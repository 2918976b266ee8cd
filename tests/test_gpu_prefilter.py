"""rerank_shared: the tensor-core pre-filter + exact re-score must return exactly what the exact
dense kernel (and the oracle, reader.rs:381-399) returns."""
import os

import numpy as np
import pytest

import arroy_b200 as ab
import oracle
from helpers import adversarial_set

pytestmark = pytest.mark.gpu
SEED = bytes([42] * 32)
CUBLAS = bool(os.environ.get("ARROY_TEST_CUBLAS"))   # engine 1 is only a cross-check of the hand-written kernel


@pytest.fixture(scope="module")
def ctx():
    c = ab.Context(0)
    yield c
    c.close()


def _both(ctx, monkeypatch, q, qh, rows, k):
    monkeypatch.setenv("ARROY_B200_XRERANK", "exact")
    exact = ctx.rerank_shared(q, qh, rows, k)
    before = ctx.rerank_stats()
    monkeypatch.setenv("ARROY_B200_XRERANK", "filter")
    filt = ctx.rerank_shared(q, qh, rows, k)
    after = ctx.rerank_stats()
    assert after["prefilter_chunks"] > before["prefilter_chunks"]
    assert exact[2].tolist() == filt[2].tolist()
    for i in range(q.shape[0]):
        n = exact[2][i]
        assert exact[0][i, :n].tolist() == filt[0][i, :n].tolist()
        assert exact[1][i, :n].tobytes() == filt[1][i, :n].tobytes()
    return filt, {k_: after[k_] - before[k_] for k_ in after}


@pytest.mark.parametrize("metric,d", [("euclidean", 96), ("cosine", 768), ("dot-product", 200), ("cosine", 33)])
def test_prefilter_matches_exact_kernel_and_oracle(ctx, monkeypatch, metric, d):
    n, nq, k = 30_000, 48, 100
    data = oracle.synth_rows(SEED, d, 0, n + nq, 0.5)
    ctx.stage_items_flat(metric, np.arange(n + nq, dtype=np.uint32), data)
    h0, _ = ctx.item_headers()
    q = data[n:]
    qh = h0[n:]
    rows = np.arange(0, n, dtype=np.uint32)                     # contiguous: GEMM reads the item matrix in place
    (out_rows, out_dist, out_len), st = _both(ctx, monkeypatch, q, qh, rows, k)
    assert st["fallback_chunks"] == 0 and st["survivors"] < 0.2 * n * nq
    m = oracle.METRICS[metric]
    hdr = h0 if metric == "cosine" else np.zeros(n + nq, np.float32)
    for i in (0, 17, nq - 1):
        wr, wd = oracle.rerank(m, q[i], (float(qh[i]), 0.0), data, hdr, None, rows, k)
        assert out_rows[i, :out_len[i]].tolist() == wr.tolist() and out_dist[i, :out_len[i]].tobytes() == wd.tobytes()
    scattered = np.arange(1, n, 3, dtype=np.uint32)             # not contiguous: gathered candidate matrix
    _both(ctx, monkeypatch, q, qh, scattered, 10)


def test_prefilter_with_ties_duplicates_and_degenerate_rows(ctx, monkeypatch):
    # many exactly equal candidates (ties broken by id), zero vectors (cosine: distance 0 via the
    # norm test), huge and tiny magnitudes; more ties than the per-query cap forces the fallback
    n, d, nq = 12_000, 64, 40
    rng = np.random.default_rng(5)
    base = rng.standard_normal((50, d)).astype(np.float32)
    data = base[rng.integers(0, 50, n)]
    data[::7] = 0.0
    data[1::11] *= np.float32(1e18)
    data[2::13] *= np.float32(1e-18)
    q = np.concatenate([base[:20], rng.standard_normal((nq - 20, d)).astype(np.float32)])
    for metric in ("cosine", "euclidean", "dot-product"):
        ctx.stage_items_flat(metric, np.arange(n, dtype=np.uint32), data)
        if metric == "cosine":
            qh = np.sqrt((q.astype(np.float64) ** 2).sum(1)).astype(np.float32)
        else:
            qh = None
        rows = np.arange(n, dtype=np.uint32)
        _, st = _both(ctx, monkeypatch, q, qh, rows, 100)
        _both(ctx, monkeypatch, q, qh, rows, 1)


def test_prefilter_nan_and_inf_inputs(ctx, monkeypatch):
    n, d, nq = 8_000, 48, 36
    rng = np.random.default_rng(9)
    data = rng.standard_normal((n, d)).astype(np.float32)
    data[5, 3] = np.nan
    data[77, 0] = np.inf
    data[78, 1] = -np.inf
    q = rng.standard_normal((nq, d)).astype(np.float32)
    q[3, 2] = np.nan
    for metric in ("euclidean", "dot-product"):
        ctx.stage_items_flat(metric, np.arange(n, dtype=np.uint32), data)
        _both(ctx, monkeypatch, q, None, np.arange(n, dtype=np.uint32), 20)


@pytest.mark.parametrize("d,nq,nc", [(768, 300, 5001), (33, 7, 258), (100, 129, 1000), (64, 1, 40)])
def test_tensor_core_scores_are_within_the_bound(ctx, d, nq, nc):
    # the bound the whole pre-filter rests on: |S - q.c| <= 2^-8 |q| |c|, for the hand-written wgmma
    # kernel (engine 0, single-CTA and 2-CTA multicast variants) and optionally for cuBLAS (engine 1); ragged tile
    # edges in both directions
    n = nc + 50
    data = oracle.synth_rows(SEED, d, 0, n + nq, 0.5)
    data[3] *= np.float32(1e10)
    data[4] *= np.float32(1e-10)
    ctx.stage_items_flat("euclidean", np.arange(n + nq, dtype=np.uint32), data)
    q = data[n:]
    for rows in (np.arange(10, 10 + nc, dtype=np.uint32), np.sort(np.random.default_rng(1).choice(n, nc, replace=False)).astype(np.uint32)):
        exact = q.astype(np.float64) @ data[rows].astype(np.float64).T
        bound = np.linalg.norm(q.astype(np.float64), axis=1)[:, None] * np.linalg.norm(data[rows].astype(np.float64), axis=1)[None, :] / 256.0
        own = ctx.prefilter_scores(q, rows, engine=0)
        assert np.all(np.abs(own - exact) <= bound), float(np.max(np.abs(own - exact) / bound))
        if CUBLAS:
            lib = ctx.prefilter_scores(q, rows, engine=1)
            assert np.all(np.abs(lib - exact) <= bound)
        # far tighter in practice: the truncation errors are not all aligned
        assert float(np.max(np.abs(own - exact) / bound)) < 0.25


@pytest.mark.skipif(not CUBLAS, reason="cuBLAS cross-check engine: set ARROY_TEST_CUBLAS=1 (loading libcublasLt on a fresh box takes minutes)")
def test_prefilter_engines_agree(ctx, monkeypatch):
    n, d, nq, k = 20_000, 128, 130, 50
    data = oracle.synth_rows(SEED, d, 0, n + nq, 0.5)
    ctx.stage_items_flat("cosine", np.arange(n + nq, dtype=np.uint32), data)
    h0, _ = ctx.item_headers()
    rows = np.arange(n, dtype=np.uint32)
    monkeypatch.setenv("ARROY_B200_XRERANK", "filter")
    monkeypatch.setenv("ARROY_B200_XGEMM", "cublas")
    a = ctx.rerank_shared(data[n:], h0[n:], rows, k)
    monkeypatch.setenv("ARROY_B200_XGEMM", "wgmma")
    b = ctx.rerank_shared(data[n:], h0[n:], rows, k)
    assert a[0].tolist() == b[0].tolist() and a[1].tobytes() == b[1].tobytes()


def _tf32_rows(signs, exps, low):
    """sign * 2^e with the low 13 mantissa bits set to `low` (0x0FFF: just below the TF32 midpoint 1 + 2^-11, lost by rounding
    and by truncation alike; 0x1FFF: almost 2^-10 lost by truncation, almost nothing by rounding)"""
    bits = ((127 + exps.astype(np.int64)) << 23) | low
    return (signs * bits.astype(np.uint32).view(np.float32)).astype(np.float32)


def test_tensor_core_scores_at_worst_case_rounding(ctx, capsys):
    # both operands just below a TF32 midpoint, with the rows' signs taken from the query: every element of the pair loses
    # 2^-11 of itself in the same direction, ~2^-10 |q| |c| in all, a quarter of the bound 2^-8 |q| |c|. The truncation pattern
    # reports which conversion wgmma does: ~0.5 of the bound if it truncates, ~0 if it rounds.
    rng = np.random.default_rng(21)
    for d in (33, 100, 768):
        nq = 16
        signs = rng.choice([-1.0, 1.0], (nq, d))
        exps = np.where(np.arange(nq)[:, None] % 4 < 2, 0, rng.integers(-8, 9, (nq, d)))     # all ones, or mixed exponents
        low = np.where(np.arange(nq) < nq // 2, 0x0FFF, 0x1FFF)[:, None]
        q = _tf32_rows(signs, exps, low)
        rows_v = np.concatenate([_tf32_rows(signs, exps, low), rng.standard_normal((200, d)).astype(np.float32)])   # row j = query j
        n = rows_v.shape[0]
        ctx.stage_items_flat("euclidean", np.arange(n, dtype=np.uint32), rows_v)
        rows = np.arange(n, dtype=np.uint32)
        exact = q.astype(np.float64) @ rows_v.astype(np.float64).T
        bound = np.linalg.norm(q.astype(np.float64), axis=1)[:, None] * np.linalg.norm(rows_v.astype(np.float64), axis=1)[None, :] / 256.0
        own = ctx.prefilter_scores(q, rows, engine=0)
        ratio = np.abs(own - exact) / bound
        assert np.all(ratio <= 1.0), (d, float(ratio.max()))
        matched = ratio[np.arange(nq), np.arange(nq)]                  # query j against its own row j
        assert matched[: nq // 2].min() >= 0.2, (d, matched[: nq // 2])
        with capsys.disabled():
            print("\nTF32 scores d=%d: midpoint rows %.3f of the bound, all-ones low bits %.3f (0.5: truncation, ~0: rounding)"
                  % (d, float(matched[: nq // 2].min()), float(matched[nq // 2:].max())))


def _tf32_matrix(kind, metric, d, n_random=800):   # fewer candidates than the 1024 survivors a query may keep
    q, adv = adversarial_set(kind, metric, d, shift=13, delta=1, seed=d)
    rng = np.random.default_rng(d + 5)
    fill = rng.standard_normal((n_random, d))
    shortest = np.linalg.norm(adv.astype(np.float64), axis=1).min()
    fill *= rng.uniform(0.2, 0.95, (n_random, 1)) * shortest / np.linalg.norm(fill, axis=1, keepdims=True)
    return q, adv.shape[0], np.concatenate([adv, fill.astype(np.float32)])


@pytest.mark.parametrize("d", [33, 100, 768])
@pytest.mark.parametrize("metric", ["euclidean", "cosine", "dot-product"])
def test_prefilter_on_adversarial_rows(ctx, monkeypatch, metric, d):
    # the bf16 A / B construction rebuilt at TF32's midpoints (rows 0 .. nc-1 of the candidates), plus candidate sets of rows
    # whose f32 squared norm underflows and of subnormal rows: exact = filter = oracle. The bound has about 2x slack over
    # TF32's rounding, so A must survive.
    m = oracle.METRICS[metric]
    for kind in ("ones", "signs", "mixed", "near-duplicate", "underflow", "subnormal", "tiny-normal", "underflow-tail"):
        q, nc, data = _tf32_matrix(kind, metric, d)
        n = data.shape[0]
        ctx.stage_items_flat(metric, np.arange(n, dtype=np.uint32), data)
        hdr = np.array([oracle.new_header(oracle.COSINE, r)[0] for r in data], np.float32) if metric == "cosine" else np.zeros(n, np.float32)
        rng = np.random.default_rng(d)
        queries = np.concatenate([np.repeat(q[None, :], 8, axis=0), (rng.standard_normal((24, d)) * np.abs(q).max()).astype(np.float32)])
        qh = np.array([oracle.new_header(oracle.COSINE, v)[0] for v in queries], np.float32) if metric == "cosine" else None
        rows = np.arange(n, dtype=np.uint32)
        for k in (1, 10):
            (out_rows, out_dist, out_len), st = _both(ctx, monkeypatch, queries, qh, rows, k)
            assert st["fallback_chunks"] == 0, (kind, k)
            for i in (0, 8, 31):
                wr, wd = oracle.rerank(m, queries[i], (float(qh[i]) if qh is not None else 0.0, 0.0), data, hdr, None, rows, k)
                assert out_rows[i, :out_len[i]].tolist() == wr.tolist() and out_dist[i, :out_len[i]].tobytes() == wd.tobytes(), (kind, k, i)


def test_tensor_core_scores_of_tiny_rows(ctx, capsys):
    # subnormal rows and rows whose squared norm underflows, against a large query: the scores must stay within the bound the
    # pre-filter charges, 2^-8 (|q| + sub) (|c| + sub) + 1e-30 with sub = sqrt(d + 64) 2^-74 (xf_query_prep_kernel), whether
    # the conversion keeps subnormal operands or flushes them (reported)
    for d in (33, 768):
        q, adv = adversarial_set("subnormal", "dot-product", d, shift=13, delta=1, seed=d)
        _, und = adversarial_set("underflow", "dot-product", d, shift=13, delta=1, seed=d)
        rows_v = np.concatenate([adv, und])
        n = rows_v.shape[0]
        ctx.stage_items_flat("dot-product", np.arange(n, dtype=np.uint32), rows_v)
        queries = np.stack([q, -q, np.abs(q)])
        exact = queries.astype(np.float64) @ rows_v.astype(np.float64).T
        sub = np.sqrt(d + 64.0) * 2.0 ** -74
        qn = np.linalg.norm(queries.astype(np.float64), axis=1)[:, None]
        cn = np.linalg.norm(rows_v.astype(np.float64), axis=1)[None, :]
        bound = (2.0 ** -8 + d * 2.0 ** -22) * (qn + sub) * (cn + sub) + 1e-30
        own = ctx.prefilter_scores(queries, np.arange(n, dtype=np.uint32), engine=0)
        assert np.all(np.abs(own - exact) <= bound), d
        rel = np.abs(own[:, :adv.shape[0]] - exact[:, :adv.shape[0]]) / np.abs(exact[:, :adv.shape[0]])
        with capsys.disabled():
            print("\nTF32 scores of subnormal rows d=%d: relative error up to %.3g (1: flushed to zero)" % (d, float(rel.max())))
