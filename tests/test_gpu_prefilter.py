"""rerank_shared: the tensor-core pre-filter + exact re-score must return exactly what the exact
dense kernel (and the oracle, reader.rs:381-399) returns."""
import os

import numpy as np
import pytest

import arroy_b200 as ab
import oracle

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
def test_tensor_core_scores_are_within_the_bound(ctx, monkeypatch, d, nq, nc):
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
        for mc in ("1", "2"):
            monkeypatch.setenv("ARROY_B200_XGEMM_MC", mc)
            own = ctx.prefilter_scores(q, rows, engine=0)
            assert np.all(np.abs(own - exact) <= bound), (mc, float(np.max(np.abs(own - exact) / bound)))
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
