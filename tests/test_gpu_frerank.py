"""Fused re-rank (bf16 shadow pre-filter + exact re-score, frerank.cuh) must return exactly what the
plain distance + top-k kernels and the oracle (reader.rs:381-399) return, also on rows built to put the bf16 rounding at its
worst, and through the filtered searches that use it."""
import numpy as np
import pytest

import arroy_b200 as ab
import oracle
from helpers import ADVERSARIAL_KINDS, adversarial_set

pytestmark = pytest.mark.gpu
SEED = bytes([42] * 32)


@pytest.fixture(scope="module")
def ctx():
    c = ab.Context(0)
    yield c
    c.close()


def _both(ctx, monkeypatch, q, qh, rows_per_query, k):
    offs = np.zeros(len(rows_per_query) + 1, dtype=np.uint64)
    offs[1:] = np.cumsum([len(r) for r in rows_per_query])
    rows = np.concatenate(rows_per_query).astype(np.uint32)
    monkeypatch.setenv("ARROY_B200_FRERANK", "0")
    plain = ctx.rerank_batch(q, qh, rows, offs, k)
    monkeypatch.setenv("ARROY_B200_FRERANK", "1")
    c0 = ctx.counters()
    fused = ctx.rerank_batch(q, qh, rows, offs, k)
    c1 = ctx.counters()
    assert c1["fused_rerank_batches"] > c0["fused_rerank_batches"]
    assert plain[2].tolist() == fused[2].tolist()
    for i in range(q.shape[0]):
        n = plain[2][i]
        assert plain[0][i, :n].tolist() == fused[0][i, :n].tolist()
        assert plain[1][i, :n].tobytes() == fused[1][i, :n].tobytes()
    return fused, c1["fused_rerank_fallbacks"] - c0["fused_rerank_fallbacks"]


@pytest.mark.parametrize("metric,d", [("euclidean", 96), ("cosine", 768), ("dot-product", 200), ("cosine", 33), ("euclidean", 20)])
def test_fused_rerank_matches_plain_kernels_and_oracle(ctx, monkeypatch, metric, d):
    n, nq, k = 20_000, 24, 100
    data = oracle.synth_rows(SEED, d, 0, n + nq, 0.5)
    ctx.stage_items_flat(metric, np.arange(n + nq, dtype=np.uint32), data)
    h0, _ = ctx.item_headers()
    q, qh = data[n:], h0[n:]
    rng = np.random.default_rng(3)
    lists = [np.sort(rng.choice(n, int(rng.integers(600, 7000)), replace=False)) for _ in range(nq)]   # ragged candidate lists
    (out_rows, out_dist, out_len), fallbacks = _both(ctx, monkeypatch, q, qh, lists, k)
    assert fallbacks == 0
    m = oracle.METRICS[metric]
    hdr = h0 if metric == "cosine" else np.zeros(n + nq, np.float32)
    for i in (0, 11, nq - 1):
        wr, wd = oracle.rerank(m, q[i], (float(qh[i]), 0.0), data, hdr, None, lists[i].astype(np.uint32), k)
        assert out_rows[i, :out_len[i]].tolist() == wr.tolist() and out_dist[i, :out_len[i]].tobytes() == wd.tobytes()
    _both(ctx, monkeypatch, q, qh, lists, 1)
    _both(ctx, monkeypatch, q, qh, [l[:700] for l in lists], 650)   # k close to the number of candidates


def test_fused_rerank_with_ties_and_degenerate_rows(ctx, monkeypatch):
    n, d, nq = 9_000, 64, 16
    rng = np.random.default_rng(5)
    base = rng.standard_normal((40, d)).astype(np.float32)
    data = base[rng.integers(0, 40, n)]           # many exactly equal candidates: ties are broken by id
    data[::7] = 0.0
    data[1::11] *= np.float32(1e18)
    data[2::13] *= np.float32(1e-18)
    data[5, 3] = np.nan
    data[77, 0] = np.inf
    q = np.concatenate([base[:8], rng.standard_normal((nq - 8, d)).astype(np.float32)])
    lists = [np.arange(0, n, 1 + (i % 3)) for i in range(nq)]
    lists = [l[:8000] for l in lists]
    for metric in ("cosine", "euclidean", "dot-product"):
        ctx.stage_items_flat(metric, np.arange(n, dtype=np.uint32), data)
        qh = np.sqrt((q.astype(np.float64) ** 2).sum(1)).astype(np.float32) if metric == "cosine" else None
        _both(ctx, monkeypatch, q, qh, lists, 50)   # too many survivors -> falls back inside, results still identical


ADV_DIMS = [20, 32, 33, 64, 96, 100, 200, 768, 1536, 4096]   # 20: d < 32; 32, 96, 200: a trailing 32-element chunk (ld % 64 == 32)


def _adversarial_matrix(kind, metric, d, n_random=2000):
    """the adversarial set of helpers.adversarial_set in rows 0 .. nc-1, then random rows no longer than its shortest row, so
    the largest norm of the staged items (gmax) is the construction's"""
    q, adv = adversarial_set(kind, metric, d, seed=d)
    rng = np.random.default_rng(d + 1)
    fill = rng.standard_normal((n_random, d))
    shortest = np.linalg.norm(adv.astype(np.float64), axis=1).min()
    fill *= rng.uniform(0.2, 0.95, (n_random, 1)) * shortest / np.linalg.norm(fill, axis=1, keepdims=True)
    return q, adv.shape[0], np.concatenate([adv, fill.astype(np.float32)])


def _cos_header(v):
    return oracle.new_header(oracle.COSINE, v)[0]


@pytest.mark.parametrize("d", ADV_DIMS)
@pytest.mark.parametrize("metric", ["euclidean", "cosine", "dot-product"])
def test_fused_rerank_on_adversarial_rows(ctx, monkeypatch, metric, d):
    # rows whose bf16 rounding errors all line up with the query (tests/test_frerank_bound_cpu.py restates the kernel's rule on
    # them): A is the true nearest row and its shadow looks farther than the k rows B. The fused kernel must keep A, with no
    # fallback, and return what the plain kernels and the oracle return; random queries share the batch.
    m = oracle.METRICS[metric]
    for kind in ADVERSARIAL_KINDS:
        q, nc, data = _adversarial_matrix(kind, metric, d)
        n = data.shape[0]
        ctx.stage_items_flat(metric, np.arange(n, dtype=np.uint32), data)
        hdr = np.array([_cos_header(r) for r in data], np.float32) if metric == "cosine" else np.zeros(n, np.float32)
        rng = np.random.default_rng(d + 2)
        rq = (rng.standard_normal((2, d)) * (np.linalg.norm(q.astype(np.float64)) / np.sqrt(d))).astype(np.float32)
        queries = np.concatenate([q[None, :], rq])
        qh = np.array([_cos_header(v) for v in queries], np.float32) if metric == "cosine" else None
        lists = [np.arange(nc)] + [np.sort(rng.choice(n, 1500, replace=False)) for _ in range(2)]
        for k in (1, 10, nc - 1):
            (rows, dist, lens), fallbacks = _both(ctx, monkeypatch, queries, qh, lists, k)
            assert fallbacks == 0, (kind, k)
            for i in range(queries.shape[0]):
                wr, wd = oracle.rerank(m, queries[i], (float(qh[i]) if qh is not None else 0.0, 0.0), data, hdr, None,
                                       lists[i].astype(np.uint32), k)
                assert rows[i, :lens[i]].tolist() == wr.tolist() and dist[i, :lens[i]].tobytes() == wd.tobytes(), (kind, k, i)


def _env(ctx):
    e = ab.Env(0)
    e._ctx = ctx
    return e


@pytest.mark.parametrize("metric,d", [("dot-product", 33), ("euclidean", 200), ("cosine", 768), ("dot-product", 768)])
def test_adversarial_rows_through_filtered_queries(ctx, monkeypatch, metric, d):
    # the same sets through QueryBuilder::candidates: a filter of exactly {A, B_1 .. B_k} (the small-filter shortcut, or a
    # walk with search_k below the filter's rows in the forest), single queries and batches (walk1_kernel, walk_kernel), one
    # shared filter and one filter per query, against the oracle's Reader
    n_trees, count = 8, 10
    q, nc, data = _adversarial_matrix("ones", metric, d)
    n = data.shape[0]
    ids = np.arange(n, dtype=np.uint32)
    odb = oracle.Db(metric, d)
    odb.set_items(ids, data)
    odb.build(oracle.StdRng(SEED), n_trees=n_trees, threads=8)
    env = _env(ctx)
    try:
        w = ab.Writer(env, 0, d, metric)
        w.add_items(ids, data)
        w.builder(ab.StdRng.from_seed(SEED)).n_trees(n_trees).build()
        r = ab.Reader.open(env, 0, metric)
        F = list(range(nc))
        rng = np.random.default_rng(4)
        G = np.sort(rng.choice(n, 40, replace=False)).tolist()
        c0 = ctx.counters()
        for sk in (None, 2**64 - 1, 30):
            got = r.nns(count).search_k(sk).candidates(F).by_vector(q) if sk else r.nns(count).candidates(F).by_vector(q)
            want = odb.nns_by_vector(q, count, search_k=sk, candidates=F)
            assert sk == 30 or want[0][0] == 0            # every row of the filter is a candidate: A comes first
            assert got == want, sk
            for nq in (3, 40):
                vecs = np.repeat(q[None, :], nq, axis=0)
                vecs[1::2] = (rng.standard_normal((nq // 2, d)) * np.abs(q).mean()).astype(np.float32)
                bi, bd, bl, _ = r.nns_batch_by_vector(vecs, count, search_k=sk, candidates=F)
                fq = np.arange(nq) % 2
                mi, md, ml, _ = r.nns_batch_by_vector(vecs, count, search_k=sk, filters=[F, G], filter_of_query=fq)
                for i in range(nq):
                    wv = odb.nns_by_vector(vecs[i], count, search_k=sk, candidates=F)
                    assert list(zip(bi[i, :bl[i]].tolist(), bd[i, :bl[i]].tolist())) == wv, (sk, nq, i)
                    wm = wv if fq[i] == 0 else odb.nns_by_vector(vecs[i], count, search_k=sk, candidates=G)
                    assert list(zip(mi[i, :ml[i]].tolist(), md[i, :ml[i]].tolist())) == wm, (sk, nq, i)
        c1 = ctx.counters()
        assert c1["fused_rerank_batches"] > c0["fused_rerank_batches"]
        assert c1["fused_rerank_fallbacks"] == c0["fused_rerank_fallbacks"]
    finally:
        env._ctx = None
