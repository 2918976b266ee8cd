"""Batched queries and re-ranks of host-placed indexes through the plane pre-filter (frerank.cuh frerank_kernel<FR_PLANES>), with
the placement forced by ARROY_B200_HOST_ITEMS=1: every result must equal the device-placed context and the oracle byte for
byte, the kernel must read fewer rows from host memory than it estimates, its survivor count must equal the CPU restatement's
(tests/test_host_rerank_bound_cpu.py), and the cases it does not take must give the same results.
To keep the file's GPU time to a few minutes, the four search paths are compared with the device placement only (which the
filtered-search, mirror and parity tests tie to the oracle), `rerank` and `rerank_batch` with both; and d = 8192 runs 256
queries per batch on 1500 rows instead of 1000 on 4000."""
import numpy as np
import pytest

import oracle
from arroy_b200 import _capi
from test_gpu_filtered_search import forest_arrays
from test_gpu_host_items import build, ctx, ld_of, query_headers, stage   # noqa: F401  (ctx: the module's context fixture)
from test_host_rerank_bound_cpu import estimates, make_set, plane_set, survivors

pytestmark = pytest.mark.gpu
SEED = bytes([42] * 32)
FLOAT_METRICS = ["euclidean", "cosine", "dot-product", "manhattan"]


def synth(metric, n, d):
    return oracle.synth_rows(SEED, d, 0, n, 0.0 if metric == "euclidean" else 0.5, threads=8)


def same(a, b):
    a = a if isinstance(a, tuple) else (a,)
    b = b if isinstance(b, tuple) else (b,)
    return all(np.asarray(x).tobytes() == np.asarray(y).tobytes() for x, y in zip(a, b))


def batched_paths(ctx, metric, data, nq, ks, rng_seed=9):
    """the batched query and re-rank paths the plane kernel serves, as (name, result) pairs"""
    n, d = data.shape
    rng = np.random.default_rng(rng_seed)
    qv = (data[rng.choice(n, nq)] + rng.standard_normal((nq, d)).astype(np.float32) * np.float32(0.1)).astype(np.float32)
    qh = query_headers(metric, qv)
    bits = _capi.row_bitmap(np.flatnonzero(rng.random(n) < 0.3), n)
    filters = [np.sort(rng.choice(n, size=s, replace=False)) for s in (5, 400, min(2000, n // 2))]
    cand = np.sort(rng.choice(n, size=800, replace=False)).astype(np.uint32)
    offs = np.arange(0, 16 * 800 + 1, 800, dtype=np.uint64)
    out = []
    for k in ks:
        out.append(("search by vector k=%d" % k, ctx.search_batch(k, queries=qv, qhdr0=qh)))
        out.append(("search by item k=%d" % k, ctx.search_batch(k, query_rows=(np.arange(nq, dtype=np.uint32) * 3) % n)))
        out.append(("filtered k=%d" % k, ctx.search_batch_filtered(k, bits, queries=qv[:64], qhdr0=qh[:64])))
        out.append(("multi-filtered k=%d" % k, ctx.search_batch_multi_filtered(k, filters, np.arange(64) % 3, queries=qv[:64], qhdr0=qh[:64])))
        out.append(("rerank k=%d" % k, ctx.rerank(qv[0], (float(qh[0]), 0.0), cand, k)))
        out.append(("rerank_batch k=%d" % k, ctx.rerank_batch(qv[:16], qh[:16], np.tile(cand, 16), offs, k)))
    return out, (qv, qh, cand)


def check_reranks_against_the_oracle(metric, data, ctx_results, qv, qh, cand):
    h0 = np.array([oracle.new_header(oracle.COSINE, v)[0] for v in data], np.float32) if metric == "cosine" else np.zeros(len(data), np.float32)
    m = oracle.METRICS[metric]
    for name, res in ctx_results:
        if name.startswith("rerank k="):
            k = int(name.split("=")[1])
            want = oracle.rerank(m, qv[0], (float(qh[0]), 0.0), data, h0, None, cand, k)
            assert same(res, want), name
        elif name.startswith("rerank_batch"):
            k = int(name.split("=")[1])
            rows, dist, lens = res
            for q in (0, 7, 15):
                wr, wd = oracle.rerank(m, qv[q], (float(qh[q]), 0.0), data, h0, None, cand, k)
                assert rows[q, :lens[q]].tobytes() == np.asarray(wr).tobytes() and dist[q, :lens[q]].tobytes() == np.asarray(wd).tobytes(), (name, q)


@pytest.mark.parametrize("d", [64, 100, 768, 1000, 8192])
@pytest.mark.parametrize("metric", FLOAT_METRICS)
def test_batched_paths_equal_device_placement_and_the_oracle(ctx, monkeypatch, metric, d):
    n, T, nq = (1500, 3, 256) if d == 8192 else (4000, 4, 1000)
    data = synth(metric, n, d)
    stage(ctx, monkeypatch, metric, data, host=False)
    nodes = build(ctx, T, split_after=64 if d > n else 0)   # (a leaf holds up to d items by default)
    ctx.load_forest(roots=np.arange(T, dtype=np.uint32), **forest_arrays(nodes, oracle.METRICS[metric], d))
    want, _ = batched_paths(ctx, metric, data, nq, (1, 10, 100))
    stage(ctx, monkeypatch, metric, data, host=True)
    ctx.load_forest(roots=np.arange(T, dtype=np.uint32), **forest_arrays(nodes, oracle.METRICS[metric], d))
    s0, c0 = ctx.plane_rerank_stats(), ctx.counters()
    got, (qv, qh, cand) = batched_paths(ctx, metric, data, nq, (1, 10, 100))
    s1, c1 = ctx.plane_rerank_stats(), ctx.counters()
    for (name, a), (_, b) in zip(got, want):
        assert same(a, b), (metric, d, name)
    check_reranks_against_the_oracle(metric, data, got, qv, qh, cand)
    assert s1["batches"] > s0["batches"], (s0, s1)
    assert s1["fallbacks"] == s0["fallbacks"], (s0, s1)
    est, resc = s1["rows_estimated"] - s0["rows_estimated"], s1["rows_rescored"] - s0["rows_rescored"]
    assert 0 < resc < est, (est, resc)
    assert c1["fused_rerank_batches"] == c0["fused_rerank_batches"]   # the bf16 kernel's counter is not touched


def test_device_placement_leaves_the_plane_counters_at_zero():
    import arroy_b200 as ab
    c = ab.Context(0)
    try:
        data = synth("cosine", 4000, 128)
        c.stage_items_flat("cosine", np.arange(4000, dtype=np.uint32), data)
        assert c.item_placement()["placement"] == "device"
        rng = np.random.default_rng(1)
        qv = data[rng.choice(4000, 16)]
        qh = query_headers("cosine", qv)
        cand = np.sort(rng.choice(4000, size=800, replace=False)).astype(np.uint32)
        c.rerank_batch(qv, qh, np.tile(cand, 16), np.arange(0, 16 * 800 + 1, 800, dtype=np.uint64), 10)
        assert c.counters()["fused_rerank_batches"] == 1
        assert c.plane_rerank_stats() == {"batches": 0, "fallbacks": 0, "rows_estimated": 0, "rows_rescored": 0}
    finally:
        c.close()


@pytest.mark.parametrize("d", [100, 768])
@pytest.mark.parametrize("metric", FLOAT_METRICS)
def test_adversarial_rows_inside_a_larger_matrix(ctx, monkeypatch, metric, d):
    rng = np.random.default_rng(d)
    base = synth(metric, 3000, d)
    kinds = ["ones", "mixed", "big", "small", "tiny", "subnormal-products", "special", "near-duplicate"]
    kinds += ["underflow-tail"] if metric == "cosine" else []
    sets = [make_set(kind, metric, d, seed=d + i) for i, kind in enumerate(kinds)]
    # the sets that a bound without its absolute terms gets wrong (test_the_bound_without_its_absolute_terms_is_caught)
    if metric == "euclidean":
        sets.append(plane_set(metric, d, mag=-74, seed=0))
    elif metric == "dot-product":
        sets.append(plane_set(metric, d, mag=-80, qmag=-72, seed=2))
    data, queries, cands, at = base.copy(), [], [], 0
    for q, rows in sets:
        data[at:at + len(rows)] = rows
        extra = rng.choice(np.arange(200, 3000), size=600, replace=False)
        cands.append(np.sort(np.concatenate([np.arange(at, at + len(rows)), extra])).astype(np.uint32))
        queries.append(q)
        at += len(rows)
    qv = np.stack(queries).astype(np.float32)
    qh = query_headers(metric, qv)
    offs = np.concatenate([[0], np.cumsum([len(c) for c in cands])]).astype(np.uint64)
    rows = np.concatenate(cands)
    results = []
    for host in (False, True):
        stage(ctx, monkeypatch, metric, data, host=host)
        s0 = ctx.plane_rerank_stats()
        results.append([ctx.rerank_batch(qv, qh, rows, offs, k) for k in (1, 10)])
        s1 = ctx.plane_rerank_stats()
    assert s1["batches"] - s0["batches"] == 2 and s1["fallbacks"] == s0["fallbacks"], (s0, s1)
    for a, b in zip(*results):
        assert same(a, b), (metric, d)
    h0 = ctx.item_headers()[0] if metric == "cosine" else np.zeros(len(data), np.float32)
    m = oracle.METRICS[metric]
    for ki, k in enumerate((1, 10)):
        r, dist, lens = results[1][ki]
        for q in range(len(qv)):
            wr, wd = oracle.rerank(m, qv[q], (float(qh[q]), 0.0), data, h0, None, cands[q], k)
            assert r[q, :lens[q]].tobytes() == np.asarray(wr).tobytes() and dist[q, :lens[q]].tobytes() == np.asarray(wd).tobytes(), (metric, d, k, q)


@pytest.mark.parametrize("metric", FLOAT_METRICS)
def test_survivor_count_equals_the_restatement(ctx, monkeypatch, metric):
    n, d, nq, nc, k = 4000, 100, 8, 1000, 10
    data = synth(metric, n, d)
    stage(ctx, monkeypatch, metric, data, host=True)
    hi, lo, sc = ctx.prefilter_planes(n, ld_of(d))
    ch = ctx.item_headers()[0] if metric == "cosine" else np.zeros(n, np.float32)
    rng = np.random.default_rng(5)
    qv = (data[rng.choice(n, nq)] + rng.standard_normal((nq, d)).astype(np.float32) * np.float32(0.1)).astype(np.float32)
    qh = query_headers(metric, qv)
    cands = [np.sort(rng.choice(n, size=nc, replace=False)).astype(np.uint32) for _ in range(nq)]
    want = 0
    for q in range(nq):
        c = cands[q]
        a, E = estimates(metric, qv[q], qh[q], hi[c], lo[c], sc[c], ch[c])
        want += int(survivors(a, E, k).sum())
    s0 = ctx.plane_rerank_stats()
    ctx.rerank_batch(qv, qh, np.concatenate(cands), np.arange(0, nq * nc + 1, nc, dtype=np.uint64), k)
    s1 = ctx.plane_rerank_stats()
    assert s1["batches"] - s0["batches"] == 1 and s1["fallbacks"] == s0["fallbacks"]
    assert s1["rows_estimated"] - s0["rows_estimated"] == nq * nc
    assert s1["rows_rescored"] - s0["rows_rescored"] == want, (s1["rows_rescored"] - s0["rows_rescored"], want)


def test_cases_the_plane_kernel_does_not_take(ctx, monkeypatch):
    n, d = 12000, 64
    data = synth("cosine", n, d)
    rng = np.random.default_rng(2)
    qv = data[rng.choice(n, 4)]
    qh = query_headers("cosine", qv)
    big = np.sort(rng.choice(n, size=9000, replace=False)).astype(np.uint32)   # more than FR_CAP = 8192 candidates
    mid = np.sort(rng.choice(n, size=4000, replace=False)).astype(np.uint32)
    cases = [("over FR_CAP", np.tile(big, 4), np.arange(0, 4 * 9000 + 1, 9000, dtype=np.uint64), 10, None),
             ("k over FR_SURV", np.tile(mid, 4), np.arange(0, 4 * 4000 + 1, 4000, dtype=np.uint64), 2100, None),
             ("FRERANK=0", np.tile(mid, 4), np.arange(0, 4 * 4000 + 1, 4000, dtype=np.uint64), 10, "0")]
    results = []
    for host in (False, True):
        stage(ctx, monkeypatch, "cosine", data, host=host)
        out = []
        for name, rows, offs, k, env in cases:
            if env is not None:
                monkeypatch.setenv("ARROY_B200_FRERANK", env)
            s0 = ctx.plane_rerank_stats()
            out.append(ctx.rerank_batch(qv, qh, rows, offs, k))
            s1 = ctx.plane_rerank_stats()
            monkeypatch.delenv("ARROY_B200_FRERANK", raising=False)
            assert s1 == s0, (name, host, s0, s1)   # not taken
        results.append(out)
    for (name, *_), a, b in zip(cases, *results):
        assert same(a, b), name
    # a query with more than FR_CAP candidates inside a batch the host sends to the kernel: the batch falls back
    stage(ctx, monkeypatch, "cosine", data, host=True)
    qv2 = data[rng.choice(n, 32)]
    qh2 = query_headers("cosine", qv2)
    # rerank_batch sends a batch to the kernel only when every query fits; a walk's batch is sent as it is, so a large search_k
    # reaches the kernel's status path
    nodes = build(ctx, 2)
    ctx.load_forest(roots=np.arange(2, dtype=np.uint32), **forest_arrays(nodes, oracle.COSINE, d))
    s0 = ctx.plane_rerank_stats()
    got = ctx.search_batch(10, queries=qv2, qhdr0=qh2, search_k=11000)
    s1 = ctx.plane_rerank_stats()
    assert s1["batches"] - s0["batches"] == 1 and s1["fallbacks"] - s0["fallbacks"] == 1, (s0, s1)
    stage(ctx, monkeypatch, "cosine", data, host=False)
    ctx.load_forest(roots=np.arange(2, dtype=np.uint32), **forest_arrays(nodes, oracle.COSINE, d))
    assert same(got, ctx.search_batch(10, queries=qv2, qhdr0=qh2, search_k=11000))
