"""Indexes whose f32 rows live in mapped pinned host memory (host placement, arroy_b200_item_placement_plan), forced on small
data with ARROY_B200_HOST_ITEMS=1. The device then holds the 8-bit planes written at staging time; builds scan through them and
read only the rows they cannot decide (and the two_means gathers) over PCIe, routing goes through them too, and queries read the
host rows. Everything here must equal the oracle and the device-placed context byte for byte."""
import ctypes as C
import os

import numpy as np
import pytest
import torch

import arroy_b200 as ab
import oracle
from arroy_b200 import _capi
from test_gpu_filtered_search import forest_arrays

pytestmark = pytest.mark.gpu
SEED = bytes([42] * 32)
THREADS = min(os.cpu_count() or 4, 32)
FLOAT_METRICS = ["euclidean", "cosine", "dot-product", "manhattan"]
PERSISTENT, LOCKSTEP, ASYNC, CLUSTER8, CLUSTER16, GLOBAL_WS, SPECULATIVE = 1, 2, 4, 8, 16, 32, 64


@pytest.fixture(scope="module")
def ctx():
    c = ab.Context(0)
    yield c
    c.close()


def tree_seeds(user_seed, T):
    r1 = oracle.StdRng(oracle.StdRng(user_seed).gen_seed())
    return [r1.gen_seed() for _ in range(T)]


def ld_of(d):
    return (d + 31) // 32 * 32


def stage(ctx, monkeypatch, metric, data, host, hdr0=None):
    """stage_items_flat with the placement forced to host (or left to the plan, which keeps small data on the device)"""
    if host:
        monkeypatch.setenv("ARROY_B200_HOST_ITEMS", "1")
    else:
        monkeypatch.delenv("ARROY_B200_HOST_ITEMS", raising=False)
    n, d = data.shape
    ctx.stage_items_flat(metric, np.arange(n, dtype=np.uint32), data, hdr0)
    monkeypatch.delenv("ARROY_B200_HOST_ITEMS", raising=False)
    pl = ctx.item_placement()
    if host:
        assert pl["placement"] == "host", pl
        assert pl["device_bytes"] == 2 * n * ld_of(d) + 4 * n, pl     # both planes and the scales, nothing else
        assert 4 * n * ld_of(d) <= pl["host_bytes"] <= 8 * n * ld_of(d), pl   # (a buffer at most twice the size is reused)
    else:
        assert pl["placement"] == "device" and pl["host_bytes"] == 0, pl
    if metric == "dot-product":
        return ctx.dot_preprocess()
    return None


def build(ctx, T, split_after=0, user_seed=SEED):
    return ctx.build_trees(tree_seeds(user_seed, T), list(range(T)), T, split_after)


def assert_same_forest(got, want, what):
    bad = [k for k in sorted(set(got) | set(want)) if got.get(k) != want.get(k)]
    assert not bad, "%s: %d node ids differ (%d vs %d nodes), first id %d" % (what, len(bad), len(got), len(want), bad[0])


def oracle_nodes(metric, data, T, split_after=0, user_seed=SEED):
    odb = oracle.Db(metric, data.shape[1])
    odb.set_items(np.arange(data.shape[0], dtype=np.uint32), data)
    odb.build(oracle.StdRng(user_seed), n_trees=T, split_after=split_after, threads=min(T, THREADS))
    return odb


def assert_all_scans_through_planes(ctx):
    st, pre = ctx.build_stats(), ctx.build_prefilter_stats()
    assert pre["rows_via_prefilter"] == st["scanned_rows"] > 0, (pre, st)
    assert pre["rows_in_fused_root_pass"] == 0 and pre["fused_root_rows_read"] == 0, pre
    return pre


# ---- forests ------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("T", [3, 40])
@pytest.mark.parametrize("d", [64, 768, 1000])
@pytest.mark.parametrize("metric", FLOAT_METRICS)
def test_forest_matches_the_oracle_and_device_placement(ctx, monkeypatch, metric, d, T):
    n = 6000 if d == 64 else 3000
    data = oracle.synth_rows(SEED, d, 0, n, 0.0 if metric == "euclidean" else 0.5, threads=THREADS)
    hdr_dev = stage(ctx, monkeypatch, metric, data, host=False)
    want_dev = build(ctx, T)
    st_dev = ctx.build_stats()
    hdr_host = stage(ctx, monkeypatch, metric, data, host=True)
    if metric == "dot-product":   # DotProduct::preprocess reads the host rows
        assert hdr_host[0].tobytes() == hdr_dev[0].tobytes() and hdr_host[1].tobytes() == hdr_dev[1].tobytes()
    got = build(ctx, T)
    assert_all_scans_through_planes(ctx)
    assert ctx.build_stats()["scanned_rows"] == st_dev["scanned_rows"]
    assert_same_forest(got, want_dev, (metric, d, T, "device placement"))
    odb = oracle_nodes(metric, data, T)
    assert_same_forest(got, odb.nodes(), (metric, d, T, "oracle"))
    assert ctx.build_stats()["scanned_rows"] == odb.scanned_rows


# ---- schedules ----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("case", ["lockstep", "async-3000", "async-8192"])
def test_schedules_match_the_oracle(ctx, monkeypatch, case):
    metric = "cosine"
    if case == "lockstep":
        n, d, T, want = 6000, 128, 8, LOCKSTEP | SPECULATIVE
        monkeypatch.setenv("ARROY_B200_LOCKSTEP", "1")
    elif case == "async-3000":
        n, d, T, want = 3000, 3000, 3, ASYNC
    else:
        n, d, T, want = 2000, 8192, 3, ASYNC | GLOBAL_WS
    data = oracle.synth_rows(SEED, d, 0, n, 0.5, threads=THREADS)
    stage(ctx, monkeypatch, metric, data, host=True)
    got = build(ctx, T, split_after=64)
    sched = int(ctx.build_breakdown()["schedules"])
    monkeypatch.delenv("ARROY_B200_LOCKSTEP", raising=False)
    assert sched == want, (sched, want)
    assert_all_scans_through_planes(ctx)
    odb = oracle_nodes(metric, data, T, split_after=64)
    assert_same_forest(got, odb.nodes(), case)
    assert ctx.build_stats()["scanned_rows"] == odb.scanned_rows


def test_few_small_trees_take_no_cluster_kernel(ctx, monkeypatch):
    # d <= 256 with <= 8 trees runs the async schedule's 16-CTA cluster on the device; its small-node scans read f32 rows, so a
    # host-placed index keeps one control CTA per tree
    n, d, T = 20_000, 128, 4
    data = oracle.synth_rows(SEED, d, 0, n, 0.0, threads=THREADS)
    monkeypatch.setenv("ARROY_B200_MAX_WAVE", "4")
    stage(ctx, monkeypatch, "euclidean", data, host=True)
    got = build(ctx, T)
    sched = int(ctx.build_breakdown()["schedules"])
    assert not sched & (CLUSTER8 | CLUSTER16), sched
    assert_all_scans_through_planes(ctx)
    assert_same_forest(got, oracle_nodes("euclidean", data, T).nodes(), "few trees")


# ---- hard data: stage 3 reads host rows ---------------------------------------------------------------------------------
@pytest.mark.parametrize("metric", ["euclidean", "cosine"])
def test_tiny_rows_rescore_from_host_memory(ctx, monkeypatch, metric):
    n, d, T = 20_000, 128, 8
    data = (oracle.synth_rows(SEED, d, 0, n, 0.5, threads=THREADS).astype(np.float64) * 2.0 ** -80).astype(np.float32)
    stage(ctx, monkeypatch, metric, data, host=True)
    got = build(ctx, T)
    pre = assert_all_scans_through_planes(ctx)
    assert pre["rows_rescored_f32"] > 0, pre
    odb = oracle_nodes(metric, data, T)
    assert_same_forest(got, odb.nodes(), ("tiny", metric))
    assert ctx.build_stats()["scanned_rows"] == odb.scanned_rows
    assert ctx.build_stats()["random_splits"] > 0


# ---- routing: side_multi through the planes -------------------------------------------------------------------------------
@pytest.mark.parametrize("metric", FLOAT_METRICS)
def test_side_multi_equals_side_batch(ctx, monkeypatch, metric):
    n, d, n_jobs = 5000, 96, 40
    data = oracle.synth_rows(SEED, d, 0, n, 0.0 if metric == "euclidean" else 0.5, threads=THREADS)
    stage(ctx, monkeypatch, metric, data, host=True)
    rng = np.random.default_rng(3)
    normals = rng.standard_normal((n_jobs, d)).astype(np.float32)
    normals[1] *= 2.0 ** -80                      # rows the planes cannot decide
    normals[2] = 0.0
    h0 = rng.standard_normal(n_jobs).astype(np.float32)
    lists = [np.sort(rng.choice(n, size=int(rng.integers(0, 3000)), replace=False)).astype(np.uint32) for _ in range(n_jobs)]
    rows = np.concatenate(lists)
    offs = np.concatenate([[0], np.cumsum([len(x) for x in lists])]).astype(np.uint64)
    out = np.empty(rows.size, dtype=np.uint8)
    lib = ctx.lib
    ctx._ck(lib.arroy_b200_side_multi(ctx.h, n_jobs, normals.ctypes.data_as(_capi._f32p), h0.ctypes.data_as(_capi._f32p), None,
                                      rows.ctypes.data_as(_capi._u32p), offs.ctypes.data_as(_capi._u64p), out.ctypes.data_as(_capi._u8p)))
    for j in range(n_jobs):
        if len(lists[j]) == 0:
            continue
        want, _ = ctx.side_batch(normals[j], (float(h0[j]), 0.0), lists[j])
        assert out[offs[j]:offs[j + 1]].tobytes() == want.tobytes(), j


# ---- the host mirror -------------------------------------------------------------------------------------------------------
def make_env(ctx):
    e = ab.Env(0)
    e._ctx = ctx
    return e


@pytest.mark.parametrize("metric,d,n_trees", [("cosine", 96, 4), ("euclidean", 64, 3), ("dot-product", 80, 3), ("manhattan", 70, 2)])
def test_mirror_updates_and_queries_match_the_oracle(ctx, monkeypatch, metric, d, n_trees):
    monkeypatch.setenv("ARROY_B200_HOST_ITEMS", "1")
    n0 = 3000
    data = oracle.synth_rows(SEED, d, 0, n0 + 2000, 0.5, threads=4)
    env = make_env(ctx)
    w = ab.Writer(env, 0, d, metric)
    odb = oracle.Db(metric, d)
    prng, orng = ab.StdRng.from_seed(SEED), oracle.StdRng(SEED)
    r = np.random.default_rng(5)
    for i in range(n0):
        w.add_item(i, data[i]); odb.add_item(i, data[i])
    live = set(range(n0))
    next_new = n0
    for rnd in range(3):
        w.builder(prng).n_trees(n_trees).build()
        odb.build_incremental(orng, n_trees=n_trees)
        assert env.tree_nodes() == odb.nodes(), (metric, rnd)
        assert ctx.item_placement()["placement"] == "host"
        if rnd:
            assert ctx.stage_stats()["delta"] == 0   # a host-placed index stages in full
        for i in r.choice(sorted(live), size=150, replace=False):
            w.del_item(int(i)); odb.del_item(int(i)); live.discard(int(i))
        for i in r.choice(sorted(live), size=100, replace=False):
            v = data[int(r.integers(0, len(data)))] * np.float32(0.5)
            w.add_item(int(i), v); odb.add_item(int(i), v)
        for _ in range(int(r.integers(50, 700))):
            w.add_item(next_new, data[next_new % len(data)]); odb.add_item(next_new, data[next_new % len(data)])
            live.add(next_new); next_new += 1
    w.builder(prng).n_trees(n_trees + 2).build()
    odb.build_incremental(orng, n_trees=n_trees + 2)
    assert env.tree_nodes() == odb.nodes()
    assert ctx.stage_stats()["delta"] == 0
    rd = ab.Reader.open(env, 0, metric)
    for it in sorted(live)[:40]:
        want = odb.nns_by_item(it, 10)
        got = rd.nns(10).by_item(it)
        assert [g[0] for g in got] == [x[0] for x in want]
    env._ctx = None


@pytest.mark.parametrize("metric,n,d,trees,pages", [("euclidean", 3000, 64, 3, 24), ("cosine", 2500, 100, 2, 40)])
def test_mirror_memory_limited_build_matches_the_oracle(ctx, monkeypatch, metric, n, d, trees, pages):
    monkeypatch.setenv("ARROY_B200_HOST_ITEMS", "1")
    data = oracle.synth_rows(SEED, d, 0, n, 0.5, threads=4)
    ids = np.arange(0, 2 * n, 2, dtype=np.uint32)   # sparse ids: rows != ids
    odb = oracle.Db(metric, d)
    odb.set_items(ids, data)
    odb.build_memory_limited(oracle.StdRng(SEED), n_trees=trees, available_memory=pages * 4096)
    env = make_env(ctx)
    w = ab.Writer(env, 0, d, metric)
    w.add_items(ids, data)
    w.builder(ab.StdRng.from_seed(SEED)).available_memory(pages * 4096).n_trees(trees).build()
    assert ctx.item_placement()["placement"] == "host"
    assert env.tree_nodes() == odb.nodes()
    env._ctx = None


# ---- queries and re-ranks -----------------------------------------------------------------------------------------------------
def query_headers(metric, vecs):
    if metric == "cosine":
        return np.array([oracle.new_header(oracle.COSINE, v)[0] for v in vecs], dtype=np.float32)
    return np.zeros(len(vecs), dtype=np.float32)


def run_queries(ctx, monkeypatch, metric, data, nodes, T):
    """every query path, as (name, arrays) pairs to compare byte for byte"""
    n, d = data.shape
    out = []
    ctx.load_forest(roots=np.arange(T, dtype=np.uint32), **forest_arrays(nodes, oracle.METRICS[metric], d))
    rng = np.random.default_rng(9)
    qv = (data[rng.choice(n, 1000)] + rng.standard_normal((1000, d)).astype(np.float32) * np.float32(0.1)).astype(np.float32)
    qh = query_headers(metric, qv)
    for nq in (1, 1000):
        out.append(("search nq=%d by vector" % nq, ctx.search_batch(10, queries=qv[:nq], qhdr0=qh[:nq])))
        out.append(("search nq=%d by item" % nq, ctx.search_batch(10, query_rows=np.arange(nq, dtype=np.uint32) * 3)))
    bits = _capi.row_bitmap(np.flatnonzero(rng.random(n) < 0.3), n)
    out.append(("filtered", ctx.search_batch_filtered(10, bits, queries=qv[:64], qhdr0=qh[:64])))
    filters = [np.sort(rng.choice(n, size=s, replace=False)) for s in (5, 400, 2000)]
    out.append(("multi-filtered", ctx.search_batch_multi_filtered(10, filters, np.arange(64) % 3, queries=qv[:64], qhdr0=qh[:64])))
    cand = np.sort(rng.choice(n, size=800, replace=False)).astype(np.uint32)
    out.append(("rerank", ctx.rerank(qv[0], (float(qh[0]), 0.0), cand, 20)))
    offs = np.arange(0, 16 * 800 + 1, 800, dtype=np.uint64)
    out.append(("rerank_batch", ctx.rerank_batch(qv[:16], qh[:16], np.tile(cand, 16), offs, 20)))
    contiguous = np.arange(100, 100 + 2048, dtype=np.uint32)
    scattered = np.sort(rng.choice(n, size=2048, replace=False)).astype(np.uint32)
    for mode in ("filter", "exact"):
        monkeypatch.setenv("ARROY_B200_XRERANK", mode)
        for name, rows in (("contiguous", contiguous), ("scattered", scattered)):
            out.append(("rerank_shared %s %s" % (mode, name), ctx.rerank_shared(qv[:256], qh[:256], rows, 50)))
    monkeypatch.delenv("ARROY_B200_XRERANK", raising=False)
    return out


@pytest.mark.parametrize("metric", FLOAT_METRICS)
def test_queries_equal_device_placement(ctx, monkeypatch, metric):
    n, d, T = 8000, 192, 6
    data = oracle.synth_rows(SEED, d, 0, n, 0.0 if metric == "euclidean" else 0.5, threads=THREADS)
    stage(ctx, monkeypatch, metric, data, host=False)
    nodes = build(ctx, T)
    want = run_queries(ctx, monkeypatch, metric, data, nodes, T)
    stage(ctx, monkeypatch, metric, data, host=True)
    c0 = ctx.counters()
    got = run_queries(ctx, monkeypatch, metric, data, nodes, T)
    assert ctx.counters()["fused_rerank_batches"] == c0["fused_rerank_batches"]   # no bf16 shadow in host placement
    for (name, a), (_, b) in zip(got, want):
        a = a if isinstance(a, tuple) else (a,)
        b = b if isinstance(b, tuple) else (b,)
        for x, y in zip(a, b):
            assert np.asarray(x).tobytes() == np.asarray(y).tobytes(), (metric, name)


def test_cosine_default_headers_come_from_the_encoder(ctx, monkeypatch):
    n, d = 5000, 100
    data = oracle.synth_rows(SEED, d, 0, n, 0.5, threads=THREADS)
    data[7] = 0.0
    data[8] *= np.float32(2.0 ** -70)
    stage(ctx, monkeypatch, "cosine", data, host=False)
    want = ctx.item_headers()[0]
    hi_d, lo_d, sc_d = ctx.prefilter_planes(n, ld_of(d))
    stage(ctx, monkeypatch, "cosine", data, host=True)
    assert ctx.item_headers()[0].tobytes() == want.tobytes()
    hi, lo, sc = ctx.prefilter_planes(n, ld_of(d))
    assert hi.tobytes() == hi_d.tobytes() and lo.tobytes() == lo_d.tobytes() and sc.tobytes() == sc_d.tobytes()
    rows = np.array([0, 7, 8, n - 1], dtype=np.uint32)
    padded = np.zeros((n, ld_of(d)), dtype=np.float32)
    padded[:, :d] = data
    assert ctx.read_items(rows).tobytes() == padded[rows].tobytes()


# ---- what stays on the device ------------------------------------------------------------------------------------------------
def test_edges_stay_on_the_device(ctx, monkeypatch):
    monkeypatch.setenv("ARROY_B200_HOST_ITEMS", "1")
    n = 2000
    data = oracle.synth_rows(SEED, 128, 0, n, 0.5, threads=THREADS)
    ids = np.arange(n, dtype=np.uint32)
    ctx.stage_items_flat("binary quantized cosine", ids, data)
    assert ctx.item_placement()["placement"] == "device"
    ctx.stage_items_flat("euclidean", ids, np.ascontiguousarray(data[:, :32]))
    assert ctx.item_placement()["placement"] == "device"
    dev = torch.from_numpy(data).cuda()
    ctx.stage_items_device("euclidean", ids, 128, dev.data_ptr())
    torch.cuda.synchronize()
    assert ctx.item_placement()["placement"] == "device"
    ctx.device_ptrs()
    ctx.stage_items_flat("euclidean", ids, data)
    assert ctx.item_placement()["placement"] == "host"
    with pytest.raises(ab.ArroyB200Error) as ei:
        ctx.device_ptrs()
    assert ei.value.code == _capi.ERR_INVALID
    del dev


def test_restaging_frees_what_the_placement_reports(monkeypatch):
    c = ab.Context(0)
    try:
        n, d = 400_000, 512   # 819 MB of f32 rows
        data = oracle.synth_rows(SEED, d, 0, n, 0.5, threads=THREADS)
        torch.cuda.init()
        stage(c, monkeypatch, "cosine", data, host=True)
        host1 = c.item_placement()
        free_h1 = torch.cuda.mem_get_info()[0]
        stage(c, monkeypatch, "cosine", data, host=False)
        dev = c.item_placement()
        free_d = torch.cuda.mem_get_info()[0]
        stage(c, monkeypatch, "cosine", data, host=True)
        host2 = c.item_placement()
        free_h2 = torch.cuda.mem_get_info()[0]
        assert host1 == host2
        slack = 16 << 20
        # device placement adds its f32 rows (the planes stay allocated for its first build); host placement frees them again
        assert abs((free_h1 - free_d) - dev["device_bytes"]) <= slack, (free_h1, free_d, dev)
        assert abs((free_h2 - free_d) - dev["device_bytes"]) <= slack, (free_h2, free_d, dev)
    finally:
        c.close()
