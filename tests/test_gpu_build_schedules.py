"""The build's schedules other than the persistent kernel, against the oracle.

build_wave picks a schedule per wave from what it observes: the persistent kernel (rows of at most 2048 floats and
n x trees <= 2e8), or the async CUDA graph, with one control CTA per tree or, for d <= 256 and float metrics, a thread-block
cluster of 8 (9-16 trees in the wave) or 16 (<= 8 trees) CTAs that scans small nodes itself. Rows wider than 3648 floats keep
two_means' workspace in global memory; rows wider than 2112 floats give up the speculative two_means. Every case here checks
the NodeCodec bytes of the device forest against the oracle, the rows scanned against the oracle's count, and the schedule
bits the build reports (build_breakdown()["schedules"]), so that a change of a threshold cannot quietly move a case back
onto the persistent kernel."""
import ctypes as C
import os
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import pytest

import arroy_b200 as ab
import oracle
from arroy_b200 import _capi
from test_gpu_filtered_search import forest_arrays

pytestmark = pytest.mark.gpu
SEED = bytes([42] * 32)
THREADS = min(os.cpu_count() or 4, 32)
# build_breakdown()["schedules"] bits (include/arroy_b200.h)
PERSISTENT, LOCKSTEP, ASYNC, CLUSTER8, CLUSTER16, GLOBAL_WS, SPECULATIVE = 1, 2, 4, 8, 16, 32, 64


@pytest.fixture(scope="module")
def ctx():
    c = ab.Context(0)
    yield c
    c.close()


def tree_seeds(user_seed, T):
    """the tree seeds Writer::build derives from the user's StdRng (src/writer.rs:575, :795)"""
    r1 = oracle.StdRng(oracle.StdRng(user_seed).gen_seed())
    return [r1.gen_seed() for _ in range(T)]


def schedules(ctx):
    return int(ctx.build_breakdown()["schedules"])


def assert_same_forest(got, want, what):
    assert sorted(got) == sorted(want), (what, len(got), len(want))
    bad = [k for k in sorted(want) if want[k] != got[k]]
    assert not bad, "%s: node bytes differ for %d of %d nodes, first ids %s" % (what, len(bad), len(want), bad[:8])


def oracle_forest(metric, ids, vectors, user_seed, T, split_after, threads=None, user_dims=None):
    odb = oracle.Db(metric, vectors.shape[1])
    odb.set_items(ids, vectors)
    if user_dims is not None:
        odb.set_user_dims(user_dims)
    odb.build(oracle.StdRng(user_seed), n_trees=T, split_after=split_after, threads=threads or min(T, THREADS))
    return odb


def device_forest(ctx, metric, data, T, split_after, user_seed=SEED, cancel=None):
    ctx.stage_items_flat(metric, np.arange(data.shape[0], dtype=np.uint32), data)
    if metric == "dot-product":
        ctx.dot_preprocess()
    return ctx.build_trees(tree_seeds(user_seed, T), list(range(T)), T, split_after, cancel=cancel)


# ---- (a) rows wider than 2048 floats: the async graph ---------------------------------------------------------------------
# d -> the schedule bits of a 3-tree build of a few thousand rows
WIDE = {
    2048: PERSISTENT,                  # control: the widest row of the persistent kernel
    2080: ASYNC | SPECULATIVE,         # 24-vector speculative workspace still fits in shared memory
    2144: ASYNC,                       # ... no longer does
    3648: ASYNC,                       # the largest 14-vector workspace in shared memory
    3680: ASYNC | GLOBAL_WS,           # workspace in global memory
    8192: ASYNC | GLOBAL_WS,           # the widest row with the 8-bit pre-filter planes (work_kernel_planes)
    8224: ASYNC | GLOBAL_WS,           # f32 work_kernel scans
}
WIDE_CASES = [(m, d) for d in WIDE for m in ("euclidean", "cosine")] + \
             [(m, d) for d in (2080, 3680, 8224) for m in ("dot-product", "manhattan")]


@pytest.mark.parametrize("metric,d", WIDE_CASES)
def test_wide_rows_match_the_oracle(ctx, metric, d):
    n, T, split_after = (5000 if d <= 3680 else 3000), 3, 64
    data = oracle.synth_rows(SEED, d, 0, n, 0.0 if metric == "euclidean" else 0.5, threads=THREADS)
    got = device_forest(ctx, metric, data, T, split_after)
    st, sched, pre = ctx.build_stats(), schedules(ctx), ctx.build_prefilter_stats()
    odb = oracle_forest(metric, np.arange(n, dtype=np.uint32), data, SEED, T, split_after)
    assert_same_forest(got, odb.nodes(), (metric, d))
    assert st["scanned_rows"] == odb.scanned_rows
    assert sched == WIDE[d], (sched, WIDE[d])
    if d >= 8192:
        assert (pre["rows_via_prefilter"] > 0) == (d == 8192), pre
        # queries on both sides of walk1_kernel's widest row (search.cuh W1_MAX_LD = 8192): 8224 takes the batched walker
        m = oracle.METRICS[metric]
        ctx.load_forest(roots=np.arange(T, dtype=np.uint32), **forest_arrays(got, m, d))
        qitems = np.array([0, 7, 1234, n - 1], dtype=np.uint32)
        for count, sk in ((10, 0), (50, 600)):
            out_rows, out_dist, out_len, status = ctx.search_batch(count, query_rows=qitems, search_k=sk)
            assert not status.any()
            for i, it in enumerate(qitems):
                w = odb.nns_by_item(int(it), count, search_k=sk or None)
                assert out_rows[i, :out_len[i]].tolist() == [x[0] for x in w], (count, sk, int(it))
                assert out_dist[i, :out_len[i]].tobytes() == np.array([x[1] for x in w], dtype=np.float32).tobytes()


@pytest.mark.parametrize("metric,d,want", [("binary quantized euclidean", 2100, ASYNC | SPECULATIVE),
                                           ("binary quantized cosine", 4000, ASYNC | GLOBAL_WS)])
def test_wide_binary_quantized_rows_match_the_oracle(ctx, metric, d, want):
    # the bit strings are padded to a multiple of 64 (2112 / 4032 floats), which is what takes them off the persistent kernel
    n, T, split_after = 4000, 3, 64
    raw = oracle.synth_rows(SEED, d, 0, n, 0.5, threads=THREADS)
    got = device_forest(ctx, metric, raw, T, split_after)
    st, sched = ctx.build_stats(), schedules(ctx)
    pm1 = oracle.bq_quantize(raw)
    odb = oracle_forest(metric, np.arange(n, dtype=np.uint32), pm1, SEED, T, split_after, user_dims=d)
    assert_same_forest(got, odb.nodes(), metric)
    assert st["scanned_rows"] == odb.scanned_rows
    assert sched == want, (sched, want)


# ---- (b) the async schedule's cached graph and cancellation ---------------------------------------------------------------
def test_async_graph_reuse_restage_and_cancel(ctx):
    # same shapes => the CUDA graph captured by the first build is launched again by the later ones
    metric, n, d, T, split_after = "cosine", 4000, 2144, 3, 32
    seed_a, seed_b = SEED, bytes([7] * 32)
    ids = np.arange(n, dtype=np.uint32)
    data = oracle.synth_rows(SEED, d, 0, n, 0.5, threads=THREADS)
    other = oracle.synth_rows(SEED, d, n, n, 0.5, threads=THREADS)

    def check(got, vectors, user_seed, what):
        odb = oracle_forest(metric, ids, vectors, user_seed, T, split_after)
        assert_same_forest(got, odb.nodes(), what)
        assert ctx.build_stats()["scanned_rows"] == odb.scanned_rows, what
        assert schedules(ctx) == ASYNC, (what, schedules(ctx))

    check(device_forest(ctx, metric, data, T, split_after, seed_a), data, seed_a, "seeds A")
    check(ctx.build_trees(tree_seeds(seed_b, T), list(range(T)), T, split_after), data, seed_b, "seeds B")
    check(device_forest(ctx, metric, other, T, split_after, seed_a), other, seed_a, "restaged items")
    polls = []

    def cancel():
        polls.append(1)
        return len(polls) >= 2   # the first poll is before the build, the second after the first graph launch

    with pytest.raises(ab.ArroyB200Error) as ei:
        ctx.build_trees(tree_seeds(seed_b, T), list(range(T)), T, split_after, cancel=cancel)
    assert ei.value.code == _capi.ERR_CANCELLED and len(polls) == 2
    check(ctx.build_trees(tree_seeds(seed_b, T), list(range(T)), T, split_after), other, seed_b, "after a cancelled build")


# ---- (c) the cluster control kernels on a full index ----------------------------------------------------------------------
def test_cluster_kernels_on_a_full_index(ctx, monkeypatch):
    # 16 trees x 12.6M rows > 2e8: the first wave runs the async graph with clusters of 8 CTAs per tree; the second wave of 4
    # trees (50.4M) runs the persistent kernel. Nodes of more than small_max = 24576 rows are scanned by work_kernel_planes,
    # smaller ones inside the cluster, and every tree crosses the 1024-attempt limit of one control launch many times.
    # split_after = 1000 keeps the forest at tens of thousands of nodes per tree: at the default (64) the host-side comparison
    # of ~8M nodes takes minutes, while the nodes of 1000 ... 24576 rows still go through the cluster scans.
    metric, n, d, T, split_after = "euclidean", 12_600_000, 64, 20, 1000
    data = oracle.synth_rows(SEED, d, 0, n, 0.0, threads=THREADS)
    monkeypatch.setenv("ARROY_B200_MAX_WAVE", "16")
    got = device_forest(ctx, metric, data, T, split_after)
    st, sched = ctx.build_stats(), schedules(ctx)
    assert sched == CLUSTER8 | PERSISTENT | SPECULATIVE, \
        "schedules %d: expected clusters of 8 for the 16-tree wave and the persistent kernel for the 4-tree wave" % sched
    odb = oracle_forest(metric, np.arange(n, dtype=np.uint32), data, SEED, T, split_after)
    del data
    assert_same_forest(got, odb.nodes(), "12.6M x 64, 20 trees")
    assert st["scanned_rows"] == odb.scanned_rows


# ---- (d) the cluster control kernels for every float metric, through subtree builds ------------------------------------
# The schedule rule looks at the staged n, so subtrees over row subsets of a 25 000 064-row index reach it: 8 subtrees
# (25 000 064 x 8 > 2e8) run clusters of 16 CTAs, 12 subtrees clusters of 8. Each subtree is one tree of an oracle index over
# its rows. Rows are synthesized on the device; the oracle synthesizes the windows the subsets are drawn from.
BIG_N, BIG_D, SUB_SPLIT = 25_000_064, 64, 64
WINDOWS = [(0, 300_000), ((1 << 24) - 150_000, 300_000), (BIG_N - 300_000, 300_000)]   # row 0, across 2^24, the last row


def build_subtrees(ctx, seeds, subsets, split_after):
    """arroy_b200_build_subtrees_begin + arroy_b200_build_trees_emit_mapped: subtree s gets root id s << 22 and its other
    nodes (s << 22) + 1 + post-order index, so that subtracting s << 22 gives the numbering of a one-tree index."""
    S = len(subsets)
    seed_buf = (C.c_uint8 * (32 * S))(*b"".join(seeds))
    rows = np.ascontiguousarray(np.concatenate(subsets), dtype=np.uint32)
    off = np.zeros(S + 1, dtype=np.uint64)
    off[1:] = np.cumsum([s.size for s in subsets])
    counts = np.zeros(S, dtype=np.uint32)
    lib = ctx.lib
    ctx._ck(lib.arroy_b200_build_subtrees_begin(ctx.h, S, C.cast(seed_buf, C.c_void_p), _capi._up(rows), off.ctypes.data_as(_capi._u64p),
                                                split_after, C.cast(None, _capi.CANCEL_FN), None, _capi._up(counts)))
    root_ids = (np.arange(S, dtype=np.uint32) << 22).astype(np.uint32)
    node_ids = np.concatenate([(s << 22) + 1 + np.arange(int(counts[s]) - 1, dtype=np.uint32) for s in range(S)]).astype(np.uint32)
    out = [dict() for _ in range(S)]

    def sink(_arg, node_id, ptr, length):
        s, b = node_id >> 22, bytearray(C.string_at(ptr, length))
        if b[0] == 2:   # split node: child ids, big-endian
            for o in (1, 5):
                b[o:o + 4] = (int.from_bytes(b[o:o + 4], "big") - (s << 22)).to_bytes(4, "big")
        out[s][node_id - (s << 22)] = bytes(b)
        return 0

    cb = _capi.NODE_SINK(sink)
    ctx._ck(lib.arroy_b200_build_trees_emit_mapped(ctx.h, _capi._up(root_ids), _capi._up(node_ids), cb, None))
    return out


@pytest.fixture(scope="module")
def window_rows():
    return [oracle.synth_rows(SEED, BIG_D, r0, w, 0.5, threads=THREADS) for r0, w in WINDOWS]


def subset_plan(S, rng):
    """S ascending random samples: two small enough to be scanned in the cluster from their root on (<= 24576 rows), the
    others 30k - 250k rows; windows taken in turn"""
    sizes = [5_000, 20_000] + [int(x) for x in rng.integers(30_000, 250_001, S - 2)]
    plan = []
    for s, size in enumerate(sizes):
        wi = s % len(WINDOWS)
        r0, w = WINDOWS[wi]
        plan.append((wi, np.sort(rng.choice(w, size=size, replace=False)).astype(np.uint32) + np.uint32(r0)))
    return plan


@pytest.mark.parametrize("metric", ["euclidean", "cosine", "dot-product", "manhattan"])
def test_cluster_kernels_through_subtrees(ctx, window_rows, metric):
    import torch
    t = torch.empty((BIG_N, BIG_D), dtype=torch.float32, device="cuda:0")
    ctx.synth_device(SEED, BIG_D, 0, BIG_N, 0.5, t.data_ptr())
    torch.cuda.synchronize()
    ctx.stage_items_device(metric, np.arange(BIG_N, dtype=np.uint32), BIG_D, t.data_ptr())
    del t
    torch.cuda.empty_cache()
    extra_row = None
    if metric == "dot-product":
        # preprocess takes the largest norm over all staged rows: the row it belongs to goes into every subset, so that each
        # subset's oracle index sees the same maximum
        extra, _ = ctx.dot_preprocess()
        extra_row = int(np.argmin(extra))
        assert extra[extra_row] == 0.0
        extra_vec = oracle.synth_rows(SEED, BIG_D, extra_row, 1, 0.5)[0]
    rng = np.random.default_rng(len(metric))
    for S, want in ((8, CLUSTER16), (12, CLUSTER8)):
        plan = subset_plan(S, rng)
        subsets, vectors = [], []
        for wi, rows in plan:
            vec = window_rows[wi][rows - np.uint32(WINDOWS[wi][0])]
            if extra_row is not None and extra_row not in rows:
                at = int(np.searchsorted(rows, extra_row))
                rows, vec = np.insert(rows, at, extra_row), np.insert(vec, at, extra_vec, axis=0)
            subsets.append(rows.astype(np.uint32))
            vectors.append(vec)
        user_seeds = [bytes([(S * 16 + s) % 256] * 32) for s in range(S)]
        got = build_subtrees(ctx, [tree_seeds(u, 1)[0] for u in user_seeds], subsets, SUB_SPLIT)
        st, sched = ctx.build_stats(), schedules(ctx)
        assert sched == want | SPECULATIVE, \
            "%d subtrees: schedules %d, expected %d (a smaller wave than %d trees, e.g. for lack of free device memory, " \
            "changes the cluster size)" % (S, sched, want | SPECULATIVE, S)

        def one(s):
            return oracle_forest(metric, subsets[s], vectors[s], user_seeds[s], 1, SUB_SPLIT, threads=1)
        with ThreadPoolExecutor(max_workers=THREADS) as ex:
            odbs = list(ex.map(one, range(S)))
        for s in range(S):
            assert_same_forest(got[s], odbs[s].nodes(), (metric, S, s, subsets[s].size))
        assert st["scanned_rows"] == sum(o.scanned_rows for o in odbs)


# ---- (e) work_kernel's shared-memory attribute at rows of 12 800 floats -------------------------------------------------
def side_multi(ctx, normals, hdr0, subsets):
    normals = np.ascontiguousarray(normals, dtype=np.float32)
    hdr0 = np.ascontiguousarray(hdr0, dtype=np.float32)
    rows = np.ascontiguousarray(np.concatenate(subsets), dtype=np.uint32)
    off = np.zeros(len(subsets) + 1, dtype=np.uint64)
    off[1:] = np.cumsum([s.size for s in subsets])
    side = np.empty(rows.size, dtype=np.uint8)
    ctx._ck(ctx.lib.arroy_b200_side_multi(ctx.h, len(subsets), _capi._fp(normals), _capi._fp(hdr0), None, _capi._up(rows),
                                          off.ctypes.data_as(_capi._u64p), side.ctypes.data_as(_capi._u8p)))
    return np.split(side, off[1:-1].astype(np.int64))


def test_side_multi_around_a_build_at_12800_floats(ctx):
    # side_multi with 40 jobs asks work_kernel for ld * 4 + 41 * 4 + 16 bytes of shared memory (> 48 KiB); a build of 2 trees
    # sets the kernel's limit to its own, smaller request; the same side_multi afterwards must still launch
    metric, n, d, jobs, T, split_after = "euclidean", 2000, 12800, 40, 2, 64
    data = oracle.synth_rows(SEED, d, 0, n, 0.0, threads=THREADS)
    ctx.stage_items_flat(metric, np.arange(n, dtype=np.uint32), data)
    r = np.random.default_rng(12800)
    normals = (r.standard_normal((jobs, d)) / np.sqrt(d)).astype(np.float32)
    hdr0 = (r.standard_normal(jobs) * 0.1).astype(np.float32)
    subsets = [np.sort(r.choice(n, size=int(r.integers(1, n)), replace=False)).astype(np.uint32) for _ in range(jobs)]
    h0 = np.zeros(n, dtype=np.float32)
    want = [oracle.side_batch(oracle.EUCLIDEAN, normals[j], (float(hdr0[j]), 0.0), data, h0, None, subsets[j], want_margin=False)[0]
            for j in range(jobs)]
    before = side_multi(ctx, normals, hdr0, subsets)
    got = ctx.build_trees(tree_seeds(SEED, T), list(range(T)), T, split_after)
    after = side_multi(ctx, normals, hdr0, subsets)
    for j in range(jobs):
        assert before[j].tobytes() == want[j].tobytes(), j
        assert after[j].tobytes() == want[j].tobytes(), j
    assert schedules(ctx) == ASYNC | GLOBAL_WS
    odb = oracle_forest(metric, np.arange(n, dtype=np.uint32), data, SEED, T, split_after)
    assert_same_forest(got, odb.nodes(), "d = 12800")


def test_incremental_updates_at_12800_floats(ctx):
    # Writer::build on an existing index routes new items with side_multi, rebuilds the subtrees that grew, and routes again
    metric, d, T, split_after, n0 = "euclidean", 12800, 3, 64, 1500
    data = oracle.synth_rows(SEED, d, 0, n0 + 600, 0.0, threads=THREADS)
    env = ab.Env(0)
    env._ctx = ctx
    w = ab.Writer(env, 0, d, metric)
    odb = oracle.Db(metric, d)
    prng, orng = ab.StdRng.from_seed(SEED), oracle.StdRng(SEED)
    r = np.random.default_rng(3)
    for i in range(n0):
        w.add_item(i, data[i])
        odb.add_item(i, data[i])
    live, next_new = set(range(n0)), n0
    for rnd in range(3):
        w.builder(prng).n_trees(T).split_after(split_after).build()
        odb.build_incremental(orng, n_trees=T, split_after=split_after)
        assert env.tree_nodes() == odb.nodes(), rnd
        for i in r.choice(sorted(live), size=60, replace=False):
            w.del_item(int(i)); odb.del_item(int(i)); live.discard(int(i))
        for i in r.choice(sorted(live), size=40, replace=False):
            v = data[int(r.integers(0, len(data)))] * np.float32(0.5)
            w.add_item(int(i), v); odb.add_item(int(i), v)
        for _ in range(int(r.integers(100, 200))):
            w.add_item(next_new, data[next_new]); odb.add_item(next_new, data[next_new])
            live.add(next_new); next_new += 1
    w.builder(prng).n_trees(T).split_after(split_after).build()
    odb.build_incremental(orng, n_trees=T, split_after=split_after)
    assert env.tree_nodes() == odb.nodes()
    env._ctx = None
