"""Binary-quantized items on the device as bit strings (kernels.cuh bq_row_u4): the layout every staging path writes, and the
builds, side() scans and searches that read it, against the oracle.

A row is the reference's bit string (binary_quantized.rs:80-92): bit i of u64 word w set when element 64 w + i is positive,
padded with zero bytes to a multiple of 16. device_ptrs reports the row stride as bytes / 4, so the item buffer is an
n x ld float32 view of the bit rows."""
import os

import numpy as np
import pytest

import arroy_b200 as ab
import oracle
from arroy_b200._capi import ArroyB200Error, ERR_INVALID
from arroy_b200.parallel import _DevView
from test_gpu_bq_search import GRID, Index, run_searches
from test_gpu_build_schedules import build_subtrees, oracle_forest
from test_gpu_filtered_search import decode_node, forest_arrays

pytestmark = pytest.mark.gpu
SEED = bytes([42] * 32)
THREADS = min(os.cpu_count() or 4, 32)
BQ = ["binary quantized euclidean", "binary quantized cosine", "binary quantized manhattan"]
DIMS = [64, 100, 768, 1000, 1536, 8192]
PERSISTENT, ASYNC = 1, 4


@pytest.fixture(scope="module")
def ctx():
    c = ab.Context(0)
    yield c
    c.close()


def row_bytes(d):
    """ceil(d / 64) u64 words, rounded up to 16 bytes"""
    return (d + 127) // 128 * 16


def expected_rows(raw):
    """the reference's bit strings of `raw`, padded to row_bytes"""
    pm1 = oracle.bq_quantize(raw)
    bits = np.packbits(pm1 > 0, axis=1, bitorder="little")
    out = np.zeros((raw.shape[0], row_bytes(raw.shape[1])), np.uint8)
    out[:, :bits.shape[1]] = bits
    return out


def device_rows(ctx, n):
    import torch
    (p_items, _, _), ld = ctx.device_ptrs()
    t = torch.as_tensor(_DevView(p_items, (n, ld)), device="cuda:0")
    return t.cpu().numpy().view(np.uint8), ld


def signed_data(d, n):
    """synthetic rows with +0.0, -0.0 and NaNs of both signs among the components"""
    raw = oracle.synth_rows(SEED, d, 0, n, 0.5, threads=THREADS)
    u = raw.view(np.uint32)
    u[0, :4] = [0x00000000, 0x80000000, 0x7fc00000, 0xffc00000]
    u[1, d - 1] = 0x80000000
    u[2, d // 2] = 0x7fc00001
    u[3, ::7] = 0x00000000
    return raw


def leaf_values(raw, metric):
    """stored Leaf values of the BQ items: [0x00][h0 f32][bit string], one contiguous buffer"""
    d = raw.shape[1]
    dp = (d + 63) // 64 * 64
    bits = np.packbits(oracle.bq_quantize(raw) > 0, axis=1, bitorder="little")
    buf = np.zeros((raw.shape[0], 5 + dp // 8), np.uint8)
    h0 = np.float32(np.sqrt(np.float32(dp))) if metric.endswith("cosine") else np.float32(0)
    buf[:, 1:5] = np.frombuffer(np.full(raw.shape[0], h0, np.float32).tobytes(), np.uint8).reshape(-1, 4)
    buf[:, 5:] = bits
    ptrs = buf.ctypes.data + np.arange(raw.shape[0], dtype=np.uint64) * np.uint64(buf.shape[1])
    return buf, ptrs


@pytest.mark.parametrize("d", DIMS)
def test_every_staging_path_writes_the_reference_bit_strings(ctx, d):
    import torch
    n, metric = 300, "binary quantized cosine"
    raw = signed_data(d, n)
    want = expected_rows(raw)
    ids = np.arange(n, dtype=np.uint32)
    dp = (d + 63) // 64 * 64
    h0 = np.float32(np.sqrt(np.float32(dp)))

    def check(what):
        got, ld = device_rows(ctx, n)
        assert ld * 4 == row_bytes(d) <= ((dp // 64) * 8 + 15) // 16 * 16, (what, ld)
        assert np.array_equal(got, want), what
        assert ctx.item_headers()[0].tobytes() == np.full(n, h0, np.float32).tobytes(), what

    ctx.stage_items_flat(metric, ids, raw)
    check("stage_items_flat")
    dev = torch.from_numpy(raw).to("cuda:0")
    ctx.stage_items_device(metric, ids, d, dev.data_ptr())
    torch.cuda.synchronize()
    check("stage_items_device")
    buf, ptrs = leaf_values(raw, metric)
    ctx.stage_items_ptrs(metric, d, ids, ptrs)
    check("stage_items")
    ctx.stage_begin(metric, d, ids)
    for a in range(0, n, 128):
        ctx.stage_rows(a, ptrs[a:a + 128])
    ctx.stage_end()
    check("stage_begin / _rows / _end")
    del buf


def tree_seeds(T):
    r1 = oracle.StdRng(oracle.StdRng(SEED).gen_seed())
    return [r1.gen_seed() for _ in range(T)]


@pytest.mark.parametrize("metric", BQ)
@pytest.mark.parametrize("d", DIMS)
def test_forests_match_the_oracle(ctx, monkeypatch, metric, d):
    # rows of up to 2048 bits run on the persistent kernel (two waves of 3 and 2 trees), wider ones on the async graph
    n, T, split_after = 3000, 5, 64
    raw = signed_data(d, n)
    ids = np.arange(n, dtype=np.uint32)
    ctx.stage_items_flat(metric, ids, raw)
    monkeypatch.setenv("ARROY_B200_MAX_WAVE", "3")
    got = ctx.build_trees(tree_seeds(T), list(range(T)), T, split_after)
    sched = int(ctx.build_breakdown()["schedules"])
    assert sched & (PERSISTENT if d <= 2048 else ASYNC), sched
    pm1 = oracle.bq_quantize(raw)
    odb = oracle.Db(metric, pm1.shape[1])
    odb.set_items(ids, pm1)
    odb.set_user_dims(d)
    odb.build(oracle.StdRng(SEED), n_trees=T, split_after=split_after, threads=min(T, THREADS))
    want = odb.nodes()
    assert sorted(got) == sorted(want)
    bad = [k for k in want if want[k] != got[k]]
    assert not bad, bad[:8]
    assert ctx.build_stats()["scanned_rows"] == odb.scanned_rows


@pytest.mark.parametrize("metric", BQ)
@pytest.mark.parametrize("d", [64, 1000, 1536])
def test_side_batch_matches_the_oracle(ctx, metric, d):
    n = 5000
    raw = signed_data(d, n)
    ctx.stage_items_flat(metric, np.arange(n, dtype=np.uint32), raw)
    pm1 = oracle.bq_quantize(raw)
    dp = pm1.shape[1]
    rng = np.random.default_rng(d)
    h0, h1 = ctx.item_headers()
    for trial in range(4):
        normal = np.where(rng.random(dp) < 0.5, -1.0, 1.0).astype(np.float32)
        if trial == 0:
            normal = pm1[7].copy()   # margins of exactly 0 on the row's complement, d on the row itself
        bias = float(np.float32(rng.integers(-dp, dp) * 0.5))
        rows = np.sort(rng.choice(n, size=n - 17 * trial, replace=False)).astype(np.uint32)
        gs, gm = ctx.side_batch(normal, (bias, 0.0), rows)
        ws, wm = oracle.side_batch(oracle.METRICS[metric], normal, (bias, 0.0), pm1, h0, h1, rows)
        assert gs.tobytes() == ws.tobytes(), trial
        assert gm.tobytes() == wm.tobytes(), trial


@pytest.mark.parametrize("metric", BQ)
def test_searches_at_1536_dimensions_match_the_oracle(ctx, metric):
    n, d, trees = 3000, 1536, 6
    idx = Index(ctx, metric, oracle.synth_rows(SEED, d, 0, n, 0.5, threads=THREADS), trees)
    idx.qv = oracle.bq_quantize(oracle.synth_rows(SEED, d, n + 7, 40, 0.5, threads=THREADS))
    items = np.random.default_rng(d).choice(n, size=40, replace=False).astype(np.uint32)
    run_searches(ctx, idx, (1, 4, 17, 40), GRID[:6], items)


@pytest.mark.parametrize("metric", BQ)
@pytest.mark.parametrize("d", [64, 100, 768, 1000, 1536])
def test_subtree_builds_on_the_async_graph_match_the_oracle(ctx, metric, d):
    # the schedule rule looks at the staged n: 101 subtrees over a 2 000 064-row index (n x trees > 2e8) run the async graph,
    # which scans through work_kernel<true>; each subtree is one tree of an oracle index over its rows. (The normal pool is
    # sized from the staged n / split_after: split_after = 512 keeps all 101 trees in one wave up to d = 1536.)
    import torch
    n, S, split_after = 2_000_064, 101, 512
    t = torch.empty((n, d), dtype=torch.float32, device="cuda:0")
    ctx.synth_device(SEED, d, 0, n, 0.5, t.data_ptr())
    torch.cuda.synchronize()
    ctx.stage_items_device(metric, np.arange(n, dtype=np.uint32), d, t.data_ptr())
    del t
    torch.cuda.empty_cache()
    window = oracle.synth_rows(SEED, d, 0, 40_000, 0.5, threads=THREADS)
    rng = np.random.default_rng(d)
    subsets = [np.sort(rng.choice(40_000, size=int(rng.integers(2000, 6000)), replace=False)).astype(np.uint32) for _ in range(S)]
    user_seeds = [bytes([(d + s) % 256] * 32) for s in range(S)]
    got = build_subtrees(ctx, [tree_seeds_of(u) for u in user_seeds], subsets, split_after)
    sched = int(ctx.build_breakdown()["schedules"])
    assert sched & ASYNC and not sched & PERSISTENT, sched
    scanned = ctx.build_stats()["scanned_rows"]
    total = 0
    for s in range(S):
        odb = oracle_forest(metric, subsets[s], oracle.bq_quantize(window[subsets[s]]), user_seeds[s], 1, split_after, threads=1, user_dims=d)
        assert got[s] == odb.nodes(), (s, subsets[s].size)
        total += odb.scanned_rows
    assert scanned == total


def tree_seeds_of(user_seed):
    """the seed of the one tree Writer::build derives from the user's StdRng"""
    return oracle.StdRng(oracle.StdRng(user_seed).gen_seed()).gen_seed()


def test_float_only_entry_points_reject_bit_string_items(ctx):
    n, d = 500, 128
    ctx.stage_items_flat("binary quantized euclidean", np.arange(n, dtype=np.uint32), signed_data(d, n))
    with pytest.raises(ArroyB200Error) as e:
        ctx.prefilter_planes(n, d)
    assert e.value.code == ERR_INVALID
    with pytest.raises(ArroyB200Error) as e:
        ctx.prefilter_scores(np.ones((2, d), np.float32), np.arange(n, dtype=np.uint32))
    assert e.value.code == ERR_INVALID
    # the context stays usable
    side, _ = ctx.side_batch(np.ones(d, np.float32), (0.0, 0.0), np.arange(n, dtype=np.uint32))
    assert side.size == n


def mem_available():
    with open("/proc/meminfo") as f:
        for line in f:
            if line.startswith("MemAvailable:"):
                return int(line.split()[1]) * 1024
    return 0


POPC = np.array([bin(i).count("1") for i in range(256)], dtype=np.int32)


def test_twenty_million_rows_of_1536_bits(ctx):
    # the capability itself: 20M x 1536 BQ Cosine staged from host bit strings is 3.8 GB on the device (as +-1 floats it would
    # be 123 GB). The oracle cannot hold it, so the forest and the searches are checked against numpy recomputations.
    import torch
    # (leaves of up to 100k rows keep the forest at a few thousand nodes, so that decoding it in Python takes seconds)
    n, d, T, split_after = 20_000_000, 1536, 4, 100_000
    nbytes = d // 8
    free, _ = torch.cuda.mem_get_info()
    if free < 12 << 30:
        pytest.skip("needs 12 GiB of free device memory, %.1f GiB free" % (free / 2**30))
    if mem_available() < 28 << 30:
        pytest.skip("needs 28 GiB of available host memory, %.1f GiB available" % (mem_available() / 2**30))
    metric, m = "binary quantized cosine", oracle.BQ_COSINE
    h = np.float32(np.sqrt(np.float32(d)))
    buf = np.empty((n, 5 + nbytes), np.uint8)
    buf[:, 0] = 0
    buf[:, 1:5] = np.frombuffer(h.tobytes(), np.uint8)
    rng = np.random.default_rng(20)
    for a in range(0, n, 1 << 21):
        b = min(n, a + (1 << 21))
        buf[a:b, 5:] = np.frombuffer(rng.bytes((b - a) * nbytes), np.uint8).reshape(b - a, nbytes)
    bits = buf[:, 5:]
    ptrs = buf.ctypes.data + np.arange(n, dtype=np.uint64) * np.uint64(buf.shape[1])
    ctx.stage_items_ptrs(metric, d, np.arange(n, dtype=np.uint32), ptrs)
    del ptrs
    _, ld = ctx.device_ptrs()
    assert ld * 4 * n == 3_840_000_000
    got = ctx.build_trees(tree_seeds(T), list(range(T)), T, split_after)
    nodes = {k: decode_node(v, m, d) for k, v in got.items()}

    def rows_under(nid):
        out, stack = [], [nid]
        while stack:
            nd = nodes[stack.pop()]
            if nd["kind"] == "descendants":
                out.append(np.asarray(nd["descendants"], dtype=np.uint32))
            else:
                stack += [nd["left"], nd["right"]]
        return np.concatenate(out)

    for t in range(T):   # every row in exactly one leaf of each tree
        assert np.array_equal(np.sort(rows_under(t)), np.arange(n, dtype=np.uint32)), t
    for nd in nodes.values():
        if nd["kind"] == "descendants":
            assert len(nd["descendants"]) <= split_after
    # sides of sampled split nodes: Left rows have a margin with the sign bit set, Right rows not (Cosine: margin = dot)
    splits = [k for k, nd in nodes.items() if nd["kind"] == "split" and nd["normal"] is not None and k >= T]
    checked = 0
    for k in np.random.default_rng(1).permutation(splits):
        nd = nodes[int(k)]
        left, right = rows_under(nd["left"]), rows_under(nd["right"])
        if left.size + right.size > 250_000:
            continue
        nb = np.packbits(nd["normal"] > 0, bitorder="little")
        for rows, side in ((left, 0), (right, 1)):
            dot = (d - 2 * POPC[bits[rows] ^ nb].sum(axis=1)).astype(np.float32)
            got_side = np.where(np.signbit(dot), 0, 1)
            assert (got_side == side).all(), int(k)
        checked += 1
        if checked == 64:
            break
    assert checked == 64
    ctx.load_forest(roots=np.arange(T, dtype=np.uint32), **forest_arrays(got, m, d))
    del nodes, got
    items = np.random.default_rng(2).choice(n, size=1000, replace=False).astype(np.uint32)
    rows_b, dist_b, len_b, st_b = ctx.search_batch(10, query_rows=items)
    assert not st_b.any()
    pnqn = np.float32(h) * np.float32(h)

    def distances(q, rows):
        dot = (d - 2 * POPC[bits[rows] ^ bits[q]].sum(axis=1)).astype(np.float32)
        return ((np.float32(1) - dot / pnqn) / np.float32(2)).astype(np.float32)

    for i in range(20):   # single queries agree with the batch; distances and order recomputed from the bits
        r1, d1, l1, s1 = ctx.search_batch(10, query_rows=items[i:i + 1])
        assert not s1.any() and l1[0] == len_b[i] > 0
        assert r1[0].tobytes() == rows_b[i].tobytes() and d1[0].tobytes() == dist_b[i].tobytes()
        rr, dd = rows_b[i, :len_b[i]], dist_b[i, :len_b[i]]
        assert dd.tobytes() == distances(items[i], rr).tobytes()
        assert all((dd[j], rr[j]) < (dd[j + 1], rr[j + 1]) for j in range(len(rr) - 1))
    # the re-rank of a candidate set: top 10 of 200k rows recomputed in numpy
    for i in range(4):
        q = int(items[i])
        cand = np.sort(np.random.default_rng(10 + i).choice(n, size=200_000, replace=False)).astype(np.uint32)
        qv = np.where(np.unpackbits(bits[q], bitorder="little") == 1, 1.0, -1.0).astype(np.float32)
        gr, gd = ctx.rerank(qv, (float(h), 0.0), cand, 10)
        dist = distances(q, cand)
        order = np.lexsort((cand, dist))[:10]
        assert gr.tolist() == cand[order].tolist() and gd.tobytes() == dist[order].tobytes()
