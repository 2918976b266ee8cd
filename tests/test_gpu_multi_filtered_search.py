"""Batches in which every query carries its own QueryBuilder::candidates filter (arroy_b200_search_batch_multi_filtered,
Reader.nns_batch_by_item / nns_batch_by_vector with filters= / filter_of_query=): each row must equal the same query issued
alone with its filter, on the device and in the oracle (ids and float32 bytes)."""
import ctypes
import os
import re

import numpy as np
import pytest

import arroy_b200 as ab
import oracle
from arroy_b200._capi import ERR_INVALID, _u32p, _u64p, row_bitmap

pytestmark = pytest.mark.gpu
SEED = bytes([42] * 32)
U64_MAX = 2**64 - 1


@pytest.fixture(scope="module")
def shared_ctx():
    c = ab.Context(0)
    c.envs = []   # an Env closes its context when collected: keep them until the module is done, then detach them
    yield c
    for e in c.envs:
        e._ctx = None
    c.close()


def build_pair(ctx, metric, n, d, trees, ids=None):
    data = oracle.synth_rows(SEED, d, 0, n, 0.5, threads=8)
    ids = np.arange(n, dtype=np.uint32) if ids is None else ids
    odb = oracle.Db(metric, d)
    odb.set_items(ids, data)
    odb.build(oracle.StdRng(SEED), n_trees=trees, threads=8)
    env = ab.Env(0)
    env._ctx = ctx
    ctx.envs.append(env)
    w = ab.Writer(env, 0, d, metric)
    w.add_items(ids, data)
    w.builder(ab.StdRng.from_seed(SEED)).n_trees(trees).build()
    return ab.Reader.open(env, 0, metric), odb, ids


def filter_grid(ids, count):
    """all items, 50 %, 5 %, 0.5 %, exactly `count` items, fewer than `count`, one item, empty, only ids outside the index, ids
    mixed in and out"""
    rng = np.random.default_rng(7)
    n = ids.size
    pick = lambda m: np.sort(rng.choice(ids, size=m, replace=False)).tolist()
    outside = (int(ids.max()) + 1 + np.arange(50)).tolist()
    return [ids.tolist(), pick(n // 2), pick(n // 20), pick(max(1, n // 200)), pick(count), pick(count // 2), pick(1), [], outside,
            sorted(pick(30) + outside[:20])]


def same(got, want):
    assert [g[0] for g in got] == [w[0] for w in want]
    assert np.array([g[1] for g in got], dtype=np.float32).tobytes() == np.array([w[1] for w in want], dtype=np.float32).tobytes()


def row(res, i):
    return list(zip(res[0][i, :res[2][i]].tolist(), res[1][i, :res[2][i]].tolist()))


def same_rows(a, i, b, j):   # row i of one device result and row j of another: ids and float32 bytes
    assert a[2][i] == b[2][j]
    assert a[0][i, :a[2][i]].tobytes() == b[0][j, :b[2][j]].tobytes() and a[1][i, :a[2][i]].tobytes() == b[1][j, :b[2][j]].tobytes()


@pytest.mark.parametrize("metric,d", [("euclidean", 24), ("cosine", 48), ("dot-product", 96), ("manhattan", 128)])
def test_per_query_filters_match_the_oracle(shared_ctx, metric, d):
    n, trees, count, nq = 3000, 8, 10, 24
    r, odb, ids = build_pair(shared_ctx, metric, n, d, trees)
    grid = filter_grid(ids, count)
    fl = grid[:5] + [list(range(0, n, 7))] + grid[5:] + [list(range(3, n, 11))]   # filters 5 and 11 are not used
    used = [f for f in range(len(fl)) if f not in (5, 11)]
    fq = [used[i % len(used)] for i in range(nq)]   # every used filter twice or three times
    rng = np.random.default_rng(17)
    items = rng.choice(n, size=nq, replace=False)
    vecs = oracle.synth_rows(SEED, d, n + 11, nq, 0.5)
    s0 = shared_ctx.search_stats()
    for sk in (None, 1, 3000, U64_MAX):
        bi = r.nns_batch_by_item(items, count, search_k=sk, filters=fl, filter_of_query=fq)
        bv = r.nns_batch_by_vector(vecs, count, search_k=sk, filters=fl, filter_of_query=fq)
        for i in range(nq):
            F = fl[fq[i]]
            want = odb.nns_by_item(int(items[i]), count, search_k=sk, candidates=F)
            same(row(bi, i), want)
            same(r.nns(count).search_k(sk).candidates(F).by_item(int(items[i])), want)
            wv = odb.nns_by_vector(vecs[i], count, search_k=sk, candidates=F)
            same(row(bv, i), wv)
            same(r.nns(count).search_k(sk).candidates(F).by_vector(vecs[i]), wv)
    ob = r.nns_batch_by_item(items, count, oversampling=3, filters=fl, filter_of_query=fq)
    for i in range(nq):
        same(row(ob, i), odb.nns_by_item(int(items[i]), count, oversampling=3, candidates=fl[fq[i]]))
    s1 = shared_ctx.search_stats()
    assert s1["failed_queries"] == s0["failed_queries"]


def test_both_walkers_summary_groups_and_the_shortcut(shared_ctx, capfd):
    # 12 queries walk in walk1_kernel (its ARROY_B200_WALK1_DEBUG line is printed once per completed walk), 40 in walk_kernel; 70
    # distinct filters take three summary passes of 32. Filters of at most `count` items take the shortcut (with the default
    # search_k = count x trees, their rows in the forest number at most search_k) in the same calls as the walked ones.
    n, d, trees, count = 5000, 40, 12, 10
    r, odb, ids = build_pair(shared_ctx, "cosine", n, d, trees, ids=np.arange(0, 2 * 5000, 2, dtype=np.uint32))   # rows != ids
    rng = np.random.default_rng(21)
    for nq, n_filters, walk1 in ((12, 12, True), (40, 30, False), (80, 70, False)):
        # unsorted id arrays, one of them with duplicates; the last filter is unused
        fl = [rng.choice(ids, size=int(rng.integers(1, count + 1)) if j % 3 == 0 else int(rng.choice([n // 10, n // 100, 300])), replace=False)
              for j in range(n_filters + 1)]
        fl[1] = np.concatenate([fl[1], fl[1][:7]])
        fq = rng.permutation([j % n_filters for j in range(nq)])
        items = rng.choice(ids, size=nq, replace=False)
        shortcut = sum(1 for f in fq if np.unique(fl[f]).size <= count)
        assert 0 < shortcut < nq
        s0, m0 = shared_ctx.search_stats(), shared_ctx.multi_filter_stats()
        if walk1:
            os.environ["ARROY_B200_WALK1_DEBUG"] = "1"
            capfd.readouterr()
        try:
            got = r.nns_batch_by_item(items, count, filters=fl, filter_of_query=fq)
            if walk1:
                ctypes.CDLL(None).fflush(None)   # the device printf lands in the C stdout buffer
                out = capfd.readouterr().out
        finally:
            os.environ.pop("ARROY_B200_WALK1_DEBUG", None)
        s1, m1 = shared_ctx.search_stats(), shared_ctx.multi_filter_stats()
        assert s1["filtered_queries"] - s0["filtered_queries"] == nq
        assert s1["shortcut_queries"] - s0["shortcut_queries"] == shortcut
        assert s1["failed_queries"] == s0["failed_queries"]
        assert m1["summary_passes"] - m0["summary_passes"] == (n_filters + 31) // 32
        assert m1["filters_summarised"] - m0["filters_summarised"] == n_filters
        if walk1:
            assert len(re.findall(r"\[walk1\] q \d+", out)) == nq - shortcut, out
        for i in range(nq):
            F = fl[fq[i]].tolist()
            want = odb.nns_by_item(int(items[i]), count, candidates=F)
            same(row(got, i), want)
            same(r.nns(count).candidates(F).by_item(int(items[i])), want)


def decode_node(b, metric, d):
    """oracle.decode_node, plus the binary-quantized normals: a bit string of 64-bit words, bit i of word w = element 64 w + i,
    set = +1, clear = -1 (d = the padded length)."""
    if metric < oracle.BQ_EUCLIDEAN or b[0] != 2 or len(b) == 9:
        return oracle.decode_node(b, metric, d)
    bits = np.unpackbits(np.frombuffer(b[13:], dtype=np.uint8), bitorder="little")
    return {"kind": "split", "left": int.from_bytes(b[1:5], "big"), "right": int.from_bytes(b[5:9], "big"),
            "header": np.frombuffer(b[9:13], dtype=np.float32).copy(), "normal": np.where(bits == 1, 1.0, -1.0).astype(np.float32)}


def forest_arrays(nodes, metric, d):
    """{node id: NodeCodec bytes} -> the arrays arroy_b200_load_forest takes (rows == item ids here)."""
    nn = max(nodes) + 1
    kind = np.zeros(nn, np.uint8)
    left, right, nidx = np.zeros(nn, np.uint32), np.zeros(nn, np.uint32), np.full(nn, 0xffffffff, np.uint32)
    nh0, doff, dlen = np.zeros(nn, np.float32), np.zeros(nn, np.uint32), np.zeros(nn, np.uint32)
    normals, desc = [], []
    for i, b in nodes.items():
        nd = decode_node(b, metric, d)
        if nd["kind"] == "descendants":
            kind[i] = 1
            doff[i], dlen[i] = sum(x.size for x in desc), len(nd["descendants"])
            desc.append(np.asarray(nd["descendants"], dtype=np.uint32))
        else:
            kind[i] = 2
            left[i], right[i] = nd["left"], nd["right"]
            if nd["normal"] is not None:
                nidx[i] = len(normals)
                nh0[i] = nd["header"][0]
                normals.append(nd["normal"])
    normals = np.stack(normals) if normals else np.zeros((0, d), np.float32)
    return dict(kind=kind, left=left, right=right, normal_idx=nidx, normal_hdr0=nh0, desc_off=doff, desc_len=dlen, normals=normals,
                desc_rows=np.concatenate(desc) if desc else np.zeros(0, np.uint32))


def load_built_forest(ctx, metric, n, d, trees, data, quantized=None):
    """stage `data`, build `trees` trees on the device (checked against the oracle's) and load them with load_forest; for the
    binary-quantized metrics the oracle takes the +-1 vectors `quantized`"""
    vectors = data if quantized is None else quantized
    ctx.stage_items_flat(metric, np.arange(n, dtype=np.uint32), data)
    r1 = oracle.StdRng(oracle.StdRng(SEED).gen_seed())
    seeds = [r1.gen_seed() for _ in range(trees)]
    odb = oracle.Db(metric, vectors.shape[1])
    odb.set_items(np.arange(n, dtype=np.uint32), vectors)
    split_after = 0 if quantized is None else d
    if quantized is not None:
        odb.set_user_dims(d)
    odb.build(oracle.StdRng(SEED), n_trees=trees, split_after=split_after, threads=trees)
    got = ctx.build_trees(seeds, list(range(trees)), trees, split_after=split_after)
    assert got == odb.nodes()
    ctx.load_forest(roots=np.arange(trees, dtype=np.uint32), **forest_arrays(got, oracle.METRICS[metric], vectors.shape[1]))
    return odb


def test_c_abi_rows_equal_the_one_filter_call(shared_ctx):
    # on a load_forest'ed forest: each row of a multi-filter call equals search_batch_filtered with its filter's bitmap, and one
    # all-rows filter equals the unfiltered search
    metric, n, d, trees, count = "euclidean", 3000, 64, 6, 10
    data = oracle.synth_rows(SEED, d, 0, n, 0.5, threads=4)
    load_built_forest(shared_ctx, metric, n, d, trees, data)
    rng = np.random.default_rng(5)
    fl = [np.sort(rng.choice(n, size=300, replace=False)), np.sort(rng.choice(n, size=8, replace=False)), np.arange(100, 700), np.arange(n),
          np.zeros(0, np.uint32), np.array([5, 6, 2999]), np.sort(rng.choice(n, size=30, replace=False))]
    vecs = oracle.synth_rows(SEED, d, n + 3, 40, 0.5)
    for nq in (6, 40):
        q = rng.choice(n, size=nq, replace=False).astype(np.uint32)
        fq = np.array([i % (len(fl) - 1) for i in range(nq)], dtype=np.uint32)   # the last filter is unused
        for sk in (0, 1, 3000):
            for kw, sub in ((dict(query_rows=q), lambda s: dict(query_rows=q[s])), (dict(queries=vecs[:nq]), lambda s: dict(queries=vecs[:nq][s]))):
                got = shared_ctx.search_batch_multi_filtered(count, fl, fq, search_k=sk, **kw)
                assert not got[3].any()
                for f in set(fq.tolist()):
                    sel = np.flatnonzero(fq == f)
                    want = shared_ctx.search_batch_filtered(count, row_bitmap(fl[f], n), search_k=sk, **sub(sel))
                    for j, i in enumerate(sel):
                        same_rows(got, i, want, j)
                allq = shared_ctx.search_batch_multi_filtered(count, [np.arange(n)], np.zeros(nq, np.uint32), search_k=sk, **kw)
                plain = shared_ctx.search_batch(count, search_k=sk, **kw)
                for i in range(nq):
                    same_rows(allq, i, plain, i)


def test_binary_quantized_multi_filters_match_the_oracle(shared_ctx):
    metric, n, d, trees, count = "binary quantized euclidean", 3000, 64, 6, 10
    raw = oracle.synth_rows(SEED, d, 0, n, 0.5, threads=4)
    odb = load_built_forest(shared_ctx, metric, n, d, trees, raw, quantized=oracle.bq_quantize(raw))
    ids = np.arange(n, dtype=np.uint32)
    grid = filter_grid(ids, count)
    rows = [[f for f in F if f < n] for F in grid]
    qv = oracle.bq_quantize(oracle.synth_rows(SEED, d, n + 7, 40, 0.5))
    s0 = shared_ctx.search_stats()
    oracle.set_rerank_dims(d)
    try:
        for nq in (3, 40):
            fq = np.array([i % len(grid) for i in range(nq)], dtype=np.uint32)
            q = np.random.default_rng(nq).choice(n, size=nq, replace=False).astype(np.uint32)
            for sk in (0, 1, 3000, U64_MAX):
                got = shared_ctx.search_batch_multi_filtered(count, rows, fq, query_rows=q, search_k=sk)
                gv = shared_ctx.search_batch_multi_filtered(count, rows, fq, queries=qv[:nq], qhdr0=np.zeros(nq, np.float32), search_k=sk)
                assert not got[3].any() and not gv[3].any()
                for i in range(nq):
                    same(row(got, i), odb.nns_by_item(int(q[i]), count, search_k=sk or None, candidates=grid[fq[i]]))
                    same(row(gv, i), odb.nns_by_vector(qv[i], count, search_k=sk or None, candidates=grid[fq[i]]))
    finally:
        oracle.set_rerank_dims(0)
    assert shared_ctx.search_stats()["failed_queries"] == s0["failed_queries"]


def test_missing_node_surfaces_whatever_the_filter(shared_ctx):
    # node 0 splits into a leaf (node 1) and node 2, which is missing: every query must report MissingKey (status 3)
    n, d = 600, 16
    shared_ctx.stage_items_flat("euclidean", np.arange(n, dtype=np.uint32), oracle.synth_rows(SEED, d, 0, n, 0.5))
    shared_ctx.load_forest(kind=[2, 1, 0], left=[1, 0, 0], right=[2, 0, 0], normal_idx=[0xffffffff, 0, 0], normal_hdr0=[0, 0, 0],
                           desc_off=[0, 0, 0], desc_len=[0, n, 0], normals=np.zeros((0, d), np.float32), desc_rows=np.arange(n, dtype=np.uint32), roots=[0])
    fl = [[], [3, 4, 5], list(range(n))]
    s0 = shared_ctx.search_stats()
    for nq in (2, 20):
        _, _, _, status = shared_ctx.search_batch_multi_filtered(5, fl, [i % 3 for i in range(nq)], query_rows=list(range(nq)), search_k=U64_MAX)
        assert status.tolist() == [3] * nq
    assert shared_ctx.search_stats()["failed_queries"] == s0["failed_queries"] + 22


def test_host_walk_takes_per_query_filters(shared_ctx):
    # ARROY_B200_HOST_WALK=1 and count > 2048 walk on the host, each query with its own filter
    n, d, trees, nq = 3000, 24, 8, 8
    r, odb, ids = build_pair(shared_ctx, "euclidean", n, d, trees)
    grid = filter_grid(ids, 10)
    fq = [i % len(grid) for i in range(nq)]
    items = np.random.default_rng(2).choice(n, size=nq, replace=False)
    for count, env in ((10, True), (2100, False)):
        if env:
            os.environ["ARROY_B200_HOST_WALK"] = "1"
        try:
            got = r.nns_batch_by_item(items, count, filters=grid, filter_of_query=fq)
        finally:
            os.environ.pop("ARROY_B200_HOST_WALK", None)
        for i in range(nq):
            same(row(got, i), odb.nns_by_item(int(items[i]), count, candidates=grid[fq[i]]))


def test_argument_errors_leave_the_context_usable(shared_ctx):
    n, d, count = 2000, 32, 5
    data = oracle.synth_rows(SEED, d, 0, n, 0.5, threads=4)
    load_built_forest(shared_ctx, "euclidean", n, d, 4, data)
    q = np.array([1, 2, 3], dtype=np.uint32)
    good = shared_ctx.search_batch_multi_filtered(count, [[1, 5, 9], np.arange(100)], [0, 1, 1], query_rows=q)
    assert not good[3].any()

    def rejected(fn):
        with pytest.raises(ab.ArroyB200Error) as e:
            fn()
        assert e.value.code == ERR_INVALID
        again = shared_ctx.search_batch_multi_filtered(count, [[1, 5, 9], np.arange(100)], [0, 1, 1], query_rows=q)
        for i in range(3):
            same_rows(again, i, good, i)

    rejected(lambda: shared_ctx.search_batch_multi_filtered(count, [[1, 2]], [0, 1, 0], query_rows=q))        # query_filter >= n_filters
    rejected(lambda: shared_ctx.search_batch_multi_filtered(count, [], [0, 0, 0], query_rows=q))              # no filters
    rejected(lambda: shared_ctx.search_batch_multi_filtered(count, [[1, n]], [0, 0, 0], query_rows=q))        # row >= n
    rejected(lambda: shared_ctx.search_batch_multi_filtered(count, [[4, 3]], [0, 0, 0], query_rows=q))        # descending
    rejected(lambda: shared_ctx.search_batch_multi_filtered(count, [[3], [4, 4]], [0, 1, 0], query_rows=q))   # duplicate

    def bad_offsets():   # offsets 0, 3, 1: filter 1 would end before it starts
        offs = np.array([0, 3, 1], dtype=np.uint64)
        rows = np.array([1, 2, 3], dtype=np.uint32)
        fq = np.zeros(3, dtype=np.uint32)
        out_rows, out_dist = np.empty((3, count), np.uint32), np.empty((3, count), np.float32)
        out_len, st = np.zeros(3, np.uint32), np.zeros(3, np.int32)
        shared_ctx._ck(shared_ctx.lib.arroy_b200_search_batch_multi_filtered(shared_ctx.h, 3, q.ctypes.data_as(_u32p), None, None, count, 0, 2,
                                                                             offs.ctypes.data_as(_u64p), rows.ctypes.data_as(_u32p), fq.ctypes.data_as(_u32p),
                                                                             out_rows.ctypes.data_as(_u32p), out_dist.ctypes.data_as(ctypes.POINTER(ctypes.c_float)),
                                                                             out_len.ctypes.data_as(_u32p), st.ctypes.data_as(ctypes.POINTER(ctypes.c_int32))))
    rejected(bad_offsets)
    # the Reader checks its own arguments
    r, _, ids = build_pair(shared_ctx, "euclidean", 500, 8, 2)
    with pytest.raises(ab.ArroyError):
        r.nns_batch_by_item([1, 2], 5, filters=[[1]], filter_of_query=[0, 3])
    with pytest.raises(ValueError):
        r.nns_batch_by_item([1, 2], 5, candidates=[1], filters=[[1]], filter_of_query=[0, 0])
    got = r.nns_batch_by_item([1, 2], 5, filters=[[1, 2, 3]], filter_of_query=[0, 0])
    assert got[2].tolist() == [3, 3]
