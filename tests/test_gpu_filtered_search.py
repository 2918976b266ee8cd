"""Filtered queries (QueryBuilder::candidates, src/reader.rs:110-123, :350-357) on the device: the filter-aware forest walks
(walk1_kernel / walk_kernel with FILTER), the small-filter shortcut and arroy_b200_search_batch_filtered, against the oracle
(ids and float32 bytes) and against the host walk."""
import ctypes
import os
import re

import numpy as np
import pytest

import arroy_b200 as ab
import oracle
from arroy_b200._capi import row_bitmap
from helpers import golden

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


def make_env(ctx):
    e = ab.Env(0)
    e._ctx = ctx
    ctx.envs.append(e)
    return e


def build_pair(ctx, metric, n, d, trees, centre=0.5, ids=None):
    data = oracle.synth_rows(SEED, d, 0, n, centre, threads=8)
    ids = np.arange(n, dtype=np.uint32) if ids is None else ids
    odb = oracle.Db(metric, d)
    odb.set_items(ids, data)
    odb.build(oracle.StdRng(SEED), n_trees=trees, threads=8)
    env = make_env(ctx)
    w = ab.Writer(env, 0, d, metric)
    w.add_items(ids, data)
    w.builder(ab.StdRng.from_seed(SEED)).n_trees(trees).build()
    return env, ab.Reader.open(env, 0, metric), odb, data, ids


def filters(ids, count):
    """The filter grid: all items, 50 %, 5 %, 0.5 %, exactly `count` items, fewer than `count`, one item, empty, only ids
    outside the index, ids mixed in and out."""
    rng = np.random.default_rng(7)
    n = ids.size
    pick = lambda m: np.sort(rng.choice(ids, size=m, replace=False)).tolist()
    outside = (int(ids.max()) + 1 + np.arange(50)).tolist()
    return {
        "all": ids.tolist(), "50%": pick(n // 2), "5%": pick(n // 20), "0.5%": pick(max(1, n // 200)),
        "count": pick(count), "fewer": pick(count // 2), "one": pick(1), "empty": [],
        "outside": outside, "mixed": sorted(pick(30) + outside[:20]),
    }


def same(got, want):
    assert [g[0] for g in got] == [w[0] for w in want]
    assert np.array([g[1] for g in got], dtype=np.float32).tobytes() == np.array([w[1] for w in want], dtype=np.float32).tobytes()


def test_reference_filter_goldens_through_the_device(shared_ctx):  # src/tests/reader.rs:194-227
    env = make_env(shared_ctx)
    w = ab.Writer(env, 0, 2, "euclidean")
    for i in range(100):
        w.add_item(i, [0.0, float(i)])
    w.builder(ab.StdRng.from_seed(SEED)).n_trees(50).build()
    r = ab.Reader.open(env, 0, "euclidean")
    q = golden()["reader_inline"]
    s0 = shared_ctx.search_stats()
    assert r.nns(5).candidates(range(0, 2)).by_item(0) == [tuple(x) for x in q["216"]]
    assert r.nns(5).candidates(range(98, 1000)).by_item(0) == [tuple(x) for x in q["223"]]
    s1 = shared_ctx.search_stats()
    assert s1["filtered_queries"] == s0["filtered_queries"] + 2
    assert s1["failed_queries"] == s0["failed_queries"]


@pytest.mark.parametrize("metric,d", [("euclidean", 24), ("cosine", 48), ("dot-product", 96), ("manhattan", 128)])
def test_filtered_queries_match_the_oracle(shared_ctx, metric, d):
    n, trees, count = 3000, 8, 10
    env, r, odb, data, ids = build_pair(shared_ctx, metric, n, d, trees)
    qv = oracle.synth_rows(SEED, d, n + 11, 1, 0.5)[0]
    s0 = shared_ctx.search_stats()
    for name, F in filters(ids, count).items():
        inside = set(F)
        outside_item = next(i for i in range(n) if i not in inside) if len(inside & set(range(n))) < n else None
        items = [7, 1500] + ([outside_item] if outside_item is not None else [])
        for sk in (None, 1, 3000, U64_MAX):
            for it in items:
                same(r.nns(count).search_k(sk).candidates(F).by_item(it) if sk else r.nns(count).candidates(F).by_item(it),
                     odb.nns_by_item(it, count, search_k=sk, candidates=F))
            same(r.nns(count).search_k(sk).candidates(F).by_vector(qv) if sk else r.nns(count).candidates(F).by_vector(qv),
                 odb.nns_by_vector(qv, count, search_k=sk, candidates=F))
        same(r.nns(count).oversampling(3).candidates(F).by_item(7), odb.nns_by_item(7, count, oversampling=3, candidates=F))
    s1 = shared_ctx.search_stats()
    assert s1["failed_queries"] == s0["failed_queries"]
    assert s1["shortcut_queries"] > s0["shortcut_queries"]          # the small filters skip the walk
    assert s1["filtered_queries"] - s1["shortcut_queries"] > s0["filtered_queries"] - s0["shortcut_queries"]


@pytest.mark.parametrize("metric", ["euclidean", "cosine"])
def test_candidate_sets_equal_the_oracle(shared_ctx, metric):
    # with count >= the number of candidates, the result is the whole candidate set: this checks what pruning and the shortcut
    # collect, not only the top of it
    n, d, trees = 4000, 32, 10
    env, r, odb, data, ids = build_pair(shared_ctx, metric, n, d, trees)
    count = 2048
    for name, F in filters(ids, 40).items():
        for sk in (None, 50, 600, U64_MAX):
            for it in (3, 2222):
                want, cand = odb.nns_by_item(it, count, search_k=sk, candidates=F, want_candidates=True)
                if cand.size > count:
                    continue
                got = r.nns(count).search_k(sk).candidates(F).by_item(it) if sk else r.nns(count).candidates(F).by_item(it)
                assert sorted(g[0] for g in got) == sorted(cand.tolist()), (name, sk, it)
                same(got, want)


@pytest.mark.parametrize("nq", [5, 40])   # 5: walk1_kernel, 40: walk_kernel
def test_batched_filtered_queries(shared_ctx, nq):
    n, d, trees, count = 5000, 40, 12, 10
    env, r, odb, data, ids = build_pair(shared_ctx, "cosine", n, d, trees, ids=np.arange(0, 2 * 5000, 2, dtype=np.uint32))   # rows != ids
    rng = np.random.default_rng(3)
    items = rng.choice(ids, size=nq, replace=False)
    vecs = oracle.synth_rows(SEED, d, n + 100, nq, 0.5)
    for F in (np.sort(rng.choice(ids, size=n // 10, replace=False)).tolist(), np.sort(rng.choice(ids, size=n // 100, replace=False)).tolist(), [],
              list(range(1000, 1400))):
        for sk in (None, 3000):
            bi, bd, bl, _ = r.nns_batch_by_item(items, count, search_k=sk, candidates=F)
            vi, vd, vl, _ = r.nns_batch_by_vector(vecs, count, search_k=sk, candidates=F)
            for i in range(nq):
                single = r.nns(count).search_k(sk).candidates(F).by_item(int(items[i])) if sk else r.nns(count).candidates(F).by_item(int(items[i]))
                want = odb.nns_by_item(int(items[i]), count, search_k=sk, candidates=F)
                same(single, want)
                same(list(zip(bi[i, :bl[i]].tolist(), bd[i, :bl[i]].tolist())), want)
                wv = odb.nns_by_vector(vecs[i], count, search_k=sk, candidates=F)
                same(list(zip(vi[i, :vl[i]].tolist(), vd[i, :vl[i]].tolist())), wv)
            os.environ["ARROY_B200_HOST_WALK"] = "1"
            try:
                hi, hd, hl, _ = r.nns_batch_by_item(items, count, search_k=sk, candidates=F)
                hvi, hvd, hvl, _ = r.nns_batch_by_vector(vecs, count, search_k=sk, candidates=F)
            finally:
                os.environ.pop("ARROY_B200_HOST_WALK")
            assert hl.tolist() == bl.tolist() and hvl.tolist() == vl.tolist()
            for i in range(nq):
                assert hi[i, :hl[i]].tobytes() == bi[i, :bl[i]].tobytes() and hd[i, :hl[i]].tobytes() == bd[i, :bl[i]].tobytes()
                assert hvi[i, :hvl[i]].tobytes() == vi[i, :vl[i]].tobytes() and hvd[i, :hvl[i]].tobytes() == vd[i, :vl[i]].tobytes()


def test_large_frontier_past_the_shared_memory_slots(shared_ctx, capfd):
    # 50 000 x 32, 50 trees, a 0.2 % filter (100 items, 5000 filtered rows in the forest), query 17, search_k = 2000. A replay of
    # the pruned walk on the oracle's forest pops ~1 954 leaves with filtered rows (under walk1_kernel's 2048-entry leaf queue)
    # and its frontier peaks at 1 383 entries, past the 1024 shared-memory slots: the entries beyond them live in the query's
    # global spill slot. The ARROY_B200_WALK1_DEBUG line is printed only by a walk1_kernel query that completed, so it shows that
    # walk1_kernel (not the batched walk_kernel after a fallback) produced the result, and how large its frontier grew.
    n, d, trees, count, sk = 50_000, 32, 50, 10, 2000
    env, r, odb, data, ids = build_pair(shared_ctx, "euclidean", n, d, trees)
    F = np.sort(np.random.default_rng(11).choice(ids, size=n // 500, replace=False)).tolist()
    s0 = shared_ctx.search_stats()
    os.environ["ARROY_B200_WALK1_DEBUG"] = "1"
    try:
        capfd.readouterr()
        got = r.nns(count).search_k(sk).candidates(F).by_item(17)
        ctypes.CDLL(None).fflush(None)   # the device printf lands in the C stdout buffer
        out = capfd.readouterr().out
    finally:
        os.environ.pop("ARROY_B200_WALK1_DEBUG")
    fronts = [int(x) for x in re.findall(r"largest frontier (\d+)", out)]
    assert len(fronts) == 1 and fronts[0] > 1024, out
    same(got, odb.nns_by_item(17, count, search_k=sk, candidates=F))
    s1 = shared_ctx.search_stats()
    assert s1["failed_queries"] == s0["failed_queries"] and s1["filtered_queries"] == s0["filtered_queries"] + 1


def test_missing_node_still_surfaces_under_a_filter(shared_ctx):
    # node 0 splits into a leaf (node 1) and node 2, which is missing: whatever the filter holds, the walk must reach node 2
    # and report MissingKey (status 3), as the reference does
    n, d = 600, 16
    data = oracle.synth_rows(SEED, d, 0, n, 0.5)
    shared_ctx.stage_items_flat("euclidean", np.arange(n, dtype=np.uint32), data)
    shared_ctx.load_forest(kind=[2, 1, 0], left=[1, 0, 0], right=[2, 0, 0], normal_idx=[0xffffffff, 0, 0], normal_hdr0=[0, 0, 0],
                           desc_off=[0, 0, 0], desc_len=[0, n, 0], normals=np.zeros((0, d), np.float32), desc_rows=np.arange(n, dtype=np.uint32), roots=[0])
    s0 = shared_ctx.search_stats()
    for rows in ([], [3, 4, 5], list(range(n))):
        _, _, _, status = shared_ctx.search_batch_filtered(5, row_bitmap(rows, n), query_rows=[0, 9], search_k=U64_MAX)
        assert status.tolist() == [3, 3], rows
        _, _, _, status = shared_ctx.search_batch_filtered(5, row_bitmap(rows, n), query_rows=list(range(20)), search_k=U64_MAX)
        assert status.tolist() == [3] * 20, rows
    s1 = shared_ctx.search_stats()
    assert s1["failed_queries"] == s0["failed_queries"] + 3 * 22


def decode_node(b, metric, d):
    """oracle.decode_node, plus the binary-quantized normals: a bit string of 64-bit words, bit i of word w = element 64 w + i,
    set = +1, clear = -1 (d = the padded length)."""
    if metric < oracle.BQ_EUCLIDEAN or b[0] != 2 or len(b) == 9:
        return oracle.decode_node(b, metric, d)
    bits = np.unpackbits(np.frombuffer(b[13:], dtype=np.uint8), bitorder="little")
    assert bits.size == d
    return {"kind": "split", "left": int.from_bytes(b[1:5], "big"), "right": int.from_bytes(b[5:9], "big"),
            "header": np.frombuffer(b[9:13], dtype=np.float32).copy(), "normal": np.where(bits == 1, 1.0, -1.0).astype(np.float32)}


def forest_arrays(nodes, metric, d):
    """{node id: NodeCodec bytes} -> the arrays arroy_b200_load_forest takes (rows == item ids here)."""
    nn = max(nodes) + 1
    kind = np.zeros(nn, np.uint8)
    left, right, nidx = np.zeros(nn, np.uint32), np.zeros(nn, np.uint32), np.full(nn, 0xffffffff, np.uint32)
    nh0, doff, dlen = np.zeros(nn, np.float32), np.zeros(nn, np.uint32), np.zeros(nn, np.uint32)
    normals, desc = [], []
    n_desc = 0
    for i, b in nodes.items():
        nd = decode_node(b, metric, d)
        if nd["kind"] == "descendants":
            kind[i] = 1
            doff[i], dlen[i] = n_desc, len(nd["descendants"])
            desc.append(np.asarray(nd["descendants"], dtype=np.uint32))
            n_desc += dlen[i]
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


def test_identity_filter_and_c_abi_filters(shared_ctx):
    # through the C ABI on a forest loaded with load_forest: an all-ones bitmap equals the unfiltered search, and filtered
    # searches equal the oracle's
    metric, n, d, trees, count = "euclidean", 3000, 64, 6, 10
    data = oracle.synth_rows(SEED, d, 0, n, 0.5, threads=4)
    ids = np.arange(n, dtype=np.uint32)
    shared_ctx.stage_items_flat(metric, ids, data)
    user = oracle.StdRng(SEED)
    r1 = oracle.StdRng(user.gen_seed())
    seeds = [r1.gen_seed() for _ in range(trees)]
    odb = oracle.Db(metric, d)
    odb.set_items(ids, data)
    odb.build(oracle.StdRng(SEED), n_trees=trees, threads=trees)
    got = shared_ctx.build_trees(seeds, list(range(trees)), trees)
    assert got == odb.nodes()
    shared_ctx.load_forest(roots=np.arange(trees, dtype=np.uint32), **forest_arrays(got, oracle.METRICS[metric], d))
    q = np.array([0, 5, 77, 2999], dtype=np.uint32)
    for nq_rows in (q, np.arange(40, dtype=np.uint32)):
        for sk in (0, 500):
            a = shared_ctx.search_batch(count, query_rows=nq_rows, search_k=sk)
            b = shared_ctx.search_batch_filtered(count, np.full((n + 31) // 32, 0xffffffff, np.uint32), query_rows=nq_rows, search_k=sk)
            for i in range(nq_rows.size):
                assert a[2][i] == b[2][i] and a[3][i] == b[3][i] == 0
                assert a[0][i, :a[2][i]].tobytes() == b[0][i, :b[2][i]].tobytes() and a[1][i, :a[2][i]].tobytes() == b[1][i, :b[2][i]].tobytes()
    rng = np.random.default_rng(5)
    for F in (np.sort(rng.choice(n, size=300, replace=False)), np.sort(rng.choice(n, size=8, replace=False)), np.arange(100, 700)):
        for sk in (0, 1, 3000):
            out_rows, out_dist, out_len, status = shared_ctx.search_batch_filtered(count, row_bitmap(F, n), query_rows=q, search_k=sk)
            assert not status.any()
            for i, it in enumerate(q):
                want = odb.nns_by_item(int(it), count, search_k=sk or None, candidates=F.tolist())
                same(list(zip(out_rows[i, :out_len[i]].tolist(), out_dist[i, :out_len[i]].tolist())), want)


def test_binary_quantized_filtered_queries_match_the_oracle(shared_ctx):
    # binary quantized euclidean at d = 64 through the C ABI (the Writer / Reader mirror covers the four float metrics), over the
    # filter grid and the search_k values of the float test: by_item (query rows, one of them outside the filter) and by_vector
    # (+-1 query vectors; their header is 0 for this metric), single queries and batches of 40
    metric, n, d, trees, count = "binary quantized euclidean", 3000, 64, 6, 10
    m = oracle.METRICS[metric]
    raw = oracle.synth_rows(SEED, d, 0, n, 0.5, threads=4)
    pm1 = oracle.bq_quantize(raw)
    ids = np.arange(n, dtype=np.uint32)
    shared_ctx.stage_items_flat(metric, ids, raw)
    user = oracle.StdRng(SEED)
    r1 = oracle.StdRng(user.gen_seed())
    seeds = [r1.gen_seed() for _ in range(trees)]
    odb = oracle.Db(metric, pm1.shape[1])
    odb.set_items(ids, pm1)
    odb.set_user_dims(d)
    odb.build(oracle.StdRng(SEED), n_trees=trees, split_after=d, threads=trees)
    got = shared_ctx.build_trees(seeds, list(range(trees)), trees, split_after=d)
    assert got == odb.nodes()
    shared_ctx.load_forest(roots=np.arange(trees, dtype=np.uint32), **forest_arrays(got, m, pm1.shape[1]))
    qv = oracle.bq_quantize(oracle.synth_rows(SEED, d, n + 7, 40, 0.5))
    s0 = shared_ctx.search_stats()
    oracle.set_rerank_dims(d)
    try:
        for name, F in filters(ids, count).items():
            inside = set(F)
            outside_item = next((i for i in range(n) if i not in inside), None)
            items = np.array([7, 1500] + ([outside_item] if outside_item is not None else []), dtype=np.uint32)
            bits = row_bitmap([f for f in F if f < n], n)
            for sk in (0, 1, 3000, U64_MAX):
                for rows_q in (items, np.arange(40, dtype=np.uint32)):
                    out_rows, out_dist, out_len, status = shared_ctx.search_batch_filtered(count, bits, query_rows=rows_q, search_k=sk)
                    assert not status.any(), (name, sk)
                    for i, it in enumerate(rows_q):
                        want = odb.nns_by_item(int(it), count, search_k=sk or None, candidates=F)
                        same(list(zip(out_rows[i, :out_len[i]].tolist(), out_dist[i, :out_len[i]].tolist())), want)
                for nq in (1, 40):
                    out_rows, out_dist, out_len, status = shared_ctx.search_batch_filtered(count, bits, queries=qv[:nq], qhdr0=np.zeros(nq, np.float32), search_k=sk)
                    assert not status.any(), (name, sk)
                    for i in range(nq):
                        want = odb.nns_by_vector(qv[i], count, search_k=sk or None, candidates=F)
                        same(list(zip(out_rows[i, :out_len[i]].tolist(), out_dist[i, :out_len[i]].tolist())), want)
    finally:
        oracle.set_rerank_dims(0)
    assert shared_ctx.search_stats()["failed_queries"] == s0["failed_queries"]
