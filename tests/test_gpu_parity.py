"""GPU parity tests (run with -m gpu on an H100): the CUDA path, called through the C ABI,
against the CPU oracle on the same seeded inputs. Bit-exact for ids, sides, margins, node bytes;
distances bit-exact too (the tolerance the north star allows is 1e-5 relative — we assert 0)."""
import numpy as np
import pytest

import arroy_b200
import oracle
from helpers import check_dump, golden

pytestmark = pytest.mark.gpu

SEED = bytes([42] * 32)
MET = ["euclidean", "cosine", "dot-product", "manhattan"]


@pytest.fixture(scope="module")
def ctx():
    c = arroy_b200.Context(0)
    yield c
    c.close()


def synth(n, d, centre=0.5, seed=SEED, row0=0):
    return oracle.synth_rows(seed, d, row0, n, centre, threads=4)


def headers_for(metric, data):
    m = oracle.METRICS[metric]
    if m == oracle.COSINE:
        return np.array([oracle.new_header(m, v)[0] for v in data], dtype=np.float32), None
    if m == oracle.DOT_PRODUCT:
        return oracle.dot_preprocess(data)
    return np.zeros(len(data), dtype=np.float32), None


@pytest.mark.parametrize("d", [3, 15, 16, 30, 31, 32, 33, 64, 100, 768, 795, 1536])
@pytest.mark.parametrize("metric", MET)
def test_side_batch_margins_bit_exact(ctx, metric, d):
    n = 700
    data = synth(n, d)
    ids = np.arange(n, dtype=np.uint32)
    h0, h1 = headers_for(metric, data)
    ctx.stage_items_flat(metric, ids, data, h0, h1)
    if metric == "dot-product":
        e, nn = ctx.dot_preprocess()
        assert e.tobytes() == h0.tobytes() and nn.tobytes() == h1.tobytes()
    r = np.random.default_rng(d)
    normal = (r.standard_normal(d) / np.sqrt(d)).astype(np.float32)
    hdr = (float(np.float32(r.standard_normal() * 0.1)), 0.0)
    rows = np.sort(r.choice(n, size=n - 37, replace=False)).astype(np.uint32)
    side, mg = ctx.side_batch(normal, hdr, rows)
    wside, wmg = oracle.side_batch(oracle.METRICS[metric], normal, hdr, data, h0, h1, rows)
    assert mg.tobytes() == wmg.tobytes(), np.nonzero(mg.view(np.uint32) != wmg.view(np.uint32))[0][:10]
    assert side.tobytes() == wside.tobytes()


def test_side_of_signed_zero(ctx):
    # +0.0 margin => Right, -0.0 => Left (src/distance/mod.rs:103-110)
    d = 64
    data = np.zeros((4, d), dtype=np.float32)
    data[1, 0] = 1.0
    data[2, 0] = -1.0
    ctx.stage_items_flat("cosine", np.arange(4, dtype=np.uint32), data)
    normal = np.zeros(d, dtype=np.float32)
    normal[0] = -0.0
    side, mg = ctx.side_batch(normal, (0.0, 0.0), np.arange(4, dtype=np.uint32))
    wside, wmg = oracle.side_batch(oracle.COSINE, normal, (0.0, 0.0), data, np.zeros(4, np.float32), None, np.arange(4, dtype=np.uint32))
    assert mg.tobytes() == wmg.tobytes() and side.tolist() == wside.tolist()


@pytest.mark.parametrize("metric,d", [("euclidean", 30), ("euclidean", 64), ("cosine", 3), ("cosine", 100), ("cosine", 768),
                                      ("dot-product", 48), ("dot-product", 768), ("manhattan", 40), ("euclidean", 1536)])
def test_create_split_matches_and_consumes_rng_identically(ctx, metric, d):
    n = 900
    data = synth(n, d, centre=0.5 if metric != "euclidean" else 0.0)
    ids = np.arange(n, dtype=np.uint32)
    h0, h1 = headers_for(metric, data)
    ctx.stage_items_flat(metric, ids, data, h0, h1)
    m = oracle.METRICS[metric]
    for trial in range(6):
        seed = bytes([(7 * trial + 3) % 256] * 32)
        r = np.random.default_rng(trial)
        rows = np.sort(r.choice(n, size=int(r.integers(2, n)), replace=False)).astype(np.uint32)
        rng = oracle.StdRng(seed)
        start_words = int(r.integers(0, 200))
        for _ in range(start_words):
            rng.next_u32()
        probe = rng.clone()
        want_n, want_h = oracle.create_split(m, rng, data, h0, h1, rows)
        key = np.frombuffer(seed, dtype="<u4")
        got_n, got_h, pos = ctx.create_split(key, start_words, rows)
        assert got_n.tobytes() == want_n.tobytes(), (trial, np.nonzero(got_n != want_n)[0][:5])
        assert np.float32(got_h[0]).tobytes() == np.float32(want_h[0]).tobytes() and got_h[1] == want_h[1]
        # same number of words consumed: the next draw of the oracle rng equals word `pos` of the stream
        for _ in range(pos - start_words):
            probe.next_u32()
        assert probe.next_u32() == rng.next_u32()


def derive_seeds(user_rng, n_trees):
    rng1 = oracle.StdRng(user_rng.gen_seed())         # src/writer.rs:575
    return [rng1.gen_seed() for _ in range(n_trees)]  # src/writer.rs:795


def build_both(ctx, metric, data, n_trees, split_after=None, user_seed=SEED, ids=None):
    n, d = data.shape
    ids = np.arange(n, dtype=np.uint32) if ids is None else np.asarray(ids, dtype=np.uint32)
    odb = oracle.Db(metric, d)
    odb.set_items(ids, data)
    rng = oracle.StdRng(user_seed)
    user = rng.clone()
    odb.build(rng, n_trees=n_trees, split_after=split_after, threads=8)
    ctx.stage_items_flat(metric, ids, data)
    if metric == "dot-product":
        ctx.dot_preprocess()
    seeds = derive_seeds(user, n_trees)
    got = ctx.build_trees(seeds, list(range(n_trees)), n_trees, split_after or 0)
    return odb, got


def assert_same_forest(odb, got):
    want = odb.nodes()
    assert sorted(got.keys()) == sorted(want.keys()), (len(got), len(want))
    bad = [k for k in sorted(want) if want[k] != got[k]]
    assert not bad, "node bytes differ for %d nodes, first ids %s" % (len(bad), bad[:8])


@pytest.mark.parametrize("metric,n,d,trees,split_after", [
    ("euclidean", 100, 30, 10, None),
    ("euclidean", 3000, 64, 10, None),
    ("cosine", 5000, 96, 6, None),
    ("cosine", 4000, 768, 3, 200),
    ("dot-product", 5000, 128, 5, None),
    ("manhattan", 2000, 40, 4, None),
    ("euclidean", 2500, 33, 7, 20),
    ("cosine", 20000, 64, 8, None),
])
def test_forest_node_bytes_identical(ctx, metric, n, d, trees, split_after):
    data = synth(n, d, centre=0.0 if metric == "euclidean" else 0.5)
    odb, got = build_both(ctx, metric, data, trees, split_after)
    assert_same_forest(odb, got)
    st = ctx.build_stats()
    assert st["scanned_rows"] == odb.scanned_rows


def test_reference_snapshot_lot_of_random_points(ctx):
    # the reference's own golden (100 x 30 Euclidean, 10 trees), straight against the GPU path
    gold = golden()["lot_of_random_points"]
    rng = oracle.StdRng(SEED)
    data = rng.fill_f32(100 * 30).reshape(100, 30)
    ctx.stage_items_flat("euclidean", np.arange(100, dtype=np.uint32), data)
    got = ctx.build_trees(derive_seeds(rng, 10), list(range(10)), 10)
    check_dump(gold, got, list(range(10)), oracle.EUCLIDEAN, 30, oracle.decode_node)


def test_degenerate_data_takes_the_random_split_path(ctx):
    # identical vectors: every split is 100% imbalanced -> randomly_split_children (writer.rs:1220-1227)
    n, d = 600, 32
    data = np.ones((n, d), dtype=np.float32)
    odb, got = build_both(ctx, "euclidean", data, 3, split_after=50)
    assert_same_forest(odb, got)
    assert ctx.build_stats()["random_splits"] > 0


def test_sparse_item_ids_and_large_roaring_containers(ctx):
    n, d = 12000, 32
    data = synth(n, d)
    ids = (np.arange(n, dtype=np.uint64) * 7 + 65530).astype(np.uint32)
    odb, got = build_both(ctx, "cosine", data, 2, split_after=6000, ids=ids)
    assert_same_forest(odb, got)


def test_build_cancel(ctx):
    data = synth(3000, 64)
    ctx.stage_items_flat("cosine", np.arange(3000, dtype=np.uint32), data)
    seeds = derive_seeds(oracle.StdRng(SEED), 4)
    with pytest.raises(arroy_b200.ArroyB200Error) as ei:
        ctx.build_trees(seeds, [0, 1, 2, 3], 4, cancel=lambda: True)
    assert ei.value.code == arroy_b200._capi.ERR_CANCELLED
    assert "cancelled" in ei.value.message


@pytest.mark.parametrize("metric", MET)
@pytest.mark.parametrize("d,n_cand,k", [(30, 500, 10), (64, 3000, 100), (768, 6000, 100), (100, 9000, 1500), (16, 100, 200)])
def test_rerank_ids_and_distances(ctx, metric, d, n_cand, k):
    n = 10000
    data = synth(n, d)
    h0, h1 = headers_for(metric, data)
    ctx.stage_items_flat(metric, np.arange(n, dtype=np.uint32), data, h0, h1)
    m = oracle.METRICS[metric]
    r = np.random.default_rng(d + k)
    rows = np.sort(r.choice(n, size=n_cand, replace=False)).astype(np.uint32)
    q = synth(1, d, row0=n + 5)[0]
    qh = oracle.new_header(m, q)
    wr, wd = oracle.rerank(m, q, qh, data, h0, h1, rows, k)
    gr, gd = ctx.rerank(q, qh, rows, k)
    assert gr.tolist() == wr.tolist()
    assert gd.tobytes() == wd.tobytes()


def test_rerank_ties_nan_and_signed_zero_order(ctx):
    # (OrderedFloat, id) order: NaN greatest, -0 == +0, ties by id (src/reader.rs:390-395)
    n, d = 400, 32
    data = np.zeros((n, d), dtype=np.float32)
    r = np.random.default_rng(0)
    vals = r.integers(-3, 4, size=n).astype(np.float32)  # many exact ties
    data[:, 0] = -vals                                   # dot-product distance = -(q . v) = vals for q = e0
    data[5, 0] = np.nan
    data[77, 0] = np.nan
    data[9, 0] = 0.0
    data[10, 0] = -0.0
    ctx.stage_items_flat("dot-product", np.arange(n, dtype=np.uint32), data, np.zeros(n, np.float32), np.zeros(n, np.float32))
    q = np.zeros(d, dtype=np.float32)
    q[0] = 1.0
    rows = np.arange(n, dtype=np.uint32)
    for k in (1, 7, 150, 400):
        wr, wd = oracle.rerank(oracle.DOT_PRODUCT, q, (0, 0), data, np.zeros(n, np.float32), np.zeros(n, np.float32), rows, k)
        gr, gd = ctx.rerank(q, (0, 0), rows, k)
        assert gr.tolist() == wr.tolist()
        assert np.array_equal(gd, wd, equal_nan=True)


def test_rerank_batch_ragged_and_empty(ctx):
    n, d, k = 5000, 96, 20
    data = synth(n, d)
    h0, _ = headers_for("cosine", data)
    ctx.stage_items_flat("cosine", np.arange(n, dtype=np.uint32), data, h0)
    r = np.random.default_rng(3)
    sizes = [0, 5, 1200, 20, 4097, 1]
    lists = [np.sort(r.choice(n, size=s, replace=False)).astype(np.uint32) for s in sizes]
    offs = np.concatenate([[0], np.cumsum(sizes)]).astype(np.uint64)
    qs = synth(len(sizes), d, row0=n)
    qh0 = np.array([oracle.new_header(oracle.COSINE, q)[0] for q in qs], dtype=np.float32)
    out_rows, out_dist, out_len = ctx.rerank_batch(qs, qh0, np.concatenate(lists), offs, k)
    for i, rows in enumerate(lists):
        wr, wd = oracle.rerank(oracle.COSINE, qs[i], (qh0[i], 0), data, h0, None, rows, k)
        assert out_len[i] == len(wr)
        assert out_rows[i, :len(wr)].tolist() == wr.tolist()
        assert out_dist[i, :len(wr)].tobytes() == wd.tobytes()


@pytest.mark.parametrize("metric", MET)
@pytest.mark.parametrize("d,nq,nc,k", [(768, 37, 1500, 100), (100, 16, 333, 10), (64, 5, 40, 50), (30, 9, 200, 7), (1536, 20, 700, 64)])
def test_rerank_shared_matches_per_query_rerank_and_oracle(ctx, metric, d, nq, nc, k):
    # config 5 shape (many queries x one candidate list) on the exact register-tiled kernel
    n = 4000
    data = synth(n, d)
    h0, h1 = headers_for(metric, data)
    ctx.stage_items_flat(metric, np.arange(n, dtype=np.uint32), data, h0, h1)
    m = oracle.METRICS[metric]
    r = np.random.default_rng(nq * 1000 + nc)
    rows = np.sort(r.choice(n, size=nc, replace=False)).astype(np.uint32)
    qs = synth(nq, d, row0=n + 11)
    qh = np.array([oracle.new_header(m, q)[0] for q in qs], dtype=np.float32)
    out_rows, out_dist, out_len = ctx.rerank_shared(qs, qh, rows, k)
    for i in range(nq):
        wr, wd = oracle.rerank(m, qs[i], (qh[i], 0.0), data, h0, h1, rows, k)
        assert out_len[i] == len(wr)
        assert out_rows[i, :len(wr)].tolist() == wr.tolist(), (i,)
        assert out_dist[i, :len(wr)].tobytes() == wd.tobytes()


def test_stage_from_unaligned_leaf_values(ctx):
    # the raw LMDB value layout: [0x00][header][dim x f32], byte aligned only (src/node.rs:224-228)
    n, d = 300, 40
    data = synth(n, d)
    extra, norm = oracle.dot_preprocess(data)
    values = [b"\x00" + np.float32(extra[i]).tobytes() + np.float32(norm[i]).tobytes() + data[i].tobytes() for i in range(n)]
    ctx.stage_items_leaf_values("dot-product", d, np.arange(n, dtype=np.uint32), values)
    g0, g1 = ctx.item_headers()
    assert g0.tobytes() == extra.tobytes() and g1.tobytes() == norm.tobytes()
    normal = synth(1, d, row0=999)[0]
    rows = np.arange(n, dtype=np.uint32)
    side, mg = ctx.side_batch(normal, (0.25, 0.0), rows)
    wside, wmg = oracle.side_batch(oracle.DOT_PRODUCT, normal, (0.25, 0.0), data, extra, norm, rows)
    assert mg.tobytes() == wmg.tobytes() and side.tobytes() == wside.tobytes()


def test_synth_device_matches_oracle_stream(ctx):
    import torch
    n, d = 1000, 96
    t = torch.empty((n, d), dtype=torch.float32, device="cuda:0")
    ctx.synth_device(SEED, d, 17, n, 0.5, t.data_ptr())
    torch.cuda.synchronize()
    want = oracle.synth_rows(SEED, d, 17, n, 0.5)
    assert t.cpu().numpy().tobytes() == want.tobytes()


def test_invalid_arguments_are_reported(ctx):
    data = synth(100, 32)
    ctx.stage_items_flat("cosine", np.arange(100, dtype=np.uint32), data)
    with pytest.raises(arroy_b200.ArroyB200Error) as ei:
        ctx.side_batch(np.zeros(32, np.float32), (0, 0), np.array([5, 100], dtype=np.uint32))
    assert ei.value.code == arroy_b200._capi.ERR_INVALID
    with pytest.raises(arroy_b200.ArroyB200Error) as ei:
        ctx.build_trees([SEED], [0], 1, split_after=100)  # n <= split_after: single-leaf case is the caller's
    assert ei.value.code == arroy_b200._capi.ERR_INVALID
    fresh = arroy_b200.Context(0)
    with pytest.raises(arroy_b200.ArroyB200Error) as ei:
        fresh.side_batch(np.zeros(32, np.float32), (0, 0), np.array([0], dtype=np.uint32))
    assert ei.value.code == arroy_b200._capi.ERR_NOT_STAGED
    fresh.close()
