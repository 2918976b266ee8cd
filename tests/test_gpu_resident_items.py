"""Items that stay resident on the device across an update (arroy_b200_stage_items_delta, csrc/restage.cuh) and across the
Writers and Readers of one Env (the host mirror's residency record): rows and headers byte for byte against a full staging,
the byte counters, every fallback, the derived state, and builds / queries through the host mirror against the oracle."""
import numpy as np
import pytest

import arroy_b200 as ab
import oracle

pytestmark = pytest.mark.gpu
SEED = bytes([42] * 32)
SCRATCH_BYTES = 192 << 20   # one window of the in-place move (arroy_b200.cu RESTAGE_SCRATCH_BYTES)
PIECE_BYTES = 64 << 10


@pytest.fixture(scope="module")
def ctx():
    c = ab.Context(0)
    # a first staging of 64 MB: the item buffer only grows, so the small indexes below all fit its capacity whatever the order
    # the tests run in (growth past the capacity is test_fallbacks_stage_in_full's, on a context of its own)
    c.stage_items_flat("euclidean", np.arange(16384, dtype=np.uint32), np.zeros((16384, 1024), np.float32))
    yield c
    c.close()


@pytest.fixture(scope="module")
def fresh():
    c = ab.Context(0)
    yield c
    c.close()


def row_bytes(metric, d):
    m = ab.METRICS[metric] if isinstance(metric, str) else metric
    return 16 * ((d + 127) // 128) if m >= 4 else 4 * ((d + 31) // 32 * 32)


def leaf_len(metric, d):
    m = ab.METRICS[metric] if isinstance(metric, str) else metric
    return 1 + (8 if m == 2 else 4) + ((d + 63) // 64 * 8 if m >= 4 else 4 * d)


class Items:
    """id -> stored Leaf value, the values in one pool buffer ([0x00][header][vector], random bytes)."""

    def __init__(self, metric, d, pool_rows, seed):
        self.metric, self.d = metric, d
        rng = np.random.default_rng(seed)
        self.pool = np.frombuffer(rng.bytes(pool_rows * leaf_len(metric, d)), np.uint8).reshape(pool_rows, -1).copy()
        self.pool[:, 0] = 0
        self.next_pool = 0
        self.at = {}

    def put(self, ids):
        for i in ids:
            self.at[int(i)] = self.next_pool
            self.next_pool += 1
        assert self.next_pool <= self.pool.shape[0]

    def delete(self, ids):
        for i in ids:
            del self.at[int(i)]

    def ids(self):
        return np.array(sorted(self.at), dtype=np.uint32)

    def ptrs(self):
        rows = np.array([self.at[int(i)] for i in self.ids()], dtype=np.uint64)
        return np.uint64(self.pool.ctypes.data) + rows * np.uint64(self.pool.shape[1])

    def stage_full(self, c):
        c.stage_items_ptrs(self.metric, self.d, self.ids(), self.ptrs())

    def stage_delta(self, c, changed):
        c.stage_items_delta(self.metric, self.d, self.ids(), self.ptrs(), np.array(sorted(set(int(i) for i in changed)), dtype=np.uint32))


def n_pieces(src, rb):
    """pieces of the copy plan: runs of consecutive rows that move or are uploaded, cut at 64 KB and at the window size"""
    per, win = max(1, PIECE_BYTES // rb), max(1, SCRATCH_BYTES // rb)

    def count(runs):
        n, used = 0, 0
        for ln in runs:
            while ln:
                if used == win:
                    used = 0
                take = min(ln, per, win - used)
                n, used, ln = n + 1, used + take, ln - take
        return n

    src = np.asarray(src)
    r = np.arange(src.size)
    down, up, upl = [], [], []
    i = 0
    while i < src.size:
        e = i + 1
        if src[i] < 0:
            while e < src.size and src[e] < 0:
                e += 1
            upl.append(e - i)
        else:
            while e < src.size and src[e] == src[e - 1] + 1:
                e += 1
            if src[i] > r[i]:
                down.append(e - i)
            elif src[i] < r[i]:
                up.append(e - i)
        i = e
    return count(down + up[::-1]) + count(upl)


def same_as_full_staging(ctx, fresh, items):
    items.stage_full(fresh)
    assert ctx.n == fresh.n
    assert ctx.read_items().tobytes() == fresh.read_items().tobytes()
    a, b = ctx.item_headers(), fresh.item_headers()
    assert a[0].tobytes() == b[0].tobytes() and a[1].tobytes() == b[1].tobytes()


def check_delta(ctx, fresh, items, old_ids, changed, moved=None):
    """stage the current items as a delta over old_ids and check stats, byte counters, rows and headers"""
    rb = row_bytes(items.metric, items.d)
    src, n_upload = ab.stage_delta_plan(old_ids, items.ids(), np.array(sorted(set(int(i) for i in changed)), dtype=np.uint32))
    n = items.ids().size
    h0 = ctx.counters()["h2d_bytes"]
    e0 = ctx.epochs()[0]
    items.stage_delta(ctx, changed)
    st = ctx.stage_stats()
    assert st["delta"] == 1 and st["uploaded_rows"] == n_upload
    assert st["moved_rows"] == int(np.sum((src >= 0) & (src != np.arange(n))))
    if moved is not None:
        assert st["moved_rows"] == moved
    assert st["h2d_bytes"] == n_upload * rb + 8 * n + 16 * n_pieces(src, rb)
    assert ctx.counters()["h2d_bytes"] - h0 == st["h2d_bytes"]
    assert ctx.epochs()[0] not in (0, e0)
    same_as_full_staging(ctx, fresh, items)
    return st


BASE, STEP = 100000, 4


def scenarios(n0):
    """name -> (deleted ids, replaced ids, inserted ids) over the ids BASE + STEP * [0, n0)"""
    ids0 = BASE + STEP * np.arange(n0)
    r = np.random.default_rng(n0)
    pick = lambda k: np.sort(r.choice(ids0, size=k, replace=False))   # noqa: E731
    run = lambda a, b: ids0[a:b]   # noqa: E731
    gap = lambda a, b, o=1: ids0[a:b] + o   # noqa: E731
    q = n0 // 10
    out = {
        "mixed": (pick(n0 // 30), pick(n0 // 30), np.unique(np.concatenate([pick(n0 // 25) + 1, pick(n0 // 50) + 2]))),
        "append_only": ([], [], ids0[-1] + 1 + np.arange(n0 // 5)),
        "front_run": ([], [], BASE - 1 - np.arange(n0 // 6)),
        "single_rows": ([ids0[5]], [ids0[n0 // 2]], [ids0[n0 // 3] + 1, ids0[0] - 7, ids0[-1] + 9]),
        # the shift changes sign several times: -, +, -, +, and back to 0 at the end
        "alternating": (np.concatenate([run(q, q + 40), run(4 * q, 4 * q + 150), run(9 * q, 9 * q + 5)]), run(5 * q, 5 * q + 3),
                        np.concatenate([gap(2 * q, 2 * q + 90), gap(2 * q, 2 * q + 30, 2), gap(6 * q, 6 * q + 75)])),
        "more_deletions": (np.concatenate([pick(n0 // 8), run(3 * q, 3 * q + q // 2)]), pick(5), gap(7 * q, 7 * q + 20)),
        "more_insertions": (pick(7), pick(5), np.concatenate([gap(q, q + q // 2), gap(q, q + q // 2, 3), gap(8 * q, 8 * q + 11)])),
        "replace_only": ([], pick(n0 // 20), []),
        "nothing": ([], [], []),
    }
    return ids0, out


@pytest.mark.parametrize("d", [20, 64, 100, 768, 1000])
@pytest.mark.parametrize("metric", sorted(ab.METRICS, key=ab.METRICS.get))
def test_rows_and_headers_after_a_delta_equal_a_full_staging(ctx, fresh, metric, d):
    n0 = 3000
    ids0, scen = scenarios(n0)
    for name, (dele, repl, ins) in scen.items():
        items = Items(metric, d, 2 * n0, seed=len(name) + d)
        items.put(ids0)
        items.stage_full(ctx)
        st = ctx.stage_stats()
        assert st == {"uploaded_rows": n0, "moved_rows": 0, "delta": 0, "h2d_bytes": n0 * (row_bytes(metric, d) + 8)}, name
        dele, ins = np.unique(np.asarray(dele, dtype=np.int64)), np.unique(np.asarray(ins, dtype=np.int64))
        repl = np.setdiff1d(np.asarray(repl, dtype=np.int64), dele)
        items.delete(dele)
        items.put(repl)
        items.put(ins)
        # deleted ids are listed too, as a Writer's Updated keys would; they are ignored
        st = check_delta(ctx, fresh, items, ids0, list(dele) + list(repl) + list(ins), moved=0 if name in ("append_only", "replace_only", "nothing") else None)
        assert st["uploaded_rows"] == len(repl) + len(ins), name
        if name == "front_run":
            assert st["moved_rows"] == n0
        # a second delta on top of the first (the resident ids are now the updated ones): undo part of it
        old = items.ids()
        back = list(dele)[: len(dele) // 2]
        items.put(back)
        gone = list(ins)[::3]
        items.delete(gone)
        check_delta(ctx, fresh, items, old, back + gone)


def test_unlisted_new_ids_are_uploaded_and_unlisted_resident_ids_are_kept(ctx, fresh):
    items = Items("euclidean", 40, 5000, seed=1)
    ids0 = np.arange(0, 4000, 2)
    items.put(ids0)
    items.stage_full(ctx)
    items.put([1, 3, 999, 5001])
    st = check_delta(ctx, fresh, items, ids0, [])
    assert st["uploaded_rows"] == 4


@pytest.mark.parametrize("metric,d", [("euclidean", 768), ("binary quantized cosine", 1536)])
def test_a_matrix_of_several_windows(ctx, fresh, metric, d):
    # 400k x 768 f32 = 1.2 GB: more than six windows of the move, in regions that go down, up and down again
    n0 = 400_000 if metric == "euclidean" else 4_000_000
    assert n0 * row_bytes(metric, d) > 3 * SCRATCH_BYTES
    ll = leaf_len(metric, d)
    rng = np.random.default_rng(9)
    pool = np.frombuffer(rng.bytes((n0 + 4096) * ll), np.uint8).reshape(-1, ll).copy()
    pool[:, 0] = 0
    ids0 = 10 + 2 * np.arange(n0, dtype=np.int64)
    q = n0 // 8
    dele = np.concatenate([ids0[100:1100], ids0[5 * q:5 * q + 2500]])
    ins = np.concatenate([ids0[2 * q:2 * q + 2000] + 1, [3, 5], ids0[-1] + 1 + np.arange(90)])
    repl = ids0[7 * q:7 * q + 4]
    keep = np.setdiff1d(ids0, dele)
    new_ids = np.union1d(keep, ins)
    rows0 = np.arange(n0, dtype=np.uint64)
    base = np.uint64(pool.ctypes.data)
    ctx.stage_items_ptrs(metric, d, ids0.astype(np.uint32), base + rows0 * np.uint64(ll))
    rows1 = (new_ids - 10) // 2
    special = np.concatenate([ins, repl])
    rows1[np.searchsorted(new_ids, special)] = n0 + np.arange(special.size)       # their values are the pool's spare rows
    rows1 = rows1.astype(np.uint64)
    changed = np.sort(np.concatenate([dele, ins, repl])).astype(np.uint32)
    ctx.stage_items_delta(metric, d, new_ids.astype(np.uint32), base + rows1 * np.uint64(ll), changed)
    st = ctx.stage_stats()
    assert st["delta"] == 1 and st["uploaded_rows"] == len(ins) + len(repl)
    assert st["moved_rows"] > 3 * (SCRATCH_BYTES // row_bytes(metric, d))
    fresh.stage_items_ptrs(metric, d, new_ids.astype(np.uint32), base + rows1 * np.uint64(ll))
    step = 50_000
    for a in range(0, new_ids.size, step):
        rows = np.arange(a, min(a + step, new_ids.size), dtype=np.uint32)
        assert ctx.read_items(rows).tobytes() == fresh.read_items(rows).tobytes(), a
    # leave the module's contexts small again
    small = Items("euclidean", 32, 64, seed=0)
    small.put(range(64))
    small.stage_full(ctx)
    small.stage_full(fresh)


def test_fallbacks_stage_in_full(fresh):
    c = ab.Context(0)
    try:
        d, n0 = 48, 4000
        items = Items("euclidean", d, 3 * n0, seed=3)
        ids0 = np.arange(n0) * 2
        items.put(ids0)

        def full(why):
            st = c.stage_stats()
            assert st["delta"] == 0 and st["uploaded_rows"] == c.n and st["moved_rows"] == 0, why
            assert st["h2d_bytes"] == c.n * (row_bytes(items.metric, items.d) + 8), why
            same_as_full_staging(c, fresh, items)

        items.stage_delta(c, [])
        full("nothing staged")
        items.stage_delta(c, [])
        assert c.stage_stats()["delta"] == 1 and c.stage_stats()["uploaded_rows"] == 0
        other = Items("manhattan", d, n0, seed=4)
        other.put(ids0)
        items, keep = other, items
        items.stage_delta(c, [])
        full("other metric")
        items = Items("manhattan", d + 1, n0, seed=5)
        items.put(ids0)
        items.stage_delta(c, [])
        full("other dim")
        items = keep
        items.stage_full(c)
        c.stage_begin("euclidean", d, ids0.astype(np.uint32))
        items.stage_delta(c, [])
        full("a staging was open")
        ch = ids0[: n0 // 4 + 1]
        items.put(ch)
        items.stage_delta(c, ch)
        full("more than a quarter of the rows")
        ch = ids0[: n0 // 4]
        items.put(ch)
        items.stage_delta(c, ch)
        assert c.stage_stats()["delta"] == 1 and c.stage_stats()["uploaded_rows"] == n0 // 4
        same_as_full_staging(c, fresh, items)
        # growth: the buffer has 25 % of slack, so + 20 % stays in place and a further + 20 % does not fit
        items.put(2 * n0 + np.arange(n0 // 5))
        items.stage_delta(c, [])
        assert c.stage_stats()["delta"] == 1 and c.stage_stats()["moved_rows"] == 0
        same_as_full_staging(c, fresh, items)
        items.put(3 * n0 + np.arange(n0 // 5))
        items.stage_delta(c, [])
        full("growth past the capacity of the buffer")
        with pytest.raises(ab.ArroyB200Error):
            c.stage_items_delta("euclidean", d, items.ids(), items.ptrs(), np.array([5, 5], dtype=np.uint32))
    finally:
        c.close()


def cosine_leaves(ids, data):
    buf = np.zeros((len(ids), 5 + 4 * data.shape[1]), np.uint8)
    h0 = np.array([oracle.new_header(oracle.COSINE, v)[0] for v in data], dtype=np.float32)
    buf[:, 1:5] = h0.view(np.uint8).reshape(-1, 4)
    buf[:, 5:] = np.ascontiguousarray(data).view(np.uint8).reshape(len(ids), -1)
    return buf, np.uint64(buf.ctypes.data) + np.arange(len(ids), dtype=np.uint64) * np.uint64(buf.shape[1])


def test_derived_state_is_rebuilt_after_a_delta(ctx):
    n, d, n_trees = 12000, 64, 32
    data = oracle.synth_rows(SEED, d, 0, n + 600, 0.5, threads=4)
    ids0 = np.arange(n, dtype=np.uint32) * 2
    buf0, ptrs0 = cosine_leaves(ids0, data[:n])
    ctx.stage_items_ptrs("cosine", d, ids0, ptrs0)
    seeds = [bytes([t + 1] * 32) for t in range(n_trees)]
    ctx.build_trees(seeds, list(range(n_trees)), n_trees)      # builds the 8-bit planes of the old rows
    ctx.rerank_shared(data[:64], np.ones(64, np.float32), np.arange(0, n, 2, dtype=np.uint32), 10)   # and the bf16 shadow
    rows = np.arange(n, dtype=np.uint32)
    ctx.load_forest(kind=[2, 1, 1], left=[1, 0, 0], right=[2, 0, 0], normal_idx=[0xffffffff, 0, 0], normal_hdr0=[0, 0, 0],
                    desc_off=[0, 0, n // 2], desc_len=[0, n // 2, n - n // 2], normals=np.zeros((0, d), np.float32), desc_rows=rows, roots=[0])
    assert ctx.epochs()[1] != 0
    # update: delete 300, replace 300, insert 600 between the old ids
    r = np.random.default_rng(2)
    dele = np.sort(r.choice(ids0, 300, replace=False))
    live = np.setdiff1d(ids0, dele)
    repl = np.sort(r.choice(live, 300, replace=False))
    ins = np.sort(r.choice(ids0, 600, replace=False)) + 1
    new_ids = np.union1d(live, ins).astype(np.uint32)
    vec = {int(i): data[k] for k, i in enumerate(ids0)}
    for k, i in enumerate(repl):
        vec[int(i)] = data[k] * np.float32(0.5) + data[k + 1]
    for k, i in enumerate(ins):
        vec[int(i)] = data[n + k]
    new_data = np.stack([vec[int(i)] for i in new_ids])
    buf1, ptrs1 = cosine_leaves(new_ids, new_data)
    ctx.stage_items_delta("cosine", d, new_ids, ptrs1, np.sort(np.concatenate([dele, repl, ins])).astype(np.uint32))
    assert ctx.stage_stats()["delta"] == 1 and ctx.stage_stats()["uploaded_rows"] == 900
    assert ctx.epochs()[1] == 0          # the forest loaded before the update is gone
    with pytest.raises(ab.ArroyB200Error):
        ctx.search_batch(5, query_rows=[0, 1], search_k=100)
    odb = oracle.Db("cosine", d)
    odb.set_items(new_ids, new_data)
    rng = oracle.StdRng(SEED)
    user = rng.clone()
    odb.build(rng, n_trees=n_trees)
    want = odb.nodes()
    rng1 = oracle.StdRng(user.gen_seed())
    seeds = [rng1.gen_seed() for _ in range(n_trees)]
    got = ctx.build_trees(seeds, list(range(n_trees)), n_trees)
    assert got.keys() == want.keys() and not [k for k in want if want[k] != got[k]]
    h0 = np.array([oracle.new_header(oracle.COSINE, v)[0] for v in new_data], dtype=np.float32)
    cand = np.arange(0, new_ids.size, 3, dtype=np.uint32)
    for qi in (0, 5, 4000):
        q = new_data[qi]
        qh = oracle.new_header(oracle.COSINE, q)
        wr, wd = oracle.rerank(oracle.COSINE, q, qh, new_data, h0, None, cand, 10)
        gr, gd = ctx.rerank(q, qh, cand, 10)
        assert wr.tolist() == gr.tolist() and wd.tobytes() == gd.tobytes()
    gr, gd, gl = ctx.rerank_shared(new_data[:48], h0[:48], cand, 10)    # batched: the fused bf16 re-rank over the new shadow
    for qi in range(48):
        wr, wd = oracle.rerank(oracle.COSINE, new_data[qi], (h0[qi], 0.0), new_data, h0, None, cand, 10)
        assert gr[qi, :gl[qi]].tolist() == wr.tolist() and gd[qi, :gl[qi]].tobytes() == wd.tobytes()


# ---- through the host mirror -------------------------------------------------------------------------------------------------

def make_env(c):
    e = ab.Env(0)
    e._ctx = c
    return e


class Pair:
    """one index written through the host mirror and through the oracle"""

    def __init__(self, env, index, metric, d, n_trees):
        self.env, self.index, self.metric, self.d, self.n_trees = env, index, metric, d, n_trees
        self.w = ab.Writer(env, index, d, metric)
        self.odb = oracle.Db(metric, d)
        self.prng, self.orng = ab.StdRng.from_seed(SEED), oracle.StdRng(SEED)
        self.live = set()

    def add(self, i, v):
        self.w.add_item(int(i), v); self.odb.add_item(int(i), v); self.live.add(int(i))

    def delete(self, i):
        self.w.del_item(int(i)); self.odb.del_item(int(i)); self.live.discard(int(i))

    def build(self, n_trees=None):
        self.w.builder(self.prng).n_trees(n_trees or self.n_trees).build()
        self.odb.build_incremental(self.orng, n_trees=n_trees or self.n_trees)
        assert self.env.tree_nodes(self.index) == self.odb.nodes()
        return self.env.ctx.stage_stats()

    def check_queries(self, k=25):
        rd = ab.Reader.open(self.env, self.index, self.metric)
        for it in sorted(self.live)[:k]:
            assert [g[0] for g in rd.nns(10).by_item(it)] == [x[0] for x in self.odb.nns_by_item(it, 10)]
        return rd


def run_update_sequence(c, metric, d, n_trees, expect_delta):
    n0 = 3000
    data = oracle.synth_rows(SEED, d, 0, n0 + 2000, 0.5, threads=4)
    env = make_env(c)
    p = Pair(env, 0, metric, d, n_trees)
    r = np.random.default_rng(5)
    for i in range(n0):
        p.add(i, data[i])
    next_new = n0
    written = None
    for rnd in range(4):
        st = p.build()
        n = len(p.live)
        if not expect_delta:
            assert st["delta"] == 0 and st["uploaded_rows"] == n and env.resident() is None
        elif written is None or 4 * written > n:
            assert st["delta"] == 0 and st["uploaded_rows"] == n, rnd       # the first build, or more than a quarter is new
        else:
            assert st["delta"] == 1 and st["uploaded_rows"] == written, rnd
            assert st["h2d_bytes"] < (written + 1) * 4 * ((d + 31) // 32 * 32) + 8 * n + 16 * (2 * 250 + 2 * written + 8)
        if expect_delta:
            assert env.resident() == {"index": 0, "epoch": c.epochs()[0], "dirty": 0}
        assert p.w.build_timings()["h2d_bytes"] == st["h2d_bytes"]
        dele = r.choice(sorted(p.live), size=150, replace=False)
        for i in dele:
            p.delete(i)
        over = r.choice(sorted(p.live), size=100, replace=False)
        for i in over:
            p.add(i, data[int(r.integers(0, len(data)))] * np.float32(0.5))
        added = int(r.integers(50, 700))
        for _ in range(added):
            p.add(next_new, data[next_new % len(data)])
            next_new += 1
        written = 100 + added
        if expect_delta:
            assert env.resident()["dirty"] == 250 + added
    p.build(n_trees + 2)
    p.check_queries()
    nodes = env.tree_nodes()
    env._ctx = None
    return nodes


@pytest.mark.parametrize("metric,d,n_trees", [("cosine", 32, 4), ("euclidean", 48, 3), ("dot-product", 40, 3), ("manhattan", 33, 2)])
def test_update_sequences_upload_only_what_was_written(ctx, monkeypatch, metric, d, n_trees):
    # the Writers of the host mirror store f32 vectors (the four float metrics); bit-string rows take the same path below the
    # C ABI and are covered there
    nodes = run_update_sequence(ctx, metric, d, n_trees, expect_delta=True)
    monkeypatch.setenv("ARROY_B200_FULL_RESTAGE", "1")
    assert run_update_sequence(ctx, metric, d, n_trees, expect_delta=False) == nodes


def test_a_reader_opened_after_a_build_uploads_no_items(ctx, monkeypatch):
    n, d = 6000, 96
    data = oracle.synth_rows(SEED, d, 0, n, 0.5, threads=4)
    matrix = n * 4 * d
    grown = {}
    for mode in ("resident", "full"):
        if mode == "full":
            monkeypatch.setenv("ARROY_B200_FULL_RESTAGE", "1")
        env = make_env(ctx)
        p = Pair(env, 0, "euclidean", d, 3)
        for i in range(n):
            p.add(i, data[i])
        p.build()
        e0, h0 = ctx.epochs()[0], ctx.counters()["h2d_bytes"]
        rd = ab.Reader.open(env, 0, "euclidean")
        got = rd.nns(10).by_item(17)
        assert [g[0] for g in got] == [x[0] for x in p.odb.nns_by_item(17, 10)]
        ids, dist, lens, _ = rd.nns_batch_by_item(np.arange(40), 10)
        for i in range(40):
            assert ids[i, :lens[i]].tolist() == [x[0] for x in p.odb.nns_by_item(i, 10)]
        grown[mode] = ctx.counters()["h2d_bytes"] - h0
        assert (ctx.epochs()[0] == e0) == (mode == "resident")
        env._ctx = None
    assert grown["resident"] < matrix // 2 < matrix <= grown["full"]      # the forest and the queries, not the item matrix
    assert grown["full"] - grown["resident"] == n * (4 * d + 8)


def test_two_envs_and_two_indexes_sharing_one_context(ctx):
    d = 32
    data = oracle.synth_rows(SEED, d, 0, 6000, 0.5, threads=4)
    env_a, env_b = make_env(ctx), make_env(ctx)
    a, b = Pair(env_a, 0, "euclidean", d, 3), Pair(env_b, 0, "cosine", d, 3)
    a2 = Pair(env_a, 1, "euclidean", d, 2)
    for i in range(2000):
        a.add(i, data[i]); b.add(i, data[3000 + i]); a2.add(3 * i, data[1000 + i])
    assert a.build()["delta"] == 0
    a.add(5000, data[5000])
    assert a.build() == {"uploaded_rows": 1, "moved_rows": 0, "delta": 1, "h2d_bytes": 4 * d + 8 * 2001 + 16}
    assert b.build()["delta"] == 0                 # another Env's rows were resident
    a.add(5001, data[5001])
    assert a.build()["delta"] == 0                 # ... and now b's are: a's record is stale
    a.check_queries()
    b.delete(7)
    st = b.build()
    assert st["delta"] == 0 and st["uploaded_rows"] == 1999     # a's reader staged a's items in between
    assert a2.build()["delta"] == 0                # the other index of env_a
    a.add(5002, data[5002])
    assert a.build()["delta"] == 0                 # env_a's record was about index 1
    a2.delete(0)
    assert a2.build()["delta"] == 0
    a2.add(1, data[1])
    st = a2.build()
    assert st["delta"] == 1 and st["uploaded_rows"] == 1 and st["moved_rows"] == 1999     # id 1 goes in front of all the others
    for p in (a, b, a2):
        p.check_queries(10)
    env_a._ctx = None
    env_b._ctx = None


def test_cancelled_build_then_clear_and_refill(ctx):
    d = 32
    data = oracle.synth_rows(SEED, d, 0, 5000, 0.5, threads=4)
    env = make_env(ctx)
    p = Pair(env, 0, "euclidean", d, 3)
    for i in range(2500):
        p.add(i, data[i])
    p.build()
    for i in range(2500, 2600):
        p.add(i, data[i])
    p.delete(3)
    calls = []
    with pytest.raises(ab.ArroyError) as ei:     # cancelled after the items were staged
        p.w.builder(ab.StdRng.from_seed(SEED)).n_trees(3).cancel(lambda: calls.append(1) or len(calls) > 1).build()
    assert ei.value.kind == "BuildCancelled" and p.w.need_build()
    st = ctx.stage_stats()
    assert st["delta"] == 1 and st["uploaded_rows"] == 100 and env.resident()["dirty"] == 0
    st = p.build()                               # nothing was written since: nothing is uploaded, the trees are the oracle's
    assert st["delta"] == 1 and st["uploaded_rows"] == 0 and st["moved_rows"] == 0
    # delete every item, build the empty index, fill it again with other vectors
    ids = sorted(p.live)
    for i in ids:
        p.delete(i)
    p.build()
    for i in ids:
        p.add(i, data[i + 2000])
    st = p.build()
    assert st["delta"] == 0 and st["uploaded_rows"] == len(ids)
    p.check_queries()
    # what drops the record
    assert env.resident() is not None
    ab.Writer(env, 0, d, "euclidean")
    assert env.resident() is not None
    ab.Writer(env, 0, d, "cosine")
    assert env.resident() is None
    p.add(9000, data[0])
    assert p.build()["delta"] == 0 and env.resident() is not None
    k, v = next((k, v) for k, v in env.items() if k[2] == 3)
    env.put_raw(k, v)
    assert env.resident() is None
    p.add(9001, data[1])
    assert p.build()["delta"] == 0
    p.w.clear()
    assert env.resident() is None
    env._ctx = None
