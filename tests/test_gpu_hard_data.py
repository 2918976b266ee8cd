"""Builds, scans, splits, searches and re-ranks on data that makes the low-precision filters give up, against the oracle.

Every low-precision shortcut of the device path is only a filter in front of exact arithmetic, and each has a give-up path:
the speculative two_means (TF32 Gram prediction) re-runs sequentially after a misspeculation, the 8-bit side() pre-filter
leaves rows near the hyperplane to the f32 re-score (stage 3), the fused bf16 re-rank hands a query with too many survivors to
the plain kernels, and rerank_shared's TF32 pre-filter hands a chunk with too many survivors to the exact dense kernel. The
uniform rows most tests use almost never reach these paths. The families here do, and each test asserts that its path ran:

  tiny        rows scaled to 2^-72 ... 2^-100 (or mixed per row): the reference's products underflow, its margins are +-0
              and its splits fall back to random ones; the pre-filter must leave every such row to the f32 re-score
  clusters    32 centres and rows a relative 2^-8 or 2^-18 around them: two_means meets near-ties far below the TF32
              prediction's rounding, so it misspeculates
  duplicates  every row copied 1-8 times and one block of 3000 identical rows: random splits nested in real ones, distance
              ties broken by id
  sparse      1-4 nonzeros from {+-1, +-0.5, +-0.25}, 1 % zero rows and -0.0 elements: margins of exactly +-0, Cosine rows of
              norm 0, DotProduct preprocess with zero rows
"""
import functools
import os

import numpy as np
import pytest

import arroy_b200 as ab
import oracle
from test_gpu_build_schedules import tree_seeds
from test_gpu_filtered_search import forest_arrays
from test_gpu_parity import headers_for

pytestmark = pytest.mark.gpu
SEED = bytes([42] * 32)
THREADS = min(os.cpu_count() or 4, 32)
F32 = np.float32
MET = ["euclidean", "cosine", "dot-product", "manhattan"]
BLOCK = 3000          # identical rows in the duplicates family


@pytest.fixture(scope="module")
def ctx():
    c = ab.Context(0)
    yield c
    c.close()


# ---- the data families ----------------------------------------------------------------------------------------------------
def tiny(n, d, e):
    base = oracle.synth_rows(SEED, d, 0, n, 0.5, threads=THREADS).astype(np.float64)
    if e == "mixed":
        ex = np.random.default_rng(1).integers(-90, -69, size=(n, 1))
        return (base * np.exp2(ex)).astype(np.float32)
    return (base * 2.0 ** e).astype(np.float32)


def clusters(n, d, shift, n_centres=32, big_first=False):
    """(rows, labels): rows = centre + 2^-shift mean|centre| noise"""
    rng = np.random.default_rng(shift * 100 + n_centres)
    centres = oracle.synth_rows(SEED, d, 10_000_000, n_centres, 0.5).astype(np.float64)
    if big_first:
        centres[0] *= 2.0            # the largest dot products too, for DotProduct queries in cluster 0
    lab = rng.integers(0, n_centres, size=n)
    noise = rng.standard_normal((n, d)) * 2.0 ** -shift * np.abs(centres).mean(axis=1)[lab, None]
    return (centres[lab] + noise).astype(np.float32), lab


def duplicates(n, d, block=BLOCK):
    """(rows, the rows of the identical block): the block vector is twice a synthesized row, so that it is also every
    metric's nearest row to itself (DotProduct included)"""
    rng = np.random.default_rng(7)
    uniq = oracle.synth_rows(SEED, d, 20_000_000, n, 0.5, threads=THREADS)
    reps = rng.integers(1, 9, size=n)
    idx = np.repeat(np.arange(n), reps)[: n - block]
    rows = np.concatenate([uniq[idx], np.repeat(uniq[-1:] * F32(2), block, axis=0)])
    perm = rng.permutation(n)
    rows = rows[perm]
    return rows, np.sort(np.flatnonzero(perm >= n - block)).astype(np.uint32)


def sparse(n, d):
    rng = np.random.default_rng(11)
    rows = np.zeros((n, d), dtype=np.float32)
    vals = np.array([1.0, -1.0, 0.5, -0.5, 0.25, -0.25], dtype=np.float32)
    k = rng.integers(1, 5, size=n)
    for i in range(n):
        rows[i, rng.choice(d, size=min(int(k[i]), d), replace=False)] = rng.choice(vals, size=min(int(k[i]), d))
    rows[rng.random(n) < 0.01] = 0.0
    neg = rng.random((n, d)) < 0.05
    rows[neg & (rows == 0)] = -0.0
    rows[rng.random(n) < 0.005] = -0.0
    return rows


@functools.lru_cache(maxsize=None)
def family_rows(family, n, d):
    if family.startswith("tiny-"):
        tail = family[5:]
        return tiny(n, d, "mixed" if tail == "mixed" else -int(tail))
    if family.startswith("clusters-"):
        return clusters(n, d, int(family[9:]))[0]
    if family == "duplicates":
        return duplicates(n, d, min(BLOCK, n // 2))[0]
    assert family == "sparse"
    return sparse(n, d)


def assert_same_forest(got, want, what):
    """node bytes of every node id either forest has; the message names the first id that differs"""
    bad = [k for k in sorted(set(got) | set(want)) if got.get(k) != want.get(k)]
    assert not bad, "%s: %d node ids differ (%d nodes built, %d in the oracle's forest), first id %d: %r vs the oracle's %r" % (
        what, len(bad), len(got), len(want), bad[0], got.get(bad[0], b"")[:48], want.get(bad[0], b"")[:48])


def query_headers(metric, vecs):
    if metric == "cosine":
        return np.array([oracle.new_header(oracle.COSINE, v)[0] for v in vecs], dtype=np.float32)
    return np.zeros(len(vecs), dtype=np.float32)


# ---- forests under three build setups, and queries on them ------------------------------------------------------------------
# 40 000 x 128: n ld >= 2^22 and d >= 64, so nodes go through the 8-bit planes. 32 trees: every node (fused root pass);
# 3 trees: nodes of more than 8192 rows; lockstep: the schedule the others are tested against.
FN, FD = 40_000, 128
FAMILIES = ["tiny-72", "tiny-76", "tiny-80", "tiny-100", "tiny-mixed", "clusters-8", "clusters-18", "duplicates", "sparse"]
SETUPS = {"all-planes": 32, "few-trees": 3, "lockstep": 32}
RANDOM_SPLITS = {"tiny-76", "tiny-80", "tiny-100", "duplicates"}
_ORACLE = {}


def oracle_db(family, metric, T):
    key = (family, metric, T)
    if key not in _ORACLE:
        data = family_rows(family, FN, FD)
        odb = oracle.Db(metric, FD)
        odb.set_items(np.arange(FN, dtype=np.uint32), data)
        odb.build(oracle.StdRng(SEED), n_trees=T, threads=min(T, THREADS))
        _ORACLE[key] = (odb, odb.nodes())
    return _ORACLE[key]


@pytest.mark.parametrize("setup", list(SETUPS))
@pytest.mark.parametrize("metric", MET)
@pytest.mark.parametrize("family", FAMILIES)
def test_forest_matches_the_oracle(ctx, monkeypatch, family, metric, setup):
    T = SETUPS[setup]
    data = family_rows(family, FN, FD)
    ctx.stage_items_flat(metric, np.arange(FN, dtype=np.uint32), data)
    if metric == "dot-product":
        ctx.dot_preprocess()
    if setup == "lockstep":
        monkeypatch.setenv("ARROY_B200_LOCKSTEP", "1")
    got = ctx.build_trees(tree_seeds(SEED, T), list(range(T)), T)
    monkeypatch.delenv("ARROY_B200_LOCKSTEP", raising=False)
    st, pre = ctx.build_stats(), ctx.build_prefilter_stats()
    odb, want = oracle_db(family, metric, T)
    assert_same_forest(got, want, (family, metric, setup))
    assert st["scanned_rows"] == odb.scanned_rows
    assert pre["rows_via_prefilter"] > 0, pre
    if family.startswith("tiny"):
        assert pre["rows_rescored_f32"] > 0, pre
    if family in RANDOM_SPLITS:
        assert st["random_splits"] > 0, st
    if family.startswith("clusters"):
        # Manhattan's two_means is always the sequential loop
        assert (st["misspeculated_splits"] > 0) == (metric != "manhattan"), st
    if setup != "all-planes":
        return
    m = oracle.METRICS[metric]
    ctx.load_forest(roots=np.arange(T, dtype=np.uint32), **forest_arrays(got, m, FD))
    rng = np.random.default_rng(len(family) + len(metric))
    count = 10
    for nq in (3, 12, 40):        # walk1_kernel with forest_dots_kernel, walk1_kernel alone, walk_kernel
        qitems = np.sort(rng.choice(FN, size=nq, replace=False)).astype(np.uint32)
        out_rows, out_dist, out_len, status = ctx.search_batch(count, query_rows=qitems)
        assert not status.any()
        for i, it in enumerate(qitems):
            w = odb.nns_by_item(int(it), count)
            assert out_rows[i, :out_len[i]].tolist() == [x[0] for x in w], (nq, int(it))
            assert out_dist[i, :out_len[i]].tobytes() == np.array([x[1] for x in w], dtype=np.float32).tobytes(), (nq, int(it))
        qv = data[rng.choice(FN, size=nq, replace=False)]
        out_rows, out_dist, out_len, status = ctx.search_batch(count, queries=qv, qhdr0=query_headers(metric, qv))
        assert not status.any()
        for i in range(nq):
            w = odb.nns_by_vector(qv[i], count)
            assert out_rows[i, :out_len[i]].tolist() == [x[0] for x in w], (nq, i)
            assert out_dist[i, :out_len[i]].tobytes() == np.array([x[1] for x in w], dtype=np.float32).tobytes(), (nq, i)


@pytest.mark.parametrize("metric", MET)
def test_clusters_below_32_dimensions_never_speculate(ctx, metric):
    n, d, T = 8000, 16, 8
    data = family_rows("clusters-18", n, d)
    ctx.stage_items_flat(metric, np.arange(n, dtype=np.uint32), data)
    if metric == "dot-product":
        ctx.dot_preprocess()
    got = ctx.build_trees(tree_seeds(SEED, T), list(range(T)), T)
    st = ctx.build_stats()
    odb = oracle.Db(metric, d)
    odb.set_items(np.arange(n, dtype=np.uint32), data)
    odb.build(oracle.StdRng(SEED), n_trees=T, threads=min(T, THREADS))
    assert_same_forest(got, odb.nodes(), (metric, d))
    assert st["scanned_rows"] == odb.scanned_rows
    assert st["misspeculated_splits"] == 0


# ---- create_split on subsets inside one cluster, one duplicate block and the tiny rows --------------------------------------
@pytest.mark.parametrize("d", [32, 64, 768, 2080, 2144])      # 2080 still speculates, 2144 does not
@pytest.mark.parametrize("metric", MET)
def test_create_split_on_hard_subsets(ctx, metric, d):
    ca, la = clusters(400, d, 8, n_centres=4)
    cb, lb = clusters(400, d, 18, n_centres=4)
    dup, block = duplicates(600, d, block=250)
    ti = tiny(300, d, -80)
    data = np.concatenate([ca, cb, dup, ti])
    n = data.shape[0]
    h0, h1 = headers_for(metric, data)
    ctx.stage_items_flat(metric, np.arange(n, dtype=np.uint32), data, h0, h1)
    m = oracle.METRICS[metric]
    o_dup, o_ti = 800, 1400
    subsets = {"cluster 2^-8": np.flatnonzero(la == 0), "cluster 2^-18": 400 + np.flatnonzero(lb == 1),
               "identical block": o_dup + block, "duplicates": o_dup + np.arange(600), "tiny": o_ti + np.arange(300),
               "tiny sample": o_ti + np.sort(np.random.default_rng(d).choice(300, 57, replace=False))}
    for name, rows in subsets.items():
        rows = np.ascontiguousarray(rows, dtype=np.uint32)
        for trial in range(2):
            seed = bytes([(11 * trial + d) % 256] * 32)
            start_words = 17 * trial
            rng = oracle.StdRng(seed)
            for _ in range(start_words):
                rng.next_u32()
            probe = rng.clone()
            want_n, want_h = oracle.create_split(m, rng, data, h0, h1, rows)
            got_n, got_h, pos = ctx.create_split(np.frombuffer(seed, dtype="<u4"), start_words, rows)
            assert got_n.tobytes() == want_n.tobytes(), (name, trial, np.nonzero(got_n.view(np.uint32) != want_n.view(np.uint32))[0][:5])
            assert np.float32(got_h[0]).tobytes() == np.float32(want_h[0]).tobytes() and got_h[1] == want_h[1], (name, trial)
            for _ in range(pos - start_words):
                probe.next_u32()
            assert probe.next_u32() == rng.next_u32(), (name, trial)


# ---- side_batch margins, signed zeros included ----------------------------------------------------------------------------
@pytest.mark.parametrize("d", [16, 31, 32, 33, 64, 768])
@pytest.mark.parametrize("metric", MET)
def test_side_batch_margins_on_hard_rows(ctx, metric, d):
    n = 1500
    m = oracle.METRICS[metric]
    rng = np.random.default_rng(d)
    for family in ("tiny-80", "tiny-mixed", "clusters-18", "duplicates", "sparse"):
        data = family_rows(family, n, d)
        h0, h1 = headers_for(metric, data)
        ctx.stage_items_flat(metric, np.arange(n, dtype=np.uint32), data, h0, h1)
        rows = np.sort(rng.choice(n, size=n - 41, replace=False)).astype(np.uint32)
        normal, hdr = oracle.create_split(m, oracle.StdRng(SEED), data, h0, h1, rows)
        cases = [(normal, hdr)]
        if family == "sparse":     # a sparse normal: the rows off its support have margins of exactly +-0
            sn = np.zeros(d, dtype=np.float32)
            sn[:2] = (1.0, -0.5)
            cases.append((sn, (0.0, 0.0)))
        for j, (nrm, hd) in enumerate(cases):
            side, mg = ctx.side_batch(nrm, hd, rows)
            wside, wmg = oracle.side_batch(m, nrm, hd, data, h0, h1, rows)
            assert mg.tobytes() == wmg.tobytes(), (family, j, np.nonzero(mg.view(np.uint32) != wmg.view(np.uint32))[0][:10])
            assert side.tobytes() == wside.tobytes(), (family, j)
            if j == 1:
                assert (wmg == 0).sum() > 0.5 * rows.size


# ---- re-rank give-ups on ties -----------------------------------------------------------------------------------------------
def tied_rows(family, d):
    """(rows, a query row, 8000 candidates): more than 2048 of the candidates tie (duplicates) or sit within 2^-18 (clusters)
    of the query's nearest row. 8000: the fused re-rank holds at most 8192 candidates per query."""
    n = 12_000
    if family == "duplicates":
        data, tied = duplicates(n, d)
    else:
        data, lab = clusters(n, d, 18, n_centres=4, big_first=True)
        tied = np.flatnonzero(lab == 0)
    assert 2048 < tied.size < 8000
    rest = np.setdiff1d(np.arange(n), tied)
    others = np.random.default_rng(d).choice(rest, 8000 - tied.size, replace=False)
    return data, int(tied[0]), np.sort(np.concatenate([tied, others])).astype(np.uint32)


def _oracle_check(metric, data, queries, qh, lists, k, got):
    m = oracle.METRICS[metric]
    h0 = headers_for(metric, data)[0] if metric == "cosine" else np.zeros(data.shape[0], dtype=np.float32)
    out_rows, out_dist, out_len = got
    for i in range(len(lists)):
        wr, wd = oracle.rerank(m, queries[i], (float(qh[i]), 0.0), data, h0, None, lists[i], k)
        assert out_rows[i, :out_len[i]].tolist() == wr.tolist(), i
        assert out_dist[i, :out_len[i]].tobytes() == wd.tobytes(), i


@pytest.mark.parametrize("family", ["duplicates", "clusters"])
@pytest.mark.parametrize("metric", ["euclidean", "cosine", "dot-product"])
def test_fused_rerank_falls_back_on_ties(ctx, monkeypatch, family, metric):
    d, k = 64, 10
    data, qi, cand = tied_rows(family, d)
    n = data.shape[0]
    ctx.stage_items_flat(metric, np.arange(n, dtype=np.uint32), data)
    rng = np.random.default_rng(2)
    queries = np.stack([data[qi], data[qi], data[int(rng.integers(n))]])
    qh = query_headers(metric, queries)
    lists = [cand, cand[::2], np.sort(rng.choice(n, 1500, replace=False)).astype(np.uint32)]
    offs = np.zeros(len(lists) + 1, dtype=np.uint64)
    offs[1:] = np.cumsum([len(r) for r in lists])
    flat = np.concatenate(lists)
    monkeypatch.setenv("ARROY_B200_FRERANK", "0")
    plain = ctx.rerank_batch(queries, qh, flat, offs, k)
    monkeypatch.setenv("ARROY_B200_FRERANK", "1")
    c0 = ctx.counters()
    fused = ctx.rerank_batch(queries, qh, flat, offs, k)
    c1 = ctx.counters()
    assert c1["fused_rerank_batches"] > c0["fused_rerank_batches"]
    assert c1["fused_rerank_fallbacks"] > c0["fused_rerank_fallbacks"]
    assert plain[2].tolist() == fused[2].tolist()
    for i in range(len(lists)):
        assert plain[0][i, :plain[2][i]].tolist() == fused[0][i, :fused[2][i]].tolist(), i
        assert plain[1][i, :plain[2][i]].tobytes() == fused[1][i, :fused[2][i]].tobytes(), i
    _oracle_check(metric, data, queries, qh, lists, k, fused)


@pytest.mark.parametrize("family", ["duplicates", "clusters"])
@pytest.mark.parametrize("metric", ["euclidean", "cosine", "dot-product"])
def test_shared_rerank_falls_back_on_ties(ctx, monkeypatch, family, metric):
    d, k = 64, 10            # at most max(1024, 4k) = 1024 survivors per query
    data, qi, cand = tied_rows(family, d)
    n = data.shape[0]
    ctx.stage_items_flat(metric, np.arange(n, dtype=np.uint32), data)
    rng = np.random.default_rng(3)
    queries = np.concatenate([data[qi][None, :], data[rng.choice(n, 7, replace=False)]])
    qh = query_headers(metric, queries)
    monkeypatch.setenv("ARROY_B200_XRERANK", "exact")
    exact = ctx.rerank_shared(queries, qh, cand, k)
    before = ctx.rerank_stats()
    monkeypatch.setenv("ARROY_B200_XRERANK", "filter")
    filt = ctx.rerank_shared(queries, qh, cand, k)
    after = ctx.rerank_stats()
    assert after["prefilter_chunks"] > before["prefilter_chunks"]
    assert after["fallback_chunks"] > before["fallback_chunks"]
    assert exact[2].tolist() == filt[2].tolist()
    for i in range(queries.shape[0]):
        assert exact[0][i, :exact[2][i]].tolist() == filt[0][i, :filt[2][i]].tolist(), i
        assert exact[1][i, :exact[2][i]].tobytes() == filt[1][i, :filt[2][i]].tobytes(), i
    _oracle_check(metric, data, queries[:3], qh[:3], [cand] * 3, k, filt)
