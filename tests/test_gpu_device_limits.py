"""Launches that take more than 48 KB of dynamic shared memory need their kernel's limit raised, and that limit belongs to the
kernel on one device. Such launches must work on every device of a process, whichever device raised the limit first, and a
smaller request from one context must not lower the limit another context on the same device relies on. Every result is
checked against the oracle."""
import numpy as np
import pytest

import arroy_b200 as ab
import oracle
from arroy_b200._capi import row_bitmap
from test_gpu_build_schedules import side_multi, tree_seeds
from test_gpu_filtered_search import forest_arrays

pytestmark = pytest.mark.gpu
SEED = bytes([42] * 32)


def filtered_walk1(ctxs):
    # one filtered query at d = 768: walk1_kernel<FILTER> (Walk1Shared<true> alone is above 64 KB)
    metric, n, d, T, count = "euclidean", 3000, 768, 4, 10
    data = oracle.synth_rows(SEED, d, 0, n, 0.5, threads=8)
    ids = np.arange(n, dtype=np.uint32)
    odb = oracle.Db(metric, d)
    odb.set_items(ids, data)
    odb.build(oracle.StdRng(SEED), n_trees=T, threads=T)
    F = np.arange(0, n, 2, dtype=np.uint32)   # more rows than search_k = count x trees: the query walks, no small-filter shortcut
    want = odb.nns_by_item(7, count, candidates=F.tolist())
    for ctx in ctxs:
        ctx.stage_items_flat(metric, ids, data)
        ctx.load_forest(roots=np.arange(T, dtype=np.uint32), **forest_arrays(odb.nodes(), oracle.EUCLIDEAN, d))
        s0 = ctx.search_stats()
        rows, dist, length, status = ctx.search_batch_filtered(count, row_bitmap(F, n), query_rows=[7])
        assert status[0] == 0 and ctx.search_stats()["shortcut_queries"] == s0["shortcut_queries"]
        assert rows[0, :length[0]].tolist() == [w[0] for w in want]
        assert dist[0, :length[0]].tobytes() == np.array([w[1] for w in want], dtype=np.float32).tobytes()


def fused_rerank(ctxs):
    # the fused re-rank at d = 2560 (frerank_smem is above 48 KB from ld = 2080 on)
    metric, n, d, nq, k = "cosine", 4000, 2560, 8, 10
    data = oracle.synth_rows(SEED, d, 0, n + nq, 0.5, threads=8)
    rng = np.random.default_rng(2560)
    lists = [np.sort(rng.choice(n, int(rng.integers(600, 2000)), replace=False)).astype(np.uint32) for _ in range(nq)]
    offs = np.zeros(nq + 1, dtype=np.uint64)
    offs[1:] = np.cumsum([len(r) for r in lists])
    for ctx in ctxs:
        ctx.stage_items_flat(metric, np.arange(n + nq, dtype=np.uint32), data)
        h0, _ = ctx.item_headers()
        c0 = ctx.counters()
        out_rows, out_dist, out_len = ctx.rerank_batch(data[n:], h0[n:], np.concatenate(lists), offs, k)
        assert ctx.counters()["fused_rerank_batches"] > c0["fused_rerank_batches"]
        for i in range(nq):
            wr, wd = oracle.rerank(oracle.COSINE, data[n + i], (float(h0[n + i]), 0.0), data, h0, None, lists[i], k)
            assert out_rows[i, :out_len[i]].tolist() == wr.tolist() and out_dist[i, :out_len[i]].tobytes() == wd.tobytes()


def tensor_core_prefilter(ctxs):
    # rerank_shared with nq x nc = 2^22 and nc >= 4k: the tensor-core pre-filter (tcgemm_tf32_kernel takes TG_SMEM > 48 KB)
    metric, n, d, nq, k = "euclidean", 32768, 96, 128, 10
    data = oracle.synth_rows(SEED, d, 0, n + nq, 0.5, threads=8)
    rows = np.arange(n, dtype=np.uint32)
    for ctx in ctxs:
        ctx.stage_items_flat(metric, np.arange(n + nq, dtype=np.uint32), data)
        h0, _ = ctx.item_headers()
        s0 = ctx.rerank_stats()
        out_rows, out_dist, out_len = ctx.rerank_shared(data[n:], h0[n:], rows, k)
        assert ctx.rerank_stats()["prefilter_chunks"] > s0["prefilter_chunks"]
        for i in (0, 63, nq - 1):
            wr, wd = oracle.rerank(oracle.EUCLIDEAN, data[n + i], (float(h0[n + i]), 0.0), data, np.zeros(n + nq, np.float32), None, rows, k)
            assert out_rows[i, :out_len[i]].tolist() == wr.tolist() and out_dist[i, :out_len[i]].tobytes() == wd.tobytes()


@pytest.mark.parametrize("launch", [filtered_walk1, fused_rerank, tensor_core_prefilter], ids=lambda f: f.__name__)
def test_launch_on_the_second_device_after_the_first(launch):
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two visible GPUs")
    ctxs = [ab.Context(0), ab.Context(1)]
    try:
        launch(ctxs)
    finally:
        for c in ctxs:
            c.close()


def test_smaller_request_of_another_context_keeps_the_limit():
    # side_multi with 40 jobs at d = 12800 asks work_kernel for more shared memory than a build of 2 trees on another context of
    # the same device; after that build, the first context's side_multi must still launch
    metric, n, d, jobs, T = "euclidean", 2000, 12800, 40, 2
    data = oracle.synth_rows(SEED, d, 0, n, 0.0, threads=8)
    r = np.random.default_rng(12800)
    normals = (r.standard_normal((jobs, d)) / np.sqrt(d)).astype(np.float32)
    hdr0 = (r.standard_normal(jobs) * 0.1).astype(np.float32)
    subsets = [np.sort(r.choice(n, size=int(r.integers(1, n)), replace=False)).astype(np.uint32) for _ in range(jobs)]
    h0 = np.zeros(n, dtype=np.float32)
    want = [oracle.side_batch(oracle.EUCLIDEAN, normals[j], (float(hdr0[j]), 0.0), data, h0, None, subsets[j], want_margin=False)[0]
            for j in range(jobs)]
    a, b = ab.Context(0), ab.Context(0)
    try:
        for c in (a, b):
            c.stage_items_flat(metric, np.arange(n, dtype=np.uint32), data)
        before = side_multi(a, normals, hdr0, subsets)
        b.build_trees(tree_seeds(SEED, T), list(range(T)), T, 64)
        after = side_multi(a, normals, hdr0, subsets)
        for j in range(jobs):
            assert before[j].tobytes() == want[j].tobytes(), j
            assert after[j].tobytes() == want[j].tobytes(), j
    finally:
        a.close()
        b.close()
