"""A context frees everything it allocates. The process-wide allocation census (arroy_b200_allocations) counts live device
buffers, pinned host buffers and CUDA handles. After a context has used every family of scratch and has been closed, the census
equals what it was before the context was created, in every field."""
import gc

import numpy as np
import pytest

import arroy_b200 as ab
import oracle
from arroy_b200._capi import allocations, bq_quantize, row_bitmap
from test_gpu_filtered_search import forest_arrays

ZERO = {"device_buffers": 0, "device_bytes": 0, "pinned_buffers": 0, "pinned_bytes": 0, "handles": 0}


def test_census_is_zero_without_a_device():
    import torch
    if torch.cuda.is_available():
        return   # the GPU case below checks the census on a device
    assert allocations() == ZERO
    with pytest.raises(ab.ArroyB200Error):
        ab.Context(0)
    assert allocations() == ZERO


def census():
    gc.collect()
    return allocations()


def leaf_pointers(data):
    """Leaf values ([0x00][header f32][vector]) of the rows of `data`: the pool that owns them and their addresses."""
    n, d = data.shape
    pool = np.zeros((n, 5 + 4 * d), np.uint8)
    pool[:, 5:] = data.view(np.uint8).reshape(n, 4 * d)
    return pool, np.uint64(pool.ctypes.data) + np.arange(n, dtype=np.uint64) * np.uint64(pool.shape[1])


def exercise(ctx, monkeypatch):
    rng = np.random.default_rng(3)
    n, d, T = 65536, 64, 4   # n x d = 2^22: the build scans through the 8-bit planes
    data = rng.standard_normal((n, d), dtype=np.float32)
    ids = np.arange(n, dtype=np.uint32)
    seeds = [bytes([t + 1] * 32) for t in range(T)]
    ctx.stage_items_flat("euclidean", ids, data)
    nodes = ctx.build_trees(seeds, list(range(T)), T)
    assert ctx.build_prefilter_stats()["rows_via_prefilter"] > 0
    for schedule in ("ARROY_B200_LOCKSTEP", "ARROY_B200_PROFILE"):   # (the profiled build times its steps with events)
        monkeypatch.setenv(schedule, "1")
        assert ctx.build_trees(seeds, list(range(T)), T) == nodes
        monkeypatch.delenv(schedule)

    ctx.load_forest(roots=np.arange(T, dtype=np.uint32), **forest_arrays(nodes, oracle.EUCLIDEAN, d))
    for nq in (3, 300):
        assert not ctx.search_batch(10, query_rows=np.arange(nq, dtype=np.uint32))[3].any()
    queries = np.arange(40, dtype=np.uint32)
    s0 = ctx.search_stats()
    for rows in (np.arange(0, n, 2), np.arange(5)):   # a filter the queries walk, and one that takes the small-filter shortcut
        assert not ctx.search_batch_filtered(10, row_bitmap(rows, n), query_rows=queries)[3].any()
    s1 = ctx.search_stats()
    assert s1["shortcut_queries"] > s0["shortcut_queries"]
    assert s1["filtered_queries"] - s1["shortcut_queries"] > s0["filtered_queries"] - s0["shortcut_queries"]
    assert not ctx.search_batch_multi_filtered(10, [np.arange(0, n, 3), np.arange(100)], queries % 2, query_rows=queries)[3].any()

    q = data[:8]
    cand = np.arange(0, n, 16, dtype=np.uint32)
    offsets = np.arange(9, dtype=np.uint64) * np.uint64(cand.size)
    c0 = ctx.counters()["fused_rerank_batches"]
    ctx.rerank_batch(q, None, np.tile(cand, 8), offsets, 10)     # the fused re-rank
    assert ctx.counters()["fused_rerank_batches"] == c0 + 1
    ctx.rerank_batch(q, None, np.tile(cand, 8), offsets, 2100)   # more than it keeps: the plain kernels
    ctx.rerank_shared(q, None, cand, 10)
    ctx.prefilter_scores(q, cand, engine=1)                       # cuBLAS
    ctx.side_batch(data[0], (0.0, 0.0), cand)
    pool, ptrs = leaf_pointers(data)
    ctx.stage_items_delta("euclidean", d, ids, ptrs, np.array([5, 77], dtype=np.uint32))
    assert ctx.stage_stats()["delta"] == 1
    del pool

    bq_n, bq_T = 3000, 2
    ctx.stage_items_flat("binary quantized euclidean", ids[:bq_n], data[:bq_n])
    bq_nodes = ctx.build_trees(seeds[:bq_T], list(range(bq_T)), bq_T, split_after=d)
    ctx.load_forest(roots=np.arange(bq_T, dtype=np.uint32), **forest_arrays(bq_nodes, oracle.BQ_EUCLIDEAN, d))
    assert not ctx.search_batch(10, query_rows=queries)[3].any()
    qv = np.stack([bq_quantize(v) for v in data[:4]])
    assert not ctx.search_batch(10, queries=qv, qhdr0=np.zeros(4, np.float32))[3].any()

    monkeypatch.setenv("ARROY_B200_HOST_ITEMS", "1")
    ctx.stage_items_flat("euclidean", ids[:bq_n], data[:bq_n])
    monkeypatch.delenv("ARROY_B200_HOST_ITEMS")
    assert ctx.item_placement()["placement"] == "host"
    ctx.build_trees(seeds[:bq_T], list(range(bq_T)), bq_T)
    ctx.rerank_batch(q, None, np.tile(ids[:bq_n], 8), np.arange(9, dtype=np.uint64) * np.uint64(bq_n), 10)   # the plane pre-filter
    assert ctx.plane_rerank_stats()["batches"] == 1

    with pytest.raises(ab.ArroyB200Error):
        ctx.stage_items_flat("euclidean", np.array([2, 1], dtype=np.uint32), np.zeros((2, d), np.float32))
    ctx.stage_begin("euclidean", d, ids[:100])   # never ended


@pytest.mark.gpu
def test_closing_a_context_frees_everything_it_allocated(monkeypatch):
    start = census()
    for _ in range(3):
        ctx = ab.Context(0)
        exercise(ctx, monkeypatch)
        assert census() != start
        ctx.close()
        assert census() == start
    g = ab.Group([0])
    g.close()
    assert census() == start
