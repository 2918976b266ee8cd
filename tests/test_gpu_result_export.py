"""The build's results reach host memory while the wave builds: each control CTA copies its tree's records, the ids of its
leaves and the normals of its splits to mapped pinned host memory as they close (build.cuh export_records), and only the
slots the host pool has no room for are copied after the kernel. Every case compares the forest byte for byte with the oracle
on one schedule or path through that export: the persistent kernel (with its exports in the wait windows), the async graph,
its cluster control kernels, lockstep, several waves, subtree builds, a host pool smaller than the split count, and a
cancelled build followed by a rebuild on the same context."""
import os

import numpy as np
import pytest

import arroy_b200 as ab
import oracle
from arroy_b200 import _capi
from test_gpu_build_schedules import (ASYNC, CLUSTER16, LOCKSTEP, PERSISTENT, SEED, assert_same_forest, build_subtrees,
                                      oracle_forest, schedules, tree_seeds)

pytestmark = pytest.mark.gpu
THREADS = min(os.cpu_count() or 4, 32)
NORMAL_HDR = 4          # floats ahead of each normal in a pool slot (kernels.cuh)
TREE_STATE_BYTES = 96   # sizeof(TreeState) (build.cuh): read back per tree after the kernel


@pytest.fixture(scope="module")
def ctx():
    c = ab.Context(0)
    yield c
    c.close()


def export_bytes(nodes, n_rows, d, n_trees):
    """What a build writes to host memory: every record (16 B per node), every row's id once per tree, one pool slot
    (header + normal, ld + 4 floats) per split that has a normal, and the tree states read back after the kernel."""
    ld = (d + 31) // 32 * 32
    normals = sum(1 for b in nodes.values() if b[0] == 2 and len(b) > 9)
    return 16 * len(nodes) + 4 * n_rows + 4 * (ld + NORMAL_HDR) * normals + TREE_STATE_BYTES * n_trees


def build_and_check(ctx, metric, data, T, split_after, want_sched, user_seed=SEED, check_bytes=True):
    n, d = data.shape
    ctx.stage_items_flat(metric, np.arange(n, dtype=np.uint32), data)

    def build():
        c0 = ctx.counters()
        got = ctx.build_trees(tree_seeds(user_seed, T), list(range(T)), T, split_after)
        return got, ctx.counters()["d2h_bytes"] - c0["d2h_bytes"], ctx.build_breakdown()
    got, d2h, bd = build()
    sched = schedules(ctx)
    assert sched & want_sched == want_sched, (sched, want_sched)
    odb = oracle_forest(metric, np.arange(n, dtype=np.uint32), data, user_seed, T, split_after)
    assert_same_forest(got, odb.nodes(), (metric, n, d, T))
    assert ctx.build_stats()["scanned_rows"] == odb.scanned_rows
    if check_bytes:
        if bd["late_pool_slots"]:
            # the first build of these shapes used more slots than the host pool's first estimate (2 per expected leaf); the
            # same build again finds a pool sized from what that one used
            again, d2h, bd = build()
            assert again == got and bd["late_pool_slots"] == 0, bd
        assert d2h == export_bytes(got, n * T, d, T)
    return got, bd


def test_persistent_schedule(ctx):
    data = oracle.synth_rows(SEED, 96, 0, 20_000, 0.5, threads=THREADS)
    build_and_check(ctx, "cosine", data, 4, 64, PERSISTENT)


def test_async_graph(ctx):
    data = oracle.synth_rows(SEED, 2144, 0, 4000, 0.5, threads=THREADS)
    build_and_check(ctx, "euclidean", data, 3, 32, ASYNC)


def test_lockstep(ctx, monkeypatch):
    monkeypatch.setenv("ARROY_B200_LOCKSTEP", "1")
    data = oracle.synth_rows(SEED, 96, 0, 20_000, 0.5, threads=THREADS)
    build_and_check(ctx, "manhattan", data, 3, 64, LOCKSTEP)


def test_several_waves(ctx, monkeypatch):
    # 5 trees in waves of 2, 2 and 1: each wave has its own host buffers
    monkeypatch.setenv("ARROY_B200_MAX_WAVE", "2")
    data = oracle.synth_rows(SEED, 128, 0, 12_000, 0.0, threads=THREADS)
    build_and_check(ctx, "euclidean", data, 5, 64, PERSISTENT)


@pytest.mark.parametrize("d,want", [(96, PERSISTENT), (2144, ASYNC)], ids=["persistent", "async"])
def test_host_pool_smaller_than_the_splits(ctx, monkeypatch, d, want):
    # ten slots of host pool: the kernel exports the normals in slots below 10, the host copies the rest after the kernel
    monkeypatch.setenv("ARROY_B200_EXPORT_SLOTS", "10")
    data = oracle.synth_rows(SEED, d, 0, 6000, 0.5, threads=THREADS)
    _, bd = build_and_check(ctx, "cosine", data, 3, 32, want, check_bytes=False)
    assert bd["late_pool_slots"] > 0, bd
    monkeypatch.delenv("ARROY_B200_EXPORT_SLOTS")
    # ... and the next build of the same shapes sizes its pool from the slots this one used
    _, bd = build_and_check(ctx, "cosine", data, 3, 32, want)
    assert bd["late_pool_slots"] == 0, bd


def test_subtrees(ctx):
    n, d, split_after = 30_000, 96, 64
    data = oracle.synth_rows(SEED, d, 0, n, 0.5, threads=THREADS)
    ctx.stage_items_flat("cosine", np.arange(n, dtype=np.uint32), data)
    rng = np.random.default_rng(5)
    subsets = [np.sort(rng.choice(n, size=s, replace=False)).astype(np.uint32) for s in (500, 4000, 12_000)]
    user_seeds = [bytes([s + 1] * 32) for s in range(len(subsets))]
    c0 = ctx.counters()
    got = build_subtrees(ctx, [tree_seeds(u, 1)[0] for u in user_seeds], subsets, split_after)
    c1 = ctx.counters()
    assert schedules(ctx) & PERSISTENT
    for s, rows in enumerate(subsets):
        odb = oracle_forest("cosine", rows, data[rows], user_seeds[s], 1, split_after, threads=1)
        assert_same_forest(got[s], odb.nodes(), ("subtree", s))
    total_nodes = {i: b for s in range(len(subsets)) for i, b in ((s << 22 | k, v) for k, v in got[s].items())}
    assert c1["d2h_bytes"] - c0["d2h_bytes"] == export_bytes(total_nodes, sum(r.size for r in subsets), d, len(subsets))


def test_cluster_control_kernels(ctx):
    # the schedule rule looks at the staged n: 8 small subtrees of a 25 000 064-row index run clusters of 16 CTAs per tree
    import torch
    big_n, d, window, split_after = 25_000_064, 64, 60_000, 64
    t = torch.empty((big_n, d), dtype=torch.float32, device="cuda:0")
    ctx.synth_device(SEED, d, 0, big_n, 0.5, t.data_ptr())
    torch.cuda.synchronize()
    ctx.stage_items_device("euclidean", np.arange(big_n, dtype=np.uint32), d, t.data_ptr())
    del t
    torch.cuda.empty_cache()
    rows_w = oracle.synth_rows(SEED, d, 0, window, 0.5, threads=THREADS)
    rng = np.random.default_rng(16)
    subsets = [np.sort(rng.choice(window, size=int(s), replace=False)).astype(np.uint32) for s in rng.integers(2000, 8000, 8)]
    user_seeds = [bytes([s + 40] * 32) for s in range(len(subsets))]
    got = build_subtrees(ctx, [tree_seeds(u, 1)[0] for u in user_seeds], subsets, split_after)
    assert schedules(ctx) & CLUSTER16, schedules(ctx)
    for s, rows in enumerate(subsets):
        odb = oracle_forest("euclidean", rows, rows_w[rows], user_seeds[s], 1, split_after, threads=1)
        assert_same_forest(got[s], odb.nodes(), ("cluster subtree", s))


@pytest.mark.parametrize("d,want", [(96, PERSISTENT), (2144, ASYNC)], ids=["persistent", "async"])
def test_cancelled_build_then_rebuild(ctx, d, want):
    # a build cancelled mid-kernel leaves partial results in the host buffers; the rebuild on the same context must not see them
    n, T, split_after = (60_000 if d == 96 else 4000), 4, 32
    data = oracle.synth_rows(SEED, d, 0, n, 0.5, threads=THREADS)
    ctx.stage_items_flat("cosine", np.arange(n, dtype=np.uint32), data)
    polls = []

    def cancel():
        polls.append(1)
        return len(polls) >= 2   # the first poll is before the build, the second while its kernels run
    with pytest.raises(ab.ArroyB200Error) as ei:
        ctx.build_trees(tree_seeds(bytes([3] * 32), T), list(range(T)), T, split_after, cancel=cancel)
    assert ei.value.code == _capi.ERR_CANCELLED
    build_and_check(ctx, "cosine", data, T, split_after, want)
