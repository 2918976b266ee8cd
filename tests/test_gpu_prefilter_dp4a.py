"""The device's integer pre-filter (kernels.cuh scan_claim_planes, timed through time_scan variant 1) makes exactly the calls of
the numpy restatement in test_prefilter_dp4a_cpu.py, whose rule is checked there against the oracle: on fixed rows and a fixed
normal the rows left by stage 1 and by stage 2 are counted equal, and the Left count is the f32 scan's."""
import numpy as np
import pytest

import arroy_b200 as ab
from test_prefilter_dp4a_cpu import decide_planes
from test_prefilter_planes_cpu import make_case

pytestmark = pytest.mark.gpu
F32 = np.float32


def device_counts(metric, normal, nh0, rows, ih0):
    """(restated stage-1 certain, stage-2 certain, device prefilter stats, Left of variant 1, Left of the f32 scan)"""
    n, d = rows.shape
    ld = (d + 31) // 32 * 32
    ctx = ab.Context(0)
    try:
        ctx.stage_items_flat(metric, np.arange(n, dtype=np.uint32), rows)
        hi, lo, s = ctx.prefilter_planes(n, ld)
        nrm = np.zeros(ld, dtype=np.float32)
        nrm[:d] = normal
        c1, _, c2, _ = decide_planes(metric, nrm, nh0, hi, lo, s, ih0, d)
        _, left = ctx.time_scan(normal, (nh0, 0.0), n, iters=1, flush_l2=False, variant=1)
        st = ctx.build_prefilter_stats()
        _, left_f32 = ctx.time_scan(normal, (nh0, 0.0), n, iters=1, flush_l2=False, variant=0)
    finally:
        ctx.close()
    return c1, c2, st, left, left_f32


@pytest.mark.parametrize("metric,d", [("cosine", 768), ("euclidean", 96), ("manhattan", 1000)])
def test_stage_counts_equal_the_restatement(metric, d):
    normal, nh0, rows, ih0 = make_case(metric, d, 7 * d + len(metric))
    n = rows.shape[0]
    c1, c2, st, left, left_f32 = device_counts(metric, normal, nh0, rows, ih0)
    assert st["rows_via_prefilter"] == n
    assert st["rows_stage2"] == int((~c1).sum())
    assert st["rows_rescored_f32"] == int((~c1 & ~c2).sum())
    assert 0 < st["rows_rescored_f32"] < st["rows_stage2"] < n
    assert left == left_f32


def test_largest_sums_at_the_largest_d():
    """d = PLANES_MAX_D, every row element at +-127 s and every normal element in [126.5, 127) sigma, so every limb a is +-127:
    rows aligned with sign(n) reach the largest int32 sums the kernel can form (127 * 127 * 8192 in magnitude); random-sign rows
    and half-aligned, half-opposed rows (near the hyperplane) fill the other stages. A wrapped int32 sum would flip a certain
    call, and the counts and the Left count would differ from the restatement's and the f32 scan's."""
    d = 8192
    rng = np.random.default_rng(11)
    sg = np.where(rng.random(d) < 0.5, F32(-1), F32(1)).astype(np.float32)
    normal = (sg * rng.uniform(126.5, 126.999, size=d)).astype(np.float32)
    rows = np.empty((96, d), dtype=np.float32)
    rows[:16] = 127.0 * sg
    rows[16:32] = -127.0 * sg
    rows[32:64] = 127.0 * np.where(rng.random((32, d)) < 0.5, -1.0, 1.0)
    half = np.where(np.arange(d) < d // 2, 1.0, -1.0)
    rows[64:] = 127.0 * sg * np.stack([half[rng.permutation(d)] for _ in range(32)])
    rows *= np.float32(2.0 ** -7)
    ih0 = np.zeros(96, dtype=np.float32)
    c1, c2, st, left, left_f32 = device_counts("cosine", normal, 0.0, rows, ih0)
    assert c1[:32].all()                              # the extreme rows are decided by stage 1
    assert st["rows_via_prefilter"] == 96
    assert st["rows_stage2"] == int((~c1).sum()) > 0
    assert st["rows_rescored_f32"] == int((~c1 & ~c2).sum())
    assert left == left_f32
