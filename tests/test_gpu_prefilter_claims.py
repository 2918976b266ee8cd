"""The 8-bit pre-filter scan (kernels.cuh scan_claim_planes) takes each claim's row ids, scales and DotProduct headers into shared
memory once and reads them from there in all three stages. These tests pin what depends on that bookkeeping: claims over an id
list (not the identity), claims whose row count is not a multiple of the 128-row stage-1 block, the DotProduct header term, and
forests of the persistent, lockstep and async schedules against the oracle, with the pre-filter counters pinned."""
import numpy as np
import pytest

import arroy_b200 as ab
import oracle
from test_gpu_build_schedules import ASYNC, LOCKSTEP, PERSISTENT, assert_same_forest, device_forest, oracle_forest, schedules
from test_prefilter_dp4a_cpu import decide_planes
from test_prefilter_planes_cpu import make_case

pytestmark = pytest.mark.gpu
SEED = bytes([7] * 32)


@pytest.mark.parametrize("metric,d,n_rows", [("cosine", 768, 1000), ("dot-product", 768, 1000), ("euclidean", 96, 129),
                                             ("manhattan", 1000, 300), ("dot-product", 200, 383)])
def test_claims_over_an_id_list(metric, d, n_rows):
    """time_scan variant 1 over a shuffled subset of the rows: claims of 256 positions whose last one is cut short; every stage
    reads the ids, scales and headers of its positions, so the stage counts equal the restatement's on those rows and the Left
    count equals the f32 scan's over the same id list."""
    normal, nh0, rows, ih0 = make_case(metric, d, 3 * d + n_rows)
    n = rows.shape[0]
    assert n >= n_rows
    ld = (d + 31) // 32 * 32
    sel = np.random.default_rng(d + n_rows).permutation(n)[:n_rows].astype(np.uint32)
    ctx = ab.Context(0)
    try:
        ctx.stage_items_flat(metric, np.arange(n, dtype=np.uint32), rows, hdr0=ih0 if metric == "dot-product" else None)
        hi, lo, s = ctx.prefilter_planes(n, ld)
        nrm = np.zeros(ld, dtype=np.float32)
        nrm[:d] = normal
        c1, _, c2, _ = decide_planes(metric, nrm, nh0, hi[sel], lo[sel], s[sel], ih0[sel], d)
        _, left = ctx.time_scan(normal, (nh0, 0.0), n_rows, rows=sel, iters=1, flush_l2=False, variant=1)
        st = ctx.build_prefilter_stats()
        _, left_f32 = ctx.time_scan(normal, (nh0, 0.0), n_rows, rows=sel, iters=1, flush_l2=False, variant=0)
    finally:
        ctx.close()
    assert st["rows_via_prefilter"] == n_rows
    assert st["rows_stage2"] == int((~c1).sum())
    assert st["rows_rescored_f32"] == int((~c1 & ~c2).sum())
    assert 0 < st["rows_stage2"]
    assert left == left_f32


# (metric, schedule, d, n, trees) -> the pre-filter counters (rows_via_prefilter, rows_stage2, rows_rescored_f32) of the build.
# Every node above 12 scan units goes through the pre-filter: on the persistent kernel's workers (32 trees), on work_kernel_planes
# in the lockstep schedule, and in the async graph (rows wider than 2048 floats). Node sizes are arbitrary, so most claims end
# inside a 128-row block. The counters are those the builds gave before claims kept their ids and scales in shared memory.
FOREST_CASES = {
    ("cosine", "persistent", 768, 9000, 32): (864000, 106041, 986),
    ("dot-product", "persistent", 768, 9000, 32): (1504975, 126691, 1222),
    ("euclidean", "lockstep", 768, 9000, 32): (1273763, 286375, 2789),
    ("dot-product", "lockstep", 768, 9000, 32): (1792975, 148846, 1431),
    ("cosine", "async", 2080, 5000, 3): (45000, 9087, 152),
    ("manhattan", "async", 2080, 5000, 3): (49694, 9700, 222),
}


def build_case(metric, schedule, d, n, T, monkeypatch):
    """(device forest, build_stats, schedule bits, pre-filter counters)"""
    if schedule == "lockstep":
        monkeypatch.setenv("ARROY_B200_LOCKSTEP", "1")
    else:
        monkeypatch.delenv("ARROY_B200_LOCKSTEP", raising=False)
    data = data_of(metric, d, n)
    ctx = ab.Context(0)
    try:
        got = device_forest(ctx, metric, data, T, 64, user_seed=SEED)
        st, sched, pre = ctx.build_stats(), schedules(ctx), ctx.build_prefilter_stats()
    finally:
        ctx.close()
    counts = (pre["rows_via_prefilter"], pre["rows_stage2"], pre["rows_rescored_f32"])
    return got, st, sched, counts


@pytest.mark.parametrize("case", list(FOREST_CASES), ids=lambda c: "-".join(map(str, c)))
def test_forests_through_the_prefilter_match_the_oracle(case, monkeypatch):
    metric, schedule, d, n, T = case
    got, st, sched, counts = build_case(metric, schedule, d, n, T, monkeypatch)
    odb = oracle_forest(metric, np.arange(n, dtype=np.uint32), data_of(metric, d, n), SEED, T, 64)
    assert_same_forest(got, odb.nodes(), case)
    assert st["scanned_rows"] == odb.scanned_rows
    assert sched & {"persistent": PERSISTENT, "lockstep": LOCKSTEP, "async": ASYNC}[schedule], sched
    assert counts == FOREST_CASES[case], counts


def data_of(metric, d, n):
    return oracle.synth_rows(SEED, d, 0, n, 0.0 if metric == "euclidean" else 0.5, threads=8)
