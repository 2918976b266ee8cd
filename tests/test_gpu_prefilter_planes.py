"""The device encoder of side()'s 8-bit pre-filter (kernels.cuh planes_encode_kernel) produces exactly the planes and scales of
the numpy restatement in test_prefilter_planes_cpu.py, so the CPU proof of the decision rules speaks for the device; and the
build's per-stage row counts are consistent with the older two-stage accounting."""
import numpy as np
import pytest

import arroy_b200 as ab
import oracle
from test_prefilter_planes_cpu import encode

pytestmark = pytest.mark.gpu
SEED = bytes([42] * 32)


@pytest.fixture(scope="module")
def ctx():
    c = ab.Context(0)
    yield c
    c.close()


def rows_for(n, d, seed):
    rng = np.random.default_rng(seed)
    rows = (rng.standard_normal((n, d)) * rng.choice([1e-30, 1e-3, 1.0, 1e30], size=(n, 1))).astype(np.float32)
    rows[rng.integers(0, n, size=n // 10), rng.integers(0, d, size=n // 10)] *= 1000.0
    rows[0] = 0.0
    rows[1, d - 1] = np.nan
    rows[2, d // 2] = -np.inf
    rows[3] = 0.0
    rows[3, 1] = -1e-37
    return rows


@pytest.mark.parametrize("n,d", [(1000, 64), (777, 200), (300, 1000), (33, 8192)])
def test_device_planes_equal_the_restatement(ctx, n, d):
    rows = rows_for(n, d, n + d)
    ctx.stage_items_flat("euclidean", np.arange(n, dtype=np.uint32), rows)
    ld = (d + 31) // 32 * 32
    hi, lo, s = ctx.prefilter_planes(n, ld)
    whi, wlo, ws = encode(rows, ld)
    assert np.array_equal(s.view(np.uint32), ws.view(np.uint32))
    assert np.array_equal(hi, whi)
    assert np.array_equal(lo, wlo)


def test_restage_rebuilds_the_planes(ctx):
    a, b = rows_for(500, 96, 1), rows_for(500, 96, 2)
    ids = np.arange(500, dtype=np.uint32)
    ctx.stage_items_flat("cosine", ids, a)
    ctx.prefilter_planes(500, 96)
    ctx.stage_items_flat("cosine", ids, b)
    hi, lo, s = ctx.prefilter_planes(500, 96)
    whi, wlo, ws = encode(b, 96)
    assert np.array_equal(s.view(np.uint32), ws.view(np.uint32)) and np.array_equal(hi, whi) and np.array_equal(lo, wlo)


def test_stage_counts(ctx):
    n, d, T = 70_000, 64, 2
    data = oracle.synth_rows(SEED, d, 0, n, 0.5, threads=8)
    ctx.stage_items_flat("euclidean", np.arange(n, dtype=np.uint32), data)
    user = oracle.StdRng(SEED)
    r1 = oracle.StdRng(user.gen_seed())
    ctx.build_trees([r1.gen_seed() for _ in range(T)], list(range(T)), T)
    sh, pf = ctx.build_shadow_stats(), ctx.build_prefilter_stats()
    assert pf["rows_via_prefilter"] == sh["rows_via_bf16_shadow"] > n
    assert pf["rows_rescored_f32"] == sh["rows_rescored_f32"]
    assert 0 < pf["rows_rescored_f32"] <= pf["rows_stage2"] < pf["rows_via_prefilter"]
