"""Stage 2 of the 8-bit pre-filter (kernels.cuh scan_claim_planes) reads only the lo plane: stage 1 forms every hi-plane sum while
it streams the hi row and keeps them, with the row's position, for the rows it leaves. These tests pin that hand-off: rows left in
both 128-row blocks of a claim and in a short last block, rows whose words do not fill the last 8-lane step (d = 96, 800, 2080),
the DotProduct header term, the largest hi-plane sums at d = 8192, and claims whose every row goes to stage 2. Each case compares
the stage counts with the numpy restatement, the Left count with the f32 scan's, and every row's flag (host-placed items, whose
routing goes through the planes) with the f32 flag."""
import numpy as np
import pytest

import arroy_b200 as ab
from arroy_b200 import _capi
from test_prefilter_dp4a_cpu import decide_planes
from test_prefilter_planes_cpu import make_case

pytestmark = pytest.mark.gpu
F32 = np.float32
CLAIM = 256     # rows of one scan_claim_planes call: two stage-1 blocks of 128


def counts_and_left(metric, normal, nh0, rows, ih0, sel, gathered):
    """(restated stage-1 certain, stage-2 certain over sel, device prefilter stats, Left of variant 1, Left of the f32 scan)"""
    n, d = rows.shape
    ld = (d + 31) // 32 * 32
    ctx = ab.Context(0)
    try:
        ctx.stage_items_flat(metric, np.arange(n, dtype=np.uint32), rows, hdr0=ih0 if metric == "dot-product" else None)
        hi, lo, s = ctx.prefilter_planes(n, ld)
        nrm = np.zeros(ld, dtype=np.float32)
        nrm[:d] = normal
        c1, _, c2, _ = decide_planes(metric, nrm, nh0, hi[sel], lo[sel], s[sel], ih0[sel], d)
        arg = sel if gathered else None
        _, left = ctx.time_scan(normal, (nh0, 0.0), sel.size, rows=arg, iters=1, flush_l2=False, variant=1)
        st = ctx.build_prefilter_stats()
        _, left_f32 = ctx.time_scan(normal, (nh0, 0.0), sel.size, rows=arg, iters=1, flush_l2=False, variant=0)
    finally:
        ctx.close()
    return c1, c2, st, left, left_f32


def flags_through_planes(metric, normal, nh0, rows, ih0, sel, monkeypatch):
    """(flags of side_multi, which scans host-placed items through scan_claim_planes, flags of the f32 side_batch) over sel"""
    n = rows.shape[0]
    monkeypatch.setenv("ARROY_B200_HOST_ITEMS", "1")
    ctx = ab.Context(0)
    try:
        ctx.stage_items_flat(metric, np.arange(n, dtype=np.uint32), rows, hdr0=ih0 if metric == "dot-product" else None)
        monkeypatch.delenv("ARROY_B200_HOST_ITEMS")
        assert ctx.item_placement()["placement"] == "host"
        nrm = np.ascontiguousarray(normal, dtype=np.float32)
        h0 = np.array([nh0], dtype=np.float32)
        r = np.ascontiguousarray(sel, dtype=np.uint32)
        offs = np.array([0, r.size], dtype=np.uint64)
        got = np.empty(r.size, dtype=np.uint8)
        ctx._ck(ctx.lib.arroy_b200_side_multi(ctx.h, 1, _capi._fp(nrm), _capi._fp(h0), None, _capi._up(r),
                                              offs.ctypes.data_as(_capi._u64p), got.ctypes.data_as(_capi._u8p)))
        want, _ = ctx.side_batch(nrm, (nh0, 0.0), r)
    finally:
        ctx.close()
    return got, want


def check(metric, normal, nh0, rows, ih0, sel, gathered, monkeypatch):
    c1, c2, st, left, left_f32 = counts_and_left(metric, normal, nh0, rows, ih0, sel, gathered)
    assert st["rows_via_prefilter"] == sel.size
    assert st["rows_stage2"] == int((~c1).sum()) > 0
    assert st["rows_rescored_f32"] == int((~c1 & ~c2).sum())
    assert left == left_f32
    got, want = flags_through_planes(metric, normal, nh0, rows, ih0, sel, monkeypatch)
    assert got.tobytes() == want.tobytes(), np.flatnonzero(got != want)[:10]
    return c1, c2, st


# (metric, d, rows scanned, through an id list): d = 96, 800 and 2080 leave 6, 50 and 130 16-byte words per plane row, so the
# last 8-lane step of both stages has masked words; 1000 and 300 rows end in a short claim
@pytest.mark.parametrize("metric,d,n_rows,gathered", [("cosine", 96, 1000, False), ("dot-product", 96, 1000, True),
                                                      ("euclidean", 800, 300, True), ("dot-product", 800, 300, False),
                                                      ("manhattan", 2080, 300, True)])
def test_kept_sums_over_both_blocks_and_a_short_claim(metric, d, n_rows, gathered, monkeypatch):
    normal, nh0, rows, ih0 = make_case(metric, d, 5 * d + n_rows)
    n = rows.shape[0]
    sel = np.random.default_rng(d).permutation(n)[:n_rows].astype(np.uint32) if gathered else np.arange(n_rows, dtype=np.uint32)
    c1, _, _ = check(metric, normal, nh0, rows, ih0, sel, gathered, monkeypatch)
    left_pos = np.flatnonzero(~c1)
    assert (left_pos % CLAIM < 128).any() and (left_pos % CLAIM >= 128).any()     # both stage-1 blocks of a claim
    assert (left_pos >= (n_rows - 1) // CLAIM * CLAIM).any()                       # and the short last claim


def test_largest_hi_sums_at_the_largest_d(monkeypatch):
    """d = PLANES_MAX_D, every normal element a limb a = +-127 and U = 254, and its third limb c = +-127 with the sign of a
    pattern w (half +1, half -1) whose second limbs b are equal: rows at +-127 s along sign(n) w have sum h a = sum h b = 0, so
    stage 1 leaves them, with sum h c = +-127 * 127 * 8192 and sum |h| U = 127 * 254 * 8192, the largest the kernel keeps. Rows
    of test_largest_sums_at_the_largest_d's kinds (aligned, opposed, random signs, half and half) fill the other outcomes."""
    d = 8192
    rng = np.random.default_rng(12)
    cand = np.arange(F32(126.5).view(np.uint32) + 1, F32(127.0).view(np.uint32), dtype=np.uint32).view(np.float32)
    t = cand.astype(np.float64)                               # sigma = 1: the limbs of v in [126.5, 127)
    a = np.rint(t)
    r1 = 254.0 * (t - a)
    b = np.rint(r1)
    c = np.rint(254.0 * (r1 - b))
    beta = sorted(set(b[c == 127]) & set(b[c == -127]))[0]
    v_plus, v_minus = cand[(c == 127) & (b == beta)][0], cand[(c == -127) & (b == beta)][0]
    sg = np.where(rng.random(d) < 0.5, F32(-1), F32(1)).astype(np.float32)
    w = np.where(rng.permutation(d) < d // 2, F32(1), F32(-1)).astype(np.float32)
    normal = (sg * np.where(w > 0, v_plus, v_minus)).astype(np.float32)
    rows = np.empty((160, d), dtype=np.float32)
    rows[:32] = 127.0 * sg * w
    rows[32:64] = -127.0 * sg * w
    rows[64:80] = 127.0 * sg
    rows[80:96] = -127.0 * sg
    rows[96:128] = 127.0 * np.where(rng.random((32, d)) < 0.5, -1.0, 1.0)
    half = np.where(np.arange(d) < d // 2, 1.0, -1.0)
    rows[128:] = 127.0 * sg * np.stack([half[rng.permutation(d)] for _ in range(32)])
    rows *= np.float32(2.0 ** -7)
    ih0 = np.zeros(rows.shape[0], dtype=np.float32)
    sel = np.arange(rows.shape[0], dtype=np.uint32)
    c1, _, _ = check("cosine", normal, 0.0, rows, ih0, sel, False, monkeypatch)
    assert not c1[:64].any() and c1[64:96].all()


def near_plane_case(metric, d):
    """(normal, nh0, rows, ih0, id list): rows on the normal's hyperplane or 0.3 % of their length off it, in shuffled order"""
    rng = np.random.default_rng(d)
    n = 2 * CLAIM + 77
    normal = rng.standard_normal(d).astype(np.float32)
    x = rng.standard_normal((n, d)) * rng.choice([1e-2, 1.0, 100.0], size=(n, 1))
    nn = normal.astype(np.float64)
    off = rng.choice([0.0, 3e-3, -3e-3], size=n) * np.linalg.norm(x, axis=1) / np.linalg.norm(nn)
    rows = (x - np.outer(x @ nn / (nn @ nn) - off, nn)).astype(np.float32)
    nh0 = 0.37 if metric == "dot-product" else 0.0
    ih0 = (np.abs(rng.standard_normal(n)) * 1e-6).astype(np.float32) if metric == "dot-product" else np.zeros(n, dtype=np.float32)
    return normal, nh0, rows, ih0, rng.permutation(n).astype(np.uint32)


@pytest.mark.parametrize("metric,d", [("cosine", 800), ("dot-product", 2080)])
def test_every_row_through_stage_2(metric, d, monkeypatch):
    """Rows at most 0.3 % of their length off the normal's hyperplane: stage 1 decides none of them, so every claim keeps the
    sums of all its rows (two full claims and a short one), and stage 2 decides a part of them."""
    normal, nh0, rows, ih0, sel = near_plane_case(metric, d)
    _, _, st = check(metric, normal, nh0, rows, ih0, sel, True, monkeypatch)
    assert st["rows_stage2"] == sel.size
