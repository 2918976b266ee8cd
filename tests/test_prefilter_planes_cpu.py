"""The two-plane 8-bit pre-filter of side() (kernels.cuh planes_encode_kernel / scan_claim_planes), restated in numpy and checked
on the CPU against the oracle's margins: every row that stage 1 (hi plane) or stage 2 (hi + lo planes) calls certain must have
the sign of the margin the reference computes from the f32 row in its own summation order. The sums are taken in the kernel's
lane order (eight lanes per row, two f32 chains per lane, then a butterfly). The rows include ones built on the decision
boundary, mixed magnitudes, rows with one dominant element, zero and non-finite rows, and rows whose quantization error is
aligned with the normal, so that a rule with half the bound makes wrong calls (test_half_the_bound_is_caught)."""
import numpy as np
import pytest

import oracle

F32 = np.float32
TINY = np.finfo(np.float32).tiny
FMAX = np.finfo(np.float32).max


def k1(d):
    return F32(0.5002) + F32(d) * F32(8.6e-6)


def w2(d):
    return F32(0.50216) * (F32(1.0) + F32(6.1e-8) * F32(d + 16))


def rel2(d):
    return F32(1.3e-6) + F32(d) * F32(6.8e-8)


def encode(rows, ld):
    """planes_encode_kernel: (hi int8 n x ld, lo int8 n x ld, scale f32 n)."""
    n, d = rows.shape
    x = np.zeros((n, ld), dtype=np.float32)
    x[:, :d] = rows
    bits = np.abs(x).view(np.uint32).max(axis=1)           # NaN sorts above +inf as bits
    with np.errstate(all="ignore"):
        s = (bits.view(np.float32) / F32(127)).astype(np.float32)
    ok = (s >= TINY) & (s <= FMAX)
    s.view(np.uint32)[~ok & (bits != 0) & (bits != 0x7F800000)] = 0x7FFFFFFF
    hi = np.zeros((n, ld), dtype=np.int8)
    lo = np.zeros((n, ld), dtype=np.int8)
    q = x[ok] / s[ok, None]
    h = np.rint(q)
    hi[ok] = h.astype(np.int8)
    lo[ok] = np.rint((q - h) * F32(254)).astype(np.int8)
    return hi, lo, s


def fma32(a, b, c):
    return (a.astype(np.float64) * b.astype(np.float64) + c.astype(np.float64)).astype(np.float32)


def lane_sum(v, nrm, absolute=False):
    """f32 sum of v * nrm over a row in scan_claim_planes' order (v: n x ld, nrm: ld)."""
    n, ld = v.shape
    nq = ld // 16
    if absolute:
        v, nrm = np.abs(v), np.abs(nrm)
    acc = [np.zeros((n, 8), dtype=np.float32), np.zeros((n, 8), dtype=np.float32)]
    for c in range((nq + 7) // 8):
        g = np.arange(8)
        live = 8 * c + g < nq
        g = g[live]
        for e in range(16):
            idx = 16 * (8 * c + g) + e
            a = acc[e & 1]
            a[:, live] = fma32(v[:, idx], nrm[idx][None, :], a[:, live])
    t = acc[0] + acc[1]
    t = t[:, 0::2] + t[:, 1::2]
    t = t[:, 0::2] + t[:, 1::2]
    return t[:, 0] + t[:, 1]


def up32(x):
    f = np.float32(x)
    return np.nextafter(f, F32(np.inf)) if float(f) < x else f


def with_c(metric, v, nh0, ih0):
    if metric == "cosine":
        return v
    if metric == "dot-product":
        return v + (F32(nh0) * ih0).astype(np.float32)
    return F32(nh0) + v


def decide(metric, normal, nh0, rows, ih0, factor=1.0):
    """(stage-1 certain, stage-2 certain, side called) for every row; factor scales the bounds."""
    n, d = rows.shape
    ld = (d + 31) // 32 * 32
    nrm = np.zeros(ld, dtype=np.float32)
    nrm[:d] = normal
    hi, lo, s = encode(rows, ld)
    n1 = np.abs(nrm.astype(np.float64)).sum() * (1.0 + 2.0 ** -30)
    f = F32(factor)
    w1 = up32(n1 * float(k1(d))) * f
    w2j = up32(n1 * float(w2(d))) * f
    with np.errstate(all="ignore"):
        t = lane_sum(hi.astype(np.float32), nrm)
        mt1 = with_c(metric, s * t, nh0, ih0)
        c1 = np.abs(mt1) > s * w1
        y = hi.astype(np.float32) * F32(254) + lo.astype(np.float32)
        m = lane_sum(y, nrm)
        a = lane_sum(y, nrm, absolute=True)
        s2 = s / F32(254)
        mt2 = with_c(metric, s2 * m, nh0, ih0)
        c2 = np.abs(mt2) > s2 * (w2j + rel2(d) * f * a)
    return c1, mt1 > 0, c2, mt2 > 0


def greedy_half(absn, frac=0.45):
    """a 0/1 mask whose |n|-weighted sum is just below frac * |n|_1"""
    order = np.argsort(-absn)
    b = np.zeros(absn.size, dtype=bool)
    tot, goal = 0.0, frac * float(absn.sum())
    for i in order:
        if tot + absn[i] <= goal:
            b[i] = True
            tot += absn[i]
    return b


def make_case(metric, d, seed):
    rng = np.random.default_rng(seed)
    n = 3000 if d <= 768 else 300
    normal = (rng.standard_normal(d) * rng.choice([1e-3, 1.0, 30.0], size=d)).astype(np.float32)
    normal[0] = 0.0    # the adversarial rows below put their largest element here
    rows = (rng.standard_normal((n, d)) * rng.choice([1e-2, 1.0, 100.0], size=(n, 1))).astype(np.float32)
    dom = rng.random(n) < 0.1                                   # one dominant element: a large scale for the rest
    rows[dom, rng.integers(0, d, size=n)[dom]] *= 1000.0
    nn = normal.astype(np.float64)
    proj = (rows.astype(np.float64) @ nn) / (nn @ nn)
    eps = rng.choice([0.0, 1e-7, -1e-7, 1e-4, -1e-4, 3e-3, -3e-3], size=n)
    near = rng.random(n) < 0.6                                  # on the hyperplane up to rounding, or a tiny step off it
    rows[near] = (rows[near].astype(np.float64) - np.outer(proj[near] - eps[near] * np.abs(proj[near] + 1e-3), nn)).astype(np.float32)
    # quantization error aligned with the normal, the f32 dot a small step to the other side of the plane than the encoded one
    sg = np.sign(normal).astype(np.float32)
    b = greedy_half(np.abs(normal))
    k = n // 10
    adv = rng.permutation(n)[:2 * k]
    for j, r in enumerate(adv):
        sigma = F32(1 if j % 2 else -1)
        sc = F32(2.0 ** int(rng.integers(-9, 3)))
        if j < k:      # stage 1: h = -sigma sign(n) on the subset, x/s = h + 0.49 sigma sign(n)
            xs = np.where(b, -sigma * sg, F32(0)) + F32(0.49) * sigma * sg
        else:          # stage 2: h = 0, l = -sigma sign(n) on the subset, x/s = l/254 + 0.49/254 sigma sign(n)
            xs = (np.where(b, -sigma * sg, F32(0)) + F32(0.49) * sigma * sg) / F32(254)
        xs[0] = 127.0
        rows[r] = (xs * sc).astype(np.float32)
    zero = rng.permutation(n)[:5]
    rows[zero] = 0.0
    rows[zero[0], 3] = np.nan
    rows[zero[1], 5] = np.inf
    rows[zero[2], 1] = 1e-37                                     # a scale below FLT_MIN
    if metric in ("euclidean", "manhattan"):
        nh0 = float(np.float32(rng.standard_normal() * 1e-4))
    elif metric == "dot-product":
        nh0 = float(np.float32(0.37))                           # normal.extra_dim
    else:
        nh0 = 0.0
    ih0 = (np.abs(rng.standard_normal(n)) * 1e-4).astype(np.float32) if metric == "dot-product" else np.zeros(n, dtype=np.float32)
    return normal, nh0, rows, ih0


def reference_sides(metric, normal, nh0, rows, ih0):
    side, _ = oracle.side_batch(oracle.METRICS[metric], normal, (nh0, 0.0), rows, ih0, np.zeros_like(ih0), np.arange(rows.shape[0]))
    return side.astype(bool)


CASES = [("cosine", 64), ("euclidean", 96), ("manhattan", 200), ("cosine", 768), ("dot-product", 768), ("euclidean", 768),
         ("manhattan", 1000), ("dot-product", 8192)]


@pytest.mark.parametrize("metric,d", CASES)
def test_certain_rows_have_the_reference_sign(metric, d):
    normal, nh0, rows, ih0 = make_case(metric, d, d * 11 + len(metric))
    ref = reference_sides(metric, normal, nh0, rows, ih0)
    c1, r1, c2, r2 = decide(metric, normal, nh0, rows, ih0)
    assert not np.any(c1 & (r1 != ref)), np.flatnonzero(c1 & (r1 != ref))[:10]
    assert not np.any(c2 & (r2 != ref)), np.flatnonzero(c2 & (r2 != ref))[:10]
    n = rows.shape[0]
    assert 0 < c1.sum() < n and 0 < c2.sum() < n      # both outcomes occur in both stages
    assert c2[~c1].sum() > 0                          # stage 2 decides rows stage 1 left


@pytest.mark.parametrize("metric,d", CASES)
def test_half_the_bound_is_caught(metric, d):
    normal, nh0, rows, ih0 = make_case(metric, d, d * 11 + len(metric))
    ref = reference_sides(metric, normal, nh0, rows, ih0)
    c1, r1, c2, r2 = decide(metric, normal, nh0, rows, ih0, factor=0.5)
    assert np.any(c1 & (r1 != ref)) and np.any(c2 & (r2 != ref))


def test_encoder_bounds_and_special_rows():
    rng = np.random.default_rng(5)
    rows = (rng.standard_normal((400, 200)) * rng.choice([1e-30, 1e-3, 1.0, 1e30], size=(400, 1))).astype(np.float32)
    rows[0] = 0.0
    rows[1, 7] = np.nan
    rows[2, 9] = -np.inf
    rows[3] = 0.0
    rows[3, 0] = 1e-37
    hi, lo, s = encode(rows, 224)
    assert s[0] == 0.0 and s.view(np.uint32)[1] == 0x7FFFFFFF and s[2] == np.inf and s.view(np.uint32)[3] == 0x7FFFFFFF
    assert not hi[:4].any() and not lo[:4].any() and not hi[:, 200:].any() and not lo[:, 200:].any()
    x = rows[4:].astype(np.float64)
    sc = s[4:, None].astype(np.float64)
    h, y = hi[4:, :200].astype(np.float64), hi[4:, :200] * 254.0 + lo[4:, :200]
    assert np.all(np.abs(x - sc * h) <= sc * (0.5 + 128 * 2.0 ** -24))
    assert np.all(np.abs(x - sc * y / 254.0) <= sc * 0.001977)
    assert np.abs(hi).max() == 127 and np.abs(lo).max() <= 127
