"""side()'s 8-bit pre-filter on integer dot products (kernels.cuh planes_job_factors / scan_claim_planes), restated in numpy and
checked on the CPU against the oracle's margins. The normal is read as int8 limbs (a + b / 254 for stage 1, + c / 254^2 for
stage 2, and an unsigned bound U of |n|), the plane sums are exact integers, and the bounds carry the normal's limb error D1 / D2
summed per job. The factors are computed in the device's order and rounding (f64 sums over 8 warps x 32 lanes, then rounded
up), so the restatement makes the device's calls row for row (test_gpu_prefilter_dp4a.py checks that on the device)."""
import math
from fractions import Fraction

import numpy as np
import pytest

from test_prefilter_planes_cpu import CASES, encode, make_case, reference_sides

F32 = np.float32


def _ru(x):
    """the least double >= the exact rational x"""
    r = float(x)
    return r if Fraction(r) >= x else math.nextafter(r, math.inf)


def mul_ru(a, b):
    return _ru(Fraction(a) * Fraction(b))


def add_ru(a, b):
    return _ru(Fraction(a) + Fraction(b))


def div_ru(a, b):
    return _ru(Fraction(a) / Fraction(b))


def cta_sum(v):
    """f64 sum in the device's order: thread t sums elements t, t + 256, ...; xor butterfly over 32 lanes; lane 0 of 8 warps."""
    ld = v.size
    acc = np.zeros(256, dtype=np.float64)
    for k in range(0, ld, 256):
        part = v[k:k + 256]
        acc[:part.size] = acc[:part.size] + part
    w = acc.reshape(8, 32)
    for o in (16, 8, 4, 2, 1):
        w = w + w[:, np.arange(32) ^ o]
    s = 0.0
    for x in w[:, 0]:
        s += float(x)
    return s


def limbs(nrm):
    """planes_job_factors: (a, b, c, U as int64 arrays, factors dict). nrm: f32, ld elements."""
    bits = np.abs(nrm).view(np.uint32)
    mb = int(bits.max())
    finite = mb < 0x7F800000
    e = 0
    if finite and mb != 0:
        e = math.frexp(float(np.uint32(mb).view(np.float32)) / 127.0)[1]
    t = nrm.astype(np.float64) * math.ldexp(1.0, -e) if finite else np.zeros(nrm.size)
    a = np.rint(t)
    r1 = 254.0 * (t - a)
    b = np.rint(r1)
    r2 = 254.0 * (r1 - b)
    c = np.rint(r2)
    u = np.ceil(2.0 * np.abs(t))
    with np.errstate(all="ignore"):
        n1s = cta_sum(np.abs(nrm).astype(np.float64))
    s1, s2 = cta_sum(np.abs(r1 - b)), cta_sum(np.abs(r2 - c))
    return a.astype(np.int64), b.astype(np.int64), c.astype(np.int64), u.astype(np.int64), (finite, e, n1s, s1, s2)


def factors(d, raw, factor=1.0, drop_limb_error=False):
    finite, e, n1s, s1, s2 = raw
    g, slack, u = 1.0 + 2.0 ** -30, 1.0 + 2.0 ** -20, 2.0 ** -24
    sigma = math.ldexp(1.0, e)
    r254, r64516 = div_ru(1.0, 254.0), div_ru(1.0, 64516.0)     # 1 / q rounded up; sigma times them is exact
    k1, k2 = sigma * (1.0 / 254.0), sigma * (1.0 / 16387064.0)
    if not finite:
        nan = float("nan")
        return dict(w1=nan, k1=k1, w2=nan, rel2=0.0, k2=k2)
    n1 = mul_ru(n1s, g)
    D1 = mul_ru(mul_ru(s1, g), sigma * r254)
    D2 = mul_ru(mul_ru(s2, g), sigma * r64516)
    if drop_limb_error:
        D1 = D2 = 0.0
    gR = mul_ru(1.001 * u, float(d))
    E1, E2x254 = 0.5 + 128.0 * u, 0.5 + 32766.0 * u
    w1 = mul_ru(add_ru(mul_ru(n1, add_ru(E1, mul_ru(127.001, gR))), mul_ru(127.0, D1)), slack)
    w2 = mul_ru(mul_ru(add_ru(mul_ru(mul_ru(n1, E2x254), add_ru(1.0, gR)), mul_ru(32385.0, D2)), slack), r254)
    rel2 = mul_ru(mul_ru(gR, sigma * (0.5 * r254)), slack)
    return dict(w1=w1 * factor, k1=k1, w2=w2 * factor, rel2=rel2 * factor, k2=k2)


def c_term(metric, nh0, ih0):
    if metric == "cosine":
        return np.zeros(ih0.size)
    if metric == "dot-product":
        return (F32(nh0) * ih0).astype(np.float32).astype(np.float64)
    return np.full(ih0.size, float(F32(nh0)))


def decide_planes(metric, nrm, nh0, hi, lo, s, ih0, d, factor=1.0, drop_limb_error=False):
    """(stage-1 certain, stage-1 side, stage-2 certain, stage-2 side) for every row from its planes and scale."""
    a, b, c, u, raw = limbs(nrm)
    f = factors(d, raw, factor, drop_limb_error)
    h, l = hi.astype(np.int64), lo.astype(np.int64)
    cc = c_term(metric, nh0, ih0)
    sd = s.astype(np.float64)
    with np.errstate(all="ignore"):
        t1 = (254 * (h @ a) + h @ b).astype(np.float64)
        mt1 = (t1 * sd) * f["k1"] + cc
        c1 = np.abs(mt1) > sd * f["w1"]
        t2 = (16387064 * (h @ a) + 64516 * (h @ b + l @ a) + 254 * (h @ c + l @ b) + l @ c).astype(np.float64)
        aa = (254 * (np.abs(h) @ u) + np.abs(l) @ u).astype(np.float64)
        mt2 = (t2 * sd) * f["k2"] + cc
        c2 = np.abs(mt2) > sd * (f["w2"] + f["rel2"] * aa)
    return c1, mt1 > 0, c2, mt2 > 0


def decide(metric, normal, nh0, rows, ih0, **kw):
    n, d = rows.shape
    ld = (d + 31) // 32 * 32
    nrm = np.zeros(ld, dtype=np.float32)
    nrm[:d] = normal
    hi, lo, s = encode(rows, ld)
    return decide_planes(metric, nrm, nh0, hi, lo, s, ih0, d, **kw)


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


def test_the_limb_error_term_is_needed():
    """A normal whose small elements all round to zero limbs (n_i = 0.99 / 508, sigma = 1) and a row that puts every one of
    them at +127 against one element -1 on the big n_0 = 126: n~ puts the row on the far side of its own hyperplane, n on the
    other. Without the 127 D1 term stage 1 calls it wrong; with it, the row is left to the later stages."""
    d = 768
    normal = np.full(d, F32(0.99 / 508), dtype=np.float32)
    normal[0] = 126.0
    rows = np.full((1, d), 127.0, dtype=np.float32)
    rows[0, 0] = -1.0
    ih0 = np.zeros(1, dtype=np.float32)
    ref = reference_sides("cosine", normal, 0.0, rows, ih0)
    assert ref[0]                                     # 127 * 767 * 0.99 / 508 > 126
    c1, r1, _, _ = decide("cosine", normal, 0.0, rows, ih0, drop_limb_error=True)
    assert c1[0] and r1[0] != ref[0]
    c1, r1, c2, r2 = decide("cosine", normal, 0.0, rows, ih0)
    assert not c1[0] and not (c2[0] and r2[0] != ref[0])


def test_no_int32_overflow_at_the_largest_d():
    """d = PLANES_MAX_D, every plane byte and limb at +-127 (U at 254): each lane's int32 dp4a sum and the 8-lane butterfly stay
    exact, and T2 and A stay below 2^53."""
    d = 8192
    x = np.full(d, 127, dtype=np.int64)
    for y in (x, -x):
        lanes = (x * y).reshape(-1, 8, 16).transpose(1, 0, 2).reshape(8, -1)   # lane g holds words 8 c + g
        exact = int((x * y).sum())
        assert abs(exact) < 2 ** 31
        lane32 = lanes.astype(np.int32).sum(axis=1, dtype=np.int32)
        assert int(lane32.sum(dtype=np.int32)) == exact
        assert int(lanes.astype(np.int32).sum(dtype=np.int32)) == exact
    one = 127 * 127 * d
    assert 16387064 * one + 64516 * 2 * one + 254 * 2 * one + one < 2 ** 53     # T2
    assert 254 * 127 * d < 2 ** 31                                                 # each unsigned sum of U |h|, U |l|
    assert 254 * (254 * 127 * d) + 254 * 127 * d < 2 ** 53                         # A


def test_limbs_fit_their_bytes_and_the_errors_are_bounded_above():
    """In exact rationals: the limbs fit int8 (U: u8), |n_i| <= sigma U_i / 2, and the factors' D1, D2 are at least the limb
    errors sum |n_i - n1_i|, sum |n_i - n2_i|."""
    rng = np.random.default_rng(9)
    for scale in (1e-30, 1e-3, 1.0, 1e30):
        nrm = (rng.standard_normal(512) * scale * rng.choice([1e-3, 1.0, 30.0], size=512)).astype(np.float32)
        a, b, c, u, raw = limbs(nrm)
        assert raw[0] and np.abs(a).max() <= 127 and np.abs(b).max() <= 127 and np.abs(c).max() <= 127 and u.max() <= 254
        sigma = Fraction(2) ** raw[1]
        n = [Fraction(float(v)) for v in nrm]
        n1 = [sigma * (int(a[i]) + Fraction(int(b[i]), 254)) for i in range(512)]
        n2 = [n1[i] + sigma * Fraction(int(c[i]), 64516) for i in range(512)]
        assert all(abs(n[i]) <= sigma * int(u[i]) / 2 for i in range(512))
        g = Fraction(1) + Fraction(1, 2 ** 30)
        D1 = mul_ru(mul_ru(raw[3], float(g)), float(sigma) * div_ru(1.0, 254.0))
        D2 = mul_ru(mul_ru(raw[4], float(g)), float(sigma) * div_ru(1.0, 64516.0))
        assert Fraction(D1) >= sum(abs(n[i] - n1[i]) for i in range(512)) > 0
        assert Fraction(D2) >= sum(abs(n[i] - n2[i]) for i in range(512)) > 0
