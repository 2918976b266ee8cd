"""side()'s 8-bit pre-filter on integer dot products (kernels.cuh planes_job_factors / scan_claim_planes), restated in numpy and
checked on the CPU against the oracle's margins. The normal is read as int8 limbs (a + b / 254 for stage 1, + c / 254^2 for
stage 2, and an unsigned bound U of |n|), the plane sums are exact integers, and the bounds carry the normal's limb error D1 / D2
summed per job. The factors are computed in the device's order and rounding (f64 sums over 8 warps x 32 lanes, then rounded
up), so the restatement makes the device's calls row for row (test_gpu_prefilter_dp4a.py checks that on the device)."""
import math
from fractions import Fraction

import numpy as np
import pytest

import oracle
from test_prefilter_planes_cpu import CASES, TINY, encode, make_case, reference_sides

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


def factors(d, raw, factor=1.0, drop_limb_error=False, drop_abs_term=False):
    finite, e, n1s, s1, s2 = raw
    g, slack, u = 1.0 + 2.0 ** -30, 1.0 + 2.0 ** -20, 2.0 ** -24
    sigma = math.ldexp(1.0, e)
    r254, r64516 = div_ru(1.0, 254.0), div_ru(1.0, 64516.0)     # 1 / q rounded up; sigma times them is exact
    k1, k2 = sigma * (1.0 / 254.0), sigma * (1.0 / 16387064.0)
    if not finite:
        nan = float("nan")
        return dict(w1=nan, k1=k1, w2=nan, rel2=0.0, k2=k2, wa=0.0)
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
    wa = 0.0 if drop_abs_term else math.ldexp(float(d + 32), -150)   # products that underflow: 2^-150 each, exact in f64
    return dict(w1=w1 * factor, k1=k1, w2=w2 * factor, rel2=rel2 * factor, k2=k2, wa=wa * factor)


def c_term(metric, nh0, ih0):
    if metric == "cosine":
        return np.zeros(ih0.size)
    if metric == "dot-product":
        return (F32(nh0) * ih0).astype(np.float32).astype(np.float64)
    return np.full(ih0.size, float(F32(nh0)))


def decide_planes(metric, nrm, nh0, hi, lo, s, ih0, d, factor=1.0, drop_limb_error=False, drop_abs_term=False):
    """(stage-1 certain, stage-1 side, stage-2 certain, stage-2 side) for every row from its planes and scale."""
    a, b, c, u, raw = limbs(nrm)
    f = factors(d, raw, factor, drop_limb_error, drop_abs_term)
    h, l = hi.astype(np.int64), lo.astype(np.int64)
    cc = c_term(metric, nh0, ih0)
    sd = s.astype(np.float64)
    with np.errstate(all="ignore"):
        t1 = (254 * (h @ a) + h @ b).astype(np.float64)
        mt1 = (t1 * sd) * f["k1"] + cc
        c1 = np.abs(mt1) > sd * f["w1"] + f["wa"]
        t2 = (16387064 * (h @ a) + 64516 * (h @ b + l @ a) + 254 * (h @ c + l @ b) + l @ c).astype(np.float64)
        aa = (254 * (np.abs(h) @ u) + np.abs(l) @ u).astype(np.float64)
        mt2 = (t2 * sd) * f["k2"] + cc
        c2 = np.abs(mt2) > sd * (f["w2"] + f["rel2"] * aa) + f["wa"]
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


# ---- rows whose products n_i x_i underflow ---------------------------------------------------------------------------------
# Below about 2^-73 the reference's split normal keeps the magnitude of the rows (|p - q|^2 underflows, so normalize leaves it
# as it is) and every product rounds to +-0: its margins are all +0, every row goes Right. The planes see the exact products in
# f64, so only the absolute term wa keeps them from calling those rows certain.
SEED = bytes([42] * 32)
METRICS = ["euclidean", "cosine", "dot-product", "manhattan"]
SWEEP_ROWS = {64: 3000, 768: 1000, 8192: 150}


def headers(metric, rows):
    """the items' header columns as the reference forms them: (h0, h1, the h0 the pre-filter reads)"""
    n = rows.shape[0]
    if metric == "cosine":
        return np.array([oracle.new_header(oracle.COSINE, r)[0] for r in rows], dtype=np.float32), None, np.zeros(n, np.float32)
    if metric == "dot-product":
        h0, h1 = oracle.dot_preprocess(rows)
        return h0, h1, h0
    z = np.zeros(n, dtype=np.float32)
    return z, None, z


def split_case(metric, rows, normal=None):
    """(oracle sides, pre-filter call) on rows for the normal create_split draws over all of them (or the normal given)"""
    m = oracle.METRICS[metric]
    h0, h1, ih0 = headers(metric, rows)
    idx = np.arange(rows.shape[0], dtype=np.uint32)
    hdr = (0.0, 0.0)
    if normal is None:
        normal, hdr = oracle.create_split(m, oracle.StdRng(SEED), rows, h0, h1, idx)
    side, mg = oracle.side_batch(m, normal, hdr, rows, h0, h1, idx)

    def call(**kw):
        return decide(metric, normal, hdr[0], rows, ih0, **kw)
    return side.astype(bool), mg, call


def wrong_calls(ref, calls):
    c1, r1, c2, r2 = calls
    return int((c1 & (r1 != ref)).sum()), int((c2 & (r2 != ref)).sum())


@pytest.mark.parametrize("d", sorted(SWEEP_ROWS))
@pytest.mark.parametrize("metric", METRICS)
def test_exponent_sweep_makes_no_wrong_call(metric, d):
    base = oracle.synth_rows(SEED, d, 0, SWEEP_ROWS[d], 0.5)
    underflowed = 0
    for e in range(-60, -127, -1):
        rows = (base * F32(2.0 ** e)).astype(np.float32)
        ref, mg, call = split_case(metric, rows)
        assert wrong_calls(ref, call()) == (0, 0), e
        underflowed += bool(e <= -75 and not mg.view(np.uint32).any())
    assert underflowed >= 40          # the sweep does reach the rows whose margins all round to +0


@pytest.mark.parametrize("metric", METRICS)
def test_the_absolute_term_is_needed(metric):
    """Without wa both stages call rows Left whose reference margin is +0 (Right), at every exponent from -75 on."""
    base = oracle.synth_rows(SEED, 768, 0, 1000, 0.5)
    for e in (-75, -80, -100, -118):
        ref, mg, call = split_case(metric, (base * F32(2.0 ** e)).astype(np.float32))
        assert not mg.view(np.uint32).any() and ref.all(), e
        w1, w2 = wrong_calls(ref, call(drop_abs_term=True))
        assert w1 > 0 and w2 > 0, (e, w1, w2)


@pytest.mark.parametrize("metric", METRICS)
def test_the_absolute_term_changes_no_call_at_ordinary_magnitudes(metric):
    base = oracle.synth_rows(SEED, 768, 0, 1000, 0.5)
    for e in (0, -20, -40, -60):
        _, _, call = split_case(metric, (base * F32(2.0 ** e)).astype(np.float32))
        c1, r1, c2, r2 = call()
        d1, s1, d2, s2 = call(drop_abs_term=True)
        assert np.array_equal(c1, d1) and np.array_equal(c2, d2) and np.array_equal(r1, s1) and np.array_equal(r2, s2), e
        assert (c1 | c2).sum() > 0.8 * c1.size


@pytest.mark.parametrize("metric", METRICS)
def test_mixed_row_exponents(metric):
    rng = np.random.default_rng(len(metric))
    base = oracle.synth_rows(SEED, 768, 0, 2000, 0.5)
    for lo, hi in ((-126, -60), (-110, -74), (-20, 0)):
        ex = rng.integers(lo, hi + 1, size=(base.shape[0], 1)).astype(np.float64)
        rows = (base * np.exp2(ex)).astype(np.float32)
        ref, _, call = split_case(metric, rows)
        assert wrong_calls(ref, call()) == (0, 0), (lo, hi)


@pytest.mark.parametrize("metric", METRICS)
def test_rows_at_the_scale_threshold(metric):
    """Rows whose largest element sits a few ulps above and below 127 FLT_MIN: above it the encoder stores a normal scale and
    the rows go through the planes, below it they are left to stage 3. Once with the normal create_split draws over them
    (products underflow) and once with a normal of ordinary magnitude."""
    d, n = 768, 1200
    rng = np.random.default_rng(3)
    base = oracle.synth_rows(SEED, d, 0, n, 0.5).astype(np.float64)
    base /= np.abs(base).max(axis=1, keepdims=True)
    steps = rng.integers(-6, 7, size=n)
    m = np.full(n, F32(127) * TINY, dtype=np.float32)      # exact: the threshold itself
    for i, k in enumerate(steps):                            # k ulps from it
        for _ in range(abs(int(k))):
            m[i] = np.nextafter(m[i], F32(np.inf) if k > 0 else F32(0))
    rows = (base * m[:, None].astype(np.float64)).astype(np.float32)
    rows[np.arange(n), np.abs(base).argmax(axis=1)] = m * np.sign(base[np.arange(n), np.abs(base).argmax(axis=1)]).astype(np.float32)
    _, _, s = encode(rows, d)
    planes = (s >= TINY) & (s <= np.finfo(np.float32).max)
    assert 0 < planes.sum() < n                    # both sides of the threshold occur
    ordinary = (rng.standard_normal(d) / np.sqrt(d)).astype(np.float32)
    for normal in (None, ordinary):
        ref, _, call = split_case(metric, rows, normal)
        c1, r1, c2, r2 = call()
        assert wrong_calls(ref, (c1, r1, c2, r2)) == (0, 0)
        assert not (c1 | c2)[~planes].any()       # the rows below the threshold are never certain
        if normal is not None:
            assert (c1 | c2)[planes].sum() > 0.5 * planes.sum()
