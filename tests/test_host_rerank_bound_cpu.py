"""The plane pre-filter of host-placed indexes' re-rank (frerank.cuh frerank_kernel<FR_PLANES>, phases 1-3), restated in numpy
float32 and checked on the CPU against the oracle (built_distance / rerank). The restatement follows the kernel: the encoder's
planes and scales (test_prefilter_planes_cpu.encode), the dequantized x~_i = fl(y_i fl(s fl(1/254))), the phase-1 sums in lane
order (eight lanes per row, each running over its 16-element slices of every 128-element chunk and of a trailing partial chunk,
then the xor-shuffle adds 4, 2, 1), |q|_1 in the kernel's order, the per-row bounds E_r, the per-query E (their maximum over the
finite estimates), and the survivor rule with phase 2's histogram threshold. It asserts (a) |estimate - reference| <= E for
every pair with a finite estimate and (b) every member of the oracle's top-k survives, on rows built to put the 8-bit rounding
at its worst: every element of row A sits a few ulps below a half-step of the lo plane and rounds the way that hides part of
q.A, the B rows sit just above and round the other way, and B's element 0 is one lo step less aligned, so A is truly nearest
while every B looks nearer. These come at magnitudes 1, 2^+-60 (~1e+-18) and 2^-80, with mixed exponents, with products or
squares in the subnormal range (rows at 2^-80 against a query at 2^-72; rows at 2^-74 for Euclidean), next to zero rows,
rows with a NaN scale (2^-126, subnormal, or just below the encoder's 127 FLT_MIN threshold), rows just above that threshold,
near-duplicates of the query, and the Cosine rows whose header lost an underflowed tail (helpers.adversarial_set)."""
import numpy as np
import pytest

import oracle
from helpers import adversarial_set
from test_prefilter_planes_cpu import encode

F32 = np.float32
U = 2.0 ** -24
EPS32 = F32(1.1920928955078125e-07)
METRICS = ["euclidean", "cosine", "dot-product", "manhattan"]
DIMS = [64, 100, 768, 1000, 4096, 8192]
FR_SURV = 2048
TINY = float(np.finfo(np.float32).tiny)


def fma32(a, b, c):
    return (np.asarray(a, np.float64) * np.asarray(b, np.float64) + np.asarray(c, np.float64)).astype(np.float32)


def ld_of(d):
    return (d + 31) // 32 * 32


def consts(metric, d, quant=1.0, absolute=True):
    """fr_plane_consts: (e2, wq, wa, rel_a); quant scales the quantization part E2' and absolute=False drops the absolute
    terms wq and wa (for the tests that weaken the bound)."""
    e2p = (1.0 / 508.0 + 512.0 * U) * quant
    e2 = e2p + 127.5 * (d / 6.0 + 48.0) * U if metric in ("dot-product", "cosine") else e2p
    rel = (d / 6.0 + 64.0 if metric == "euclidean" else 1.25 * d + 16.0) * U * 1.01 * (1.0 + 2.0 ** -20)
    wq, wa = (2.0 ** -132, (d + 32.0) * 2.0 ** -148) if absolute else (0.0, 0.0)
    return F32(e2 * (1.0 + 2.0 ** -10) * (1.0 + 2.0 ** -20)), F32(wq), F32(wa), F32(rel)


def dequantized(hi, lo, s):
    y = 254 * hi.astype(np.int32) + lo.astype(np.int32)
    with np.errstate(all="ignore"):
        ks = (s * F32(1.0 / 254.0)).astype(np.float32)
        return (y.astype(np.float32) * ks[:, None]).astype(np.float32)


def lane_sums(metric, q, xt):
    """phase 1's sums (a0, a1) of every row, in the kernel's lane order"""
    n, ld = xt.shape
    qp = np.zeros(ld, np.float32)
    qp[:q.size] = q
    a0 = np.zeros((n, 8), np.float32)
    a1 = np.zeros((n, 8), np.float32)
    nch, tail = ld // 128, (ld % 128) // 16
    spans = [(c * 128, 8) for c in range(nch)] + ([(nch * 128, tail)] if tail else [])
    with np.errstate(all="ignore"):
        for base, lanes in spans:
            for e in range(16):
                idx = base + np.arange(lanes) * 16 + e
                if metric in ("dot-product", "cosine"):
                    a0[:, :lanes] = fma32(qp[idx], xt[:, idx], a0[:, :lanes])
                    continue
                t = (qp[idx] - xt[:, idx]).astype(np.float32)
                if metric == "euclidean":
                    a0[:, :lanes] = fma32(t, t, a0[:, :lanes])
                    a1[:, :lanes] = (a1[:, :lanes] + np.abs(t)).astype(np.float32)
                else:
                    a0[:, :lanes] = (a0[:, :lanes] + np.abs(t)).astype(np.float32)
        lanes = np.arange(8)
        for o in (4, 2, 1):
            a0 = (a0 + a0[:, lanes ^ o]).astype(np.float32)
            a1 = (a1 + a1[:, lanes ^ o]).astype(np.float32)
    return a0[:, 0], a1[:, 0]


def query_l1(q):
    """|q|_1 * 1.001 as the kernel sums it: 256 threads stride, xor-shuffles 16..1, the 8 warps in order"""
    part = np.zeros(256, np.float32)
    for s0 in range(0, q.size, 256):
        seg = q[s0:s0 + 256]
        part[:seg.size] = (part[:seg.size] + np.abs(seg)).astype(np.float32)
    w = part.reshape(8, 32)
    for o in (16, 8, 4, 2, 1):
        w = (w + w[:, np.arange(32) ^ o]).astype(np.float32)
    t = F32(0)
    for i in range(8):
        t = F32(t + w[i, 0])
    return F32(t * F32(1.001))


def hmin(d):  # xrerank.cuh cos_header_min
    return F32(np.sqrt(F32(d) + F32(64))) * F32(8.470329472543003e-22)


def estimates(metric, q, qh, hi, lo, s, ch, quant=1.0, absolute=True):
    """(estimates, per-row bounds E_r) of phase 1 for one query; E_r is 0 where the estimate is not finite"""
    d = q.size
    e2, wq, wa, rel = consts(metric, d, quant, absolute)
    a0, a1 = lane_sums(metric, q, dequantized(hi, lo, s))
    l1q = query_l1(q)
    sfin = s <= F32(3.40282347e38)
    with np.errstate(all="ignore"):
        er = fma32(s, e2, wq)
        if metric == "dot-product":
            a = np.where(sfin, -a0, np.nan).astype(np.float32)
            E = fma32(er, l1q, wa)
        elif metric == "euclidean":
            a = np.where(sfin, a0, np.nan).astype(np.float32)
            Q = (er * fma32(F32(2.002), a1, (F32(d) * er).astype(np.float32))).astype(np.float32)
            E = fma32(rel, a, fma32(Q, F32(1.001), wa))
        elif metric == "manhattan":
            a = np.where(sfin, a0, np.nan).astype(np.float32)
            E = fma32(rel, a, fma32((F32(d) * er).astype(np.float32), F32(1.001), wa))
        else:
            qa = F32(1) / qh if qh >= F32(1e-30) else F32(np.nan)
            pnqn = (qh * ch).astype(np.float32)
            ich = (F32(1) / ch).astype(np.float32)
            cs = np.where((ch >= hmin(d)) & sfin, (a0 * (qa * ich).astype(np.float32)).astype(np.float32), F32(np.nan))
            cs = np.where(cs < -1, F32(-1), np.where(cs > 1, F32(1), cs)).astype(np.float32)
            a = np.where(pnqn > EPS32, (F32(0.5) * (F32(1) - cs)).astype(np.float32), np.where(pnqn == pnqn, F32(0), pnqn)).astype(np.float32)
            E = fma32(fma32(er, l1q, wa), (F32(0.5005) * (qa * ich).astype(np.float32)).astype(np.float32), F32(1.9073486328125e-06))
            E = np.where(pnqn > EPS32, E, F32(0)).astype(np.float32)
        known = np.abs(a) <= F32(3.0e38)
        E = np.where(known, np.where(E == E, E, F32(np.inf)), F32(0)).astype(np.float32)
    return a, E


def xf_key(a):
    b = np.asarray(a, np.float32).view(np.uint32).astype(np.uint64)
    k = np.where(b & 0x80000000, b ^ 0xFFFFFFFF, b ^ 0x80000000)
    return np.where(np.abs(a) <= F32(3.0e38), k, 0xFFFFFFFF).astype(np.uint64)


def xf_unkey(k):
    k = np.uint64(k)
    b = k ^ (np.uint64(0x80000000) if k & np.uint64(0x80000000) else np.uint64(0xFFFFFFFF))
    return np.array([b], np.uint64).astype(np.uint32).view(np.float32)[0]


def threshold_key(keys, k, two_e):
    """phase 2: the histogram's upper edge of the k-th smallest estimate, widened by 2E (key of t + 2E)"""
    nc = keys.size
    if nc <= k or not (F32(0) <= two_e <= F32(3.0e38)):
        return 0xFFFFFFFF
    rlo, rhi, want = int(keys.min()), int(keys.max()), k
    for _ in range(3):
        if not rhi > rlo:
            break
        span = rhi - rlo
        shift = 0 if span < 2048 else span.bit_length() - 11
        sel = keys[(keys >= rlo) & (keys <= rhi)].astype(np.int64)
        hist = np.bincount((sel - rlo) >> shift, minlength=2048)
        cum = np.cumsum(hist)
        b = int(np.argmax(cum >= want)) if cum[-1] >= want else 2047
        before = int(cum[b] - hist[b]) if cum[-1] >= want else int(cum[-1])
        in_bin = int(hist[b])
        top = min(rhi, rlo + ((b + 1) << shift) - 1)
        want -= before
        rlo, rhi = rlo + (b << shift), top
        if in_bin <= 8 or shift == 0:
            break
    if rhi == 0xFFFFFFFF:
        return rhi
    return int(xf_key(F32(xf_unkey(rhi) + two_e)))


def survivors(a, E, k):
    """phase 3 with one E per query: the largest E_r"""
    two_e = F32(F32(F32(2) * F32(E.max() if E.size else 0)) * F32(1.001))
    keys = xf_key(a)
    T = threshold_key(keys, k, two_e)
    return (keys <= T) | (keys == 0xFFFFFFFF)


def survivors_per_row(a, E, k):
    """the alternative rule: keep the rows whose lower bound a - E_r is at most the k-th smallest upper bound a + E_r"""
    known = np.abs(a) <= F32(3.0e38)
    if a.size <= k:
        return np.ones(a.size, bool)
    up = np.sort(np.where(known, a.astype(np.float64) + E, np.inf))[k - 1]
    return ~known | (a.astype(np.float64) - E <= up)


def headers(rows):
    return np.array([oracle.new_header(oracle.COSINE, r)[0] for r in rows], dtype=np.float32)


def run(metric, q, rows, **kw):
    m = oracle.METRICS[metric]
    d = q.size
    hi, lo, s = encode(rows, ld_of(d))
    ch = headers(rows) if metric == "cosine" else np.zeros(rows.shape[0], np.float32)
    qh = F32(oracle.new_header(oracle.COSINE, q)[0]) if metric == "cosine" else F32(0)
    a, E = estimates(metric, q, qh, hi, lo, s, ch, **kw)
    ref = np.array([oracle.built_distance(m, q, (float(qh), 0.0), r, (float(h), 0.0)) for r, h in zip(rows, ch)], dtype=np.float32)
    return a, E, ref, qh, ch


def bound_violations(a, E, ref):
    fin = np.abs(a) <= F32(3.0e38)
    with np.errstate(invalid="ignore"):
        err = np.abs(a.astype(np.float64) - ref.astype(np.float64))
    return np.flatnonzero(fin & ~(err <= float(E.max())))


def dropped(metric, q, rows, qh, ch, a, E, k):
    want, _ = oracle.rerank(oracle.METRICS[metric], q, (float(qh), 0.0), rows, ch, None, np.arange(rows.shape[0], dtype=np.uint32), k)
    keep = survivors(a, E, k)
    return [int(r) for r in want if not keep[r]]


# ---- adversarial rows for the planes ---------------------------------------------------------------------------------------
def plane_set(metric, d, mag=0, mixed=False, delta=2, nb=12, seed=0, qmag=None):
    """(query, rows): row A and nb rows B around the lo plane's half-steps at scale s = 2^mag (one element of every row is
    127 s, which the query's matches or ignores), so A truly nearest while every B's planes make it look nearer (see the module docstring).
    mixed: the elements' integer parts range over 1..126 with random signs instead of 64. The query is scaled by 2^qmag; by
    default 2^-mag for DotProduct and Cosine (products of magnitude ~2^12) and 2^mag for Euclidean and Manhattan (the rows'
    scale)."""
    rng = np.random.default_rng(seed)
    sign = rng.choice([-1.0, 1.0], d) if mixed else np.ones(d)
    hpart = rng.integers(1, 127, d).astype(np.float64) if mixed else np.full(d, 64.0)
    lpart = rng.integers(-100, 100, d).astype(np.float64)
    # the element sits delta f32 ulps below / above the half step between lo values l and l + 1 (s = 1 before scaling)
    def ulps(x, k):
        return (np.asarray(x, np.float32).view(np.uint32).astype(np.int64) + k).astype(np.uint32).view(np.float32).astype(np.float64)
    A = ulps(hpart + (lpart + 0.5) / 254.0, -delta)
    B = ulps(hpart + (lpart + 0.5) / 254.0, delta)
    B[0] = ulps(hpart[0] + (lpart[0] - 0.5) / 254.0, delta)
    if metric in ("euclidean", "manhattan"):
        # the errors x - x~ must point away from the query: A rounds towards it, the B rows away; query beyond the rows
        q = (hpart + 1.0) * sign
    else:
        q = hpart * sign
    A, B = A * sign, B * sign
    A[-1] = B[-1] = 127.0
    q[-1] = 127.0 if metric in ("euclidean", "manhattan") else 0.0   # an element without quantization error that adds nothing
    if metric == "cosine":
        h = max(1, d // 2)
        q[h:-1] = 0.0
    rows = np.stack([A] + [B] * nb) * 2.0 ** mag
    if qmag is None:
        qmag = -mag if metric in ("dot-product", "cosine") else mag
    qs = q * 2.0 ** qmag
    return qs.astype(np.float32), rows.astype(np.float32)


def special_rows(q, d, rng):
    """zero rows, NaN-scale rows (2^-126, subnormal, just below 127 FLT_MIN) and rows just above the threshold"""
    out = [np.zeros(d)]
    for mx in (2.0 ** -126, 2.0 ** -140, 127.0 * TINY * (1 - 2.0 ** -20), 127.0 * TINY, 127.0 * TINY * (1 + 2.0 ** -20), 254.0 * TINY):
        r = rng.uniform(-1, 1, d)
        r = r / np.max(np.abs(r)) * mx
        out.append(r)
    return np.stack(out).astype(np.float32)


KINDS = ["ones", "mixed", "big", "small", "tiny", "subnormal-products", "special", "near-duplicate", "underflow-tail"]


def make_set(kind, metric, d, seed):
    rng = np.random.default_rng(seed)
    if kind == "near-duplicate":
        return adversarial_set("near-duplicate", metric, d, seed=seed)
    if kind == "underflow-tail":
        return adversarial_set("underflow-tail", "cosine", d, seed=seed)
    if kind == "subnormal-products":   # DotProduct / Cosine: rows at 2^-80, query at 2^-72 (products ~2^-140); squares ~2^-148
        q, rows = plane_set(metric, d, mag=-80 if metric in ("dot-product", "cosine") else -74, seed=seed,
                            qmag=-72 if metric in ("dot-product", "cosine") else None)
        return q, rows
    mag = {"ones": 0, "mixed": 0, "big": 60, "small": -60, "tiny": -80, "special": 0}[kind]
    q, rows = plane_set(metric, d, mag=mag, mixed=kind == "mixed", seed=seed)
    if kind == "special":
        rows = np.concatenate([rows, special_rows(q, d, rng)])
    return q, rows


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("d", DIMS)
@pytest.mark.parametrize("metric", METRICS)
def test_estimates_within_the_bound_and_top_k_survives(metric, d, kind):
    if kind == "underflow-tail" and metric != "cosine":
        pytest.skip("a Cosine construction")
    q, rows = make_set(kind, metric, d, seed=d)
    a, E, ref, qh, ch = run(metric, q, rows)
    bad = bound_violations(a, E, ref)
    assert bad.size == 0, [(int(i), float(a[i]), float(ref[i]), float(E.max())) for i in bad[:5]]
    nc = rows.shape[0]
    for k in (1, 10, nc - 1):
        lost = dropped(metric, q, rows, qh, ch, a, E, k)
        assert not lost, (k, lost)


def quant_term(metric, q, rows, a):
    """the quantization part of the bound for row A: s E2' |q|_1 (DotProduct), its Cosine image, 2 s E2' L1 (Euclidean), d s E2'"""
    s = float(np.max(np.abs(rows[0]))) / 127.0
    e = s * (1.0 / 508.0)
    d = q.size
    if metric == "dot-product":
        return e * float(np.sum(np.abs(q.astype(np.float64))))
    if metric == "cosine":
        qn = float(np.sqrt(np.sum(q.astype(np.float64) ** 2)))
        cn = float(np.sqrt(np.sum(rows[0].astype(np.float64) ** 2)))
        return 0.5 * e * float(np.sum(np.abs(q.astype(np.float64)))) / (qn * cn)
    if metric == "euclidean":
        return 2.0 * e * float(np.sum(np.abs(q.astype(np.float64) - rows[0].astype(np.float64))))
    return d * e


@pytest.mark.parametrize("metric", METRICS)
def test_the_construction_reaches_the_quantization_term(metric):
    # row A's estimate moves by at least 0.9 of the quantization part of its bound (Cosine: the query covers half of the row)
    for d in (64, 768, 4096):
        q, rows = plane_set(metric, d, seed=d)
        a, E, ref, qh, ch = run(metric, q, rows)
        got = abs(float(a[0]) - float(ref[0])) / quant_term(metric, q, rows, a)
        assert got >= (0.9 if metric != "cosine" else 0.45), (d, got)
        assert got <= 1.01


@pytest.mark.parametrize("d", [64, 100, 128])
@pytest.mark.parametrize("metric", METRICS)
def test_half_the_quantization_term_is_caught(metric, d):
    # at small d the quantization term is most of E (from d ~ 500 on the fp32 terms of the two sums are as large), so halving
    # it lets the B rows, which look nearer by about twice the quantization term, push the true nearest row A out
    q, rows = plane_set(metric, d, seed=d)
    a, E, ref, qh, ch = run(metric, q, rows, quant=0.5)
    assert dropped(metric, q, rows, qh, ch, a, E, 1) == [0]
    a, E, ref, qh, ch = run(metric, q, rows)
    assert dropped(metric, q, rows, qh, ch, a, E, 1) == []


def test_an_exponent_sweep_makes_no_wrong_drop():
    # rows from 2^0 down to 2^-76, where Euclidean's squares and Manhattan's differences reach the subnormal range, and for
    # DotProduct / Cosine rows at 2^-80 against queries from 2^-40 down to 2^-76, whose products (~2^12 2^(mag + qmag)) go
    # from normal to deep in the subnormal range
    for metric in METRICS:
        sweep = [dict(mag=mag) for mag in range(0, -77, -2)]
        if metric in ("dot-product", "cosine"):
            sweep += [dict(mag=-80, qmag=qmag) for qmag in range(-40, -77, -2)]
        for kw in sweep:
            for d in (64, 100):
                q, rows = plane_set(metric, d, seed=d - kw.get("qmag", kw["mag"]), **kw)
                a, E, ref, qh, ch = run(metric, q, rows)
                assert bound_violations(a, E, ref).size == 0, (metric, d, kw)
                assert dropped(metric, q, rows, qh, ch, a, E, 1) == [], (metric, d, kw)


@pytest.mark.parametrize("metric,d,kw", [("euclidean", 64, dict(mag=-74, seed=0)), ("euclidean", 100, dict(mag=-74, seed=0)),
                                         ("euclidean", 768, dict(mag=-74, seed=0)),
                                         ("dot-product", 64, dict(mag=-80, qmag=-72, seed=2)),
                                         ("dot-product", 100, dict(mag=-80, qmag=-72, seed=2))])
def test_the_bound_without_its_absolute_terms_is_caught(metric, d, kw):
    # squares (Euclidean) or products (DotProduct) in the subnormal range lose up to 2^-150 each in both sums, more than the
    # quantization term of rows this small charges: without wq and wa the estimate leaves its bound and A, the true nearest
    # row, is discarded behind the B rows. (Cosine's 2^-19 term is far above these losses, so it cannot be caught this way.)
    q, rows = plane_set(metric, d, **kw)
    a, E, ref, qh, ch = run(metric, q, rows, absolute=False)
    assert bound_violations(a, E, ref).size > 0
    assert dropped(metric, q, rows, qh, ch, a, E, 1) == [0]
    a, E, ref, qh, ch = run(metric, q, rows)
    assert bound_violations(a, E, ref).size == 0
    assert dropped(metric, q, rows, qh, ch, a, E, 1) == []


def walk_like(metric, d, nc, seed):
    """a query and nc candidates around it, the way a forest walk's candidates are: uniform centred rows, nearer ones first"""
    rng = np.random.default_rng(seed)
    q = rng.uniform(-1, 1, d).astype(np.float32)
    spread = np.linspace(0.05, 1.0, nc)[:, None]
    rows = (q[None, :] * (1 - spread) + rng.uniform(-1, 1, (nc, d)) * spread).astype(np.float32)
    return q, rows


@pytest.mark.parametrize("metric", METRICS)
def test_walk_candidates_leave_about_k_survivors(metric):
    # the reason for the feature: about k of a walk's candidates survive, and the per-query E keeps no more rows than per-row
    # bounds would (so the simpler rule is kept)
    d = 768
    for k, nc in ((10, 500), (100, 2000)):
        q, rows = walk_like(metric, d, nc, seed=k)
        a, E, ref, qh, ch = run(metric, q, rows)
        assert bound_violations(a, E, ref).size == 0
        keep = survivors(a, E, k)
        assert dropped(metric, q, rows, qh, ch, a, E, k) == []
        assert k <= keep.sum() <= k + 8, (k, int(keep.sum()))
        assert keep.sum() <= survivors_per_row(a, E, k).sum() + 3


def test_restatement_of_the_lane_order():
    # the lane sums equal float64 sums of the dequantized rows up to f32 rounding, and every element is visited once
    rng = np.random.default_rng(1)
    for d in (64, 96, 100, 200, 1000):
        q = rng.standard_normal(d).astype(np.float32)
        rows = rng.standard_normal((5, d)).astype(np.float32)
        hi, lo, s = encode(rows, ld_of(d))
        xt = dequantized(hi, lo, s)
        got, _ = lane_sums("dot-product", q, xt)
        want = xt[:, :d].astype(np.float64) @ q.astype(np.float64)
        assert np.all(np.abs(got - want) <= d * 2.0 ** -22 * np.abs(xt[:, :d]).astype(np.float64) @ np.abs(q)), d
        got, _ = lane_sums("manhattan", np.ones(d, np.float32), np.zeros((1, ld_of(d)), np.float32))
        assert float(got[0]) == d
    assert float(query_l1(np.arange(1, 300, dtype=np.float32))) == float(F32(F32(np.sum(np.arange(1, 300))) * F32(1.001)))
