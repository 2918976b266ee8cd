"""The survivor rule of the fused per-query re-rank (frerank.cuh frerank_kernel, phases 1-3), restated in numpy float32 and checked
on the CPU against the oracle (built_distance / rerank). The restatement follows the kernel: the bf16 shadow (round to nearest
even), the phase-1 dot in lane order (eight lanes per row, each FMAs its 8-element slices of every 64-element chunk and of a
trailing 32-element chunk, then the xor-shuffle adds 4, 2, 1), the three estimate formulas, qn, gmax, eps, e and 2e, and the
survivor test against the exact k-th smallest estimate (the kernel's histogram threshold is never below it, so a row kept here is
kept by the kernel). It asserts (a) |estimate - reference| <= E for every pair and (b) every member of the oracle's top-k survives,
on inputs built to put the bf16 rounding at its worst (tests/helpers.py adversarial_set): aligned half-ulp losses, random signs,
mixed exponents, near-duplicates of the query, rows at 1e+-18, rows whose squared norm underflows, subnormal rows, rows just above
2^-126, and Cosine rows whose header lost an underflowed tail. The construction reaches 0.996 of the rounding term of the bound for
DotProduct and Euclidean; Cosine, whose query covers half of the row, reaches 0.71 to 0.97 of it, asserted >= 0.9 / sqrt(2) ~ 0.64
(test_the_construction_reaches_the_rounding_term). The former constant 1.25 * 2^-9 + d 2^-22, the bound without its underflow
term, or the former Cosine header floor of 1e-30 drop true neighbours on these rows (test_*_is_caught)."""
import numpy as np
import pytest

import oracle
from helpers import ADVERSARIAL_KINDS, adversarial_set, bf16_rn

F32 = np.float32
EPS32 = F32(1.1920928955078125e-07)
DIMS = [32, 33, 64, 96, 100, 200, 768, 1536, 4096]
METRICS = ["euclidean", "cosine", "dot-product"]


def fr_rel(d):   # frerank.cuh fr_rel: 1.0625 * 2^-8 + d 2^-22
    return F32(0.004150390625) + F32(d) * F32(2.384185791015625e-07)


def fr_sub(d):   # frerank.cuh fr_sub: sqrt(d + 64) 2^-74, what fp32 norms can lose to underflow (and bf16's subnormal rounding)
    return F32(np.sqrt(F32(d) + F32(64))) * F32(5.293955920339377e-23)


def fr_hmin(d):  # xrerank.cuh cos_header_min: sqrt(d + 64) 2^-70, the smallest Cosine header with a known estimate
    return F32(np.sqrt(F32(d) + F32(64))) * F32(8.470329472543003e-22)


def old_rel(d):  # the constant before: 1.25 * 2^-9 + d 2^-22
    return F32(0.00244140625) + F32(d) * F32(2.384185791015625e-07)


def fma32(a, b, c):
    return (np.asarray(a, np.float64) * np.asarray(b, np.float64) + np.asarray(c, np.float64)).astype(np.float32)


def shadow_dot(q, rows):
    """Phase 1's f32 dot of the query with the bf16 rows, in the kernel's lane order."""
    n, d = rows.shape
    ld = (d + 31) // 32 * 32
    S = np.zeros((n, ld), np.float32)
    S[:, :d] = bf16_rn(rows)
    qp = np.zeros(ld, np.float32)
    qp[:d] = q
    acc = np.zeros((n, 8), np.float32)
    for c in range(ld // 64):
        for j in range(8):
            idx = c * 64 + np.arange(8) * 8 + j
            acc = fma32(S[:, idx], qp[idx], acc)
    if ld & 32:                                          # trailing 32-element chunk: lanes 0..3
        c = ld // 64
        for j in range(8):
            idx = c * 64 + np.arange(4) * 8 + j
            acc[:, :4] = fma32(S[:, idx], qp[idx], acc[:, :4])
    lanes = np.arange(8)
    for o in (4, 2, 1):
        acc = acc + acc[:, lanes ^ o]
    return acc[:, 0]


def query_qq(q):
    """|q|^2 as the kernel sums it: 256 threads stride over the elements, then xor-shuffles 16..1, then the 8 warps in order."""
    part = np.zeros(256, np.float32)
    for s0 in range(0, q.size, 256):
        seg = q[s0:s0 + 256]
        part[:seg.size] = fma32(seg, seg, part[:seg.size])
    w = part.reshape(8, 32)
    for o in (16, 8, 4, 2, 1):
        w = w + w[:, np.arange(32) ^ o]
    qq = F32(0)
    for i in range(8):
        qq = F32(qq + w[i, 0])
    return qq


def headers(rows):
    return np.array([oracle.new_header(oracle.COSINE, r)[0] for r in rows], dtype=np.float32)


def estimates(metric, q, qh, rows, cnorm, ch, gmax, rel, sub, hmin):
    """(estimates, E, 2E) of frerank_kernel for one query; gmax = the largest |c| (Cosine: |c| / header) of the staged items."""
    d = q.size
    qq = query_qq(q)
    qn = F32(np.sqrt(qq)) * F32(1.000001)
    with np.errstate(all="ignore"):
        eps = fma32(rel, F32(F32(qn + sub) * F32(gmax + sub)), F32(1e-30))
        acc = shadow_dot(q, rows)
        if metric == "dot-product":
            e = eps
            a = -acc
        elif metric == "euclidean":
            e = fma32(F32(F32(d // 32) + F32(16)) * F32(2.384185791015625e-07), F32(qq + F32(gmax * gmax)), F32(2) * eps)
            a = (qq + cnorm * cnorm) - F32(2) * acc
        else:
            if qh >= F32(1e-30):
                qa = F32(1) / qh
                e = fma32(F32(0.5) * eps, qa, F32(1.9073486328125e-06))
            else:
                qa = F32(np.nan)
                e = F32(1.9073486328125e-06)
            pnqn = qh * ch
            inv = np.where(ch >= hmin, F32(1) / ch, F32(np.nan)).astype(np.float32)
            cs = np.clip(acc * (qa * inv), F32(-1), F32(1)).astype(np.float32)
            a = np.where(pnqn > EPS32, F32(0.5) * (F32(1) - cs), np.where(pnqn == pnqn, F32(0), pnqn)).astype(np.float32)
        two_e = F32(F32(2) * e) * F32(1.001)
    return a.astype(np.float32), F32(e), two_e


def survivors(a, k, two_e):
    nc = a.size
    known = np.abs(a) <= F32(3.0e38)
    if nc <= k or not (F32(0) <= two_e <= F32(3.0e38)):
        return np.ones(nc, bool)
    t = np.sort(np.where(known, a, np.inf).astype(np.float32))[k - 1]
    if not np.isfinite(t):
        return np.ones(nc, bool)
    return (a <= F32(t + two_e)) | ~known


def run(metric, q, rows, rel=fr_rel, sub=fr_sub, hmin=fr_hmin):
    m = oracle.METRICS[metric]
    d = q.size
    cnorm = headers(rows)                               # norms_kernel: sqrt of the reference-order dot (the Cosine header)
    ch = cnorm if metric == "cosine" else np.zeros_like(cnorm)
    qh = F32(oracle.new_header(oracle.COSINE, q)[0]) if metric == "cosine" else F32(0)
    with np.errstate(all="ignore"):
        g = cnorm * np.where(ch >= F32(1e-30), F32(1) / ch, F32(0)) if metric == "cosine" else cnorm
    gmax = F32(np.max(np.where(g == g, np.abs(g), np.inf)))   # fr_gmax_kernel: NaN counts as infinite
    a, e, two_e = estimates(metric, q, qh, rows, cnorm, ch, gmax, rel(d), sub(d), hmin(d))
    ref = np.array([oracle.built_distance(m, q, (float(qh), 0.0), r, (float(h), 0.0)) for r, h in zip(rows, ch)], dtype=np.float32)
    return a, e, two_e, ref, qh, ch, gmax


def bound_violations(a, e, ref):
    """pairs whose finite estimate is farther than E from the reference (or whose reference is not finite)"""
    fin = np.abs(a) <= F32(3.0e38)
    with np.errstate(invalid="ignore"):
        err = np.abs(a.astype(np.float64) - ref.astype(np.float64))
    return np.flatnonzero(fin & ~(err <= float(e)))


def dropped(metric, q, rows, qh, ch, a, two_e, k):
    m = oracle.METRICS[metric]
    want, _ = oracle.rerank(m, q, (float(qh), 0.0), rows, ch, None, np.arange(rows.shape[0], dtype=np.uint32), k)
    keep = survivors(a, k, two_e)
    return [int(r) for r in want if not keep[r]]


@pytest.mark.parametrize("kind", ADVERSARIAL_KINDS)
@pytest.mark.parametrize("d", DIMS)
@pytest.mark.parametrize("metric", METRICS)
def test_estimates_within_the_bound_and_top_k_survives(metric, d, kind):
    q, rows = adversarial_set(kind, metric, d, seed=d)
    a, e, two_e, ref, qh, ch, _ = run(metric, q, rows)
    bad = bound_violations(a, e, ref)
    assert bad.size == 0, [(int(i), float(a[i]), float(ref[i]), float(e)) for i in bad[:5]]
    nc = rows.shape[0]
    for k in (1, 10, nc - 1):
        lost = dropped(metric, q, rows, qh, ch, a, two_e, k)
        assert not lost, (k, lost)


@pytest.mark.parametrize("metric", ["euclidean", "dot-product", "cosine"])
def test_the_construction_reaches_the_rounding_term(metric):
    # the bf16 part of the bound is 2^-8 |q| gmax (Euclidean: twice that, Cosine: half of it over |q| |c|); the aligned rows
    # must come within 0.9 of it (Cosine: of 2^-1/2 of it, since only half of the row is aligned with the query), at every d
    for d in DIMS:
        worst = 0.0
        for kind in ("ones", "signs", "mixed"):
            q, rows = adversarial_set(kind, metric, d, seed=d)
            a, e, two_e, ref, qh, ch, gmax = run(metric, q, rows)
            qn = np.sqrt(np.sum(q.astype(np.float64) ** 2))
            scale = 0.5 / float(qh) if metric == "cosine" else (2.0 if metric == "euclidean" else 1.0)
            term = scale * 2.0 ** -8 * qn * float(gmax)
            worst = max(worst, float(np.max(np.abs(a.astype(np.float64) - ref))) / term)
        assert worst >= (0.9 if metric != "cosine" else 0.9 * 2 ** -0.5), (d, worst)
        assert worst <= 1.0625


@pytest.mark.parametrize("metric,d", [("dot-product", 33), ("dot-product", 768), ("dot-product", 4096), ("euclidean", 33), ("euclidean", 200),
                                      ("euclidean", 4096), ("cosine", 64), ("cosine", 200), ("cosine", 768)])
def test_the_former_constant_is_caught(metric, d):
    # rel = 1.25 * 2^-9 + d 2^-22 charges half of bf16's unit roundoff: on the aligned rows the estimate moves by up to 1.6 E,
    # and A, the true nearest row, is discarded behind k rows B that look closer
    q, rows = adversarial_set("ones", metric, d, seed=d)
    a, e, two_e, ref, qh, ch, _ = run(metric, q, rows, rel=old_rel)
    assert bound_violations(a, e, ref).size > 0
    for k in (1, 10):
        assert dropped(metric, q, rows, qh, ch, a, two_e, k) == [0], k
    a, e, two_e, ref, qh, ch, _ = run(metric, q, rows)
    assert dropped(metric, q, rows, qh, ch, a, two_e, 10) == []


@pytest.mark.parametrize("kind", ["underflow", "subnormal", "tiny-normal"])
@pytest.mark.parametrize("d", [33, 768])
def test_the_bound_without_its_underflow_term_is_caught(d, kind):
    # rows this small have an f32 squared norm of 0, so gmax = 0 and rel qn gmax says nothing; a large query turns their bf16
    # error (relative, or absolute below 2^-126) into far more than the 1e-30 floor. The sub term keeps E above it.
    q, rows = adversarial_set(kind, "dot-product", d, seed=d)
    a, e, two_e, ref, qh, ch, gmax = run("dot-product", q, rows, sub=lambda d: F32(0))
    assert gmax == 0.0
    assert bound_violations(a, e, ref).size > 0
    assert dropped("dot-product", q, rows, qh, ch, a, two_e, 1) == [0]
    a, e, two_e, ref, qh, ch, _ = run("dot-product", q, rows)
    assert bound_violations(a, e, ref).size == 0
    assert dropped("dot-product", q, rows, qh, ch, a, two_e, 1) == []


@pytest.mark.parametrize("d", [768, 1536, 4096])
def test_the_cosine_header_floor_is_caught(d):
    # Cosine divides by the headers, and a header loses what underflows of the row's squared norm: on rows whose tail squares
    # underflow, |c| / header is 2 to 4, far beyond what gmax = cnorm / header = 1 charges. With the former floor (a header of
    # 1e-30 gets a known estimate) A is discarded; with cos_header_min those rows are unknown and survive.
    q, rows = adversarial_set("underflow-tail", "cosine", d, seed=d)
    a, e, two_e, ref, qh, ch, _ = run("cosine", q, rows, hmin=lambda d: F32(1e-30))
    assert bound_violations(a, e, ref).size > 0
    assert dropped("cosine", q, rows, qh, ch, a, two_e, 1) == [0]
    a, e, two_e, ref, qh, ch, _ = run("cosine", q, rows)
    assert bound_violations(a, e, ref).size == 0
    assert dropped("cosine", q, rows, qh, ch, a, two_e, 1) == []


def test_restatement_of_the_lane_order():
    # the lane-order dot equals a float64 dot of the bf16 rows up to f32 rounding, and a 32-element tail reaches lanes 0..3 only
    rng = np.random.default_rng(1)
    for d in (20, 32, 33, 96, 100, 200):
        q = rng.standard_normal(d).astype(np.float32)
        rows = rng.standard_normal((5, d)).astype(np.float32)
        want = bf16_rn(rows).astype(np.float64) @ q.astype(np.float64)
        got = shadow_dot(q, rows)
        assert np.all(np.abs(got - want) <= d * 2.0 ** -22 * np.abs(bf16_rn(rows)).astype(np.float64) @ np.abs(q)), d
    assert float(query_qq(np.arange(1, 300, dtype=np.float32))) == float(np.sum(np.arange(1, 300, dtype=np.float64) ** 2))
