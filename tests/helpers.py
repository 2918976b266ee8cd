"""Shared helpers for the parity tests (golden comparison, node decoding)."""
import json
import os

import numpy as np

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "reference_golden.json")


def golden():
    with open(GOLDEN) as f:
        return json.load(f)


def fmt4(x):
    """Rust `{:0.4}` of an f32 (exact value, correctly rounded) == C printf of the widened double."""
    return "%.4f" % float(np.float32(x))


def bf16_rn(x):
    """f32 -> nearest bf16 (ties to even), returned as f32 (what fr_shadow_kernel stores)."""
    b = np.ascontiguousarray(x, dtype=np.float32).view(np.uint32).astype(np.uint64)
    r = ((b + 0x7FFF + ((b >> 16) & 1)) >> 16) << 16
    return (r & 0xFFFFFFFF).astype(np.uint32).view(np.float32)


ADVERSARIAL_KINDS = ("ones", "signs", "mixed", "near-duplicate", "big", "small", "underflow", "subnormal", "tiny-normal",
                     "underflow-tail")


def _from_bits(bits):
    return np.asarray(bits, dtype=np.uint64).astype(np.uint32).view(np.float32)


def adversarial_set(kind, metric, d, nb=12, shift=16, delta=8, seed=0):
    """(query, rows) that put the rounding of a low-precision copy of the rows (bf16: shift 16; TF32: shift 13) at its worst.

    Every element of row A lies `delta` f32 ulps below the midpoint between two low-precision values, so it rounds towards zero
    and loses almost half a low-precision ulp; the query's sign pattern matches, so all of those losses push q.A in the same
    direction. Rows B_1 .. B_nb lie `delta` ulps above the midpoints and round away from zero, except element 0, which sits just
    above the low-precision value one step down: that makes every B truly farther from the query than A, while its rounded copy
    looks closer. The query's magnitudes follow the rows' (Cauchy-Schwarz equality), so the error is ~ 2^-(p+1) |q| |c|.
    For Cosine the query covers only the first half of the elements (an aligned query would clamp the cosine at 1).
    Kinds: "ones" (all magnitudes 1, query all +1), "signs" (random signs), "mixed" (magnitudes 2^-20 .. 2^20),
    "near-duplicate" (A and B straddle a random query, plus rows equal to the query up to a few ulps), "big" / "small" (rows at
    2^60 / 2^-60 ~ 1e+-18 with a query of magnitude 1), "underflow" (rows at 2^-80, whose f32 squared norm is 0), "subnormal"
    (the smallest subnormal low-precision step) and "tiny-normal" (rows at 2^-126); the last three with a query of magnitude 2^50.
    "underflow-tail" (_underflow_tail) targets Cosine, whose headers lose the part of the squared norm that underflows."""
    rng = np.random.default_rng(seed)
    if kind == "underflow-tail":
        return _underflow_tail(d, nb, shift, rng)
    m = 23 - shift                                         # low-precision mantissa bits
    pow2 = lambda e: np.asarray((127 + np.asarray(e, dtype=np.int64)) << m, dtype=np.uint64)
    s = np.ones(d) if kind == "ones" else rng.choice([-1.0, 1.0], d)
    b = np.full(d, pow2(0), dtype=np.uint64)
    qscale, q = 1.0, None
    if kind == "mixed":
        e = rng.integers(-20, 21, d)
        e[0] = 20
        b = pow2(e)
    elif kind == "near-duplicate":
        q = (rng.standard_normal(d) * rng.choice([1e-3, 1.0, 30.0], d)).astype(np.float32)
        s = np.where(q < 0, -1.0, 1.0)
        b = np.maximum(np.abs(q).view(np.uint32).astype(np.uint64) >> shift, np.uint64(1))
    elif kind in ("big", "small"):
        e = 60 if kind == "big" else -60
        b[:] = pow2(e)
        qscale = 2.0 ** -e
    elif kind == "underflow":
        b[:] = pow2(-80)
        qscale = 2.0 ** (50 + 80)
    elif kind == "subnormal":
        b[:] = 1
        qscale = 2.0 ** (50 + 126 + m)
    elif kind == "tiny-normal":
        b[:] = pow2(-126)
        qscale = 2.0 ** (50 + 126)
    exact = _from_bits(b << shift).astype(np.float64)
    half = 1 << (shift - 1)
    A = _from_bits((b << shift) + half - delta).astype(np.float64)
    B = _from_bits((b << shift) + half + delta).astype(np.float64)
    B[0] = _from_bits(((b[0] - 1) << shift) + 2 * delta)
    if q is None:
        q = (s * exact * qscale).astype(np.float32)
    if metric == "cosine" and kind != "near-duplicate":
        h = max(1, d // 2)
        outside = exact[h:] if kind not in ("underflow", "subnormal", "tiny-normal") else np.full(d - h, 2.0 ** -60)   # keep |c| normal
        q[h:] = 0.0
        A[h:] = outside
        B[h:] = outside
    rows = [s * A] + [s * B] * nb
    if kind == "near-duplicate":
        rows += [q, np.nextafter(q, np.float32(np.inf)), q * (1.0 + 2.0 ** -20)]
    return q, np.stack(rows).astype(np.float32)


def _underflow_tail(d, nb, shift, rng):
    """Rows of element 0 = 2^-72 and a tail of magnitude ~2^-76, whose squares underflow: every row's f32 header is 2^-72, while
    |c| is 2.2 2^-72 at d = 1024. Query: 0 at element 0, +-2^50 elsewhere, with signs independent of the rows', so the cosine
    stays far from the clamp. Each tail element sits 2 ulps from a low-precision midpoint, on the side that makes q_i e_i < 0 for
    every element of A and > 0 for every element of the B rows; B's element 1 is one low-precision step less aligned, which
    makes A truly nearest (the reference divides both by the same header)."""
    m = 23 - shift
    b = (127 - 76) << m
    half, delta = 1 << (shift - 1), 2
    below = float(_from_bits((b << shift) + half - delta))
    above = float(_from_bits((b << shift) + half + delta))
    s = rng.choice([-1.0, 1.0], d)
    r = rng.choice([-1.0, 1.0], d)
    aligned = r == s
    A = r * np.where(aligned, below, above)
    B = r * np.where(aligned, above, below)
    B[1] = r[1] * float(_from_bits(((b - 1 if aligned[1] else b + 1) << shift) + 2 * delta))
    A[0] = B[0] = 2.0 ** -72
    q = (s * 2.0 ** 50).astype(np.float32)
    q[0] = 0.0
    return q, np.stack([A] + [B] * nb).astype(np.float32)


def check_dump(gold, nodes, roots, metric, dims, decode_node):
    """Compare a forest ({node id: NodeCodec bytes}) with a parsed reference snapshot.

    Everything the reference's DatabaseHandle dump prints is compared: roots, node ids, node
    kinds, child ids, header values and the first 10 normal components at 4 decimals, and the
    full descendant lists.
    """
    assert list(roots) == gold["roots"]
    assert sorted(nodes.keys()) == sorted(int(k) for k in gold["tree"].keys())
    for key, g in gold["tree"].items():
        n = decode_node(nodes[int(key)], metric, dims)
        assert n["kind"] == g["kind"], (key, n, g)
        if g["kind"] == "descendants":
            assert n["descendants"] == g["descendants"], key
            continue
        assert (n["left"], n["right"]) == (g["left"], g["right"]), key
        if g["normal"] is None:
            assert n["normal"] is None, key
            continue
        hdr_vals = [fmt4(v) for v in n["header"]]
        assert hdr_vals == list(g["header"].values()), (key, hdr_vals, g["header"])
        got = [fmt4(v) for v in n["normal"][:10]]
        assert got == g["normal"], (key, got, g["normal"])
        if not g["truncated"]:
            assert len(n["normal"]) == len(g["normal"])
