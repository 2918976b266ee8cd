// frerank.cuh — fused per-query re-rank with a half-width pre-filter (reader.rs:381-399).
//
// The re-rank of a query reads every candidate row once (search_k ~ count x n_trees rows of 4d bytes:
// 15 MB per query for BASELINE config 2) although only `count` of them end up in the result: the
// scan is HBM-bound. This kernel first scores the candidates against a bf16 SHADOW copy of the item
// matrix (half the bytes) with a guaranteed error bound, keeps the few that can still reach the
// top-k, and re-scores only those from the fp32 rows in the reference's exact summation order — so
// ids and distances stay bit-identical while the bytes per query drop ~1.9x.
//
//   shadow[c][i] = bf16_rn(item[c][i])  ->  | s - dot_ref(q, item_c) | <= rel (qn + sub) (gmax + sub),   s = phase 1's fp32 dot,
//   rel = 1.0625 2^-8 + d 2^-22,   sub = sqrt(d + 64) 2^-74,   qn >= |q| and gmax >= |c| as computed in fp32.
// The terms, with u = 2^-24 (fp32) and the bf16 rounding e_i = shadow_i - c_i:
//   * bf16 keeps 8 significant bits: round to nearest even gives |e_i| <= 2^-8 |c_i| for |c_i| >= 2^-126 (an element just below
//     the midpoint 1 + 2^-8 loses almost 2^-8 of itself), and |e_i| <= 2^-134 below it (the subnormal step is 2^-133), so
//     |sum q_i e_i| <= 2^-8 |q| |c| + sqrt(d) 2^-134 |q|. The errors of all elements line up when the row's rounding
//     directions follow the query's signs: tests/test_frerank_bound_cpu.py builds such rows and reaches 0.996 of 2^-8 |q| |c|.
//   * fp32 accumulation of s: a product passes through at most d/8 + 11 roundings (its lane's FMA chain over the non-zero
//     elements, then the xor 4, 2, 1 adds). The reference's dot_ref: at most d/32 + 37 (an AVX chain, hsum256, the three adds,
//     a tail of up to 31 elements; SSE and scalar paths are shorter). Both sums run over |q_i| |c_i| (1 + 2^-8), so together
//     they stay below (0.16 d + 48) u |q| |c| <= d 2^-22 |q| |c| for d >= 13, and below 4 d u by counting the non-zero terms
//     for smaller d.
//   * underflow: |q| (the kernel's qq) and |c| (norms_kernel) are fp32 sums of squares. A square below 2^-150 rounds to zero and
//     each of the at most d + 40 roundings loses at most 2^-150 in the subnormal range, so |c| <= gmax + sqrt(d + 40) 2^-75 and
//     |q| <= qn + sqrt(d + 40) 2^-75; `sub` is twice that. It also covers the subnormal term above, sqrt(d) 2^-134 |q| <=
//     2^-8 sub |q|. Without it an index of rows whose squared norm underflows has gmax = 0 and an E far below its error.
//     Cosine divides by the headers instead: gmax is cnorm / header, the ratio of two equal fp32 sums, so sub does not bound
//     a row's |c| / header, which underflow makes unbounded (a row of one element 2^-72 and a tail of 2^-76 has header 2^-72
//     and |c| = 2.2 2^-72 at d = 1024). A row whose header is at least cos_header_min(d) = sqrt(d + 64) 2^-70 (xrerank.cuh)
//     loses at most 2^-10 of its squared norm, so |c| <= header (1 + 2^-11) (1 + small), inside the 1.0625 factor; a row
//     below it gets an unknown estimate and always survives. The query's side is covered by qn + sub over its header.
//   * the 1.0625 factor covers the roundings of the bound itself: qn = sqrt(qq) * 1.000001 and gmax (|c| by norms_kernel,
//     Cosine |c| / header) are within (d/32 + 10) u of the true norms, and eps, e and 2e take a few more roundings and the
//     1.001 factor; all of them are multiplicative, far below 2^-4.
//   The estimate a(q, c) of built_distance and E(q) follow xrerank.cuh (same formulas as the tensor-core pre-filter:
//   TgEpilogue / xf_query_prep_kernel), with eps = rel (qn + sub) (gmax + sub) + 1e-30: DotProduct E = eps; Euclidean
//   E = 2 eps + (d/32 + 16) 2^-22 (|q|^2 + gmax^2) for the roundings of |q|^2, |c|^2 and the reference's own sum of squares;
//   Cosine E = eps / (2 |q|) + 2^-19 for the roundings of the division and of the clamp formula (a row whose header is below
//   cos_header_min(d) has an unknown estimate and always survives). For ordinary data sub vanishes next to the norms and eps
//   is rel qn gmax.
//
// One CTA per query, everything in shared memory:
//   1. estimates of all candidates (fr_estimates_bf16: 8 lanes per row, 16-byte loads of 8 bf16)
//   2. t = k-th smallest estimate (linear-range histograms), threshold t + 2E
//   3. survivors (estimate <= threshold, or not finite) in candidate order = ascending ids
//   4. exact distances of the survivors (distance_kernel's row_sum8; Manhattan in the reference's sequential order), 64-bit
//      keys, bitonic sort, first k -> out_rows / normalized distances (what topk_kernel returns)
// A query with more candidates than FR_CAP or more survivors than FR_SURV sets its status to 1 and
// the host re-runs the batch on the plain kernels.
//
// Host-placed items (frerank_kernel<FR_PLANES>): the f32 rows are in mapped host memory and there is no bf16 shadow, but the
// build's two 8-bit planes and row scales are on the device (kernels.cuh planes_encode_kernel). Phase 1 (fr_estimates_planes)
// then estimates every candidate from its planes (2 bytes per element; nothing reads an f32 row, a norm or a gmax, each of which would be a pass over
// PCIe), phases 2-3 are the same, and phase 4 re-scores only the survivors from the host rows — about k rows per query instead
// of all of its candidates. The estimate and its bound, with u = 2^-24:
//   * dequantization: y_i = 254 h_i + l_i is an exact integer (|y_i| <= 32385), turned into a float exactly (the 1.5 2^23 bias
//     trick), and x~_i = fl(y_i ks), ks = fl(s fl(1/254)). Three relative roundings give |x~_i - s y_i / 254| <= 383 u s, and a
//     subnormal ks or product adds at most 32386 2^-150 < 2^-135. With the encoder's |x_i - s y_i / 254| <= s E2 (E2 = 1/508 +
//     129 u): |x_i - x~_i| <= er = s E2' + wq, E2' = 1/508 + 512 u, wq = 2^-132 (four times 2^-135: it also covers the fp32
//     roundings of er itself when er is subnormal). Every row's bound below is built from er.
//   * DotProduct: a = -fl(sum q_i x~_i) (8 lanes per row, each an FMA chain over its 16-element slices of every 128-element
//     chunk, then xor 4, 2, 1). |sum q_i x_i - sum q_i x~_i| <= er |q|_1. The estimate's chain has at most ld/8 + 3 <= d/8 + 7
//     roundings and the reference's dot_ref at most d/32 + 37 (frerank_kernel's note above), both over sum |q_i| |x_i| with
//     |x_i| <= 127.001 s and |x~_i| <= 127.5 s (1 + 3 u) + 2^-135: together at most 127.5 (d/6 + 48) u s |q|_1. Products that
//     underflow lose up to 2^-150 each in both sums, carried through at most 1 + gamma: wa = (d + 32) 2^-148 (twice what the
//     two sums need). E_r = er' |q|_1 + wa with er' = s (E2' + 127.5 (d/6 + 48) u) (1 + 2^-10) + wq, |q|_1 summed in fp32 and
//     multiplied by 1.001 (d u <= 2^-11 for d <= 8192); the two slack factors cover every fp32 rounding of the bound.
//   * Cosine: the dot above through frerank_kernel's clamp formula and header division; E_r = 0.5005 E_dot / (qh ch) + 2^-19
//     (the 2^-19 covers the roundings of the division and of the clamp formula, as for the bf16 estimate). A row whose header is
//     below cos_header_min(d) keeps an unknown estimate and always survives, so that no such row widens E; a row with
//     qh ch <= 2^-23 has the reference's exact 0.
//   * Euclidean: a = fl(sum t_i^2), t_i = fl(q_i - x~_i), and L1 = fl(sum |t_i|) in the same pass (never |c|^2: on the device it
//     would take a pass over the host rows). With d_i = q_i - x_i, t^_i = q_i - x~_i and delta_i = x_i - x~_i:
//     |sum t^_i^2 - sum d_i^2| = |sum delta_i (2 t^_i - delta_i)| <= er (2 sum |t^_i| + d er) = Q. Every term of both sums is
//     non-negative, so their fp32 roundings (the chain, the subtraction's (1 + u)^2; the reference's d/32 + 37 adds and its own
//     subtraction) are relative to the estimate: E_r = (d/6 + 64) u 1.01 a + 1.001 Q + wa, Q evaluated with L1 * 1.001 (which
//     covers L1's own roundings), wa for the squares that underflow.
//   * Manhattan: a = fl(sum |t_i|); ||t^| - |d|| <= |delta| gives Q = d er; the reference's sequential sum has d + 1 roundings:
//     E_r = (1.25 d + 16) u 1.01 a + 1.001 Q + wa. (Manhattan has no bf16 path: this is its only pre-filter.)
//   * special scales: s = 0 (an all-zero row) has x~ = 0 = x and the formulas above (Q = 0); a NaN or +inf scale (non-finite,
//     tiny or below the encoder's 127 FLT_MIN threshold) gets a NaN estimate and always survives.
//   The survivor rule is frerank_kernel's with one E per query: E = the largest E_r over the query's candidates whose estimate is
//   finite. A true top-k row r has a_r <= D_r + E_r <= D_(k) + E, and D_(k) <= t + E (the k rows with the smallest estimates
//   have D <= t + E), so a_r <= t + 2E. Per-row bounds (keep rows whose lower bound is below the k-th smallest upper bound) would
//   only differ where E_r varies across a query's candidates, which it barely does for a walk's candidates (similar scales and
//   distances); tests/test_host_rerank_bound_cpu.py counts the survivors of both rules.
#pragma once
#include <cuda_bf16.h>

#include "xrerank.cuh"

namespace ab {

constexpr int FR_THREADS = 256;
constexpr int FR_CAP = 8192;      // candidates per query held in shared memory
constexpr int FR_SURV = 2048;     // survivors per query
constexpr int FR_BINS = 2048;
enum FrSource { FR_NONE = -1, FR_BF16 = 0, FR_PLANES = 1 };   // where phase 1's estimates come from (FR_NONE: the fused kernel does not run)

inline float fr_rel(uint32_t d) { return 0.004150390625f + (float)d * 2.384185791015625e-07f; }   // 1.0625 * 2^-8 + d 2^-22
inline float fr_sub(uint32_t d) { return sqrtf((float)d + 64.0f) * 5.293955920339377e-23f; }  // sqrt(d + 64) 2^-74

// shadow copy: n x ld bf16, round to nearest even (padding stays zero)
__global__ void fr_shadow_kernel(const float4* __restrict__ items, uint2* __restrict__ shadow, uint64_t total4) {
    for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total4; i += (uint64_t)gridDim.x * blockDim.x) {
        const float4 v = items[i];
        __nv_bfloat162 a = __floats2bfloat162_rn(v.x, v.y), b = __floats2bfloat162_rn(v.z, v.w);
        uint2 o;
        o.x = *reinterpret_cast<uint32_t*>(&a); o.y = *reinterpret_cast<uint32_t*>(&b);
        shadow[i] = o;
    }
}

struct FrParams {
    const float* items; const __nv_bfloat16* shadow; const float* ih0; const float* cnorm;   // cnorm: |c| per item row (fp32)
    uint32_t d, ld; int metric;
    const float* queries; const uint32_t* qrows; const float* qh0;                            // like distance_kernel
    const uint32_t* rows; const uint64_t* seg_beg; const uint64_t* seg_end;                   // sorted candidate rows per query
    uint32_t k; float rel, sub, hmin; const uint32_t* gmax_bits;   // hmin: cos_header_min(d)
    uint32_t* out_rows; float* out_dist; uint32_t* out_len; int32_t* status;
    // FR_PLANES: the build's planes and row scales, the bound's constants (fr_plane_consts) and the counters (candidates
    // estimated, survivors re-scored)
    const int8_t* hi; const int8_t* lo; const float* scale;
    float e2, wq, wa, rel_a;
    unsigned long long* counts;
};

// Phase 1 of FR_PLANES for one row: lane g8 of the row's 8-lane group runs over its 16-element slices of every 128-element
// chunk (16-byte loads of each plane) and of a trailing partial chunk (ld % 128 = 32, 64 or 96: lanes 0..1, 0..3 or 0..5).
// MODE 0: a0 = sum q_i x~_i; MODE 1: a0 = sum t_i^2, a1 = sum |t_i|; MODE 2: a0 = sum |t_i|, with t_i = q_i - x~_i.
template <int MODE>
__device__ __forceinline__ void fr_plane_row(const int8_t* __restrict__ hi, const int8_t* __restrict__ lo, uint32_t ld, uint32_t r, float ks,
                                             const float* sq, int g8, float& a0, float& a1) {
    const uint4* H = reinterpret_cast<const uint4*>(hi + (size_t)r * ld);
    const uint4* L = reinterpret_cast<const uint4*>(lo + (size_t)r * ld);
    auto step = [&](const uint4 h, const uint4 l, const float* qp) {
        const uint32_t hw[4] = {h.x, h.y, h.z, h.w}, lw[4] = {l.x, l.y, l.z, l.w};
#pragma unroll
        for (int w = 0; w < 4; ++w) {
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                const int y = 254 * ((int)(hw[w] << (24 - 8 * j)) >> 24) + ((int)(lw[w] << (24 - 8 * j)) >> 24);
                const float xt = __fmul_rn(__fsub_rn(__int_as_float(0x4b400000 + y), 12582912.0f), ks);   // (float)y exactly, times ks
                const float qi = qp[4 * w + j];
                if (MODE == 0) a0 = fmaf(qi, xt, a0);
                else {
                    const float t = __fsub_rn(qi, xt);
                    if (MODE == 1) { a0 = fmaf(t, t, a0); a1 = __fadd_rn(a1, fabsf(t)); }
                    else a0 = __fadd_rn(a0, fabsf(t));
                }
            }
        }
    };
    const int nch = (int)(ld >> 7), tail = (int)((ld & 127u) >> 4);
#pragma unroll 2
    for (int c = 0; c < nch; ++c) step(__ldg(H + c * 8 + g8), __ldg(L + c * 8 + g8), sq + c * 128 + g8 * 16);
    if (g8 < tail) step(__ldg(H + nch * 8 + g8), __ldg(L + nch * 8 + g8), sq + nch * 128 + g8 * 16);
}

// Phase 1 from the bf16 shadow: est[p] for every candidate p, the CTA's smallest and largest key in sh_min / sh_max; returns 2E.
__device__ __forceinline__ float fr_estimates_bf16(const FrParams& P, const float* __restrict__ sq, float* __restrict__ est, const uint32_t* __restrict__ rows,
                                                   uint32_t nc, float qh, uint32_t* sh_min, uint32_t* sh_max) {
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, g8 = lane & 7, grp = lane >> 3;
    const int metric = P.metric;
    // |q| (any order: it only enters the bound) and the per-query constants of the estimate
    __shared__ float sm_f[FR_THREADS / 32];
    float part = 0.f;
    for (uint32_t i = tid; i < P.d; i += FR_THREADS) part = fmaf(sq[i], sq[i], part);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) part += __shfl_xor_sync(0xffffffffu, part, o);
    if (lane == 0) sm_f[warp] = part;
    __syncthreads();
    float qq = 0.f;
#pragma unroll
    for (int i = 0; i < FR_THREADS / 32; ++i) qq += sm_f[i];
    const float qn = sqrtf(qq) * 1.000001f;
    const float gmax = __uint_as_float(*P.gmax_bits);
    const float eps = fmaf(P.rel, (qn + P.sub) * (gmax + P.sub), 1e-30f);
    float qa = 0.f, e;
    if (metric == DOT_PRODUCT) e = eps;
    else if (metric == EUCLIDEAN) { qa = qq; e = fmaf(((float)(P.d / 32u) + 16.0f) * 2.384185791015625e-07f, qq + gmax * gmax, 2.0f * eps); }
    else { if (qh >= 1e-30f) { qa = 1.0f / qh; e = fmaf(0.5f * eps, qa, 1.9073486328125e-06f); } else { qa = __uint_as_float(0x7fc00000u); e = 1.9073486328125e-06f; } }

    // estimates: 8 lanes per row, 16-byte loads of 8 bf16
    const int nch = (int)(P.ld >> 6);                      // chunks of 64 elements (8 lanes x 8 bf16); ld % 32 == 0
    const bool half_chunk = (P.ld & 32u) != 0;             // a trailing chunk of 32 elements (lanes 0..3 of the group)
    uint32_t mn = 0xffffffffu, mx = 0u;
    for (uint32_t p0 = (uint32_t)warp * 4u; p0 < nc; p0 += (FR_THREADS / 32) * 4u) {
        const uint32_t p = p0 + (uint32_t)grp;
        const bool v = p < nc;
        const uint32_t r = v ? rows[p] : 0u;
        const uint4* S = reinterpret_cast<const uint4*>(P.shadow + (size_t)r * P.ld);
        float acc = 0.f;
        auto fma8 = [&](const uint4 w, const float* qp) {
            const __nv_bfloat162* h = reinterpret_cast<const __nv_bfloat162*>(&w);
#pragma unroll
            for (int j = 0; j < 4; ++j) { const float2 f = __bfloat1622float2(h[j]); acc = fmaf(f.x, qp[2 * j], acc); acc = fmaf(f.y, qp[2 * j + 1], acc); }
        };
#pragma unroll 4
        for (int c = 0; c < nch; ++c) fma8(__ldg(S + c * 8 + g8), sq + c * 64 + g8 * 8);
        if (half_chunk && g8 < 4) fma8(__ldg(S + nch * 8 + g8), sq + nch * 64 + g8 * 8);
        acc += __shfl_xor_sync(0xffffffffu, acc, 4); acc += __shfl_xor_sync(0xffffffffu, acc, 2); acc += __shfl_xor_sync(0xffffffffu, acc, 1);
        if (v && g8 == 0) {
            float a;
            if (metric == DOT_PRODUCT) a = -acc;
            else if (metric == EUCLIDEAN) { const float cn = P.cnorm[r]; a = (qa + cn * cn) - 2.0f * acc; }
            else {
                const float ch = P.ih0[r];
                const float pnqn = __fmul_rn(qh, ch);
                if (pnqn > 1.1920928955078125e-07f) {
                    float cs = ch >= P.hmin ? acc * (qa * (1.0f / ch)) : __uint_as_float(0x7fc00000u);
                    cs = cs < -1.0f ? -1.0f : (cs > 1.0f ? 1.0f : cs);
                    a = 0.5f * (1.0f - cs);
                } else a = pnqn == pnqn ? 0.0f : pnqn;
            }
            est[p] = a;
            const uint32_t key = xf_key(a);
            mn = min(mn, key); mx = max(mx, key);
        }
    }
    mn = __reduce_min_sync(0xffffffffu, mn); mx = __reduce_max_sync(0xffffffffu, mx);
    if (lane == 0) { atomicMin(sh_min, mn); atomicMax(sh_max, mx); }
    __syncthreads();
    return 2.0f * e * 1.001f;
}

// Phase 1 from the 8-bit planes: est[p] for every candidate p and the largest per-row bound E, the CTA's smallest and largest
// key in sh_min / sh_max; returns 2E.
__device__ __forceinline__ float fr_estimates_planes(const FrParams& P, const float* __restrict__ sq, float* __restrict__ est, const uint32_t* __restrict__ rows,
                                                     uint32_t nc, float qh, uint32_t* sh_min, uint32_t* sh_max) {
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, g8 = lane & 7, grp = lane >> 3;
    const int metric = P.metric;
    // |q|_1 (any order: it only enters the bound) and 1 / qh
    __shared__ float sm_f[FR_THREADS / 32];
    __shared__ uint32_t sh_e;
    float part = 0.f;
    for (uint32_t i = tid; i < P.d; i += FR_THREADS) part = __fadd_rn(part, fabsf(sq[i]));
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) part += __shfl_xor_sync(0xffffffffu, part, o);
    if (lane == 0) sm_f[warp] = part;
    if (tid == 0) sh_e = 0u;
    __syncthreads();
    float l1q = 0.f;
#pragma unroll
    for (int i = 0; i < FR_THREADS / 32; ++i) l1q += sm_f[i];
    l1q *= 1.001f;
    const float qa = metric == COSINE ? (qh >= 1e-30f ? 1.0f / qh : __uint_as_float(0x7fc00000u)) : 0.f;

    uint32_t mn = 0xffffffffu, mx = 0u, eb = 0u;
    for (uint32_t p0 = (uint32_t)warp * 4u; p0 < nc; p0 += (FR_THREADS / 32) * 4u) {
        const uint32_t p = p0 + (uint32_t)grp;
        const bool v = p < nc;
        const uint32_t r = v ? rows[p] : 0u;
        const float s = v ? P.scale[r] : 0.f;
        const float ks = __fmul_rn(s, 1.0f / 254.0f);
        float a0 = 0.f, a1 = 0.f;
        if (metric == EUCLIDEAN) fr_plane_row<1>(P.hi, P.lo, P.ld, r, ks, sq, g8, a0, a1);
        else if (metric == MANHATTAN) fr_plane_row<2>(P.hi, P.lo, P.ld, r, ks, sq, g8, a0, a1);
        else fr_plane_row<0>(P.hi, P.lo, P.ld, r, ks, sq, g8, a0, a1);
        a0 += __shfl_xor_sync(0xffffffffu, a0, 4); a0 += __shfl_xor_sync(0xffffffffu, a0, 2); a0 += __shfl_xor_sync(0xffffffffu, a0, 1);
        a1 += __shfl_xor_sync(0xffffffffu, a1, 4); a1 += __shfl_xor_sync(0xffffffffu, a1, 2); a1 += __shfl_xor_sync(0xffffffffu, a1, 1);
        if (v && g8 == 0) {
            const bool sfin = s <= 3.40282347e+38f;                 // false for the NaN and +inf scales
            const float er = fmaf(s, P.e2, P.wq);                    // DotProduct / Cosine: er' of the note above
            const float nan = __uint_as_float(0x7fc00000u);
            float a, E = 0.f;
            if (metric == DOT_PRODUCT) { a = sfin ? -a0 : nan; E = fmaf(er, l1q, P.wa); }
            else if (metric == EUCLIDEAN) { a = sfin ? a0 : nan; E = fmaf(P.rel_a, a, fmaf(er * fmaf(2.002f, a1, (float)P.d * er), 1.001f, P.wa)); }
            else if (metric == MANHATTAN) { a = sfin ? a0 : nan; E = fmaf(P.rel_a, a, fmaf((float)P.d * er, 1.001f, P.wa)); }
            else {
                const float ch = P.ih0[r];
                const float pnqn = __fmul_rn(qh, ch);
                if (pnqn > 1.1920928955078125e-07f) {
                    const float ich = 1.0f / ch;
                    float cs = (ch >= P.hmin && sfin) ? a0 * (qa * ich) : nan;
                    cs = cs < -1.0f ? -1.0f : (cs > 1.0f ? 1.0f : cs);
                    a = 0.5f * (1.0f - cs);
                    E = fmaf(fmaf(er, l1q, P.wa), 0.5005f * (qa * ich), 1.9073486328125e-06f);
                } else a = pnqn == pnqn ? 0.0f : pnqn;
            }
            est[p] = a;
            const uint32_t key = xf_key(a);
            mn = min(mn, key); mx = max(mx, key);
            if (key != 0xffffffffu) eb = max(eb, E == E ? __float_as_uint(E) : 0x7f800000u);   // E >= 0: uint order is float order
        }
    }
    mn = __reduce_min_sync(0xffffffffu, mn); mx = __reduce_max_sync(0xffffffffu, mx); eb = __reduce_max_sync(0xffffffffu, eb);
    if (lane == 0) { atomicMin(sh_min, mn); atomicMax(sh_max, mx); atomicMax(&sh_e, eb); }
    __syncthreads();
    return 2.0f * __uint_as_float(sh_e) * 1.001f;
}

template <int SRC>
__global__ void __launch_bounds__(FR_THREADS)
frerank_kernel(FrParams P) {
    extern __shared__ __align__(16) unsigned char fr_smem[];
    // shared memory: [query ld floats][region A: FR_CAP estimates; in phase 4 re-used for FR_SURV keys + FR_SURV distances]
    //                [FR_BINS histogram words; from phase 3 on the survivor positions] — 43 KB at d = 768, five CTAs per SM
    float* sq = reinterpret_cast<float*>(fr_smem);
    float* est = sq + P.ld;
    unsigned long long* keys = reinterpret_cast<unsigned long long*>(est);          // phase 4 (the estimates are dead by then)
    float* sdist = est + 2 * FR_SURV;                                               // phase 4: exact distance per survivor
    uint32_t* hist = reinterpret_cast<uint32_t*>(est + FR_CAP);
    __shared__ uint32_t sm_scan[FR_THREADS / 32];
    __shared__ uint32_t sh_min, sh_max, sh_bin[2];
    const uint32_t q = blockIdx.x;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, g8 = lane & 7, grp = lane >> 3;
    const uint64_t beg = P.seg_beg[q], end = P.seg_end[q];
    const uint32_t nc = (uint32_t)(end - beg);
    const uint32_t* rows = P.rows + beg;
    const uint32_t k = P.k, kk = nc < k ? nc : k;
    const float* qv = P.qrows ? P.items + (size_t)P.qrows[q] * P.ld : P.queries + (size_t)q * P.ld;
    const float qh = P.qh0 ? P.qh0[q] : 0.f;
    const int metric = P.metric;
    if (tid == 0) { sh_min = 0xffffffffu; sh_max = 0u; P.status[q] = 0; }
    if (nc > FR_CAP) { if (tid == 0) { P.status[q] = 1; P.out_len[q] = 0; } return; }
    for (uint32_t i = tid; i < P.ld; i += FR_THREADS) sq[i] = qv[i];
    __syncthreads();

    // ---- 1. estimates of all candidates ---------------------------------------------------------
    float two_e;
    if constexpr (SRC == FR_BF16) two_e = fr_estimates_bf16(P, sq, est, rows, nc, qh, &sh_min, &sh_max);
    else two_e = fr_estimates_planes(P, sq, est, rows, nc, qh, &sh_min, &sh_max);

    // ---- 2. k-th smallest estimate (upper bin edge) ---------------------------------------------
    uint32_t T = 0xffffffffu;   // key of the threshold t + 2E
    if (nc > k && two_e >= 0.0f && two_e <= 3.0e38f) {
        const uint32_t t = hist_narrow<FR_THREADS, FR_BINS>(sh_min, sh_max, k, 8u, [&](auto add) {
            for (uint32_t p = tid; p < nc; p += FR_THREADS) add(xf_key(est[p]));
        }, hist, sm_scan, sh_bin);
        T = xf_widen(t, two_e);
    }

    // ---- 3. survivors in candidate order ----------------------------------------------------------
    uint32_t* surv = hist;                                                          // FR_SURV <= FR_BINS entries
    uint32_t count = 0;
    for (uint32_t p0 = 0; p0 < nc; p0 += FR_THREADS) {
        const uint32_t p = p0 + tid;
        uint32_t keep = 0;
        if (p < nc) { const uint32_t key = xf_key(est[p]); keep = (key <= T || key == 0xffffffffu) ? 1u : 0u; }
        uint32_t total;
        const uint32_t pos = count + block_exclusive_scan<FR_THREADS>(keep, sm_scan, &total);
        if (keep && pos < FR_SURV) surv[pos] = p;
        count += total;
    }
    __syncthreads();
    if constexpr (SRC == FR_PLANES) {
        if (tid == 0) { atomicAdd(&P.counts[0], (unsigned long long)nc); if (count <= FR_SURV) atomicAdd(&P.counts[1], (unsigned long long)count); }
    }
    if (count > FR_SURV) { if (tid == 0) { P.status[q] = 1; P.out_len[q] = 0; } return; }

    // ---- 4. exact distances of the survivors, then sort by (distance, position) -------------------
    int np2 = 2;
    while ((uint32_t)np2 < count) np2 <<= 1;
    for (int i = (int)count + tid; i < np2; i += FR_THREADS) keys[i] = ~0ull;
    for (uint32_t s0 = (uint32_t)warp * 4u; s0 < count; s0 += (FR_THREADS / 32) * 4u) {
        const uint32_t s = s0 + (uint32_t)grp;
        const bool v = s < count;
        const uint32_t p = v ? surv[s] : 0u;
        const uint32_t r = v ? rows[p] : 0u;
        const float* row = P.items + (size_t)r * P.ld;
        float res;
        if (metric == MANHATTAN) {
            // the reference's strictly sequential sum in element order. The group's 8 lanes load the row in 16-byte pieces, all in
            // flight at once (host-placed rows are read over PCIe), and lane 0 adds the terms in order from their registers.
            const float4* A = reinterpret_cast<const float4*>(row);
            const float4* Q = reinterpret_cast<const float4*>(sq);
            const int src = lane & ~7, n32 = (int)(P.d >> 5);
            res = 0.f;
#pragma unroll 4
            for (int c = 0; c < n32; ++c) {
                const float4 x = Q[c * 8 + g8], y = ldg_stream(A + c * 8 + g8);
                const float t[4] = {fabsf(__fsub_rn(x.x, y.x)), fabsf(__fsub_rn(x.y, y.y)), fabsf(__fsub_rn(x.z, y.z)), fabsf(__fsub_rn(x.w, y.w))};
#pragma unroll
                for (int j = 0; j < 8; ++j)
#pragma unroll
                    for (int e = 0; e < 4; ++e) res = __fadd_rn(res, __shfl_sync(0xffffffffu, t[e], src + j));
            }
            if (g8 == 0) for (uint32_t i = (uint32_t)n32 * 32u; i < P.d; ++i) res = __fadd_rn(res, fabsf(__fsub_rn(sq[i], row[i])));
        } else res = row_sum8<false>(metric == EUCLIDEAN, sq, row, P.d, g8, v);
        if (v && g8 == 0) {
            const float dist = built_finish(metric, res, qh, (metric == COSINE) ? P.ih0[r] : 0.f);
            sdist[s] = dist;
            keys[s] = ((unsigned long long)ordered_key(dist) << 32) | (unsigned long long)s;   // s grows with the position: same tie-break
        }
    }
    __syncthreads();
    bitonic_sort_shared(keys, np2);
    if (tid == 0) P.out_len[q] = kk;
    for (uint32_t i = tid; i < kk; i += FR_THREADS) {
        const uint32_t s = (uint32_t)(keys[i] & 0xffffffffull);
        P.out_rows[(size_t)q * k + i] = rows[surv[s]];
        P.out_dist[(size_t)q * k + i] = normalized_distance_dev(metric, sdist[s]);
    }
}

// gmax = max over all items of |c| (Euclidean, DotProduct) or |c| / header norm (Cosine; 1 when the headers are the norms)
__global__ void fr_gmax_kernel(const float* __restrict__ cnorm, const float* __restrict__ ih0, uint64_t n, int metric, uint32_t* __restrict__ gmax_bits) {
    uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    float g = 0.f;
    if (i < n) {
        g = cnorm[i];
        if (metric == COSINE) { const float h = ih0[i]; g = h >= 1e-30f ? __fmul_rn(g, __fdiv_rn(1.0f, h)) : 0.f; }
        if (!(g == g)) g = __uint_as_float(0x7f800000u);
    }
    g = fabsf(g);
    const uint32_t bits = __reduce_max_sync(0xffffffffu, __float_as_uint(g));
    if ((threadIdx.x & 31) == 0 && bits) atomicMax(gmax_bits, bits);
}

// FR_PLANES's per-query constants of the bound (the note above), for d <= PLANES_MAX_D; u = 2^-24, all rounded up:
//   e2 = (E2' + 127.5 (d/6 + 48) u) (1 + 2^-10) for DotProduct / Cosine, E2' (1 + 2^-10) for Euclidean and Manhattan;
//   wq = 2^-132; wa = (d + 32) 2^-148; rel_a = (d/6 + 64) u 1.01 (Euclidean) or (1.25 d + 16) u 1.01 (Manhattan).
inline void fr_plane_consts(int metric, uint32_t d, FrParams& P) {
    const double u = 0x1p-24, E2p = 1.0 / 508.0 + 512.0 * u;
    const double e2 = (metric == DOT_PRODUCT || metric == COSINE) ? E2p + 127.5 * (d / 6.0 + 48.0) * u : E2p;
    P.e2 = (float)(e2 * (1.0 + 0x1p-10) * (1.0 + 0x1p-20));
    P.wq = 0x1p-132f;
    P.wa = (float)(((double)d + 32.0) * 0x1p-148);
    P.rel_a = (float)((metric == EUCLIDEAN ? d / 6.0 + 64.0 : 1.25 * d + 16.0) * u * 1.01 * (1.0 + 0x1p-20));
}

inline size_t frerank_smem(uint32_t ld) { return (size_t)ld * 4 + (size_t)FR_CAP * 4 + (size_t)FR_BINS * 4; }
static_assert(FR_CAP * 4 >= FR_SURV * 8 + FR_SURV * 4, "phase-4 buffers must fit in the estimate region");

}  // namespace ab
