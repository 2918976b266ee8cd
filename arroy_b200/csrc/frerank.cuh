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
//   1. estimates of all candidates (8 lanes per row, 16-byte loads of 8 bf16)
//   2. t = k-th smallest estimate (linear-range histograms), threshold t + 2E
//   3. survivors (estimate <= threshold, or not finite) in candidate order = ascending ids
//   4. exact distances of the survivors (distance_kernel's code), 64-bit keys, bitonic sort,
//      first k -> out_rows / normalized distances (what topk_kernel returns)
// A query with more candidates than FR_CAP or more survivors than FR_SURV sets its status to 1 and
// the host re-runs the batch on the plain kernels.
#pragma once
#include <cuda_bf16.h>

#include "xrerank.cuh"

namespace ab {

constexpr int FR_THREADS = 256;
constexpr int FR_CAP = 8192;      // candidates per query held in shared memory
constexpr int FR_SURV = 2048;     // survivors per query
constexpr int FR_BINS = 2048;

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

__device__ __forceinline__ uint32_t fr_block_scan(uint32_t v, uint32_t* sm /* 9 */, uint32_t* total) {   // exclusive scan over FR_THREADS
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    uint32_t inc = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) { uint32_t t = __shfl_up_sync(0xffffffffu, inc, o); if (lane >= o) inc += t; }
    __syncthreads();
    if (lane == 31) sm[warp] = inc;
    __syncthreads();
    uint32_t base = 0, tot = 0;
#pragma unroll
    for (int i = 0; i < FR_THREADS / 32; ++i) { const uint32_t y = sm[i]; if (i < warp) base += y; tot += y; }
    *total = tot;
    return base + inc - v;
}

struct FrParams {
    const float* items; const __nv_bfloat16* shadow; const float* ih0; const float* cnorm;   // cnorm: |c| per item row (fp32)
    uint32_t d, ld; int metric;
    const float* queries; const uint32_t* qrows; const float* qh0;                            // like distance_kernel
    const uint32_t* rows; const uint64_t* seg_beg; const uint64_t* seg_end;                   // sorted candidate rows per query
    uint32_t k; float rel, sub, hmin; const uint32_t* gmax_bits;   // hmin: cos_header_min(d)
    uint32_t* out_rows; float* out_dist; uint32_t* out_len; int32_t* status;
};

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
    __shared__ uint32_t sm_scan[9];
    __shared__ uint32_t sh_min, sh_max, sh_bin, sh_before;
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

    // |q| (any order: it only enters the bound) and the per-query constants of the estimate
    float part = 0.f;
    for (uint32_t i = tid; i < P.d; i += FR_THREADS) part = fmaf(sq[i], sq[i], part);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) part += __shfl_xor_sync(0xffffffffu, part, o);
    __shared__ float sm_f[FR_THREADS / 32];
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
    const float two_e = 2.0f * e * 1.001f;
    const bool e_ok = two_e >= 0.0f && two_e <= 3.0e38f;

    // ---- 1. estimates from the bf16 shadow ------------------------------------------------------
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
    if (lane == 0) { atomicMin(&sh_min, mn); atomicMax(&sh_max, mx); }
    __syncthreads();

    // ---- 2. k-th smallest estimate (upper bin edge) ---------------------------------------------
    uint32_t T = 0xffffffffu;   // key of the threshold t + 2E
    if (nc > k && e_ok) {
        uint32_t rlo = sh_min, rhi = sh_max, want = k;
        for (int level = 0; level < 3 && rhi > rlo; ++level) {
            for (int i = tid; i < FR_BINS; i += FR_THREADS) hist[i] = 0;
            __syncthreads();
            const uint32_t span = rhi - rlo;
            const int shift = span < FR_BINS ? 0 : (32 - __clz(span)) - 11;
            for (uint32_t p = tid; p < nc; p += FR_THREADS) { const uint32_t key = xf_key(est[p]); if (key >= rlo && key <= rhi) atomicAdd(&hist[(key - rlo) >> shift], 1u); }
            __syncthreads();
            // smallest bin whose cumulative count reaches `want`
            constexpr int PER = FR_BINS / FR_THREADS;
            uint32_t local = 0;
#pragma unroll
            for (int i = 0; i < PER; ++i) local += hist[tid * PER + i];
            uint32_t total;
            const uint32_t ex = fr_block_scan(local, sm_scan, &total);
            if (tid == 0) { sh_bin = FR_BINS - 1; sh_before = total; }
            __syncthreads();
            if (ex < want && ex + local >= want) {
                uint32_t cum = ex;
                for (int i = 0; i < PER; ++i) { const uint32_t h = hist[tid * PER + i]; if (cum + h >= want) { sh_bin = tid * PER + i; sh_before = cum; break; } cum += h; }
            }
            __syncthreads();
            const uint32_t b = sh_bin, in_bin = hist[b];
            const uint32_t top = (uint32_t)min((unsigned long long)rhi, (unsigned long long)rlo + (((unsigned long long)b + 1ull) << shift) - 1ull);
            want -= sh_before; rlo = rlo + (b << shift); rhi = top;
            __syncthreads();
            if (in_bin <= 8u || shift == 0) break;
        }
        T = xf_widen(rhi, two_e);
    }

    // ---- 3. survivors in candidate order ----------------------------------------------------------
    uint32_t* surv = hist;                                                          // FR_SURV <= FR_BINS entries
    uint32_t count = 0;
    for (uint32_t p0 = 0; p0 < nc; p0 += FR_THREADS) {
        const uint32_t p = p0 + tid;
        uint32_t keep = 0;
        if (p < nc) { const uint32_t key = xf_key(est[p]); keep = (key <= T || key == 0xffffffffu) ? 1u : 0u; }
        uint32_t total;
        const uint32_t pos = count + fr_block_scan(keep, sm_scan, &total);
        if (keep && pos < FR_SURV) surv[pos] = p;
        count += total;
    }
    __syncthreads();
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
        float res;
        if (metric == MANHATTAN) {   // not reached (the host keeps Manhattan on the plain kernels); kept for completeness
            res = 0.f;
            if (g8 == 0) { const float* row = P.items + (size_t)r * P.ld; for (uint32_t i = 0; i < P.d; ++i) res = __fadd_rn(res, fabsf(__fsub_rn(sq[i], row[i]))); }
        } else if (P.d >= 32) {
            const float4* A = reinterpret_cast<const float4*>(P.items + (size_t)r * P.ld);
            const float4* Q = reinterpret_cast<const float4*>(sq);
            float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
            const int n32 = (int)(P.d >> 5);
            if (metric == EUCLIDEAN) {
#pragma unroll 4
                for (int c = 0; c < n32; ++c) {
                    const float4 x = Q[c * 8 + g8], y = ldg_stream(A + c * 8 + g8);
                    const float t0 = __fsub_rn(x.x, y.x), t1 = __fsub_rn(x.y, y.y), t2 = __fsub_rn(x.z, y.z), t3 = __fsub_rn(x.w, y.w);
                    acc.x = fmaf(t0, t0, acc.x); acc.y = fmaf(t1, t1, acc.y); acc.z = fmaf(t2, t2, acc.z); acc.w = fmaf(t3, t3, acc.w);
                }
            } else {
#pragma unroll 4
                for (int c = 0; c < n32; ++c) {
                    const float4 x = Q[c * 8 + g8], y = ldg_stream(A + c * 8 + g8);
                    acc.x = fmaf(x.x, y.x, acc.x); acc.y = fmaf(x.y, y.y, acc.y); acc.z = fmaf(x.z, y.z, acc.z); acc.w = fmaf(x.w, y.w, acc.w);
                }
            }
            res = group8_hsum(acc);
            const float* row = P.items + (size_t)r * P.ld;
            for (uint32_t i = (uint32_t)n32 * 32u; i < P.d; ++i) {
                if (metric == EUCLIDEAN) { const float t = __fsub_rn(sq[i], row[i]); res = __fadd_rn(res, __fmul_rn(t, t)); }
                else res = __fadd_rn(res, __fmul_rn(sq[i], row[i]));
            }
        } else {
            res = 0.f;
            if (g8 == 0 && v) { const float* row = P.items + (size_t)r * P.ld; res = (metric == EUCLIDEAN) ? exact_thread<true>(sq, row, (int)P.d) : exact_thread<false>(sq, row, (int)P.d); }
        }
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

inline size_t frerank_smem(uint32_t ld) { return (size_t)ld * 4 + (size_t)FR_CAP * 4 + (size_t)FR_BINS * 4; }
static_assert(FR_CAP * 4 >= FR_SURV * 8 + FR_SURV * 4, "phase-4 buffers must fit in the estimate region");

}  // namespace ab
