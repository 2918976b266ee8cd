// xrerank.cuh — batched re-rank of MANY queries against ONE shared candidate list (BASELINE.json
// config 5: 4096 queries x 100k candidates, d = 768), bit-exact.
//
// D::built_distance (src/reader.rs:381-391) for every (query, candidate) pair is a dense
// Q x C x d contraction. Tensor cores cannot be used for it: the result contract is "top-k ids
// identical to the reference", and the reference's value for each pair is defined by its AVX+FMA
// summation order (src/spaces/simple_avx.rs:6-110) — 32 accumulator lanes (k mod 32), each a
// sequential FMA chain over the 32-chunks, then the hsum256 tree. So this is a register-tiled
// CUDA-core kernel that keeps exactly that order per pair:
//   * lane l of a warp IS accumulator lane l; a thread holds an 8 x 8 tile of pairs (64 chains),
//     so one chunk costs 16 shared-memory loads for 64 FMAs;
//   * operands (16 query rows x 32 candidate rows per CTA, 64 floats of k per stage) are staged with
//     cp.async, double buffered;
//   * the final reduction is a transposing butterfly (xor 4, 2, 1: each step halves the number of
//     pairs a lane keeps, 56 shuffles instead of 192), then ((h1+h2)+h3)+h4 across the four
//     accumulator groups — the same additions, in the same order, as hsum256 + the final sum.
// Manhattan (strictly sequential scalar sum) and d < 32 (SSE / scalar paths) use the generic kernels.
#pragma once
#include "kernels.cuh"

namespace ab {

constexpr int XQ = 8, XC = 8;        // register tile per warp (queries x candidates)
constexpr int XWQ = 2, XWC = 4;      // warps per CTA along q and c
constexpr int XQB = XQ * XWQ;        // 16 queries per CTA
constexpr int XCB = XC * XWC;        // 32 candidates per CTA
constexpr int XSLAB = 64;            // floats of k per pipeline stage (2 chunks)
constexpr int XTHREADS = 32 * XWQ * XWC;

__device__ __forceinline__ void cp_async16(void* smem, const void* gmem) {
    unsigned s = (unsigned)__cvta_generic_to_shared(smem);
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(s), "l"(gmem));
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;"); }
template <int N> __device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N)); }

// dist[q * nc + c] = built_distance(query q, item rows[c]); grid = (ceil(nc / XCB), ceil(nq / XQB))
template <bool EUCLID>
__global__ void __launch_bounds__(XTHREADS)
xrerank_kernel(const float* __restrict__ items, const float* __restrict__ ih0, uint32_t d, uint32_t ld, int metric,
               const float* __restrict__ queries /* nq x ld */, const float* __restrict__ qh0, uint32_t nq,
               const uint32_t* __restrict__ rows, uint32_t nc, float* __restrict__ dist) {
    __shared__ __align__(16) float sQ[2][XQB][XSLAB];
    __shared__ __align__(16) float sC[2][XCB][XSLAB];
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int wq = warp / XWC, wc = warp % XWC;
    const uint32_t qb = blockIdx.y * XQB, cb = blockIdx.x * XCB;
    const uint32_t m = d & ~31u;                       // AVX main part
    const int nstage = (int)((m + XSLAB - 1) / XSLAB);

    // this thread's cp.async sources: 1 float4 of Q, 2 float4 of C per stage
    const int qr = tid / (XSLAB / 4), qc4 = tid % (XSLAB / 4);          // 256 threads -> 16 rows x 16 float4
    const uint32_t qrow = min(qb + (uint32_t)qr, nq - 1);
    const float* qsrc = queries + (size_t)qrow * ld;
    const float* csrc[2];
    int cr[2], cc4[2];
    for (int h = 0; h < 2; ++h) {
        int idx = tid + h * XTHREADS;
        cr[h] = idx / (XSLAB / 4); cc4[h] = idx % (XSLAB / 4);
        uint32_t crow = min(cb + (uint32_t)cr[h], nc - 1);
        csrc[h] = items + (size_t)rows[crow] * ld;
    }
    auto issue = [&](int st, int buf) {
        const uint32_t k0 = (uint32_t)st * XSLAB;
        if (k0 + qc4 * 4 < m) cp_async16(&sQ[buf][qr][qc4 * 4], qsrc + k0 + qc4 * 4);
        for (int h = 0; h < 2; ++h)
            if (k0 + cc4[h] * 4 < m) cp_async16(&sC[buf][cr[h]][cc4[h] * 4], csrc[h] + k0 + cc4[h] * 4);
        cp_async_commit();
    };

    float acc[XQ][XC];
#pragma unroll
    for (int i = 0; i < XQ; ++i)
#pragma unroll
        for (int j = 0; j < XC; ++j) acc[i][j] = 0.f;

    if (nstage > 0) issue(0, 0);
    for (int st = 0; st < nstage; ++st) {
        const int buf = st & 1;
        if (st + 1 < nstage) { issue(st + 1, buf ^ 1); cp_async_wait<1>(); } else cp_async_wait<0>();
        __syncthreads();
        const uint32_t k0 = (uint32_t)st * XSLAB;
#pragma unroll
        for (int kk = 0; kk < XSLAB / 32; ++kk) {
            if (k0 + kk * 32 < m) {
                float qv[XQ], cv[XC];
#pragma unroll
                for (int i = 0; i < XQ; ++i) qv[i] = sQ[buf][wq * XQ + i][kk * 32 + lane];
#pragma unroll
                for (int j = 0; j < XC; ++j) cv[j] = sC[buf][wc * XC + j][kk * 32 + lane];
#pragma unroll
                for (int i = 0; i < XQ; ++i)
#pragma unroll
                    for (int j = 0; j < XC; ++j) {
                        if (EUCLID) { float t = __fsub_rn(qv[i], cv[j]); acc[i][j] = fmaf(t, t, acc[i][j]); }
                        else acc[i][j] = fmaf(qv[i], cv[j], acc[i][j]);
                    }
            }
        }
        __syncthreads();
    }

    // ---- hsum256 for 64 pairs at once: transposing butterfly --------------------------------------
    const unsigned full = 0xffffffffu;
    const bool b2 = (lane & 4) != 0, b1 = (lane & 2) != 0, b0 = (lane & 1) != 0;
    float v1[XQ][4];
#pragma unroll
    for (int i = 0; i < XQ; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) {   // x128[u] = x[u+4] + x[u]; this lane keeps pairs (i, j + 4*b2)
            float send = b2 ? acc[i][j] : acc[i][j + 4];
            float mine = b2 ? acc[i][j + 4] : acc[i][j];
            v1[i][j] = __fadd_rn(mine, __shfl_xor_sync(full, send, 4));
        }
    float v2[XQ][2];
#pragma unroll
    for (int i = 0; i < XQ; ++i)
#pragma unroll
        for (int j = 0; j < 2; ++j) {   // x64[0] = x128[0]+x128[2], x64[1] = x128[1]+x128[3]
            float send = b1 ? v1[i][j] : v1[i][j + 2];
            float mine = b1 ? v1[i][j + 2] : v1[i][j];
            v2[i][j] = __fadd_rn(mine, __shfl_xor_sync(full, send, 2));
        }
    float h[XQ];
#pragma unroll
    for (int i = 0; i < XQ; ++i) {      // x64[0] + x64[1]
        float send = b0 ? v2[i][0] : v2[i][1];
        float mine = b0 ? v2[i][1] : v2[i][0];
        h[i] = __fadd_rn(mine, __shfl_xor_sync(full, send, 1));
    }
    // lane (g, t) now holds accumulator g's horizontal sum for the pairs (i = 0..7, j = t)
    const int t = lane & 7;
    float res[XQ];
#pragma unroll
    for (int i = 0; i < XQ; ++i) {
        float s1 = __shfl_sync(full, h[i], t + 8), s2 = __shfl_sync(full, h[i], t + 16), s3 = __shfl_sync(full, h[i], t + 24);
        res[i] = __fadd_rn(__fadd_rn(__fadd_rn(h[i], s1), s2), s3);   // ((h1 + h2) + h3) + h4
    }
    if (lane < 8) {
        const uint32_t c = cb + wc * XC + t;
        if (c < nc) {
            const uint32_t crow = rows[c];
            const float* cptr = items + (size_t)crow * ld;
            const float ch = (metric == COSINE) ? ih0[crow] : 0.f;
#pragma unroll
            for (int i = 0; i < XQ; ++i) {
                const uint32_t q = qb + wq * XQ + i;
                if (q < nq) {
                    float r = res[i];
                    const float* qptr = queries + (size_t)q * ld;
                    for (uint32_t k = m; k < d; ++k) {   // len % 32 tail: separately rounded
                        if (EUCLID) { float tt = __fsub_rn(qptr[k], cptr[k]); r = __fadd_rn(r, __fmul_rn(tt, tt)); }
                        else r = __fadd_rn(r, __fmul_rn(qptr[k], cptr[k]));
                    }
                    dist[(size_t)q * nc + c] = built_finish(metric, r, qh0 ? qh0[q] : 0.f, ch);
                }
            }
        }
    }
}

// top-k per query straight from a dense distance row: key = ordered_key(dist) << 32 | position
__global__ void __launch_bounds__(TOPK_THREADS)
topk_dense_kernel(const float* __restrict__ dist, const uint32_t* __restrict__ rows, uint32_t nc, uint32_t k, int metric,
                  uint32_t* __restrict__ out_rows, float* __restrict__ out_dist, uint32_t* __restrict__ out_len) {
    __shared__ unsigned long long buf[TOPK_CAP];
    __shared__ uint32_t fill;
    const uint32_t q = blockIdx.x;
    const float* dq = dist + (size_t)q * nc;
    const uint32_t kk = nc < k ? nc : k;
    unsigned long long threshold = ~0ull;
    uint32_t pos = 0;
    bool have = false;
    while (pos < nc) {
        const uint32_t base = have ? kk : 0u;
        const uint32_t room = TOPK_CAP - base;
        const uint32_t take = nc - pos < room ? nc - pos : room;
        __syncthreads();
        if (threadIdx.x == 0) fill = base;
        __syncthreads();
        for (uint32_t i = threadIdx.x; i < take; i += blockDim.x) {
            unsigned long long key = ((unsigned long long)ordered_key(dq[pos + i]) << 32) | (unsigned long long)(pos + i);
            if (key < threshold) { uint32_t s = atomicAdd(&fill, 1u); buf[s] = key; }
        }
        pos += take;
        __syncthreads();
        const uint32_t f = fill;
        int mm = 2;
        while ((uint32_t)mm < f) mm <<= 1;
        for (int i = (int)f + threadIdx.x; i < mm; i += blockDim.x) buf[i] = ~0ull;
        bitonic_sort_shared(buf, mm);
        have = true;
        threshold = (f >= kk && kk > 0) ? buf[kk - 1] : ~0ull;
    }
    __syncthreads();
    if (threadIdx.x == 0) out_len[q] = kk;
    for (uint32_t i = threadIdx.x; i < kk; i += blockDim.x) {
        uint32_t p = (uint32_t)(buf[i] & 0xffffffffull);
        out_rows[(size_t)q * k + i] = rows[p];
        out_dist[(size_t)q * k + i] = normalized_distance_dev(metric, dq[p]);
    }
}

// =================================================================================================
// Tensor-core pre-filter for the shared-candidate re-rank (SURVEY.md §8a row 9: "tensor-core
// pre-filter + exact AVX-order re-score of the top-(k + margin)").
//
// The tensor cores cannot produce the reference's value of a pair, but they can bound it. With both
// operands truncated to TF32 (10-bit mantissa) and FP32 accumulation the contraction s satisfies
//     | s - dot_ref(q, c) |  <=  rel * |q| * |c|,      rel = 2^-8 + d * 2^-22
// (Cauchy-Schwarz over the per-element relative errors 2 * 2^-10, the accumulation error, and the
// reference's own FP32 rounding of dot_ref; about 2x slack). E(q) charges rel (qn + sub) (gmax + sub),
// sub = sqrt(d + 64) 2^-74: the fp32 norms qn and gmax may have underflowed (frerank.cuh derives sub),
// and sub also covers operands below 2^-126, which the conversion may flush to zero (a loss of at most
// sqrt(d) 2^-126 (|q| + |c|) over the row, far below 2^-8 sub (|q| + |c|)). tcgemm.cuh turns s into an estimate
// a(q, c) of built_distance in its epilogue; for a query q every pair then satisfies
//     | a(q, c) - built_distance_ref(q, c) |  <=  E(q)
// where E(q) uses the largest candidate norm (xf_query_prep_kernel). Let a_(k) be the k-th smallest
// estimate of the query. At least k candidates have a distance <= a_(k) + E, so a candidate of the
// true top-k has a <= a_(k) + 2 E: everything above that is discarded, the survivors (a few hundred
// of 100 000 for BASELINE config 5) are re-scored by distance_kernel in the reference's exact
// summation order and ranked by topk_kernel. Ids and distances are therefore bit-identical to the
// exact path. Survivors are kept in candidate order, which keeps the (distance, id) tie-break of
// reader.rs:390. Estimates that are NaN / infinite count as "unknown" and always survive.
// =================================================================================================
constexpr int XF_THREADS = 512;
constexpr int XF_BINS = 4096;
constexpr int XF_STAGE = 2048;
constexpr uint32_t XF_SAMPLE = 4;

inline float xf_rel(uint32_t d) { return 0.00390625f + (float)d * 2.384185791015625e-07f; }   // 2^-8 + d 2^-22
// Cosine: the smallest header norm whose row gets a known estimate. A row's fp32 sum of squares may lose up to (d + 40) 2^-150
// to underflow, so its true |c| can be many times its header; from sqrt(d + 64) 2^-70 on, |c| <= header (1 + 2^-11) (1 + small).
// Rows below it have an unknown estimate (NaN) and always survive; the reference still sees pnqn > EPSILON for them.
inline float cos_header_min(uint32_t d) { return sqrtf((float)d + 64.0f) * 8.470329472543003e-22f; }   // sqrt(d + 64) 2^-70

// dst[c] = items[rows[c]] (ld floats per row), float4 granularity
__global__ void xf_gather_kernel(float4* __restrict__ dst, const float4* __restrict__ items, const uint32_t* __restrict__ rows, uint32_t nc, uint32_t ld4) {
    const uint64_t total = (uint64_t)nc * ld4;
    for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (uint64_t)gridDim.x * blockDim.x) {
        const uint32_t c = (uint32_t)(i / ld4), k = (uint32_t)(i - (uint64_t)c * ld4);
        dst[i] = items[(uint64_t)rows[c] * ld4 + k];
    }
}

// per-candidate epilogue constants (see TgEpilogue) and gmax = max over candidates of the factor
// the error bound grows with: |c| (Euclidean, DotProduct) or |c| / header norm (Cosine, normally 1)
__global__ void xf_cand_prep_kernel(const float* __restrict__ cnorm, const float* __restrict__ ih0, const uint32_t* __restrict__ rows, uint32_t nc, int metric,
                                    float hmin, float* __restrict__ ca, float* __restrict__ cb, uint32_t* __restrict__ gmax_bits) {
    uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    float g = 0.f;
    if (i < nc) {
        const float cn = cnorm[i];
        g = cn;
        float a = 0.f, b = 0.f;
        if (metric == EUCLIDEAN) a = __fmul_rn(cn, cn);
        else if (metric == COSINE) {
            b = ih0[rows[i]];
            if (b >= hmin) { a = __fdiv_rn(1.0f, b); g = __fmul_rn(cn, a); }   // hmin = cos_header_min(d)
            else { a = __uint_as_float(0x7fc00000u); g = 0.f; }   // the estimate is exactly 0 (pnqn <= EPSILON) or unknown
        }
        ca[i] = a; cb[i] = b;
        if (!(g == g)) g = __uint_as_float(0x7f800000u);
    }
    g = fabsf(g);
    uint32_t bits = __reduce_max_sync(0xffffffffu, __float_as_uint(g));
    if ((threadIdx.x & 31) == 0 && bits) atomicMax(gmax_bits, bits);
}

// per-query epilogue constants and E(q) (stored as 2 E, slightly inflated)
__global__ void xf_query_prep_kernel(const float* __restrict__ qnorm, const float* __restrict__ qh0, uint32_t m, int metric, float rel, uint32_t d,
                                     const uint32_t* __restrict__ gmax_bits, float* __restrict__ qa, float* __restrict__ qb, float* __restrict__ two_e) {
    uint32_t q = blockIdx.x * blockDim.x + threadIdx.x;
    if (q >= m) return;
    const float qn = qnorm[q], gmax = __uint_as_float(*gmax_bits);
    const float sub = __fmul_rn(sqrtf((float)d + 64.0f), 5.293955920339377e-23f);   // sqrt(d + 64) 2^-74: underflowed norms, flushed operands
    const float eps = __fmaf_rn(rel, __fmul_rn(__fadd_rn(qn, sub), __fadd_rn(gmax, sub)), 1e-30f);
    float a = 0.f, b = 0.f, e;
    if (metric == DOT_PRODUCT) e = eps;
    else if (metric == EUCLIDEAN) {
        a = __fmul_rn(qn, qn);
        const float slack = ((float)(d / 32u) + 16.0f) * 2.384185791015625e-07f;   // reference + estimate rounding, relative to |q|^2 + |c|^2
        e = __fmaf_rn(slack, __fadd_rn(a, __fmul_rn(gmax, gmax)), __fmul_rn(2.0f, eps));
    } else {
        b = qh0[q];
        if (b >= 1e-30f) { a = __fdiv_rn(1.0f, b); e = __fmaf_rn(__fmul_rn(0.5f, eps), a, 1.9073486328125e-06f /* 2^-19 */); }
        else { a = __uint_as_float(0x7fc00000u); e = 1.9073486328125e-06f; }
    }
    qa[q] = a; qb[q] = b;
    two_e[q] = __fmul_rn(__fmul_rn(2.0f, e), 1.0009765625f);
}

// monotone float -> uint32 key for finite estimates; NaN / infinite estimates are "unknown" = max
__device__ __forceinline__ uint32_t xf_key(float a) {
    const uint32_t b = __float_as_uint(a);
    return fabsf(a) <= 3.0e38f ? (b ^ ((b & 0x80000000u) ? 0xffffffffu : 0x80000000u)) : 0xffffffffu;
}
__device__ __forceinline__ float xf_unkey(uint32_t k) {   // inverse of xf_key for finite values
    return __uint_as_float(k ^ ((k & 0x80000000u) ? 0x80000000u : 0xffffffffu));
}
__device__ __forceinline__ bool xf_unknown(float a) { return !(fabsf(a) <= 3.0e38f); }
__device__ __forceinline__ uint32_t xf_widen(uint32_t key, float two_e) {   // key of (value + 2E), max if not finite
    if (key == 0xffffffffu) return key;
    return xf_key(__fadd_rn(xf_unkey(key), two_e));
}

// exclusive scan of one value per thread over the CTA (XF_THREADS threads); returns the exclusive
// prefix, *total = sum. sm: 17 uint32.
__device__ __forceinline__ uint32_t xf_block_scan(uint32_t v, uint32_t* sm, uint32_t* total) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    uint32_t inc = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) { uint32_t t = __shfl_up_sync(0xffffffffu, inc, o); if (lane >= o) inc += t; }
    __syncthreads();
    if (lane == 31) sm[warp] = inc;
    __syncthreads();
    if (warp == 0) {
        uint32_t w = lane < (XF_THREADS / 32) ? sm[lane] : 0u, winc = w;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) { uint32_t t = __shfl_up_sync(0xffffffffu, winc, o); if (lane >= o) winc += t; }
        if (lane < (XF_THREADS / 32)) sm[lane] = winc - w;
        if (lane == 31) sm[16] = winc;
    }
    __syncthreads();
    const uint32_t res = sm[warp] + inc - v;
    *total = sm[16];
    return res;
}

// smallest bin b with (number of entries in bins <= b) >= want; *before = entries in bins < b
__device__ __forceinline__ uint32_t xf_find_bin(const uint32_t* hist, uint32_t want, uint32_t* sm, uint32_t* sh_out /* 2 uint32 */, uint32_t* before) {
    constexpr int PER = XF_BINS / XF_THREADS;
    uint32_t local = 0;
#pragma unroll
    for (int i = 0; i < PER; ++i) local += hist[threadIdx.x * PER + i];
    uint32_t total;
    uint32_t ex = xf_block_scan(local, sm, &total);
    if (threadIdx.x == 0) { sh_out[0] = XF_BINS - 1; sh_out[1] = total; }   // fewer than `want` entries: last bin
    __syncthreads();
    if (ex < want && ex + local >= want) {
        uint32_t cum = ex;
        for (int i = 0; i < PER; ++i) {
            uint32_t h = hist[threadIdx.x * PER + i];
            if (cum + h >= want) { sh_out[0] = threadIdx.x * PER + i; sh_out[1] = cum; break; }
            cum += h;
        }
    }
    __syncthreads();
    *before = sh_out[1];
    return sh_out[0];
}

__device__ __forceinline__ void xf_bitonic_u32(uint32_t* buf, int n /* power of two */) {
    for (int size = 2; size <= n; size <<= 1)
        for (int stride = size >> 1; stride > 0; stride >>= 1) {
            __syncthreads();
            for (int t = threadIdx.x; t < (n >> 1); t += XF_THREADS) {
                int i = 2 * t - (t & (stride - 1)), j = i + stride;
                bool up = ((i & size) == 0);
                uint32_t a = buf[i], b = buf[j];
                if ((a > b) == up) { buf[i] = b; buf[j] = a; }
            }
        }
    __syncthreads();
}

// One CTA per query, over the query's row of estimates A[q][0..nc).
//  1. t0: a loose upper bound of the k-th smallest estimate, from a sample (every 4th group of 32
//     candidates): the r-th smallest sample key, r = k p + 4 sqrt(k p) + 4 (p = sample fraction),
//     located with linear-range histograms (the keys of the range spread over the bins).
//  2. One pass over all candidates: count a <= t0 (t0 is valid iff that reaches k) and stage every
//     candidate with a <= t0 + 2E (or unknown) in shared memory.
//  3. t1 = the exact k-th smallest estimate (it is staged); survivors = staged with a <= t1 + 2E,
//     written in candidate order.
// Anything unusual (t0 not valid, more than XF_STAGE staged, more than `cap` survivors, E not
// finite) raises *overflow and the caller takes the exact dense kernel for the chunk.
__global__ void __launch_bounds__(XF_THREADS)
xf_select_kernel(const float* __restrict__ A, uint32_t lds, uint32_t nc, uint32_t k, const float* __restrict__ two_e_q, const uint32_t* __restrict__ rows, uint32_t cap,
                 uint32_t* __restrict__ sel_rows, uint64_t* __restrict__ seg_beg, uint64_t* __restrict__ seg_end, int* __restrict__ overflow) {
    __shared__ uint32_t u_mem[XF_BINS];               // histogram, later sort buffers
    __shared__ uint32_t st_key[XF_STAGE], st_pos[XF_STAGE];
    __shared__ uint32_t sm_scan[17];
    __shared__ uint32_t sh_out[2];
    __shared__ uint32_t sh_min, sh_max, sh_ns, sh_cnt, sh_nlow, sh_cnt2;
    const uint32_t q = blockIdx.x;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const float* a = A + (size_t)q * lds;
    const float two_e = two_e_q[q];
    if (threadIdx.x == 0) { sh_min = 0xffffffffu; sh_max = 0u; sh_ns = 0u; sh_cnt = 0u; sh_nlow = 0u; sh_cnt2 = 0u; seg_beg[q] = (uint64_t)q * cap; seg_end[q] = (uint64_t)q * cap; }
    __syncthreads();
    if (!(two_e >= 0.0f && two_e <= 3.0e38f)) { if (threadIdx.x == 0) atomicExch(overflow, 1); return; }

    // t0 (key) / t0f (float): loose upper bound of the k-th smallest estimate; T0f = t0f + 2E
    uint32_t t0 = 0xffffffffu;
    if (nc > k) {
        const uint32_t sf = (nc >= 16384u && nc >= 64u * k) ? XF_SAMPLE : 1u;
        const uint32_t groups = (nc + 31u) / 32u, sgroups = (groups + sf - 1u) / sf;
        uint32_t mn = 0xffffffffu, mx = 0u, cnt = 0u;
        for (uint32_t j = warp; j < sgroups; j += XF_THREADS / 32) {
            const uint32_t c = j * sf * 32u + lane;
            if (c < nc) { const uint32_t key = xf_key(a[c]); mn = min(mn, key); mx = max(mx, key); ++cnt; }
        }
        mn = __reduce_min_sync(0xffffffffu, mn); mx = __reduce_max_sync(0xffffffffu, mx); cnt = __reduce_add_sync(0xffffffffu, cnt);
        if (lane == 0) { atomicMin(&sh_min, mn); atomicMax(&sh_max, mx); atomicAdd(&sh_ns, cnt); }
        __syncthreads();
        const uint32_t ns = sh_ns;
        uint32_t rlo = sh_min, rhi = sh_max;
        uint32_t want;
        if (sf == 1u) want = k;
        else {
            const float mean = (float)k * (float)ns / (float)nc;
            want = (uint32_t)(mean + 4.0f * sqrtf(mean) + 4.0f) + 1u;
        }
        if (want > ns) want = ns;
        for (int level = 0; level < 3 && rhi > rlo; ++level) {
            for (int i = threadIdx.x; i < XF_BINS; i += XF_THREADS) u_mem[i] = 0;
            __syncthreads();
            // bin = (key - rlo) >> shift with the smallest shift that keeps every key of the range below XF_BINS
            const uint32_t span = rhi - rlo;
            const int shift = span < XF_BINS ? 0 : (32 - __clz(span)) - 12;
            for (uint32_t j = warp; j < sgroups; j += XF_THREADS / 32) {
                const uint32_t c = j * sf * 32u + lane;
                if (c < nc) {
                    const uint32_t key = xf_key(a[c]);
                    if (key >= rlo && key <= rhi) atomicAdd(&u_mem[(key - rlo) >> shift], 1u);
                }
            }
            __syncthreads();
            uint32_t before;
            const uint32_t b = xf_find_bin(u_mem, want, sm_scan, sh_out, &before);
            const uint32_t in_bin = u_mem[b];
            __syncthreads();
            const uint32_t nlo = rlo + (b << shift);
            const uint32_t top = (uint32_t)min((unsigned long long)rhi, (unsigned long long)rlo + (((unsigned long long)b + 1ull) << shift) - 1ull);
            want -= before; rlo = nlo; rhi = top;
            if (in_bin <= 32u || shift == 0) break;
        }
        t0 = rhi;
    }
    const bool all = t0 == 0xffffffffu;
    const float t0f = all ? 0.f : xf_unkey(t0);
    const float T0f = all ? 0.f : __fadd_rn(t0f, two_e);
    const bool wide = all || xf_unknown(T0f);          // threshold not finite: everything is staged (and overflows)

    // full pass: stage a <= t0 + 2E (or unknown), count known a <= t0
    uint32_t nlow = 0;
    auto visit = [&](float v, uint32_t c) {
        nlow += (v <= t0f && v >= -3.0e38f) ? 1u : 0u;
        if (wide || !(v > T0f && v <= 3.0e38f)) {
            const uint32_t i = atomicAdd(&sh_cnt, 1u);
            if (i < XF_STAGE) { st_key[i] = xf_key(v); st_pos[i] = c; }
        }
    };
    const uint32_t nc4 = nc & ~3u;
    const float4* a4 = reinterpret_cast<const float4*>(a);           // lds % 4 == 0 and A is 16-byte aligned
    for (uint32_t c = threadIdx.x * 4u; c < nc4; c += XF_THREADS * 4u) {
        const float4 v = __ldg(a4 + (c >> 2));
        visit(v.x, c); visit(v.y, c + 1u); visit(v.z, c + 2u); visit(v.w, c + 3u);
    }
    if (threadIdx.x < nc - nc4) visit(a[nc4 + threadIdx.x], nc4 + threadIdx.x);
    nlow = __reduce_add_sync(0xffffffffu, nlow);
    if (lane == 0 && nlow) atomicAdd(&sh_nlow, nlow);
    __syncthreads();
    const uint32_t staged = sh_cnt;
    if (staged > XF_STAGE || (nc > k && (all || sh_nlow < k))) { if (threadIdx.x == 0) atomicExch(overflow, 1); return; }

    // t1 = exact k-th smallest estimate
    uint32_t T1 = 0xffffffffu;
    if (nc > k) {
        int np2 = 2;
        while ((uint32_t)np2 < staged) np2 <<= 1;
        for (int i = threadIdx.x; i < np2; i += XF_THREADS) u_mem[i] = (uint32_t)i < staged ? st_key[i] : 0xffffffffu;
        xf_bitonic_u32(u_mem, np2);
        T1 = xf_widen(u_mem[k - 1], two_e);
        __syncthreads();
    }
    for (uint32_t i = threadIdx.x; i < staged; i += XF_THREADS)
        if (st_key[i] <= T1 || st_key[i] == 0xffffffffu) u_mem[atomicAdd(&sh_cnt2, 1u)] = st_pos[i];
    __syncthreads();
    const uint32_t keep = sh_cnt2;
    int kp2 = 2;
    while ((uint32_t)kp2 < keep) kp2 <<= 1;
    for (int i = keep + threadIdx.x; i < kp2; i += XF_THREADS) u_mem[i] = 0xffffffffu;
    xf_bitonic_u32(u_mem, kp2);                       // back to candidate order (ties are broken by id)
    uint32_t* out = sel_rows + (size_t)q * cap;
    for (uint32_t i = threadIdx.x; i < keep && i < cap; i += XF_THREADS) out[i] = rows[u_mem[i]];
    if (threadIdx.x == 0) {
        seg_end[q] = (uint64_t)q * cap + (keep < cap ? keep : cap);
        if (keep > cap) atomicExch(overflow, 1);
    }
}

}  // namespace ab
