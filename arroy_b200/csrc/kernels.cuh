// kernels.cuh — data-parallel kernels of the hot path (sm_90a):
//   work_kernel      side()/margin scan over row lists + stable left/right partition of id lists
//                    (src/writer.rs:1201-1207 and its callers :1424-1430, :1494-1500)
//   norms_kernel     per-item sqrt(dot(v,v)) (Cosine new_header, cosine.rs:39-41;
//                    DotProduct::preprocess pass 1, dot_product.rs:132-142)
//   dot_header_kernel  DotProduct::preprocess pass 2 (dot_product.rs:146-160)
//   distance_kernel  D::built_distance(query, item) per candidate (src/reader.rs:381-391)
//   topk_kernel      k smallest by (OrderedFloat(dist), id) + D::normalized_distance (reader.rs:394-399)
//   synth_kernel     counter-based ChaCha12 synthetic matrix (SURVEY.md §8d)
// All are HBM-bound streaming kernels: 128-bit coalesced loads, warp-shuffle reductions in the
// reference's exact summation order (exact.cuh), no tensor cores.
#pragma once
#include "exact.cuh"

namespace ab {

constexpr int WORK_THREADS = 256;
constexpr int SCAN_UNIT = 64;    // rows per scan unit (8 warps x 4 groups x 2 rows)
constexpr int PART_UNIT = 256;   // ids per partition unit (= 4 scan units)

enum : int { JOB_NONE = 0, JOB_SCAN = 1, JOB_PARTITION = 2 };

// A normal as the kernels read it: [h0, h1, 0, 0, v[ld]] (16-byte aligned vector part).
constexpr int NORMAL_HDR = 4;

struct Job {
    int32_t kind;
    uint32_t len;            // rows in the node
    const uint32_t* rows;    // scan: ascending row indices (NULL = identity); partition: source ids
    const float* normal;     // scan: [h0,h1,_,_,v[ld]]
    uint8_t* flags;          // scan out / partition in: 1 = Right, 0 = Left, per position
    float* margins;          // scan out, optional
    uint32_t* unit_left;     // scan out: Left count per SCAN_UNIT; partition in: exclusive prefix of it
    uint32_t* dst;           // partition out: [0,total_left) lefts then rights, both in source order
    uint32_t total_left;
    uint32_t pad;
};

__device__ __forceinline__ float4 ldg_stream(const float4* p) {
    float4 v;
    asm volatile("ld.global.nc.L1::no_allocate.v4.f32 {%0,%1,%2,%3}, [%4];"
                 : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "l"(p));
    return v;
}

__device__ __forceinline__ float margin_finish(int metric, float dot, float nh0, float item_h0) {
    // euclidean.rs:79-81 / manhattan.rs:82-84: bias + dot; cosine.rs:87-89: dot;
    // dot_product.rs:115-117: dot + n.extra_dim * q.extra_dim (two roundings)
    // binary_quantized_euclidean.rs:95-97 / _manhattan.rs:99-101: bias + dot; binary_quantized_cosine.rs:95-97: dot
    if (metric == COSINE || metric == BQ_COSINE) return dot;
    if (metric == DOT_PRODUCT) return __fadd_rn(dot, __fmul_rn(nh0, item_h0));
    return __fadd_rn(nh0, dot);
}

// One scan unit: SCAN_UNIT consecutive positions of a job. d >= 32: 8 lanes per row, float4
// loads, two rows in flight per group. sm_normal: the job's normal vector in shared memory.
// DEEP: eight 32-float chunks of both rows in flight instead of four (the persistent schedule runs fewer scanning warps per SM
// than work_kernel's three CTAs, so each warp has to keep more bytes in flight to saturate HBM).
template <bool DEEP = false>
__device__ __forceinline__ void scan_unit(const Job& jb, uint32_t unit, const float* __restrict__ items, const float* __restrict__ ih0,
                                          uint32_t d, uint32_t ld, int metric, const float* sm_normal, float nh0, uint32_t* sm_count) {
    const uint32_t base = unit * SCAN_UNIT;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    if (threadIdx.x == 0) *sm_count = 0;
    __syncthreads();
    if (d >= 32) {
        const int g8 = lane & 7, grp = lane >> 3;
        const uint32_t slot = warp * 8 + grp * 2;  // first of the two positions of this group
        uint32_t pa = base + slot, pb = base + slot + 1;
        const bool va = pa < jb.len, vb = pb < jb.len;
        uint32_t ra = 0, rb = 0;
        // (id lists, flags and unit counts change between jobs of ONE persistent kernel: they are read through L2, never L1)
        if (va) ra = jb.rows ? __ldcg(jb.rows + pa) : pa;
        if (vb) rb = jb.rows ? __ldcg(jb.rows + pb) : pb;
        const float4* A = reinterpret_cast<const float4*>(items + (size_t)ra * ld);
        const float4* B = reinterpret_cast<const float4*>(items + (size_t)rb * ld);
        const float4* N = reinterpret_cast<const float4*>(sm_normal);
        float4 acca = make_float4(0.f, 0.f, 0.f, 0.f), accb = acca;
        const int nch = d >> 5;
        int c = 0;
        if (DEEP) {
            for (; c + 8 <= nch; c += 8) {
                float4 x[8], z[8];
#pragma unroll
                for (int u = 0; u < 8; ++u) { x[u] = ldg_stream(A + (c + u) * 8 + g8); z[u] = ldg_stream(B + (c + u) * 8 + g8); }
#pragma unroll
                for (int u = 0; u < 8; ++u) {
                    const float4 y = N[(c + u) * 8 + g8];
                    acca.x = fmaf(x[u].x, y.x, acca.x); acca.y = fmaf(x[u].y, y.y, acca.y);
                    acca.z = fmaf(x[u].z, y.z, acca.z); acca.w = fmaf(x[u].w, y.w, acca.w);
                    accb.x = fmaf(z[u].x, y.x, accb.x); accb.y = fmaf(z[u].y, y.y, accb.y);
                    accb.z = fmaf(z[u].z, y.z, accb.z); accb.w = fmaf(z[u].w, y.w, accb.w);
                }
            }
        }
#pragma unroll 4
        for (; c < nch; ++c) {
            float4 x = ldg_stream(A + c * 8 + g8);
            float4 z = ldg_stream(B + c * 8 + g8);
            float4 y = N[c * 8 + g8];
            acca.x = fmaf(x.x, y.x, acca.x); acca.y = fmaf(x.y, y.y, acca.y);
            acca.z = fmaf(x.z, y.z, acca.z); acca.w = fmaf(x.w, y.w, acca.w);
            accb.x = fmaf(z.x, y.x, accb.x); accb.y = fmaf(z.y, y.y, accb.y);
            accb.z = fmaf(z.z, y.z, accb.z); accb.w = fmaf(z.w, y.w, accb.w);
        }
        float da = group8_hsum(acca), db = group8_hsum(accb);
        const float* rowa = items + (size_t)ra * ld;
        const float* rowb = items + (size_t)rb * ld;
        for (uint32_t i = nch * 32; i < d; ++i) {  // len % 32 tail: separately rounded mul, add
            da = __fadd_rn(da, __fmul_rn(rowa[i], sm_normal[i]));
            db = __fadd_rn(db, __fmul_rn(rowb[i], sm_normal[i]));
        }
        float ma = margin_finish(metric, da, nh0, (metric == DOT_PRODUCT) ? ih0[ra] : 0.f);
        float mb = margin_finish(metric, db, nh0, (metric == DOT_PRODUCT) ? ih0[rb] : 0.f);
        int sa = side_of(ma), sb = side_of(mb);
        const bool leader = g8 == 0;
        if (leader && va) { if (jb.flags) jb.flags[pa] = (uint8_t)sa; if (jb.margins) jb.margins[pa] = ma; }
        if (leader && vb) { if (jb.flags) jb.flags[pb] = (uint8_t)sb; if (jb.margins) jb.margins[pb] = mb; }
        unsigned la = __ballot_sync(0xffffffffu, leader && va && sa == 0);
        unsigned lb = __ballot_sync(0xffffffffu, leader && vb && sb == 0);
        if (lane == 0) { int c = __popc(la) + __popc(lb); if (c) atomicAdd(sm_count, (uint32_t)c); }
    } else {
        // d < 32: SSE (16..31) or scalar (<16) order, one thread per row
        int left = 0;
        if (threadIdx.x < SCAN_UNIT) {
            uint32_t p = base + threadIdx.x;
            if (p < jb.len) {
                uint32_t r = jb.rows ? __ldcg(jb.rows + p) : p;
                float dt = exact_thread<false>(items + (size_t)r * ld, sm_normal, (int)d);
                float m = margin_finish(metric, dt, nh0, (metric == DOT_PRODUCT) ? ih0[r] : 0.f);
                int s = side_of(m);
                if (jb.flags) jb.flags[p] = (uint8_t)s;
                if (jb.margins) jb.margins[p] = m;
                left = (s == 0);
            }
        }
        unsigned l = __ballot_sync(0xffffffffu, left);
        if (lane == 0 && l) atomicAdd(sm_count, (uint32_t)__popc(l));
    }
    __syncthreads();
    if (threadIdx.x == 0 && jb.unit_left) jb.unit_left[unit] = *sm_count;
}

// ---- side() through a two-plane 8-bit pre-filter of the items -----------------------------------------------------------
// side() only needs the SIGN of the margin, and a scan is bound by the bytes of the rows it reads. Every row is encoded once per
// staging (planes_encode_kernel) as a scale s = fl(M / 127), M = max_i |x_i|, and two int8 planes (u = 2^-24):
//     q_i = fl(x_i / s),   h_i = rint(q_i),   l_i = rint(fl((q_i - h_i) * 254))      (q_i - h_i is exact)
// The quotient is rounded once and the constants are rounded up to cover it (|q_i| <= 127 (1 + u)): |x_i - s h_i| <= s E1,
// E1 = 1/2 + 128 u, and with y_i = 254 h_i + l_i (an exact integer in f32), |x_i - s y_i / 254| <= s E2, E2 = 1/508 + 129 u < 0.001977.
// A row whose scale is not a normal finite f32 keeps zero planes and is never decided through them: M = 0 stores s = 0 (the
// row's dot is exactly 0), M = inf stores +inf, a NaN or tiny (M < 127 FLT_MIN) row stores NaN (0x7fffffff); the tests below
// are false for NaN and +inf.
// The reference's margin is fl(dot + c) (c = the bias / extra-dim term, formed exactly as the reference forms it; fl keeps the
// sign of dot + c), with |dot - sum n_i x_i| <= gamma_R sum |n_i x_i|, gamma_R <= 1.001 d u in any summation order, and
// sum |n_i x_i| <= 127.001 s |n|_1. A lane sums a row in two f32 chains of at most ld/16 + 7 terms, then 1 + 3 adds: gamma_k <=
// (d/8 + 16) u for either stage. N1 >= |n|_1 is summed in f64 once per job and rounded up.
//  stage 1, hi plane only (d bytes per row): t = f32 sum n_i h_i (sum |n_i h_i| <= 127 |n|_1), and
//    |dot - fl(s t)| <= s |n|_1 (E1 + 127.001 (gamma_R + gamma_k + u)) <= s N1 K1(d) / (1 + 2^-20),  K1(d) = 0.5002 + 8.6e-6 d;
//    the row is certain when |fl(fl(s t) + c)| > fl(s w1), w1 = N1 K1(d) rounded up (the factor 1 + 2^-20 covers the test's
//    own roundings).
//  stage 2, the rows stage 1 left (both planes; the hi row was just streamed by this CTA): m = f32 sum n_i y_i,
//    A = f32 sum |n_i| |y_i|, s2 = fl(s / 254), and
//    |dot - fl(s2 m)| <= s2 (254 E2 |n|_1 (1 + gamma_R) + A (gamma_R + gamma_k + 4 u)) <= s2 (N1 W2(d) + rel2(d) A) / (1 + 2^-20),
//    W2(d) = 0.50216 (1 + 6.1e-8 (d + 16)), rel2(d) = 1.3e-6 + 6.8e-8 d; certain when |fl(fl(s2 m) + c)| > fl(s2 fl(w2 + fl(rel2 A))),
//    w2 = N1 W2(d) rounded up.
//  stage 3: every other row — near the hyperplane, zero, non-finite — is scored from the f32 row in the reference's summation
//    order (scan_unit's arithmetic). Flags and unit counts are the exact scan's.
// The bounds are relative: like any such rule they assume that no product n_i x_i underflows.
// sm_perm: the normal re-laid for the planes' lane order: the 16 elements of 16-byte word q = 8 c + g of a row sit at float4
// 32 c + 8 j + g (j = 0..3, four elements each), so that the eight lanes of a row read consecutive float4s.
__host__ __device__ __forceinline__ float planes_k1(uint32_t d) { return 0.5002f + (float)d * 8.6e-6f; }
__host__ __device__ __forceinline__ float planes_w2(uint32_t d) { return 0.50216f * (1.0f + 6.1e-8f * (float)(d + 16u)); }
__host__ __device__ __forceinline__ float planes_rel2(uint32_t d) { return 1.3e-6f + (float)d * 6.8e-8f; }
__host__ __device__ __forceinline__ uint32_t planes_perm_floats(uint32_t ld) { return (ld + 127u) & ~127u; }   // sm_perm's size
__host__ __device__ __forceinline__ uint32_t planes_perm_index(uint32_t i) {
    const uint32_t q = i >> 4, w = i & 15u;
    return (((q >> 3) * 32u + (w >> 2) * 8u + (q & 7u)) << 2) + (w & 3u);
}
constexpr uint32_t PLANES_MAX_D = 8192;
constexpr uint32_t PLANES_CHUNK = 4;          // scan units per claim on this path (256 rows)

struct PlaneRows {
    const int8_t* hi;       // n x ld, h_i
    const int8_t* lo;       // n x ld, l_i
    const float* scale;     // n, s
};

// Encoder: one warp per row. Padding columns are zero in the items, so they are zero in both planes.
__global__ void __launch_bounds__(256) planes_encode_kernel(const float* __restrict__ items, uint64_t n, uint32_t ld, int8_t* __restrict__ hi,
                                                            int8_t* __restrict__ lo, float* __restrict__ scale) {
    const int lane = threadIdx.x & 31;
    const uint32_t n4 = ld >> 2;
    const uint64_t nw = (uint64_t)gridDim.x * (blockDim.x >> 5);
    for (uint64_t r = (uint64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); r < n; r += nw) {
        const float4* row = reinterpret_cast<const float4*>(items + r * ld);
        uint32_t mb = 0;   // max of |x| as bits: the uint order of non-negative floats, with NaN above +inf
        for (uint32_t k = lane; k < n4; k += 32) {
            const float4 v = row[k];
            mb = max(max(mb, __float_as_uint(fabsf(v.x))), max(__float_as_uint(fabsf(v.y)), max(__float_as_uint(fabsf(v.z)), __float_as_uint(fabsf(v.w)))));
        }
        mb = __reduce_max_sync(0xffffffffu, mb);
        const float M = __uint_as_float(mb);
        float s = __fdiv_rn(M, 127.0f);
        const bool ok = s >= 1.17549435e-38f && s <= 3.40282347e+38f;
        if (!ok && mb != 0u && mb != 0x7f800000u) s = __int_as_float(0x7fffffff);
        uint32_t* H = reinterpret_cast<uint32_t*>(hi + r * ld);
        uint32_t* L = reinterpret_cast<uint32_t*>(lo + r * ld);
        for (uint32_t k = lane; k < n4; k += 32) {
            const float4 v = row[k];
            const float x[4] = {v.x, v.y, v.z, v.w};
            uint32_t hw = 0, lw = 0;
            if (ok) {
#pragma unroll
                for (int j = 0; j < 4; ++j) {
                    const float q = __fdiv_rn(x[j], s), h = rintf(q);
                    const float l = rintf(__fmul_rn(__fsub_rn(q, h), 254.0f));
                    hw |= ((uint32_t)(int)h & 0xffu) << (8 * j);
                    lw |= ((uint32_t)(int)l & 0xffu) << (8 * j);
                }
            }
            H[k] = hw; L[k] = lw;
        }
        if (lane == 0) scale[r] = s;
    }
}

__device__ __forceinline__ uint4 ldg_stream_u4(const uint4* p) {
    uint4 v;
    asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(p));
    return v;
}
// byte k of w (signed) as a float, without I2F: b ^ 0x80 = b + 128 is put into the mantissa of 2^23 (exactly 2^23 + 128 + b),
// one add removes the offset. wx = w ^ 0x80808080.
__device__ __forceinline__ float s8_to_f32(uint32_t wx, uint32_t k) {
    return __fsub_rn(__uint_as_float(__byte_perm(wx, 0x4B000000u, 0x7540u | k)), 8388736.0f);
}
// 16 hi-plane elements of one word times their normal elements (y: the four float4s of sm_perm for this word): two chains
__device__ __forceinline__ void planes_fma16(const uint4 v, const float4 (&y)[4], float& m0, float& m1) {
    const uint32_t w[4] = {v.x ^ 0x80808080u, v.y ^ 0x80808080u, v.z ^ 0x80808080u, v.w ^ 0x80808080u};
#pragma unroll
    for (int j = 0; j < 4; ++j) {
        m0 = fmaf(s8_to_f32(w[j], 0), y[j].x, m0); m1 = fmaf(s8_to_f32(w[j], 1), y[j].y, m1);
        m0 = fmaf(s8_to_f32(w[j], 2), y[j].z, m0); m1 = fmaf(s8_to_f32(w[j], 3), y[j].w, m1);
    }
}
// the same word of both planes: y = 254 h + l (exact), m += n y, a += |n| |y|
__device__ __forceinline__ void planes_fma16x2(const uint4 vh, const uint4 vl, const float4 (&y)[4], float& m0, float& m1, float& a0, float& a1) {
    const uint32_t wh[4] = {vh.x ^ 0x80808080u, vh.y ^ 0x80808080u, vh.z ^ 0x80808080u, vh.w ^ 0x80808080u};
    const uint32_t wl[4] = {vl.x ^ 0x80808080u, vl.y ^ 0x80808080u, vl.z ^ 0x80808080u, vl.w ^ 0x80808080u};
#pragma unroll
    for (int j = 0; j < 4; ++j) {
        const float n4[4] = {y[j].x, y[j].y, y[j].z, y[j].w};
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            const float v = fmaf(s8_to_f32(wh[j], (uint32_t)k), 254.0f, s8_to_f32(wl[j], (uint32_t)k));
            if (k & 1) { m1 = fmaf(v, n4[k], m1); a1 = fmaf(fabsf(v), fabsf(n4[k]), a1); }
            else { m0 = fmaf(v, n4[k], m0); a0 = fmaf(fabsf(v), fabsf(n4[k]), a0); }
        }
    }
}

__device__ __forceinline__ float prefilter_finish(int metric, float v, float nh0, float item_h0) {
    if (metric == COSINE) return v;
    if (metric == DOT_PRODUCT) return __fadd_rn(v, __fmul_rn(nh0, item_h0));
    return __fadd_rn(nh0, v);
}

// scan units [u0, u1) (at most PLANES_CHUNK) of a job. sm_list, sm_list2: 64 * PLANES_CHUNK positions each (the rows stage 1,
// stage 2 left); sm_cnt: PLANES_CHUNK + 2 counters. w1, w2: the job's bound factors (above). stats (optional): [0] rows through
// the pre-filter, [1] of them re-scored from the f32 row, [2] of them that went through stage 2.
__device__ __forceinline__ void scan_claim_planes(const Job& jb, uint32_t u0, uint32_t u1, const float* __restrict__ items, const PlaneRows pl,
                                                  const float* __restrict__ ih0, uint32_t d, uint32_t ld, int metric, const float* sm_normal, const float* sm_perm,
                                                  float nh0, float w1, float w2, uint32_t* sm_list, uint32_t* sm_list2, uint32_t* sm_cnt, unsigned long long* stats) {
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, g8 = lane & 7, grp = lane >> 3;
    if (tid <= (int)PLANES_CHUNK + 1) sm_cnt[tid] = 0;
    __syncthreads();
    const uint32_t base = u0 * SCAN_UNIT, end = min(jb.len, u1 * SCAN_UNIT);
    const uint32_t nq = ld >> 4;                       // 16-byte words per plane row
    const int nsteps = (int)((nq + 7) >> 3);
    const float4* PN = reinterpret_cast<const float4*>(sm_perm);
    // ---- stage 1: the hi plane of every row ----
    for (uint32_t pbase = base; pbase < end; pbase += 128) {
        uint32_t pos[4], rid[4];
        const uint4* S[4];
#pragma unroll
        for (int r = 0; r < 4; ++r) {
            pos[r] = pbase + warp * 16 + grp * 4 + r;
            rid[r] = pos[r] < end ? (jb.rows ? __ldcg(jb.rows + pos[r]) : pos[r]) : 0u;
            S[r] = reinterpret_cast<const uint4*>(pl.hi + (size_t)rid[r] * ld) + g8;
        }
        float m0[4], m1[4];
#pragma unroll
        for (int r = 0; r < 4; ++r) { m0[r] = 0.f; m1[r] = 0.f; }
        for (int c0 = 0; c0 < nsteps; c0 += 3) {
            uint4 v[3][4];
#pragma unroll
            for (int sidx = 0; sidx < 3; ++sidx)
#pragma unroll
                for (int r = 0; r < 4; ++r) {
                    const uint32_t q = (uint32_t)(c0 + sidx) * 8u + (uint32_t)g8;
                    v[sidx][r] = q < nq ? ldg_stream_u4(S[r] + (c0 + sidx) * 8) : make_uint4(0u, 0u, 0u, 0u);
                }
#pragma unroll
            for (int sidx = 0; sidx < 3; ++sidx) {
                const uint32_t q = (uint32_t)(c0 + sidx) * 8u + (uint32_t)g8;
                float4 y[4];
#pragma unroll
                for (int j = 0; j < 4; ++j) y[j] = q < nq ? PN[(c0 + sidx) * 32 + j * 8 + g8] : make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
                for (int r = 0; r < 4; ++r) planes_fma16(v[sidx][r], y, m0[r], m1[r]);
            }
        }
#pragma unroll
        for (int r = 0; r < 4; ++r) {
            float t = m0[r] + m1[r];
#pragma unroll
            for (int o = 1; o < 8; o <<= 1) t += __shfl_xor_sync(0xffffffffu, t, o);
            const bool valid = pos[r] < end;
            const float s = valid ? __ldg(pl.scale + rid[r]) : 0.f;
            const float mt = prefilter_finish(metric, __fmul_rn(s, t), nh0, (metric == DOT_PRODUCT && valid) ? ih0[rid[r]] : 0.f);
            const bool certain = fabsf(mt) > __fmul_rn(s, w1);      // false for NaN / Inf scales
            const bool leader = g8 == 0 && valid;
            const int side = mt > 0.f ? 1 : 0;
            if (leader && certain) jb.flags[pos[r]] = (uint8_t)side;
            if (leader && !certain) sm_list[atomicAdd(&sm_cnt[PLANES_CHUNK], 1u)] = pos[r];
            const unsigned lefts = __ballot_sync(0xffffffffu, leader && certain && side == 0);
            // the four groups of a warp hold positions of the same unit (16 consecutive positions per warp)
            if (lane == 0 && lefts) atomicAdd(&sm_cnt[(pbase + warp * 16 - base) / SCAN_UNIT], (uint32_t)__popc(lefts));
        }
    }
    __syncthreads();
    // ---- stage 2: both planes of the rows stage 1 left, one 8-lane group per row ----
    const uint32_t n1 = sm_cnt[PLANES_CHUNK];
    const float rel2 = planes_rel2(d);
    for (uint32_t it = 0; it * 32u < n1; ++it) {
        const uint32_t idx = it * 32u + (uint32_t)(warp * 4 + grp);
        const bool act = idx < n1;
        const uint32_t p = act ? sm_list[idx] : base;
        const uint32_t r = jb.rows ? __ldcg(jb.rows + p) : p;
        const uint4* Hr = reinterpret_cast<const uint4*>(pl.hi + (size_t)r * ld) + g8;
        const uint4* Lr = reinterpret_cast<const uint4*>(pl.lo + (size_t)r * ld) + g8;
        float m0 = 0.f, m1 = 0.f, a0 = 0.f, a1 = 0.f;
        for (int c0 = 0; c0 < nsteps; c0 += 3) {
            uint4 vh[3], vl[3];
#pragma unroll
            for (int sidx = 0; sidx < 3; ++sidx) {
                const uint32_t q = (uint32_t)(c0 + sidx) * 8u + (uint32_t)g8;
                vh[sidx] = q < nq ? ldg_stream_u4(Hr + (c0 + sidx) * 8) : make_uint4(0u, 0u, 0u, 0u);
                vl[sidx] = q < nq ? ldg_stream_u4(Lr + (c0 + sidx) * 8) : make_uint4(0u, 0u, 0u, 0u);
            }
#pragma unroll
            for (int sidx = 0; sidx < 3; ++sidx) {
                const uint32_t q = (uint32_t)(c0 + sidx) * 8u + (uint32_t)g8;
                float4 y[4];
#pragma unroll
                for (int j = 0; j < 4; ++j) y[j] = q < nq ? PN[(c0 + sidx) * 32 + j * 8 + g8] : make_float4(0.f, 0.f, 0.f, 0.f);
                planes_fma16x2(vh[sidx], vl[sidx], y, m0, m1, a0, a1);
            }
        }
        float m = m0 + m1, a = a0 + a1;
#pragma unroll
        for (int o = 1; o < 8; o <<= 1) { m += __shfl_xor_sync(0xffffffffu, m, o); a += __shfl_xor_sync(0xffffffffu, a, o); }
        const float s2 = __fdiv_rn(__ldg(pl.scale + r), 254.0f);
        const float mt = prefilter_finish(metric, __fmul_rn(s2, m), nh0, (metric == DOT_PRODUCT) ? ih0[r] : 0.f);
        const bool certain = fabsf(mt) > __fmul_rn(s2, __fadd_rn(w2, __fmul_rn(rel2, a)));
        const int side = mt > 0.f ? 1 : 0;
        if (act && g8 == 0) {
            if (certain) { jb.flags[p] = (uint8_t)side; if (side == 0) atomicAdd(&sm_cnt[(p - base) / SCAN_UNIT], 1u); }
            else sm_list2[atomicAdd(&sm_cnt[PLANES_CHUNK + 1], 1u)] = p;
        }
    }
    __syncthreads();
    // ---- stage 3: the rows left, exactly: one 8-lane group per row, scan_unit's arithmetic ----
    const uint32_t nl = sm_cnt[PLANES_CHUNK + 1];
    if (stats != nullptr && tid == 0) {
        atomicAdd(stats, (unsigned long long)(end - base));
        if (nl) atomicAdd(stats + 1, (unsigned long long)nl);
        if (n1) atomicAdd(stats + 2, (unsigned long long)n1);
    }
    const int nch = (int)(d >> 5);
    const float4* N = reinterpret_cast<const float4*>(sm_normal);
    for (uint32_t it = 0; it * 32u < nl; ++it) {
        const uint32_t idx = it * 32u + (uint32_t)(warp * 4 + grp);
        const bool act = idx < nl;
        const uint32_t p = act ? sm_list2[idx] : base;
        const uint32_t r = jb.rows ? __ldcg(jb.rows + p) : p;
        const float4* A = reinterpret_cast<const float4*>(items + (size_t)r * ld);
        float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
        int c = 0;
        for (; c + 8 <= nch; c += 8) {
            float4 x[8];
#pragma unroll
            for (int u = 0; u < 8; ++u) x[u] = ldg_stream(A + (c + u) * 8 + g8);
#pragma unroll
            for (int u = 0; u < 8; ++u) {
                const float4 y = N[(c + u) * 8 + g8];
                acc.x = fmaf(x[u].x, y.x, acc.x); acc.y = fmaf(x[u].y, y.y, acc.y); acc.z = fmaf(x[u].z, y.z, acc.z); acc.w = fmaf(x[u].w, y.w, acc.w);
            }
        }
        for (; c < nch; ++c) {
            const float4 x = ldg_stream(A + c * 8 + g8), y = N[c * 8 + g8];
            acc.x = fmaf(x.x, y.x, acc.x); acc.y = fmaf(x.y, y.y, acc.y); acc.z = fmaf(x.z, y.z, acc.z); acc.w = fmaf(x.w, y.w, acc.w);
        }
        float da = group8_hsum(acc);
        const float* row = items + (size_t)r * ld;
        for (uint32_t i = (uint32_t)nch * 32u; i < d; ++i) da = __fadd_rn(da, __fmul_rn(row[i], sm_normal[i]));
        const int sa = side_of(margin_finish(metric, da, nh0, (metric == DOT_PRODUCT) ? ih0[r] : 0.f));
        if (act && g8 == 0) { jb.flags[p] = (uint8_t)sa; if (sa == 0) atomicAdd(&sm_cnt[(p - base) / SCAN_UNIT], 1u); }
    }
    __syncthreads();
    if (tid < (int)(u1 - u0)) jb.unit_left[u0 + tid] = sm_cnt[tid];
}

// The bound factors of a job's normal from the per-warp partial sums of |n_i| (f64, eight warps): {w1, w2}, rounded up.
__device__ __forceinline__ float2 planes_job_factors(const double* sm_l1, uint32_t d) {
    double s = 0.0;
#pragma unroll
    for (int w = 0; w < 8; ++w) s += sm_l1[w];
    s *= 1.0 + 0x1p-30;    // the f64 sum's own rounding (< 8192 * 2^-53)
    return make_float2(__double2float_ru(s * (double)planes_k1(d)), __double2float_ru(s * (double)planes_w2(d)));
}
__device__ __forceinline__ double warp_sum_f64(double v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

// Stable partition of one PART_UNIT block of ids. left_before = number of Left flags in all
// earlier positions of the node. sm_w: 2*8 uint32 scratch.
__device__ __forceinline__ void partition_block(const uint32_t* __restrict__ src, const uint8_t* __restrict__ flags, uint32_t* __restrict__ dst,
                                                uint32_t base, uint32_t len, uint32_t left_before, uint32_t total_left, uint32_t* sm_w) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    uint32_t p = base + threadIdx.x;
    bool valid = p < len;
    int f = valid ? (int)__ldcg(flags + p) : 1;
    uint32_t id = valid ? __ldcg(src + p) : 0;
    unsigned lm = __ballot_sync(0xffffffffu, valid && f == 0);
    unsigned rm = __ballot_sync(0xffffffffu, valid && f != 0);
    if (lane == 0) { sm_w[warp] = __popc(lm); sm_w[8 + warp] = __popc(rm); }
    __syncthreads();
    uint32_t lw = 0, rw = 0;
    for (int w = 0; w < warp; ++w) { lw += sm_w[w]; rw += sm_w[8 + w]; }
    unsigned below = (1u << lane) - 1u;
    if (valid) {
        if (f == 0) dst[left_before + lw + __popc(lm & below)] = id;
        else dst[total_left + (base - left_before) + rw + __popc(rm & below)] = id;
    }
    __syncthreads();
}

// Persistent-style grid: every CTA strides over the units of all posted jobs.
// Dynamic shared memory: ld floats (normal) + (njobs + 1) uint32 (unit prefix).
__global__ void __launch_bounds__(WORK_THREADS, 3)
work_kernel(const Job* __restrict__ jobs, int njobs, const float* __restrict__ items, const float* __restrict__ ih0,
            uint32_t d, uint32_t ld, int metric) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    float* sm_normal = reinterpret_cast<float*>(smem_raw);
    uint32_t* sm_prefix = reinterpret_cast<uint32_t*>(sm_normal + ld);
    __shared__ uint32_t sm_count;
    __shared__ uint32_t sm_w[16];
    // exclusive prefix of the unit counts over jobs (njobs <= a few hundred)
    for (int j = threadIdx.x; j < njobs; j += blockDim.x) {
        const int k = jobs[j].kind;
        const uint32_t len = jobs[j].len;
        sm_prefix[j] = k == JOB_SCAN ? (len + SCAN_UNIT - 1) / SCAN_UNIT : (k == JOB_PARTITION ? (len + PART_UNIT - 1) / PART_UNIT : 0u);
    }
    __syncthreads();
    if (threadIdx.x < 32) {
        const int per = (njobs + 31) / 32;
        const int b = threadIdx.x * per, e = min(b + per, njobs);
        uint32_t loc = 0;
        for (int i = b; i < e; ++i) loc += sm_prefix[i];
        uint32_t inc = loc;
        for (int o = 1; o < 32; o <<= 1) { uint32_t y = __shfl_up_sync(0xffffffffu, inc, o); if ((int)threadIdx.x >= o) inc += y; }
        uint32_t run = inc - loc;
        for (int i = b; i < e; ++i) { uint32_t x = sm_prefix[i]; sm_prefix[i] = run; run += x; }
        if (threadIdx.x == 31) sm_prefix[njobs] = inc;
    }
    __syncthreads();
    const uint32_t total = sm_prefix[njobs];
    int loaded_job = -1;
    float nh0 = 0.f;
    for (uint32_t u = blockIdx.x; u < total; u += gridDim.x) {
        int lo = 0, hi = njobs;  // last j with prefix[j] <= u
        while (hi - lo > 1) { int mid = (lo + hi) >> 1; if (sm_prefix[mid] <= u) lo = mid; else hi = mid; }
        const int j = lo;
        const Job jb = jobs[j];
        const uint32_t unit = u - sm_prefix[j];
        if (jb.kind == JOB_SCAN) {
            if (loaded_job != j) {
                __syncthreads();
                for (uint32_t i = threadIdx.x; i < ld; i += blockDim.x) sm_normal[i] = jb.normal[NORMAL_HDR + i];
                nh0 = jb.normal[0];
                loaded_job = j;
                __syncthreads();
            }
            scan_unit(jb, unit, items, ih0, d, ld, metric, sm_normal, nh0, &sm_count);
        } else {
            partition_block(jb.rows, jb.flags, jb.dst, unit * PART_UNIT, jb.len, jb.unit_left[unit * (PART_UNIT / SCAN_UNIT)], jb.total_left, sm_w);
        }
    }
}

// work_kernel for contexts that hold the 8-bit planes of the items: scan jobs of more than min_units units are cut into items of
// PLANES_CHUNK units and go through scan_claim_planes; everything else is work_kernel's. Shared memory: the normal, the normal in
// the planes' lane order (planes_perm_floats(ld) floats) and the prefix table.
__global__ void __launch_bounds__(WORK_THREADS, 2)
work_kernel_shadow(const Job* __restrict__ jobs, int njobs, const float* __restrict__ items, const PlaneRows planes, const float* __restrict__ ih0,
                   uint32_t d, uint32_t ld, int metric, uint32_t min_units, unsigned long long* stats) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    float* sm_normal = reinterpret_cast<float*>(smem_raw);
    float* sm_perm = sm_normal + ld;
    uint32_t* sm_prefix = reinterpret_cast<uint32_t*>(sm_perm + planes_perm_floats(ld));
    __shared__ uint32_t sm_count;
    __shared__ uint32_t sm_w[16];
    __shared__ uint32_t sm_list[SCAN_UNIT * PLANES_CHUNK], sm_list2[SCAN_UNIT * PLANES_CHUNK];
    __shared__ uint32_t sm_cnt[PLANES_CHUNK + 2];
    __shared__ double sm_l1[WORK_THREADS / 32];
    auto via_shadow = [&](const Job& jb) { return jb.kind == JOB_SCAN && jb.margins == nullptr && (jb.len + SCAN_UNIT - 1) / SCAN_UNIT > min_units; };
    for (int j = threadIdx.x; j < njobs; j += blockDim.x) {
        const Job jb = jobs[j];
        const uint32_t units = (jb.len + SCAN_UNIT - 1) / SCAN_UNIT;
        sm_prefix[j] = jb.kind == JOB_SCAN ? (via_shadow(jb) ? (units + PLANES_CHUNK - 1) / PLANES_CHUNK : units) : (jb.kind == JOB_PARTITION ? (jb.len + PART_UNIT - 1) / PART_UNIT : 0u);
    }
    __syncthreads();
    if (threadIdx.x < 32) {
        const int per = (njobs + 31) / 32;
        const int b = threadIdx.x * per, e = min(b + per, njobs);
        uint32_t loc = 0;
        for (int i = b; i < e; ++i) loc += sm_prefix[i];
        uint32_t inc = loc;
        for (int o = 1; o < 32; o <<= 1) { uint32_t y = __shfl_up_sync(0xffffffffu, inc, o); if ((int)threadIdx.x >= o) inc += y; }
        uint32_t run = inc - loc;
        for (int i = b; i < e; ++i) { uint32_t x = sm_prefix[i]; sm_prefix[i] = run; run += x; }
        if (threadIdx.x == 31) sm_prefix[njobs] = inc;
    }
    __syncthreads();
    const uint32_t total = sm_prefix[njobs];
    int loaded_job = -1;
    float nh0 = 0.f;
    float2 wf = make_float2(0.f, 0.f);
    for (uint32_t u = blockIdx.x; u < total; u += gridDim.x) {
        int lo = 0, hi = njobs;  // last j with prefix[j] <= u
        while (hi - lo > 1) { int mid = (lo + hi) >> 1; if (sm_prefix[mid] <= u) lo = mid; else hi = mid; }
        const int j = lo;
        const Job jb = jobs[j];
        const uint32_t item = u - sm_prefix[j];
        if (jb.kind == JOB_SCAN) {
            if (loaded_job != j) {
                __syncthreads();
                double l1 = 0.0;
                for (uint32_t i = threadIdx.x; i < ld; i += blockDim.x) {
                    const float v = jb.normal[NORMAL_HDR + i];
                    sm_normal[i] = v;
                    sm_perm[planes_perm_index(i)] = v;
                    l1 += (double)fabsf(v);
                }
                l1 = warp_sum_f64(l1);
                if ((threadIdx.x & 31) == 0) sm_l1[threadIdx.x >> 5] = l1;
                nh0 = jb.normal[0];
                loaded_job = j;
                __syncthreads();
                wf = planes_job_factors(sm_l1, d);
            }
            if (via_shadow(jb)) {
                const uint32_t units = (jb.len + SCAN_UNIT - 1) / SCAN_UNIT;
                scan_claim_planes(jb, item * PLANES_CHUNK, min(units, (item + 1u) * PLANES_CHUNK), items, planes, ih0, d, ld, metric, sm_normal, sm_perm, nh0, wf.x, wf.y,
                                  sm_list, sm_list2, sm_cnt, stats);
            } else scan_unit<true>(jb, item, items, ih0, d, ld, metric, sm_normal, nh0, &sm_count);
        } else {
            partition_block(jb.rows, jb.flags, jb.dst, item * PART_UNIT, jb.len, jb.unit_left[item * (PART_UNIT / SCAN_UNIT)], jb.total_left, sm_w);
        }
    }
}

// ---- per-item norms ---------------------------------------------------------------------
// out[r] = sqrt(dot(v_r, v_r)) in the reference's order; optional atomic max over rows
// (f32::max semantics: NaN ignored; norms are >= 0 so the uint order equals the float order).
__global__ void __launch_bounds__(256) norms_kernel(const float* __restrict__ items, uint64_t n, uint32_t d, uint32_t ld, float* __restrict__ out, uint32_t* max_bits) {
    const int lane = threadIdx.x & 31;
    uint64_t warp_global = (uint64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    uint64_t nwarps = (uint64_t)gridDim.x * (blockDim.x >> 5);
    for (uint64_t r0 = warp_global * 4; r0 < n; r0 += nwarps * 4) {
        float res;
        if (d >= 32) {
            const int g8 = lane & 7, grp = lane >> 3;
            uint64_t r = r0 + grp;
            bool v = r < n;
            const float4* A = reinterpret_cast<const float4*>(items + (size_t)(v ? r : 0) * ld);
            float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
            const int nch = d >> 5;
#pragma unroll 4
            for (int c = 0; c < nch; ++c) {
                float4 x = ldg_stream(A + c * 8 + g8);
                acc.x = fmaf(x.x, x.x, acc.x); acc.y = fmaf(x.y, x.y, acc.y); acc.z = fmaf(x.z, x.z, acc.z); acc.w = fmaf(x.w, x.w, acc.w);
            }
            float dt = group8_hsum(acc);
            const float* row = items + (size_t)(v ? r : 0) * ld;
            for (uint32_t i = nch * 32; i < d; ++i) dt = __fadd_rn(dt, __fmul_rn(row[i], row[i]));
            res = __fsqrt_rn(dt);
            if (v && g8 == 0) {
                out[r] = res;
                if (max_bits && res == res) atomicMax(max_bits, __float_as_uint(res));
            }
        } else {
            if (lane < 4) {
                uint64_t r = r0 + lane;
                if (r < n) {
                    const float* row = items + (size_t)r * ld;
                    res = __fsqrt_rn(exact_thread<false>(row, row, (int)d));
                    out[r] = res;
                    if (max_bits && res == res) atomicMax(max_bits, __float_as_uint(res));
                }
            }
        }
    }
}

// DotProduct::preprocess pass 2 — dot_product.rs:146-160
__global__ void dot_header_kernel(const float* __restrict__ norms, uint64_t n, const uint32_t* max_bits, float* __restrict__ extra_dim, float* __restrict__ norm_hdr) {
    uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    float max_norm = __uint_as_float(*max_bits);
    float node_norm = norms[i];
    float mm = __fmul_rn(max_norm, max_norm);
    float diff = __fsub_rn(mm, __fmul_rn(node_norm, node_norm));
    norm_hdr[i] = mm;
    extra_dim[i] = __fsqrt_rn(diff);
}

// ---- re-rank distances --------------------------------------------------------------------
// One warp handles 4 candidates at a time (8 lanes each). Query vectors in global memory
// (read through L1/L2; nq*ld floats). keys[q][i] = ordered_key(dist) << 32 | position.
__device__ __forceinline__ float built_finish(int metric, float acc, float qh0, float item_h0) {
    if (metric == EUCLIDEAN || metric == MANHATTAN) return acc;      // euclidean.rs:45-47 / manhattan.rs:44-46
    // binary quantized: sum (a - b)^2 = 4 popcount(a ^ b) (euclidean.rs:117-124), sum |a - b| = 2 popcount (manhattan.rs:113-120)
    if (metric == BQ_EUCLIDEAN || metric == BQ_MANHATTAN) return acc;
    if (metric == BQ_COSINE) {                                       // binary_quantized_cosine.rs:51-65: no clamp, `!= 0.0`
        const float pnqn = __fmul_rn(qh0, item_h0);
        return pnqn != 0.0f ? __fdiv_rn(__fsub_rn(1.0f, __fdiv_rn(acc, pnqn)), 2.0f) : 0.0f;
    }
    if (metric == DOT_PRODUCT) return -acc;                          // dot_product.rs:52-56
    float pnqn = __fmul_rn(qh0, item_h0);                            // cosine.rs:43-59
    if (pnqn > 1.1920928955078125e-07f) {
        float c = __fdiv_rn(acc, pnqn);
        if (c < -1.0f) c = -1.0f;
        if (c > 1.0f) c = 1.0f;
        return __fdiv_rn(__fsub_rn(1.0f, c), 2.0f);
    }
    return 0.0f;
}

__global__ void __launch_bounds__(256)
distance_kernel(const float* __restrict__ items, const float* __restrict__ ih0, uint32_t d, uint32_t ld, int metric,
                const float* __restrict__ queries, const uint32_t* __restrict__ qrows, const float* __restrict__ qh0, uint32_t nq,
                const uint32_t* __restrict__ rows, const uint64_t* __restrict__ seg_beg, const uint64_t* __restrict__ seg_end,
                float* __restrict__ dists, unsigned long long* __restrict__ keys) {
    const uint32_t q = blockIdx.y;
    const uint64_t beg = seg_beg[q], end = seg_end[q];
    const float* qv = qrows ? items + (size_t)qrows[q] * ld : queries + (size_t)q * ld;
    const float qhdr = qh0 ? qh0[q] : 0.f;
    const int lane = threadIdx.x & 31;
    const uint64_t warp_global = (uint64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    const uint64_t nwarps = (uint64_t)gridDim.x * (blockDim.x >> 5);
    if (metric == MANHATTAN || metric == BQ_MANHATTAN) {
        // strictly sequential scalar sum of |p - q| per candidate (manhattan.rs:44-46): one lane per row
        for (uint64_t p0 = beg + warp_global * 32; p0 < end; p0 += nwarps * 32) {
            uint64_t p = p0 + lane;
            if (p < end) {
                const float* row = items + (size_t)rows[p] * ld;
                float s = 0.0f;
                for (uint32_t i = 0; i < d; ++i) s = __fadd_rn(s, fabsf(__fsub_rn(qv[i], row[i])));
                dists[p] = s;
                keys[p] = ((unsigned long long)ordered_key(s) << 32) | (unsigned long long)(uint32_t)(p - beg);
            }
        }
        return;
    }
    for (uint64_t p0 = beg + warp_global * 4; p0 < end; p0 += nwarps * 4) {
        float res;
        uint64_t p;
        bool v, writer;
        uint32_t r = 0;
        if (d >= 32) {
            const int g8 = lane & 7, grp = lane >> 3;
            p = p0 + grp;
            v = p < end;
            writer = g8 == 0;
            if (v) r = rows[p];
            const float4* A = reinterpret_cast<const float4*>(items + (size_t)r * ld);
            const float4* Q = reinterpret_cast<const float4*>(qv);
            float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
            const int nch = d >> 5;
            if (metric == EUCLIDEAN || metric == BQ_EUCLIDEAN) {
#pragma unroll 4
                for (int c = 0; c < nch; ++c) {
                    float4 x = __ldg(Q + c * 8 + g8);
                    float4 y = ldg_stream(A + c * 8 + g8);
                    float t0 = __fsub_rn(x.x, y.x), t1 = __fsub_rn(x.y, y.y), t2 = __fsub_rn(x.z, y.z), t3 = __fsub_rn(x.w, y.w);
                    acc.x = fmaf(t0, t0, acc.x); acc.y = fmaf(t1, t1, acc.y); acc.z = fmaf(t2, t2, acc.z); acc.w = fmaf(t3, t3, acc.w);
                }
            } else {
#pragma unroll 4
                for (int c = 0; c < nch; ++c) {
                    float4 x = __ldg(Q + c * 8 + g8);
                    float4 y = ldg_stream(A + c * 8 + g8);
                    acc.x = fmaf(x.x, y.x, acc.x); acc.y = fmaf(x.y, y.y, acc.y); acc.z = fmaf(x.z, y.z, acc.z); acc.w = fmaf(x.w, y.w, acc.w);
                }
            }
            res = group8_hsum(acc);
            const float* row = items + (size_t)r * ld;
            for (uint32_t i = nch * 32; i < d; ++i) {
                if (metric == EUCLIDEAN || metric == BQ_EUCLIDEAN) { float t = __fsub_rn(qv[i], row[i]); res = __fadd_rn(res, __fmul_rn(t, t)); }
                else res = __fadd_rn(res, __fmul_rn(qv[i], row[i]));
            }
        } else {
            p = p0 + lane;
            v = lane < 4 && p < end;
            writer = true;
            res = 0.f;
            if (v) {
                r = rows[p];
                const float* row = items + (size_t)r * ld;
                res = (metric == EUCLIDEAN || metric == BQ_EUCLIDEAN) ? exact_thread<true>(qv, row, (int)d) : exact_thread<false>(qv, row, (int)d);
            }
        }
        if (v && writer) {
            float dist = built_finish(metric, res, qhdr, (metric == COSINE || metric == BQ_COSINE) ? ih0[r] : 0.f);
            dists[p] = dist;
            keys[p] = ((unsigned long long)ordered_key(dist) << 32) | (unsigned long long)(uint32_t)(p - beg);
        }
    }
}

// ---- top-k ----------------------------------------------------------------------------------
// One CTA per query. Streaming selection: the CAP-key shared buffer keeps the best k so far in
// [0,k) (sorted) and is refilled with up to CAP-k new keys that beat the current k-th key, then
// bitonic-sorted. Equivalent to sort-ascending-take-k on (OrderedFloat, id) — which is what
// median_based_top_k returns (src/reader.rs:607-640, tests/reader.rs:283-299).
constexpr int TOPK_CAP = 4096;
constexpr int TOPK_THREADS = 256;

__device__ __forceinline__ void bitonic_sort_shared(unsigned long long* buf, int n /* power of two */) {
    for (int size = 2; size <= n; size <<= 1) {
        for (int stride = size >> 1; stride > 0; stride >>= 1) {
            __syncthreads();
            for (int t = threadIdx.x; t < (n >> 1); t += blockDim.x) {
                int i = 2 * t - (t & (stride - 1));
                int j = i + stride;
                bool up = ((i & size) == 0);
                unsigned long long a = buf[i], b = buf[j];
                if ((a > b) == up) { buf[i] = b; buf[j] = a; }
            }
        }
    }
    __syncthreads();
}

__device__ __forceinline__ float normalized_distance_dev(int metric, float dist) {
    if (metric == EUCLIDEAN) return __fsqrt_rn(dist);  // mod.rs:59-61
    if (metric == COSINE || is_bq(metric)) return dist;   // cosine.rs:61-63; binary quantized: see bq_normalize_kernel
    if (metric == DOT_PRODUCT) return -dist;           // dot_product.rs:81-83
    return (dist != dist) ? 0.0f : (dist > 0.0f ? dist : 0.0f);  // manhattan.rs:48-50 (f32::max)
}

__global__ void __launch_bounds__(TOPK_THREADS)
topk_kernel(const unsigned long long* __restrict__ keys, const float* __restrict__ dists, const uint32_t* __restrict__ rows,
            const uint64_t* __restrict__ seg_beg, const uint64_t* __restrict__ seg_end, uint32_t k, int metric,
            uint32_t* __restrict__ out_rows, float* __restrict__ out_dist, uint32_t* __restrict__ out_len) {
    __shared__ unsigned long long buf[TOPK_CAP];
    __shared__ uint32_t fill;
    const uint32_t q = blockIdx.x;
    const uint64_t beg = seg_beg[q], end = seg_end[q];
    const uint64_t n = end - beg;
    const uint32_t kk = (uint32_t)(n < (uint64_t)k ? n : (uint64_t)k);
    for (int i = threadIdx.x; i < TOPK_CAP; i += blockDim.x) buf[i] = ~0ull;
    unsigned long long threshold = ~0ull;  // keys >= threshold cannot enter the top k any more
    uint64_t pos = 0;
    bool have = false;
    while (pos < n) {  // host guarantees k <= TOPK_CAP / 2, so every round makes progress
        const uint32_t base = have ? kk : 0u;
        const uint64_t room = (uint64_t)(TOPK_CAP - base);
        const uint32_t take = (uint32_t)(n - pos < room ? n - pos : room);
        __syncthreads();
        if (threadIdx.x == 0) fill = base;
        __syncthreads();
        for (uint32_t i = threadIdx.x; i < take; i += blockDim.x) {
            unsigned long long key = keys[beg + pos + i];
            if (key < threshold) { uint32_t s = atomicAdd(&fill, 1u); buf[s] = key; }
        }
        pos += take;
        __syncthreads();
        const uint32_t f = fill;
        int m = 2;
        while ((uint32_t)m < f) m <<= 1;
        for (int i = (int)f + threadIdx.x; i < m; i += blockDim.x) buf[i] = ~0ull;
        bitonic_sort_shared(buf, m);
        have = true;
        threshold = (f >= kk && kk > 0) ? buf[kk - 1] : ~0ull;  // keys are unique, so `<` loses nothing
    }
    __syncthreads();
    if (threadIdx.x == 0) out_len[q] = kk;
    for (uint32_t i = threadIdx.x; i < kk; i += blockDim.x) {
        uint32_t p = (uint32_t)(buf[i] & 0xffffffffull);
        out_rows[(size_t)q * k + i] = rows[beg + p];
        out_dist[(size_t)q * k + i] = normalized_distance_dev(metric, dists[beg + p]);
    }
}

// k beyond the streaming buffer (k > TOPK_CAP / 2; the reference has no limit, reader.rs:396-399): the keys of every
// query were sorted completely (CUB segmented sort); this kernel takes the first min(k, n) of each segment.
__global__ void __launch_bounds__(256)
take_sorted_kernel(const unsigned long long* __restrict__ sorted_keys, const float* __restrict__ dists, const uint32_t* __restrict__ rows,
                   const uint64_t* __restrict__ seg_beg, const uint64_t* __restrict__ seg_end, uint32_t k, int metric,
                   uint32_t* __restrict__ out_rows, float* __restrict__ out_dist, uint32_t* __restrict__ out_len) {
    const uint32_t q = blockIdx.x;
    const uint64_t beg = seg_beg[q], n = seg_end[q] - beg;
    const uint32_t kk = (uint32_t)(n < (uint64_t)k ? n : (uint64_t)k);
    if (threadIdx.x == 0) out_len[q] = kk;
    for (uint32_t i = threadIdx.x; i < kk; i += blockDim.x) {
        const uint32_t p = (uint32_t)(sorted_keys[beg + i] & 0xffffffffull);
        out_rows[(size_t)q * k + i] = rows[beg + p];
        out_dist[(size_t)q * k + i] = normalized_distance_dev(metric, dists[beg + p]);
    }
}

// binary-quantized distances divide by the index' dimensions (reader.rs:398 -> binary_quantized_euclidean.rs:56-58: d / dims;
// _manhattan.rs:56-58: d.max(0.0) / dims; _cosine: unchanged): a second pass over the (few) results of the top-k kernels
__global__ void bq_normalize_kernel(float* __restrict__ dist, uint64_t n, int metric, float dims) {
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    float d = dist[i];
    if (metric == BQ_MANHATTAN) d = (d != d) ? 0.0f : (d > 0.0f ? d : 0.0f);
    if (metric != BQ_COSINE) dist[i] = __fdiv_rn(d, dims);
}

// dense f32 rows (n x d_in) -> the padded +-1 layout (n x ld, the first dpad = 64 * ceil(d_in / 64) columns +-1, the rest 0):
// BinaryQuantized::from_slice + ::iter (binary_quantized.rs:80-92, :276-289) — bit = is_sign_positive
__global__ void bq_sign_rows_kernel(const float* __restrict__ src, float* __restrict__ dst, uint64_t n, uint32_t d_in, uint32_t dpad, uint32_t ld) {
    const uint64_t total = n * ld;
    for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (uint64_t)gridDim.x * blockDim.x) {
        const uint64_t r = i / ld;
        const uint32_t c = (uint32_t)(i - r * ld);
        float v = 0.f;
        if (c < d_in) v = (__float_as_uint(src[r * d_in + c]) >> 31) ? -1.0f : 1.0f;
        else if (c < dpad) v = -1.0f;
        dst[i] = v;
    }
}

// ---- synthetic matrix -------------------------------------------------------------------------
// out[(i, j)] = gen::<f32>() number (row0+i)*d + j of StdRng::from_seed(key) minus centre; one
// thread per ChaCha block (16 words).
__global__ void synth_kernel(const uint32_t* __restrict__ key8, uint32_t d, uint64_t row0, uint64_t rows, float centre, float* __restrict__ out) {
    uint32_t key[8];
    for (int i = 0; i < 8; ++i) key[i] = key8[i];
    const uint64_t w0 = row0 * d, w1 = (row0 + rows) * d;
    const uint64_t b0 = w0 >> 4, b1 = (w1 + 15) >> 4;
    for (uint64_t b = b0 + (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; b < b1; b += (uint64_t)gridDim.x * blockDim.x) {
        uint32_t blk[16];
        chacha12_block(key, b, blk);
#pragma unroll
        for (int k = 0; k < 16; ++k) {
            uint64_t w = (b << 4) + k;
            if (w >= w0 && w < w1) out[w - w0] = __fsub_rn(__fmul_rn((float)(blk[k] >> 8), 5.9604644775390625e-08f), centre);
        }
    }
}

// copy a dense n x d matrix into the padded n x ld layout (zero fill)
__global__ void pad_rows_kernel(const float* __restrict__ src, float* __restrict__ dst, uint64_t n, uint32_t d, uint32_t ld) {
    uint64_t total = n * ld;
    for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (uint64_t)gridDim.x * blockDim.x) {
        uint64_t r = i / ld;
        uint32_t c = (uint32_t)(i - r * ld);
        dst[i] = c < d ? src[r * d + c] : 0.f;
    }
}

__global__ void fill_u32_kernel(uint32_t* p, uint64_t n, uint32_t v) {
    for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x) p[i] = v;
}
__global__ void iota_u32_kernel(uint32_t* p, uint64_t n) {
    for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x) p[i] = (uint32_t)i;
}

}  // namespace ab
