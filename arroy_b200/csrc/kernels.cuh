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
// The normal is read as integer limbs, so that both stages are exact integer dot products (IDP.4A). Once per job, with sigma the
// least power of two above max_i |n_i| / 127 and t_i = n_i / sigma (exact, |t_i| < 127):
//     a_i = rint(t_i),  b_i = rint(254 (t_i - a_i)),  c_i = rint(254 (254 (t_i - a_i) - b_i)),  U_i = ceil(2 |t_i|)
// (every step exact in f64; |a|, |b|, |c| <= 127, U <= 254), n1_i = sigma (a_i + b_i / 254), n2_i = n1_i + sigma c_i / 254^2,
// |n_i| <= sigma U_i / 2, and D1 >= sum |n_i - n1_i|, D2 >= sum |n_i - n2_i| are summed in f64 and rounded up, as is N1 >= |n|_1.
// The reference's margin is fl(dot + c) (c = the bias / extra-dim term, formed exactly as the reference forms it; fl keeps the
// sign of dot + c), with |dot - sum n_i x_i| <= gamma_R sum |n_i x_i|, gamma_R <= 1.001 d u in any summation order, and
// |x_i| <= M <= 127.001 s.
//  stage 1, hi plane only (d bytes per row): T1 = 254 sum h_i a_i + sum h_i b_i, an exact integer (each int32 sum is at most
//    127 * 127 * 8192 < 2^31 in magnitude for d <= PLANES_MAX_D), so s sigma T1 / 254 = s sum h_i n1_i and
//    |dot - s sum h_i n1_i| <= s (E1 N1 + 127 D1 + 127.001 gamma_R N1).
//    The row is certain when |p + c| > s w1 in f64, p = fl(fl(T1 s) k1), k1 = fl(sigma / 254), w1 = (N1 (E1 + 127.001 gamma_R)
//    + 127 D1) (1 + 2^-20) rounded up: the factor 1 + 2^-20 covers the relative errors of p (3 roundings on |p| <= 254 s N1)
//    and of the test (2^-53 each).
//  stage 2, the rows stage 1 left (both planes; the hi row was just streamed by this CTA): y_i = 254 h_i + l_i (|y_i| <= 32385),
//    T2 = sum y_i (254^2 a_i + 254 b_i + c_i) from the six int32 sums of h, l times a, b, c (|T2| <= 2.2e15 < 2^53: exact in f64),
//    so s sigma T2 / 254^3 = (s / 254) sum y_i n2_i, and with A = 254 sum |h_i| U_i + sum |l_i| U_i (sum |n_i| |y_i| <= sigma A / 2):
//    |dot - (s/254) sum y_i n2_i| <= s E2 N1 + (s/254) 32385 D2 + gamma_R ((s/254) sigma A / 2 + s E2 N1)
//                                  = (s/254) (254 E2 (1 + gamma_R) N1 + 32385 D2 + gamma_R sigma A / 2).
//    The row is certain when |p2 + c| > s (w2 + rel2 A) in f64, p2 = fl(fl(T2 s) k2), k2 = fl(sigma / 254^3),
//    w2 = (254 E2 (1 + gamma_R) N1 + 32385 D2) (1 + 2^-20) / 254, rel2 = gamma_R sigma / 508 (1 + 2^-20), both rounded up (the
//    factor covers p2's 3 roundings on |p2| <= 255 s N1 and the test's own).
//  stage 3: every other row — near the hyperplane, zero, non-finite — is scored from the f32 row in the reference's summation
//    order (scan_unit's arithmetic). Flags and unit counts are the exact scan's.
// A normal with a non-finite element gets NaN factors: no row is certain. The bounds are relative: like any such rule they assume
// that no product n_i x_i underflows.
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
// sum over the 16 bytes of x and y of x_k y_k: signed (planes times a, b, c limbs) and unsigned (|h|, |l| times U)
__device__ __forceinline__ int dp16(const uint4 x, const uint4 y, int acc) {
    acc = __dp4a((int)x.x, (int)y.x, acc); acc = __dp4a((int)x.y, (int)y.y, acc);
    acc = __dp4a((int)x.z, (int)y.z, acc); return __dp4a((int)x.w, (int)y.w, acc);
}
__device__ __forceinline__ uint32_t dp16u(const uint4 x, const uint4 y, uint32_t acc) {
    acc = __dp4a(x.x, y.x, acc); acc = __dp4a(x.y, y.y, acc);
    acc = __dp4a(x.z, y.z, acc); return __dp4a(x.w, y.w, acc);
}
// |b| of every signed byte b of w (the planes hold no -128): b ^ 0x80 = b + 128 as an unsigned byte, its distance to 128
__device__ __forceinline__ uint4 abs_bytes(const uint4 w) {
    return make_uint4(__vabsdiffu4(w.x ^ 0x80808080u, 0x80808080u), __vabsdiffu4(w.y ^ 0x80808080u, 0x80808080u),
                      __vabsdiffu4(w.z ^ 0x80808080u, 0x80808080u), __vabsdiffu4(w.w ^ 0x80808080u, 0x80808080u));
}

// A job's normal as the pre-filter reads it: the limbs a, b, c, U (above) as four ld-byte arrays in shared memory, natural
// element order, and its factors.
struct PlanesNormal {
    double w1, k1;               // stage 1: bound factor, sigma / 254
    double w2, rel2, k2;         // stage 2: bound factors, sigma / 254^3
};
constexpr uint32_t PLANES_LIMBS = 4;   // ld bytes each

__device__ __forceinline__ double prefilter_c(int metric, float nh0, float item_h0) {
    if (metric == COSINE) return 0.0;
    if (metric == DOT_PRODUCT) return (double)__fmul_rn(nh0, item_h0);
    return (double)nh0;
}

// scan units [u0, u1) (at most PLANES_CHUNK) of a job. sm_list, sm_list2: 64 * PLANES_CHUNK positions each (the rows stage 1,
// stage 2 left); sm_cnt: PLANES_CHUNK + 2 counters. limbs, pn: the job's normal as planes_job_factors left it. stats (optional):
// [0] rows through the pre-filter, [1] of them re-scored from the f32 row, [2] of them that went through stage 2.
__device__ __forceinline__ void scan_claim_planes(const Job& jb, uint32_t u0, uint32_t u1, const float* __restrict__ items, const PlaneRows pl,
                                                  const float* __restrict__ ih0, uint32_t d, uint32_t ld, int metric, const float* sm_normal, const uint8_t* limbs,
                                                  const PlanesNormal* pn, float nh0, uint32_t* sm_list, uint32_t* sm_list2, uint32_t* sm_cnt, unsigned long long* stats) {
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, g8 = lane & 7, grp = lane >> 3;
    if (tid <= (int)PLANES_CHUNK + 1) sm_cnt[tid] = 0;
    __syncthreads();
    const uint32_t base = u0 * SCAN_UNIT, end = min(jb.len, u1 * SCAN_UNIT);
    const uint32_t nq = ld >> 4;                       // 16-byte words per plane row
    const int nsteps = (int)((nq + 7) >> 3);
    const uint4* LA = reinterpret_cast<const uint4*>(limbs);
    const uint4* LB = LA + nq;
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
        int sa[4], sb[4];
#pragma unroll
        for (int r = 0; r < 4; ++r) { sa[r] = 0; sb[r] = 0; }
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
                const uint4 la = q < nq ? LA[q] : make_uint4(0u, 0u, 0u, 0u), lb = q < nq ? LB[q] : make_uint4(0u, 0u, 0u, 0u);
#pragma unroll
                for (int r = 0; r < 4; ++r) { sa[r] = dp16(v[sidx][r], la, sa[r]); sb[r] = dp16(v[sidx][r], lb, sb[r]); }
            }
        }
        const double w1 = pn->w1, k1 = pn->k1;
#pragma unroll
        for (int r = 0; r < 4; ++r) {
#pragma unroll
            for (int o = 1; o < 8; o <<= 1) { sa[r] += __shfl_xor_sync(0xffffffffu, sa[r], o); sb[r] += __shfl_xor_sync(0xffffffffu, sb[r], o); }
            const bool valid = pos[r] < end;
            const float s = valid ? __ldg(pl.scale + rid[r]) : 0.f;
            const double t1 = (double)(254ll * sa[r] + sb[r]);
            const double mt = __dadd_rn(__dmul_rn(__dmul_rn(t1, (double)s), k1), prefilter_c(metric, nh0, (metric == DOT_PRODUCT && valid) ? ih0[rid[r]] : 0.f));
            const bool certain = fabs(mt) > __dmul_rn((double)s, w1);      // false for NaN / Inf scales and NaN factors
            const bool leader = g8 == 0 && valid;
            const int side = mt > 0.0 ? 1 : 0;
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
    const uint4* LC = LB + nq;
    const uint4* LU = LC + nq;
    for (uint32_t it = 0; it * 32u < n1; ++it) {
        const uint32_t idx = it * 32u + (uint32_t)(warp * 4 + grp);
        const bool act = idx < n1;
        const uint32_t p = act ? sm_list[idx] : base;
        const uint32_t r = jb.rows ? __ldcg(jb.rows + p) : p;
        const uint4* Hr = reinterpret_cast<const uint4*>(pl.hi + (size_t)r * ld) + g8;
        const uint4* Lr = reinterpret_cast<const uint4*>(pl.lo + (size_t)r * ld) + g8;
        int ha = 0, hb = 0, hc = 0, la = 0, lb = 0, lc = 0;
        uint32_t hu = 0, lu = 0;
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
                if (q < nq) {   // the rows' words past nq were loaded as zeros
                    const uint4 na = LA[q], nb = LB[q], nc = LC[q], nu = LU[q];
                    ha = dp16(vh[sidx], na, ha); hb = dp16(vh[sidx], nb, hb); hc = dp16(vh[sidx], nc, hc);
                    la = dp16(vl[sidx], na, la); lb = dp16(vl[sidx], nb, lb); lc = dp16(vl[sidx], nc, lc);
                    hu = dp16u(abs_bytes(vh[sidx]), nu, hu); lu = dp16u(abs_bytes(vl[sidx]), nu, lu);
                }
            }
        }
        // this lane's share of T2 and A: integers below 2^53, so the doubles and their butterfly are exact
        double m = (double)(16387064ll * ha + 64516ll * (hb + la) + 254ll * (hc + lb) + lc);
        double a = (double)(254ull * hu + lu);
#pragma unroll
        for (int o = 1; o < 8; o <<= 1) { m += __shfl_xor_sync(0xffffffffu, m, o); a += __shfl_xor_sync(0xffffffffu, a, o); }
        const float s = __ldg(pl.scale + r);
        const double mt = __dadd_rn(__dmul_rn(__dmul_rn(m, (double)s), pn->k2), prefilter_c(metric, nh0, (metric == DOT_PRODUCT) ? ih0[r] : 0.f));
        const bool certain = fabs(mt) > __dmul_rn((double)s, __dadd_rn(pn->w2, __dmul_rn(pn->rel2, a)));
        const int side = mt > 0.0 ? 1 : 0;
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

__device__ __forceinline__ double warp_sum_f64(double v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

// Per-warp partials of planes_job_factors (eight warps): the caller's sum of |n_i| and max |n_i| (as bits, NaN above +inf), then
// the limb errors.
struct PlanesScratch { double l1[8], d1[8], d2[8]; uint32_t mx[8]; };

// The pre-filter's view of a job's normal (above). The caller has written sm_normal (ld floats) and sc.l1 / sc.mx, then passed a
// CTA barrier. Writes the limbs and, after one more barrier, pn (thread 0; scan_claim_planes reads it after its first barrier).
__device__ __forceinline__ void planes_job_factors(const float* sm_normal, uint32_t ld, uint32_t d, uint8_t* limbs, PlanesScratch& sc, PlanesNormal* pn) {
    uint32_t mb = 0;
#pragma unroll
    for (int w = 0; w < 8; ++w) mb = max(mb, sc.mx[w]);
    const bool finite = mb < 0x7f800000u;
    int e = 0;                                        // sigma = 2^e > max |n_i| / 127 (f64 rounding is monotone)
    if (finite && mb != 0u) frexp((double)__uint_as_float(mb) / 127.0, &e);
    const double inv = ldexp(1.0, -e);
    double d1 = 0.0, d2 = 0.0;
    for (uint32_t i = threadIdx.x; i < ld; i += blockDim.x) {
        const double t = finite ? (double)sm_normal[i] * inv : 0.0;     // every step exact (at most 40 significant bits)
        const double a = rint(t), r1 = 254.0 * (t - a), b = rint(r1), r2 = 254.0 * (r1 - b), c = rint(r2);
        limbs[i] = (uint8_t)(int)a;
        limbs[ld + i] = (uint8_t)(int)b;
        limbs[2 * ld + i] = (uint8_t)(int)c;
        limbs[3 * ld + i] = (uint8_t)(int)ceil(2.0 * fabs(t));
        d1 += fabs(r1 - b);                           // |n_i - n1_i| = sigma |r1 - b| / 254
        d2 += fabs(r2 - c);                           // |n_i - n2_i| = sigma |r2 - c| / 254^2
    }
    d1 = warp_sum_f64(d1);
    d2 = warp_sum_f64(d2);
    if ((threadIdx.x & 31) == 0) { sc.d1[threadIdx.x >> 5] = d1; sc.d2[threadIdx.x >> 5] = d2; }
    __syncthreads();
    if (threadIdx.x == 0) {
        double n1 = 0.0, s1 = 0.0, s2 = 0.0;
#pragma unroll
        for (int w = 0; w < 8; ++w) { n1 += sc.l1[w]; s1 += sc.d1[w]; s2 += sc.d2[w]; }
        const double g = 1.0 + 0x1p-30, slack = 1.0 + 0x1p-20, u = 0x1p-24;   // g: the f64 sums' own rounding (< 8192 * 2^-53)
        // sigma / q rounded up as sigma times 1 / q rounded up (sigma is a power of two: that product is exact)
        const double sigma = ldexp(1.0, e), r254 = 0x1.0204081020409p-8, r64516 = 0x1.040c2050c1c41p-16;
        n1 = __dmul_ru(n1, g);
        const double D1 = __dmul_ru(__dmul_ru(s1, g), sigma * r254), D2 = __dmul_ru(__dmul_ru(s2, g), sigma * r64516);
        const double gR = __dmul_ru(1.001 * u, (double)d);
        const double E1 = 0.5 + 128.0 * u, E2x254 = 0.5 + 32766.0 * u;
        PlanesNormal f;
        f.w1 = __dmul_ru(__dadd_ru(__dmul_ru(n1, __dadd_ru(E1, __dmul_ru(127.001, gR))), __dmul_ru(127.0, D1)), slack);
        f.w2 = __dmul_ru(__dmul_ru(__dadd_ru(__dmul_ru(__dmul_ru(n1, E2x254), __dadd_ru(1.0, gR)), __dmul_ru(32385.0, D2)), slack), r254);
        f.rel2 = __dmul_ru(__dmul_ru(gR, sigma * (0.5 * r254)), slack);
        f.k1 = sigma * (1.0 / 254.0);
        f.k2 = sigma * (1.0 / 16387064.0);
        if (!finite) { f.w1 = __longlong_as_double(0x7ff8000000000000ll); f.w2 = f.w1; }
        *pn = f;
    }
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
// PLANES_CHUNK units and go through scan_claim_planes; everything else is work_kernel's. Shared memory: the normal, its limbs
// (PLANES_LIMBS * ld bytes) and the prefix table.
__global__ void __launch_bounds__(WORK_THREADS, 2)
work_kernel_shadow(const Job* __restrict__ jobs, int njobs, const float* __restrict__ items, const PlaneRows planes, const float* __restrict__ ih0,
                   uint32_t d, uint32_t ld, int metric, uint32_t min_units, unsigned long long* stats) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    float* sm_normal = reinterpret_cast<float*>(smem_raw);
    uint8_t* sm_limbs = reinterpret_cast<uint8_t*>(sm_normal + ld);
    uint32_t* sm_prefix = reinterpret_cast<uint32_t*>(sm_limbs + PLANES_LIMBS * ld);
    __shared__ uint32_t sm_count;
    __shared__ uint32_t sm_w[16];
    __shared__ uint32_t sm_list[SCAN_UNIT * PLANES_CHUNK], sm_list2[SCAN_UNIT * PLANES_CHUNK];
    __shared__ uint32_t sm_cnt[PLANES_CHUNK + 2];
    __shared__ PlanesScratch sm_sc;
    __shared__ PlanesNormal sm_pn;
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
                uint32_t mb = 0;
                for (uint32_t i = threadIdx.x; i < ld; i += blockDim.x) {
                    const float v = jb.normal[NORMAL_HDR + i];
                    sm_normal[i] = v;
                    l1 += (double)fabsf(v);
                    mb = max(mb, __float_as_uint(fabsf(v)));
                }
                l1 = warp_sum_f64(l1);
                mb = __reduce_max_sync(0xffffffffu, mb);
                if ((threadIdx.x & 31) == 0) { sm_sc.l1[threadIdx.x >> 5] = l1; sm_sc.mx[threadIdx.x >> 5] = mb; }
                nh0 = jb.normal[0];
                loaded_job = j;
                __syncthreads();
                if (via_shadow(jb)) planes_job_factors(sm_normal, ld, d, sm_limbs, sm_sc, &sm_pn);
            }
            if (via_shadow(jb)) {
                const uint32_t units = (jb.len + SCAN_UNIT - 1) / SCAN_UNIT;
                scan_claim_planes(jb, item * PLANES_CHUNK, min(units, (item + 1u) * PLANES_CHUNK), items, planes, ih0, d, ld, metric, sm_normal, sm_limbs, &sm_pn, nh0,
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
