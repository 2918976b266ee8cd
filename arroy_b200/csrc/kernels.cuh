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
#include "select.cuh"

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
// sign of dot + c), with |dot - sum n_i x_i| <= gamma_R sum |n_i x_i| + wa, gamma_R <= 1.001 d u in any summation order, and
// |x_i| <= M <= 127.001 s. wa is the part of the reference's error that is not relative: a product n_i x_i (a multiply or the
// multiply of an FMA) whose result is subnormal loses up to 2^-150 absolutely, and rows far below 1 make every product do so
// (rows below 2^-73 also leave the reference's split normal unnormalized, so n is as tiny as x). An add whose result is
// subnormal is exact, and each of the d losses is carried through at most d later roundings (a factor of at most 1 + gamma_R,
// with d gamma_R <= 5 for d <= PLANES_MAX_D), so wa = (d + 32) 2^-150 covers them all, exact in f64. Both stage tests below
// add wa to their bound; at ordinary magnitudes it is far below one ulp of the bound and changes no decision.
//  stage 1, hi plane only (d bytes per row): T1 = 254 sum h_i a_i + sum h_i b_i, an exact integer (each int32 sum is at most
//    127 * 127 * 8192 < 2^31 in magnitude for d <= PLANES_MAX_D), so s sigma T1 / 254 = s sum h_i n1_i and
//    |dot - s sum h_i n1_i| <= s (E1 N1 + 127 D1 + 127.001 gamma_R N1).
//    The row is certain when |p + c| > s w1 + wa in f64, p = fl(fl(T1 s) k1), k1 = fl(sigma / 254), w1 = (N1 (E1 + 127.001
//    gamma_R) + 127 D1) (1 + 2^-20) rounded up: the factor 1 + 2^-20 covers the relative errors of p (3 roundings on
//    |p| <= 254 s N1) and of the test (2^-53 each; s w1 and wa are both positive, so the sum's rounding is relative too).
//  stage 2, the rows stage 1 left (lo plane only: stage 1 kept their hi-plane sums): y_i = 254 h_i + l_i (|y_i| <= 32385),
//    T2 = sum y_i (254^2 a_i + 254 b_i + c_i) from the six int32 sums of h, l times a, b, c (|T2| <= 2.2e15 < 2^53: exact in f64),
//    so s sigma T2 / 254^3 = (s / 254) sum y_i n2_i, and with A = 254 sum |h_i| U_i + sum |l_i| U_i (sum |n_i| |y_i| <= sigma A / 2):
//    |dot - (s/254) sum y_i n2_i| <= s E2 N1 + (s/254) 32385 D2 + gamma_R ((s/254) sigma A / 2 + s E2 N1) + wa
//                                  = (s/254) (254 E2 (1 + gamma_R) N1 + 32385 D2 + gamma_R sigma A / 2) + wa.
//    The row is certain when |p2 + c| > s (w2 + rel2 A) + wa in f64, p2 = fl(fl(T2 s) k2), k2 = fl(sigma / 254^3),
//    w2 = (254 E2 (1 + gamma_R) N1 + 32385 D2) (1 + 2^-20) / 254, rel2 = gamma_R sigma / 508 (1 + 2^-20), both rounded up (the
//    factor covers p2's 3 roundings on |p2| <= 255 s N1 and the test's own).
//  stage 3: every other row — near the hyperplane, zero, non-finite — is scored from the f32 row in the reference's summation
//    order (scan_unit's arithmetic). Flags and unit counts are the exact scan's.
// A normal with a non-finite element gets NaN factors: no row is certain.
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

// The encoder of host-placed items (arroy_b200.cu stage_rows_pipeline): the f32 rows live in mapped host memory, and each chunk
// of them crosses PCIe once, into a device bounce buffer, where this kernel reads it. It writes the chunk's planes and scales
// with planes_encode_kernel's arithmetic (the same bytes) and, when `norms` is given, sqrt(dot(v, v)) of every row in
// norms_kernel's order (d >= 32: the caller only places rows of 64 <= d <= PLANES_MAX_D on the host). One 8-lane group per row,
// four rows per warp; every lane runs every iteration, so the group shuffles see a full warp.
__global__ void __launch_bounds__(256) planes_encode_chunk_kernel(const float* __restrict__ rows_f32, uint64_t n, uint32_t d, uint32_t ld,
                                                                  int8_t* __restrict__ hi, int8_t* __restrict__ lo, float* __restrict__ scale,
                                                                  float* __restrict__ norms) {
    const unsigned full = 0xffffffffu;
    const int lane = threadIdx.x & 31, g8 = lane & 7, grp = lane >> 3;
    const uint32_t n4 = ld >> 2;   // a multiple of 8
    const uint64_t nwarps = (uint64_t)gridDim.x * (blockDim.x >> 5);
    for (uint64_t r0 = ((uint64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5)) * 4; r0 < n; r0 += nwarps * 4) {
        const uint64_t r = r0 + grp;
        const bool v = r < n;
        const float4* row = reinterpret_cast<const float4*>(rows_f32 + (v ? r : 0) * ld);
        uint32_t mb = 0;
        for (uint32_t k = g8; k < n4; k += 8) {
            const float4 x = row[k];
            mb = max(max(mb, __float_as_uint(fabsf(x.x))), max(__float_as_uint(fabsf(x.y)), max(__float_as_uint(fabsf(x.z)), __float_as_uint(fabsf(x.w)))));
        }
#pragma unroll
        for (int o = 1; o < 8; o <<= 1) mb = max(mb, __shfl_xor_sync(full, mb, o));
        const float M = __uint_as_float(mb);
        float s = __fdiv_rn(M, 127.0f);
        const bool ok = s >= 1.17549435e-38f && s <= 3.40282347e+38f;
        if (!ok && mb != 0u && mb != 0x7f800000u) s = __int_as_float(0x7fffffff);
        if (v) {
            uint32_t* H = reinterpret_cast<uint32_t*>(hi + r * ld);
            uint32_t* L = reinterpret_cast<uint32_t*>(lo + r * ld);
            for (uint32_t k = g8; k < n4; k += 8) {
                const float4 x4 = row[k];
                const float x[4] = {x4.x, x4.y, x4.z, x4.w};
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
            if (g8 == 0) scale[r] = s;
        }
        if (norms != nullptr) {   // (uniform over the grid)
            float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
            const int nch = d >> 5;
#pragma unroll 4
            for (int c = 0; c < nch; ++c) {
                const float4 x = row[c * 8 + g8];
                acc.x = fmaf(x.x, x.x, acc.x); acc.y = fmaf(x.y, x.y, acc.y); acc.z = fmaf(x.z, x.z, acc.z); acc.w = fmaf(x.w, x.w, acc.w);
            }
            float dt = group8_hsum(acc);
            const float* rf = reinterpret_cast<const float*>(row);
            for (uint32_t i = nch * 32; i < d; ++i) dt = __fadd_rn(dt, __fmul_rn(rf[i], rf[i]));
            if (v && g8 == 0) norms[r] = __fsqrt_rn(dt);
        }
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
    double wa;                   // both stages: the absolute term (d + 32) 2^-150 of products that underflow
};
constexpr uint32_t PLANES_LIMBS = 4;   // ld bytes each

__device__ __forceinline__ double prefilter_c(int metric, float nh0, float item_h0) {
    if (metric == COSINE) return 0.0;
    if (metric == DOT_PRODUCT) return (double)__fmul_rn(nh0, item_h0);
    return (double)nh0;
}

// Starts `bytes` (a multiple of 16) at p, 16-byte aligned, on their way from HBM into L2; takes no register for the data.
__device__ __forceinline__ void prefetch_l2(const void* p, uint32_t bytes) {
    // (no "memory" clobber: it writes nothing the program reads, so no load or store has to stay on either side of it)
    asm volatile("cp.async.bulk.prefetch.L2.global [%0], %1;" :: "l"(__cvta_generic_to_global(p)), "r"(bytes));
}

// A row stage 1 of scan_claim_planes leaves to stage 2: its position and its hi-plane sums over the whole row,
// mh = 254^3 sum h a + 254^2 sum h b + 254 sum h c (|mh| < 2^51) and hu = sum |h| U (< 2^32).
struct __align__(16) PlanesLeft {
    long long mh;
    uint32_t hu, pos;
};

// What scan_claim_planes keeps of the rows of its claim (position base + i at index i): the ids, fetched once in its prologue
// (zeros past the claim's end), and for the rows stage 1 leaves (the first sm_cnt[PLANES_CHUNK] entries of left) their scales
// and headers.
constexpr uint32_t PLANES_CLAIM_ROWS = SCAN_UNIT * PLANES_CHUNK;
struct PlanesClaimRows {
    uint32_t rid[PLANES_CLAIM_ROWS];   // row ids
    float scale[PLANES_CLAIM_ROWS];    // the plane scales of the rows stage 1 leaves
    float ih0[PLANES_CLAIM_ROWS];      // DotProduct: their h0 (the other metrics: 0)
    PlanesLeft left[PLANES_CLAIM_ROWS];
};

// scan units [u0, u1) (at most PLANES_CHUNK) of a job. sm_list2: 64 * PLANES_CHUNK positions (the rows stage 2 left); sm_cnt:
// PLANES_CHUNK + 2 counters. limbs, pn: the job's normal as planes_job_factors left it. stats (optional): [0] rows through the
// pre-filter, [1] of them re-scored from the f32 row, [2] of them that went through stage 2.
// Every read of a plane row is a device read (the planes never live in host memory), so their L2 prefetches are safe.
__device__ __forceinline__ void scan_claim_planes(const Job& jb, uint32_t u0, uint32_t u1, const float* __restrict__ items, const PlaneRows pl,
                                                  const float* __restrict__ ih0, uint32_t d, uint32_t ld, int metric, const float* sm_normal, const uint8_t* limbs,
                                                  const PlanesNormal* pn, float nh0, uint32_t* sm_list2, uint32_t* sm_cnt,
                                                  PlanesClaimRows& cr, unsigned long long* stats) {
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, g8 = lane & 7, grp = lane >> 3;
    const uint32_t base = u0 * SCAN_UNIT, end = min(jb.len, u1 * SCAN_UNIT);
    // ---- prologue: one round for the claim's row ids; the hi rows of the first 128 positions start towards L2 as soon as
    // their ids are known (the rows' scales and headers are loaded in stage 1, beside its hi-plane loads) ----
    if (tid <= (int)PLANES_CHUNK + 1) sm_cnt[tid] = 0;
    for (uint32_t i = tid; i < PLANES_CLAIM_ROWS; i += blockDim.x) {
        const bool v = base + i < end;
        const uint32_t r = v ? (jb.rows ? __ldcg(jb.rows + base + i) : base + i) : 0u;
        if (v && i < 128u) prefetch_l2(pl.hi + (size_t)r * ld, ld);
        cr.rid[i] = r;
    }
    __syncthreads();
    const uint32_t nq = ld >> 4;                       // 16-byte words per plane row
    const int nsteps = (int)((nq + 7) >> 3);
    const uint4* LA = reinterpret_cast<const uint4*>(limbs);
    const uint4* LB = LA + nq;
    const uint4* LC = LB + nq;
    const uint4* LU = LC + nq;
    // ---- stage 1: the hi plane of every row, and with it every hi-plane sum stage 2 needs (kept for the rows it leaves); the
    // next block's hi rows are prefetched into L2 while this block's are read ----
    for (uint32_t pbase = base; pbase < end; pbase += 128) {
        if (tid < 128 && pbase + 128u + tid < end) prefetch_l2(pl.hi + (size_t)cr.rid[pbase + 128u - base + tid] * ld, ld);
        const uint4* S[4];
#pragma unroll
        for (int r = 0; r < 4; ++r) S[r] = reinterpret_cast<const uint4*>(pl.hi + (size_t)cr.rid[pbase + warp * 16 + grp * 4 + r - base] * ld) + g8;
        // the row this lane decides once its group's sums are reduced (below): row 2 b2 + b1 of the group's four, for the lane
        // bits b2 b1 b0 of g8; its scale and header are in flight while the hi rows stream
        const uint32_t pos = pbase + warp * 16 + grp * 4 + (uint32_t)(g8 >> 1), rid = cr.rid[pos - base];
        const bool valid = pos < end;
        const float s = valid ? __ldg(pl.scale + rid) : 0.f;
        const float h0 = (valid && metric == DOT_PRODUCT) ? ih0[rid] : 0.f;
        int sa[4], sb[4], hc[4];
        uint32_t hu[4];
#pragma unroll
        for (int r = 0; r < 4; ++r) { sa[r] = 0; sb[r] = 0; hc[r] = 0; hu[r] = 0; }
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
                const uint4 z = make_uint4(0u, 0u, 0u, 0u);
                const uint4 la = q < nq ? LA[q] : z, lb = q < nq ? LB[q] : z, lc = q < nq ? LC[q] : z, lu = q < nq ? LU[q] : z;
#pragma unroll
                for (int r = 0; r < 4; ++r) {
                    sa[r] = dp16(v[sidx][r], la, sa[r]); sb[r] = dp16(v[sidx][r], lb, sb[r]); hc[r] = dp16(v[sidx][r], lc, hc[r]);
                    hu[r] = dp16u(abs_bytes(v[sidx][r]), lu, hu[r]);
                }
            }
        }
        // reduce the 16 sums (4 rows x sa, sb, hc, hu) over the group by halving: lanes b2 = 0 keep rows 0, 1 and b2 = 1 rows 2, 3
        // (xor 4), then b1 picks one of the two (xor 2), and the lane pair b0 = 0, 1 sums its row's four (xor 1): 16 shuffles
        int x[2][4];
#pragma unroll
        for (int j = 0; j < 2; ++j) {
            const int lo4[4] = {sa[j], sb[j], hc[j], (int)hu[j]}, hi4[4] = {sa[j + 2], sb[j + 2], hc[j + 2], (int)hu[j + 2]};
#pragma unroll
            for (int k = 0; k < 4; ++k) {
                const bool up = (g8 & 4) != 0;
                x[j][k] = (up ? hi4[k] : lo4[k]) + __shfl_xor_sync(0xffffffffu, up ? lo4[k] : hi4[k], 4);
            }
        }
        int y[4];
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            const bool up = (g8 & 2) != 0;
            y[k] = (up ? x[1][k] : x[0][k]) + __shfl_xor_sync(0xffffffffu, up ? x[0][k] : x[1][k], 2);
            y[k] += __shfl_xor_sync(0xffffffffu, y[k], 1);
        }
        const long long t1 = 254ll * y[0] + y[1];
        const double mt = __dadd_rn(__dmul_rn(__dmul_rn((double)t1, (double)s), pn->k1), prefilter_c(metric, nh0, h0));
        const bool certain = fabs(mt) > __dadd_rn(__dmul_rn((double)s, pn->w1), pn->wa);     // false for NaN / Inf scales and NaN factors
        const bool leader = (g8 & 1) == 0 && valid;
        const int side = mt > 0.0 ? 1 : 0;
        if (leader && certain) jb.flags[pos] = (uint8_t)side;
        if (leader && !certain) {   // stage 2 reads this row's lo plane from L2, and its scale and header from cr
            PlanesLeft e;
            e.mh = 64516ll * t1 + 254ll * y[2]; e.hu = (uint32_t)y[3]; e.pos = pos;
            cr.left[atomicAdd(&sm_cnt[PLANES_CHUNK], 1u)] = e;
            cr.scale[pos - base] = s;
            cr.ih0[pos - base] = h0;
            prefetch_l2(pl.lo + (size_t)rid * ld, ld);
        }
        const unsigned lefts = __ballot_sync(0xffffffffu, leader && certain && side == 0);
        // the four groups of a warp hold positions of the same unit (16 consecutive positions per warp)
        if (lane == 0 && lefts) atomicAdd(&sm_cnt[(pbase + warp * 16 - base) / SCAN_UNIT], (uint32_t)__popc(lefts));
    }
    __syncthreads();
    // ---- stage 2: the lo plane of the rows stage 1 left, one 8-lane group per row; six words per lane in flight (the one
    // round of a row of ld <= 768) ----
    const uint32_t n1 = sm_cnt[PLANES_CHUNK];
    for (uint32_t it = 0; it * 32u < n1; ++it) {
        const uint32_t idx = it * 32u + (uint32_t)(warp * 4 + grp);
        const bool act = idx < n1;
        PlanesLeft e;
        if (act) e = cr.left[idx];
        else { e.mh = 0; e.hu = 0u; e.pos = base; }
        const uint32_t p = e.pos;
        const uint32_t r = cr.rid[p - base];
        const uint4* Lr = reinterpret_cast<const uint4*>(pl.lo + (size_t)r * ld) + g8;
        int la = 0, lb = 0, lc = 0;
        uint32_t lu = 0;
        for (int c0 = 0; c0 < nsteps; c0 += 6) {
            uint4 vl[6];
#pragma unroll
            for (int sidx = 0; sidx < 6; ++sidx) {
                const uint32_t q = (uint32_t)(c0 + sidx) * 8u + (uint32_t)g8;
                vl[sidx] = q < nq ? ldg_stream_u4(Lr + (c0 + sidx) * 8) : make_uint4(0u, 0u, 0u, 0u);
            }
#pragma unroll
            for (int sidx = 0; sidx < 6; ++sidx) {
                const uint32_t q = (uint32_t)(c0 + sidx) * 8u + (uint32_t)g8;
                if (q < nq) {   // the row's words past nq were loaded as zeros
                    const uint4 na = LA[q], nb = LB[q], nc = LC[q], nu = LU[q];
                    la = dp16(vl[sidx], na, la); lb = dp16(vl[sidx], nb, lb); lc = dp16(vl[sidx], nc, lc);
                    lu = dp16u(abs_bytes(vl[sidx]), nu, lu);
                }
            }
        }
#pragma unroll
        for (int o = 1; o < 8; o <<= 1) {
            la += __shfl_xor_sync(0xffffffffu, la, o); lb += __shfl_xor_sync(0xffffffffu, lb, o);
            lc += __shfl_xor_sync(0xffffffffu, lc, o); lu += __shfl_xor_sync(0xffffffffu, lu, o);
        }
        // T2 and A: integers below 2^53 (the lo-plane group sums fit int32 / uint32 like the hi-plane ones), so the doubles are exact
        const double m = (double)(e.mh + 64516ll * la + 254ll * lb + lc);
        const double a = (double)(254ull * e.hu + lu);
        const float s = cr.scale[p - base];
        const double mt = __dadd_rn(__dmul_rn(__dmul_rn(m, (double)s), pn->k2), prefilter_c(metric, nh0, cr.ih0[p - base]));
        const bool certain = fabs(mt) > __dadd_rn(__dmul_rn((double)s, __dadd_rn(pn->w2, __dmul_rn(pn->rel2, a))), pn->wa);
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
        const uint32_t r = cr.rid[p - base];
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
        const int sa = side_of(margin_finish(metric, da, nh0, cr.ih0[p - base]));
        if (act && g8 == 0) { jb.flags[p] = (uint8_t)sa; if (sa == 0) atomicAdd(&sm_cnt[(p - base) / SCAN_UNIT], 1u); }
    }
    __syncthreads();
    if (jb.unit_left != nullptr && tid < (int)(u1 - u0)) jb.unit_left[u0 + tid] = sm_cnt[tid];   // (side_multi's jobs count nothing)
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
        f.wa = (double)(d + 32u) * 0x1p-150;
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

// ---- binary-quantized items: bit strings ----------------------------------------------------------------------------------
// A binary-quantized item row is the reference's bit string (binary_quantized.rs:80-92): bit i of u64 word w set when element
// 64 w + i is positive, i.e. bit j of u32 word k = element 32 k + j. `d` (the bit count) is a multiple of 64; rows are padded with
// zero words to 16 bytes. Every element is +-1, so each sum the reference forms over two such vectors is an exact integer in any
// summation order: dot = d - 2 popcount(a ^ b), sum (a - b)^2 = 4 popcount, sum |a - b| = 2 popcount.
__host__ __device__ constexpr uint32_t bq_row_u4(uint32_t d) { return (d + 127u) / 128u; }   // 16-byte words per row

// A +-1 normal (f32, d elements) as a bit string in shared memory: 4 bq_row_u4(d) u32 words, bit = is_sign_positive, padding 0.
// Every thread of the CTA calls it; the caller puts a barrier between this and the first read.
__device__ __forceinline__ void bq_pack_normal(const float* __restrict__ v, uint32_t d, uint32_t* sm_bits) {
    const int lane = threadIdx.x & 31;
    const uint32_t nw = 4u * bq_row_u4(d);
    for (uint32_t w = threadIdx.x >> 5; w < nw; w += blockDim.x >> 5) {
        const uint32_t i = w * 32u + (uint32_t)lane;
        const unsigned b = __ballot_sync(0xffffffffu, i < d && !(__float_as_uint(v[i]) >> 31));
        if (lane == 0) sm_bits[w] = b;
    }
}

// scan_unit for bit-string rows: four lanes per row (a CTA of 4 SCAN_UNIT threads covers the unit's positions). The margin is
// margin_finish of the exact dot, as scan_unit forms it from its f32 sum of the same +-1 products; flags, margins and the unit's
// Left count are scan_unit's.
static_assert(WORK_THREADS == 4 * SCAN_UNIT, "bq_scan_unit: four lanes per position of a scan unit");
__device__ __forceinline__ void bq_scan_unit(const Job& jb, uint32_t unit, const uint4* __restrict__ items, uint32_t d, int metric,
                                             const uint4* sm_bits, float nh0, uint32_t* sm_count) {
    const uint32_t rq = bq_row_u4(d);
    const int lane = threadIdx.x & 31, sub = threadIdx.x & 3;
    if (threadIdx.x == 0) *sm_count = 0;
    __syncthreads();
    const uint32_t p = unit * SCAN_UNIT + (threadIdx.x >> 2);
    const bool v = p < jb.len;
    const uint32_t r = v ? (jb.rows ? __ldcg(jb.rows + p) : p) : 0u;
    const uint4* x = items + (size_t)r * rq;
    int pc = 0;
    for (uint32_t c = (uint32_t)sub; c < rq; c += 4) {
        const uint4 a = ldg_stream_u4(x + c), b = sm_bits[c];
        pc += __popc(a.x ^ b.x) + __popc(a.y ^ b.y) + __popc(a.z ^ b.z) + __popc(a.w ^ b.w);
    }
    pc += __shfl_xor_sync(0xffffffffu, pc, 1);
    pc += __shfl_xor_sync(0xffffffffu, pc, 2);
    const float m = margin_finish(metric, (float)((int)d - 2 * pc), nh0, 0.f);
    const int s = side_of(m);
    const bool leader = sub == 0 && v;
    if (leader) { if (jb.flags) jb.flags[p] = (uint8_t)s; if (jb.margins) jb.margins[p] = m; }
    const unsigned l = __ballot_sync(0xffffffffu, leader && s == 0);
    if (lane == 0 && l) atomicAdd(sm_count, (uint32_t)__popc(l));
    __syncthreads();
    if (threadIdx.x == 0 && jb.unit_left) jb.unit_left[unit] = *sm_count;
}

// Persistent-style grid: every CTA strides over the units of all posted jobs.
// Dynamic shared memory: ld floats (normal) + (njobs + 1) uint32 (unit prefix). BQ: `items` holds bit-string rows and the
// normal's first ld floats of shared memory hold its bit string (bq_scan_unit).
template <bool BQ>
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
                if constexpr (BQ) bq_pack_normal(jb.normal + NORMAL_HDR, d, reinterpret_cast<uint32_t*>(sm_normal));
                else for (uint32_t i = threadIdx.x; i < ld; i += blockDim.x) sm_normal[i] = jb.normal[NORMAL_HDR + i];
                nh0 = jb.normal[0];
                loaded_job = j;
                __syncthreads();
            }
            if constexpr (BQ) bq_scan_unit(jb, unit, reinterpret_cast<const uint4*>(items), d, metric, reinterpret_cast<const uint4*>(sm_normal), nh0, &sm_count);
            else scan_unit(jb, unit, items, ih0, d, ld, metric, sm_normal, nh0, &sm_count);
        } else {
            partition_block(jb.rows, jb.flags, jb.dst, unit * PART_UNIT, jb.len, jb.unit_left[unit * (PART_UNIT / SCAN_UNIT)], jb.total_left, sm_w);
        }
    }
}

// work_kernel for contexts that hold the 8-bit planes of the items: scan jobs of more than min_units units are cut into items of
// PLANES_CHUNK units and go through scan_claim_planes; everything else is work_kernel's. Shared memory: the normal, its limbs
// (PLANES_LIMBS * ld bytes) and the prefix table.
__global__ void __launch_bounds__(WORK_THREADS, 2)
work_kernel_planes(const Job* __restrict__ jobs, int njobs, const float* __restrict__ items, const PlaneRows planes, const float* __restrict__ ih0,
                   uint32_t d, uint32_t ld, int metric, uint32_t min_units, unsigned long long* stats) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    float* sm_normal = reinterpret_cast<float*>(smem_raw);
    uint8_t* sm_limbs = reinterpret_cast<uint8_t*>(sm_normal + ld);
    uint32_t* sm_prefix = reinterpret_cast<uint32_t*>(sm_limbs + PLANES_LIMBS * ld);
    __shared__ uint32_t sm_count;
    __shared__ uint32_t sm_w[16];
    __shared__ uint32_t sm_list2[SCAN_UNIT * PLANES_CHUNK];
    __shared__ uint32_t sm_cnt[PLANES_CHUNK + 2];
    __shared__ PlanesClaimRows sm_cr;
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
                                  sm_list2, sm_cnt, sm_cr, stats);
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

// The raw sum of built_distance (Euclidean: the sum of squared differences, else the dot product) of the query q and one row,
// in the reference's summation order, by the 8 lanes g8 of a group. d >= 32: every lane of the warp takes part (the AVX order
// over 16-byte loads, group8_hsum, then the separately rounded tail). d < 32: lane g8 == 0 alone, when v (exact_thread). The
// result is valid in lane g8 == 0. Q_LDG: q is read through the read-only cache (global memory), else with plain loads.
template <bool Q_LDG>
__device__ __forceinline__ float row_sum8(bool euclid, const float* q, const float* row, uint32_t d, int g8, bool v) {
    if (d < 32) return (g8 == 0 && v) ? (euclid ? exact_thread<true>(q, row, (int)d) : exact_thread<false>(q, row, (int)d)) : 0.f;
    const float4* A = reinterpret_cast<const float4*>(row);
    const float4* Q = reinterpret_cast<const float4*>(q);
    float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
    const int nch = (int)(d >> 5);
    if (euclid) {
#pragma unroll 4
        for (int c = 0; c < nch; ++c) {
            const float4 x = Q_LDG ? __ldg(Q + c * 8 + g8) : Q[c * 8 + g8], y = ldg_stream(A + c * 8 + g8);
            const float t0 = __fsub_rn(x.x, y.x), t1 = __fsub_rn(x.y, y.y), t2 = __fsub_rn(x.z, y.z), t3 = __fsub_rn(x.w, y.w);
            acc.x = fmaf(t0, t0, acc.x); acc.y = fmaf(t1, t1, acc.y); acc.z = fmaf(t2, t2, acc.z); acc.w = fmaf(t3, t3, acc.w);
        }
    } else {
#pragma unroll 4
        for (int c = 0; c < nch; ++c) {
            const float4 x = Q_LDG ? __ldg(Q + c * 8 + g8) : Q[c * 8 + g8], y = ldg_stream(A + c * 8 + g8);
            acc.x = fmaf(x.x, y.x, acc.x); acc.y = fmaf(x.y, y.y, acc.y); acc.z = fmaf(x.z, y.z, acc.z); acc.w = fmaf(x.w, y.w, acc.w);
        }
    }
    float res = group8_hsum(acc);
    for (uint32_t i = (uint32_t)nch * 32u; i < d; ++i) {
        if (euclid) { const float t = __fsub_rn(q[i], row[i]); res = __fadd_rn(res, __fmul_rn(t, t)); }
        else res = __fadd_rn(res, __fmul_rn(q[i], row[i]));
    }
    return res;
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
    const bool euclid = metric == EUCLIDEAN || metric == BQ_EUCLIDEAN;
    const int g8 = lane & 7, grp = lane >> 3;
    for (uint64_t p0 = beg + warp_global * 4; p0 < end; p0 += nwarps * 4) {   // one row per 8-lane group
        const uint64_t p = p0 + grp;
        const bool v = p < end;
        const uint32_t r = v ? rows[p] : 0u;
        const float res = row_sum8<true>(euclid, qv, items + (size_t)r * ld, d, g8, v);
        if (v && g8 == 0) {
            const float dist = built_finish(metric, res, qhdr, (metric == COSINE || metric == BQ_COSINE) ? ih0[r] : 0.f);
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
// The query's keys: DENSE, formed here from its row of a dense distance matrix (dists + q * nc) over one candidate list `rows`
// that all queries share, key = ordered_key(dist) << 32 | position; else distance_kernel's keys[seg_beg[q] .. seg_end[q]) over
// the query's own candidates rows + seg_beg[q].
constexpr int TOPK_CAP = 4096;
constexpr int TOPK_THREADS = 256;

__device__ __forceinline__ float normalized_distance_dev(int metric, float dist) {
    if (metric == EUCLIDEAN) return __fsqrt_rn(dist);  // mod.rs:59-61
    if (metric == COSINE || is_bq(metric)) return dist;   // cosine.rs:61-63; binary quantized: see bq_normalize_kernel
    if (metric == DOT_PRODUCT) return -dist;           // dot_product.rs:81-83
    return (dist != dist) ? 0.0f : (dist > 0.0f ? dist : 0.0f);  // manhattan.rs:48-50 (f32::max)
}

template <bool DENSE>
__global__ void __launch_bounds__(TOPK_THREADS)
topk_kernel(const unsigned long long* __restrict__ keys, const float* __restrict__ dists, const uint32_t* __restrict__ rows,
            const uint64_t* __restrict__ seg_beg, const uint64_t* __restrict__ seg_end, uint32_t nc, uint32_t k, int metric,
            uint32_t* __restrict__ out_rows, float* __restrict__ out_dist, uint32_t* __restrict__ out_len) {
    __shared__ unsigned long long buf[TOPK_CAP];
    __shared__ uint32_t fill;
    const uint32_t q = blockIdx.x;
    const uint64_t beg = DENSE ? (uint64_t)q * nc : seg_beg[q];
    const uint64_t n = DENSE ? (uint64_t)nc : seg_end[q] - beg;
    const uint32_t* qrows = DENSE ? rows : rows + beg;
    const uint32_t kk = (uint32_t)(n < (uint64_t)k ? n : (uint64_t)k);
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
            const uint32_t j = (uint32_t)pos + i;
            const unsigned long long key = DENSE ? ((unsigned long long)ordered_key(dists[beg + j]) << 32) | (unsigned long long)j : keys[beg + j];
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
        out_rows[(size_t)q * k + i] = qrows[p];
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

// dense f32 rows (n x d_in, row pitch `pitch` floats) -> bit-string rows of w32 u32 words: BinaryQuantized::from_slice
// (binary_quantized.rs:80-92) — bit = is_sign_positive, so +0.0 -> 1, -0.0 -> 0 and a NaN's sign bit decides; elements from d_in
// on are 0 (the padding of the bit string and of the row). One warp per word.
__global__ void bq_pack_rows_kernel(const float* __restrict__ src, uint64_t pitch, uint32_t* __restrict__ dst, uint64_t n, uint32_t d_in, uint32_t w32) {
    const int lane = threadIdx.x & 31;
    const uint64_t total = n * w32, nw = (uint64_t)gridDim.x * (blockDim.x >> 5);
    for (uint64_t w = (uint64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); w < total; w += nw) {
        const uint64_t r = w / w32;
        const uint32_t c = (uint32_t)(w - r * w32) * 32u + (uint32_t)lane;
        const unsigned b = __ballot_sync(0xffffffffu, c < d_in && !(__float_as_uint(src[r * pitch + c]) >> 31));
        if (lane == 0) dst[w] = b;
    }
}

// queries by item of a binary-quantized index: their bit strings (rows of w32 words) copied to bits, and expanded to the +-1
// f32 vectors (ld floats each) that the forest walks take
__global__ void bq_query_rows_kernel(const uint32_t* __restrict__ items, uint32_t w32, const uint32_t* __restrict__ rows, uint32_t m, uint32_t ld,
                                     float* __restrict__ vecs, uint32_t* __restrict__ bits) {
    const uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
    for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < (uint64_t)m * ld; i += stride) {
        const uint64_t q = i / ld;
        const uint32_t c = (uint32_t)(i - q * ld);
        vecs[i] = ((items[(size_t)rows[q] * w32 + (c >> 5)] >> (c & 31u)) & 1u) ? 1.0f : -1.0f;
    }
    for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < (uint64_t)m * w32; i += stride) {
        const uint64_t q = i / w32;
        bits[i] = items[(size_t)rows[q] * w32 + (i - q * w32)];
    }
}

// distance_kernel for bit-string rows: query q's bit string is qbits[q] (bq_row_u4(d) 16-byte words), four lanes per candidate.
// D::built_distance of binary_quantized_{euclidean,cosine,manhattan}.rs from the exact popcount sums, as distance_kernel forms it
// from its f32 sums of the same +-1 terms; keys as distance_kernel's.
__global__ void __launch_bounds__(256)
bq_distance_kernel(const uint4* __restrict__ items, const float* __restrict__ ih0, uint32_t d, int metric, const uint4* __restrict__ qbits,
                   const float* __restrict__ qh0, const uint32_t* __restrict__ rows, const uint64_t* __restrict__ seg_beg,
                   const uint64_t* __restrict__ seg_end, float* __restrict__ dists, unsigned long long* __restrict__ keys) {
    const uint32_t q = blockIdx.y, rq = bq_row_u4(d);
    const uint64_t beg = seg_beg[q], end = seg_end[q];
    const uint4* qv = qbits + (size_t)q * rq;
    const float qhdr = qh0 ? qh0[q] : 0.f;
    const int sub = threadIdx.x & 3;
    const uint64_t slot = (uint64_t)blockIdx.x * (blockDim.x >> 2) + (threadIdx.x >> 2), nslots = (uint64_t)gridDim.x * (blockDim.x >> 2);
    for (uint64_t p0 = beg; p0 < end; p0 += nslots) {   // the same trip count on every lane: the shuffles below need all 32
        const uint64_t p = p0 + slot;
        const bool v = p < end;
        const uint32_t r = v ? rows[p] : 0u;
        const uint4* x = items + (size_t)r * rq;
        int pc = 0;
        for (uint32_t c = (uint32_t)sub; c < rq; c += 4) {
            const uint4 a = ldg_stream_u4(x + c), b = __ldg(qv + c);
            pc += __popc(a.x ^ b.x) + __popc(a.y ^ b.y) + __popc(a.z ^ b.z) + __popc(a.w ^ b.w);
        }
        pc += __shfl_xor_sync(0xffffffffu, pc, 1);
        pc += __shfl_xor_sync(0xffffffffu, pc, 2);
        if (v && sub == 0) {
            const float dist = metric == BQ_EUCLIDEAN ? (float)(4 * pc)
                             : metric == BQ_MANHATTAN ? (float)(2 * pc)
                             : built_finish(BQ_COSINE, (float)((int)d - 2 * pc), qhdr, ih0[r]);
            dists[p] = dist;
            keys[p] = ((unsigned long long)ordered_key(dist) << 32) | (unsigned long long)(uint32_t)(p - beg);
        }
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
