// tcgemm.cuh — S = Q . C^T on the Hopper tensor cores (wgmma, TF32 inputs, FP32 accumulation in
// registers), hand-written for sm_90a. It is the first stage of the shared-candidate re-rank
// (xrerank.cuh, "tensor-core pre-filter"): S only has to *bound* the reference's distance of every
// (query, candidate) pair, the survivors are re-scored in the reference's exact order.
//
//   Q : m  x K  fp32, row-major, pitch ld (K = ld, padding is zero)      -> wgmma operand A, K-major
//   C : nc x K  fp32, row-major, pitch ld (item rows, in place)          -> wgmma operand B, K-major
//   S : m  x nc fp32, row-major, pitch lds
//
// Structure (one persistent CTA per SM, three warpgroups):
//   warpgroup 0     TMA producer (one thread): cp.async.bulk.tensor 2D, 128B-swizzled boxes of 32
//                   floats of K (128 x 32 of Q, 256 x 32 of C) into a 4-stage shared-memory ring,
//                   mbarrier tx-counts
//   warpgroups 1-2  consumers: 64 queries each, wgmma.mma_async m64n256k8 TF32 (four per stage) into a
//                   64 x 256 FP32 register accumulator; a stage is released as soon as the wgmma group
//                   that read it has retired (wait_group 1 keeps one group in flight), then the
//                   distance estimate of the tile is computed and stored straight from the registers
//                   while the producer already fills the ring for the next tile
// Tiles are ordered candidates-major so that the CTAs running at the same time share the same
// candidate rows in L2 and C streams from HBM once.
#pragma once
#include <cuda.h>
#include <cooperative_groups.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include <algorithm>

namespace ab {

constexpr int TG_BM = 128;     // queries per tile   (two consumer warpgroups x wgmma M = 64)
constexpr int TG_BN = 256;      // candidates per tile (wgmma N)
constexpr int TG_BK = 32;       // floats of K per stage = one 128-byte swizzle span
constexpr int TG_UK = 8;        // K of one wgmma .tf32
constexpr int TG_STAGES = 4;
constexpr int TG_THREADS = 3 * 128;
constexpr uint32_t TG_A_BYTES = TG_BM * TG_BK * 4;
constexpr uint32_t TG_B_BYTES = TG_BN * TG_BK * 4;
constexpr uint32_t TG_STAGE_BYTES = TG_A_BYTES + TG_B_BYTES;
constexpr size_t TG_SMEM = (size_t)TG_STAGES * TG_STAGE_BYTES + 1024 /* 1024-byte alignment */ + 256 /* barriers */;

__device__ __forceinline__ uint32_t tg_smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void tg_mbar_init(uint32_t bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory");
}
__device__ __forceinline__ void tg_mbar_expect_tx(uint32_t bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
// arrive on the barrier at this shared-memory offset in CTA `cta` of the cluster (the own CTA included)
__device__ __forceinline__ void tg_mbar_arrive_cluster(uint32_t bar, uint32_t cta) {
    asm volatile("{\n\t.reg .b32 ra;\n\tmapa.shared::cluster.u32 ra, %0, %1;\n\tmbarrier.arrive.release.cluster.shared::cluster.b64 _, [ra];\n\t}"
                 ::"r"(bar), "r"(cta) : "memory");
}
// Spin on a phase parity. A protocol bug must not hang the GPU: trap after ~2 s.
__device__ __forceinline__ void tg_mbar_wait(uint32_t bar, uint32_t parity) {
    uint32_t done = 0;
    long long t0 = 0;
    for (uint32_t spin = 0;; ++spin) {
        asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}"
                     : "=r"(done) : "r"(bar), "r"(parity) : "memory");
        if (done) break;
        if ((spin & 0xffffu) == 0xffffu) {
            long long now = clock64();
            if (t0 == 0) t0 = now;
            else if (now - t0 > 4000000000ll) __trap();
        }
    }
}
__device__ __forceinline__ void tg_tma_load_2d(uint32_t dst, const CUtensorMap* map, uint32_t bar, int c0, int c1) {
    asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
                 ::"r"(dst), "l"(map), "r"(bar), "r"(c0), "r"(c1) : "memory");
}
// the same load delivered to the same shared-memory offset (and mbarrier) of every CTA in `mask`
__device__ __forceinline__ void tg_tma_load_2d_mc(uint32_t dst, const CUtensorMap* map, uint32_t bar, int c0, int c1, uint16_t mask) {
    asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes.multicast::cluster [%0], [%1, {%3, %4}], [%2], %5;"
                 ::"r"(dst), "l"(map), "r"(bar), "r"(c0), "r"(c1), "h"(mask) : "memory");
}

// wgmma shared-memory matrix descriptor: K-major, 128-byte swizzle, 8-row groups 1024 bytes apart
__device__ __forceinline__ uint64_t tg_smem_desc(uint32_t addr) {
    uint64_t d = 0;
    d |= (uint64_t)((addr & 0x3ffffu) >> 4);       // start address, 16-byte units
    d |= (uint64_t)1 << 16;                         // leading byte offset (unused for swizzled K-major)
    d |= (uint64_t)(1024 >> 4) << 32;               // stride byte offset: next 8-row group
    d |= (uint64_t)1 << 62;                         // SWIZZLE_128B
    return d;
}

// d (64 x 256 FP32, wgmma accumulator fragment) (+)= A (64 x 8) . B (256 x 8)^T, both TF32 from shared memory
__device__ __forceinline__ void tg_wgmma_tf32(float* d, uint64_t desc_a, uint64_t desc_b, uint32_t accumulate) {
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %130, 0;\n\t"
                 "wgmma.mma_async.sync.aligned.m64n256k8.f32.tf32.tf32 {"
                 "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
                 "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
                 "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "
                 "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63, "
                 "%64, %65, %66, %67, %68, %69, %70, %71, %72, %73, %74, %75, %76, %77, %78, %79, "
                 "%80, %81, %82, %83, %84, %85, %86, %87, %88, %89, %90, %91, %92, %93, %94, %95, "
                 "%96, %97, %98, %99, %100, %101, %102, %103, %104, %105, %106, %107, %108, %109, %110, %111, "
                 "%112, %113, %114, %115, %116, %117, %118, %119, %120, %121, %122, %123, %124, %125, %126, %127}, "
                 "%128, %129, p, 1, 1;\n\t}"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
                   "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
                   "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
                   "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
                   "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),
                   "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),
                   "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]),
                   "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63]),
                   "+f"(d[64]), "+f"(d[65]), "+f"(d[66]), "+f"(d[67]), "+f"(d[68]), "+f"(d[69]), "+f"(d[70]), "+f"(d[71]),
                   "+f"(d[72]), "+f"(d[73]), "+f"(d[74]), "+f"(d[75]), "+f"(d[76]), "+f"(d[77]), "+f"(d[78]), "+f"(d[79]),
                   "+f"(d[80]), "+f"(d[81]), "+f"(d[82]), "+f"(d[83]), "+f"(d[84]), "+f"(d[85]), "+f"(d[86]), "+f"(d[87]),
                   "+f"(d[88]), "+f"(d[89]), "+f"(d[90]), "+f"(d[91]), "+f"(d[92]), "+f"(d[93]), "+f"(d[94]), "+f"(d[95]),
                   "+f"(d[96]), "+f"(d[97]), "+f"(d[98]), "+f"(d[99]), "+f"(d[100]), "+f"(d[101]), "+f"(d[102]), "+f"(d[103]),
                   "+f"(d[104]), "+f"(d[105]), "+f"(d[106]), "+f"(d[107]), "+f"(d[108]), "+f"(d[109]), "+f"(d[110]), "+f"(d[111]),
                   "+f"(d[112]), "+f"(d[113]), "+f"(d[114]), "+f"(d[115]), "+f"(d[116]), "+f"(d[117]), "+f"(d[118]), "+f"(d[119]),
                   "+f"(d[120]), "+f"(d[121]), "+f"(d[122]), "+f"(d[123]), "+f"(d[124]), "+f"(d[125]), "+f"(d[126]), "+f"(d[127])
                 : "l"(desc_a), "l"(desc_b), "r"(accumulate) : "memory");
}
__device__ __forceinline__ void tg_wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void tg_wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N> __device__ __forceinline__ void tg_wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }

// What the epilogue writes for pair (q, c) from the raw contraction s = Q[q] . C[c]:
//   TG_RAW     s
//   TG_NEG     -s                                             (DotProduct built_distance, dot_product.rs:52-56)
//   TG_EUCLID  (qa[q] + ca[c]) - 2 s                          (qa, ca = squared norms; euclidean.rs:45-47)
//   TG_COSINE  qb[q] * cb[c] > f32::EPSILON ? (1 - clamp(s * qa[q] * ca[c])) / 2 : 0     (cosine.rs:43-59;
//              qa, ca = reciprocal header norms, qb, cb = header norms)
// i.e. an FP32 *estimate* of the reference's built_distance; xrerank.cuh bounds its error.
enum { TG_RAW = 0, TG_NEG = 1, TG_EUCLID = 2, TG_COSINE = 3 };

struct TgEpilogue {
    int mode;
    const float* qa; const float* qb;   // per query (row)
    const float* ca; const float* cb;   // per candidate (column)
};

__device__ __forceinline__ float tg_finish(int mode, float s, float qa, float qb, float ca, float cb) {
    if (mode == TG_RAW) return s;
    if (mode == TG_NEG) return -s;
    if (mode == TG_EUCLID) return __fsub_rn(__fadd_rn(qa, ca), __fmul_rn(2.0f, s));
    const float pnqn = __fmul_rn(qb, cb);
    if (pnqn > 1.1920928955078125e-07f) {
        float c = __fmul_rn(s, __fmul_rn(qa, ca));
        c = c < -1.0f ? -1.0f : (c > 1.0f ? 1.0f : c);   // NaN stays NaN
        return __fmul_rn(0.5f, __fsub_rn(1.0f, c));
    }
    return pnqn == pnqn ? 0.0f : pnqn;
}

// MC = 1: independent CTAs. MC = 2: clusters of two CTAs that work on the same 256 candidates and two
// neighbouring blocks of 128 queries; each CTA fetches one half of the candidate tile and TMA-multicasts it
// into both CTAs' shared memory, so the operand traffic L2 -> SM per CTA drops from 48 to 32 KB per stage.
// A stage is released to both producers by the consumer warpgroups of both CTAs (remote mbarrier arrivals
// on the `empty` barriers, which therefore count 2 * MC arrivals).
template <int MC>
__global__ void __launch_bounds__(TG_THREADS, 1)
tcgemm_tf32_kernel(const __grid_constant__ CUtensorMap map_q, const __grid_constant__ CUtensorMap map_c,
                   float* __restrict__ S, uint32_t m, uint32_t nc, uint32_t lds, uint32_t nk, TgEpilogue ep) {
    extern __shared__ uint8_t tg_raw[];
    const uint32_t raw = tg_smem_u32(tg_raw);
    const uint32_t base = (raw + 1023u) & ~1023u;                      // swizzle-128B tiles need 1024-byte alignment
    const uint32_t bars = base + TG_STAGES * TG_STAGE_BYTES;           // full[4], empty[4]
    auto full = [&](int s) { return bars + 8u * s; };
    auto empty = [&](int s) { return bars + 8u * (TG_STAGES + s); };

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const uint32_t crank = MC > 1 ? cooperative_groups::this_cluster().block_rank() : 0u;
    const uint32_t num_mb = ((m + TG_BM - 1) / TG_BM + MC - 1) / MC, num_n = (nc + TG_BN - 1) / TG_BN;   // m-blocks per cluster step
    const uint32_t tiles = num_mb * num_n, first = blockIdx.x / MC, stride = gridDim.x / MC;
    auto tile_m0 = [&](uint32_t t) { return ((t % num_mb) * MC + crank) * TG_BM; };   // may lie beyond m: zero rows, nothing stored
    auto tile_n0 = [&](uint32_t t) { return (t / num_mb) * TG_BN; };

    if (threadIdx.x == 0) {
        for (int s = 0; s < TG_STAGES; ++s) { tg_mbar_init(full(s), 1); tg_mbar_init(empty(s), 2 * MC); }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
        asm volatile("prefetch.tensormap [%0];" ::"l"(&map_q) : "memory");
        asm volatile("prefetch.tensormap [%0];" ::"l"(&map_c) : "memory");
    }
    __syncthreads();
    if (MC > 1) cooperative_groups::this_cluster().sync();   // the peer's barriers exist before anything is multicast to them

    if (warp < 4) {
        if (threadIdx.x == 0) {
            int stage = 0; uint32_t phase = 0;
            for (uint32_t t = first; t < tiles; t += stride) {
                const int m0 = (int)tile_m0(t), n0 = (int)tile_n0(t);
                for (uint32_t kb = 0; kb < nk; ++kb) {
                    tg_mbar_wait(empty(stage), phase ^ 1u);
                    tg_mbar_expect_tx(full(stage), TG_STAGE_BYTES);
                    const uint32_t sa = base + stage * TG_STAGE_BYTES, sb = sa + TG_A_BYTES;
                    tg_tma_load_2d(sa, &map_q, full(stage), (int)(kb * TG_BK), m0);
                    if (MC == 1) tg_tma_load_2d(sb, &map_c, full(stage), (int)(kb * TG_BK), n0);
                    else tg_tma_load_2d_mc(sb + crank * (TG_B_BYTES / MC), &map_c, full(stage), (int)(kb * TG_BK), n0 + (int)(crank * (TG_BN / MC)), (uint16_t)((1u << MC) - 1u));
                    if (++stage == TG_STAGES) { stage = 0; phase ^= 1u; }
                }
            }
        }
    } else {
        const uint32_t wg = (uint32_t)(warp >> 2) - 1u;               // consumer warpgroup: rows wg * 64 .. + 63 of the tile
        const uint32_t wr = (uint32_t)(warp & 3) * 16u + (uint32_t)(lane >> 2);   // fragment rows wr and wr + 8
        const uint32_t wc = (uint32_t)(lane & 3) * 2u;                 // fragment columns 8 j + wc, + 1
        auto release = [&](int s) {                                    // one arrival per warpgroup on every CTA's barrier
            if ((threadIdx.x & 127u) == 0)
                for (uint32_t r = 0; r < (uint32_t)MC; ++r) tg_mbar_arrive_cluster(empty(s), r);
        };
        int stage = 0; uint32_t phase = 0;
        float acc[TG_BN / 2];
        for (uint32_t t = first; t < tiles; t += stride) {
            const uint32_t m0 = tile_m0(t), n0 = tile_n0(t);
            int prev = -1;
            for (uint32_t kb = 0; kb < nk; ++kb) {
                tg_mbar_wait(full(stage), phase);                      // TMA has landed this stage
                const uint32_t sa = base + stage * TG_STAGE_BYTES + wg * (TG_A_BYTES / 2), sb = base + stage * TG_STAGE_BYTES + TG_A_BYTES;
                const uint64_t da = tg_smem_desc(sa), db = tg_smem_desc(sb);
                tg_wgmma_fence();
#pragma unroll
                for (int k = 0; k < TG_BK / TG_UK; ++k)                // +32 bytes of K inside the swizzle span per step
                    tg_wgmma_tf32(acc, da + (uint64_t)(k * TG_UK * 4 / 16), db + (uint64_t)(k * TG_UK * 4 / 16), (kb | (uint32_t)k) != 0u);
                tg_wgmma_commit();
                tg_wgmma_wait<1>();                                    // the previous stage's group has retired
                if (prev >= 0) release(prev);
                prev = stage;
                if (++stage == TG_STAGES) { stage = 0; phase ^= 1u; }
            }
            tg_wgmma_wait<0>();
            if (prev >= 0) release(prev);

            const uint32_t r0 = m0 + wg * 64u + wr, r1 = r0 + 8u;
            float qa0 = 0.f, qb0 = 0.f, qa1 = 0.f, qb1 = 0.f;
            if (ep.mode >= TG_EUCLID) {
                if (r0 < m) { qa0 = ep.qa[r0]; if (ep.mode == TG_COSINE) qb0 = ep.qb[r0]; }
                if (r1 < m) { qa1 = ep.qa[r1]; if (ep.mode == TG_COSINE) qb1 = ep.qb[r1]; }
            }
            float* out0 = S + (size_t)r0 * lds;
            float* out1 = S + (size_t)r1 * lds;
#pragma unroll
            for (int j = 0; j < TG_BN / 8; ++j) {
                const uint32_t col = n0 + 8u * (uint32_t)j + wc;
                float ca0 = 0.f, ca1 = 0.f, cb0 = 0.f, cb1 = 0.f;
                if (ep.mode >= TG_EUCLID) {
                    if (col < nc) { ca0 = __ldg(ep.ca + col); if (ep.mode == TG_COSINE) cb0 = __ldg(ep.cb + col); }
                    if (col + 1u < nc) { ca1 = __ldg(ep.ca + col + 1u); if (ep.mode == TG_COSINE) cb1 = __ldg(ep.cb + col + 1u); }
                }
                const float v00 = tg_finish(ep.mode, acc[4 * j + 0], qa0, qb0, ca0, cb0), v01 = tg_finish(ep.mode, acc[4 * j + 1], qa0, qb0, ca1, cb1);
                const float v10 = tg_finish(ep.mode, acc[4 * j + 2], qa1, qb1, ca0, cb0), v11 = tg_finish(ep.mode, acc[4 * j + 3], qa1, qb1, ca1, cb1);
                if (col + 1u < nc) {                                   // col is even and lds % 4 == 0: 8-byte aligned
                    if (r0 < m) *reinterpret_cast<float2*>(out0 + col) = make_float2(v00, v01);
                    if (r1 < m) *reinterpret_cast<float2*>(out1 + col) = make_float2(v10, v11);
                } else if (col < nc) {
                    if (r0 < m) out0[col] = v00;
                    if (r1 < m) out1[col] = v10;
                }
            }
        }
    }
    __syncthreads();
    if (MC > 1) cooperative_groups::this_cluster().sync();   // no CTA leaves while its peer can still multicast or arrive into it
}

// the same epilogue as a separate pass (used after the cuBLAS cross-check engine)
__global__ void tg_finish_kernel(float* __restrict__ S, uint32_t m, uint32_t nc, uint32_t lds, TgEpilogue ep) {
    const uint64_t total = (uint64_t)m * nc;
    for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (uint64_t)gridDim.x * blockDim.x) {
        const uint32_t r = (uint32_t)(i / nc), c = (uint32_t)(i - (uint64_t)r * nc);
        float qa = 0.f, qb = 0.f, ca = 0.f, cb = 0.f;
        if (ep.mode >= TG_EUCLID) { qa = ep.qa[r]; ca = ep.ca[c]; if (ep.mode == TG_COSINE) { qb = ep.qb[r]; cb = ep.cb[c]; } }
        float* p = S + (size_t)r * lds + c;
        *p = tg_finish(ep.mode, *p, qa, qb, ca, cb);
    }
}

// ---- host side ---------------------------------------------------------------------------------
typedef CUresult (*tg_encode_fn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*, const cuuint32_t*,
                                 const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

inline tg_encode_fn tg_encoder() {
    static tg_encode_fn fn = [] {
        void* p = nullptr;
        cudaDriverEntryPointQueryResult q;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) != cudaSuccess || q != cudaDriverEntryPointSuccess) p = nullptr;
        return reinterpret_cast<tg_encode_fn>(p);
    }();
    return fn;
}

// rows x ld fp32 matrix, boxes of 32 floats x box_rows rows, 128-byte swizzle, zero fill outside
inline bool tg_make_map(CUtensorMap* map, const float* ptr, uint64_t rows, uint32_t ld, uint32_t box_rows) {
    tg_encode_fn enc = tg_encoder();
    if (!enc) return false;
    cuuint64_t gdim[2] = {ld, rows};
    cuuint64_t gstride[1] = {(cuuint64_t)ld * 4};
    cuuint32_t box[2] = {(cuuint32_t)TG_BK, box_rows};
    cuuint32_t estr[2] = {1, 1};
    return enc(map, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, const_cast<float*>(ptr), gdim, gstride, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
               CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}

// S[m x nc] (pitch lds, lds % 4 == 0) = Q[m x ld] . C[nc x ld]^T; false if the tensor maps cannot be built
inline bool tcgemm_tf32(const float* Q, uint32_t m, const float* C, uint32_t nc, uint32_t ld, float* S, uint32_t lds, TgEpilogue ep, int sm_count, cudaStream_t stream, int mc = 2) {
    if (mc != 1 && mc != 2) mc = 2;
    CUtensorMap mq, mcand;
    if (!tg_make_map(&mq, Q, m, ld, TG_BM) || !tg_make_map(&mcand, C, nc, ld, TG_BN / mc)) return false;
    static bool configured = false;
    static int max_clusters[3] = {0, 0, 0};   // clusters of 1 / 2 CTAs that can be resident at once (GPCs need not hold an even SM count)
    if (!configured) {
        if (cudaFuncSetAttribute(tcgemm_tf32_kernel<1>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)TG_SMEM) != cudaSuccess) return false;
        if (cudaFuncSetAttribute(tcgemm_tf32_kernel<2>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)TG_SMEM) != cudaSuccess) return false;
        configured = true;
    }
    cudaLaunchConfig_t cfg{};
    cfg.blockDim = dim3(TG_THREADS); cfg.dynamicSmemBytes = TG_SMEM; cfg.stream = stream;
    cudaLaunchAttribute at[1];
    at[0].id = cudaLaunchAttributeClusterDimension; at[0].val.clusterDim.x = (unsigned)mc; at[0].val.clusterDim.y = 1; at[0].val.clusterDim.z = 1;
    cfg.attrs = at; cfg.numAttrs = 1;
    if (max_clusters[mc] == 0) {
        cfg.gridDim = dim3((unsigned)(sm_count / mc * mc));
        int nclu = 0;
        const cudaError_t oe = mc == 1 ? cudaOccupancyMaxActiveClusters(&nclu, tcgemm_tf32_kernel<1>, &cfg) : cudaOccupancyMaxActiveClusters(&nclu, tcgemm_tf32_kernel<2>, &cfg);
        if (oe != cudaSuccess || nclu <= 0) return false;
        max_clusters[mc] = nclu;
    }
    const uint32_t num_mb = ((m + TG_BM - 1) / TG_BM + mc - 1) / mc;
    const uint32_t tiles = num_mb * ((nc + TG_BN - 1) / TG_BN);
    const uint32_t units = (uint32_t)std::min(sm_count / mc, max_clusters[mc]);
    cfg.gridDim = dim3((unsigned)((tiles < units ? tiles : units) * mc));
    const uint32_t nk = ld / TG_BK;
    cudaError_t e = mc == 1 ? cudaLaunchKernelEx(&cfg, tcgemm_tf32_kernel<1>, mq, mcand, S, m, nc, lds, nk, ep)
                            : cudaLaunchKernelEx(&cfg, tcgemm_tf32_kernel<2>, mq, mcand, S, m, nc, lds, nk, ep);
    return e == cudaSuccess;
}

}  // namespace ab
