// build.cuh — device-resident forest build.
//
// Restates the per-tree task of the reference (src/writer.rs:660-739 -> make_tree_in_file
// :1167-1261) as a device state machine. Each tree owns ONE StdRng stream that is consumed in
// depth-first order (left subtree fully before right, :1235-1254) and the number of draws is
// data dependent (retries :1193-1216, rejection sampling, random fallback :1220-1227), so a
// tree is a sequential chain of "attempts" (create_split + side() scan). Concurrency comes from
// running all trees of a wave side by side: every device step runs
//     control_kernel   one CTA per tree: finish the previous attempt (count Lefts, imbalance
//                      test, partition), advance the DFS, draw the RNG, run two_means
//                      (src/distance/mod.rs:126-171) and create_split, post one scan job;
//     work_kernel      all SMs: the side() scans (and wide partitions) of all trees.
// Node records come out tree-local and post-order; the host turns them into NodeCodec bytes.
#pragma once
#include <cooperative_groups.h>
#include "kernels.cuh"

namespace ab {

constexpr int CTRL_THREADS = 256;
constexpr int MAX_DEPTH = 4096;          // DFS frames per tree
constexpr uint32_t INLINE_PART_MAX = 8192;  // nodes up to this size are partitioned by the control CTA
constexpr uint32_t NO_SLOT = 0xffffffffu;

enum : int { PH_START = 0, PH_AWAIT_SCAN = 1, PH_AWAIT_PART = 2, PH_DONE = 3 };
enum : int { REC_DESC = 1, REC_SPLIT = 2 };
enum : int { ERR_NONE = 0, ERR_DEPTH = 1, ERR_RECORDS = 2, ERR_POOL = 3, ERR_HANG = 4, ERR_ABORT = 5 };

struct Frame {
    uint32_t start, len;     // segment of the tree's id permutation
    uint32_t left_len;       // number of ids that went Left (valid from stage 1)
    uint32_t left_id;        // local id of the finished left child (stage 3)
    uint32_t slot;           // normal pool slot, NO_SLOT = random split ("normal: none")
    uint8_t parity;          // which of the two ping-pong id buffers holds this node's ids
    uint8_t stage;           // 0 = new, 1 = split decided + partitioned, 2 = left in progress, 3 = right in progress
    uint16_t pad;
};

struct Record {  // tree-local node, in post-order; the root is the last record
    uint32_t kind;
    uint32_t a, b, c;  // DESC: start, len, parity   SPLIT: left local id, right local id, slot
};

struct TreeState {
    uint32_t key[8];
    uint64_t pos;            // StdRng words consumed
    int32_t phase;
    int32_t sp;              // top frame index
    int32_t attempts_left;
    uint32_t cur_slot;       // pool slot holding the current attempt's normal (NO_SLOT = none reserved)
    uint32_t n_recs;
    uint32_t n_splits_tried, n_random;
    uint32_t slot_next;      // pool slots are taken from the shared counter eight at a time: [slot_next, slot_end)
    uint64_t scanned;        // rows that went through side()
    uint32_t slot_end;
    uint32_t n_misspec;      // create_split calls whose speculative two_means had to be redone sequentially
};

// Persistent schedule (control_kernel<.., CS = 0>): one launch per wave holds one control CTA per tree and worker CTAs on
// every SM; a control CTA publishes its scan / wide-partition job in its tree's slot and the workers claim units of it.
// Everything a worker needs sits in ONE 128-byte line and the protocol is one word: ticket = seq:16 | total units:24 | next
// unclaimed unit:24. A claim is one atomicAdd on it and carries the epoch it belongs to, so a worker that raced with the
// publication of the next job can tell whose units it holds; a global round trip costs ~0.7 us here, so the path from
// "published" to "reported" is kept to: poll, claim (with the field and normal loads in flight), id list, item rows, report.
struct __align__(128) PSlot {
    unsigned long long ticket;
    unsigned long long done;     // seq:32 | units reported finished:32
    const uint32_t* rows; uint8_t* flags; uint32_t* unit_left; uint32_t* dst;
    uint32_t len, kind, total_left, chunk;
    uint32_t pad[16];
};
__device__ __forceinline__ unsigned long long pticket(uint32_t seq, uint32_t total, uint32_t next) { return ((unsigned long long)(seq & 0xffffu) << 48) | ((unsigned long long)(total & 0xffffffu) << 24) | (unsigned long long)(next & 0xffffffu); }
__device__ __forceinline__ uint32_t pt_seq(unsigned long long t) { return (uint32_t)(t >> 48); }
__device__ __forceinline__ uint32_t pt_total(unsigned long long t) { return (uint32_t)(t >> 24) & 0xffffffu; }
__device__ __forceinline__ uint32_t pt_next(unsigned long long t) { return (uint32_t)t & 0xffffffu; }
constexpr uint32_t LAT_MASK = 3;   // worker w is a latency worker (pworker) when (w & LAT_MASK) == 0: one in four
// units per claim of a scan through the 8-bit planes: SHADOW_CHUNK, or SHADOW_BIG_CHUNK for scans of more than SHADOW_BIG_UNITS
constexpr uint32_t SHADOW_CHUNK = 4, SHADOW_BIG_UNITS = 512, SHADOW_BIG_CHUNK = 8;

struct BuildParams {
    const float* items; const float* ih0; const float* ih1;
    uint32_t n, d, ld; int32_t metric; uint32_t K;
    uint32_t n_trees;
    TreeState* st; Frame* frames; Record* recs; uint32_t rec_cap;
    uint32_t* perm[2];       // n_trees x n each
    uint8_t* flags;          // n_trees x n
    uint32_t* unit_left;     // n_trees x units_per_tree
    uint32_t units_per_tree;
    float* pool; uint32_t pool_stride; uint32_t pool_cap; uint32_t* pool_counter;
    Job* jobs;
    float* scratch;          // n_trees x WS_VECS x ld (two_means workspace when it does not fit in smem)
    int32_t use_smem_ws;
    int32_t spec;            // speculative two_means: the shared-memory workspace holds WS_VECS_SPEC vectors
    uint32_t* active;        // trees not yet done
    int32_t* error;
    // optional: tree t is built over the ascending row subset sub_rows[sub_off[t] .. sub_off[t+1])
    // instead of all n rows (incremental builds: one subtree per over-full descendant)
    const uint32_t* sub_rows;
    const uint64_t* sub_off;
    // cluster-resident small nodes (control_kernel<.., CS > 1>): nodes of at most small_max rows are
    // scanned by the control kernel's own cluster, at most max_inner attempts per launch
    uint32_t small_max, max_inner;
    // persistent schedule
    PSlot* slots;                 // n_trees
    float* cur_normal;            // n_trees x pool_stride: the normal of each tree's open scan job, at an address workers know without the job fields
    const volatile int* abort;    // set by the host (cancel): control CTAs stop at their next wait
    // fused root scan: when every tree of the wave starts at the root of the whole index, the first split's side() scans of all
    // trees read the same rows — the workers do them in ONE pass over the item matrix (proot below)
    // the 8-bit planes of the item matrix (kernels.cuh), or NULLs: scans of more than shadow_min_units units go through them
    // (scan_claim_planes)
    PlaneRows planes;
    uint32_t shadow_min_units;
    unsigned long long* shadow_stats;   // [0] rows scanned through the planes, [1] of them re-scored from the f32 row, [2] through stage 2
    int32_t root_fused;
    uint32_t* root_ready;         // number of trees whose root normal is published
    uint32_t* root_ticket;        // next unclaimed chunk of the fused pass
};

__device__ __forceinline__ double split_imbalance_dev(uint32_t l, uint32_t r) {  // src/writer.rs:1348-1353
    double ls = (double)l, rs = (double)r;
    double f = ls / (ls + rs + 2.220446049250313e-16);
    double g = 1.0 - f;
    return f > g ? f : g;
}

// ---- two_means + create_split on one CTA ----------------------------------------------------
// ws: WS_VECS vectors of ld floats: ws[0]=p, ws[1]=q, ws[2..11]=the ten sampled k,
// ws[12], ws[13] = scratch (normal / bias terms / Manhattan terms / k / norm of the current iteration).
constexpr int WS_VECS = 14;
// Speculative two_means (spec_two_means below) keeps every centroid version of the ten iterations: ws[14 + it] = the centroid
// that iteration `it` produced. 24 vectors in all; used when they fit in shared memory.
constexpr int WS_VECS_SPEC = 24;
struct TwoMeansShared {
    uint32_t rows[12];
    float h0[12], h1[12];
    float nk[12];           // D::norm of p (0), q (1) and of the ten k (2..11)
    float res[2][2];        // di, dj, double buffered by iteration parity
    float php[2], phq[2];   // headers of p and q
    float misc[2];
    // speculative two_means
    float G[12][12];        // approximate dots between the 12 gathered vectors (0 = p, 1 = q after normalize, 2.. = the ten k)
    float Gp[8][16][16];    // its partial products, one 16 x 16 tile per warp
    float An[10][10];       // An[it][l] = (k_it / norm_it) . k_l
    float rc[10][7];        // per-iteration constants of the recurrence
    float vdot[32];         // exact dots of the verification pass
    int choice[10];         // per iteration: 0 = nothing moved, 1 = p moved, 2 = q moved
    int ready;              // iterations whose choice has been published by the speculating warp
    int mismatch;
};

// hsum256 of the four accumulators + ((h1+h2)+h3)+h4 when lane l holds accumulator lane l (simple_avx.rs:6-13)
__device__ __forceinline__ float warp_hsum_exact(float acc) {
    const unsigned full = 0xffffffffu;
    acc = __fadd_rn(acc, __shfl_xor_sync(full, acc, 4));
    acc = __fadd_rn(acc, __shfl_xor_sync(full, acc, 2));
    acc = __fadd_rn(acc, __shfl_xor_sync(full, acc, 1));
    const float h1 = __shfl_sync(full, acc, 0), h2 = __shfl_sync(full, acc, 8), h3 = __shfl_sync(full, acc, 16), h4 = __shfl_sync(full, acc, 24);
    return __fadd_rn(__fadd_rn(__fadd_rn(h1, h2), h3), h4);
}

// dot(a, b) [Euclidean: sum (a-b)^2] and dot(a, a) of one vector pair on one warp, lane l = accumulator lane l
// (scalar loads, conflict-free; two independent FMA chains per lane). All 32 lanes must call.
template <bool EUCLID>
__device__ __forceinline__ void exact_warp_ab_aa(const float* a, const float* b, int n, float& ab, float& aa) {
    const int lane = threadIdx.x & 31;
    if (n >= 32) {
        const int m = n & ~31;
        float acc = 0.f, acc2 = 0.f;
#pragma unroll 8
        for (int i = lane; i < m; i += 32) {
            const float x = a[i], y = b[i];
            if (EUCLID) { const float t = __fsub_rn(x, y); acc = fmaf(t, t, acc); }
            else { acc = fmaf(x, y, acc); acc2 = fmaf(x, x, acc2); }
        }
        float r = warp_hsum_exact(acc), r2 = EUCLID ? 0.f : warp_hsum_exact(acc2);
        for (int i = m; i < n; ++i) {
            if (EUCLID) { const float t = __fsub_rn(a[i], b[i]); r = __fadd_rn(r, __fmul_rn(t, t)); }
            else { r = __fadd_rn(r, __fmul_rn(a[i], b[i])); r2 = __fadd_rn(r2, __fmul_rn(a[i], a[i])); }
        }
        ab = r; aa = r2;
    } else {
        float r = 0.f, r2 = 0.f;
        if (lane == 0) { r = exact_thread<EUCLID>(a, b, n); if (!EUCLID) r2 = exact_thread<false>(a, a, n); }
        ab = __shfl_sync(0xffffffffu, r, 0); aa = __shfl_sync(0xffffffffu, r2, 0);
    }
}


// ---- speculative two_means ---------------------------------------------------------------------
// The ten iterations of two_means (src/distance/mod.rs:146-168) form a chain only through ten BRANCHES (which centroid
// moves); everything else is element-wise. So:
//  (1) predict the branches with ordinary float arithmetic on the 12 x 12 Gram matrix of the gathered vectors (every centroid
//      is a linear combination of them, so its dots with the ten k follow a scalar recurrence) — warp 0; meanwhile the other
//      warps produce the centroid versions element-wise, following the predictions as they are published;
//  (2) compute the reference's exact dots of ALL ten iterations at once, in the reference's summation order (32 dots, one per
//      8-lane group), and the exact di / dj from them;
//  (3) check that they take the predicted branches. If they do, the centroids are the reference's, bit for bit. If one does
//      not (|di - dj| below the prediction's rounding noise: rare), the caller runs the sequential loop instead.
// ws: slots 0 / 1 = p / q (normalized for the angular metrics), 2..11 = the ten k, 14 + it = centroid produced by iteration it.
// On success pslot / qslot are the slots of the final centroids.
template <int METRIC>
__device__ __forceinline__ bool spec_two_means(const BuildParams& P, float* ws, TwoMeansShared& S, int& pslot, int& qslot) {
    constexpr bool EUCLID = METRIC == EUCLIDEAN;
    constexpr int metric = METRIC;
    const unsigned full = 0xffffffffu;
    const int d = (int)P.d, ld = (int)P.ld;
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, grp = lane >> 3, g8 = lane & 7;
    const bool cosine = !EUCLID;
    if (tid == 0) { S.ready = 0; S.mismatch = 0; }
    // (1a) Gram matrix of the 12 gathered vectors on the tensor cores (mma.sync m16n8k8, TF32 inputs, FP32 accumulate): it only
    // has to PREDICT branches, so ~2^-10 relative input rounding is fine (a wrong prediction costs one sequential re-run). Rows
    // 12..15 of the 16 x 16 product read the neighbouring workspace slots; their entries are never used. Every warp takes the
    // 16-float chunks m = warp, warp + 8, ...; a lane (r = lane / 4, c = lane % 4) loads floats 4c..4c+3 of rows r and r + 8 of
    // the chunk — the SAME registers serve as A fragment (row-major 16 x 8) and as B fragment (col-major 8 x 8 of U^T), because
    // the k index of a dot product may be permuted freely as long as both operands use the same permutation.
    {
        float acc[2][4];
#pragma unroll
        for (int i = 0; i < 2; ++i)
#pragma unroll
            for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;
        const float* r0 = ws + (size_t)(lane >> 2) * ld + 4 * (lane & 3);
        const float* r1 = r0 + (size_t)8 * ld;
        const int nck = ld >> 4;
#pragma unroll 1
        for (int m = warp; m < nck; m += CTRL_THREADS / 32) {
            const float4 x0 = *reinterpret_cast<const float4*>(r0 + 16 * m);
            const float4 x1 = *reinterpret_cast<const float4*>(r1 + 16 * m);
            const uint32_t a0 = __float_as_uint(x0.x), a1 = __float_as_uint(x1.x), a2 = __float_as_uint(x0.y), a3 = __float_as_uint(x1.y);
            const uint32_t e0 = __float_as_uint(x0.z), e1 = __float_as_uint(x1.z), e2 = __float_as_uint(x0.w), e3 = __float_as_uint(x1.w);
            asm volatile("mma.sync.aligned.m16n8k8.row.col.f32.tf32.tf32.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
                         : "+f"(acc[0][0]), "+f"(acc[0][1]), "+f"(acc[0][2]), "+f"(acc[0][3]) : "r"(a0), "r"(a1), "r"(a2), "r"(a3), "r"(a0), "r"(a2));
            asm volatile("mma.sync.aligned.m16n8k8.row.col.f32.tf32.tf32.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
                         : "+f"(acc[1][0]), "+f"(acc[1][1]), "+f"(acc[1][2]), "+f"(acc[1][3]) : "r"(a0), "r"(a1), "r"(a2), "r"(a3), "r"(a1), "r"(a3));
            asm volatile("mma.sync.aligned.m16n8k8.row.col.f32.tf32.tf32.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
                         : "+f"(acc[0][0]), "+f"(acc[0][1]), "+f"(acc[0][2]), "+f"(acc[0][3]) : "r"(e0), "r"(e1), "r"(e2), "r"(e3), "r"(e0), "r"(e2));
            asm volatile("mma.sync.aligned.m16n8k8.row.col.f32.tf32.tf32.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
                         : "+f"(acc[1][0]), "+f"(acc[1][1]), "+f"(acc[1][2]), "+f"(acc[1][3]) : "r"(e0), "r"(e1), "r"(e2), "r"(e3), "r"(e1), "r"(e3));
        }
        // D fragment: acc[t][0..1] = D[lane / 4][8t + 2 (lane % 4) + {0, 1}], acc[t][2..3] = the same columns of row lane / 4 + 8
        float* gp = &S.Gp[warp][0][0];
#pragma unroll
        for (int t = 0; t < 2; ++t) {
            const int col = 8 * t + 2 * (lane & 3), row = lane >> 2;
            gp[row * 16 + col] = acc[t][0]; gp[row * 16 + col + 1] = acc[t][1];
            gp[(row + 8) * 16 + col] = acc[t][2]; gp[(row + 8) * 16 + col + 1] = acc[t][3];
        }
    }
    __syncthreads();
    if (tid < 144) {   // G = sum of the eight warps' partial products
        const int i = tid / 12, j = tid - 12 * i;
        float v = 0.f;
#pragma unroll
        for (int w = 0; w < CTRL_THREADS / 32; ++w) v += S.Gp[w][i][j];
        S.G[i][j] = v;
    }
    __syncthreads();
    // per-iteration constants of the recurrence (tid = iteration, or iteration x lane)
    if (tid < 10) {
        const float nrm = cosine ? S.nk[2 + tid] : 1.f;
        const float inv = __fdividef(1.f, nrm);
        S.rc[tid][0] = inv;                                      // 1 / norm_it
        S.rc[tid][1] = S.G[2 + tid][2 + tid] * inv * inv;        // (k / norm)^2
        S.rc[tid][2] = S.G[2 + tid][2 + tid];                    // k . k
        S.rc[tid][3] = (metric == COSINE) ? __fdividef(1.f, S.h0[2 + tid]) : S.h0[2 + tid];   // Cosine: 1 / |k| (stored header); DotProduct: k.extra_dim
        S.rc[tid][4] = S.h1[2 + tid];                            // DotProduct: k's norm header
        S.rc[tid][5] = (nrm != nrm || nrm <= 0.f) ? 0.f : 1.f;   // the loop's `continue` guard (mod.rs:152-155)
        S.rc[tid][6] = rsqrtf(S.h1[2 + tid]);                    // DotProduct: 1 / sqrt(k's norm header)
    }
    if (tid >= 32 && tid < 132) { const int it = (tid - 32) / 10, l = (tid - 32) - 10 * it; S.An[it][l] = S.G[2 + it][2 + l] * __fdividef(1.f, cosine ? S.nk[2 + it] : 1.f); }
    __syncthreads();
    if (warp == 0) {
        // (1b) the recurrence on SUMS: with Sp = ic * p (the sum of p0 and the k / norm assigned to it), lane l < 10 carries
        // Sp . k_l and Sq . k_l; every lane carries Sp . Sp, Sq . Sq and the counts. The warp runs alone, so what counts is the
        // length of the dependent chain from one branch to the next: the dots of the NEXT iteration are fetched from their lanes
        // before this iteration's branch is known (and patched with one add afterwards), and everything a branch changes — the
        // new Sp . Sp, its rsqrt / reciprocal, the new count — is computed for both outcomes ahead of the comparison.
        const int li = lane < 10 ? lane : 0;
        float spk = S.G[0][2 + li], sqk = S.G[1][2 + li];
        float spp = S.G[0][0], sqq = S.G[1][1], ic = 1.f, jc = 1.f;
        float a = __shfl_sync(full, spk, 0), b = __shfl_sync(full, sqk, 0);
        float rp = EUCLID ? 1.f : rsqrtf(spp), rq = EUCLID ? 1.f : rsqrtf(sqq);   // Euclidean: 1 / count; angular: 1 / |Sp|
        const float pe = S.php[0], qe = S.phq[0];   // DotProduct: extra_dim of the centroids (update_mean leaves headers alone)
#pragma unroll
        for (int it = 0; it < 10; ++it) {
            const float inv = S.rc[it][0], bb = S.rc[it][1], kk = S.rc[it][2], ka = S.rc[it][3], ok = S.rc[it][5];
            const float g = S.An[it][li];
            float a_nb = 0.f, b_nb = 0.f, g_n = 0.f;
            if (it < 9) { a_nb = __shfl_sync(full, spk, it + 1); b_nb = __shfl_sync(full, sqk, it + 1); g_n = S.An[it][it + 1]; }
            const float spp_n = spp + (2.f * a * inv + bb), sqq_n = sqq + (2.f * b * inv + bb);
            const float ic_n = ic + 1.f, jc_n = jc + 1.f;
            const float rp_n = EUCLID ? __fdividef(1.f, ic_n) : rsqrtf(spp_n), rq_n = EUCLID ? __fdividef(1.f, jc_n) : rsqrtf(sqq_n);
            float di, dj;
            if (EUCLID) { di = spp * rp - 2.f * a + ic * kk; dj = sqq * rq - 2.f * b + jc * kk; }
            else if (metric == COSINE) {
                const float cp = fminf(1.f, fmaxf(-1.f, a * rp * ka)), cq = fminf(1.f, fmaxf(-1.f, b * rq * ka));
                di = ic * (1.f - cp); dj = jc * (1.f - cq);
            } else {
                const float kb = S.rc[it][4], rkb = S.rc[it][6];   // (slot 6 of rc: 1 / sqrt(k's norm header))
                const float mp = spp * kb, mq = sqq * kb;
                di = mp >= 1.17549435e-38f * ic * ic ? ic * (2.f - 2.f * (a + ic * pe * ka) * rp * rkb) : ic * 2.f;
                dj = mq >= 1.17549435e-38f * jc * jc ? jc * (2.f - 2.f * (b + jc * qe * ka) * rq * rkb) : jc * 2.f;
            }
            const bool c1 = ok != 0.f && di < dj, c2 = ok != 0.f && dj < di;
            spk += c1 ? g : 0.f; sqk += c2 ? g : 0.f;
            a = a_nb + (c1 ? g_n : 0.f); b = b_nb + (c2 ? g_n : 0.f);
            spp = c1 ? spp_n : spp; rp = c1 ? rp_n : rp; ic = c1 ? ic_n : ic;
            sqq = c2 ? sqq_n : sqq; rq = c2 ? rq_n : rq; jc = c2 ? jc_n : jc;
            if (lane == 0) S.choice[it] = c1 ? 1 : (c2 ? 2 : 0);
        }
        asm volatile("" :: "f"(spk), "f"(sqk), "f"(spp), "f"(sqq), "f"(a), "f"(b) : "memory");
    } else if (cosine) {
        // meanwhile the other warps divide the ten k by their norms (the k / norm term of update_mean, mod.rs:172-180) into the
        // slots the centroid versions will be produced in; element i belongs to thread (i mod 224) + 32 from here on
        for (int it = 0; it < 10; ++it) {
            const float* k = ws + (size_t)(2 + it) * ld;
            float* out = ws + (size_t)(14 + it) * ld;
            const float norm = S.nk[2 + it];
            const UDiv D(norm);
            if (!(norm > 0.0f)) continue;                       // the iteration is skipped (mod.rs:152-155): nothing reads the slot
            bool bad = !D.ok;
            for (int i0 = tid - 32; i0 < ld; i0 += 4 * (CTRL_THREADS - 32)) {
                float a[4];
#pragma unroll
                for (int u = 0; u < 4; ++u) { const int i = i0 + u * (CTRL_THREADS - 32); a[u] = i < d ? k[i] : 0.f; }
#pragma unroll
                for (int u = 0; u < 4; ++u) { const int i = i0 + u * (CTRL_THREADS - 32); bad = bad || UDiv::suspect(a[u]); if (i < ld) out[i] = D.quot(a[u]); }
            }
            if (bad) S.mismatch = 1;                            // out of the fast division's range: the sequential loop decides
        }
    }
    __syncthreads();
    if (warp != 0) {
        // the centroid versions, element-wise and in the reference's exact operations; every thread only re-reads elements it
        // wrote itself, so the ten steps need no barrier
        float ic = 1.f, jc = 1.f;
        int ps = 0, qs = 1;
#pragma unroll 1
        for (int it = 0; it < 10; ++it) {
            const int ch = S.choice[it];
            if (ch == 0) continue;
            const float* kn = ws + (size_t)(cosine ? 14 + it : 2 + it) * ld;   // norm = 1: k / norm = k
            const float* cen = ws + (size_t)(ch == 1 ? ps : qs) * ld;
            float* out = ws + (size_t)(14 + it) * ld;
            const float cnt = ch == 1 ? ic : jc, c1 = __fadd_rn(cnt, 1.0f);
            const UDiv D(c1);                                   // c1 = 2 .. 11
            bool bad = false;
            for (int i0 = tid - 32; i0 < ld; i0 += 4 * (CTRL_THREADS - 32)) {
                float a[4];
#pragma unroll
                for (int u = 0; u < 4; ++u) { const int i = i0 + u * (CTRL_THREADS - 32); a[u] = i < d ? __fadd_rn(__fmul_rn(cen[i], cnt), kn[i]) : 0.f; }
#pragma unroll
                for (int u = 0; u < 4; ++u) { const int i = i0 + u * (CTRL_THREADS - 32); bad = bad || UDiv::suspect(a[u]); if (i < ld) out[i] = D.quot(a[u]); }
            }
            if (bad) S.mismatch = 1;
            if (ch == 1) { ps = 14 + it; ic = c1; } else { qs = 14 + it; jc = c1; }
        }
    }
    __syncthreads();
    // (2) the reference's dots: group j < 10: p_j . k_j, 10 + j: q_j . k_j (Euclidean: squared distances), 20 / 21: the D::init
    // dots of the initial p / q, 22 + j: of the centroid iteration j produced
    if (!EUCLID || warp < 5) {
        const int job = warp * 4 + grp;
        const float* a = ws; const float* b = ws;
        if (job < 20) {
            const int it = job % 10, side = job / 10;
            int slot = side;
            for (int j = 0; j < it; ++j) if (S.choice[j] == side + 1) slot = 14 + j;
            a = ws + (size_t)slot * ld; b = ws + (size_t)(2 + it) * ld;
        } else {
            const int v = job - 20;
            const int slot = v < 2 ? v : (S.choice[v - 2] ? 14 + (v - 2) : 0);
            a = b = ws + (size_t)slot * ld;
        }
        const float r = exact_group8<EUCLID>(a, b, d);
        if (g8 == 0) S.vdot[job] = r;
    }
    __syncthreads();
    // (3) exact di / dj of every iteration (mod.rs:148-149) against the predicted branch
    int ps = 0, qs = 1;
    if (tid < 10) {
        const int it = tid;
        float ic = 1.f, jc = 1.f;
        for (int j = 0; j < it; ++j) { const int c = S.choice[j]; if (c == 1) { ps = 14 + j; ic = __fadd_rn(ic, 1.0f); } else if (c == 2) { qs = 14 + j; jc = __fadd_rn(jc, 1.0f); } }
        const float xp = S.vdot[it], xq = S.vdot[10 + it];
        const float sp = S.vdot[ps < 2 ? 20 + ps : 22 + (ps - 14)], sq = S.vdot[qs < 2 ? 20 + qs : 22 + (qs - 14)];   // D::init dots
        const float kh0 = S.h0[2 + it], kh1 = S.h1[2 + it];
        float dvp, dvq;
        if (EUCLID) { dvp = xp; dvq = xq; }
        else if (metric == COSINE) { dvp = built_finish(COSINE, xp, __fsqrt_rn(sp), kh0); dvq = built_finish(COSINE, xq, __fsqrt_rn(sq), kh0); }
        else {   // dot_product.rs:58-70
            const float a1 = __fadd_rn(xp, __fmul_rn(S.php[0], kh0)), m1 = __fmul_rn(sp, kh1);
            dvp = (m1 >= 1.17549435e-38f) ? __fsub_rn(2.0f, __fdiv_rn(__fmul_rn(2.0f, a1), __fsqrt_rn(m1))) : 2.0f;
            const float a2 = __fadd_rn(xq, __fmul_rn(S.phq[0], kh0)), m2 = __fmul_rn(sq, kh1);
            dvq = (m2 >= 1.17549435e-38f) ? __fsub_rn(2.0f, __fdiv_rn(__fmul_rn(2.0f, a2), __fsqrt_rn(m2))) : 2.0f;
        }
        const float di = __fmul_rn(ic, dvp), dj = __fmul_rn(jc, dvq);
        const float norm = cosine ? S.nk[2 + it] : 1.0f;
        int want = 0;
        if (!(norm != norm || norm <= 0.0f)) want = di < dj ? 1 : (dj < di ? 2 : 0);
        if (want != S.choice[it]) S.mismatch = 1;
    }
    __syncthreads();
    if (S.mismatch) return false;
    ps = 0; qs = 1;
    for (int j = 0; j < 10; ++j) { const int c = S.choice[j]; if (c == 1) ps = 14 + j; else if (c == 2) qs = 14 + j; }
    pslot = ps; qslot = qs;
    return true;
}

// The sequential two_means loop (src/distance/mod.rs:146-168), in place on ws[0] / ws[1]: Manhattan, d < 32, workspaces too
// big for the speculative path, and the rare mis-speculation. Each iteration is ONE dot phase: warp 0 computes p.k and — for a
// centroid that was just moved — its D::init dot, warp 1 the same for q, then one barrier, the element-wise update_mean on all
// threads, one barrier. Out of line: it is not on the usual path and the control kernel is instruction-fetch bound.
template <int METRIC>
__device__ __noinline__ void two_means_sequential(const BuildParams& P, float* ws, TwoMeansShared& S) {
    constexpr int metric = METRIC;
    constexpr bool cosine = (METRIC == COSINE || METRIC == DOT_PRODUCT);
    const int d = (int)P.d, ld = (int)P.ld;
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    float* p = ws; float* q = ws + ld;
    float* sc0 = ws + (size_t)12 * ld; float* sc1 = ws + (size_t)13 * ld;
    float ic = 1.0f, jc = 1.0f;
    bool p_dirty = cosine, q_dirty = cosine;   // D::init pending (cosine.rs:69-71, dot_product.rs:94-96)
    // (kept rolled: the serial path runs on one or two warps, whose speed is set by instruction fetch —
    // ten unrolled copies of this body never hit the instruction cache)
#pragma unroll 1
    for (int it = 0; it < 10; ++it) {
        const float* k = ws + (size_t)(2 + it) * ld;
        const float kh0 = S.h0[2 + it], kh1 = S.h1[2 + it];
        if (metric == MANHATTAN) {  // manhattan.rs:44-46: strictly sequential sum of |p - k|
            for (int i = tid; i < d; i += blockDim.x) { sc0[i] = fabsf(__fsub_rn(p[i], k[i])); sc1[i] = fabsf(__fsub_rn(q[i], k[i])); }
            __syncthreads();
            if (tid < 2) {
                const float* t = tid ? sc1 : sc0;
                float s = 0.0f;
                int i = 0;
                for (; i + 8 <= d; i += 8) {
                    float t0 = t[i], t1 = t[i + 1], t2 = t[i + 2], t3 = t[i + 3], t4 = t[i + 4], t5 = t[i + 5], t6 = t[i + 6], t7 = t[i + 7];
                    s = __fadd_rn(s, t0); s = __fadd_rn(s, t1); s = __fadd_rn(s, t2); s = __fadd_rn(s, t3);
                    s = __fadd_rn(s, t4); s = __fadd_rn(s, t5); s = __fadd_rn(s, t6); s = __fadd_rn(s, t7);
                }
                for (; i < d; ++i) s = __fadd_rn(s, t[i]);
                S.res[it & 1][tid] = __fmul_rn(tid ? jc : ic, s);
            }
        } else if (warp < 2) {
            // warp 0: p.k and (after a move of p) p.p; warp 1: q.k and q.q — lane l = accumulator lane l, so both
            // sides run at the same time on two schedulers; lane 0 of each warp finishes its side.
            const bool qs = warp == 1;
            const float* a = qs ? q : p;
            float xk, xx;
            if (metric == EUCLIDEAN) exact_warp_ab_aa<true>(a, k, d, xk, xx); else exact_warp_ab_aa<false>(a, k, d, xk, xx);
            if (lane == 0) {
                float* hdr = qs ? S.phq : S.php;
                float h0v = hdr[0], h1v = hdr[1];
                if (qs ? q_dirty : p_dirty) { if (metric == COSINE) h0v = __fsqrt_rn(xx); else h1v = xx; hdr[0] = h0v; hdr[1] = h1v; }
                float dv;   // D::non_built_distance — mod.rs:54-56 (= built_distance) except dot_product.rs:58-70
                if (metric == EUCLIDEAN) dv = xk;
                else if (metric == COSINE) dv = built_finish(COSINE, xk, h0v, kh0);
                else {
                    const float a1 = __fadd_rn(xk, __fmul_rn(h0v, kh0));
                    const float m1 = __fmul_rn(h1v, kh1);
                    dv = (m1 >= 1.17549435e-38f) ? __fsub_rn(2.0f, __fdiv_rn(__fmul_rn(2.0f, a1), __fsqrt_rn(m1))) : 2.0f;
                }
                S.res[it & 1][qs ? 1 : 0] = __fmul_rn(qs ? jc : ic, dv);
            }
        } else if (cosine) {
            // meanwhile the other warps form k / norm for update_mean (mod.rs:86-94): it does not depend on
            // the centroids, so the division leaves the critical path
            const float nrm = S.nk[2 + it];
            for (int i = tid - 64; i < d; i += CTRL_THREADS - 64) sc1[i] = __fdiv_rn(k[i], nrm);
        }
        p_dirty = false; q_dirty = false;
        __syncthreads();
        const float di = S.res[it & 1][0], dj = S.res[it & 1][1];
        const float norm = cosine ? S.nk[2 + it] : 1.0f;
        if (norm != norm || norm <= 0.0f) continue;
        const float* kn = cosine ? sc1 : k;          // k / norm (norm == 1 for Euclidean / Manhattan: k itself)
        if (di < dj || dj < di) {                    // update_mean(c, k, norm, count) — mod.rs:86-94; D::init follows in the next dot phase
            const bool up = di < dj;
            float* cen = up ? p : q;
            const float cnt = up ? ic : jc, c1 = __fadd_rn(cnt, 1.0f);
            for (int i0 = tid; i0 < d; i0 += 4 * CTRL_THREADS) {   // four independent chains per thread
                float v[4];
#pragma unroll
                for (int u = 0; u < 4; ++u) { const int i = i0 + u * CTRL_THREADS; if (i < d) v[u] = __fdiv_rn(__fadd_rn(__fmul_rn(cen[i], cnt), cosine ? kn[i] : __fdiv_rn(kn[i], norm)), c1); }
#pragma unroll
                for (int u = 0; u < 4; ++u) { const int i = i0 + u * CTRL_THREADS; if (i < d) cen[i] = v[u]; }
            }
            if (up) { ic = c1; p_dirty = cosine; } else { jc = c1; q_dirty = cosine; }
            __syncthreads();
        }
    }
}

__device__ __forceinline__ float norm_leaf_group(int metric, const float* v, float h0, int d) {
    float dot = exact_group8<false>(v, v, d);
    if (metric == DOT_PRODUCT) return __fsqrt_rn(__fadd_rn(dot, __fmul_rn(h0, h0)));  // dot_product.rs:72-75
    return __fsqrt_rn(dot);                                                              // mod.rs:70-72
}
// Draws the RNG exactly like choose_two + 10 x choose (src/parallel.rs:342-367), runs
// two_means and the metric's create_split, writes the normal into `slot_ptr`
// ([h0,h1,0,0,v[ld]]). seg = the node's ascending id list. `ws` is the 14-vector workspace
// (shared memory in practice: the function is force-inlined so the loads become LDS).
//
// Latency matters here (this is the serial part of every tree's chain), so each two_means iteration
// is ONE dot phase: warp 0 computes p.k, q.k and — for a centroid that was just moved — its D::init
// dot (p.p / q.q) on four 8-lane groups at the same time, then one barrier, the element-wise
// update_mean on all threads, one barrier.
template <int METRIC>
__device__ __forceinline__ void create_split_cta(const BuildParams& P, Rng& rng /* thread 0 only */, const uint32_t* seg, uint32_t len,
                                                 float* ws, TwoMeansShared& S, float* slot_ptr, float* mirror = nullptr /* second copy of the slot */) {
    // Binary-quantized metrics: two_means_binary_quantized (mod.rs:173-223) turns the sampled leaves into f32 leaves of the
    // NON-quantized distance and runs the ordinary loop — on the device the items already are those +-1 vectors and their headers,
    // so everything up to the centroids is the base metric's code; only the normal differs (below).
    constexpr int metric = base_metric(METRIC);
    constexpr bool BQ = is_bq(METRIC);
    constexpr bool cosine = (metric == COSINE || metric == DOT_PRODUCT);
    const int d = (int)P.d, ld = (int)P.ld;
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, grp = lane >> 3;
    // All RNG draws of the attempt first: they do not depend on the data. choose_two = index::sample(len, 2)
    // = gen_range(0..=len-2), gen_range(0..=len-1); then ten gen_range(0..=len-1). rand 0.8.5's sample_single_inclusive accepts a
    // word v iff low32(v * range) <= zone with zone = (range << lzcnt(range)) - 1 — a deliberately loose zone: between half and
    // all of the words are accepted, so the twelve draws consume ~12-24 words. The stream is a queue: draw 0 takes the first
    // word acceptable for range len-1, every later draw the next word acceptable for range len. The blocks were computed ahead
    // (rng.pref, >= 64 words from pos), so both acceptance masks of the next 64 words are two ballots, the twelve words are found
    // with find-nth-set-bit, and the serial loop only runs when 64 words were not enough.
    if (warp == 0) {
        bool done = false;
        const uint64_t pos = rng.pos;
        const uint64_t base16 = rng.pref_base << 4;
        if (rng.pref && pos >= base16 && pos + 64 <= base16 + ((uint64_t)rng.pref_n << 4)) {
            const uint32_t r0 = len - 1u, r1 = len;
            const uint32_t z0 = (r0 << __clz((int)r0)) - 1u, z1 = (r1 << __clz((int)r1)) - 1u;
            const uint32_t off = (uint32_t)(pos - base16);
            const uint32_t vlo = rng.pref[off + lane], vhi = rng.pref[off + 32 + lane];
            const unsigned a0lo = __ballot_sync(0xffffffffu, (uint32_t)((unsigned long long)vlo * r0) <= z0), a0hi = __ballot_sync(0xffffffffu, (uint32_t)((unsigned long long)vhi * r0) <= z0);
            const unsigned a1lo = __ballot_sync(0xffffffffu, (uint32_t)((unsigned long long)vlo * r1) <= z1), a1hi = __ballot_sync(0xffffffffu, (uint32_t)((unsigned long long)vhi * r1) <= z1);
            const unsigned long long a0 = (unsigned long long)a0lo | ((unsigned long long)a0hi << 32), a1 = (unsigned long long)a1lo | ((unsigned long long)a1hi << 32);
            if (r0 != 0u && a0 != 0ull) {
                const int idx0 = __ffsll((long long)a0) - 1;
                const unsigned long long rest = idx0 >= 63 ? 0ull : (a1 & ~((2ull << idx0) - 1ull));
                if (__popcll(rest) >= 11) {
                    // lane j (1..11): the j-th acceptable word after idx0; lane 0: idx0 itself
                    const unsigned lo = (unsigned)rest, hi = (unsigned)(rest >> 32);
                    const int clo = __popc(lo);
                    int idx = idx0;
                    if (lane >= 1 && lane < 12) idx = lane <= clo ? (int)__fns(lo, 0, lane) : 32 + (int)__fns(hi, 0, lane - clo);
                    const uint32_t v = rng.pref[off + (uint32_t)(lane < 12 ? idx : 0)];
                    const uint32_t r = (uint32_t)(((unsigned long long)v * (unsigned long long)(lane == 0 ? r0 : r1)) >> 32);
                    const uint32_t t0 = __shfl_sync(0xffffffffu, r, 0), t1 = __shfl_sync(0xffffffffu, r, 1);
                    if (lane == 0) { if (t1 == t0) { S.rows[0] = len - 1u; S.rows[1] = t0; } else { S.rows[0] = t0; S.rows[1] = t1; } }
                    if (lane >= 2 && lane < 12) S.rows[lane] = r;
                    if (lane == 11) rng.pos = pos + (uint64_t)idx + 1u;
                    done = true;
                }
            }
        }
        if (!done && lane == 0) {
            uint32_t a, b;
            rng.sample2(len, a, b);
            S.rows[0] = a; S.rows[1] = b;
#pragma unroll 1
            for (int it = 0; it < 10; ++it) S.rows[2 + it] = rng.gen_range_incl(0, len - 1);
        }
    }
    __syncthreads();
    uint32_t my_row = 0;
    if (tid < 12) my_row = __ldcg(seg + S.rows[tid]);  // RoaringBitmap::select(rank) on the ascending id list
    __syncthreads();
    if (tid < 12) S.rows[tid] = my_row;
    __syncthreads();
    {   // gather: warp w copies rows w and w + 8; all loads of a thread are issued before any store
        if (tid < 12) { S.h0[tid] = P.ih0 ? P.ih0[my_row] : 0.f; S.h1[tid] = P.ih1 ? P.ih1[my_row] : 0.f; }
        const int l4 = ld >> 2;
        for (int j = warp; j < 12; j += 8) {
            const float4* src = reinterpret_cast<const float4*>(P.items + (size_t)S.rows[j] * ld);
            float4* dst = reinterpret_cast<float4*>(ws + (size_t)j * ld);
            for (int c0 = lane; c0 < l4; c0 += 32 * 8) {
                float4 v[8];
#pragma unroll
                for (int u = 0; u < 8; ++u) { int c = c0 + 32 * u; if (c < l4) v[u] = __ldg(src + c); }
#pragma unroll
                for (int u = 0; u < 8; ++u) { int c = c0 + 32 * u; if (c < l4) dst[c] = v[u]; }
            }
        }
    }
    __syncthreads();
    if (tid == 0) { S.php[0] = S.h0[0]; S.php[1] = S.h1[0]; S.phq[0] = S.h0[1]; S.phq[1] = S.h1[1]; }
    float* p = ws; float* q = ws + ld;
    float* sc0 = ws + (size_t)12 * ld; float* sc1 = ws + (size_t)13 * ld;
    if (cosine) {
        // D::norm of all 12 gathered leaves in one pass: 8 warps x 4 groups. For p and q it feeds
        // D::normalize (mod.rs:76-82, dot_product.rs:85-92); for the ten k it is the `norm` of
        // two_means' loop (mod.rs:152) — it does not depend on the centroids.
        const int gi = warp * 4 + grp;
        const int j = gi < 12 ? gi : 0;
        float x = norm_leaf_group(metric, ws + (size_t)j * ld, S.h0[j], d);
        if (gi < 12 && (lane & 7) == 0) S.nk[gi] = x;
        __syncthreads();
        const float np = S.nk[0], nq = S.nk[1];
        if (np > 0.0f) udiv_loop(tid, CTRL_THREADS, d, np, [&](int i) { return p[i]; }, [&](int i, float v) { p[i] = v; });
        if (nq > 0.0f) udiv_loop(tid, CTRL_THREADS, d, nq, [&](int i) { return q[i]; }, [&](int i, float v) { q[i] = v; });
        if (tid == 0 && metric == DOT_PRODUCT) {
            if (np > 0.0f) S.php[0] = __fdiv_rn(S.php[0], np);
            if (nq > 0.0f) S.phq[0] = __fdiv_rn(S.phq[0], nq);
        }
    }
    __syncthreads();
    bool spec_done = false;
    if constexpr (metric != MANHATTAN) {
        if (P.spec && d >= 32) {
            int ps = 0, qs = 1;
            spec_done = spec_two_means<metric>(P, ws, S, ps, qs);
            if (spec_done) { p = ws + (size_t)ps * ld; q = ws + (size_t)qs * ld; }
        }
    }
    if (!spec_done) two_means_sequential<metric>(P, ws, S);
    __syncthreads();
    // normal = normalize(p - q) (+ bias / extra_dim) — euclidean.rs:59-75, manhattan.rs:62-78,
    // cosine.rs:77-83, dot_product.rs:102-111. (A D::init still pending after the last update only
    // touches the centroid's norm header, which create_split does not read.)
    float* nv = sc0;
    if constexpr (BQ) {
        // create_split of binary_quantized_{euclidean,cosine,manhattan}.rs: p - q goes through UnalignedVector::<BinaryQuantized>::
        // from_vec, i.e. only its sign bits survive (is_sign_positive -> +1, else -1); Self::normalize then divides by a positive
        // norm (or does nothing) and re-quantizes, which cannot change a bit. bias (Euclidean / Manhattan) = sum of
        // -n * (P + Q) / 2 over the QUANTIZED centroids P, Q — every term is -1, 0 or 1, so the sum is exact in any order, and it
        // is folded left to right like the reference's anyway.
        float* out = slot_ptr + NORMAL_HDR;
        for (int i = tid; i < ld; i += blockDim.x) {
            const float v = i < d ? ((__float_as_uint(__fsub_rn(p[i], q[i])) >> 31) ? -1.0f : 1.0f) : 0.f;
            nv[i] = v; out[i] = v;
            if (mirror != nullptr) mirror[NORMAL_HDR + i] = v;
            if (METRIC != BQ_COSINE && i < d) {
                const float Pq = (__float_as_uint(p[i]) >> 31) ? -1.0f : 1.0f, Qq = (__float_as_uint(q[i]) >> 31) ? -1.0f : 1.0f;
                sc1[i] = __fdiv_rn(__fmul_rn(-v, __fadd_rn(Pq, Qq)), 2.0f);
            }
        }
        __syncthreads();
        if (tid == 0) {
            float bias = 0.0f;
            if (METRIC != BQ_COSINE) for (int i = 0; i < d; ++i) bias = __fadd_rn(bias, sc1[i]);
            slot_ptr[0] = bias; slot_ptr[1] = 0.f; slot_ptr[2] = 0.f; slot_ptr[3] = 0.f;
            if (mirror != nullptr) mirror[0] = bias;
        }
        __syncthreads();
    } else {
    for (int i = tid; i < ld; i += blockDim.x) nv[i] = i < d ? __fsub_rn(p[i], q[i]) : 0.f;
    float extra = (metric == DOT_PRODUCT) ? __fsub_rn(S.php[0], S.phq[0]) : 0.f;
    __syncthreads();
    if (warp == 0) { float x = norm_leaf_group(metric, nv, extra, d); if (lane == 0) S.misc[0] = x; }
    __syncthreads();
    const float nn = S.misc[0];
    float* out = slot_ptr + NORMAL_HDR;
    if (nn > 0.0f) { udiv_loop(tid, CTRL_THREADS, d, nn, [&](int i) { return nv[i]; }, [&](int i, float v) { nv[i] = v; }); extra = (metric == DOT_PRODUCT) ? __fdiv_rn(extra, nn) : extra; }
    for (int i = tid; i < ld; i += blockDim.x) out[i] = nv[i];  // each thread re-reads only what it wrote
    if (mirror != nullptr) for (int i = tid; i < ld; i += blockDim.x) mirror[NORMAL_HDR + i] = nv[i];
    if (metric == EUCLIDEAN || metric == MANHATTAN) {
        // bias = sum over i of ((-n_i) * (p_i + q_i)) / 2, folded left to right from +0.0
        for (int i = tid; i < d; i += blockDim.x) sc1[i] = __fmul_rn(__fmul_rn(-nv[i], __fadd_rn(p[i], q[i])), 0.5f);   // x / 2 == x * 0.5 in every rounding case
        __syncthreads();
        if (tid == 0) {
            float bias = 0.0f;
            int i = 0;
            for (; i + 8 <= d; i += 8) {
                float t0 = sc1[i], t1 = sc1[i + 1], t2 = sc1[i + 2], t3 = sc1[i + 3], t4 = sc1[i + 4], t5 = sc1[i + 5], t6 = sc1[i + 6], t7 = sc1[i + 7];
                bias = __fadd_rn(bias, t0); bias = __fadd_rn(bias, t1); bias = __fadd_rn(bias, t2); bias = __fadd_rn(bias, t3);
                bias = __fadd_rn(bias, t4); bias = __fadd_rn(bias, t5); bias = __fadd_rn(bias, t6); bias = __fadd_rn(bias, t7);
            }
            for (; i < d; ++i) bias = __fadd_rn(bias, sc1[i]);
            slot_ptr[0] = bias; slot_ptr[1] = 0.f; slot_ptr[2] = 0.f; slot_ptr[3] = 0.f;
            if (mirror != nullptr) mirror[0] = bias;
        }
    } else if (tid == 0) {
        slot_ptr[0] = (metric == DOT_PRODUCT) ? extra : 0.f;  // Cosine normal header: norm = 0.0; Dot: {extra_dim, norm = 0.0}
        slot_ptr[1] = 0.f; slot_ptr[2] = 0.f; slot_ptr[3] = 0.f;
        if (mirror != nullptr) mirror[0] = (metric == DOT_PRODUCT) ? extra : 0.f;
    }
    __syncthreads();
    }
}

// CTA-wide stable partition of a whole node (any size) by its flags. Each round handles
// PART_BATCH sub-blocks of blockDim ids: all loads of the round are issued before any is used, one
// barrier per round. sm_pw: 2 * PART_BATCH * 8 + 2 uint32.
constexpr int PART_BATCH = 8;
__device__ __noinline__ void partition_inline(const uint32_t* __restrict__ src, const uint8_t* __restrict__ flags, uint32_t* __restrict__ dst, uint32_t len, uint32_t total_left, uint32_t* sm_pw) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    uint32_t left_before = 0;
    for (uint32_t base = 0; base < len; base += PART_BATCH * CTRL_THREADS) {
        uint32_t id[PART_BATCH];
        int fl[PART_BATCH];
#pragma unroll
        for (int j = 0; j < PART_BATCH; ++j) {
            uint32_t p = base + j * CTRL_THREADS + threadIdx.x;
            bool v = p < len;
            fl[j] = v ? (int)__ldcg(flags + p) : 2;   // 2 = out of range
            id[j] = v ? __ldcg(src + p) : 0u;
        }
        unsigned lm[PART_BATCH], rm[PART_BATCH];
#pragma unroll
        for (int j = 0; j < PART_BATCH; ++j) {
            lm[j] = __ballot_sync(0xffffffffu, fl[j] == 0);
            rm[j] = __ballot_sync(0xffffffffu, fl[j] == 1);
            if (lane == 0) { sm_pw[j * 8 + warp] = __popc(lm[j]); sm_pw[PART_BATCH * 8 + j * 8 + warp] = __popc(rm[j]); }
        }
        __syncthreads();
        // source order = sub-blocks in order, warps in order inside a sub-block = the index order of sm_pw: warp 0 turns the 64
        // Left counts and the 64 Right counts into exclusive prefixes (two entries per lane), entry 128 / 129 = the totals
        if (warp == 0) {
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const uint32_t a = sm_pw[h * 64 + 2 * lane], b = sm_pw[h * 64 + 2 * lane + 1];
                uint32_t inc = a + b;
                for (int o = 1; o < 32; o <<= 1) { const uint32_t y = __shfl_up_sync(0xffffffffu, inc, o); if (lane >= o) inc += y; }
                const uint32_t ex = inc - (a + b);
                sm_pw[h * 64 + 2 * lane] = ex; sm_pw[h * 64 + 2 * lane + 1] = ex + a;
                if (lane == 31) sm_pw[128 + h] = inc;
            }
        }
        __syncthreads();
        const unsigned below = (1u << lane) - 1u;
        const uint32_t right_before = base - left_before;
#pragma unroll
        for (int j = 0; j < PART_BATCH; ++j) {
            if (fl[j] == 0) dst[left_before + sm_pw[j * 8 + warp] + __popc(lm[j] & below)] = id[j];
            else if (fl[j] == 1) dst[total_left + right_before + sm_pw[64 + j * 8 + warp] + __popc(rm[j] & below)] = id[j];
        }
        left_before += sm_pw[128];
        __syncthreads();
    }
}

// exclusive scan (in place) of v[0..n) by one CTA; returns the total to every thread
__device__ uint32_t cta_exclusive_scan(uint32_t* v, uint32_t n, uint32_t* sm_tmp /* blockDim */) {
    const int tid = threadIdx.x, nt = blockDim.x;
    const uint32_t per = (n + nt - 1) / nt;
    if (per <= 1) {   // one element per thread (small nodes): a single read of v, the value stays in a register
        const uint32_t x = (uint32_t)tid < n ? __ldcg(v + tid) : 0u;
        const int lane = tid & 31, w = tid >> 5;
        uint32_t inc = x;
        for (int o = 1; o < 32; o <<= 1) { uint32_t y = __shfl_up_sync(0xffffffffu, inc, o); if (lane >= o) inc += y; }
        if (lane == 31) sm_tmp[w] = inc;
        __syncthreads();
        uint32_t base = 0, total = 0;
        for (int i = 0; i < nt / 32; ++i) { const uint32_t y = sm_tmp[i]; if (i < w) base += y; total += y; }
        if ((uint32_t)tid < n) v[tid] = base + inc - x;
        __syncthreads();
        return total;
    }
    const uint32_t b = (uint32_t)tid * per, e = (b + per < n) ? b + per : n;
    uint32_t s = 0;
    for (uint32_t i = b; i < e; ++i) s += __ldcg(v + i);
    sm_tmp[tid] = s;
    __syncthreads();
    if (tid < 32) {  // warp 0: exclusive scan of the nt partials (nt == 8 * 32)
        const int per_lane = nt / 32;
        uint32_t loc = 0;
        for (int i = 0; i < per_lane; ++i) loc += sm_tmp[tid * per_lane + i];
        uint32_t inc = loc;
        for (int o = 1; o < 32; o <<= 1) { uint32_t y = __shfl_up_sync(0xffffffffu, inc, o); if (tid >= o) inc += y; }
        uint32_t run2 = inc - loc;
        for (int i = 0; i < per_lane; ++i) { uint32_t x = sm_tmp[tid * per_lane + i]; sm_tmp[tid * per_lane + i] = run2; run2 += x; }
        if (tid == 31) sm_tmp[nt] = inc;
    }
    __syncthreads();
    uint32_t run = sm_tmp[tid];
    for (uint32_t i = b; i < e; ++i) { uint32_t x = __ldcg(v + i); v[i] = run; run += x; }
    uint32_t total = sm_tmp[nt];
    __syncthreads();
    return total;
}

enum : int { ACT_NONE = 0, ACT_SPLIT = 1, ACT_PART_INLINE = 2, ACT_RANDOM = 3, ACT_EXIT = 4, ACT_PART_WIDE = 5 };


// ---- persistent schedule: job slots between the control CTAs and the worker CTAs of ONE launch -------------------------
__device__ __forceinline__ unsigned long long ld_vol64(const unsigned long long* p) { return *reinterpret_cast<const volatile unsigned long long*>(p); }
__device__ __forceinline__ void st_vol64(unsigned long long* p, unsigned long long v) { *reinterpret_cast<volatile unsigned long long*>(p) = v; }
__device__ __forceinline__ uint32_t ld_vol32(const uint32_t* p) { return *reinterpret_cast<const volatile uint32_t*>(p); }

// thread 0 of a control CTA, after every thread's writes were fenced and a CTA barrier: open `total` units of `jb` (epoch seq)
__device__ __forceinline__ void ppublish(PSlot& sl, const Job& jb, uint32_t seq, uint32_t total, uint32_t chunk) {
    volatile PSlot* v = &sl;
    v->rows = jb.rows; v->flags = jb.flags; v->unit_left = jb.unit_left; v->dst = jb.dst;
    v->len = jb.len; v->kind = (uint32_t)jb.kind; v->total_left = jb.total_left; v->chunk = chunk;
    v->done = (unsigned long long)seq << 32;
    __threadfence();
    v->ticket = pticket(seq, total, 0u);
}
// ... and wait until the workers have reported all of them. false: error / cancel / no progress for ~4 s (never on a sane run)
__device__ __forceinline__ bool pwait(const BuildParams& P, PSlot& sl, uint32_t seq, uint32_t total) {
    const long long t0 = clock64();
    uint32_t spins = 0;
    const unsigned long long want = ((unsigned long long)seq << 32) | total;
    for (;;) {
        if (ld_vol64(&sl.done) == want) { __threadfence(); return true; }
        if ((++spins & 63u) == 0u) {
            if (*reinterpret_cast<volatile int32_t*>(P.error) != ERR_NONE) return false;
            if (P.abort != nullptr && *P.abort != 0) { atomicCAS(P.error, ERR_NONE, ERR_ABORT); return false; }
            if (clock64() - t0 > 8000000000ll) { atomicCAS(P.error, ERR_NONE, ERR_HANG); return false; }
        }
        __nanosleep(20);
    }
}

// ---- fused root scan -------------------------------------------------------------------------------------------------------
// The root of every tree is the whole index, so the first side() scan of each of the wave's T trees reads all n rows: T passes
// over the item matrix (at 50 trees, one eleventh of all the bytes a C2 build reads). Here the workers wait until the T root
// normals are published and make ONE pass: a claim is ROOT_CHUNK scan units; for every batch of ROOT_TB normals (staged in
// shared memory) its rows are dotted with all of them — the first batch streams the rows from HBM, the others find them in
// L2 — in exactly scan_unit's summation order, so flags and unit counts are the ones T separate scans would have written.
constexpr int ROOT_TB = 8;       // normals per pass over a claim's rows (8 x 2 rows x float4 accumulators = 64 registers)
constexpr uint32_t ROOT_CHUNK = 8;   // scan units per claim (measured: 8 -> 18.8M cycles for 50 roots of 1M x 768, 4 -> 20.3M, 1 -> 21.3M)

// units [u0, u1) of the root against the NB normals staged in smN (trees tb .. tb + NB - 1). The next chunk of the two rows
// and the next normal's chunk are requested before the current one is used: the loop has to run at the FMA rate, not at the
// latency of a load.
// ask L2 for the rows of one scan unit of the root (identity id list): one bulk prefetch per row, no register is tied up
__device__ __forceinline__ void proot_prefetch(const BuildParams& P, uint32_t unit) {
    const uint32_t r = unit * SCAN_UNIT + threadIdx.x;
    if (threadIdx.x < SCAN_UNIT && r < P.n) {
        const float* row = P.items + (size_t)r * P.ld;
        asm volatile("cp.async.bulk.prefetch.L2.global [%0], %1;" :: "l"(row), "r"(P.ld * 4u) : "memory");
    }
}
template <int NB>
__device__ __forceinline__ void proot_units(const BuildParams& P, uint32_t u0, uint32_t u1, uint32_t tb, uint32_t next_u0, const float* smN, const float* r_h0, uint32_t* r_cnt) {
    const uint32_t n = P.n, d = P.d, ld = P.ld;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, g8 = lane & 7, grp = lane >> 3;
    const int nch = (int)(d >> 5);
    const uint32_t units_all = (n + SCAN_UNIT - 1) / SCAN_UNIT;
    for (uint32_t unit = u0; unit < u1; ++unit) {
        if (tid < NB) r_cnt[tid] = 0;
        if (tb == 0) {   // the first batch meets the rows in HBM: have the next unit (of this claim, then of the next one) on its way to L2
            const uint32_t nu = unit + 1 < u1 ? unit + 1 : next_u0;
            if (nu < units_all) proot_prefetch(P, nu);
        }
        __syncthreads();
        const uint32_t pa = unit * SCAN_UNIT + warp * 8 + grp * 2, pb = pa + 1;
        const bool va = pa < n, vb = pb < n;
        const uint32_t ra = va ? pa : 0u, rb = vb ? pb : 0u;   // the root's id list is the identity
        const float4* A = reinterpret_cast<const float4*>(P.items + (size_t)ra * ld) + g8;
        const float4* B = reinterpret_cast<const float4*>(P.items + (size_t)rb * ld) + g8;
        const float4* N = reinterpret_cast<const float4*>(smN) + g8;
        const int nstride = (int)(ld >> 2);   // float4 per normal
        float4 acc[NB][2];
#pragma unroll
        for (int j = 0; j < NB; ++j) { acc[j][0] = make_float4(0.f, 0.f, 0.f, 0.f); acc[j][1] = acc[j][0]; }
        float4 x = make_float4(0.f, 0.f, 0.f, 0.f), z = x, x1 = x, z1 = x;
        if (nch > 0) { x = ldg_stream(A); z = ldg_stream(B); }
        if (nch > 1) { x1 = ldg_stream(A + 8); z1 = ldg_stream(B + 8); }
#pragma unroll 1
        for (int c = 0; c < nch; ++c) {
            float4 xn = x1, zn = z1;
            if (c + 2 < nch) { x1 = ldg_stream(A + (c + 2) * 8); z1 = ldg_stream(B + (c + 2) * 8); }
            float4 y = N[c * 8];
#pragma unroll
            for (int j = 0; j < NB; ++j) {
                float4 yn = y;
                if (j + 1 < NB) yn = N[(j + 1) * nstride + c * 8];
                acc[j][0].x = fmaf(x.x, y.x, acc[j][0].x); acc[j][0].y = fmaf(x.y, y.y, acc[j][0].y);
                acc[j][0].z = fmaf(x.z, y.z, acc[j][0].z); acc[j][0].w = fmaf(x.w, y.w, acc[j][0].w);
                acc[j][1].x = fmaf(z.x, y.x, acc[j][1].x); acc[j][1].y = fmaf(z.y, y.y, acc[j][1].y);
                acc[j][1].z = fmaf(z.z, y.z, acc[j][1].z); acc[j][1].w = fmaf(z.w, y.w, acc[j][1].w);
                y = yn;
            }
            x = xn; z = zn;
        }
        const float* rowa = P.items + (size_t)ra * ld;
        const float* rowb = P.items + (size_t)rb * ld;
        const float iha = (P.metric == DOT_PRODUCT) ? P.ih0[ra] : 0.f, ihb = (P.metric == DOT_PRODUCT) ? P.ih0[rb] : 0.f;
#pragma unroll
        for (int j = 0; j < NB; ++j) {
            float da = group8_hsum(acc[j][0]), db = group8_hsum(acc[j][1]);
            const float* nv = smN + (size_t)j * ld;
            for (uint32_t i = (uint32_t)nch * 32; i < d; ++i) {   // len % 32 tail: separately rounded mul, add
                da = __fadd_rn(da, __fmul_rn(rowa[i], nv[i]));
                db = __fadd_rn(db, __fmul_rn(rowb[i], nv[i]));
            }
            const int sa = side_of(margin_finish(P.metric, da, r_h0[j], iha)), sb = side_of(margin_finish(P.metric, db, r_h0[j], ihb));
            uint8_t* fl = P.flags + (size_t)(tb + j) * n;
            const bool leader = g8 == 0;
            if (leader && va) fl[pa] = (uint8_t)sa;
            if (leader && vb) fl[pb] = (uint8_t)sb;
            const unsigned la = __ballot_sync(0xffffffffu, leader && va && sa == 0), lb = __ballot_sync(0xffffffffu, leader && vb && sb == 0);
            if (lane == 0) { const int cn = __popc(la) + __popc(lb); if (cn) atomicAdd(&r_cnt[j], (uint32_t)cn); }
        }
        __syncthreads();
        if (tid < NB) (P.unit_left + (size_t)(tb + tid) * P.units_per_tree)[unit] = r_cnt[tid];
    }
}

__device__ __noinline__ void proot(const BuildParams& P, float* smN) {
    __shared__ uint32_t r_claim, r_ok;
    __shared__ uint32_t r_cnt[ROOT_TB];
    __shared__ float r_h0[ROOT_TB];
    const uint32_t T = P.n_trees, n = P.n, ld = P.ld;
    const int tid = threadIdx.x;
    if (tid == 0) {
        uint32_t ok = 1;
        while (ld_vol32(P.root_ready) < T) {
            if (*reinterpret_cast<volatile int32_t*>(P.error) != ERR_NONE || (P.abort != nullptr && *P.abort != 0)) { ok = 0; break; }
            __nanosleep(200);
        }
        r_ok = ok;
    }
    __syncthreads();
    if (!r_ok) return;
    __threadfence();
    const uint32_t units = (n + SCAN_UNIT - 1) / SCAN_UNIT;
    // claims are taken one ahead, so that the first unit of the next claim can be prefetched during the last unit of this one
    if (tid == 0) r_claim = atomicAdd(P.root_ticket, 1u);
    __syncthreads();
    uint32_t u0 = r_claim * ROOT_CHUNK;
    if (u0 < units) proot_prefetch(P, u0);
    for (;;) {
        if (u0 >= units) break;
        __syncthreads();
        if (tid == 0) r_claim = atomicAdd(P.root_ticket, 1u);
        __syncthreads();
        const uint32_t nu0 = r_claim * ROOT_CHUNK;
        const uint32_t u1 = min(units, u0 + ROOT_CHUNK);
        for (uint32_t tb = 0; tb < T; tb += ROOT_TB) {
            const int nb = (int)min((uint32_t)ROOT_TB, T - tb);
            __syncthreads();   // the previous batch's normals are no longer read
            {   // stage the batch's normals: all of a thread's loads are issued before the first store
                const uint32_t per = ld / 4u, total = (uint32_t)nb * per;   // float4 units
                for (uint32_t i0 = tid; i0 < total; i0 += 8u * CTRL_THREADS) {
                    float4 v[8];
#pragma unroll
                    for (int u = 0; u < 8; ++u) {
                        const uint32_t i = i0 + (uint32_t)u * CTRL_THREADS;
                        if (i < total) { const uint32_t j = i / per, e = i - j * per; v[u] = __ldcg(reinterpret_cast<const float4*>(P.cur_normal + (size_t)(tb + j) * P.pool_stride + NORMAL_HDR) + e); }
                    }
#pragma unroll
                    for (int u = 0; u < 8; ++u) { const uint32_t i = i0 + (uint32_t)u * CTRL_THREADS; if (i < total) reinterpret_cast<float4*>(smN)[i] = v[u]; }
                }
                if (tid < nb) r_h0[tid] = __ldcg(P.cur_normal + (size_t)(tb + tid) * P.pool_stride);
            }
            __syncthreads();
            switch (nb) {
                case 8: proot_units<8>(P, u0, u1, tb, nu0, smN, r_h0, r_cnt); break;
                case 7: proot_units<7>(P, u0, u1, tb, nu0, smN, r_h0, r_cnt); break;
                case 6: proot_units<6>(P, u0, u1, tb, nu0, smN, r_h0, r_cnt); break;
                case 5: proot_units<5>(P, u0, u1, tb, nu0, smN, r_h0, r_cnt); break;
                case 4: proot_units<4>(P, u0, u1, tb, nu0, smN, r_h0, r_cnt); break;
                case 3: proot_units<3>(P, u0, u1, tb, nu0, smN, r_h0, r_cnt); break;
                case 2: proot_units<2>(P, u0, u1, tb, nu0, smN, r_h0, r_cnt); break;
                default: proot_units<1>(P, u0, u1, tb, nu0, smN, r_h0, r_cnt); break;
            }
        }
        // report the claim to every tree
        __threadfence();
        __syncthreads();
        for (uint32_t t = tid; t < T; t += CTRL_THREADS) atomicAdd(&P.slots[t].done, (unsigned long long)(u1 - u0));
        u0 = nu0;
    }
}

// A worker CTA: claims units of whatever the control CTAs have published and runs the same scan / partition code as work_kernel.
// Returns when every tree is done (or on error). sm_normal: ld floats of dynamic shared memory.
__device__ __noinline__ void pworker(const BuildParams& P, float* sm_normal) {
    __shared__ uint32_t w_t, w_u0, w_n, w_seq, w_pseq, w_found, w_exit, w_count;
    __shared__ PSlot w_job;        // fields of the claimed job (first 64 bytes)
    __shared__ uint32_t w_sm[16];
    __shared__ uint32_t w_list[SCAN_UNIT * PLANES_CHUNK], w_list2[SCAN_UNIT * PLANES_CHUNK];   // positions stage 1 / stage 2 could not decide
    __shared__ uint32_t w_cnt[PLANES_CHUNK + 2];
    __shared__ PlanesScratch w_sc;
    __shared__ PlanesNormal w_pn;                           // the loaded normal's pre-filter factors (scan_claim_planes)
    uint8_t* sm_limbs = reinterpret_cast<uint8_t*>(sm_normal + P.ld);   // and its limbs
    const uint32_t T = P.n_trees;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const uint32_t rot = (blockIdx.x - T) * 7u;
    const bool latency_class = ((blockIdx.x - T) & LAT_MASK) == 0u;
    uint32_t loaded_t = 0xffffffffu, loaded_seq = 0xffffffffu;
    float nh0 = 0.f;
    if (tid == 0) w_exit = 0;
    if (P.root_fused) proot(P, sm_normal);
    for (;;) {
        // ---- poll: one load per slot, 32 slots per pass; pick a slot with unclaimed units ----
        if (warp == 0) {
            uint32_t found = 0;
            for (uint32_t base = 0; base < T && !found; base += 32) {
                const uint32_t k = base + lane;
                const uint32_t t = k < T ? (rot + k) % T : 0u;
                const unsigned long long tk = k < T ? ld_vol64(&P.slots[t].ticket) : 0ull;
                // Two classes of workers. One in four is a LATENCY worker: among the open jobs it takes the one with the fewest
                // groups (small nodes sit on their tree's critical path and must not queue behind a root scan). The others are
                // THROUGHPUT workers: they take the job with the most unclaimed groups, so the big scans keep (almost) all of the
                // bandwidth and a burst of small jobs does not turn into hundreds of failed claims.
                const bool open_job = k < T && pt_next(tk) < pt_total(tk);
                uint32_t key = !open_job ? 0xffffffffu : (latency_class ? pt_total(tk) : 0x00ffffffu - (pt_total(tk) - pt_next(tk)));
                uint32_t best = key;
#pragma unroll
                for (int o = 16; o > 0; o >>= 1) best = min(best, __shfl_xor_sync(0xffffffffu, best, o));
                if (best != 0xffffffffu) {
                    const unsigned m = __ballot_sync(0xffffffffu, key == best);
                    const int src = __ffs((int)m) - 1;
                    if (lane == src) { w_t = t; w_pseq = pt_seq(tk); }
                    found = 1;
                }
            }
            if (lane == 0) {
                w_found = found;
                if (!found) {
                    if (ld_vol32(P.active) == 0u || *reinterpret_cast<volatile int32_t*>(P.error) != ERR_NONE) w_exit = 1;
                    else __nanosleep(60);
                }
            }
        }
        __syncthreads();
        if (w_exit) return;
        if (!w_found) { __syncthreads(); continue; }
        // ---- claim; the job fields and (scan jobs) the normal are loaded while the atomic is in flight ----
        const uint32_t t = w_t;
        PSlot& sl = P.slots[t];
        const float* nsrc = P.cur_normal + (size_t)t * P.pool_stride;
        const bool want_normal = !(loaded_t == t && loaded_seq == w_pseq);
        float nreg[8];   // ld <= 8 * blockDim is guaranteed by the host for this schedule
#pragma unroll
        for (int u = 0; u < 8; ++u) nreg[u] = 0.f;
        if (want_normal) {
#pragma unroll
            for (int u = 0; u < 8; ++u) { const uint32_t i = tid + u * CTRL_THREADS; if (i < P.ld) nreg[u] = __ldcg(nsrc + NORMAL_HDR + i); }
        }
        if (tid == 0) {
            const unsigned long long r = atomicAdd(&sl.ticket, 1ull);   // a claim is one group of `chunk` units
            const uint4 f0 = __ldcg(reinterpret_cast<const uint4*>(&sl) + 1), f1 = __ldcg(reinterpret_cast<const uint4*>(&sl) + 2), f2 = __ldcg(reinterpret_cast<const uint4*>(&sl) + 3);
            uint4* wj = reinterpret_cast<uint4*>(&w_job);
            wj[1] = f0; wj[2] = f1; wj[3] = f2;
            w_seq = pt_seq(r);
            w_u0 = pt_next(r);
            w_n = pt_next(r) < pt_total(r) ? 1u : 0u;
        }
        __syncthreads();
        const uint32_t seq = w_seq, g0 = w_u0;
        const bool have = w_n != 0u;
        if (have && seq != w_pseq) {
            // The claim fell into a NEWER epoch than the polled one (this CTA raced with the publication of the tree's next job):
            // the group is real and must be processed — reload the fields and the normal of that epoch. (Its fields were complete
            // before its ticket was stored, and it cannot end while this claim is unreported.)
            if (tid == 0) { uint4* wj = reinterpret_cast<uint4*>(&w_job); wj[1] = __ldcg(reinterpret_cast<const uint4*>(&sl) + 1); wj[2] = __ldcg(reinterpret_cast<const uint4*>(&sl) + 2); wj[3] = __ldcg(reinterpret_cast<const uint4*>(&sl) + 3); }
#pragma unroll
            for (int u = 0; u < 8; ++u) { const uint32_t i = tid + u * CTRL_THREADS; if (i < P.ld) nreg[u] = __ldcg(nsrc + NORMAL_HDR + i); }
            __syncthreads();
        }
        if (have) {
            Job jb;
            jb.kind = (int)w_job.kind; jb.len = w_job.len; jb.rows = w_job.rows; jb.normal = nullptr; jb.flags = w_job.flags; jb.margins = nullptr;
            jb.unit_left = w_job.unit_left; jb.dst = w_job.dst; jb.total_left = w_job.total_left; jb.pad = 0;
            const uint32_t chunk = max(1u, w_job.chunk);
            if (jb.kind == JOB_SCAN) {
                const uint32_t units = (jb.len + SCAN_UNIT - 1) / SCAN_UNIT;
                if (want_normal || seq != w_pseq) {
                    double l1 = 0.0;
                    uint32_t mb = 0;
#pragma unroll
                    for (int u = 0; u < 8; ++u) {
                        const uint32_t i = tid + u * CTRL_THREADS;
                        if (i < P.ld) {
                            sm_normal[i] = nreg[u];
                            l1 += (double)fabsf(nreg[u]);
                            mb = max(mb, __float_as_uint(fabsf(nreg[u])));
                        }
                    }
                    if (P.planes.hi != nullptr) {
                        l1 = warp_sum_f64(l1);
                        mb = __reduce_max_sync(0xffffffffu, mb);
                        if (lane == 0) { w_sc.l1[warp] = l1; w_sc.mx[warp] = mb; }
                    }
                    nh0 = __ldcg(nsrc);
                    loaded_t = t; loaded_seq = seq;
                    __syncthreads();
                    if (P.planes.hi != nullptr && units > P.shadow_min_units) planes_job_factors(sm_normal, P.ld, P.d, sm_limbs, w_sc, &w_pn);
                }
                if (P.planes.hi != nullptr && units > P.shadow_min_units)
                    for (uint32_t u = g0 * chunk; u < min(units, (g0 + 1u) * chunk); u += PLANES_CHUNK)
                        scan_claim_planes(jb, u, min(min(units, (g0 + 1u) * chunk), u + PLANES_CHUNK), P.items, P.planes, P.ih0, P.d, P.ld, P.metric, sm_normal, sm_limbs,
                                          &w_pn, nh0, w_list, w_list2, w_cnt, P.shadow_stats);
                else
                    for (uint32_t u = g0 * chunk; u < min(units, (g0 + 1u) * chunk); ++u) scan_unit<true>(jb, u, P.items, P.ih0, P.d, P.ld, P.metric, sm_normal, nh0, &w_count);
            } else if (jb.kind == JOB_PARTITION) {
                const uint32_t units = (jb.len + PART_UNIT - 1) / PART_UNIT;
                for (uint32_t u = g0 * chunk; u < min(units, (g0 + 1u) * chunk); ++u)
                    partition_block(jb.rows, jb.flags, jb.dst, u * PART_UNIT, jb.len, __ldcg(jb.unit_left + u * (PART_UNIT / SCAN_UNIT)), jb.total_left, w_sm);
            }
            __threadfence();
            __syncthreads();
            if (tid == 0) atomicAdd(&sl.done, 1ull);
        }
        __syncthreads();
    }
}

// One tree per launch unit. CS = 1: one CTA; the scan of every attempt is a separate work_kernel
// launch. CS > 1 (thread-block cluster of CS CTAs, latency-bound regime: few trees per GPU): CTA 0
// of the cluster runs the state machine; a node of at most P.small_max rows is scanned right here
// by all CS CTAs between two cluster barriers (the job table, flags and unit counts live in global
// memory; barrier.cluster has release / acquire semantics), and the state machine goes on to the
// next attempt without leaving the kernel — no launch gap, no work_kernel start-up for the deep part
// of the tree, where the chain of attempts is the critical path. Bigger nodes leave through the
// posted job exactly as with CS = 1.
template <int CS>
__device__ __forceinline__ void cluster_scan_share(const BuildParams& P, const Job& jb, float* sm_normal, uint32_t* sm_count, unsigned rank) {
    for (uint32_t i = threadIdx.x; i < P.ld; i += blockDim.x) sm_normal[i] = jb.normal[NORMAL_HDR + i];
    const float nh0 = jb.normal[0];
    __syncthreads();
    const uint32_t units = (jb.len + SCAN_UNIT - 1) / SCAN_UNIT;
    for (uint32_t u = rank; u < units; u += CS) scan_unit(jb, u, P.items, P.ih0, P.d, P.ld, P.metric, sm_normal, nh0, sm_count);
}

// CS = 0: the PERSISTENT schedule. One launch per wave: CTAs [0, n_trees) each run one tree's state machine to the end, the other
// CTAs are workers (pworker). Nothing is launched per attempt: a control CTA publishes its scan (or wide partition) in its slot,
// the workers on all SMs claim units of it, the control CTA waits for their reports and goes on — the tree's state, its DFS
// frames and its ChaCha blocks never leave shared memory. All CTAs must be resident together (cooperative launch).
template <bool SMEM_WS, int CS, int METRIC>
__global__ void __launch_bounds__(CTRL_THREADS, (CS == 0 ? 2 : 1)) control_kernel(BuildParams P, uint32_t tree_base) {
    static_assert(CS <= 1 || SMEM_WS, "the cluster path keeps the normal in the shared-memory workspace");
    constexpr bool PERSIST = CS == 0;
    constexpr int CSD = CS < 1 ? 1 : CS;
    extern __shared__ __align__(16) unsigned char ctrl_smem[];
    if (PERSIST && blockIdx.x >= P.n_trees) { pworker(P, reinterpret_cast<float*>(ctrl_smem)); return; }
    __shared__ uint32_t s_scan_count;
    __shared__ TwoMeansShared TM;
    __shared__ uint32_t sm_tmp[CTRL_THREADS + 1];
    __shared__ uint32_t sm_w[2 * PART_BATCH * 8 + 2];
    __shared__ int s_action;
    __shared__ uint32_t s_total_left;
    __shared__ Rng s_rng;  // thread 0 only
    __shared__ uint32_t s_pref[8][16];   // eight ChaCha blocks of this tree's stream computed ahead (one per quad of warp 1)

    constexpr int SMF = 96;  // DFS frames cached in shared memory (deeper ones stay in global)
    __shared__ Frame sm_frames[SMF];
    __shared__ TreeState S;

    __shared__ int s_wait_ok;
    __shared__ uint32_t s_pseq;   // epoch of this tree's job slot (persistent schedule)
    const uint32_t t = blockIdx.x / CSD + tree_base;
    Job& job = P.jobs[t];
    unsigned crank = 0;
    if (CS > 1) crank = cooperative_groups::this_cluster().block_rank();
    if (CS > 1 && crank != 0) {
        // helper CTA: [A] wait for the leader's decision; scan a share; [B]; repeat until released
        float* sm_normal = reinterpret_cast<float*>(ctrl_smem);
        for (;;) {
            cooperative_groups::this_cluster().sync();
            const volatile Job* vj = &job;
            if (vj->pad != 1u) return;
            Job jb;
            jb.kind = JOB_SCAN; jb.len = vj->len; jb.rows = vj->rows; jb.normal = vj->normal; jb.flags = vj->flags; jb.margins = nullptr;
            jb.unit_left = vj->unit_left; jb.dst = nullptr; jb.total_left = 0; jb.pad = 1;
            cluster_scan_share<CS>(P, jb, sm_normal, &s_scan_count, crank);
            cooperative_groups::this_cluster().sync();
        }
    }
    // job.kind is already JOB_NONE and job.pad 0 for a finished tree / after an error
    if (P.st[t].phase == PH_DONE || *P.error != ERR_NONE) { if (CS > 1) cooperative_groups::this_cluster().sync(); return; }
    uint32_t inner = 0;
    Frame* gframes = P.frames + (size_t)t * MAX_DEPTH;
    if (threadIdx.x == 0) S = P.st[t];
    __syncthreads();
    for (int i = threadIdx.x; i <= S.sp && i < SMF; i += blockDim.x) sm_frames[i] = gframes[i];
    __syncthreads();
    auto FR = [&](int i) -> Frame& { return i < SMF ? sm_frames[i] : gframes[i]; };
    Record* recs = P.recs + (size_t)t * P.rec_cap;
    uint32_t* perm0 = P.perm[0] + (size_t)t * P.n;
    uint32_t* perm1 = P.perm[1] + (size_t)t * P.n;
    uint8_t* flags = P.flags + (size_t)t * P.n;
    uint32_t* unit_left = P.unit_left + (size_t)t * P.units_per_tree;
    const int tid = threadIdx.x;

    if (tid == 0) { s_rng.init(S.key, S.pos); job.kind = JOB_NONE; TM.mismatch = 0; s_pseq = 0; }
    uint32_t total_left = 0;
    if (S.phase == PH_AWAIT_SCAN) {
        const Frame f = FR(S.sp);
        total_left = cta_exclusive_scan(unit_left, (f.len + SCAN_UNIT - 1) / SCAN_UNIT, sm_tmp);
    }
    __syncthreads();

    uint64_t pref_base = ~0ull;   // block number held in s_pref[0] (every thread tracks the same value)
    for (;;) {
        // warp 1 keeps eight ChaCha blocks of this tree's stream computed ahead (four lanes per block, all eight quads at once)
        // while thread 0 walks the DFS; they are renewed when fewer than 64 words are left ahead of the stream position
        {
            const uint64_t blk0 = s_rng.pos >> 4;
            if (pref_base == ~0ull || blk0 < pref_base || blk0 >= pref_base + 4) {
                if ((tid >> 5) == 1) {
                    const int l = tid & 31, g = l >> 2;
                    uint32_t o[4];
                    chacha12_block_quad(S.key, blk0 + (uint64_t)g, o);
                    s_pref[g][l & 3] = o[0]; s_pref[g][4 + (l & 3)] = o[1]; s_pref[g][8 + (l & 3)] = o[2]; s_pref[g][12 + (l & 3)] = o[3];
                }
                pref_base = blk0;
            }
        }
        // ---- thread 0: advance the DFS until CTA-wide work is needed --------------------------
        if (tid == 0) {
            int action = ACT_NONE;
            if (S.phase == PH_START) {
                Frame r; r.start = 0; r.len = P.sub_off ? (uint32_t)(P.sub_off[t + 1] - P.sub_off[t]) : P.n; r.left_len = 0; r.left_id = 0; r.slot = NO_SLOT; r.parity = 0; r.stage = 0; r.pad = 0;
                FR(0) = r; S.sp = 0; S.phase = PH_AWAIT_PART;  // falls into the descend loop below
            } else if (S.phase == PH_AWAIT_SCAN) {
                Frame& f = FR(S.sp);
                const uint32_t left = total_left, right = f.len - total_left;
                S.scanned += f.len;
                const double imb = split_imbalance_dev(left, right);
                if (imb < 0.95 || S.attempts_left == 0) {            // src/writer.rs:1209-1213
                    if (imb > 0.99) { action = ACT_RANDOM; }         // :1220-1227
                    else {
                        f.slot = S.cur_slot; S.cur_slot = NO_SLOT;   // the normal is kept
                        f.left_len = left;
                        if (f.len <= INLINE_PART_MAX) action = ACT_PART_INLINE;
                        else {  // wide partition by all SMs (this step's work kernel / the workers)
                            job.kind = JOB_PARTITION; job.len = f.len;
                            job.rows = (f.parity ? perm1 : perm0) + f.start;
                            job.dst = (f.parity ? perm0 : perm1) + f.start;
                            job.flags = flags + f.start; job.unit_left = unit_left; job.total_left = left;
                            job.normal = nullptr; job.margins = nullptr;
                            if (PERSIST) action = ACT_PART_WIDE;
                            else { f.stage = 1; S.phase = PH_AWAIT_PART; action = ACT_EXIT; }
                        }
                    }
                } else { S.attempts_left -= 1; action = ACT_SPLIT; }  // :1215
            }
            if (action == ACT_NONE) {
                // descend: emit leaves, close finished splits, stop at the next node to split
                S.phase = PH_AWAIT_PART;
                bool have_ret = false; uint32_t ret = 0;
                for (;;) {
                    if (have_ret) {
                        if (S.sp < 0) { S.phase = PH_DONE; atomicSub(P.active, 1u); action = ACT_EXIT; break; }
                        Frame& par = FR(S.sp);
                        if (par.stage == 2) {          // left child finished -> open the right child
                            par.left_id = ret; par.stage = 3; have_ret = false;
                            if (S.sp + 1 >= MAX_DEPTH) { atomicExch(P.error, ERR_DEPTH); action = ACT_EXIT; break; }
                            Frame c; c.start = par.start + par.left_len; c.len = par.len - par.left_len; c.left_len = 0; c.left_id = 0;
                            c.slot = NO_SLOT; c.parity = par.parity ^ 1; c.stage = 0; c.pad = 0;
                            S.sp += 1; FR(S.sp) = c;
                        } else {                       // right child finished -> emit the split node (post-order)
                            if (S.n_recs >= P.rec_cap) { atomicExch(P.error, ERR_RECORDS); action = ACT_EXIT; break; }
                            Record rc; rc.kind = REC_SPLIT; rc.a = par.left_id; rc.b = ret; rc.c = par.slot;
                            recs[S.n_recs] = rc; ret = S.n_recs++; S.sp -= 1;
                        }
                        continue;
                    }
                    Frame& f = FR(S.sp);
                    if (f.stage == 0) {
                        if (f.len <= P.K) {            // fit_in_descendant — src/writer.rs:1184-1189
                            if (S.n_recs >= P.rec_cap) { atomicExch(P.error, ERR_RECORDS); action = ACT_EXIT; break; }
                            Record rc; rc.kind = REC_DESC; rc.a = f.start; rc.b = f.len; rc.c = f.parity;
                            recs[S.n_recs] = rc; ret = S.n_recs++; have_ret = true; S.sp -= 1;
                        } else { S.attempts_left = 3; action = ACT_SPLIT; break; }
                    } else {                           // stage 1: children are known -> open the left child
                        f.stage = 2;
                        if (S.sp + 1 >= MAX_DEPTH) { atomicExch(P.error, ERR_DEPTH); action = ACT_EXIT; break; }
                        Frame c; c.start = f.start; c.len = f.left_len; c.left_len = 0; c.left_id = 0;
                        c.slot = NO_SLOT; c.parity = f.parity ^ 1; c.stage = 0; c.pad = 0;
                        S.sp += 1; FR(S.sp) = c;
                    }
                }
            }
            if (action == ACT_SPLIT && S.cur_slot == NO_SLOT) {
                if (S.slot_next == S.slot_end) { S.slot_next = atomicAdd(P.pool_counter, 8u); S.slot_end = S.slot_next + 8u; }
                if (S.slot_next >= P.pool_cap) { atomicExch(P.error, ERR_POOL); action = ACT_EXIT; }
                else S.cur_slot = S.slot_next++;
            }
            s_action = action;
            s_total_left = total_left;
            s_rng.pref = &s_pref[0][0]; s_rng.pref_base = pref_base; s_rng.pref_n = 8;
        }
        __syncthreads();
        const int action = s_action;
        if (action == ACT_EXIT) break;
        const Frame f = FR(S.sp);
        const uint32_t* src = (f.parity ? perm1 : perm0) + f.start;
        uint32_t* dst = (f.parity ? perm0 : perm1) + f.start;
        if (action == ACT_SPLIT) {
            float* slot_ptr = P.pool + (size_t)S.cur_slot * P.pool_stride;
            float* mirror = PERSIST ? P.cur_normal + (size_t)t * P.pool_stride : nullptr;   // where the workers fetch the open job's normal
            if (SMEM_WS) create_split_cta<METRIC>(P, s_rng, src, f.len, reinterpret_cast<float*>(ctrl_smem), TM, slot_ptr, mirror);
            else create_split_cta<METRIC>(P, s_rng, src, f.len, P.scratch + (size_t)t * WS_VECS * P.ld, TM, slot_ptr, mirror);
            if (tid == 0) {
                if (TM.mismatch) { S.n_misspec += 1; TM.mismatch = 0; }
                S.n_splits_tried += 1;
                job.kind = JOB_SCAN; job.len = f.len; job.rows = src; job.normal = slot_ptr;
                job.flags = flags + f.start; job.margins = nullptr; job.unit_left = unit_left; job.dst = nullptr; job.total_left = 0;
                S.phase = PH_AWAIT_SCAN;
                if (CS > 1 && f.len <= P.small_max && inner < P.max_inner) job.pad = 1;
            }
            if (PERSIST) {
                // the normal (create_split also wrote it to the tree's fixed place, where workers fetch it while their claim is in
                // flight) and the job fields must be visible device-wide before the job opens
                __threadfence();
                __syncthreads();
                const uint32_t units = (f.len + SCAN_UNIT - 1) / SCAN_UNIT;
                if (tid == 0) {
                    s_pseq += 1;
                    if (P.root_fused && s_pseq == 1u && f.len == P.n) {
                        // the tree's first scan is its root's: the workers take it in their fused pass over all trees' roots
                        // (proot). The slot shows a job whose units are all claimed; each fused claim reports its units here.
                        volatile PSlot* v = &P.slots[t];
                        v->len = job.len; v->kind = (uint32_t)JOB_SCAN; v->chunk = 1u;
                        v->done = (unsigned long long)s_pseq << 32;
                        v->ticket = pticket(s_pseq, units, units);
                        __threadfence();
                        atomicAdd(P.root_ready, 1u);
                        s_wait_ok = pwait(P, P.slots[t], s_pseq, units) ? 1 : 0;
                    } else {
                    // a claim = `chunk` units: four for the big scans (and for everything that goes through the 8-bit planes)
                    const bool via_shadow = P.planes.hi != nullptr && units > P.shadow_min_units;
                    const uint32_t chunk = via_shadow ? (units > SHADOW_BIG_UNITS ? SHADOW_BIG_CHUNK : SHADOW_CHUNK) : (units > 1024u ? 4u : 1u), groups = (units + chunk - 1) / chunk;
                    ppublish(P.slots[t], job, s_pseq, groups, chunk);
                    s_wait_ok = pwait(P, P.slots[t], s_pseq, groups) ? 1 : 0;
                    }
                }
                __syncthreads();
                if (!s_wait_ok) break;
                total_left = cta_exclusive_scan(unit_left, units, sm_tmp);
                __syncthreads();
                continue;
            }
            if (CS > 1 && f.len <= P.small_max && inner < P.max_inner) {
                // cluster-resident attempt: scan here, then straight on to the decision
                cooperative_groups::this_cluster().sync();                       // [A] job visible to the helpers
                Job jb = job;
                cluster_scan_share<CS>(P, jb, reinterpret_cast<float*>(ctrl_smem) + (size_t)12 * P.ld, &s_scan_count, 0);
                cooperative_groups::this_cluster().sync();                       // [B] flags / unit counts visible to this CTA
                if (tid == 0) { job.kind = JOB_NONE; job.pad = 0; }
                total_left = cta_exclusive_scan(unit_left, (f.len + SCAN_UNIT - 1) / SCAN_UNIT, sm_tmp);
                ++inner;
                __syncthreads();
                continue;
            }
            break;
        }
        if (action == ACT_RANDOM) {
            // randomly_split_children — src/writer.rs:1310-1326: one gen::<bool>() per id, ascending;
            // bool = top bit of next_u32 (rand 0.8.5 Standard), true => Left
            const uint64_t pos0 = s_rng.pos;
            uint32_t cnt = 0;
            for (uint32_t i = tid; i < f.len; i += blockDim.x) {
                uint32_t blk[16];
                const uint64_t w = pos0 + i;
                chacha12_block(S.key, w >> 4, blk);
                const int left = (int)(blk[w & 15] >> 31);
                flags[f.start + i] = left ? 0 : 1;
                cnt += left;
            }
            sm_tmp[tid] = cnt;
            __syncthreads();
            if (tid == 0) {
                uint32_t tot = 0; for (int i = 0; i < blockDim.x; ++i) tot += sm_tmp[i];
                s_total_left = tot; s_rng.pos = pos0 + f.len; s_rng.blk_no = ~0ull;
                S.n_random += 1;
                FR(S.sp).slot = NO_SLOT; FR(S.sp).left_len = tot;
                if (S.cur_slot != NO_SLOT) { /* keep the reserved slot for the next split */ }
            }
            __syncthreads();
            partition_inline(src, flags + f.start, dst, f.len, s_total_left, sm_w);
            if (tid == 0) { FR(S.sp).stage = 1; S.phase = PH_AWAIT_PART; }
            total_left = 0;
            __syncthreads();
            continue;
        }
        if (PERSIST && action == ACT_PART_WIDE) {
            // the exclusive prefix of the unit counts (written by every thread above) feeds the workers' partition blocks
            __threadfence();
            __syncthreads();
            const uint32_t units = (f.len + PART_UNIT - 1) / PART_UNIT;
            if (tid == 0) { s_pseq += 1; const uint32_t groups = (units + 3u) / 4u; ppublish(P.slots[t], job, s_pseq, groups, 4u); s_wait_ok = pwait(P, P.slots[t], s_pseq, groups) ? 1 : 0; }
            __syncthreads();
            if (!s_wait_ok) break;
            if (tid == 0) { FR(S.sp).stage = 1; S.phase = PH_AWAIT_PART; }
            total_left = 0;
            __syncthreads();
            continue;
        }
        if (action == ACT_PART_INLINE) {
            // flags came from the scan; ids keep their ascending order on both sides (writer.rs:1201-1207)
            partition_inline(src, flags + f.start, dst, f.len, f.left_len, sm_w);
            if (tid == 0) { FR(S.sp).stage = 1; S.phase = PH_AWAIT_PART; }
            total_left = 0;
            __syncthreads();
            continue;
        }
    }
    __syncthreads();
    if (CS > 1) cooperative_groups::this_cluster().sync();   // releases the helpers (job.pad == 0)
    for (int i = tid; i <= S.sp && i < SMF; i += blockDim.x) gframes[i] = sm_frames[i];
    if (tid == 0) { S.pos = s_rng.pos; P.st[t] = S; }
}

// Merge the two ping-pong id buffers into `final_ids` following each leaf's parity.
__global__ void finalize_kernel(BuildParams P, uint32_t* __restrict__ final_ids) {
    const uint32_t t = blockIdx.y;
    const TreeState& S = P.st[t];
    const Record* recs = P.recs + (size_t)t * P.rec_cap;
    for (uint32_t r = blockIdx.x; r < S.n_recs; r += gridDim.x) {
        const Record rc = recs[r];
        if (rc.kind != REC_DESC) continue;
        const uint32_t* src = P.perm[rc.c & 1] + (size_t)t * P.n + rc.a;
        uint32_t* dst = final_ids + (size_t)t * P.n + rc.a;
        for (uint32_t i = threadIdx.x; i < rc.b; i += blockDim.x) dst[i] = src[i];
    }
}

__global__ void init_trees_kernel(BuildParams P, const uint32_t* __restrict__ keys /* n_trees x 8 */, const uint64_t* __restrict__ start_pos /* words already consumed, or NULL */) {
    const uint32_t t = blockIdx.x;
    if (threadIdx.x == 0) {
        TreeState s;
        for (int i = 0; i < 8; ++i) s.key[i] = keys[t * 8 + i];
        s.pos = start_pos ? start_pos[t] : 0; s.phase = PH_START; s.sp = -1; s.attempts_left = 0; s.cur_slot = NO_SLOT; s.n_recs = 0;
        s.n_splits_tried = 0; s.n_random = 0; s.n_misspec = 0; s.scanned = 0; s.slot_next = 0; s.slot_end = 0;
        P.st[t] = s;
        P.jobs[t].kind = JOB_NONE;
        P.jobs[t].pad = 0;
    }
    uint32_t* perm0 = P.perm[0] + (size_t)t * P.n;
    if (P.sub_off) {
        const uint64_t b = P.sub_off[t], len = P.sub_off[t + 1] - b;
        for (uint64_t i = threadIdx.x; i < len; i += blockDim.x) perm0[i] = P.sub_rows[b + i];
    } else {
        for (uint32_t i = threadIdx.x; i < P.n; i += blockDim.x) perm0[i] = i;
    }
}

}  // namespace ab
