// search.cuh — batched query path on the device (SURVEY.md §8f "next" #1).
//
// walk_kernel restates the candidate-collecting loop of Reader::nns_by_leaf
// (src/reader.rs:328-374): a max-heap of (OrderedFloat(dist), NodeId), pop the greatest, a
// Descendants node appends its items, a SplitPlaneNormal node pushes both children with
// D::pq_distance(dist, D::margin(normal, query), side) (src/distance/mod.rs:63-68). One warp per
// query: lane 0 owns the binary heap (global memory, per query), all 32 lanes compute the margin
// in the reference's exact summation order. Items are de-duplicated with a per-query bitmap while
// they are appended (the reference sorts + dedups afterwards, reader.rs:378-379; the *count* that
// stops the walk includes duplicates, as in the reference). The unique candidates are then sorted
// (CUB segmented sort) and go through distance_kernel + topk_kernel unchanged.
#pragma once
#include <cub/cub.cuh>

#include "kernels.cuh"

namespace ab {

struct DevForest {
    const uint8_t* kind;        // per node id: 0 = missing, 1 = Descendants, 2 = SplitPlaneNormal
    const uint32_t* left;
    const uint32_t* right;
    const uint32_t* normal_idx; // index into normals, 0xffffffff = "normal: none"
    const float* nh0;           // normal header 0 (bias / extra_dim)
    const uint32_t* desc_off;
    const uint32_t* desc_len;
    const float* normals;       // n_normals x ld
    const uint32_t* desc_rows;  // concatenated descendant lists, as ROW indices
    const uint32_t* roots;
    uint32_t n_roots, n_nodes;
    // the same per-node fields packed for the latency path (walk1_kernel): two 16-byte words per node
    //   [kind, left, right, normal_idx] [bits(nh0), desc_off, desc_len, 0]  — one round trip per pop, prefetchable at push time
    const uint4* rec;
    const uint32_t* node_of_normal;   // split node that owns normal ni
};

__global__ void forest_pack_kernel(DevForest F, uint4* __restrict__ rec, uint32_t* __restrict__ node_of_normal) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= F.n_nodes) return;
    const uint32_t k = F.kind[i], ni = F.normal_idx[i];
    rec[2 * (size_t)i] = make_uint4(k, F.left[i], F.right[i], ni);
    rec[2 * (size_t)i + 1] = make_uint4(__float_as_uint(F.nh0[i]), F.desc_off[i], F.desc_len[i], 0u);
    if (k == 2u && ni != 0xffffffffu) node_of_normal[ni] = i;
}

__device__ __forceinline__ float key_to_dist(uint32_t k) {  // inverse of ordered_key (canonical +0 / NaN)
    if (k == 0xffffffffu) return __uint_as_float(0x7fc00000u);
    uint32_t b = (k & 0x80000000u) ? (k & 0x7fffffffu) : ~k;
    return __uint_as_float(b);
}
__device__ __forceinline__ float f32_min_dev(float a, float b) {  // Rust f32::min: NaN loses
    if (a != a) return b;
    if (b != b) return a;
    return a < b ? a : b;
}

__device__ __forceinline__ void heap_push(unsigned long long* h, uint32_t& size, unsigned long long v) {
    uint32_t i = size++;
    while (i > 0) {
        uint32_t p = (i - 1) >> 1;
        unsigned long long pv = h[p];
        if (pv >= v) break;
        h[i] = pv;
        i = p;
    }
    h[i] = v;
}
__device__ __forceinline__ unsigned long long heap_pop(unsigned long long* h, uint32_t& size) {
    unsigned long long top = h[0];
    unsigned long long last = h[--size];
    uint32_t i = 0;
    for (;;) {
        uint32_t l = 2 * i + 1, r = l + 1;
        if (l >= size) break;
        unsigned long long lv = h[l];
        uint32_t c = l;
        unsigned long long cv = lv;
        if (r < size) { unsigned long long rv = h[r]; if (rv > lv) { c = r; cv = rv; } }
        if (cv <= last) break;
        h[i] = cv;
        i = c;
    }
    if (size > 0) h[i] = last;
    return top;
}

constexpr int WALK_WARPS = 8;
constexpr uint32_t WALK_SHEAP = 512;    // heap entries per query kept in shared memory (spills to the global heap beyond)
constexpr uint32_t NO_PARENT = 0xffffffffu;

// ---- filtered walks (QueryBuilder::candidates, reader.rs:350-357) -----------------------------------------------------
// One row filter is shared by every query of a call. The reference keeps only `descendants & candidates` of each popped
// Descendants node and stops once it holds search_k of those (duplicates included), so a walk adds fcount[node] to its stop
// count and appends only the filtered rows. It also never pushes a child whose live flag is 0: such a subtree holds no filtered
// row (and no missing node, whose ancestors load_forest pins live), so it adds nothing to the count or the candidates, and
// since every key is distinct (the node id is its low half) the remaining nodes pop in the reference's order.
struct WalkFilter {
    const uint32_t* bits;       // bit r set = row r passes
    const uint32_t* fcount;     // per Descendants node: |desc(node) & filter|
    const uint8_t* live;        // per node: its subtree holds a filtered row or a missing node
    uint32_t* pops;             // per query: nodes popped
    unsigned long long* spill;  // walk1_kernel: per query, frontier entries past the shared-memory slots (spill_cap each)
    uint32_t spill_cap;
    // MULTI walks (one filter per query, arroy_b200_search_batch_multi_filtered): query q reads bit qfilter[q] % 32 of the
    // summaries of group qfilter[q] / 32 (GroupSummaries) in place of bits / fcount / live
    const uint32_t* qfilter;
    const uint32_t* summary;
    unsigned long long group_words, live_off, count_off;
};

// The summaries of up to 32 filters (a group), group_words words per group in one buffer:
//   [0, n_rows)             row masks: bit b of word r = row r passes filter b of the group
//   [live_off, + n_nodes)   live masks: bit b = the node's subtree holds a row of filter b (or a missing node)
//   [count_off, + 32 n_nodes) fcount: word 32 node + b = |desc(node) & filter b| (Descendants nodes)
// One block per group keeps a walker's filter state at one pointer and one bit.
struct GroupSummaries {
    uint32_t* sum;
    unsigned long long group_words, live_off, count_off;
};

// ---- many filters per call: one summary pass per group of 32 ----------------------------------------------------------
// Each filter sets its bit in its group's row masks (one block row per filter of the call).
__global__ void multi_filter_mask_kernel(const uint32_t* __restrict__ rows, const uint64_t* __restrict__ offs, GroupSummaries G) {
    const uint32_t f = blockIdx.y;
    const uint64_t e = offs[f + 1];
    uint32_t* m = G.sum + (f >> 5) * G.group_words;
    const uint32_t bit = 1u << (f & 31);
    for (uint64_t i = offs[f] + (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < e; i += (uint64_t)gridDim.x * blockDim.x) atomicOr(&m[rows[i]], bit);
}

// live masks before the summary pass: all bits on pinned nodes (a missing node and its ancestors), or on every node when the
// forest is not tree-shaped (no pruning)
__global__ void multi_filter_live_init_kernel(const uint8_t* __restrict__ pin, uint32_t n_nodes, GroupSummaries G) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n_nodes) G.sum[blockIdx.y * G.group_words + G.live_off + i] = (!pin || pin[i]) ? 0xffffffffu : 0u;
}

// filter_count_kernel for the 32 filters of group blockIdx.y at once: one warp per Descendants node reads its rows' masks once;
// lane b ends with fcount of filter b, and the OR of the masks is ORed into the live masks of the node and its ancestors
// (`parent`: tree-shaped forests), stopping at the first that already holds those bits.
__global__ void multi_filter_count_kernel(DevForest F, GroupSummaries G, const uint8_t* __restrict__ reach, const uint32_t* __restrict__ parent,
                                          unsigned long long* __restrict__ ftotal) {
    const uint32_t node = (uint32_t)(((size_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5);
    const int lane = threadIdx.x & 31;
    const uint32_t g = blockIdx.y;
    if (node >= F.n_nodes || F.kind[node] != 1) return;
    uint32_t* gs = G.sum + g * G.group_words;
    const uint32_t* m = gs;
    const uint32_t off = F.desc_off[node], len = F.desc_len[node];
    uint32_t cnt = 0, any = 0;
    for (uint32_t i0 = 0; i0 < len; i0 += 32) {
        const uint32_t x = i0 + lane < len ? m[F.desc_rows[off + i0 + lane]] : 0u;
        uint32_t u = __reduce_or_sync(0xffffffffu, x);
        any |= u;
        for (; u; u &= u - 1) {   // only the filters present in these 32 rows
            const int b = __ffs((int)u) - 1;
            const unsigned v = __ballot_sync(0xffffffffu, (x >> b) & 1u);
            if (lane == b) cnt += __popc(v);
        }
    }
    gs[G.count_off + (size_t)node * 32 + lane] = cnt;
    if (cnt && reach[node]) atomicAdd(&ftotal[g * 32 + lane], (unsigned long long)cnt);
    if (lane == 0 && any && parent) {
        uint32_t* lv = gs + G.live_off;
        for (uint32_t x = node; x != NO_PARENT; x = parent[x]) if ((atomicOr(&lv[x], any) & any) == any) break;
    }
}

// The small-filter shortcut of a multi-filter call, one warp per query: the query's filter rows that some reachable leaf
// holds, already ascending (a compaction of the filter's row list).
__global__ void multi_filter_select_kernel(const uint32_t* __restrict__ rows, const uint64_t* __restrict__ offs, const uint32_t* __restrict__ qfilter,
                                           const uint32_t* __restrict__ inleaf, uint32_t nq, uint32_t* __restrict__ cand, uint32_t cand_cap,
                                           uint32_t* __restrict__ cand_count, int32_t* __restrict__ status) {
    const uint32_t q = (uint32_t)(((size_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5);
    const int lane = threadIdx.x & 31;
    if (q >= nq) return;
    const uint32_t f = qfilter[q];
    const uint64_t b = offs[f], e = offs[f + 1];
    uint32_t* out = cand + (size_t)q * cand_cap;
    uint32_t o = 0;
    int st = 0;
    for (uint64_t i0 = b; i0 < e; i0 += 32) {
        const uint64_t i = i0 + lane;
        uint32_t row = 0;
        bool keep = false;
        if (i < e) { row = rows[i]; keep = (inleaf[row >> 5] >> (row & 31)) & 1u; }
        const unsigned m = __ballot_sync(0xffffffffu, keep);
        if (keep) { const uint32_t p = o + __popc(m & ((1u << lane) - 1u)); if (p < cand_cap) out[p] = row; else st = 1; }
        o += __popc(m);
    }
    st = __reduce_max_sync(0xffffffffu, st);
    if (lane == 0) { cand_count[q] = o < cand_cap ? o : cand_cap; status[q] = st; }
}

// fcount for every Descendants node (one warp per node) and ftotal = their sum over the nodes reachable from the roots. With
// `parent` (a tree-shaped forest), a node with a filtered row flags itself and its ancestors live, stopping at the first one
// already flagged; without it the caller has set every flag.
__global__ void filter_count_kernel(DevForest F, const uint32_t* __restrict__ bits, const uint8_t* __restrict__ reach, const uint32_t* __restrict__ parent,
                                    uint32_t* __restrict__ fcount, volatile uint8_t* live, unsigned long long* __restrict__ ftotal) {
    const uint32_t node = (uint32_t)(((size_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5);
    const int lane = threadIdx.x & 31;
    if (node >= F.n_nodes || F.kind[node] != 1) return;
    const uint32_t off = F.desc_off[node], len = F.desc_len[node];
    uint32_t cnt = 0;
    for (uint32_t i = lane; i < len; i += 32) { const uint32_t row = F.desc_rows[off + i]; cnt += (bits[row >> 5] >> (row & 31)) & 1u; }
    cnt = __reduce_add_sync(0xffffffffu, cnt);
    if (lane != 0) return;
    fcount[node] = cnt;
    if (cnt == 0) return;
    if (reach[node]) atomicAdd(ftotal, (unsigned long long)cnt);
    if (parent) for (uint32_t x = node; x != NO_PARENT && !live[x]; x = parent[x]) live[x] = 1;
}

// bit r of `inleaf` = row r is a descendant of some reachable Descendants node (once per forest upload)
__global__ void forest_inleaf_kernel(DevForest F, const uint8_t* __restrict__ reach, uint32_t* __restrict__ inleaf) {
    const uint32_t node = (uint32_t)(((size_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5);
    const int lane = threadIdx.x & 31;
    if (node >= F.n_nodes || F.kind[node] != 1 || !reach[node]) return;
    const uint32_t off = F.desc_off[node], len = F.desc_len[node];
    for (uint32_t i = lane; i < len; i += 32) { const uint32_t row = F.desc_rows[off + i]; atomicOr(&inleaf[row >> 5], 1u << (row & 31)); }
}

// The small-filter shortcut: every filtered row of a reachable leaf, ascending, copied to each query's candidate segment.
__global__ void filter_select_count_kernel(const uint32_t* __restrict__ bits, const uint32_t* __restrict__ inleaf, uint32_t words, uint32_t* __restrict__ counts) {
    const uint32_t w = blockIdx.x * blockDim.x + threadIdx.x;
    if (w < words) counts[w] = __popc(bits[w] & inleaf[w]);
}
__global__ void filter_select_scatter_kernel(const uint32_t* __restrict__ bits, const uint32_t* __restrict__ inleaf, const uint32_t* __restrict__ offs, uint32_t words,
                                             uint32_t* __restrict__ cand, uint32_t cand_cap, uint32_t* __restrict__ cand_count, int32_t* __restrict__ status) {
    const uint32_t w = blockIdx.x * blockDim.x + threadIdx.x, q = blockIdx.y;
    if (w >= words) return;
    uint32_t m = bits[w] & inleaf[w], o = offs[w];
    uint32_t* out = cand + (size_t)q * cand_cap;
    for (; m; m &= m - 1) out[o++] = w * 32 + (uint32_t)(__ffs((int)m) - 1);
    if (w == words - 1) { cand_count[q] = o; status[q] = 0; }
}

// query q: vector = qrows ? items[qrows[q]] : queries[q] (ld floats); qh0 = extra_dim for DotProduct margins.
// FILTER: one filter for every query (Fl.bits / fcount / live); with MULTI, each query's own (Fl.qfilter, the group summaries).
template <bool FILTER, bool MULTI = false>
__global__ void __launch_bounds__(WALK_WARPS * 32)
walk_kernel(DevForest F, const float* __restrict__ items, uint32_t d, uint32_t ld, int metric, uint32_t nq,
            const uint32_t* __restrict__ qrows, const float* __restrict__ queries, const float* __restrict__ qh0,
            unsigned long long search_k, unsigned long long* __restrict__ heaps, uint32_t heap_cap,
            uint32_t* __restrict__ cand, uint32_t cand_cap, uint32_t* __restrict__ cand_count,
            uint32_t* __restrict__ bitmap, uint32_t bitmap_words, int32_t* __restrict__ status, WalkFilter Fl) {
    static_assert(FILTER || !MULTI, "MULTI is a filtered walk");
    const int lane = threadIdx.x & 31;
    const uint32_t q = blockIdx.x * WALK_WARPS + (threadIdx.x >> 5);
    if (q >= nq) return;
    const float* qv = qrows ? items + (size_t)qrows[q] * ld : queries + (size_t)q * ld;
    const float qhdr = qh0 ? qh0[q] : 0.f;
    // MULTI: this query's filter is bit fb of the group summaries at gs
    const uint32_t qf = MULTI ? Fl.qfilter[q] : 0u, fb = qf & 31u;
    const uint32_t* gs = MULTI ? Fl.summary + (qf >> 5) * Fl.group_words : nullptr;
    auto live = [&](uint32_t node) -> bool { return MULTI ? (gs[Fl.live_off + node] >> fb) & 1u : Fl.live[node]; };
    // The heap lives in shared memory (a walk pushes two entries per pop: a few hundred in practice) and moves to
    // its global-memory slot only if it outgrows WALK_SHEAP: every pop / push is a chain of dependent accesses.
    extern __shared__ unsigned long long walk_sheap[];
    unsigned long long* gheap = heaps + (size_t)q * heap_cap;
    unsigned long long* heap = walk_sheap + (size_t)(threadIdx.x >> 5) * WALK_SHEAP;
    uint32_t cap = WALK_SHEAP < heap_cap ? WALK_SHEAP : heap_cap;
    uint32_t* out = cand + (size_t)q * cand_cap;
    uint32_t* bm = bitmap + (size_t)q * bitmap_words;
    uint32_t size = 0;
    if (F.n_roots > cap) { heap = gheap; cap = heap_cap; }
    if (lane == 0) {
        const unsigned long long inf_key = (unsigned long long)ordered_key(__uint_as_float(0x7f800000u)) << 32;
        for (uint32_t r = 0; r < F.n_roots && size < cap; ++r) if (!FILTER || live(F.roots[r])) heap_push(heap, size, inf_key | F.roots[r]);
    }
    unsigned long long total = 0;   // nns.len() of the reference (duplicates included)
    uint32_t unique = 0, pops = 0;
    int st = 0;
    for (;;) {
        size = __shfl_sync(0xffffffffu, size, 0);
        if (total >= search_k || size == 0) break;
        unsigned long long top = 0;
        if (lane == 0) top = heap_pop(heap, size);
        top = __shfl_sync(0xffffffffu, top, 0);
        pops += 1;
        const uint32_t node = (uint32_t)top;
        const float dist = key_to_dist((uint32_t)(top >> 32));
        const int kind = node < F.n_nodes ? F.kind[node] : 0;
        if (kind == 1) {
            const uint32_t off = F.desc_off[node], len = F.desc_len[node];
            for (uint32_t i0 = 0; i0 < len; i0 += 32) {
                uint32_t i = i0 + lane;
                bool fresh = false;
                uint32_t row = 0;
                if (i < len) {
                    row = F.desc_rows[off + i];
                    uint32_t bit = 1u << (row & 31);
                    fresh = (!FILTER || (MULTI ? ((gs[row] >> fb) & 1u) : (Fl.bits[row >> 5] & bit))) && (atomicOr(&bm[row >> 5], bit) & bit) == 0;
                }
                unsigned m = __ballot_sync(0xffffffffu, fresh);
                if (fresh) {
                    uint32_t p = unique + __popc(m & ((1u << lane) - 1u));
                    if (p < cand_cap) out[p] = row; else st = 1;
                }
                unique += __popc(m);
            }
            total += FILTER ? (MULTI ? gs[Fl.count_off + (size_t)node * 32 + fb] : Fl.fcount[node]) : len;
        } else if (kind == 2) {
            const uint32_t ni = F.normal_idx[node];
            bool push_l = true, push_r = true;
            if (FILTER && lane == 0) { push_l = live(F.left[node]); push_r = live(F.right[node]); }
            float mg = 0.0f;
            if (ni != 0xffffffffu) {
                const float* nv = F.normals + (size_t)ni * ld;
                float dt = exact_warp<false>(nv, qv, (int)d);
                mg = margin_finish(metric, dt, F.nh0[node], qhdr);
            }
            // outgrown the shared-memory heap: move it (the array *is* the heap) to the global slot
            const int spill = __shfl_sync(0xffffffffu, (int)(size + 2 > cap && heap != gheap), 0);
            if (spill) {
                const uint32_t sz = __shfl_sync(0xffffffffu, size, 0);
                for (uint32_t i = lane; i < sz; i += 32) gheap[i] = heap[i];
                __syncwarp();
                heap = gheap; cap = heap_cap;
            }
            if (lane == 0) {
                if (size + 2 > cap) st = 2;
                else {
                    if (push_l) heap_push(heap, size, ((unsigned long long)ordered_key(f32_min_dev(-mg, dist)) << 32) | F.left[node]);
                    if (push_r) heap_push(heap, size, ((unsigned long long)ordered_key(f32_min_dev(mg, dist)) << 32) | F.right[node]);
                }
            }
        } else {
            st = 3;  // missing node (Error::MissingKey)
        }
        st = __reduce_max_sync(0xffffffffu, st);
        if (st) break;
    }
    if (lane == 0) { cand_count[q] = unique < cand_cap ? unique : cand_cap; status[q] = st; if (FILTER) Fl.pops[q] = pops; }
}

// offsets[q] = q * cand_cap (begin), ends[q] = begin + count — segment descriptors for the sort
__global__ void walk_segments_kernel(const uint32_t* __restrict__ cand_count, uint32_t nq, uint32_t cand_cap, uint64_t* __restrict__ begins, uint64_t* __restrict__ ends) {
    uint32_t q = blockIdx.x * blockDim.x + threadIdx.x;
    if (q < nq) { begins[q] = (uint64_t)q * cand_cap; ends[q] = (uint64_t)q * cand_cap + cand_count[q]; }
    if (q == nq) { begins[q] = (uint64_t)q * cand_cap; }
}

__global__ void gather_f32_kernel(float* __restrict__ dst, const float* __restrict__ src, const uint32_t* __restrict__ idx, uint32_t n) {
    uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) dst[i] = src[idx[i]];
}

}  // namespace ab

namespace ab {

// ---- few queries at a time: one CTA per query -------------------------------------------------------------------
// walk_kernel above is built for throughput (one WARP per query, thousands of queries per launch). A single
// Reader::nns_by_item / nns_by_vector call is a latency problem instead: the same priority-queue walk runs on warp 0 of a
// CTA with the query vector and the heap in shared memory, a Descendants node only costs the walker its length (the stop
// count includes duplicates, reader.rs:344-373) while the other seven warps copy its items into the candidate buffer, and the
// candidates are sorted + de-duplicated right here (bitonic sort in shared memory; reader.rs:378-379) instead of going
// through a per-query bitmap and a device-wide segmented sort. The re-rank then uses every SM (distance_kernel + topk_kernel).
constexpr int W1_THREADS = 256;
constexpr uint32_t W1_HEAP = 1024;     // heap entries in shared memory
constexpr uint32_t W1_CAND = 8192;     // candidate slots in shared memory (duplicates included)
constexpr uint32_t W1_LEAFQ = 128;     // Descendants nodes queued for the copier warps
constexpr uint32_t W1_LEAFQ_FILTER = 2048;   // a filtered walk publishes more, smaller leaves (only those with a filtered row)

template <uint32_t LEAFQ>
struct Walk1SharedT {
    unsigned long long heap[W1_HEAP];
    uint32_t cand[W1_CAND];
    volatile uint32_t lq_off[LEAFQ], lq_len[LEAFQ], lq_dst[LEAFQ];   // (volatile: read by the copier warps right after `produced`)
    uint32_t scan[W1_THREADS / 32];
    volatile uint32_t produced;
    volatile int done;
    uint32_t total;
    int status;
};
template <bool FILTER> using Walk1Shared = Walk1SharedT<FILTER ? W1_LEAFQ_FILTER : W1_LEAFQ>;
constexpr size_t W1_MAX_LD = 8192;
template <bool FILTER> inline size_t walk1_smem(uint32_t ld) { return sizeof(Walk1Shared<FILTER>) + (size_t)ld * 4 + 16; }

// dots[q][node] = the reference's dot of query q with the normal of split node `node`, for EVERY normal of the forest (one warp per pair, the same
// exact_warp the walker would call). A single query's walk is a chain of ~160 dependent pops, each of which would otherwise load
// a 3 KB normal and reduce it on one warp; reading the whole forest's normals once (C2: 313 MB = 50 us of HBM) turns every pop
// into a table lookup. Only worth it while the forest's normals are a few hundred MB (the caller decides).
__global__ void __launch_bounds__(256)
forest_dots_kernel(DevForest F, uint32_t n_normals, const float* __restrict__ items, uint32_t d, uint32_t ld,
                   const uint32_t* __restrict__ qrows, const float* __restrict__ queries, float* __restrict__ dots) {
    extern __shared__ __align__(16) float fd_q[];
    const uint32_t q = blockIdx.y;
    const float* qv = qrows ? items + (size_t)qrows[q] * ld : queries + (size_t)q * ld;
    for (uint32_t i = threadIdx.x; i < ld; i += blockDim.x) fd_q[i] = qv[i];
    __syncthreads();
    const uint32_t warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    for (uint32_t ni = blockIdx.x * 8u + warp; ni < n_normals; ni += gridDim.x * 8u) {
        const float dt = exact_warp<false>(F.normals + (size_t)ni * ld, fd_q, (int)d);
        if (lane == 0) dots[(size_t)q * F.n_nodes + F.node_of_normal[ni]] = dt;   // indexed by NODE: the walker can prefetch it when it pushes the node
    }
}

// FILTER: the frontier may outgrow the W1_HEAP shared-memory slots (a selective filter keeps the walk going through many more
// splits); entries past them continue the same unsorted array in the query's global spill slot, so the arg-max, and with it
// the pop order, is unchanged. MULTI: each query reads its own filter's bit, as in walk_kernel.
template <bool FILTER, bool MULTI = false>
__global__ void __launch_bounds__(W1_THREADS)
walk1_kernel(DevForest F, const float* __restrict__ items, uint32_t d, uint32_t ld, int metric, uint32_t nq,
             const uint32_t* __restrict__ qrows, const float* __restrict__ queries, const float* __restrict__ qh0,
             const float* __restrict__ pre_dots, uint32_t n_normals, int debug, unsigned long long search_k, uint32_t* __restrict__ out_cand, uint32_t cand_cap, uint32_t* __restrict__ out_count, int32_t* __restrict__ status,
             WalkFilter Fl) {
    extern __shared__ __align__(16) unsigned char w1_smem[];
    Walk1Shared<FILTER>& S = *reinterpret_cast<Walk1Shared<FILTER>*>(w1_smem);
    float* sq = reinterpret_cast<float*>(w1_smem + ((sizeof(Walk1Shared<FILTER>) + 15) & ~(size_t)15));
    constexpr uint32_t LEAFQ = FILTER ? W1_LEAFQ_FILTER : W1_LEAFQ;
    const uint32_t q = blockIdx.x;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const float* qv = qrows ? items + (size_t)qrows[q] * ld : queries + (size_t)q * ld;
    const float qhdr = qh0 ? qh0[q] : 0.f;
    static_assert(FILTER || !MULTI, "MULTI is a filtered walk");
    const uint32_t qf = MULTI ? Fl.qfilter[q] : 0u, fb = qf & 31u;
    const uint32_t* gs = MULTI ? Fl.summary + (qf >> 5) * Fl.group_words : nullptr;
    unsigned long long* spill = FILTER ? Fl.spill + (size_t)q * Fl.spill_cap : nullptr;
    const uint32_t hcap = FILTER ? W1_HEAP + Fl.spill_cap : W1_HEAP;
    auto hget = [&](uint32_t i) -> unsigned long long { return (!FILTER || i < W1_HEAP) ? S.heap[i] : spill[i - W1_HEAP]; };
    auto hset = [&](uint32_t i, unsigned long long v) { if (!FILTER || i < W1_HEAP) S.heap[i] = v; else spill[i - W1_HEAP] = v; };
    for (uint32_t i = tid; i < ld; i += W1_THREADS) sq[i] = qv[i];
    if (tid == 0) { S.produced = 0; S.done = 0; S.total = 0; S.status = 0; }
    __syncthreads();
    const long long dbg_t0 = clock64();
    uint32_t dbg_pops = 0, dbg_leaves = 0, dbg_front = 0;
    if (warp == 0) {
        uint32_t size = 0, produced = 0, total32 = 0;
        unsigned long long total = 0;
        int st = 0;
        if (lane == 0) {
            const unsigned long long inf_key = (unsigned long long)ordered_key(__uint_as_float(0x7f800000u)) << 32;
            uint32_t r = 0;
            for (; r < F.n_roots && size < hcap; ++r) if (!FILTER || (MULTI ? (gs[Fl.live_off + F.roots[r]] >> fb) & 1u : Fl.live[F.roots[r]])) hset(size++, inf_key | F.roots[r]);
            if (FILTER ? r < F.n_roots : F.n_roots > W1_HEAP) st = 2;
        }
        st = __shfl_sync(0xffffffffu, st, 0);
        // The priority queue is an UNSORTED array: a push appends (lane 0), a pop is a warp-wide arg-max over the <= 1024 entries
        // (every key is distinct — the node id is its low half — so the pop sequence is the BinaryHeap's of the reference whatever
        // the container). On one lane a binary heap costs ~1300 cycles per pop + two pushes; this is ~300.
        while (!st) {
            size = __shfl_sync(0xffffffffu, size, 0);
            if (total >= search_k || size == 0) break;
            __syncwarp();
            unsigned long long top = 0;
            uint32_t ti = 0xffffffffu;
            for (uint32_t i = lane; i < size; i += 32) { const unsigned long long v = hget(i); if (ti == 0xffffffffu || v > top) { top = v; ti = i; } }
            {   // warp arg-max of a 64-bit key in two REDUX steps: the high halves, then the low halves among the lanes that hold the
                // winning high half (a lane without an entry contributes 0 / loses the ballot)
                const uint32_t hi = ti != 0xffffffffu ? (uint32_t)(top >> 32) : 0u;
                const uint32_t mh = __reduce_max_sync(0xffffffffu, hi);
                const bool in = ti != 0xffffffffu && hi == mh;
                const uint32_t ml = __reduce_max_sync(0xffffffffu, in ? (uint32_t)top : 0u);
                const unsigned win = __ballot_sync(0xffffffffu, in && (uint32_t)top == ml);
                const int src = __ffs((int)win) - 1;
                ti = __shfl_sync(0xffffffffu, ti, src);
                top = ((unsigned long long)mh << 32) | ml;
            }
            if (lane == 0) { hset(ti, hget(size - 1)); size -= 1; }
            __syncwarp();
            dbg_pops += 1;
            const uint32_t node = (uint32_t)top;
            const float dist = key_to_dist((uint32_t)(top >> 32));
            uint4 r0 = make_uint4(0u, 0u, 0u, 0u), r1 = r0;
            if (node < F.n_nodes) { r0 = F.rec[2 * (size_t)node]; r1 = F.rec[2 * (size_t)node + 1]; }
            const int kind = (int)r0.x;
            if (kind == 1) {
                const uint32_t off = r1.y, len = r1.z;
                const uint32_t cnt = FILTER ? (MULTI ? gs[Fl.count_off + (size_t)node * 32 + fb] : Fl.fcount[node]) : len;   // slots this leaf fills
                if (total32 + cnt > W1_CAND || produced >= LEAFQ) { st = 1; break; }
                if (!FILTER || cnt) {
                    if (lane == 0) { S.lq_off[produced] = off; S.lq_len[produced] = len; S.lq_dst[produced] = total32; __threadfence_block(); S.produced = produced + 1; }
                    produced += 1;
                }
                total32 += cnt; total += cnt; dbg_leaves += 1;
            } else if (kind == 2) {
                const uint32_t ni = r0.w;
                const uint32_t lc = r0.y, rc = r0.z;
                // the children will be popped soon (one of them usually next): have their records and dots on the way
                uint32_t lv = 1;
                if (lane < 2) {
                    const uint32_t ch = lane == 0 ? lc : rc;
                    if (ch < F.n_nodes) {
                        asm volatile("prefetch.global.L1 [%0];" :: "l"(F.rec + 2 * (size_t)ch));
                        if (pre_dots) asm volatile("prefetch.global.L1 [%0];" :: "l"(pre_dots + (size_t)q * F.n_nodes + ch));
                        if (FILTER) { asm volatile("prefetch.global.L1 [%0];" :: "l"(MULTI ? gs + Fl.count_off + (size_t)ch * 32 + fb : Fl.fcount + ch)); lv = MULTI ? (gs[Fl.live_off + ch] >> fb) & 1u : Fl.live[ch]; }
                    }
                }
                float mg = 0.0f;
                if (ni != 0xffffffffu) {
                    const float* nv = F.normals + (size_t)ni * ld;
                    const float dt = pre_dots ? pre_dots[(size_t)q * F.n_nodes + node] : exact_warp<false>(nv, sq, (int)d);
                    mg = margin_finish(metric, dt, __uint_as_float(r1.x), qhdr);
                }
                const uint32_t live_r = FILTER ? __shfl_sync(0xffffffffu, lv, 1) : 1u;
                if (lane == 0) {
                    if (size + 2 > hcap) st = 2;
                    else {
                        if (!FILTER || lv) hset(size++, ((unsigned long long)ordered_key(f32_min_dev(-mg, dist)) << 32) | lc);
                        if (!FILTER || live_r) hset(size++, ((unsigned long long)ordered_key(f32_min_dev(mg, dist)) << 32) | rc);
                    }
                    if (FILTER) dbg_front = max(dbg_front, size);
                }
                st = __shfl_sync(0xffffffffu, st, 0);
            } else st = 3;
        }
        if (lane == 0) { S.total = total32; S.status = st; __threadfence_block(); S.done = 1; if (FILTER) Fl.pops[q] = dbg_pops; }
    } else if (FILTER) {
        // copier warps, filtered: the 32-row slices of all published leaves, numbered in publishing order, go round-robin to the
        // warps (so leaves of 32 rows or fewer spread over all of them); a warp appends the rows whose filter bit is set at the
        // leaf's cursor (lq_dst, bumped atomically), and reads `produced` / `done` once, through lane 0
        const uint32_t cw = warp - 1, ncw = W1_THREADS / 32 - 1;
        uint32_t e = 0, slice0 = 0;   // slice0: number of the first slice of leaf e
        for (;;) {
            int dn = 0;
            uint32_t p = 0;
            if (lane == 0) { dn = S.done; __threadfence_block(); p = S.produced; }
            dn = __shfl_sync(0xffffffffu, dn, 0);
            p = __shfl_sync(0xffffffffu, p, 0);
            if (e < p) {
                for (; e < p; ++e) {
                    const uint32_t off = S.lq_off[e], len = S.lq_len[e];
                    const uint32_t first = (cw + ncw - slice0 % ncw) % ncw;   // this warp's first slice of the leaf
                    slice0 += (len + 31) / 32;
                    for (uint32_t i0 = first * 32; i0 < len; i0 += ncw * 32) {
                        const uint32_t i = i0 + lane;
                        uint32_t row = 0;
                        bool pass = false;
                        if (i < len) { row = F.desc_rows[off + i]; pass = MULTI ? (gs[row] >> fb) & 1u : (Fl.bits[row >> 5] >> (row & 31)) & 1u; }
                        const unsigned m = __ballot_sync(0xffffffffu, pass);
                        uint32_t base = 0;
                        if (lane == 0 && m) base = atomicAdd(const_cast<uint32_t*>(&S.lq_dst[e]), (uint32_t)__popc(m));
                        base = __shfl_sync(0xffffffffu, base, 0);
                        if (pass) S.cand[base + __popc(m & ((1u << lane) - 1u))] = row;
                    }
                }
            } else if (dn) break;
            else __nanosleep(100);
        }
    } else {
        // copier warps: Descendants nodes as they are published
        const int t = tid - 32, nt = W1_THREADS - 32;
        uint32_t e = 0;
        for (;;) {
            const uint32_t p = S.produced;
            if (e < p) {
                const uint32_t off = S.lq_off[e], len = S.lq_len[e], dst = S.lq_dst[e];
                for (uint32_t i = t; i < len; i += nt) S.cand[dst + i] = F.desc_rows[off + i];
                ++e;
            } else if (S.done) { if (e >= S.produced) break; }
            else __nanosleep(100);
        }
    }
    __syncthreads();
    const long long dbg_t1 = clock64();
    const int st = S.status;
    const uint32_t n = S.total;
    if (st != 0 || n > cand_cap) { if (tid == 0) { status[q] = st ? st : 1; out_count[q] = 0; } return; }
    uint32_t m = 2;
    while (m < n) m <<= 1;
    for (uint32_t i = n + tid; i < m; i += W1_THREADS) S.cand[i] = 0xffffffffu;
    // bitonic sort, ascending (= ascending item ids)
    for (uint32_t size = 2; size <= m; size <<= 1) {
        for (uint32_t stride = size >> 1; stride > 0; stride >>= 1) {
            __syncthreads();
            for (uint32_t t = tid; t < (m >> 1); t += W1_THREADS) {
                const uint32_t i = 2 * t - (t & (stride - 1)), j = i + stride;
                const bool up = ((i & size) == 0);
                const uint32_t a = S.cand[i], b = S.cand[j];
                if ((a > b) == up) { S.cand[i] = b; S.cand[j] = a; }
            }
        }
    }
    __syncthreads();
    // unique + compaction (stable): every thread owns a contiguous slice
    const uint32_t per = (n + W1_THREADS - 1) / W1_THREADS;
    const uint32_t b0 = min(n, (uint32_t)tid * per), e0 = min(n, b0 + per);
    uint32_t cnt = 0;
    for (uint32_t i = b0; i < e0; ++i) cnt += (i == 0 || S.cand[i] != S.cand[i - 1]) ? 1u : 0u;
    uint32_t inc = cnt;
    for (int o = 1; o < 32; o <<= 1) { const uint32_t y = __shfl_up_sync(0xffffffffu, inc, o); if (lane >= o) inc += y; }
    if (lane == 31) S.scan[warp] = inc;
    __syncthreads();
    uint32_t base = 0, uniq = 0;
    for (int w = 0; w < W1_THREADS / 32; ++w) { const uint32_t y = S.scan[w]; if (w < warp) base += y; uniq += y; }
    uint32_t o = base + inc - cnt;
    uint32_t* out = out_cand + (size_t)q * cand_cap;
    for (uint32_t i = b0; i < e0; ++i) if (i == 0 || S.cand[i] != S.cand[i - 1]) out[o++] = S.cand[i];
    if (tid == 0) { out_count[q] = uniq; status[q] = 0; }
    if (debug && tid == 0) {
        if (FILTER) printf("[walk1] q %u: %u pops (%u leaves), largest frontier %u, walk %lld cycles, sort + unique %lld cycles, %u candidates (%u unique)\n", q, dbg_pops, dbg_leaves, dbg_front, dbg_t1 - dbg_t0, clock64() - dbg_t1, n, uniq);
        else printf("[walk1] q %u: %u pops (%u leaves), walk %lld cycles, sort + unique %lld cycles, %u candidates (%u unique)\n", q, dbg_pops, dbg_leaves, dbg_t1 - dbg_t0, clock64() - dbg_t1, n, uniq);
    }
}

}  // namespace ab
