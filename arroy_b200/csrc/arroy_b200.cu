// arroy_b200.cu — context, item staging, forest-build driver, re-rank and the extern "C"
// boundary declared in include/arroy_b200.h. Product code: there is no CPU fallback and no
// dependency on oracle/.
#include <cuda_runtime.h>

#include <algorithm>
#include <atomic>
#include <chrono>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <map>
#include <memory>
#include <mutex>
#include <stdexcept>
#include <string>
#include <thread>
#include <utility>
#include <vector>

#include "../../include/arroy_b200.h"
#include "build.cuh"
#include "search.cuh"
#include <cublas_v2.h>

#include "xrerank.cuh"
#include "tcgemm.cuh"
#include "frerank.cuh"
#include "restage.cuh"

using namespace ab;

namespace {

struct CudaError : std::runtime_error { using std::runtime_error::runtime_error; };
struct ArgError : std::runtime_error { using std::runtime_error::runtime_error; };
struct CapacityError : std::runtime_error { using std::runtime_error::runtime_error; };
struct Cancelled : std::runtime_error { using std::runtime_error::runtime_error; };
struct NotStaged : std::runtime_error { using std::runtime_error::runtime_error; };

#define CK(call)                                                                                      \
    do {                                                                                              \
        cudaError_t e_ = (call);                                                                      \
        if (e_ != cudaSuccess)                                                                        \
            throw CudaError(std::string(#call) + ": " + cudaGetErrorString(e_) + " (" __FILE__ ":" + \
                            std::to_string(__LINE__) + ")");                                          \
    } while (0)

// Live allocations of the owning types below, in the whole process (arroy_b200_allocations): device buffers and their bytes,
// pinned host buffers and their bytes, CUDA handles. Kept on the allocate and free paths only.
enum { LIVE_DEV, LIVE_DEV_BYTES, LIVE_PIN, LIVE_PIN_BYTES, LIVE_HANDLES, LIVE_N };
std::atomic<uint64_t> g_live[LIVE_N];
void live_add(int kind, size_t bytes) { g_live[kind].fetch_add(1, std::memory_order_relaxed); g_live[kind + 1].fetch_add(bytes, std::memory_order_relaxed); }
void live_sub(int kind, size_t bytes) { g_live[kind].fetch_sub(1, std::memory_order_relaxed); g_live[kind + 1].fetch_sub(bytes, std::memory_order_relaxed); }

// The buffers below free their memory when they are destroyed and are move-only. Destructors ignore return codes: a context may
// be destroyed at interpreter exit, after the CUDA runtime has begun unloading.
struct DevBuf {
    void* p = nullptr;
    size_t cap = 0;
    DevBuf() = default;
    DevBuf(DevBuf&& o) noexcept { *this = std::move(o); }
    DevBuf& operator=(DevBuf&& o) noexcept { if (this != &o) { release(); p = std::exchange(o.p, nullptr); cap = std::exchange(o.cap, 0); } return *this; }
    ~DevBuf() { release(); }
    void ensure(size_t bytes) {
        if (bytes <= cap) return;
        release();
        alloc(bytes + bytes / 4 + 256);
    }
    // exactly `bytes` (no slack, nothing larger kept): for the planes of host-placed items, which are most of what such an index
    // holds on the device
    void ensure_exact(size_t bytes) {
        if (bytes == cap) return;
        release();
        alloc(bytes);
    }
    void release() { if (p) { cudaFree(p); live_sub(LIVE_DEV, cap); } p = nullptr; cap = 0; }
    template <class T> T* as() { return static_cast<T*>(p); }
  private:
    void alloc(size_t bytes) { CK(cudaMalloc(&p, bytes)); cap = bytes; if (p) live_add(LIVE_DEV, cap); }
};
// Mapped pinned host memory that kernels address through `dev`: the f32 item matrix of a host-placed index, and the host result
// buffers the build kernels write (HostWave). Allocated to size; a buffer more than twice the size asked for is given back rather
// than kept pinned.
struct MappedBuf {
    void* p = nullptr;
    void* dev = nullptr;
    size_t cap = 0;
    MappedBuf() = default;
    MappedBuf(MappedBuf&& o) noexcept { *this = std::move(o); }
    MappedBuf& operator=(MappedBuf&& o) noexcept {
        if (this != &o) { release(); p = std::exchange(o.p, nullptr); dev = std::exchange(o.dev, nullptr); cap = std::exchange(o.cap, 0); }
        return *this;
    }
    ~MappedBuf() { release(); }
    void ensure(size_t bytes) {
        if (bytes <= cap && cap / 2 <= bytes) return;
        release();
        const cudaError_t e = cudaHostAlloc(&p, bytes, cudaHostAllocMapped | cudaHostAllocPortable);
        if (e != cudaSuccess) {
            p = nullptr;
            cudaGetLastError();
            throw CudaError("cudaHostAlloc of " + std::to_string(bytes) + " bytes of mapped pinned host memory failed: " + cudaGetErrorString(e));
        }
        cap = bytes;
        live_add(LIVE_PIN, cap);
        CK(cudaHostGetDevicePointer(&dev, p, 0));
    }
    void release() { if (p) { cudaFreeHost(p); live_sub(LIVE_PIN, cap); } p = nullptr; dev = nullptr; cap = 0; }
    template <class T> T* as() { return static_cast<T*>(p); }
};
struct PinBuf {
    void* p = nullptr;
    size_t cap = 0;
    PinBuf() = default;
    PinBuf(PinBuf&& o) noexcept { *this = std::move(o); }
    PinBuf& operator=(PinBuf&& o) noexcept { if (this != &o) { release(); p = std::exchange(o.p, nullptr); cap = std::exchange(o.cap, 0); } return *this; }
    ~PinBuf() { release(); }
    void ensure(size_t bytes) {
        if (bytes <= cap) return;
        release();
        CK(cudaMallocHost(&p, bytes));
        cap = bytes;
        live_add(LIVE_PIN, cap);
    }
    void release() { if (p) { cudaFreeHost(p); live_sub(LIVE_PIN, cap); } p = nullptr; cap = 0; }
    template <class T> T* as() { return static_cast<T*>(p); }
};

// A CUDA or cuBLAS handle that destroys itself. It converts to the raw handle, so it is passed to the API as one.
template <class T, auto Destroy>
struct Handle {
    T h = nullptr;
    Handle() = default;
    explicit Handle(T raw) : h(raw) { if (h) g_live[LIVE_HANDLES].fetch_add(1, std::memory_order_relaxed); }
    Handle(Handle&& o) noexcept { *this = std::move(o); }
    Handle& operator=(Handle&& o) noexcept { if (this != &o) { reset(); h = std::exchange(o.h, nullptr); } return *this; }
    ~Handle() { reset(); }
    operator T() const { return h; }
    void reset() { if (h) { Destroy(h); g_live[LIVE_HANDLES].fetch_sub(1, std::memory_order_relaxed); } h = nullptr; }
};
using Stream = Handle<cudaStream_t, cudaStreamDestroy>;
using Event = Handle<cudaEvent_t, cudaEventDestroy>;
using Graph = Handle<cudaGraph_t, cudaGraphDestroy>;
using GraphExec = Handle<cudaGraphExec_t, cudaGraphExecDestroy>;
using Blas = Handle<cublasHandle_t, cublasDestroy>;

Stream new_stream() { cudaStream_t s = nullptr; CK(cudaStreamCreateWithFlags(&s, cudaStreamNonBlocking)); return Stream(s); }
Event new_event(unsigned flags = cudaEventDefault) { cudaEvent_t e = nullptr; CK(cudaEventCreateWithFlags(&e, flags)); return Event(e); }

struct Wave {  // device buffers of one wave of trees; kept across builds
    DevBuf st, frames, recs, perm0, perm1, flags, unit_left, pool, pool_counter, jobs, scratch, active, error, keys, sub_rows, sub_off, slots, abort, cur_normal, start_pos, root, shadow_stats;
};
struct BuiltTreeView {  // views into the HostWave buffers of the context
    const void* recs = nullptr;
    uint32_t n_recs = 0;
    const uint32_t* final_rows = nullptr;  // n entries
    const float* pool = nullptr;
};
struct StageWorker {  // one H2D lane of the staging pipeline: own stream, two pinned bounce buffers
    Stream st;
    PinBuf pin[2];
    DevBuf dev[2];   // host placement: the device bounce buffers the chunk encoder reads
    Event ev[2];
};
// One wave's results in mapped pinned host memory, written by the control kernel while the wave builds (build.cuh
// export_records); kept across builds. Records of tree t start at t * rec_cap, its ids in final order at t * n.
struct HostWave {
    MappedBuf recs, final_rows, pool;
    uint64_t shape[5] = {0, 0, 0, 0, 0};   // (n, K, ld, trees, subsets) of the last build of this wave, the slot capacity of its
    uint32_t slots = 0, pool_used = 0;     // host pool and the slots it used (build_wave sizes the next pool from them)
};

}  // namespace

struct arroy_ctx {
    int device = 0;
    int sm_count = 132;
    Stream stream;   // declared first, destroyed last: ~arroy_ctx synchronises it and the other members free themselves
    std::mutex mu;
    std::string err;
    // staged items
    bool staged = false;
    int metric = 0;
    uint32_t dim = 0, ld = 0;   // dim = the vectors' length on the device (binary-quantized metrics: the padded bit count)
    uint32_t user_dim = 0;      // the index' dimensions (what normalized_distance of the binary-quantized metrics divides by)
    uint32_t row_bytes = 0;     // bytes per item row: 4 ld, binary-quantized metrics: the bit string (kernels.cuh bq_row_u4)
    uint64_t n = 0;
    DevBuf items, h0, h1, norms, maxbits;
    // host placement (arroy_b200_item_placement_plan): the f32 rows live in mapped pinned host memory, `items` is released and
    // the 8-bit planes are written at staging time
    bool host_items = false;
    MappedBuf host_rows;
    int32_t placed_metric = -1; uint32_t placed_dim = 0; uint64_t placed_n = 0;   // the last device-placed staging that asked
    std::vector<uint32_t> ids;
    // scratch
    DevBuf s_rows, s_flags, s_margins, s_normal, s_unit, s_job, s_keys, s_keys2, s_dists, s_q, s_qbits, s_qh0, s_off, s_orows, s_odist, s_olen, s_misc;
    PinBuf pin;
    Event ev0, ev1;
    Stream side_stream;   // host -> device flags while the persistent build kernel occupies `stream`
    Event ev_done, ev_p0, ev_p1;   // ev_p0 / ev_p1 bracket the persistent build kernel
    double stats[8] = {0, 0, 0, 0, 0, 0, 0, 0};
    uint64_t shadow_rows = 0, shadow_rescored = 0, shadow_stage2 = 0, fused_root_rows = 0, fused_root_read = 0;
    uint64_t wave_key[4] = {0, 0, 0, 0}, wave_max = 0, wave_trees_ok = 0; bool wave_key_valid = false;   // shapes of the last successful build (do_build_begin)   // last build: rows scanned through the bf16 shadow / re-scored from f32
    uint64_t n_launches = 0, h2d_bytes = 0, d2h_bytes = 0;  // since create (arroy_b200_counters)
    Event tev0, tev1;
    std::vector<StageWorker> stage_workers;
    bool staging_open = false;             // between arroy_b200_stage_begin and arroy_b200_stage_end
    std::vector<float> stage_h0, stage_h1;  // headers decoded from the leaf values staged so far
    uint64_t stage_stats[4] = {0, 0, 0, 0};  // the last arroy_b200_stage_items / _delta call (arroy_b200_stage_stats)
    // device-resident forest for the batched query path (arroy_b200_load_forest)
    DevBuf f_kind, f_left, f_right, f_nidx, f_nh0, f_doff, f_dlen, f_normals, f_desc, f_roots, f_rec, f_nofn;
    DevForest forest{};
    bool forest_loaded = false;
    uint32_t forest_max_desc = 0;
    uint64_t forest_n = 0;                       // the item count the loaded forest's rows were validated against
    uint64_t stage_epoch = 0, forest_epoch = 0;  // bumped by every (re)staging / forest upload: owners compare them (arroy_b200_epochs)
    DevBuf w_heaps, w_cand, w_cand2, w_count, w_bitmap, w_status, w_beg, w_end, w_qrows, w_tmp, w_pre;
    uint32_t f_n_normals = 0;
    // what filtered searches need from the forest (load_forest): parent per node (tree-shaped forests), nodes reachable from the
    // roots, nodes pinned live (a missing node and its ancestors), rows that some reachable leaf holds
    DevBuf f_parent, f_reach, f_pin, f_inleaf;
    bool f_tree = false;       // every reachable node has one parent: pruning by the live flags is exact
    bool f_complete = false;   // no reachable node is missing: the small-filter shortcut is exact
    // per-call scratch of filtered searches (arroy_b200_search_batch_filtered)
    DevBuf w_fbits, w_fcount, w_live, w_ftotal, w_pops, w_spill, w_scount, w_soff;
    uint64_t filter_stats[4] = {0, 0, 0, 0};   // arroy_b200_search_stats
    // per-call scratch of multi-filter searches (arroy_b200_search_batch_multi_filtered): the filters' row lists and offsets, the
    // group summaries (search.cuh GroupSummaries), each query's filter (w_ftotal / w_pops are shared with the one-filter path)
    DevBuf w_mrows, w_moffs, w_msum, w_mqf;
    uint64_t multi_stats[2] = {0, 0};          // arroy_b200_multi_filter_stats
    // results of the last build_trees_begin, waiting for build_trees_emit
    std::vector<std::vector<struct BuiltTreeView>> pending_waves;
    std::vector<uint32_t> pending_wave_t0;
    uint32_t pending_pool_stride = 0, pending_n_trees = 0;
    Wave wave;
    Graph cached_graph;
    GraphExec cached_exec;
    std::vector<uint8_t> cached_graph_key;  // BuildParams bytes + schedule the cached graph was captured for
    std::vector<HostWave> host_waves;
    double breakdown[8] = {0, 0, 0, 0, 0, 0, 0, 0};
    std::vector<Stream> tree_streams;   // one per tree of a wave (asynchronous per-tree chains)
    std::vector<Event> tree_events;     // join events, [0] = fork
    // tensor-core pre-filter of rerank_shared
    Blas blas;
    DevBuf x_gather, x_cnorm, x_ca, x_cb, x_gmax, x_qa, x_qb, x_twoe, x_qnorm, x_S, x_sel, x_beg, x_end, x_flag;
    DevBuf x_gh0, x_iota;   // host placement: the gathered candidates' headers and their positions for the exact dense path
    uint64_t xf_calls = 0, xf_fallbacks = 0, xf_selected = 0, xf_queries = 0;
    int tg_clusters = 0;   // tcgemm_tf32's resident clusters on this device, once measured
    Event xev[8];
    double xbreak[8] = {0, 0, 0, 0, 0, 0, 0, 0};
    double sbreak[8] = {0, 0, 0, 0, 0, 0, 0, 0};
    // fused re-rank with a bf16 shadow of the items (frerank.cuh); built lazily by the first query after staging
    DevBuf fr_shadow, fr_norm, fr_gmax, fr_status;
    bool fr_valid = false;
    bool shadow_valid = false;   // fr_shadow holds the bf16 copy of the staged items
    // the build's side() pre-filter (kernels.cuh scan_claim_planes): 8-bit planes + row scales of the staged items, built by the
    // first build after staging
    DevBuf pl_hi, pl_lo, pl_scale;
    bool planes_valid = false;
    // the plane pre-filter of host-placed items' re-rank (frerank_kernel<FR_PLANES>): device counters of candidates estimated
    // and survivors re-scored, allocated by the first such batch
    DevBuf pr_counts;
    uint64_t fr_batches[2] = {0, 0}, fr_fallbacks[2] = {0, 0};   // fused re-rank batches and fallbacks since create, per FrSource

    ~arroy_ctx() {
        cudaSetDevice(device);
        if (stream) cudaStreamSynchronize(stream);
    }
};

namespace {

int metric_header_floats(int m) { return m == DOT_PRODUCT ? 2 : 1; }

void set_device(arroy_ctx* c) { CK(cudaSetDevice(c->device)); }

void require_staged(arroy_ctx* c) { if (!c->staged) throw NotStaged("items have not been staged on this context"); }

// The f32 item matrix as kernels address it: device memory, or for host-placed items the device address of the mapped host rows.
// Kernels that read through it take ordinary loads; TMA and cp.async are only given device copies (xf_candidates).
const float* items_f32(arroy_ctx* c) { return c->host_items ? static_cast<const float*>(c->host_rows.dev) : c->items.as<float>(); }

// Indexes whose f32 rows may live in host memory: float metrics whose rows the 8-bit planes encode (kernels.cuh PLANES_MAX_D).
bool host_placement_eligible(int metric, uint32_t dim) { return metric >= EUCLIDEAN && metric <= MANHATTAN && dim >= 64 && dim <= PLANES_MAX_D; }

// Device bytes of a device-placed index and one tree of its build: f32 rows, both planes, scales, headers, and the wave buffers
// do_build_begin sizes one tree with (split_after = dim).
uint64_t device_placement_bytes(uint32_t dim, uint64_t n) {
    const uint64_t ld = (dim + 31u) & ~31u;
    const uint64_t leaves_est = n / std::max<uint32_t>(dim, 1) + 1;
    const uint64_t per_tree = n * (4 + 4 + 1) + (n / SCAN_UNIT + 1) * 4 + sizeof(Frame) * (uint64_t)MAX_DEPTH + 16ull * 8 * leaves_est +
                              4ull * (ld + NORMAL_HDR) * 4 * leaves_est + 4096;
    return n * ld * 4 + 2 * n * ld + 4 * n + 8 * n + per_tree;
}

uint32_t placement_plan(int32_t metric, uint32_t dim, uint64_t n, uint64_t free_bytes) {
    if (!host_placement_eligible(metric, dim)) return 0;
    return (double)device_placement_bytes(dim, n) <= (double)free_bytes * 0.7 ? 0u : 1u;
}

bool host_items_forced() { const char* e = getenv("ARROY_B200_HOST_ITEMS"); return e != nullptr && atoi(e) == 1; }

// Lets kernel `fn` take `bytes` of dynamic shared memory on `device` (the current device) where that is above the 48 KB any kernel
// may take. The limit belongs to the kernel on one device, whichever context set it, so it is only ever raised: a launch that asks
// for less must not take away what another launch still needs. One table for the process, read and set under one lock.
void raise_smem_limit(int device, const void* fn, size_t bytes) {
    if (bytes <= 48 * 1024) return;
    static std::mutex mu;
    static std::map<std::pair<int, const void*>, size_t> limits;
    std::lock_guard<std::mutex> lk(mu);
    size_t& limit = limits[{device, fn}];
    if (bytes <= limit) return;
    CK(cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes));
    limit = bytes;
}

PlaneRows plane_rows(arroy_ctx* c) { return PlaneRows{c->pl_hi.as<int8_t>(), c->pl_lo.as<int8_t>(), c->pl_scale.as<float>()}; }

// A side() scan through the 8-bit planes: jobs of more than min_units units go through them, their stage counts to stats (or null).
struct ScanPlanes { uint32_t min_units; unsigned long long* stats; };

// The dynamic shared memory of a side() scan over njobs jobs, its kernel's limit raised to it: the normal, the jobs' unit-prefix
// table and, through the planes, the normal's limbs.
size_t scan_smem(arroy_ctx* c, int njobs, bool planes) {
    const size_t smem = (size_t)c->ld * 4 + (size_t)(njobs + 1) * 4 + 16 + (planes ? (size_t)PLANES_LIMBS * c->ld : 0);
    raise_smem_limit(c->device, planes ? (const void*)work_kernel_planes : is_bq(c->metric) ? (const void*)work_kernel<true> : (const void*)work_kernel<false>, smem);
    return smem;
}

// A side() scan of the staged items over njobs jobs on `grid` CTAs: work_kernel (binary-quantized metrics: on the bit strings), or
// with `pl` work_kernel_planes. Once the limit is raised, the launch is its only CUDA call (build_wave captures it in a graph);
// the caller checks and counts it.
void launch_scan(arroy_ctx* c, cudaStream_t s, const Job* jobs, int njobs, unsigned grid, const ScanPlanes* pl) {
    const size_t smem = scan_smem(c, njobs, pl != nullptr);
    const float *items = items_f32(c), *ih0 = c->h0.as<float>();
    if (pl) work_kernel_planes<<<grid, WORK_THREADS, smem, s>>>(jobs, njobs, items, plane_rows(c), ih0, c->dim, c->ld, c->metric, pl->min_units, pl->stats);
    else if (is_bq(c->metric)) work_kernel<true><<<grid, WORK_THREADS, smem, s>>>(jobs, njobs, items, ih0, c->dim, c->ld, c->metric);
    else work_kernel<false><<<grid, WORK_THREADS, smem, s>>>(jobs, njobs, items, ih0, c->dim, c->ld, c->metric);
}

// norms_kernel over n rows of d = c->dim in a matrix of pitch c->ld (one 8-lane group per row); max_bits: their atomic max, or null
void launch_norms(arroy_ctx* c, const float* rows, uint64_t n, float* out, uint32_t* max_bits) {
    const uint64_t warps = (n + 3) / 4;
    const int grid = (int)std::max<uint64_t>(1, std::min<uint64_t>((warps + 7) / 8, (uint64_t)c->sm_count * 16));
    norms_kernel<<<grid, 256, 0, c->stream>>>(rows, n, c->dim, c->ld, out, max_bits);
    CK(cudaGetLastError());
}

void compute_norms(arroy_ctx* c, bool with_max) {
    c->norms.ensure(c->n * 4);
    c->maxbits.ensure(4);
    if (with_max) CK(cudaMemsetAsync(c->maxbits.p, 0, 4, c->stream));
    launch_norms(c, items_f32(c), c->n, c->norms.as<float>(), with_max ? c->maxbits.as<uint32_t>() : nullptr);
    c->n_launches += 1;
}

// A (re)staging forgets everything derived from the previous items: the bf16 shadow, the 8-bit planes and the device forest (its
// descendant rows were validated against the previous item count). Their buffers are kept for reuse. Stage epochs are unique in
// the process, not per context: an owner that remembers (context, epoch) is not fooled by a new context that was created at the
// address of a destroyed one.
void forget_staged(arroy_ctx* c) {
    static std::atomic<uint64_t> last_epoch{0};
    c->staged = false; c->fr_valid = false; c->shadow_valid = false; c->planes_valid = false; c->forest_loaded = false; c->staging_open = false;
    c->stage_epoch = ++last_epoch;
}

// Where the f32 rows of a staging go (may_host: the staging calls that can write host-placed rows, arroy_b200_stage_items and
// _flat). The plan sees the free device memory plus what this context already holds for items, their derived copies and the wave
// buffers, since the staging replaces or reuses all of it. A staging with the shapes of the last device-placed one that asked
// takes its answer again: cudaMemGetInfo is a driver round trip of up to tens of milliseconds.
bool choose_host_placement(arroy_ctx* c, int metric, uint32_t dim, uint64_t n, bool may_host) {
    if (!may_host || n == 0 || !host_placement_eligible(metric, dim)) return false;
    if (host_items_forced()) return true;
    if (c->placed_metric == metric && c->placed_dim == dim && c->placed_n == n) return false;
    size_t free_b = 0, total_b = 0;
    CK(cudaMemGetInfo(&free_b, &total_b));
    const Wave& W = c->wave;
    const uint64_t held = c->items.cap + c->pl_hi.cap + c->pl_lo.cap + c->pl_scale.cap + c->fr_shadow.cap + c->fr_norm.cap + W.perm0.cap + W.perm1.cap +
                          W.flags.cap + W.pool.cap + W.recs.cap;
    if (placement_plan(metric, dim, n, (uint64_t)free_b + held) == 1) return true;
    c->placed_metric = metric; c->placed_dim = dim; c->placed_n = n;
    return false;
}

void alloc_items(arroy_ctx* c, int metric, uint32_t dim, uint64_t n, const uint32_t* ids, bool may_host = false) {
    if (metric < 0 || metric > BQ_MANHATTAN) throw ArgError("unknown metric");
    if (dim == 0) throw ArgError("dim must be > 0");
    c->staged = false;
    const bool host = choose_host_placement(c, metric, dim, n, may_host);
    c->user_dim = dim;
    if (is_bq(metric)) dim = (dim + 63u) / 64u * 64u;   // the bit string's length (binary_quantized.rs:80-92)
    if (n > 0xffffffffull) throw ArgError("too many items");
    for (uint64_t i = 1; i < n; ++i) if (ids[i] <= ids[i - 1]) throw ArgError("ids must be strictly ascending");
    forget_staged(c);
    c->metric = metric; c->dim = dim; c->ld = (dim + 31u) & ~31u; c->n = n;
    c->row_bytes = is_bq(metric) ? 16u * bq_row_u4(dim) : 4u * c->ld;
    c->ids.assign(ids, ids + n);
    c->host_items = host;
    if (host) {   // the device keeps the planes and scales (written by the staging), no f32 rows and no bf16 shadow
        CK(cudaStreamSynchronize(c->stream));
        c->items.release(); c->fr_shadow.release(); c->fr_norm.release();
        c->host_rows.ensure((size_t)n * c->row_bytes);
        c->pl_hi.ensure_exact((size_t)n * c->ld);
        c->pl_lo.ensure_exact((size_t)n * c->ld);
        c->pl_scale.ensure_exact((size_t)n * 4);
    } else {
        c->host_rows.release();
        c->items.ensure(std::max<size_t>(16, (size_t)n * c->row_bytes));
    }
    c->h0.ensure(std::max<size_t>(16, n * 4));
    c->h1.ensure(std::max<size_t>(16, n * 4));
    CK(cudaMemsetAsync(c->h0.p, 0, std::max<size_t>(16, n * 4), c->stream));
    CK(cudaMemsetAsync(c->h1.p, 0, std::max<size_t>(16, n * 4), c->stream));
}

// headers as Writer::add_item stores them: D::new_header(vector) (src/writer.rs:388-390)
void default_headers(arroy_ctx* c) {
    if (c->metric == BQ_COSINE && c->n > 0) {   // sqrt(dot(v, v)) of a +-1 vector: sqrt(dim), dim exact in f32
        const float h = sqrtf((float)c->dim);
        uint32_t bits;
        memcpy(&bits, &h, 4);
        fill_u32_kernel<<<(unsigned)std::min<uint64_t>((c->n + 255) / 256, (uint64_t)c->sm_count * 8), 256, 0, c->stream>>>(c->h0.as<uint32_t>(), c->n, bits);
        CK(cudaGetLastError());
        c->n_launches += 1;
    } else if (c->metric == COSINE && c->n > 0) {
        compute_norms(c, false);
        CK(cudaMemcpyAsync(c->h0.p, c->norms.p, c->n * 4, cudaMemcpyDeviceToDevice, c->stream));
    }
}

// Staging pipeline: W host threads, each decoding row chunks into its own pinned bounce buffers and
// issuing its own cudaMemcpyAsync on its own stream, so decode (host memcpy of unaligned values)
// and PCIe transfers of different chunks overlap. Rows of row_bytes bytes, zero padded.
// mode 0: row_src(i) = dim f32 (byte aligned only); mode 1 (binary quantized): row_src(i) = src_dim f32 to be quantized to a
// bit string (is_sign_positive); mode 2 (binary quantized): row_src(i) = the stored bit string (dim / 8 bytes), copied.
// Host placement (c->host_items, mode 0): the rows are decoded straight into the mapped host matrix, each chunk is copied into a
// device bounce buffer of its lane and planes_encode_chunk_kernel writes its planes and scales there (and its norms into
// `norms`, when given), on the lane's stream: the rows cross PCIe once and the planes are complete when the pipeline returns.
template <class RowSrc>
void stage_rows_pipeline(arroy_ctx* c, uint64_t n, uint32_t dim, uint32_t row_bytes, RowSrc row_src, uint8_t* dst_override = nullptr, size_t chunk_mb_override = 0, bool count_bytes = true,
                         int mode = 0, uint32_t src_dim = 0, float* norms = nullptr) {
    if (n == 0) return;
    // 8 lanes x 4 MB chunks: decode of one chunk overlaps the PCIe copies of the others
    unsigned W = std::min(8u, std::max(1u, std::thread::hardware_concurrency()));
    const size_t chunk_mb = chunk_mb_override ? chunk_mb_override : 4;
    const uint64_t chunk_rows = std::max<uint64_t>(1, (chunk_mb << 20) / row_bytes);
    const uint64_t n_chunks = (n + chunk_rows - 1) / chunk_rows;
    W = (unsigned)std::min<uint64_t>(W, n_chunks);
    const bool host = c->host_items && !dst_override;
    if (c->stage_workers.size() < W) c->stage_workers.resize(W);
    for (unsigned w = 0; w < W; ++w) {
        StageWorker& sw = c->stage_workers[w];
        if (!sw.st) sw.st = new_stream();
        for (int k = 0; k < 2; ++k) {
            if (host) sw.dev[k].ensure(chunk_rows * row_bytes);
            else sw.pin[k].ensure(chunk_rows * row_bytes);
            if (!sw.ev[k]) sw.ev[k] = new_event(cudaEventDisableTiming);
        }
    }
    CK(cudaStreamSynchronize(c->stream));  // the destination buffer must not be in use
    std::mutex emu;
    std::string err;
    uint8_t* dst = dst_override ? dst_override : host ? static_cast<uint8_t*>(c->host_rows.p) : c->items.as<uint8_t>();
    const unsigned enc_grid = (unsigned)std::max<uint64_t>(1, std::min<uint64_t>((chunk_rows + 31) / 32, (uint64_t)c->sm_count * 4));
    auto worker = [&](unsigned w) {
        try {
            CK(cudaSetDevice(c->device));
            StageWorker& sw = c->stage_workers[w];
            bool used[2] = {false, false};
            int k = 0;
            for (uint64_t ch = w; ch < n_chunks; ch += W, k ^= 1) {
                const uint64_t r0 = ch * chunk_rows, rows = std::min<uint64_t>(chunk_rows, n - r0);
                if (used[k] && !host) CK(cudaEventSynchronize(sw.ev[k]));
                uint8_t* b = host ? dst + r0 * row_bytes : sw.pin[k].as<uint8_t>();
                for (uint64_t i = 0; i < rows; ++i) {
                    uint8_t* o = b + i * row_bytes;
                    const size_t used = mode == 0 ? 4ull * dim : dim / 8;
                    if (mode == 0) memcpy(o, row_src(r0 + i), used);
                    else if (mode == 1) {   // little-endian words: bit t of the string is bit t & 7 of byte t >> 3
                        const uint8_t* sp = row_src(r0 + i);
                        memset(o, 0, used);
                        for (uint32_t t = 0; t < src_dim; ++t) { uint32_t bits; memcpy(&bits, sp + 4ull * t, 4); if (!(bits >> 31)) o[t >> 3] |= (uint8_t)(1u << (t & 7)); }
                    } else memcpy(o, row_src(r0 + i), used);
                    memset(o + used, 0, row_bytes - used);
                }
                if (host) {   // (the bounce buffer's previous chunk was encoded by an earlier launch on this stream)
                    CK(cudaMemcpyAsync(sw.dev[k].p, b, rows * row_bytes, cudaMemcpyHostToDevice, sw.st));
                    planes_encode_chunk_kernel<<<enc_grid, 256, 0, sw.st>>>(sw.dev[k].as<float>(), rows, dim, c->ld, c->pl_hi.as<int8_t>() + r0 * c->ld,
                                                                           c->pl_lo.as<int8_t>() + r0 * c->ld, c->pl_scale.as<float>() + r0, norms ? norms + r0 : nullptr);
                    CK(cudaGetLastError());
                } else CK(cudaMemcpyAsync(dst + r0 * row_bytes, b, rows * row_bytes, cudaMemcpyHostToDevice, sw.st));
                CK(cudaEventRecord(sw.ev[k], sw.st));
                used[k] = true;
            }
            CK(cudaStreamSynchronize(sw.st));
        } catch (const std::exception& e) { std::lock_guard<std::mutex> lk(emu); if (err.empty()) err = e.what(); }
    };
    if (W == 1) worker(0);
    else { std::vector<std::thread> th; for (unsigned w = 0; w < W; ++w) th.emplace_back(worker, w); for (auto& x : th) x.join(); }
    if (!err.empty()) throw CudaError(err);
    if (count_bytes) c->h2d_bytes += n * (uint64_t)row_bytes;
    if (host) { c->n_launches += n_chunks; c->planes_valid = true; }
}

// ---- RoaringBitmap::serialize_into (roaring 0.10.9, portable format, no run containers) ------
void roaring_serialize(const uint32_t* ids, size_t n, std::vector<uint8_t>& out) {
    struct C { uint16_t key; size_t b, e; };
    std::vector<C> cs;
    for (size_t i = 0; i < n;) {
        uint16_t key = (uint16_t)(ids[i] >> 16);
        size_t j = i + 1;
        while (j < n && (uint16_t)(ids[j] >> 16) == key) ++j;
        cs.push_back({key, i, j});
        i = j;
    }
    size_t header = 8 + 8 * cs.size();
    size_t total = header;
    for (auto& c : cs) total += (c.e - c.b > 4096) ? 8192 : (c.e - c.b) * 2;
    size_t base = out.size();
    out.resize(base + total);
    uint8_t* w = out.data() + base;
    auto p32 = [&](size_t off, uint32_t v) { memcpy(w + off, &v, 4); };
    auto p16 = [&](size_t off, uint16_t v) { memcpy(w + off, &v, 2); };
    p32(0, 12346u);
    p32(4, (uint32_t)cs.size());
    size_t off = 8;
    for (auto& c : cs) { p16(off, c.key); p16(off + 2, (uint16_t)(c.e - c.b - 1)); off += 4; }
    uint32_t data_off = (uint32_t)header;
    for (auto& c : cs) { p32(off, data_off); off += 4; data_off += (c.e - c.b > 4096) ? 8192u : (uint32_t)(c.e - c.b) * 2u; }
    for (auto& c : cs) {
        size_t len = c.e - c.b;
        if (len > 4096) {
            memset(w + off, 0, 8192);
            for (size_t i = c.b; i < c.e; ++i) { uint16_t lo = (uint16_t)ids[i]; w[off + (lo >> 3)] |= (uint8_t)(1u << (lo & 7)); }
            off += 8192;
        } else {
            for (size_t i = c.b; i < c.e; ++i) { p16(off, (uint16_t)ids[i]); off += 2; }
        }
    }
}

}  // namespace

// ================================================================================================
// forest build
// ================================================================================================
namespace {

using BuiltTree = BuiltTreeView;

struct Subsets {   // host arrays, indexed by global tree
    const uint32_t* rows = nullptr; const uint64_t* off = nullptr;
    const uint64_t* start_pos = nullptr;   // optional: StdRng words each tree's stream has already consumed
    uint64_t* end_pos = nullptr;           // optional: ... and has consumed when its tree is finished
};

// f(std::integral_constant<int, METRIC>{}) for the metric: kernels are instantiated per metric, and this is their one dispatch
template <class F>
decltype(auto) with_metric(int metric, F&& f) {
    switch (metric) {
        case EUCLIDEAN: return f(std::integral_constant<int, EUCLIDEAN>{});
        case COSINE: return f(std::integral_constant<int, COSINE>{});
        case DOT_PRODUCT: return f(std::integral_constant<int, DOT_PRODUCT>{});
        case MANHATTAN: return f(std::integral_constant<int, MANHATTAN>{});
        case BQ_EUCLIDEAN: return f(std::integral_constant<int, BQ_EUCLIDEAN>{});
        case BQ_COSINE: return f(std::integral_constant<int, BQ_COSINE>{});
        default: return f(std::integral_constant<int, BQ_MANHATTAN>{});
    }
}

// The control kernel is compiled once per metric (and per cluster size): it is bound by instruction fetch, so every
// instantiation only carries its own metric's code. The binary-quantized metrics have no cluster variants (null).
template <bool SMEM_WS, int CS>
const void* control_fn(int metric) {
    return with_metric(metric, [](auto m) -> const void* {
        if constexpr (CS > 1 && is_bq(decltype(m)::value)) return nullptr;
        else return reinterpret_cast<const void*>(&control_kernel<SMEM_WS, CS, decltype(m)::value>);
    });
}
inline const void* control_fn(bool smem_ws, int cs, int metric) {
    if (!smem_ws) return control_fn<false, 1>(metric);
    if (cs == 0) return control_fn<true, 0>(metric);   // persistent schedule
    return cs == 16 ? control_fn<true, 16>(metric) : (cs == 8 ? control_fn<true, 8>(metric) : control_fn<true, 1>(metric));
}
// The two_means workspace of a control CTA at row pitch ld (build.cuh): WS_VECS vectors, in shared memory when they fit in
// 200 KB, and WS_VECS_SPEC vectors for the speculative two_means when those fit as well.
struct TwoMeansWs { size_t bytes; bool smem, spec; };   // bytes per CTA
TwoMeansWs two_means_ws(uint32_t ld) {
    const size_t plain = (size_t)WS_VECS * ld * 4, spec = (size_t)WS_VECS_SPEC * ld * 4;
    if (spec <= 200 * 1024) return {spec, true, true};
    return {plain, plain <= 200 * 1024, false};
}
// launch (cluster dimension cs > 1: thread-block cluster of cs CTAs per tree)
inline void launch_control(const void* fn, unsigned n_trees, int cs, size_t smem, cudaStream_t s, BuildParams& P, uint32_t tree_base) {
    cudaLaunchConfig_t cfg{};
    cfg.gridDim = dim3(n_trees * (unsigned)cs); cfg.blockDim = dim3(CTRL_THREADS); cfg.dynamicSmemBytes = smem; cfg.stream = s;
    cudaLaunchAttribute at[1];
    cfg.attrs = at; cfg.numAttrs = 0;
    if (cs > 1) { at[0].id = cudaLaunchAttributeClusterDimension; at[0].val.clusterDim.x = (unsigned)cs; at[0].val.clusterDim.y = 1; at[0].val.clusterDim.z = 1; cfg.numAttrs = 1; }
    void* args[2] = {&P, &tree_base};
    CK(cudaLaunchKernelExC(&cfg, fn, args));
}

void planes_prepare(arroy_ctx* c);
void build_wave(arroy_ctx* c, size_t wave_no, uint32_t t0, uint32_t tw, const uint8_t (*seeds)[32], uint32_t K, uint32_t cap_mult,
                arroy_b200_cancel_fn cancel, void* cancel_arg, std::vector<BuiltTree>& out_trees, uint32_t& out_pool_stride, Subsets sub = Subsets{}) {
    const uint64_t n = c->n;
    const uint32_t ld = c->ld;
    Wave& W = c->wave;
    auto t_setup = std::chrono::steady_clock::now();
    auto ms_since = [](std::chrono::steady_clock::time_point t) { return std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t).count(); };
    const uint32_t units = (uint32_t)((n + SCAN_UNIT - 1) / SCAN_UNIT);
    const uint64_t leaves_est = n / std::max<uint32_t>(K, 1) + 1;
    const uint64_t rec_cap64 = std::min<uint64_t>(2 * n + 2, std::max<uint64_t>(64, 8 * leaves_est * cap_mult));
    const uint32_t rec_cap = (uint32_t)rec_cap64;
    // (+ 8 per tree: slots are handed out eight at a time)
    const uint64_t pool_cap64 = std::min<uint64_t>((uint64_t)tw * (n + 1), (uint64_t)tw * (4 * leaves_est * cap_mult + 2)) + 8ull * tw;
    if (pool_cap64 > 0xfffffff0ull) throw CapacityError("normal pool too large");
    const uint32_t pool_cap = (uint32_t)pool_cap64;
    const uint32_t pool_stride = ld + NORMAL_HDR;

    W.st.ensure(sizeof(TreeState) * tw);
    W.frames.ensure(sizeof(Frame) * (size_t)MAX_DEPTH * tw);
    W.recs.ensure(sizeof(Record) * (size_t)rec_cap * tw);
    W.perm0.ensure(4ull * n * tw);
    W.perm1.ensure(4ull * n * tw);
    W.flags.ensure(1ull * n * tw);
    W.unit_left.ensure(4ull * units * tw);
    W.pool.ensure(4ull * pool_stride * pool_cap);
    W.pool_counter.ensure(4);
    W.jobs.ensure(sizeof(Job) * tw);
    W.active.ensure(4);
    W.error.ensure(4);
    W.keys.ensure(32ull * tw);
    const TwoMeansWs ws = two_means_ws(ld);
    if (!ws.smem) W.scratch.ensure(ws.bytes * tw);

    BuildParams P{};
    P.items = items_f32(c); P.ih0 = c->h0.as<float>(); P.ih1 = c->h1.as<float>();
    P.n = (uint32_t)n; P.d = c->dim; P.ld = ld; P.metric = c->metric; P.K = K; P.n_trees = tw;
    P.st = W.st.as<TreeState>(); P.frames = W.frames.as<Frame>(); P.recs = W.recs.as<Record>(); P.rec_cap = rec_cap;
    P.perm[0] = W.perm0.as<uint32_t>(); P.perm[1] = W.perm1.as<uint32_t>();
    P.flags = W.flags.as<uint8_t>(); P.unit_left = W.unit_left.as<uint32_t>(); P.units_per_tree = units;
    P.pool = W.pool.as<float>(); P.pool_stride = pool_stride; P.pool_cap = pool_cap; P.pool_counter = W.pool_counter.as<uint32_t>();
    P.jobs = W.jobs.as<Job>(); P.scratch = W.scratch.as<float>(); P.use_smem_ws = ws.smem; P.spec = ws.spec;
    P.active = W.active.as<uint32_t>(); P.error = W.error.as<int32_t>();
    P.sub_rows = nullptr; P.sub_off = nullptr;
    // cluster-resident nodes: up to ~6 MB of item rows per scan (2048 rows at d = 768, every node of a 10k x 64 index)
    P.small_max = (uint32_t)std::max<uint64_t>(2048, (6ull << 20) / (4ull * ld));
    P.max_inner = 1024u;   // attempts per launch; `cancel` is polled between launches
    // host result buffers: the control kernel writes each record, leaf's ids and accepted normal there as it closes
    // (build.cuh export_records), so no copy of the results follows the kernel. The host pool keeps the slot capacity of the
    // last build of these shapes while that build's slots fit in it, and otherwise takes the slots it used plus an eighth; slots
    // above the capacity are copied after the kernel. A capacity that stays put keeps BuildParams, and so the async schedule's
    // cached graph, the same from build to build.
    if (c->host_waves.size() <= wave_no) c->host_waves.resize(wave_no + 1);
    HostWave& H = c->host_waves[wave_no];
    const uint64_t shape[5] = {n, K, ld, tw, (uint64_t)(sub.rows ? 1 : 0)};
    const bool same_shape = memcmp(shape, H.shape, sizeof shape) == 0;
    uint64_t h_slots = !same_shape ? 2 * leaves_est * tw + 8ull * tw : H.pool_used <= H.slots ? H.slots : (uint64_t)H.pool_used + H.pool_used / 8;
    h_slots = std::min<uint64_t>(h_slots, pool_cap);
    if (const char* e = getenv("ARROY_B200_EXPORT_SLOTS")) h_slots = std::min<uint64_t>(h_slots, strtoull(e, nullptr, 10));
    H.recs.ensure(sizeof(Record) * (size_t)rec_cap * tw);
    H.final_rows.ensure(std::max<size_t>(16, 4ull * n * tw));
    H.pool.ensure(std::max<size_t>(16, (size_t)h_slots * pool_stride * 4));
    P.h_recs = static_cast<Record*>(H.recs.dev); P.h_rows = static_cast<uint32_t*>(H.final_rows.dev);
    P.h_pool = static_cast<float*>(H.pool.dev); P.h_pool_slots = (uint32_t)h_slots;
    if (sub.rows) {   // this wave's subsets, offsets rebased to the wave
        const uint64_t b = sub.off[t0], e = sub.off[t0 + tw];
        std::vector<uint64_t> off(tw + 1);
        for (uint32_t t = 0; t <= tw; ++t) off[t] = sub.off[t0 + t] - b;
        W.sub_rows.ensure(std::max<size_t>(16, 4ull * (e - b)));
        W.sub_off.ensure(8ull * (tw + 1));
        if (e > b) CK(cudaMemcpyAsync(W.sub_rows.p, sub.rows + b, 4ull * (e - b), cudaMemcpyHostToDevice, c->stream));
        CK(cudaMemcpy(W.sub_off.p, off.data(), 8ull * (tw + 1), cudaMemcpyHostToDevice));
        P.sub_rows = W.sub_rows.as<uint32_t>(); P.sub_off = W.sub_off.as<uint64_t>();
    }

    // tree keys = the 8 little-endian words of each 32-byte seed (StdRng::from_seed)
    std::vector<uint32_t> keys((size_t)tw * 8);
    for (uint32_t t = 0; t < tw; ++t)
        for (int i = 0; i < 8; ++i) {
            const uint8_t* s = seeds[t0 + t] + 4 * i;
            keys[(size_t)t * 8 + i] = (uint32_t)s[0] | ((uint32_t)s[1] << 8) | ((uint32_t)s[2] << 16) | ((uint32_t)s[3] << 24);
        }
    CK(cudaMemcpyAsync(W.keys.p, keys.data(), keys.size() * 4, cudaMemcpyHostToDevice, c->stream));
    CK(cudaMemsetAsync(W.pool_counter.p, 0, 4, c->stream));
    CK(cudaMemsetAsync(W.error.p, 0, 4, c->stream));
    CK(cudaMemcpyAsync(W.active.p, &tw, 4, cudaMemcpyHostToDevice, c->stream));
    const uint64_t* d_start = nullptr;
    if (sub.start_pos) {
        W.start_pos.ensure(8ull * tw);
        CK(cudaMemcpyAsync(W.start_pos.p, sub.start_pos + t0, 8ull * tw, cudaMemcpyHostToDevice, c->stream));
        d_start = W.start_pos.as<uint64_t>();
    }
    init_trees_kernel<<<tw, 256, 0, c->stream>>>(P, W.keys.as<uint32_t>(), d_start);
    CK(cudaGetLastError());
    c->n_launches += 1;

    const size_t ctrl_smem = ws.smem ? ws.bytes : 0;

    // Three schedules over the same kernels:
    //  * persistent (below): one cooperative launch for the whole wave.
    //  * async: every tree is its own chain control -> work -> control -> ... on its own stream; all chains of the wave are
    //    branches of ONE CUDA graph of ASYNC_BATCH steps each, so the two_means latency of one tree overlaps the scans of the
    //    others (trees only share the read-only item matrix).
    //  * lockstep (ARROY_B200_LOCKSTEP=1, also used by ARROY_B200_PROFILE=1): one control launch for all trees, then one work
    //    launch for all posted jobs, launched directly; every kernel runs alone, which is what the per-launch roofline
    //    measurement needs. It is the reference the other two schedules are tested against.
    constexpr int ASYNC_BATCH = 64, LOCKSTEP_BATCH = 32;   // steps per graph launch / per batch of direct launches
    const bool profile = getenv("ARROY_B200_PROFILE") != nullptr && atoi(getenv("ARROY_B200_PROFILE")) != 0;
    const bool lockstep = profile || (getenv("ARROY_B200_LOCKSTEP") != nullptr && atoi(getenv("ARROY_B200_LOCKSTEP")) != 0);
    const int steps_per_batch = lockstep ? LOCKSTEP_BATCH : ASYNC_BATCH;
    const void* ctrl1 = control_fn(ws.smem, 1, c->metric);
    raise_smem_limit(c->device, ctrl1, ctrl_smem);
    // Few trees on this GPU = the chain of attempts of each tree is the critical path: the async schedule runs the control kernel
    // as a thread-block cluster that scans small nodes itself (build.cuh control_kernel<.., CS = 8 | 16>).
    // measured: d = 64, 1-10 trees: 24 -> 20 us per attempt; d = 768: 38 -> 37 us for one tree but slower from ~6 trees on
    // (not for host-placed items: the cluster kernels scan their small nodes from the f32 rows)
    const int cluster = (!lockstep && ws.smem && c->dim <= 256 && !is_bq(c->metric) && !c->host_items) ? (tw <= 8 ? 16 : (tw <= 16 ? 8 : 1)) : 1;
    const void* ctrlc = control_fn(ws.smem, cluster, c->metric);
    raise_smem_limit(c->device, ctrlc, ctrl_smem);
    if (cluster == 16) CK(cudaFuncSetAttribute(ctrlc, cudaFuncAttributeNonPortableClusterSizeAllowed, 1));

    // Persistent schedule (default): ONE cooperative launch per wave — a control CTA per tree plus worker CTAs on every SM
    // (build.cuh control_kernel<.., CS = 0>). Needs two CTAs per SM to have enough workers next to the control CTAs; with
    // a big workspace (d > 1152) that means giving up the speculative two_means.
    bool persist = false;
    int pgrid = 0;
    size_t psmem = ctrl_smem;
    const void* ctrlp = nullptr;
    // It wins where the chain of attempts is the critical path (few trees per GPU, small indexes); a wave that is bandwidth-bound
    // from start to end (10M x 100 trees) runs a little faster on work_kernel's three scanning CTAs per SM.
    if ((double)n * (double)tw <= 2.0e8 && !lockstep && ws.smem && ld <= 8u * CTRL_THREADS && n < (1ull << 29)) {
        ctrlp = control_fn(true, 0, c->metric);
        const size_t cand[2] = {persistent_smem(ctrl_smem, ld), persistent_smem((size_t)WS_VECS * ld * 4, ld)};
        for (int k = 0; k < 2 && !persist; ++k) {
            if (k == 1 && !P.spec) break;
            raise_smem_limit(c->device, ctrlp, cand[k]);
            int nb = 0;
            CK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&nb, ctrlp, CTRL_THREADS, cand[k]));
            const int cap = nb * c->sm_count;
            if ((nb >= 2 || k == 1) && cap >= (int)tw + std::max(16, c->sm_count / 2)) { persist = true; pgrid = cap; psmem = cand[k]; if (k == 1) P.spec = 0; }
        }
    }
    // scans through the 8-bit planes of the items (kernels.cuh scan_claim_planes): nodes of more than shadow_min_units units.
    // Host-placed items: every scan, so that only the rows the planes cannot decide are read over PCIe.
    if (!is_bq(c->metric) && P.d >= 64 && P.d <= PLANES_MAX_D && (n * (uint64_t)ld >= (1ull << 22) || c->host_items)) {
        planes_prepare(c);
        P.planes = plane_rows(c);
        W.shadow_stats.ensure(24);
        CK(cudaMemsetAsync(W.shadow_stats.p, 0, 24, c->stream));
        P.shadow_stats = W.shadow_stats.as<unsigned long long>();
        // many trees per GPU: bandwidth decides, every node goes through the shadow; few: the chain of attempts decides and
        // small nodes keep the one-unit claims of the exact scan (more CTAs per node)
        P.shadow_min_units = c->host_items ? 0u : (!persist || tw >= 32) ? 12u : (tw >= 12 ? 64u : 128u);
    }
    const ScanPlanes scan_planes{P.shadow_min_units, P.shadow_stats};
    const ScanPlanes* pl = P.planes.hi ? &scan_planes : nullptr;
    scan_smem(c, (int)tw, pl != nullptr);   // the limit of the wave's largest scan, raised before the graph is captured
    if (persist) {
        W.slots.ensure(sizeof(PSlot) * tw);
        W.abort.ensure(4);
        CK(cudaMemsetAsync(W.slots.p, 0, sizeof(PSlot) * tw, c->stream));
        CK(cudaMemsetAsync(W.abort.p, 0, 4, c->stream));
        W.cur_normal.ensure(4ull * pool_stride * tw);
        P.slots = W.slots.as<PSlot>();
        P.cur_normal = W.cur_normal.as<float>();
        P.abort = W.abort.as<int>();
        // fused root scan: every tree of the wave starts at the root of the whole index (no subtree mode), rows go through the
        // 8-lanes-per-row path, and a batch of normals fits next to nothing else in the workers' shared memory (f32 rows only: the
        // bit-string rows of the binary-quantized metrics take the popcount scan, kernels.cuh bq_scan_unit)
        // (not for host-placed items: the pass streams every f32 row and prefetches them into L2 with bulk copies)
        P.root_fused = (!is_bq(c->metric) && !sub.rows && tw >= 2 && P.d >= 32 && (size_t)ROOT_TB * ld * 4 <= psmem && !c->host_items) ? 1 : 0;
        W.root.ensure(8);
        CK(cudaMemsetAsync(W.root.p, 0, 8, c->stream));
        P.root_ready = W.root.as<uint32_t>(); P.root_ticket = W.root.as<uint32_t>() + 1;
    }
    // the schedule this wave runs, OR-ed over the waves of the build (bits: arroy_b200_build_breakdown in arroy_b200.h)
    {
        const uint32_t sched = persist ? 1u : lockstep ? 2u : cluster == 16 ? 16u : cluster == 8 ? 8u : 4u;
        c->breakdown[6] = (double)((uint32_t)c->breakdown[6] | sched | (ws.smem ? 0u : 32u) | (P.spec ? 64u : 0u));
    }

    CK(cudaStreamSynchronize(c->stream));
    c->breakdown[0] += ms_since(t_setup);
    auto t_graph = std::chrono::steady_clock::now();
    // The async schedule's graph only depends on the kernel arguments (BuildParams: buffer pointers are stable because the wave
    // buffers live in the context), the wave's size and the cluster size, so it is reused by later builds with the same shapes.
    cudaGraphExec_t gexec = nullptr;
    if (!persist && !lockstep) {
        std::vector<uint8_t> key(sizeof(BuildParams) + 12);
        memcpy(key.data(), &P, sizeof(BuildParams));
        const int32_t shape[3] = {(int32_t)tw, (int32_t)ctrl_smem, cluster};
        memcpy(key.data() + sizeof(BuildParams), shape, 12);
        if (c->cached_exec && key == c->cached_graph_key) gexec = c->cached_exec;
        else {
            c->cached_graph_key.clear();
            while (c->tree_streams.size() < tw) c->tree_streams.push_back(new_stream());
            while (c->tree_events.size() < (size_t)tw + 1) c->tree_events.push_back(new_event(cudaEventDisableTiming));
            cudaGraph_t graph = nullptr;
            CK(cudaStreamBeginCapture(c->stream, cudaStreamCaptureModeThreadLocal));
            CK(cudaEventRecord(c->tree_events[0], c->stream));
            for (uint32_t t = 0; t < tw; ++t) {   // one tree (one cluster) per control launch, sm_count work CTAs per work launch
                cudaStream_t st = c->tree_streams[t];
                CK(cudaStreamWaitEvent(st, c->tree_events[0], 0));
                for (int i = 0; i < ASYNC_BATCH; ++i) {
                    launch_control(ctrlc, 1, cluster, ctrl_smem, st, P, t);
                    launch_scan(c, st, P.jobs + t, 1, c->sm_count, pl);
                }
                CK(cudaEventRecord(c->tree_events[1 + t], st));
                CK(cudaStreamWaitEvent(c->stream, c->tree_events[1 + t], 0));
            }
            CK(cudaStreamEndCapture(c->stream, &graph));
            c->cached_graph = Graph(graph);
            CK(cudaGraphInstantiate(&gexec, graph, 0));
            c->cached_exec = GraphExec(gexec);
            c->cached_graph_key = key;
        }
    }

    c->breakdown[1] += ms_since(t_graph);
    auto t_loop = std::chrono::steady_clock::now();
    c->pin.ensure(64);
    volatile uint32_t* h_active = c->pin.as<uint32_t>();
    volatile int32_t* h_error = reinterpret_cast<volatile int32_t*>(c->pin.as<uint32_t>() + 1);
    std::vector<Event> pev;
    if (profile) for (int i = 0; i < 2 * LOCKSTEP_BATCH; ++i) pev.push_back(new_event());
    uint64_t steps = 0;
    // safety net against a stuck state machine (never hit by a correct build): every step each
    // live tree completes one attempt or one partition
    const uint64_t max_steps = 40ull * (8 * leaves_est + 64) + 4096;
    if (persist) {
        cudaLaunchConfig_t cfg{};
        cfg.gridDim = dim3((unsigned)pgrid); cfg.blockDim = dim3(CTRL_THREADS); cfg.dynamicSmemBytes = psmem; cfg.stream = c->stream;
        cudaLaunchAttribute at[1];
        at[0].id = cudaLaunchAttributeCooperative; at[0].val.cooperative = 1;   // all CTAs resident together, or the launch fails
        cfg.attrs = at; cfg.numAttrs = 1;
        uint32_t tree_base = 0;
        void* args[2] = {&P, &tree_base};
        CK(cudaEventRecord(c->ev_p0, c->stream));
        CK(cudaLaunchKernelExC(&cfg, ctrlp, args));
        CK(cudaEventRecord(c->ev_p1, c->stream));
        CK(cudaEventRecord(c->ev_done, c->stream));
        if (cancel) {   // polled while the kernel runs (BuildOption::cancel, src/writer.rs:116-124)
            bool aborted = false;
            for (;;) {
                const cudaError_t q = cudaEventQuery(c->ev_done);
                if (q == cudaSuccess) break;
                if (q != cudaErrorNotReady) CK(q);
                if (!aborted && cancel(cancel_arg)) {
                    const int one = 1;
                    CK(cudaMemcpyAsync(W.abort.p, &one, 4, cudaMemcpyHostToDevice, c->side_stream));
                    aborted = true;
                }
                std::this_thread::sleep_for(std::chrono::microseconds(aborted ? 50 : 500));
            }
        }
        CK(cudaMemcpyAsync((void*)h_active, W.active.p, 4, cudaMemcpyDeviceToHost, c->stream));
        CK(cudaMemcpyAsync((void*)h_error, W.error.p, 4, cudaMemcpyDeviceToHost, c->stream));
        CK(cudaStreamSynchronize(c->stream));
        steps = 1;
        c->n_launches += 1;
        { float kms = 0; CK(cudaEventElapsedTime(&kms, c->ev_p0, c->ev_p1)); c->stats[5] += kms; }   // the kernel that holds every scan of the wave
        if (*h_error != ERR_NONE) {
            const int e = *h_error;
            if (e == ERR_ABORT) throw Cancelled("The corresponding build process has been cancelled");
            if (e == ERR_HANG) throw std::runtime_error("forest build made no progress (persistent schedule watchdog)");
            throw CapacityError(e == ERR_DEPTH ? "tree deeper than MAX_DEPTH frames" : e == ERR_RECORDS ? "node record table overflow" : "normal pool overflow");
        }
        if (*h_active != 0) throw std::runtime_error("forest build ended with unfinished trees (internal state machine error)");
    } else
    for (;;) {
        if (steps > max_steps) throw std::runtime_error("forest build did not converge (internal state machine error)");
        if (!lockstep) CK(cudaGraphLaunch(gexec, c->stream));
        else {   // all trees per launch; with `profile`, each work launch is timed by a pair of events
            for (int i = 0; i < LOCKSTEP_BATCH; ++i) {
                launch_control(ctrl1, tw, 1, ctrl_smem, c->stream, P, 0u);
                if (profile) CK(cudaEventRecord(pev[2 * i], c->stream));
                launch_scan(c, c->stream, P.jobs, (int)tw, c->sm_count * (pl ? 2 : 3), pl);
                if (profile) CK(cudaEventRecord(pev[2 * i + 1], c->stream));
            }
            CK(cudaGetLastError());
            if (profile) {
                CK(cudaStreamSynchronize(c->stream));
                for (int i = 0; i < LOCKSTEP_BATCH; ++i) {
                    float ms = 0; CK(cudaEventElapsedTime(&ms, pev[2 * i], pev[2 * i + 1])); c->stats[5] += ms;
                    if (getenv("ARROY_B200_TRACE") && steps + i < 48) fprintf(stderr, "[trace] step %llu work_kernel %.3f ms\n", (unsigned long long)(steps + i), ms);
                }
            }
        }
        steps += steps_per_batch;
        c->n_launches += 2ull * steps_per_batch * (lockstep ? 1 : tw);
        CK(cudaMemcpyAsync((void*)h_active, W.active.p, 4, cudaMemcpyDeviceToHost, c->stream));
        CK(cudaMemcpyAsync((void*)h_error, W.error.p, 4, cudaMemcpyDeviceToHost, c->stream));
        CK(cudaStreamSynchronize(c->stream));
        if (*h_error != ERR_NONE) {
            int e = *h_error;
            throw CapacityError(e == ERR_DEPTH ? "tree deeper than MAX_DEPTH frames" : e == ERR_RECORDS ? "node record table overflow" : "normal pool overflow");
        }
        if (*h_active == 0) break;
        if (cancel && cancel(cancel_arg)) throw Cancelled("The corresponding build process has been cancelled");
    }
    c->stats[1] += (double)steps;
    c->breakdown[2] += ms_since(t_loop);
    c->breakdown[5] += (double)(steps / steps_per_batch);
    auto t_d2h = std::chrono::steady_clock::now();

    // results: the kernel has written them to the host buffers; only the tree states, the pool's fill and the pre-filter's
    // stage counters come back here
    std::vector<TreeState> st(tw);
    uint32_t pool_used = 0;
    unsigned long long hs[3] = {0, 0, 0};
    CK(cudaMemcpyAsync(st.data(), W.st.p, sizeof(TreeState) * tw, cudaMemcpyDeviceToHost, c->stream));
    CK(cudaMemcpyAsync(&pool_used, W.pool_counter.p, 4, cudaMemcpyDeviceToHost, c->stream));
    if (P.shadow_stats) CK(cudaMemcpyAsync(hs, P.shadow_stats, 24, cudaMemcpyDeviceToHost, c->stream));
    CK(cudaStreamSynchronize(c->stream));
    memcpy(H.shape, shape, sizeof shape); H.slots = (uint32_t)h_slots; H.pool_used = pool_used;
    uint64_t late_bytes = 0;
    if (pool_used > h_slots) {   // the slots the host pool had no room for: a bigger pool keeps the exported ones
        const size_t kept = (size_t)h_slots * pool_stride * 4;
        late_bytes = ((size_t)pool_used - h_slots) * pool_stride * 4;
        MappedBuf grown;
        grown.ensure(kept + late_bytes);
        memcpy(grown.p, H.pool.p, kept);
        H.pool = std::move(grown);
        CK(cudaMemcpyAsync(static_cast<uint8_t*>(H.pool.p) + kept, W.pool.as<uint8_t>() + kept, late_bytes, cudaMemcpyDeviceToHost, c->stream));
        c->breakdown[7] += (double)(pool_used - h_slots);
    }
    out_pool_stride = pool_stride;
    out_trees.resize(tw);
    // bytes the kernel wrote to host memory: every record, the ids of every row of the tree (its leaves partition them) and
    // one normal per split that is not random ((n_recs - 1) / 2 splits), less the normals in slots the host copied itself
    uint64_t exported = 0;
    for (uint32_t t = 0; t < tw; ++t) {
        const Record* recs = H.recs.as<Record>() + (size_t)t * rec_cap;
        out_trees[t].recs = static_cast<const void*>(recs);
        out_trees[t].n_recs = st[t].n_recs;
        out_trees[t].final_rows = H.final_rows.as<uint32_t>() + (size_t)t * n;
        out_trees[t].pool = H.pool.as<float>();
        const uint64_t rows = sub.rows ? sub.off[t0 + t + 1] - sub.off[t0 + t] : n;
        uint64_t normals = (st[t].n_recs - 1) / 2 - st[t].n_random;
        if (late_bytes)
            for (uint32_t i = 0; i < st[t].n_recs; ++i) normals -= recs[i].kind == REC_SPLIT && recs[i].c != NO_SLOT && recs[i].c >= h_slots;
        exported += sizeof(Record) * (uint64_t)st[t].n_recs + 4 * rows + 4ull * pool_stride * normals;
        c->stats[0] += (double)st[t].scanned;
        c->stats[2] += (double)st[t].n_splits_tried;
        c->stats[3] += (double)st[t].n_random;
        c->stats[7] += (double)st[t].n_misspec;
        if (sub.end_pos) sub.end_pos[t0 + t] = st[t].pos;
    }
    if (persist && P.root_fused) { c->fused_root_rows += (uint64_t)tw * n; c->fused_root_read += n; }
    if (P.shadow_stats) { c->shadow_rows += hs[0]; c->shadow_rescored += hs[1]; c->shadow_stage2 += hs[2]; }
    if (late_bytes) CK(cudaStreamSynchronize(c->stream));
    c->d2h_bytes += sizeof(TreeState) * tw + exported + late_bytes;
    c->breakdown[3] += ms_since(t_d2h);
}

// Phase 1: device build of `n_trees` trees; results stay parked in the context.
void do_build_begin(arroy_ctx* c, uint32_t n_trees, const uint8_t (*seeds)[32], uint32_t split_after, arroy_b200_cancel_fn cancel, void* cancel_arg, uint32_t* out_counts,
                    Subsets sub = Subsets{}) {
    require_staged(c);
    set_device(c);
    for (auto& s : c->stats) s = 0;
    c->shadow_rows = 0; c->shadow_rescored = 0; c->shadow_stage2 = 0; c->fused_root_rows = 0; c->fused_root_read = 0;
    c->pending_waves.clear(); c->pending_wave_t0.clear(); c->pending_n_trees = 0;
    const uint32_t K = split_after ? split_after : c->dim;
    if (!sub.rows && c->n <= K) throw ArgError("build_trees needs more items than split_after (a single Descendants node is the caller's job, src/writer.rs:499-501)");
    if (sub.rows)
        for (uint32_t t = 0; t < n_trees; ++t) {
            if (sub.off[t + 1] - sub.off[t] <= K) throw ArgError("build_subtrees: every subset must hold more rows than split_after");
            for (uint64_t i = sub.off[t]; i < sub.off[t + 1]; ++i) { if (sub.rows[i] >= c->n) throw ArgError("row index out of range"); if (i > sub.off[t] && sub.rows[i] <= sub.rows[i - 1]) throw ArgError("subset rows must be ascending"); }
        }
    if (n_trees == 0) return;
    if (cancel && cancel(cancel_arg)) throw Cancelled("The corresponding build process has been cancelled");

    // wave size from free memory. cudaMemGetInfo is a driver round trip that takes anything from 0.5 to 30 ms on this part: a
    // rebuild with the shapes of the previous build (whose wave buffers are still held by the context) reuses its answer.
    const uint64_t n = c->n;
    const uint64_t wave_key[4] = {n, K, c->ld, (uint64_t)(sub.rows ? 1 : 0)};
    const bool same_shape = c->wave_key_valid && memcmp(wave_key, c->wave_key, sizeof wave_key) == 0 && n_trees <= c->wave_trees_ok;
    size_t free_b = 0, total_b = 0;
    if (!same_shape) CK(cudaMemGetInfo(&free_b, &total_b));
    const uint64_t leaves_est = n / K + 1;
    const uint64_t per_tree = n * (4 + 4 + 1) + (n / SCAN_UNIT + 1) * 4 + sizeof(Frame) * (uint64_t)MAX_DEPTH + 16ull * 8 * leaves_est +
                              4ull * (c->ld + NORMAL_HDR) * 4 * leaves_est + 4096;
    uint64_t reusable = c->wave.perm0.cap + c->wave.perm1.cap + c->wave.flags.cap + c->wave.pool.cap + c->wave.recs.cap;
    uint64_t max_wave = same_shape ? c->wave_max : (uint64_t)((free_b + reusable) * 0.7) / std::max<uint64_t>(per_tree, 1);
    if (!same_shape) c->wave_max = max_wave;
    if (const char* e = getenv("ARROY_B200_MAX_WAVE")) max_wave = std::min<uint64_t>(max_wave, (uint64_t)atoi(e));
    max_wave = std::max<uint64_t>(1, std::min<uint64_t>(max_wave, 120));  // <= 128 concurrent kernels

    for (auto& b : c->breakdown) b = 0;
    CK(cudaEventRecord(c->ev0, c->stream));
    uint32_t pool_stride = 0;
    for (uint32_t t0 = 0; t0 < n_trees;) {
        uint32_t tw = (uint32_t)std::min<uint64_t>(max_wave, n_trees - t0);
        std::vector<BuiltTree> trees;
        uint32_t cap_mult = 1;
        for (;;) {
            try { build_wave(c, c->pending_waves.size(), t0, tw, seeds, K, cap_mult, cancel, cancel_arg, trees, pool_stride, sub); break; }
            catch (const CapacityError&) { if (cap_mult >= 64) throw; cap_mult *= 4; }
        }
        c->pending_waves.push_back(std::move(trees));
        c->pending_wave_t0.push_back(t0);
        t0 += tw;
    }
    CK(cudaEventRecord(c->ev1, c->stream));
    CK(cudaEventSynchronize(c->ev1));
    float ms = 0;
    CK(cudaEventElapsedTime(&ms, c->ev0, c->ev1));
    c->stats[4] = ms;
    c->pending_pool_stride = pool_stride;
    c->pending_n_trees = n_trees;
    memcpy(c->wave_key, wave_key, sizeof wave_key); c->wave_key_valid = true; c->wave_trees_ok = std::max<uint64_t>(same_shape ? c->wave_trees_ok : 0, n_trees);
    uint64_t total_nodes = 0;
    for (size_t w = 0; w < c->pending_waves.size(); ++w)
        for (size_t i = 0; i < c->pending_waves[w].size(); ++i) {
            if (out_counts) out_counts[c->pending_wave_t0[w] + i] = c->pending_waves[w][i].n_recs;
            total_nodes += c->pending_waves[w][i].n_recs;
        }
    c->stats[6] = (double)total_nodes;
}

// Phase 2: NodeCodec encoding of the parked trees. Non-root node li of tree t gets id base_ids[t] + li.
// node_ids (optional): explicit ids of the non-root nodes, concatenated per tree in post-order
// (tree t contributes n_recs[t] - 1 entries); otherwise node li of tree t gets base[t] + li.
void do_build_emit(arroy_ctx* c, const uint32_t* root_ids, const uint64_t* base, arroy_b200_node_sink sink, void* sink_arg, const uint32_t* node_ids = nullptr) {
    const uint32_t n_trees = c->pending_n_trees;
    if (n_trees == 0 || !sink) return;
    std::vector<const BuiltTree*> tree_ptr(n_trees);
    for (size_t w = 0; w < c->pending_waves.size(); ++w)
        for (size_t i = 0; i < c->pending_waves[w].size(); ++i) tree_ptr[c->pending_wave_t0[w] + i] = &c->pending_waves[w][i];
    std::vector<uint64_t> id_off(n_trees + 1, 0);
    for (uint32_t t = 0; t < n_trees; ++t) id_off[t + 1] = id_off[t] + tree_ptr[t]->n_recs - 1;
    if (!node_ids)
        for (uint32_t t = 0; t < n_trees; ++t)
            if (base[t] + tree_ptr[t]->n_recs > 0x100000000ull) throw CapacityError("node ids exceed u32 (Error::DatabaseFull)");
    const uint32_t pool_stride = c->pending_pool_stride;
    auto t_enc = std::chrono::steady_clock::now();

    // encode NodeCodec bytes (src/node.rs:229-241); trees in parallel, the sink is called concurrently
    const int hdrf = metric_header_floats(c->metric);
    const uint32_t d = c->dim;
    std::mutex sink_mu;
    // work items = (tree, block of ENC_BLOCK records): finer than one tree per thread, so that 50 trees keep 64 threads busy
    constexpr uint32_t ENC_BLOCK = 256;
    std::vector<uint64_t> blk_off(n_trees + 1, 0);
    for (uint32_t t = 0; t < n_trees; ++t) blk_off[t + 1] = blk_off[t] + (tree_ptr[t]->n_recs + ENC_BLOCK - 1) / ENC_BLOCK;
    const uint64_t n_blocks = blk_off[n_trees];
    std::atomic<uint64_t> next_block{0};
    std::atomic<int> abort_flag{0};
    std::string worker_err;
    auto worker = [&]() {
        std::vector<uint8_t> buf;
        std::vector<uint32_t> ids;
        try {
            for (;;) {
                const uint64_t w = next_block.fetch_add(1);
                if (w >= n_blocks || abort_flag.load()) return;
                const uint32_t t = (uint32_t)(std::upper_bound(blk_off.begin(), blk_off.end(), w) - blk_off.begin() - 1);
                const BuiltTree& T = *tree_ptr[t];
                const Record* recs = static_cast<const Record*>(T.recs);
                const float* pool = T.pool;
                const uint32_t root_local = T.n_recs - 1;
                auto gid = [&](uint32_t li) { return li == root_local ? root_ids[t] : (node_ids ? node_ids[id_off[t] + li] : (uint32_t)(base[t] + li)); };
                const uint32_t li0 = (uint32_t)(w - blk_off[t]) * ENC_BLOCK, li1 = std::min<uint32_t>(T.n_recs, li0 + ENC_BLOCK);
                for (uint32_t li = li0; li < li1; ++li) {
                    const Record& r = recs[li];
                    buf.clear();
                    if (r.kind == REC_DESC) {
                        buf.push_back(1);
                        ids.resize(r.b);
                        for (uint32_t i = 0; i < r.b; ++i) ids[i] = c->ids[T.final_rows[r.a + i]];
                        roaring_serialize(ids.data(), ids.size(), buf);
                    } else {
                        buf.push_back(2);
                        uint32_t l = gid(r.a), rr = gid(r.b);
                        for (int k = 3; k >= 0; --k) buf.push_back((uint8_t)(l >> (8 * k)));
                        for (int k = 3; k >= 0; --k) buf.push_back((uint8_t)(rr >> (8 * k)));
                        if (r.c != NO_SLOT && is_bq(c->metric)) {
                            // the vector part of a binary-quantized normal is its bit string: 64-bit words, bit i of word w = element
                            // 64 w + i positive (binary_quantized.rs:80-92)
                            const float* s = pool + (size_t)r.c * pool_stride;
                            size_t o = buf.size();
                            buf.resize(o + 4 + d / 8, 0);
                            memcpy(buf.data() + o, s, 4);
                            for (uint32_t i = 0; i < d; ++i) if (s[NORMAL_HDR + i] > 0.f) buf[o + 4 + (i >> 3)] |= (uint8_t)(1u << (i & 7));
                        } else if (r.c != NO_SLOT) {
                            const float* s = pool + (size_t)r.c * pool_stride;
                            size_t o = buf.size();
                            buf.resize(o + 4 * hdrf + 4ull * d);
                            memcpy(buf.data() + o, s, 4 * hdrf);
                            memcpy(buf.data() + o + 4 * hdrf, s + NORMAL_HDR, 4ull * d);
                        }
                    }
                    if (abort_flag.load()) return;
                    if (sink(sink_arg, gid(li), buf.data(), buf.size()) != 0) { abort_flag = 1; return; }
                }
            }
        } catch (const std::exception& e) { std::lock_guard<std::mutex> lk(sink_mu); worker_err = e.what(); abort_flag = 2; }
    };
    const int nthreads = c->n < 100000 ? 1 : (int)std::min<uint64_t>(n_blocks, std::max(1u, std::min(64u, std::thread::hardware_concurrency())));
    if (nthreads <= 1) worker();
    else { std::vector<std::thread> th; for (int i = 0; i < nthreads; ++i) th.emplace_back(worker); for (auto& x : th) x.join(); }
    c->breakdown[4] = std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t_enc).count();
    if (abort_flag.load() == 1) throw Cancelled("node sink aborted the build");
    if (abort_flag.load() == 2) throw std::runtime_error(worker_err);
}

void do_build(arroy_ctx* c, uint32_t n_trees, const uint8_t (*seeds)[32], const uint32_t* root_ids, uint32_t first_free, uint32_t split_after,
              arroy_b200_cancel_fn cancel, void* cancel_arg, arroy_b200_node_sink sink, void* sink_arg, uint64_t* out_n_nodes) {
    std::vector<uint32_t> counts(n_trees, 0);
    do_build_begin(c, n_trees, seeds, split_after, cancel, cancel_arg, counts.data());
    // node ids: roots pre-allocated; the rest numbered as a 1-thread rayon pool would (tree tasks
    // LIFO => last tree first; post-order inside a tree) — SURVEY.md Appendix B.4
    std::vector<uint64_t> base(n_trees);
    uint64_t counter = first_free, total = 0;
    for (uint32_t k = 0; k < n_trees; ++k) { uint32_t t = n_trees - 1 - k; base[t] = counter; counter += counts[t] - 1; total += counts[t]; }
    if (counter > 0xffffffffull) throw CapacityError("node ids exceed u32 (Error::DatabaseFull)");
    if (out_n_nodes) *out_n_nodes = total;
    do_build_emit(c, root_ids, base.data(), sink, sink_arg);
}

// ================================================================================================
// side_batch / rerank
// ================================================================================================

void upload_normal(arroy_ctx* c, const float* normal, float h0, float h1) {
    const uint32_t ld = c->ld;
    c->s_normal.ensure((size_t)(ld + NORMAL_HDR) * 4);
    c->pin.ensure(std::max<size_t>(c->pin.cap, (size_t)(ld + NORMAL_HDR) * 4));
    float* h = c->pin.as<float>();
    h[0] = h0; h[1] = h1; h[2] = 0.f; h[3] = 0.f;
    memcpy(h + NORMAL_HDR, normal, 4ull * c->dim);
    for (uint32_t i = c->dim; i < ld; ++i) h[NORMAL_HDR + i] = 0.f;
    CK(cudaMemcpyAsync(c->s_normal.p, h, (size_t)(ld + NORMAL_HDR) * 4, cudaMemcpyHostToDevice, c->stream));
}

void do_side_batch(arroy_ctx* c, const float* normal, float h0, float h1, const uint32_t* rows, uint64_t n_rows, uint8_t* out_side, float* out_margin) {
    require_staged(c);
    set_device(c);
    if (n_rows == 0) return;
    if (n_rows > 0xffffffffull) throw ArgError("too many rows");
    for (uint64_t i = 0; i < n_rows; ++i) if (rows[i] >= c->n) throw ArgError("row index out of range");
    upload_normal(c, normal, h0, h1);
    CK(cudaStreamSynchronize(c->stream));  // pinned staging buffer is reused below
    c->s_rows.ensure(n_rows * 4);
    c->s_flags.ensure(n_rows);
    c->s_margins.ensure(n_rows * 4);
    c->s_unit.ensure(((n_rows + SCAN_UNIT - 1) / SCAN_UNIT) * 4);
    c->s_job.ensure(sizeof(Job));
    CK(cudaMemcpyAsync(c->s_rows.p, rows, n_rows * 4, cudaMemcpyHostToDevice, c->stream));
    Job jb{};
    jb.kind = JOB_SCAN; jb.len = (uint32_t)n_rows; jb.rows = c->s_rows.as<uint32_t>(); jb.normal = c->s_normal.as<float>();
    jb.flags = c->s_flags.as<uint8_t>(); jb.margins = out_margin ? c->s_margins.as<float>() : nullptr; jb.unit_left = c->s_unit.as<uint32_t>();
    CK(cudaMemcpyAsync(c->s_job.p, &jb, sizeof(Job), cudaMemcpyHostToDevice, c->stream));
    uint64_t units = (n_rows + SCAN_UNIT - 1) / SCAN_UNIT;
    launch_scan(c, c->stream, c->s_job.as<Job>(), 1, (unsigned)std::min<uint64_t>(units, (uint64_t)c->sm_count * 3), nullptr);
    CK(cudaGetLastError());
    c->n_launches += 1;
    CK(cudaMemcpyAsync(out_side, c->s_flags.p, n_rows, cudaMemcpyDeviceToHost, c->stream));
    if (out_margin) CK(cudaMemcpyAsync(out_margin, c->s_margins.p, n_rows * 4, cudaMemcpyDeviceToHost, c->stream));
    CK(cudaStreamSynchronize(c->stream));
}

// ---- tensor-core pre-filter helpers (rerank_shared) ---------------------------------------------
// candidate matrix for the score GEMM: the item matrix in place when `rows` is a contiguous range,
// else a gathered copy. Host-placed items are always gathered: the GEMM reads its operands with TMA, which takes device memory.
const float* xf_candidates(arroy_ctx* c, const uint32_t* rows, uint32_t nc) {
    bool contiguous = !c->host_items;
    for (uint64_t i = 1; i < nc && contiguous; ++i) contiguous = rows[i] == rows[0] + i;
    if (contiguous) return c->items.as<float>() + (size_t)rows[0] * c->ld;
    c->x_gather.ensure(4ull * nc * c->ld);
    xf_gather_kernel<<<c->sm_count * 8, 256, 0, c->stream>>>(c->x_gather.as<float4>(), reinterpret_cast<const float4*>(items_f32(c)), c->s_rows.as<uint32_t>(), nc, c->ld / 4);
    CK(cudaGetLastError());
    c->n_launches += 1;
    return c->x_gather.as<float>();
}

// S (m x nc, pitch lds) = Q . cand^T with TF32 inputs and FP32 accumulation. engine 0: the wgmma
// kernel of tcgemm.cuh; engine 1: cuBLAS (kept as the cross-check of the hand-written kernel)
void xf_scores(arroy_ctx* c, const float* q, uint32_t m, const float* cand, uint32_t nc, float* S, uint32_t lds, TgEpilogue ep, int engine) {
    if (engine == 0) {
        raise_smem_limit(c->device, (const void*)tcgemm_tf32_kernel, TG_SMEM);
        if (!tcgemm_tf32(q, m, cand, nc, c->ld, S, lds, ep, c->sm_count, c->tg_clusters, c->stream)) throw CudaError(std::string("tcgemm_tf32 launch failed: ") + cudaGetErrorString(cudaGetLastError()));
        c->n_launches += 1;
        return;
    }
    if (!c->blas) { cublasHandle_t b = nullptr; if (cublasCreate(&b) != CUBLAS_STATUS_SUCCESS) throw CudaError("cublasCreate failed"); c->blas = Blas(b); }
    if (cublasSetStream(c->blas, c->stream) != CUBLAS_STATUS_SUCCESS) throw CudaError("cublasSetStream failed");
    const float one = 1.0f, zero = 0.0f;
    cublasStatus_t st = cublasGemmEx(c->blas, CUBLAS_OP_T, CUBLAS_OP_N, (int)nc, (int)m, (int)c->ld, &one, cand, CUDA_R_32F, (int)c->ld,
                                     q, CUDA_R_32F, (int)c->ld, &zero, S, CUDA_R_32F, (int)lds, CUBLAS_COMPUTE_32F_FAST_TF32, CUBLAS_GEMM_DEFAULT);
    if (st != CUBLAS_STATUS_SUCCESS) throw CudaError("cublasGemmEx failed with status " + std::to_string((int)st));
    if (ep.mode != TG_RAW) { tg_finish_kernel<<<c->sm_count * 8, 256, 0, c->stream>>>(S, m, nc, lds, ep); CK(cudaGetLastError()); }
    c->n_launches += 2;
}

int xf_engine() { const char* e = getenv("ARROY_B200_XGEMM"); return (e && strcmp(e, "cublas") == 0) ? 1 : 0; }

// A call's queries on the device: by item their rows (vecs == nullptr), by vector their vectors (rows == nullptr), and their
// first header. Binary-quantized metrics: always their +-1 vectors (rows == nullptr), and their bit strings.
struct DevQueries {
    const float* vecs = nullptr;
    const uint32_t* rows = nullptr;
    const float* h0 = nullptr;
    const uint4* bits = nullptr;
};

// ---- fused re-rank (frerank.cuh) -------------------------------------------------------------------
// The estimate source of the fused re-rank for this context and k: device-placed items estimate from the bf16 shadow (Manhattan
// has none), host-placed items from the build's 8-bit planes, which reads only the survivors' rows from host memory.
// FR_NONE: the plain kernels re-rank (ARROY_B200_FRERANK=0, binary-quantized metrics, k or rows beyond the kernel's buffers).
int frerank_source(arroy_ctx* c, uint32_t k) {
    const char* e = getenv("ARROY_B200_FRERANK");
    if ((e != nullptr && atoi(e) == 0) || is_bq(c->metric) || k > (uint32_t)FR_SURV || frerank_smem(c->ld) > 200 * 1024) return FR_NONE;
    if (c->host_items) return c->planes_valid ? FR_PLANES : FR_NONE;
    return c->metric != MANHATTAN ? FR_BF16 : FR_NONE;
}

// bf16 copy of the staged items (round to nearest even; padding stays zero) for the fused re-rank
void shadow_prepare(arroy_ctx* c) {
    if (c->shadow_valid) return;
    const uint64_t total4 = (uint64_t)c->n * c->ld / 4;
    c->fr_shadow.ensure(std::max<size_t>(16, (size_t)c->n * c->ld * 2));
    fr_shadow_kernel<<<c->sm_count * 8, 256, 0, c->stream>>>(c->items.as<float4>(), c->fr_shadow.as<uint2>(), total4);
    CK(cudaGetLastError());
    c->n_launches += 1;
    c->shadow_valid = true;
}

// the build's pre-filter encoding of the staged items (kernels.cuh planes_encode_kernel): two int8 planes and a scale per row
void planes_prepare(arroy_ctx* c) {
    if (c->planes_valid) return;
    const size_t bytes = std::max<size_t>(16, (size_t)c->n * c->ld);
    c->pl_hi.ensure(bytes);
    c->pl_lo.ensure(bytes);
    c->pl_scale.ensure(std::max<size_t>(16, (size_t)c->n * 4));
    const uint64_t blocks = std::max<uint64_t>(1, std::min<uint64_t>((c->n + 7) / 8, (uint64_t)c->sm_count * 16));
    planes_encode_kernel<<<(unsigned)blocks, 256, 0, c->stream>>>(items_f32(c), c->n, c->ld, c->pl_hi.as<int8_t>(), c->pl_lo.as<int8_t>(), c->pl_scale.as<float>());
    CK(cudaGetLastError());
    c->n_launches += 1;
    c->planes_valid = true;
}

// the bf16 source's per-item norms and gmax, built with the shadow
void frerank_prepare(arroy_ctx* c) {
    if (c->fr_valid) return;
    shadow_prepare(c);
    c->fr_norm.ensure(std::max<size_t>(16, c->n * 4));
    c->fr_gmax.ensure(4);
    launch_norms(c, c->items.as<float>(), c->n, c->fr_norm.as<float>(), nullptr);
    CK(cudaMemsetAsync(c->fr_gmax.p, 0, 4, c->stream));
    fr_gmax_kernel<<<(unsigned)((c->n + 255) / 256), 256, 0, c->stream>>>(c->fr_norm.as<float>(), c->h0.as<float>(), c->n, c->metric, c->fr_gmax.as<uint32_t>());
    CK(cudaGetLastError());
    c->n_launches += 2;
    c->fr_valid = true;
}

// launches the fused kernel with estimates from `src` for m queries whose sorted candidate rows are rows[beg[q] .. end[q]);
// results in s_orows / s_odist / s_olen, per-query status in fr_status (0 = done, 1 = needs the plain kernels). The plane source
// reads the planes, scales and headers on the device and needs nothing prepared.
void frerank_launch(arroy_ctx* c, int src, uint32_t m, const DevQueries& Q, const uint32_t* d_rows, const uint64_t* d_beg, const uint64_t* d_end,
                    uint32_t k) {
    c->fr_status.ensure(4ull * m);
    FrParams P{};
    P.items = items_f32(c); P.ih0 = c->h0.as<float>();
    P.d = c->dim; P.ld = c->ld; P.metric = c->metric;
    P.queries = Q.vecs; P.qrows = Q.rows; P.qh0 = Q.h0;
    P.rows = d_rows; P.seg_beg = d_beg; P.seg_end = d_end;
    P.k = k; P.hmin = cos_header_min(c->dim);
    P.out_rows = c->s_orows.as<uint32_t>(); P.out_dist = c->s_odist.as<float>(); P.out_len = c->s_olen.as<uint32_t>(); P.status = c->fr_status.as<int32_t>();
    if (src == FR_BF16) {
        frerank_prepare(c);
        P.shadow = c->fr_shadow.as<__nv_bfloat16>(); P.cnorm = c->fr_norm.as<float>();
        P.rel = fr_rel(c->dim); P.sub = fr_sub(c->dim); P.gmax_bits = c->fr_gmax.as<uint32_t>();
    } else {
        if (!c->pr_counts.p) { c->pr_counts.ensure(16); CK(cudaMemsetAsync(c->pr_counts.p, 0, 16, c->stream)); }
        P.hi = c->pl_hi.as<int8_t>(); P.lo = c->pl_lo.as<int8_t>(); P.scale = c->pl_scale.as<float>();
        fr_plane_consts(c->metric, c->dim, P);
        P.counts = c->pr_counts.as<unsigned long long>();
    }
    const auto kernel = src == FR_BF16 ? frerank_kernel<FR_BF16> : frerank_kernel<FR_PLANES>;
    const size_t smem = frerank_smem(c->ld);
    raise_smem_limit(c->device, (const void*)kernel, smem);
    kernel<<<m, FR_THREADS, smem, c->stream>>>(P);
    CK(cudaGetLastError());
    c->n_launches += 1;
    c->fr_batches[src] += 1;
}

// after the stream is idle: did every query of the batch from `src` finish in the fused kernel? (else counts a fallback)
bool frerank_ok(arroy_ctx* c, int src, uint32_t m) {
    std::vector<int32_t> st(m);
    CK(cudaMemcpy(st.data(), c->fr_status.p, 4ull * m, cudaMemcpyDeviceToHost));
    for (int32_t x : st) if (x != 0) { c->fr_fallbacks[src] += 1; return false; }
    return true;
}

// binary-quantized distances: normalized_distance divides by the index' dimensions (reader.rs:398); one pass over the results
void bq_normalize(arroy_ctx* c, float* d_dist, uint64_t count) {
    if (!is_bq(c->metric) || c->metric == BQ_COSINE || count == 0) return;
    bq_normalize_kernel<<<(unsigned)((count + 255) / 256), 256, 0, c->stream>>>(d_dist, count, c->metric, (float)c->user_dim);
    CK(cudaGetLastError());
    c->n_launches += 1;
}

// Event marks on the stream, in c->xev. Once the stream is idle, add_to(b) adds the time from mark i to mark i + 1 to b[i].
struct Marks {
    arroy_ctx* c;
    int n = 0;
    void operator()() { if (!c->xev[n]) c->xev[n] = new_event(); CK(cudaEventRecord(c->xev[n], c->stream)); ++n; }
    void add_to(double* b) const { for (int i = 0; i + 1 < n; ++i) { float ms = 0; CK(cudaEventElapsedTime(&ms, c->xev[i], c->xev[i + 1])); b[i] += ms; } }
};

// Uploads queries q0 .. q0 + m of a call: by item their rows into w_qrows, by vector their vectors into s_q (rows padded to ld
// with zeros). Their headers go to s_qh0: the caller's, else by item the stored header of the item, else zero.
DevQueries upload_queries(arroy_ctx* c, uint32_t q0, uint32_t m, const uint32_t* query_rows, const float* queries, const float* qhdr0) {
    const uint32_t ld = c->ld, d = c->dim;
    DevQueries Q;
    c->s_qh0.ensure(4ull * m);
    if (query_rows) {
        c->w_qrows.ensure(4ull * m);
        CK(cudaMemcpyAsync(c->w_qrows.p, query_rows + q0, 4ull * m, cudaMemcpyHostToDevice, c->stream));
        Q.rows = c->w_qrows.as<uint32_t>();
    } else {
        c->s_q.ensure((size_t)m * ld * 4);
        if (ld != d) CK(cudaMemsetAsync(c->s_q.p, 0, (size_t)m * ld * 4, c->stream));
        CK(cudaMemcpy2DAsync(c->s_q.p, (size_t)ld * 4, queries + (size_t)q0 * d, (size_t)d * 4, (size_t)d * 4, m, cudaMemcpyHostToDevice, c->stream));
        Q.vecs = c->s_q.as<float>();
    }
    if (qhdr0) CK(cudaMemcpyAsync(c->s_qh0.p, qhdr0 + q0, 4ull * m, cudaMemcpyHostToDevice, c->stream));
    else if (query_rows) { gather_f32_kernel<<<(m + 255) / 256, 256, 0, c->stream>>>(c->s_qh0.as<float>(), c->h0.as<float>(), Q.rows, m); CK(cudaGetLastError()); }
    else CK(cudaMemsetAsync(c->s_qh0.p, 0, 4ull * m, c->stream));
    Q.h0 = c->s_qh0.as<float>();
    if (is_bq(c->metric) && m) {   // the walks take the +-1 vector, the re-rank the bit string (ld = dim for these metrics)
        const uint32_t w32 = c->row_bytes / 4;
        c->s_qbits.ensure((size_t)m * c->row_bytes);
        const unsigned grid = (unsigned)std::min<uint64_t>(((uint64_t)m * ld + 255) / 256, (uint64_t)c->sm_count * 8);
        if (Q.rows) {
            c->s_q.ensure((size_t)m * ld * 4);
            bq_query_rows_kernel<<<grid, 256, 0, c->stream>>>(c->items.as<uint32_t>(), w32, Q.rows, m, ld, c->s_q.as<float>(), c->s_qbits.as<uint32_t>());
            Q.vecs = c->s_q.as<float>();
            Q.rows = nullptr;
        } else bq_pack_rows_kernel<<<grid, 256, 0, c->stream>>>(Q.vecs, ld, c->s_qbits.as<uint32_t>(), m, ld, w32);
        CK(cudaGetLastError());
        c->n_launches += 1;
        Q.bits = c->s_qbits.as<uint4>();
    }
    return Q;
}

// The re-rank of m queries whose sorted candidate rows are rows[beg[q] .. end[q]): at most max_len rows per query, n_keys rows
// in the whole array (s_keys / s_dists hold as many). Results in s_orows / s_odist / s_olen. With try_fused the fused kernel
// goes first, and the plain kernels run only if a query needs them: distance_kernel, then topk_kernel, or for k beyond the
// top-k buffer a full segmented sort of the keys and take_sorted_kernel. `mark`, when given, is recorded after the distances.
// (beg / end are not const: the key sort stays the CUB instantiation with uint64_t* offsets, as the walk's candidate sort)
void rerank_segments(arroy_ctx* c, uint32_t m, const DevQueries& Q, const uint32_t* rows, uint64_t* beg, uint64_t* end,
                     uint64_t n_keys, uint64_t max_len, uint32_t k, bool try_fused, Marks* mark) {
    const int src = try_fused ? frerank_source(c, k) : FR_NONE;
    if (src != FR_NONE) {   // one fused kernel per query: pre-filter + exact re-score + top-k (frerank.cuh)
        frerank_launch(c, src, m, Q, rows, beg, end, k);
        CK(cudaStreamSynchronize(c->stream));
        if (frerank_ok(c, src, m)) { if (mark) (*mark)(); return; }
    }
    if (max_len) {
        // (Manhattan sums one row per lane, the bit-string rows take four lanes per row, the other metrics eight)
        const uint64_t per = c->metric == MANHATTAN ? 32 : is_bq(c->metric) ? 8 : 4;
        const uint64_t warps = (max_len + per - 1) / per;
        const uint32_t gx = (uint32_t)std::max<uint64_t>(1, std::min<uint64_t>((warps + 7) / 8, std::max<uint64_t>(1, ((uint64_t)c->sm_count * 8) / std::min<uint32_t>(m, c->sm_count * 8u))));
        if (is_bq(c->metric))
            bq_distance_kernel<<<dim3(gx, m), 256, 0, c->stream>>>(c->items.as<uint4>(), c->h0.as<float>(), c->dim, c->metric, Q.bits, Q.h0, rows, beg, end,
                                                                  c->s_dists.as<float>(), c->s_keys.as<unsigned long long>());
        else
            distance_kernel<<<dim3(gx, m), 256, 0, c->stream>>>(items_f32(c), c->h0.as<float>(), c->dim, c->ld, c->metric, Q.vecs, Q.rows, Q.h0, m,
                                                               rows, beg, end, c->s_dists.as<float>(), c->s_keys.as<unsigned long long>());
        CK(cudaGetLastError());
    }
    if (mark) (*mark)();
    if (k > TOPK_CAP / 2) {
        c->s_keys2.ensure(std::max<uint64_t>(n_keys, 1) * 8);
        size_t tmp_bytes = 0;
        CK(cub::DeviceSegmentedSort::SortKeys(nullptr, tmp_bytes, c->s_keys.as<unsigned long long>(), c->s_keys2.as<unsigned long long>(), (int64_t)n_keys, (int64_t)m,
                                              beg, end, c->stream));
        c->w_tmp.ensure(std::max<size_t>(tmp_bytes, 16));
        CK(cub::DeviceSegmentedSort::SortKeys(c->w_tmp.p, tmp_bytes, c->s_keys.as<unsigned long long>(), c->s_keys2.as<unsigned long long>(), (int64_t)n_keys, (int64_t)m,
                                              beg, end, c->stream));
        take_sorted_kernel<<<m, 256, 0, c->stream>>>(c->s_keys2.as<unsigned long long>(), c->s_dists.as<float>(), rows, beg, end, k, c->metric,
                                                     c->s_orows.as<uint32_t>(), c->s_odist.as<float>(), c->s_olen.as<uint32_t>());
    } else
        topk_kernel<false><<<m, TOPK_THREADS, 0, c->stream>>>(c->s_keys.as<unsigned long long>(), c->s_dists.as<float>(), rows, beg, end, 0, k, c->metric,
                                                       c->s_orows.as<uint32_t>(), c->s_odist.as<float>(), c->s_olen.as<uint32_t>());
    CK(cudaGetLastError());
}

// The results of queries q0 .. q0 + m (k slots each) to the caller's arrays, with the walk status when out_status is given.
// The top-k kernels write only a query's first out_len slots; the others are set to 0 here, so that a result does not depend
// on what earlier calls left in the device buffers.
void copy_results(arroy_ctx* c, uint32_t q0, uint32_t m, uint32_t k, uint32_t* out_rows, float* out_dist, uint32_t* out_len, int32_t* out_status = nullptr) {
    CK(cudaMemcpyAsync(out_rows + (size_t)q0 * k, c->s_orows.p, 4ull * m * k, cudaMemcpyDeviceToHost, c->stream));
    CK(cudaMemcpyAsync(out_dist + (size_t)q0 * k, c->s_odist.p, 4ull * m * k, cudaMemcpyDeviceToHost, c->stream));
    CK(cudaMemcpyAsync(out_len + q0, c->s_olen.p, 4ull * m, cudaMemcpyDeviceToHost, c->stream));
    if (out_status) CK(cudaMemcpyAsync(out_status + q0, c->w_status.p, 4ull * m, cudaMemcpyDeviceToHost, c->stream));
    CK(cudaStreamSynchronize(c->stream));
    for (uint32_t q = q0; q < q0 + m; ++q) {
        const uint32_t len = std::min(out_len[q], k);
        memset(out_rows + (size_t)q * k + len, 0, 4ull * (k - len));
        memset(out_dist + (size_t)q * k + len, 0, 4ull * (k - len));
    }
}

void do_rerank_batch(arroy_ctx* c, uint32_t nq, const float* queries, const float* qh0, const uint32_t* rows, const uint64_t* offsets, uint32_t k,
                     uint32_t* out_rows, float* out_dist, uint32_t* out_len) {
    require_staged(c);
    set_device(c);
    if (nq == 0) return;
    if (k == 0) { for (uint32_t q = 0; q < nq; ++q) out_len[q] = 0; return; }
    if (nq > 65535) throw ArgError("at most 65535 queries per rerank_batch call");
    const uint64_t total = offsets[nq];
    if (total && !rows) throw ArgError("null rows");
    for (uint32_t q = 0; q < nq; ++q) {
        if (offsets[q + 1] < offsets[q]) throw ArgError("row_offsets must be non-decreasing");
        if (offsets[q + 1] - offsets[q] > 0xffffffffull) throw ArgError("too many candidates for one query");
    }
    for (uint64_t i = 0; i < total; ++i) if (rows[i] >= c->n) throw ArgError("row index out of range");
    c->s_off.ensure((size_t)(nq + 1) * 8);
    c->s_rows.ensure(std::max<uint64_t>(total, 1) * 4);
    c->s_keys.ensure(std::max<uint64_t>(total, 1) * 8);
    c->s_dists.ensure(std::max<uint64_t>(total, 1) * 4);
    c->s_orows.ensure((size_t)nq * k * 4);
    c->s_odist.ensure((size_t)nq * k * 4);
    c->s_olen.ensure((size_t)nq * 4);
    const DevQueries Q = upload_queries(c, 0, nq, nullptr, queries, qh0);
    CK(cudaMemcpyAsync(c->s_off.p, offsets, (size_t)(nq + 1) * 8, cudaMemcpyHostToDevice, c->stream));
    if (total) CK(cudaMemcpyAsync(c->s_rows.p, rows, total * 4, cudaMemcpyHostToDevice, c->stream));
    uint64_t max_c = 0;
    for (uint32_t q = 0; q < nq; ++q) max_c = std::max<uint64_t>(max_c, offsets[q + 1] - offsets[q]);
    // (the fused kernel's (distance, id) tie-break needs each query's rows ascending; the callers of this path pass sorted lists)
    rerank_segments(c, nq, Q, c->s_rows.as<uint32_t>(), c->s_off.as<uint64_t>(), c->s_off.as<uint64_t>() + 1, total, max_c, k,
                    total >= 512ull * nq && max_c <= (uint64_t)FR_CAP, nullptr);
    c->n_launches += total ? 2 : 1;
    bq_normalize(c, c->s_odist.as<float>(), (uint64_t)nq * k);
    c->h2d_bytes += (uint64_t)nq * c->dim * 4 + (uint64_t)nq * 4 + (uint64_t)(nq + 1) * 8 + total * 4;
    c->d2h_bytes += (uint64_t)nq * k * 8 + (uint64_t)nq * 4;
    copy_results(c, 0, nq, k, out_rows, out_dist, out_len);
}

// single-CTA create_split over a host row list (exposes D::create_split for parity tests and for
// hosts that keep the DFS on their side)
template <bool SMEM_WS, int METRIC>
__global__ void __launch_bounds__(CTRL_THREADS, 1) create_split_kernel(BuildParams P, const uint32_t* rows, uint32_t len, const uint32_t* key8, uint64_t pos, float* slot, uint64_t* out_pos) {
    extern __shared__ __align__(16) unsigned char cs_smem[];
    __shared__ TwoMeansShared TM;
    __shared__ Rng rng;
    if (threadIdx.x == 0) rng.init(key8, pos);
    __syncthreads();
    if (SMEM_WS) create_split_cta<METRIC>(P, rng, rows, len, reinterpret_cast<float*>(cs_smem), TM, slot);
    else create_split_cta<METRIC>(P, rng, rows, len, P.scratch, TM, slot);
    if (threadIdx.x == 0) *out_pos = rng.pos;
}

template <class F>
int32_t guarded(arroy_ctx* c, F&& f) {
    if (!c) return ARROY_B200_ERR_INVALID;
    std::lock_guard<std::mutex> lk(c->mu);
    {   // an asynchronous fault of an EARLIER call must not be blamed on this one
        const cudaError_t pending = cudaPeekAtLastError();
        if (pending != cudaSuccess) { c->err = std::string("a CUDA error was already pending when this call started: ") + cudaGetErrorString(pending); return ARROY_B200_ERR_CUDA; }
    }
    try { f(); return ARROY_B200_OK; }
    catch (const CudaError& e) { c->err = e.what(); cudaGetLastError(); return ARROY_B200_ERR_CUDA; }
    catch (const ArgError& e) { c->err = e.what(); return ARROY_B200_ERR_INVALID; }
    catch (const CapacityError& e) { c->err = e.what(); return ARROY_B200_ERR_CAPACITY; }
    catch (const Cancelled& e) { c->err = e.what(); return ARROY_B200_ERR_CANCELLED; }
    catch (const NotStaged& e) { c->err = e.what(); return ARROY_B200_ERR_NOT_STAGED; }
    catch (const std::exception& e) { c->err = std::string("internal error: ") + e.what(); return ARROY_B200_ERR_INTERNAL; }
    catch (...) { c->err = "internal error: unknown exception"; return ARROY_B200_ERR_INTERNAL; }
}

}  // namespace

// ================================================================================================
// extern "C"
// ================================================================================================
extern "C" {

const char* arroy_b200_version(void) { return "arroy_b200 0.1.0 (sm_90a)"; }

int32_t arroy_b200_allocations(uint64_t out[5]) {
    if (!out) return ARROY_B200_ERR_INVALID;
    for (int i = 0; i < LIVE_N; ++i) out[i] = g_live[i].load(std::memory_order_relaxed);
    return ARROY_B200_OK;
}

int32_t arroy_b200_create(int32_t device, arroy_ctx** out) {
    if (!out) return ARROY_B200_ERR_INVALID;
    *out = nullptr;
    int count = 0;
    if (cudaGetDeviceCount(&count) != cudaSuccess || count <= 0 || device < 0 || device >= count) { cudaGetLastError(); return ARROY_B200_ERR_CUDA; }
    try {
        auto c = std::make_unique<arroy_ctx>();
        c->device = device;
        CK(cudaSetDevice(device));
        cudaDeviceProp prop;
        CK(cudaGetDeviceProperties(&prop, device));
        c->sm_count = prop.multiProcessorCount;
        c->stream = new_stream();
        c->ev0 = new_event();
        c->ev1 = new_event();
        c->side_stream = new_stream();
        c->ev_done = new_event(cudaEventDisableTiming);
        c->ev_p0 = new_event();
        c->ev_p1 = new_event();
        c->tev0 = new_event();
        c->tev1 = new_event();
        // fail loudly if the kernels were not built for this device
        cudaFuncAttributes fa;
        CK(cudaFuncGetAttributes(&fa, work_kernel<false>));
        *out = c.release();
    } catch (const std::exception& e) {
        fprintf(stderr, "arroy_b200_create: %s\n", e.what());
        cudaGetLastError();
        return ARROY_B200_ERR_CUDA;
    }
    return ARROY_B200_OK;
}

void arroy_b200_destroy(arroy_ctx* c) { delete c; }

const char* arroy_b200_last_error(arroy_ctx* c) { return c ? c->err.c_str() : "null context"; }

}  // extern "C"

namespace {

// h0 / h1 of the raw stored Leaf values: [tag 0x00][Header POD][vector], byte aligned only
void decode_leaf_headers(const uint8_t* const* leaf_values, uint64_t n, int hf, std::vector<float>& h0, std::vector<float>& h1) {
    h0.assign(n, 0.f); h1.assign(n, 0.f);
    std::atomic<int> bad{0};
    const unsigned nt = n < 65536 ? 1u : std::max(1u, std::min(16u, std::thread::hardware_concurrency()));
    auto hdrs = [&](uint64_t i0, uint64_t i1) {
        for (uint64_t i = i0; i < i1; ++i) {
            const uint8_t* v = leaf_values[i];
            if (!v || v[0] != 0) { bad = 1; return; }
            memcpy(&h0[i], v + 1, 4);
            if (hf == 2) memcpy(&h1[i], v + 5, 4);
        }
    };
    if (nt <= 1) hdrs(0, n);
    else { std::vector<std::thread> th; for (unsigned t = 0; t < nt; ++t) th.emplace_back(hdrs, n * t / nt, n * (t + 1) / nt); for (auto& x : th) x.join(); }
    if (bad.load()) throw ArgError("leaf value does not start with the Leaf tag 0x00");
}

void upload_headers(arroy_ctx* c, const std::vector<float>& h0, const std::vector<float>& h1) {
    const uint64_t n = c->n;
    if (n) {
        CK(cudaMemcpyAsync(c->h0.p, h0.data(), n * 4, cudaMemcpyHostToDevice, c->stream));
        CK(cudaMemcpyAsync(c->h1.p, h1.data(), n * 4, cudaMemcpyHostToDevice, c->stream));
    }
    CK(cudaStreamSynchronize(c->stream));
    c->h2d_bytes += 8 * n;
}

void stage_items_full(arroy_ctx* c, int32_t metric, uint32_t dim, uint64_t n, const uint32_t* ids, const uint8_t* const* leaf_values) {
    const uint64_t h2d0 = c->h2d_bytes;
    alloc_items(c, metric, dim, n, ids, true);
    const int hf = metric_header_floats(metric);
    std::vector<float> h0, h1;
    decode_leaf_headers(leaf_values, n, hf, h0, h1);
    const size_t voff = 1 + 4 * (size_t)hf;
    // binary-quantized leaves store the bit string (node.rs:224-228 with VectorCodec = BinaryQuantized)
    stage_rows_pipeline(c, n, c->dim, c->row_bytes, [&](uint64_t i) { return leaf_values[i] + voff; }, nullptr, 0, true, is_bq(metric) ? 2 : 0);
    upload_headers(c, h0, h1);
    c->staged = true;
    c->stage_stats[0] = n; c->stage_stats[1] = 0; c->stage_stats[2] = 0; c->stage_stats[3] = c->h2d_bytes - h2d0;
}

constexpr size_t RESTAGE_SCRATCH_BYTES = 192ull << 20;   // with DevBuf's slack: at most 240 MB + 256 bytes, whatever the index size
constexpr size_t RESTAGE_PIECE_BYTES = 64ull << 10;

void launch_restage(arroy_ctx* c, const RestagePiece* pieces, uint64_t n_pieces, uint4* scratch, int phase) {
    if (n_pieces == 0) return;
    const unsigned grid = (unsigned)std::min<uint64_t>(n_pieces, (uint64_t)c->sm_count * 8);
    restage_copy_rows_kernel<<<grid, RESTAGE_THREADS, 0, c->stream>>>(c->items.as<uint4>(), scratch, pieces, n_pieces, c->row_bytes / 16, phase);
    CK(cudaGetLastError());
    c->n_launches += 1;
}

// The delta path of arroy_b200_stage_items_delta; false = one of the conditions for it does not hold (nothing was changed).
bool stage_items_delta(arroy_ctx* c, int32_t metric, uint32_t dim, uint64_t n, const uint32_t* ids, const uint8_t* const* leaf_values, uint64_t n_changed,
                       const uint32_t* changed_ids) {
    if (!c->staged || c->staging_open || n == 0 || c->n == 0 || c->host_items) return false;
    if (metric != c->metric || dim != c->user_dim) return false;   // row_bytes follows from the two
    if ((size_t)n * c->row_bytes > c->items.cap) return false;     // the resident buffer cannot hold the new matrix
    std::vector<int64_t> src(n);
    const uint64_t n_upload = stage_delta_plan(c->ids.data(), c->n, ids, n, changed_ids, n_changed, src.data());
    if (n_upload * 4 > n) return false;   // more than a quarter of the matrix crosses PCIe anyway: the plain pipeline is as good
    const uint64_t window_rows = std::max<uint64_t>(1, RESTAGE_SCRATCH_BYTES / c->row_bytes), piece_rows = std::max<uint64_t>(1, RESTAGE_PIECE_BYTES / c->row_bytes);
    const RestagePieces mv = restage_move_pieces(src.data(), n, window_rows, piece_rows), up = restage_upload_pieces(src.data(), n, window_rows, piece_rows);
    const int hf = metric_header_floats(metric);
    std::vector<float> h0, h1;
    decode_leaf_headers(leaf_values, n, hf, h0, h1);
    // scratch for one window, freed when this call returns: a card filled by its index has no room to lend for longer
    DevBuf scratch, d_pieces;
    const uint64_t n_pieces = mv.pieces.size() + up.pieces.size();
    if (n_pieces) {
        try {
            scratch.ensure(std::min<size_t>(RESTAGE_SCRATCH_BYTES, (size_t)std::min<uint64_t>(window_rows, std::max(mv.rows, up.rows)) * c->row_bytes));
            d_pieces.ensure(n_pieces * sizeof(RestagePiece));
        } catch (const CudaError&) { cudaGetLastError(); return false; }   // no room for the scratch: the full staging needs none
    }
    // from here on the context changes: the derived state follows rows, not ids
    const uint64_t h2d0 = c->h2d_bytes;
    forget_staged(c);
    c->n = n;
    c->ids.assign(ids, ids + n);
    CK(cudaStreamSynchronize(c->stream));   // h0 / h1 may be reallocated: nothing may still read them
    c->h0.ensure(std::max<size_t>(16, n * 4));
    c->h1.ensure(std::max<size_t>(16, n * 4));
    if (n_pieces) {
        RestagePiece* dp = d_pieces.as<RestagePiece>();
        if (!mv.pieces.empty()) CK(cudaMemcpyAsync(dp, mv.pieces.data(), mv.pieces.size() * sizeof(RestagePiece), cudaMemcpyHostToDevice, c->stream));
        if (!up.pieces.empty()) CK(cudaMemcpyAsync(dp + mv.pieces.size(), up.pieces.data(), up.pieces.size() * sizeof(RestagePiece), cudaMemcpyHostToDevice, c->stream));
        c->h2d_bytes += n_pieces * sizeof(RestagePiece);
        for (const RestageWindow& w : mv.windows) {
            launch_restage(c, dp + w.piece0, w.n_pieces, scratch.as<uint4>(), 0);
            launch_restage(c, dp + w.piece0, w.n_pieces, scratch.as<uint4>(), 1);
        }
        // the uploaded rows, after every move (they overwrite rows the moves read): host -> scratch through the bounce buffers of
        // the staging pipeline, scratch -> their rows
        std::vector<uint64_t> up_rows;
        up_rows.reserve(n_upload);
        for (uint64_t r = 0; r < n; ++r) if (src[r] < 0) up_rows.push_back(r);
        const size_t voff = 1 + 4 * (size_t)hf;
        uint64_t k0 = 0;
        for (const RestageWindow& w : up.windows) {
            uint64_t rows = 0;
            for (uint64_t p = 0; p < w.n_pieces; ++p) rows += up.pieces[w.piece0 + p].len;
            stage_rows_pipeline(c, rows, c->dim, c->row_bytes, [&](uint64_t i) { return leaf_values[up_rows[k0 + i]] + voff; }, scratch.as<uint8_t>(), 0, true,
                                is_bq(metric) ? 2 : 0);
            launch_restage(c, dp + mv.pieces.size() + w.piece0, w.n_pieces, scratch.as<uint4>(), 1);
            k0 += rows;
        }
    }
    upload_headers(c, h0, h1);   // ends in a stream synchronise: the scratch buffer is idle when it is freed
    c->staged = true;
    c->stage_stats[0] = n_upload; c->stage_stats[1] = mv.rows; c->stage_stats[2] = 1; c->stage_stats[3] = c->h2d_bytes - h2d0;
    return true;
}

}  // namespace

extern "C" {

int32_t arroy_b200_stage_items(arroy_ctx* c, int32_t metric, uint32_t dim, uint64_t n, const uint32_t* ids, const uint8_t* const* leaf_values) {
    return guarded(c, [&] {
        set_device(c);
        if (n && (!ids || !leaf_values)) throw ArgError("null ids / leaf_values");
        stage_items_full(c, metric, dim, n, ids, leaf_values);
    });
}

int32_t arroy_b200_stage_items_delta(arroy_ctx* c, int32_t metric, uint32_t dim, uint64_t n, const uint32_t* ids, const uint8_t* const* leaf_values, uint64_t n_changed,
                                     const uint32_t* changed_ids) {
    return guarded(c, [&] {
        set_device(c);
        if (n && (!ids || !leaf_values)) throw ArgError("null ids / leaf_values");
        if (n_changed && !changed_ids) throw ArgError("null changed_ids");
        if (n > 0xffffffffull) throw ArgError("too many items");
        for (uint64_t i = 1; i < n; ++i) if (ids[i] <= ids[i - 1]) throw ArgError("ids must be strictly ascending");
        for (uint64_t i = 1; i < n_changed; ++i) if (changed_ids[i] <= changed_ids[i - 1]) throw ArgError("changed_ids must be strictly ascending");
        if (!stage_items_delta(c, metric, dim, n, ids, leaf_values, n_changed, changed_ids)) stage_items_full(c, metric, dim, n, ids, leaf_values);
    });
}

int32_t arroy_b200_stage_stats(arroy_ctx* c, uint64_t out[4]) {
    return guarded(c, [&] { if (!out) throw ArgError("null argument"); for (int i = 0; i < 4; ++i) out[i] = c->stage_stats[i]; });
}

int32_t arroy_b200_read_items(arroy_ctx* c, const uint32_t* rows, uint64_t n_rows, uint8_t* out) {
    return guarded(c, [&] {
        require_staged(c); set_device(c);
        if (n_rows == 0) return;
        if (!rows || !out) throw ArgError("null argument");
        for (uint64_t i = 0; i < n_rows; ++i) if (rows[i] >= c->n) throw ArgError("row index out of range");
        if (c->host_items) {   // host-placed rows: read where they are
            const uint8_t* src = static_cast<const uint8_t*>(c->host_rows.p);
            for (uint64_t i = 0; i < n_rows; ++i) memcpy(out + i * c->row_bytes, src + (size_t)rows[i] * c->row_bytes, c->row_bytes);
            return;
        }
        for (uint64_t i = 0; i < n_rows;) {   // one copy per run of consecutive rows
            uint64_t e = i + 1;
            while (e < n_rows && rows[e] == rows[e - 1] + 1) ++e;
            CK(cudaMemcpyAsync(out + i * c->row_bytes, c->items.as<uint8_t>() + (size_t)rows[i] * c->row_bytes, (e - i) * (size_t)c->row_bytes, cudaMemcpyDeviceToHost, c->stream));
            i = e;
        }
        CK(cudaStreamSynchronize(c->stream));
        c->d2h_bytes += n_rows * (uint64_t)c->row_bytes;
    });
}

uint64_t arroy_b200_stage_delta_plan(const uint32_t* old_ids, uint64_t n_old, const uint32_t* new_ids, uint64_t n_new, const uint32_t* changed_ids, uint64_t n_changed,
                                     int64_t* out_src) {
    return stage_delta_plan(old_ids, n_old, new_ids, n_new, changed_ids, n_changed, out_src);
}

uint32_t arroy_b200_item_placement_plan(int32_t metric, uint32_t dim, uint64_t n, uint64_t free_bytes) {
    return placement_plan(metric, dim, n, free_bytes);
}

int32_t arroy_b200_item_placement(arroy_ctx* c, uint64_t out[3]) {
    return guarded(c, [&] {
        if (!out) throw ArgError("null argument");
        require_staged(c);
        out[0] = c->host_items ? 1 : 0;
        out[1] = c->host_items ? c->pl_hi.cap + c->pl_lo.cap + c->pl_scale.cap : c->items.cap;
        out[2] = c->host_items ? c->host_rows.cap : 0;
    });
}

// ---- staging in pieces (multi-GPU: the H2D copy of chunk k + 1 overlaps the broadcast of chunk k) ---------------------------
int32_t arroy_b200_stage_begin(arroy_ctx* c, int32_t metric, uint32_t dim, uint64_t n, const uint32_t* ids) {
    return guarded(c, [&] {
        set_device(c);
        if (n && !ids) throw ArgError("null ids");
        alloc_items(c, metric, dim, n, ids);
        c->stage_h0.assign(n, 0.f); c->stage_h1.assign(n, 0.f);
        CK(cudaStreamSynchronize(c->stream));
        c->staging_open = true;
    });
}

int32_t arroy_b200_stage_rows(arroy_ctx* c, uint64_t row0, uint64_t n_rows, const uint8_t* const* leaf_values) {
    return guarded(c, [&] {
        set_device(c);
        if (!c->staging_open) throw NotStaged("arroy_b200_stage_rows without arroy_b200_stage_begin");
        if (row0 > c->n || n_rows > c->n - row0) throw ArgError("row range out of bounds");
        if (n_rows == 0) return;
        if (!leaf_values) throw ArgError("null leaf_values");
        const int hf = metric_header_floats(c->metric);
        for (uint64_t i = 0; i < n_rows; ++i) {
            const uint8_t* v = leaf_values[i];
            if (!v || v[0] != 0) throw ArgError("leaf value does not start with the Leaf tag 0x00");
            memcpy(&c->stage_h0[row0 + i], v + 1, 4);
            if (hf == 2) memcpy(&c->stage_h1[row0 + i], v + 5, 4);
        }
        const size_t voff = 1 + 4 * (size_t)hf;
        stage_rows_pipeline(c, n_rows, c->dim, c->row_bytes, [&](uint64_t i) { return leaf_values[i] + voff; }, c->items.as<uint8_t>() + (size_t)row0 * c->row_bytes, 0, true,
                            is_bq(c->metric) ? 2 : 0);
    });
}

int32_t arroy_b200_stage_end(arroy_ctx* c, int32_t headers_on_device) {
    return guarded(c, [&] {
        set_device(c);
        if (!c->staging_open) throw NotStaged("arroy_b200_stage_end without arroy_b200_stage_begin");
        if (!headers_on_device && c->n) {
            CK(cudaMemcpyAsync(c->h0.p, c->stage_h0.data(), c->n * 4, cudaMemcpyHostToDevice, c->stream));
            CK(cudaMemcpyAsync(c->h1.p, c->stage_h1.data(), c->n * 4, cudaMemcpyHostToDevice, c->stream));
            c->h2d_bytes += 8 * c->n;
        }
        CK(cudaStreamSynchronize(c->stream));
        c->stage_h0.clear(); c->stage_h0.shrink_to_fit(); c->stage_h1.clear(); c->stage_h1.shrink_to_fit();
        c->staging_open = false;
        c->staged = true;
    });
}

int32_t arroy_b200_stage_items_flat(arroy_ctx* c, int32_t metric, uint32_t dim, uint64_t n, const uint32_t* ids, const float* vectors, const float* hdr0, const float* hdr1) {
    return guarded(c, [&] {
        set_device(c);
        if (n && (!ids || !vectors)) throw ArgError("null ids / vectors");
        alloc_items(c, metric, dim, n, ids, true);
        if (n) {
            const uint8_t* base = reinterpret_cast<const uint8_t*>(vectors);
            const size_t stride = 4ull * dim;
            // host placement: the Cosine default headers (the norms) come out of the chunk encoder, which reads every row anyway
            const bool enc_norms = c->host_items && !hdr0 && metric == COSINE;
            // binary-quantized metrics: the f32 vectors are quantized on the way (Writer::add_item -> UnalignedVector::from_slice)
            stage_rows_pipeline(c, n, c->dim, c->row_bytes, [&](uint64_t i) { return base + i * stride; }, nullptr, 0, true, is_bq(metric) ? 1 : 0, dim,
                                enc_norms ? c->h0.as<float>() : nullptr);
            if (hdr0) CK(cudaMemcpyAsync(c->h0.p, hdr0, n * 4, cudaMemcpyHostToDevice, c->stream));
            else if (!enc_norms) default_headers(c);
            if (hdr1) CK(cudaMemcpyAsync(c->h1.p, hdr1, n * 4, cudaMemcpyHostToDevice, c->stream));
        }
        CK(cudaStreamSynchronize(c->stream));
        c->h2d_bytes += (hdr0 ? 4 * n : 0) + (hdr1 ? 4 * n : 0);
        c->staged = true;
    });
}

int32_t arroy_b200_stage_items_device(arroy_ctx* c, int32_t metric, uint32_t dim, uint64_t n, const uint32_t* ids, const void* device_vectors) {
    return guarded(c, [&] {
        set_device(c);
        if (n && (!ids || !device_vectors)) throw ArgError("null ids / vectors");
        alloc_items(c, metric, dim, n, ids);
        if (n && is_bq(metric)) {
            bq_pack_rows_kernel<<<c->sm_count * 8, 256, 0, c->stream>>>(static_cast<const float*>(device_vectors), dim, c->items.as<uint32_t>(), n, dim, c->row_bytes / 4);
            CK(cudaGetLastError());
            c->n_launches += 1;
            default_headers(c);
        } else if (n) {
            if (c->ld != dim) CK(cudaMemsetAsync(c->items.p, 0, (size_t)n * c->ld * 4, c->stream));
            CK(cudaMemcpy2DAsync(c->items.p, (size_t)c->ld * 4, device_vectors, (size_t)dim * 4, (size_t)dim * 4, n, cudaMemcpyDeviceToDevice, c->stream));
            default_headers(c);
        }
        CK(cudaStreamSynchronize(c->stream));
        c->staged = true;
    });
}

int32_t arroy_b200_item_headers(arroy_ctx* c, float* out_hdr0, float* out_hdr1) {
    return guarded(c, [&] {
        require_staged(c); set_device(c);
        if (c->n == 0) return;
        if (out_hdr0) CK(cudaMemcpyAsync(out_hdr0, c->h0.p, c->n * 4, cudaMemcpyDeviceToHost, c->stream));
        if (out_hdr1) CK(cudaMemcpyAsync(out_hdr1, c->h1.p, c->n * 4, cudaMemcpyDeviceToHost, c->stream));
        CK(cudaStreamSynchronize(c->stream));
    });
}

int32_t arroy_b200_dot_preprocess(arroy_ctx* c, float* out_extra_dim, float* out_norm) {
    return guarded(c, [&] {
        require_staged(c); set_device(c);
        if (c->metric != DOT_PRODUCT || c->n == 0) return;  // Distance::preprocess default: no-op (src/distance/mod.rs:112-119)
        compute_norms(c, true);
        dot_header_kernel<<<(unsigned)((c->n + 255) / 256), 256, 0, c->stream>>>(c->norms.as<float>(), c->n, c->maxbits.as<uint32_t>(), c->h0.as<float>(), c->h1.as<float>());
        CK(cudaGetLastError());
        if (out_extra_dim) CK(cudaMemcpyAsync(out_extra_dim, c->h0.p, c->n * 4, cudaMemcpyDeviceToHost, c->stream));
        if (out_norm) CK(cudaMemcpyAsync(out_norm, c->h1.p, c->n * 4, cudaMemcpyDeviceToHost, c->stream));
        CK(cudaStreamSynchronize(c->stream));
    });
}

int32_t arroy_b200_side_batch(arroy_ctx* c, const float* normal, float hdr0, float hdr1, const uint32_t* rows, uint64_t n_rows, uint8_t* out_side, float* out_margin) {
    return guarded(c, [&] {
        if (n_rows && (!normal || !rows || !out_side)) throw ArgError("null argument");
        do_side_batch(c, normal, hdr0, hdr1, rows, n_rows, out_side, out_margin);
    });
}

int32_t arroy_b200_side_multi(arroy_ctx* c, uint32_t n_jobs, const float* normals, const float* hdr0, const float* hdr1,
                              const uint32_t* rows, const uint64_t* row_offsets, uint8_t* out_side) {
    return guarded(c, [&] {
        (void)hdr1;
        require_staged(c); set_device(c);
        if (n_jobs == 0) return;
        if (!normals || !hdr0 || !rows || !row_offsets || !out_side) throw ArgError("null argument");
        const uint64_t total = row_offsets[n_jobs];
        for (uint32_t j = 0; j < n_jobs; ++j) if (row_offsets[j + 1] < row_offsets[j] || row_offsets[j + 1] - row_offsets[j] > 0xffffffffull) throw ArgError("bad row_offsets");
        for (uint64_t i = 0; i < total; ++i) if (rows[i] >= c->n) throw ArgError("row index out of range");
        if (total == 0) return;
        const uint32_t ld = c->ld, slot = ld + NORMAL_HDR;
        // Host-placed items: every job goes through the 8-bit planes (work_kernel_planes, no minimum size), so that only the rows
        // the planes cannot decide are read over PCIe; the flags are the f32 scan's.
        const bool planes = c->host_items;
        if (planes) planes_prepare(c);
        const size_t limb_smem = planes ? (size_t)PLANES_LIMBS * ld : 0;
        // jobs per launch bounded by the shared-memory unit-prefix table of work_kernel (and next to the limbs of work_kernel_planes)
        const uint32_t max_jobs = planes ? (uint32_t)std::min<size_t>(40000, (160 * 1024 - 4ull * ld - limb_smem) / 4 - 1) : 40000;
        c->s_rows.ensure(4ull * total);
        c->s_flags.ensure(total);
        CK(cudaMemcpyAsync(c->s_rows.p, rows, 4ull * total, cudaMemcpyHostToDevice, c->stream));
        std::vector<float> slots;
        std::vector<Job> jobs;
        for (uint32_t j0 = 0; j0 < n_jobs; j0 += max_jobs) {
            const uint32_t m = std::min(max_jobs, n_jobs - j0);
            slots.assign((size_t)m * slot, 0.f);
            jobs.assign(m, Job{});
            c->s_normal.ensure((size_t)m * slot * 4);
            c->s_job.ensure(sizeof(Job) * m);
            uint64_t units = 0;
            for (uint32_t j = 0; j < m; ++j) {
                float* sp = slots.data() + (size_t)j * slot;
                sp[0] = hdr0[j0 + j];
                memcpy(sp + NORMAL_HDR, normals + (size_t)(j0 + j) * c->dim, 4ull * c->dim);
                Job& jb = jobs[j];
                const uint64_t b = row_offsets[j0 + j], len = row_offsets[j0 + j + 1] - b;
                jb.kind = len ? JOB_SCAN : JOB_NONE; jb.len = (uint32_t)len;
                jb.rows = c->s_rows.as<uint32_t>() + b; jb.normal = c->s_normal.as<float>() + (size_t)j * slot;
                jb.flags = c->s_flags.as<uint8_t>() + b; jb.margins = nullptr; jb.unit_left = nullptr;
                units += (len + SCAN_UNIT - 1) / SCAN_UNIT;
            }
            CK(cudaMemcpyAsync(c->s_normal.p, slots.data(), slots.size() * 4, cudaMemcpyHostToDevice, c->stream));
            CK(cudaMemcpyAsync(c->s_job.p, jobs.data(), sizeof(Job) * m, cudaMemcpyHostToDevice, c->stream));
            const int grid = (int)std::max<uint64_t>(1, std::min<uint64_t>(units, (uint64_t)c->sm_count * 3));
            const ScanPlanes all{0u, nullptr};
            launch_scan(c, c->stream, c->s_job.as<Job>(), (int)m, (unsigned)(planes ? std::min<int>(grid, c->sm_count * 2) : grid), planes ? &all : nullptr);
            CK(cudaGetLastError());
            c->n_launches += 1;
            CK(cudaStreamSynchronize(c->stream));   // slots / jobs host vectors are reused by the next chunk
        }
        CK(cudaMemcpyAsync(out_side, c->s_flags.p, total, cudaMemcpyDeviceToHost, c->stream));
        CK(cudaStreamSynchronize(c->stream));
        c->h2d_bytes += 4ull * total + (uint64_t)n_jobs * slot * 4;
        c->d2h_bytes += total;
    });
}

int32_t arroy_b200_create_split(arroy_ctx* c, const uint32_t rng_key[8], uint64_t* rng_word_pos, const uint32_t* rows, uint64_t n_rows, float* out_normal, float* out_hdr) {
    return guarded(c, [&] {
        require_staged(c); set_device(c);
        if (!rng_key || !rng_word_pos || !rows || !out_normal || !out_hdr) throw ArgError("null argument");
        if (n_rows < 2 || n_rows > 0xffffffffull) throw ArgError("create_split needs at least two rows");
        for (uint64_t i = 0; i < n_rows; ++i) { if (rows[i] >= c->n) throw ArgError("row index out of range"); if (i && rows[i] <= rows[i - 1]) throw ArgError("rows must be ascending"); }
        const uint32_t ld = c->ld;
        c->s_rows.ensure(n_rows * 4);
        c->s_normal.ensure((size_t)(ld + NORMAL_HDR) * 4);
        c->s_misc.ensure(64 + (size_t)WS_VECS * ld * 4);
        CK(cudaMemcpyAsync(c->s_rows.p, rows, n_rows * 4, cudaMemcpyHostToDevice, c->stream));
        CK(cudaMemcpyAsync(c->s_misc.p, rng_key, 32, cudaMemcpyHostToDevice, c->stream));
        BuildParams P{};
        P.items = items_f32(c); P.ih0 = c->h0.as<float>(); P.ih1 = c->h1.as<float>();
        P.n = (uint32_t)c->n; P.d = c->dim; P.ld = ld; P.metric = c->metric;
        const TwoMeansWs ws = two_means_ws(ld);
        P.use_smem_ws = ws.smem; P.spec = ws.spec;
        P.scratch = reinterpret_cast<float*>(c->s_misc.as<uint8_t>() + 64);
        const size_t smem = ws.smem ? ws.bytes : 0;
        const void* fn = with_metric(c->metric, [&](auto m) {
            return ws.smem ? (const void*)&create_split_kernel<true, decltype(m)::value> : (const void*)&create_split_kernel<false, decltype(m)::value>;
        });
        raise_smem_limit(c->device, fn, smem);
        {
            const uint32_t* d_rows = c->s_rows.as<uint32_t>(); uint32_t len32 = (uint32_t)n_rows; const uint32_t* d_key = c->s_misc.as<uint32_t>(); uint64_t pos0 = *rng_word_pos;
            float* d_slot = c->s_normal.as<float>(); uint64_t* d_pos = reinterpret_cast<uint64_t*>(c->s_misc.as<uint8_t>() + 32);
            void* args[7] = {&P, &d_rows, &len32, &d_key, &pos0, &d_slot, &d_pos};
            CK(cudaLaunchKernel(fn, dim3(1), dim3(CTRL_THREADS), args, smem, c->stream));
        }
        CK(cudaGetLastError());
        std::vector<float> slot(ld + NORMAL_HDR);
        uint64_t new_pos = 0;
        CK(cudaMemcpyAsync(slot.data(), c->s_normal.p, slot.size() * 4, cudaMemcpyDeviceToHost, c->stream));
        CK(cudaMemcpyAsync(&new_pos, c->s_misc.as<uint8_t>() + 32, 8, cudaMemcpyDeviceToHost, c->stream));
        CK(cudaStreamSynchronize(c->stream));
        memcpy(out_normal, slot.data() + NORMAL_HDR, 4ull * c->dim);
        out_hdr[0] = slot[0]; out_hdr[1] = slot[1];
        *rng_word_pos = new_pos;
    });
}

int32_t arroy_b200_build_trees(arroy_ctx* c, uint32_t n_trees, const uint8_t (*tree_seeds)[32], const uint32_t* root_ids, uint32_t first_free_node_id,
                               uint32_t split_after, arroy_b200_cancel_fn cancel, void* cancel_arg, arroy_b200_node_sink sink, void* sink_arg, uint64_t* out_n_nodes) {
    return guarded(c, [&] {
        if (n_trees && (!tree_seeds || !root_ids)) throw ArgError("null seeds / root ids");
        do_build(c, n_trees, tree_seeds, root_ids, first_free_node_id, split_after, cancel, cancel_arg, sink, sink_arg, out_n_nodes);
    });
}

int32_t arroy_b200_build_trees_begin(arroy_ctx* c, uint32_t n_trees, const uint8_t (*tree_seeds)[32], uint32_t split_after,
                                     arroy_b200_cancel_fn cancel, void* cancel_arg, uint32_t* out_node_counts) {
    return guarded(c, [&] {
        if (n_trees && !tree_seeds) throw ArgError("null seeds");
        do_build_begin(c, n_trees, tree_seeds, split_after, cancel, cancel_arg, out_node_counts);
    });
}
int32_t arroy_b200_build_trees_emit(arroy_ctx* c, const uint32_t* root_ids, const uint64_t* base_ids, arroy_b200_node_sink sink, void* sink_arg) {
    return guarded(c, [&] {
        if (c->pending_n_trees && (!root_ids || !base_ids)) throw ArgError("null root / base ids");
        do_build_emit(c, root_ids, base_ids, sink, sink_arg);
    });
}

int32_t arroy_b200_build_subtrees_begin(arroy_ctx* c, uint32_t n_subtrees, const uint8_t (*seeds)[32], const uint32_t* rows, const uint64_t* row_offsets,
                                        uint32_t split_after, arroy_b200_cancel_fn cancel, void* cancel_arg, uint32_t* out_node_counts) {
    return guarded(c, [&] {
        if (n_subtrees && (!seeds || !rows || !row_offsets)) throw ArgError("null argument");
        Subsets sub; sub.rows = rows; sub.off = row_offsets;
        do_build_begin(c, n_subtrees, seeds, split_after, cancel, cancel_arg, out_node_counts, sub);
    });
}
int32_t arroy_b200_build_subtrees_begin_at(arroy_ctx* c, uint32_t n_subtrees, const uint8_t (*seeds)[32], const uint64_t* start_pos, const uint32_t* rows,
                                           const uint64_t* row_offsets, uint32_t split_after, arroy_b200_cancel_fn cancel, void* cancel_arg,
                                           uint32_t* out_node_counts, uint64_t* out_end_pos) {
    return guarded(c, [&] {
        if (n_subtrees && (!seeds || !rows || !row_offsets)) throw ArgError("null argument");
        Subsets sub; sub.rows = rows; sub.off = row_offsets; sub.start_pos = start_pos; sub.end_pos = out_end_pos;
        do_build_begin(c, n_subtrees, seeds, split_after, cancel, cancel_arg, out_node_counts, sub);
    });
}
int32_t arroy_b200_build_trees_emit_mapped(arroy_ctx* c, const uint32_t* root_ids, const uint32_t* node_ids, arroy_b200_node_sink sink, void* sink_arg) {
    return guarded(c, [&] {
        if (c->pending_n_trees && (!root_ids || !node_ids)) throw ArgError("null root / node ids");
        do_build_emit(c, root_ids, nullptr, sink, sink_arg, node_ids);
    });
}

int32_t arroy_b200_build_stats(arroy_ctx* c, double stats[8]) {
    return guarded(c, [&] { for (int i = 0; i < 8; ++i) stats[i] = c->stats[i]; });
}
int32_t arroy_b200_build_shadow_stats(arroy_ctx* c, uint64_t out[4]) {
    return guarded(c, [&] { if (!out) throw ArgError("null argument"); out[0] = c->shadow_rows; out[1] = c->shadow_rescored; out[2] = c->fused_root_rows; out[3] = c->fused_root_read; });
}
int32_t arroy_b200_build_prefilter_stats(arroy_ctx* c, uint64_t out[5]) {
    return guarded(c, [&] {
        if (!out) throw ArgError("null argument");
        out[0] = c->shadow_rows; out[1] = c->shadow_stage2; out[2] = c->shadow_rescored; out[3] = c->fused_root_rows; out[4] = c->fused_root_read;
    });
}
int32_t arroy_b200_prefilter_planes(arroy_ctx* c, int8_t* hi, int8_t* lo, float* scale) {
    return guarded(c, [&] {
        if (!hi || !lo || !scale) throw ArgError("null argument");
        require_staged(c);
        if (is_bq(c->metric)) throw ArgError("prefilter_planes needs a float metric (binary-quantized items are bit strings)");
        set_device(c);
        planes_prepare(c);
        const size_t bytes = (size_t)c->n * c->ld;
        CK(cudaMemcpyAsync(hi, c->pl_hi.p, bytes, cudaMemcpyDeviceToHost, c->stream));
        CK(cudaMemcpyAsync(lo, c->pl_lo.p, bytes, cudaMemcpyDeviceToHost, c->stream));
        CK(cudaMemcpyAsync(scale, c->pl_scale.p, (size_t)c->n * 4, cudaMemcpyDeviceToHost, c->stream));
        CK(cudaStreamSynchronize(c->stream));
    });
}

int32_t arroy_b200_rerank(arroy_ctx* c, const float* query, float qhdr0, float qhdr1, const uint32_t* rows, uint64_t n_rows, uint32_t k,
                          uint32_t* out_rows, float* out_dist, uint32_t* out_len) {
    return guarded(c, [&] {
        if (!query || (n_rows && !rows) || !out_len) throw ArgError("null argument");
        uint64_t offs[2] = {0, n_rows};
        do_rerank_batch(c, 1, query, &qhdr0, rows, offs, k, out_rows, out_dist, out_len);
    });
}

int32_t arroy_b200_rerank_batch(arroy_ctx* c, uint32_t nq, const float* queries, const float* qhdr0, const float* qhdr1, const uint32_t* rows,
                                const uint64_t* row_offsets, uint32_t k, uint32_t* out_rows, float* out_dist, uint32_t* out_len) {
    return guarded(c, [&] {
        if (nq && (!queries || !row_offsets || !out_len)) throw ArgError("null argument");
        do_rerank_batch(c, nq, queries, qhdr0, rows, row_offsets, k, out_rows, out_dist, out_len);
    });
}

int32_t arroy_b200_rerank_shared(arroy_ctx* c, uint32_t nq, const float* queries, const float* qhdr0, const uint32_t* rows, uint64_t n_rows,
                                 uint32_t k, uint32_t* out_rows, float* out_dist, uint32_t* out_len) {
    return guarded(c, [&] {
        require_staged(c); set_device(c);
        if (nq == 0) return;
        if (!queries || (n_rows && !rows) || !out_len) throw ArgError("null argument");
        if (k == 0 || n_rows == 0) { for (uint32_t q = 0; q < nq; ++q) out_len[q] = 0; return; }
        if (n_rows > 0x7fffffffull) throw ArgError("too many candidates");
        for (uint64_t i = 0; i < n_rows; ++i) { if (rows[i] >= c->n) throw ArgError("row index out of range"); if (i && rows[i] <= rows[i - 1]) throw ArgError("rows must be ascending and unique"); }
        if (c->metric == MANHATTAN || is_bq(c->metric) || c->dim < 32 || k > TOPK_CAP / 2) {
            // sequential-sum metric / SSE + scalar paths / k beyond the top-k buffer: generic per-pair kernels over replicated row lists
            if ((uint64_t)nq * n_rows > (1ull << 28)) throw ArgError("rerank_shared: this metric / dimension only supports nq * n_rows <= 2^28");
            std::vector<uint32_t> rep((size_t)nq * n_rows);
            std::vector<uint64_t> offs(nq + 1);
            for (uint32_t q = 0; q <= nq; ++q) offs[q] = (uint64_t)q * n_rows;
            for (uint32_t q = 0; q < nq; ++q) memcpy(rep.data() + (size_t)q * n_rows, rows, 4 * n_rows);
            do_rerank_batch(c, nq, queries, qhdr0, rep.data(), offs.data(), k, out_rows, out_dist, out_len);
            return;
        }
        const uint32_t ld = c->ld, nc = (uint32_t)n_rows;
        for (double& x : c->xbreak) x = 0;
        c->s_rows.ensure(4ull * nc);
        CK(cudaMemcpyAsync(c->s_rows.p, rows, 4ull * nc, cudaMemcpyHostToDevice, c->stream));
        // ARROY_B200_XRERANK = exact | filter; default: the tensor-core pre-filter once the problem is big enough to pay for it
        const char* mode = getenv("ARROY_B200_XRERANK");
        bool filter = mode ? strcmp(mode, "filter") == 0 : ((uint64_t)nq * nc >= (1ull << 22) && nc >= 4u * k);
        const uint32_t cap = std::max<uint32_t>(1024u, 4u * k);
        const uint32_t lds = (nc + 3u) & ~3u;   // pitch of the score matrix
        const float* cand = nullptr;   // nc x ld candidate matrix for the GEMM
        if (filter) {
            cand = xf_candidates(c, rows, nc);
            c->x_cnorm.ensure(4ull * nc);
            launch_norms(c, cand, nc, c->x_cnorm.as<float>(), nullptr);
            c->x_ca.ensure(4ull * nc); c->x_cb.ensure(4ull * nc); c->x_gmax.ensure(4);
            CK(cudaMemsetAsync(c->x_gmax.p, 0, 4, c->stream));
            xf_cand_prep_kernel<<<(nc + 255) / 256, 256, 0, c->stream>>>(c->x_cnorm.as<float>(), c->h0.as<float>(), c->s_rows.as<uint32_t>(), nc, c->metric, cos_header_min(c->dim),
                                                                         c->x_ca.as<float>(), c->x_cb.as<float>(), c->x_gmax.as<uint32_t>());
            CK(cudaGetLastError());
            c->n_launches += 2;
            c->x_flag.ensure(4);
        }
        // queries in chunks so the dense score / distance matrix stays <= 2 GiB
        const uint32_t chunk = (uint32_t)std::max<uint64_t>(XQB, std::min<uint64_t>(nq, ((2ull << 30) / (4ull * lds)) / XQB * XQB));
        for (uint32_t q0 = 0; q0 < nq; q0 += chunk) {
            const uint32_t m = std::min(chunk, nq - q0);
            c->s_orows.ensure(4ull * m * k); c->s_odist.ensure(4ull * m * k); c->s_olen.ensure(4ull * m);
            // (a pinned multi-thread bounce of the 12.6 MB of config 5 was measured: not faster than the driver's own staging)
            const DevQueries Q = upload_queries(c, q0, m, nullptr, queries, qhdr0);
            bool done = false;
            Marks mark{c};
            if (filter) {
                c->xf_calls += 1;
                mark();
                c->x_S.ensure(4ull * m * lds); c->x_qnorm.ensure(4ull * m); c->x_qa.ensure(4ull * m); c->x_qb.ensure(4ull * m); c->x_twoe.ensure(4ull * m);
                c->x_sel.ensure(4ull * m * cap); c->x_beg.ensure(8ull * m); c->x_end.ensure(8ull * m);
                c->s_dists.ensure(4ull * m * cap); c->s_keys.ensure(8ull * m * cap);
                launch_norms(c, Q.vecs, m, c->x_qnorm.as<float>(), nullptr);
                xf_query_prep_kernel<<<(m + 255) / 256, 256, 0, c->stream>>>(c->x_qnorm.as<float>(), Q.h0, m, c->metric, xf_rel(c->dim), c->dim, c->x_gmax.as<uint32_t>(),
                                                                             c->x_qa.as<float>(), c->x_qb.as<float>(), c->x_twoe.as<float>());
                CK(cudaGetLastError());
                mark();
                // A (m x nc, row-major) = distance estimates: Q . cand^T on the tensor cores (TF32 inputs, FP32 accumulate) + fused epilogue
                TgEpilogue ep{c->metric == EUCLIDEAN ? TG_EUCLID : (c->metric == COSINE ? TG_COSINE : TG_NEG), c->x_qa.as<float>(), c->x_qb.as<float>(), c->x_ca.as<float>(), c->x_cb.as<float>()};
                xf_scores(c, Q.vecs, m, cand, nc, c->x_S.as<float>(), lds, ep, xf_engine());
                mark();
                CK(cudaMemsetAsync(c->x_flag.p, 0, 4, c->stream));
                xf_select_kernel<<<m, XF_THREADS, 0, c->stream>>>(c->x_S.as<float>(), lds, nc, k, c->x_twoe.as<float>(), c->s_rows.as<uint32_t>(), cap,
                                                                  c->x_sel.as<uint32_t>(), c->x_beg.as<uint64_t>(), c->x_end.as<uint64_t>(), c->x_flag.as<int>());
                CK(cudaGetLastError());
                mark();
                // exact re-score of the survivors, in the reference's summation order
                rerank_segments(c, m, Q, c->x_sel.as<uint32_t>(), c->x_beg.as<uint64_t>(), c->x_end.as<uint64_t>(), (uint64_t)m * cap, cap, k, false, &mark);
                c->n_launches += 6;
                mark();
                int flag = 0;
                CK(cudaMemcpyAsync(&flag, c->x_flag.p, 4, cudaMemcpyDeviceToHost, c->stream));
                CK(cudaStreamSynchronize(c->stream));
                mark.add_to(c->xbreak);
                done = flag == 0;
                { std::vector<uint64_t> ends(m); CK(cudaMemcpy(ends.data(), c->x_end.p, 8ull * m, cudaMemcpyDeviceToHost));
                  for (uint32_t q = 0; q < m; ++q) c->xf_selected += ends[q] - (uint64_t)q * cap; c->xf_queries += m; }
                if (!done) c->xf_fallbacks += 1;   // more survivors than `cap` for some query: take the exact path for this chunk
            }
            if (!done) {
                c->s_dists.ensure(4ull * m * nc);
                mark.n = 0; mark();
                // the kernel stages its operands with cp.async, which takes device memory: host-placed items are read from the
                // gathered candidates (candidate i at row i, its header gathered alongside)
                const float* x_items = c->items.as<float>();
                const float* x_h0 = c->h0.as<float>();
                const uint32_t* x_rows = c->s_rows.as<uint32_t>();
                if (c->host_items) {
                    if (!cand) cand = xf_candidates(c, rows, nc);
                    c->x_gh0.ensure(4ull * nc); c->x_iota.ensure(4ull * nc);
                    gather_f32_kernel<<<(nc + 255) / 256, 256, 0, c->stream>>>(c->x_gh0.as<float>(), c->h0.as<float>(), c->s_rows.as<uint32_t>(), nc);
                    iota_u32_kernel<<<(unsigned)std::min<uint64_t>((nc + 255) / 256, (uint64_t)c->sm_count * 8), 256, 0, c->stream>>>(c->x_iota.as<uint32_t>(), nc);
                    CK(cudaGetLastError());
                    c->n_launches += 2;
                    x_items = cand; x_h0 = c->x_gh0.as<float>(); x_rows = c->x_iota.as<uint32_t>();
                }
                dim3 grid((nc + XCB - 1) / XCB, (m + XQB - 1) / XQB);
                if (c->metric == EUCLIDEAN)
                    xrerank_kernel<true><<<grid, XTHREADS, 0, c->stream>>>(x_items, x_h0, c->dim, ld, c->metric, Q.vecs, Q.h0, m, x_rows, nc, c->s_dists.as<float>());
                else
                    xrerank_kernel<false><<<grid, XTHREADS, 0, c->stream>>>(x_items, x_h0, c->dim, ld, c->metric, Q.vecs, Q.h0, m, x_rows, nc, c->s_dists.as<float>());
                CK(cudaGetLastError());
                topk_kernel<true><<<m, TOPK_THREADS, 0, c->stream>>>(nullptr, c->s_dists.as<float>(), c->s_rows.as<uint32_t>(), nullptr, nullptr, nc, k, c->metric,
                                                                     c->s_orows.as<uint32_t>(), c->s_odist.as<float>(), c->s_olen.as<uint32_t>());
                CK(cudaGetLastError());
                c->n_launches += 2;
                mark();
                CK(cudaStreamSynchronize(c->stream));
                mark.add_to(c->xbreak + 5);
            }
            copy_results(c, q0, m, k, out_rows, out_dist, out_len);
        }
        c->h2d_bytes += (uint64_t)nq * c->dim * 4 + 4ull * nc;
        c->d2h_bytes += 8ull * nq * k + 4ull * nq;
    });
}

int32_t arroy_b200_load_forest(arroy_ctx* c, uint32_t n_nodes, const uint8_t* kind, const uint32_t* left, const uint32_t* right,
                               const uint32_t* normal_idx, const float* normal_hdr0, const uint32_t* desc_off, const uint32_t* desc_len,
                               uint32_t n_normals, const float* normals, uint64_t n_desc, const uint32_t* desc_rows,
                               uint32_t n_roots, const uint32_t* roots) {
    return guarded(c, [&] {
        require_staged(c); set_device(c);
        c->forest_loaded = false;
        if (n_nodes && (!kind || !left || !right || !normal_idx || !normal_hdr0 || !desc_off || !desc_len)) throw ArgError("null node arrays");
        if (n_roots && !roots) throw ArgError("null roots");
        uint32_t max_desc = 0;
        for (uint32_t i = 0; i < n_nodes; ++i) {
            if (kind[i] == 1) { if ((uint64_t)desc_off[i] + desc_len[i] > n_desc) throw ArgError("descendants out of range"); max_desc = std::max(max_desc, desc_len[i]); }
            else if (kind[i] == 2) { if (left[i] >= n_nodes || right[i] >= n_nodes) throw ArgError("child id out of range"); if (normal_idx[i] != 0xffffffffu && normal_idx[i] >= n_normals) throw ArgError("normal index out of range"); }
        }
        for (uint64_t i = 0; i < n_desc; ++i) if (desc_rows[i] >= c->n) throw ArgError("descendant row out of range");
        for (uint32_t i = 0; i < n_roots; ++i) if (roots[i] >= n_nodes) throw ArgError("root id out of range");
        const uint32_t ld = c->ld;
        auto up = [&](DevBuf& b, const void* src, size_t bytes) { b.ensure(std::max<size_t>(16, bytes)); if (bytes) CK(cudaMemcpyAsync(b.p, src, bytes, cudaMemcpyHostToDevice, c->stream)); };
        up(c->f_kind, kind, n_nodes); up(c->f_left, left, 4ull * n_nodes); up(c->f_right, right, 4ull * n_nodes); up(c->f_nidx, normal_idx, 4ull * n_nodes);
        up(c->f_nh0, normal_hdr0, 4ull * n_nodes); up(c->f_doff, desc_off, 4ull * n_nodes); up(c->f_dlen, desc_len, 4ull * n_nodes);
        up(c->f_desc, desc_rows, 4ull * n_desc); up(c->f_roots, roots, 4ull * n_roots);
        c->f_n_normals = n_normals;
        c->f_normals.ensure(std::max<size_t>(16, (size_t)n_normals * ld * 4));
        if (n_normals) {
            if (ld != c->dim) CK(cudaMemsetAsync(c->f_normals.p, 0, (size_t)n_normals * ld * 4, c->stream));
            CK(cudaMemcpy2DAsync(c->f_normals.p, (size_t)ld * 4, normals, (size_t)c->dim * 4, (size_t)c->dim * 4, n_normals, cudaMemcpyHostToDevice, c->stream));
        }
        CK(cudaStreamSynchronize(c->stream));
        c->h2d_bytes += 25ull * n_nodes + 4ull * n_desc + (uint64_t)n_normals * c->dim * 4;
        DevForest F{};
        F.kind = c->f_kind.as<uint8_t>(); F.left = c->f_left.as<uint32_t>(); F.right = c->f_right.as<uint32_t>(); F.normal_idx = c->f_nidx.as<uint32_t>();
        F.nh0 = c->f_nh0.as<float>(); F.desc_off = c->f_doff.as<uint32_t>(); F.desc_len = c->f_dlen.as<uint32_t>(); F.normals = c->f_normals.as<float>();
        F.desc_rows = c->f_desc.as<uint32_t>(); F.roots = c->f_roots.as<uint32_t>(); F.n_roots = n_roots; F.n_nodes = n_nodes;
        c->f_rec.ensure(std::max<size_t>(32, 32ull * n_nodes)); c->f_nofn.ensure(std::max<size_t>(16, 4ull * n_normals));
        if (n_nodes) { forest_pack_kernel<<<(n_nodes + 255) / 256, 256, 0, c->stream>>>(F, c->f_rec.as<uint4>(), c->f_nofn.as<uint32_t>()); CK(cudaGetLastError()); CK(cudaStreamSynchronize(c->stream)); }
        F.rec = c->f_rec.as<uint4>(); F.node_of_normal = c->f_nofn.as<uint32_t>();
        // One depth-first pass from the roots for filtered searches: parents, reachability, and the pins that keep every
        // ancestor of a missing node live, so that a pruned walk still pops it exactly when the reference would.
        std::vector<uint32_t> parent(n_nodes, NO_PARENT), stack(roots, roots + n_roots);
        std::vector<uint8_t> reach(n_nodes, 0), pin(n_nodes, 0);
        bool tree = true, complete = true;
        while (!stack.empty()) {
            const uint32_t x = stack.back();
            stack.pop_back();
            if (reach[x]) { tree = false; continue; }
            reach[x] = 1;
            if (kind[x] == 0) { complete = false; for (uint32_t y = x; y != NO_PARENT && !pin[y]; y = parent[y]) pin[y] = 1; }
            else if (kind[x] == 2)
                for (uint32_t ch : {left[x], right[x]}) {
                    if (reach[ch] || parent[ch] != NO_PARENT) tree = false;
                    else parent[ch] = x;
                    stack.push_back(ch);
                }
        }
        const uint32_t words = (uint32_t)((c->n + 31) / 32);
        up(c->f_parent, parent.data(), 4ull * n_nodes); up(c->f_reach, reach.data(), n_nodes); up(c->f_pin, pin.data(), n_nodes);
        c->f_inleaf.ensure(std::max<size_t>(16, 4ull * words));
        CK(cudaMemsetAsync(c->f_inleaf.p, 0, 4ull * words, c->stream));
        if (n_nodes) { forest_inleaf_kernel<<<(uint32_t)(((uint64_t)n_nodes * 32 + 255) / 256), 256, 0, c->stream>>>(F, c->f_reach.as<uint8_t>(), c->f_inleaf.as<uint32_t>()); CK(cudaGetLastError()); }
        CK(cudaStreamSynchronize(c->stream));
        c->f_tree = tree; c->f_complete = complete;
        c->forest = F; c->forest_max_desc = max_desc; c->forest_n = c->n; c->forest_epoch += 1; c->forest_loaded = true;
    });
}

extern "C++" {
namespace {

// The checks every batched search starts with. false: nothing to search (nq == 0, or count == 0 and the results are empty).
bool batch_begin(arroy_ctx* c, uint32_t nq, const uint32_t* query_rows, const float* queries, uint64_t count, uint32_t* out_rows, float* out_dist,
                 uint32_t* out_len, int32_t* out_status) {
        require_staged(c); set_device(c);
        if (!c->forest_loaded || c->forest_n != c->n) throw NotStaged("no forest loaded on this context for the staged items (arroy_b200_load_forest)");
        if (nq == 0) return false;
        if ((!query_rows && !queries) || !out_rows || !out_dist || !out_len) throw ArgError("null argument");
        if (count == 0) { for (uint32_t q = 0; q < nq; ++q) { out_len[q] = 0; if (out_status) out_status[q] = 0; } return false; }
        if (count > TOPK_CAP / 2) throw ArgError("count larger than the top-k buffer (TOPK_CAP/2 = 2048)");
        if (query_rows) for (uint32_t q = 0; q < nq; ++q) if (query_rows[q] >= c->n) throw ArgError("query row out of range");
        return true;
}

// The per-query buffer sizes of a call's walks.
struct BatchShape {
    uint32_t k;
    uint64_t search_k, cand_cap64;
    uint32_t cand_cap, heap_cap, bm_words;
};

BatchShape batch_shape(arroy_ctx* c, uint64_t count, uint64_t search_k, bool filtered) {
        const DevForest& F = c->forest;
        if (search_k == 0) {   // count x roots x D::DEFAULT_OVERSAMPLING, saturating (reader.rs:330-335): 3 for binary-quantized metrics
            const unsigned __int128 sk = (unsigned __int128)count * F.n_roots * (is_bq(c->metric) ? 3u : 1u);
            search_k = sk > (unsigned __int128)UINT64_MAX ? UINT64_MAX : (uint64_t)sk;
        }
        // (saturating, so that search_k near 2^64 still leaves room for every row a walk or the shortcut may take)
        const uint64_t sk_plus = search_k > UINT64_MAX - c->forest_max_desc ? UINT64_MAX : search_k + c->forest_max_desc;
        const uint64_t cand_cap64 = std::min<uint64_t>(c->n, sk_plus);
        // a filtered walk may push every node once (a filter can keep it going through the whole forest)
        const uint64_t heap_cap64 = (uint64_t)F.n_roots + (filtered ? (uint64_t)F.n_nodes : std::min<uint64_t>(F.n_nodes, 2 * std::min<uint64_t>(search_k, c->n) + 1024));
        if (cand_cap64 > 0x7fffffffull || heap_cap64 > 0x7fffffffull) throw ArgError("search_k too large for the device walk");
        BatchShape S{};
        S.k = (uint32_t)count; S.search_k = search_k; S.cand_cap64 = cand_cap64;
        S.cand_cap = (uint32_t)std::max<uint64_t>(cand_cap64, 1); S.heap_cap = (uint32_t)heap_cap64;
        S.bm_words = (uint32_t)((c->n + 31) / 32);
        return S;
}

enum FilterMode { FM_NONE, FM_SHARED, FM_MULTI };

// How the walks of one run_batch call are filtered. Queries [0, n_walk) walk; the others take the small-filter shortcut: with
// FM_SHARED every query or none (the shared filter's rows from w_fbits / w_soff), with FM_MULTI per filter (the rows of the
// query's filter f, rows[offs[f] .. offs[f + 1])).
struct BatchFilter {
    FilterMode mode = FM_NONE;
    WalkFilter Fl{};
    uint32_t n_walk = 0;
    const uint32_t* rows = nullptr;
    const uint64_t* offs = nullptr;
};

// The stages every batched search shares once its filters are summarised: the walks (or the shortcut), the candidate sort, the
// re-rank and top-k, bq_normalize and the results, in the order of the nq queries given.
void run_batch(arroy_ctx* c, uint32_t nq, const uint32_t* query_rows, const float* queries, const float* qhdr0, const BatchShape& S,
               const BatchFilter& bf, uint32_t* out_rows, float* out_dist, uint32_t* out_len, int32_t* out_status) {
        const uint32_t ld = c->ld, k = S.k, cand_cap = S.cand_cap, heap_cap = S.heap_cap, bm_words = S.bm_words;
        const uint64_t search_k = S.search_k, cand_cap64 = S.cand_cap64;
        const DevForest& F = c->forest;
        const bool filtered = bf.mode != FM_NONE, multi = bf.mode == FM_MULTI;
        const WalkFilter& Fl0 = bf.Fl;
        const size_t walk_smem = (size_t)WALK_WARPS * WALK_SHEAP * 8;
        std::vector<int32_t> h_status;
        std::vector<uint32_t> h_pops;
        auto filter_tally = [&](uint32_t m, uint32_t m_walk) {   // after the stream is idle: statistics of m filtered queries, the first m_walk walked
            if (!filtered) return;
            h_status.resize(m); h_pops.resize(m);
            CK(cudaMemcpy(h_status.data(), c->w_status.p, 4ull * m, cudaMemcpyDeviceToHost));
            if (m_walk) CK(cudaMemcpy(h_pops.data(), c->w_pops.p, 4ull * m_walk, cudaMemcpyDeviceToHost));
            for (uint32_t q = 0; q < m; ++q) {
                if (h_status[q] == 0) { c->filter_stats[0] += 1; c->filter_stats[1] += q < m_walk ? 0 : 1; }
                else c->filter_stats[2] += 1;
                if (q < m_walk) c->filter_stats[3] += h_pops[q];
            }
        };
        // the shortcut for queries q0 + [m_walk, m) of the call, their candidate segments [m_walk, m) of `cand`
        auto shortcut = [&](uint32_t q0, uint32_t m_walk, uint32_t m, uint32_t* cand) {
            if (multi) multi_filter_select_kernel<<<(m - m_walk + 7) / 8, 256, 0, c->stream>>>(bf.rows, bf.offs, Fl0.qfilter + q0 + m_walk, c->f_inleaf.as<uint32_t>(), m - m_walk,
                                                                                              cand + (size_t)m_walk * cand_cap, cand_cap, c->w_count.as<uint32_t>() + m_walk,
                                                                                              c->w_status.as<int32_t>() + m_walk);
            else filter_select_scatter_kernel<<<dim3((bm_words + 255) / 256, m), 256, 0, c->stream>>>(c->w_fbits.as<uint32_t>(), c->f_inleaf.as<uint32_t>(), c->w_soff.as<uint32_t>(), bm_words,
                                                                                                      cand, cand_cap, c->w_count.as<uint32_t>(), c->w_status.as<int32_t>());
            CK(cudaGetLastError());
        };
        // ---- a few queries: latency path, one CTA per query (search.cuh walk1_kernel), then the plain distance + top-k kernels on
        //      all SMs. Any query it cannot hold (heap / candidate overflow) sends the call through the general path below.
        if (bf.n_walk > 0 && nq <= 16 && cand_cap64 <= (uint64_t)W1_CAND && getenv("ARROY_B200_NO_WALK1") == nullptr) {
            const uint32_t m = nq, m_walk = bf.n_walk;
            if (ld <= W1_MAX_LD) {
                c->w_cand2.ensure(4ull * cand_cap * m); c->w_count.ensure(4ull * m); c->w_status.ensure(4ull * m);
                c->w_beg.ensure(8ull * (m + 1)); c->w_end.ensure(8ull * (m + 1));
                c->s_keys.ensure(8ull * cand_cap * m); c->s_dists.ensure(4ull * cand_cap * m);
                c->s_orows.ensure(4ull * m * k); c->s_odist.ensure(4ull * m * k); c->s_olen.ensure(4ull * m);
                const DevQueries Q = upload_queries(c, 0, m, query_rows, queries, qhdr0);
                Marks mark{c};
                mark();
                // every split normal's dot with the query in one pass over the forest's normals, when that is cheaper than the
                // walker's chain of per-pop reductions (up to a 768 MB normals matrix)
                const float* d_pre = nullptr;
                {
                    constexpr uint64_t DOTS_MAX_BYTES = 768ull << 20;
                    const uint64_t nbytes = (uint64_t)c->f_n_normals * ld * 4;
                    if (c->f_n_normals > 0 && m <= 4 && nbytes <= DOTS_MAX_BYTES && c->dim >= 32) {
                        c->w_pre.ensure(4ull * F.n_nodes * m);
                        const uint32_t gx = (uint32_t)std::min<uint64_t>(((uint64_t)c->f_n_normals + 7) / 8, (uint64_t)c->sm_count * 8);
                        forest_dots_kernel<<<dim3(gx, m), 256, (size_t)ld * 4, c->stream>>>(F, c->f_n_normals, items_f32(c), c->dim, ld, Q.rows, Q.vecs, c->w_pre.as<float>());
                        CK(cudaGetLastError());
                        c->n_launches += 1;
                        d_pre = c->w_pre.as<float>();
                    }
                }
                const int w1debug = getenv("ARROY_B200_WALK1_DEBUG") ? 1 : 0;
                if (m_walk < m) shortcut(0, m_walk, m, c->w_cand2.as<uint32_t>());   // (multi only: a shared filter walks every query or none)
                WalkFilter Fl = Fl0;
                if (filtered) {
                    Fl.spill_cap = F.n_roots + F.n_nodes;
                    c->w_spill.ensure(8ull * Fl.spill_cap * m_walk);
                    Fl.spill = c->w_spill.as<unsigned long long>();
                }
                const auto walk1 = multi ? &walk1_kernel<true, true> : filtered ? &walk1_kernel<true> : &walk1_kernel<false>;
                const size_t w1smem = filtered ? walk1_smem<true>(ld) : walk1_smem<false>(ld);
                raise_smem_limit(c->device, (const void*)walk1, w1smem);
                walk1<<<m_walk, W1_THREADS, w1smem, c->stream>>>(F, items_f32(c), c->dim, ld, c->metric, m_walk, Q.rows, Q.vecs, Q.h0, d_pre, c->f_n_normals, w1debug,
                                                                 search_k, c->w_cand2.as<uint32_t>(), cand_cap, c->w_count.as<uint32_t>(), c->w_status.as<int32_t>(), Fl);
                CK(cudaGetLastError());
                mark();
                walk_segments_kernel<<<(m + 256) / 256, 256, 0, c->stream>>>(c->w_count.as<uint32_t>(), m, cand_cap, c->w_beg.as<uint64_t>(), c->w_end.as<uint64_t>());
                CK(cudaGetLastError());
                mark();
                // (no fused re-rank: its one CTA per query would leave all but <= 16 SMs idle)
                rerank_segments(c, m, Q, c->w_cand2.as<uint32_t>(), c->w_beg.as<uint64_t>(), c->w_end.as<uint64_t>(), (uint64_t)cand_cap * m, cand_cap, k, false, &mark);
                c->n_launches += 4;
                bq_normalize(c, c->s_odist.as<float>(), (uint64_t)m * k);
                mark();
                c->pin.ensure(std::max<size_t>(c->pin.cap, 4ull * m));
                int32_t* h_st = c->pin.as<int32_t>();
                CK(cudaMemcpyAsync(h_st, c->w_status.p, 4ull * m, cudaMemcpyDeviceToHost, c->stream));
                copy_results(c, 0, m, k, out_rows, out_dist, out_len);
                mark.add_to(c->sbreak);
                bool all_ok = true;
                for (uint32_t q = 0; q < m; ++q) all_ok = all_ok && h_st[q] == 0;
                if (all_ok) {
                    if (out_status) for (uint32_t q = 0; q < m; ++q) out_status[q] = 0;
                    filter_tally(m, m_walk);
                    c->d2h_bytes += 8ull * m * k + 8ull * m;
                    return;
                }
            }
        }
        // process the queries in chunks that keep the scratch memory bounded (~1 GiB)
        const uint64_t per_q = 8ull * heap_cap + 8ull * cand_cap + 4ull * bm_words + 12ull * cand_cap + 64;
        uint32_t chunk = (uint32_t)std::max<uint64_t>(1, std::min<uint64_t>({(uint64_t)nq, (1ull << 30) / per_q, 65535ull}));
        for (uint32_t q0 = 0; q0 < nq; q0 += chunk) {
            const uint32_t m = std::min(chunk, nq - q0);
            const uint32_t m_walk = q0 < bf.n_walk ? std::min(m, bf.n_walk - q0) : 0u;   // the chunk's first m_walk queries walk
            c->w_heaps.ensure(8ull * heap_cap * m); c->w_cand.ensure(4ull * cand_cap * m); c->w_cand2.ensure(4ull * cand_cap * m);
            c->w_count.ensure(4ull * m); c->w_bitmap.ensure(4ull * bm_words * m); c->w_status.ensure(4ull * m);
            c->w_beg.ensure(8ull * (m + 1)); c->w_end.ensure(8ull * (m + 1));
            c->s_keys.ensure(8ull * cand_cap * m); c->s_dists.ensure(4ull * cand_cap * m);
            c->s_orows.ensure(4ull * m * k); c->s_odist.ensure(4ull * m * k); c->s_olen.ensure(4ull * m);
            const DevQueries Q = upload_queries(c, q0, m, query_rows, queries, qhdr0);
            Marks mark{c};
            mark();
            if (m_walk == 0)   // every query of the chunk takes the shortcut: its segments are already sorted
                shortcut(q0, 0, m, c->w_cand2.as<uint32_t>());
            else {
                if (m_walk < m) shortcut(q0, m_walk, m, c->w_cand.as<uint32_t>());   // (multi only) sorted with the walked segments below
                CK(cudaMemsetAsync(c->w_bitmap.p, 0, 4ull * bm_words * m_walk, c->stream));
                WalkFilter Fl = Fl0;
                if (multi) Fl.qfilter += q0;
                const auto walk = multi ? &walk_kernel<true, true> : filtered ? &walk_kernel<true> : &walk_kernel<false>;
                raise_smem_limit(c->device, (const void*)walk, walk_smem);
                walk<<<(m_walk + WALK_WARPS - 1) / WALK_WARPS, WALK_WARPS * 32, walk_smem, c->stream>>>(F, items_f32(c), c->dim, ld, c->metric, m_walk, Q.rows, Q.vecs, Q.h0,
                                                                                                        search_k, c->w_heaps.as<unsigned long long>(), heap_cap, c->w_cand.as<uint32_t>(), cand_cap,
                                                                                                        c->w_count.as<uint32_t>(), c->w_bitmap.as<uint32_t>(), bm_words, c->w_status.as<int32_t>(), Fl);
                CK(cudaGetLastError());
            }
            mark();
            walk_segments_kernel<<<(m + 256) / 256, 256, 0, c->stream>>>(c->w_count.as<uint32_t>(), m, cand_cap, c->w_beg.as<uint64_t>(), c->w_end.as<uint64_t>());
            CK(cudaGetLastError());
            if (m_walk) {   // sort every query's unique candidates ascending (= ascending item ids): reader.rs:378
                size_t tmp_bytes = 0;
                CK(cub::DeviceSegmentedSort::SortKeys(nullptr, tmp_bytes, c->w_cand.as<uint32_t>(), c->w_cand2.as<uint32_t>(), (int64_t)cand_cap * m, (int64_t)m,
                                                      c->w_beg.as<uint64_t>(), c->w_end.as<uint64_t>(), c->stream));
                c->w_tmp.ensure(std::max<size_t>(tmp_bytes, 16));
                CK(cub::DeviceSegmentedSort::SortKeys(c->w_tmp.p, tmp_bytes, c->w_cand.as<uint32_t>(), c->w_cand2.as<uint32_t>(), (int64_t)cand_cap * m, (int64_t)m,
                                                      c->w_beg.as<uint64_t>(), c->w_end.as<uint64_t>(), c->stream));
            }
            mark();
            rerank_segments(c, m, Q, c->w_cand2.as<uint32_t>(), c->w_beg.as<uint64_t>(), c->w_end.as<uint64_t>(), (uint64_t)cand_cap * m, cand_cap, k, true, &mark);
            c->n_launches += 5;
            bq_normalize(c, c->s_odist.as<float>(), (uint64_t)m * k);
            mark();
            copy_results(c, q0, m, k, out_rows, out_dist, out_len, out_status);
            mark.add_to(c->sbreak);
            filter_tally(m, m_walk);
            c->d2h_bytes += 8ull * m * k + 8ull * m;
        }
}

// arroy_b200_search_batch, and with filter_bits != NULL arroy_b200_search_batch_filtered: one row filter for every query
void search_batch_body(arroy_ctx* c, uint32_t nq, const uint32_t* query_rows, const float* queries, const float* qhdr0,
                       uint64_t count, uint64_t search_k, const uint32_t* filter_bits, uint32_t* out_rows, float* out_dist, uint32_t* out_len,
                       int32_t* out_status) {
        if (!batch_begin(c, nq, query_rows, queries, count, out_rows, out_dist, out_len, out_status)) return;
        const DevForest& F = c->forest;
        const bool filtered = filter_bits != nullptr;
        const BatchShape S = batch_shape(c, count, search_k, filtered);
        const uint32_t bm_words = S.bm_words;
        for (double& x : c->sbreak) x = 0;
        // ---- the filter's summary: fcount / live per node and ftotal (search.cuh filter_count_kernel). When ftotal <= search_k
        //      the reference's walk only ends with an empty queue, so its candidates are every filtered row of a reachable leaf:
        //      the shortcut takes those without a walk (only where no reachable node is missing and pruning is exact).
        BatchFilter bf;
        bf.mode = filtered ? FM_SHARED : FM_NONE;
        bf.n_walk = nq;
        if (filtered) {
            c->w_fbits.ensure(4ull * bm_words); c->w_fcount.ensure(std::max<size_t>(16, 4ull * F.n_nodes)); c->w_live.ensure(std::max<size_t>(16, F.n_nodes));
            c->w_ftotal.ensure(16); c->w_pops.ensure(4ull * std::max<uint32_t>(nq, 1));
            CK(cudaMemcpyAsync(c->w_fbits.p, filter_bits, 4ull * bm_words, cudaMemcpyHostToDevice, c->stream));
            if (c->f_tree) CK(cudaMemcpyAsync(c->w_live.p, c->f_pin.p, F.n_nodes, cudaMemcpyDeviceToDevice, c->stream));
            else CK(cudaMemsetAsync(c->w_live.p, 1, F.n_nodes, c->stream));
            CK(cudaMemsetAsync(c->w_ftotal.p, 0, 8, c->stream));
            if (F.n_nodes) {
                filter_count_kernel<<<(uint32_t)(((uint64_t)F.n_nodes * 32 + 255) / 256), 256, 0, c->stream>>>(F, c->w_fbits.as<uint32_t>(), c->f_reach.as<uint8_t>(),
                                                                                                              c->f_tree ? c->f_parent.as<uint32_t>() : nullptr, c->w_fcount.as<uint32_t>(),
                                                                                                              c->w_live.as<uint8_t>(), c->w_ftotal.as<unsigned long long>());
                CK(cudaGetLastError());
                c->n_launches += 1;
            }
            unsigned long long ftotal = 0;
            CK(cudaMemcpyAsync(&ftotal, c->w_ftotal.p, 8, cudaMemcpyDeviceToHost, c->stream));
            CK(cudaStreamSynchronize(c->stream));
            c->h2d_bytes += 4ull * bm_words;
            WalkFilter& Fl = bf.Fl;
            Fl.bits = c->w_fbits.as<uint32_t>(); Fl.fcount = c->w_fcount.as<uint32_t>(); Fl.live = c->w_live.as<uint8_t>(); Fl.pops = c->w_pops.as<uint32_t>();
            const bool shortcut = c->f_tree && c->f_complete && ftotal <= S.search_k;
            if (shortcut) {   // the rows, ascending: popcounts per word, an exclusive scan, then every query's segment is written
                bf.n_walk = 0;
                c->w_scount.ensure(4ull * bm_words); c->w_soff.ensure(4ull * bm_words);
                filter_select_count_kernel<<<(bm_words + 255) / 256, 256, 0, c->stream>>>(c->w_fbits.as<uint32_t>(), c->f_inleaf.as<uint32_t>(), bm_words, c->w_scount.as<uint32_t>());
                CK(cudaGetLastError());
                size_t tmp_bytes = 0;
                CK(cub::DeviceScan::ExclusiveSum(nullptr, tmp_bytes, c->w_scount.as<uint32_t>(), c->w_soff.as<uint32_t>(), (int)bm_words, c->stream));
                c->w_tmp.ensure(std::max<size_t>(tmp_bytes, 16));
                CK(cub::DeviceScan::ExclusiveSum(c->w_tmp.p, tmp_bytes, c->w_scount.as<uint32_t>(), c->w_soff.as<uint32_t>(), (int)bm_words, c->stream));
                c->n_launches += 2;
            }
        }
        run_batch(c, nq, query_rows, queries, qhdr0, S, bf, out_rows, out_dist, out_len, out_status);
}

// arroy_b200_search_batch_multi_filtered. The distinct filters the queries use are summarised 32 to a group (one row-mask
// scatter and one multi_filter_count_kernel pass per group), as many groups at a time as fit the scratch bound of the summaries
// (1 GiB); each such set of filters then runs its queries through run_batch, those whose filter takes the shortcut after the
// ones that walk, and their results go back to the caller's query order.
void multi_filter_body(arroy_ctx* c, uint32_t nq, const uint32_t* query_rows, const float* queries, const float* qhdr0, uint64_t count,
                       uint64_t search_k, uint32_t n_filters, const uint64_t* filter_offsets, const uint32_t* filter_rows, const uint32_t* query_filter,
                       uint32_t* out_rows, float* out_dist, uint32_t* out_len, int32_t* out_status) {
        require_staged(c);
        if (nq > 0) {
            if (n_filters == 0) throw ArgError("no filters for the queries");
            if (!filter_offsets || !query_filter) throw ArgError("null filter argument");
            for (uint32_t q = 0; q < nq; ++q) if (query_filter[q] >= n_filters) throw ArgError("query_filter out of range");
            for (uint32_t f = 0; f < n_filters; ++f) {
                const uint64_t b = filter_offsets[f], e = filter_offsets[f + 1];
                if (e < b) throw ArgError("filter offsets must not decrease");
                if (e > b && !filter_rows) throw ArgError("null filter rows");
                for (uint64_t i = b; i < e; ++i) {
                    if (filter_rows[i] >= c->n) throw ArgError("filter row out of range");
                    if (i > b && filter_rows[i] <= filter_rows[i - 1]) throw ArgError("filter rows must be strictly ascending");
                }
            }
        }
        if (!batch_begin(c, nq, query_rows, queries, count, out_rows, out_dist, out_len, out_status)) return;
        const DevForest& F = c->forest;
        const BatchShape S = batch_shape(c, count, search_k, true);
        const uint32_t k = S.k, d = c->dim;
        for (double& x : c->sbreak) x = 0;
        // the used filters in order of first use: filter used[u] is bit u % 32 of group u / 32
        std::vector<uint32_t> used, slot(n_filters, UINT32_MAX);
        for (uint32_t q = 0; q < nq; ++q) {
            const uint32_t f = query_filter[q];
            if (slot[f] == UINT32_MAX) { slot[f] = (uint32_t)used.size(); used.push_back(f); }
        }
        const uint32_t n_used = (uint32_t)used.size();
        // per group (search.cuh GroupSummaries): a row mask per row, a live mask and 32 counts per node, plus 32 totals
        GroupSummaries G{};
        G.live_off = (c->n + 31) / 32 * 32;
        G.count_off = G.live_off + ((uint64_t)F.n_nodes + 31) / 32 * 32;
        G.group_words = G.count_off + 32ull * F.n_nodes;
        const uint64_t group_bytes = 4ull * G.group_words + 256;
        const uint32_t set_groups = (uint32_t)std::max<uint64_t>(1, std::min<uint64_t>((1ull << 30) / group_bytes, 65535 / 32));
        const bool shortcut_ok = c->f_tree && c->f_complete;
        std::vector<uint32_t> h_rows, h_qf, order, s_qrows, o_rows, o_len;
        std::vector<uint64_t> h_offs;
        std::vector<unsigned long long> ftotal;
        std::vector<float> s_q, s_qh0, o_dist;
        std::vector<int32_t> o_status;
        for (uint32_t u0 = 0; u0 < n_used; u0 += 32 * set_groups) {
            const uint32_t nf = std::min(32 * set_groups, n_used - u0), groups = (nf + 31) / 32;
            h_offs.assign(1, 0); h_rows.clear();
            uint64_t longest = 0;
            for (uint32_t u = u0; u < u0 + nf; ++u) {
                const uint64_t b = filter_offsets[used[u]], e = filter_offsets[used[u] + 1];
                h_rows.insert(h_rows.end(), filter_rows + b, filter_rows + e);
                h_offs.push_back(h_rows.size());
                longest = std::max(longest, e - b);
            }
            Marks mark{c};
            mark();
            c->w_mrows.ensure(std::max<size_t>(16, 4ull * h_rows.size())); c->w_moffs.ensure(8ull * (nf + 1));
            c->w_msum.ensure(4ull * G.group_words * groups); c->w_ftotal.ensure(256ull * groups);
            G.sum = c->w_msum.as<uint32_t>();
            c->w_pops.ensure(4ull * nq);
            if (!h_rows.empty()) CK(cudaMemcpyAsync(c->w_mrows.p, h_rows.data(), 4ull * h_rows.size(), cudaMemcpyHostToDevice, c->stream));
            CK(cudaMemcpyAsync(c->w_moffs.p, h_offs.data(), 8ull * (nf + 1), cudaMemcpyHostToDevice, c->stream));
            CK(cudaMemset2DAsync(c->w_msum.p, 4ull * G.group_words, 0, 4ull * c->n, groups, c->stream));   // the row masks
            if (longest) {
                const uint32_t gx = (uint32_t)std::min<uint64_t>((longest + 255) / 256, (uint64_t)c->sm_count * 4);
                multi_filter_mask_kernel<<<dim3(gx, nf), 256, 0, c->stream>>>(c->w_mrows.as<uint32_t>(), c->w_moffs.as<uint64_t>(), G);
                CK(cudaGetLastError());
                c->n_launches += 1;
            }
            mark();
            CK(cudaMemsetAsync(c->w_ftotal.p, 0, 256ull * groups, c->stream));
            if (F.n_nodes) {
                multi_filter_live_init_kernel<<<dim3((F.n_nodes + 255) / 256, groups), 256, 0, c->stream>>>(c->f_tree ? c->f_pin.as<uint8_t>() : nullptr, F.n_nodes, G);
                CK(cudaGetLastError());
                multi_filter_count_kernel<<<dim3((uint32_t)(((uint64_t)F.n_nodes * 32 + 255) / 256), groups), 256, 0, c->stream>>>(F, G, c->f_reach.as<uint8_t>(),
                                                                                                                                  c->f_tree ? c->f_parent.as<uint32_t>() : nullptr,
                                                                                                                                  c->w_ftotal.as<unsigned long long>());
                CK(cudaGetLastError());
                c->n_launches += 2;
            }
            ftotal.resize(32ull * groups);
            CK(cudaMemcpyAsync(ftotal.data(), c->w_ftotal.p, 256ull * groups, cudaMemcpyDeviceToHost, c->stream));
            mark();
            CK(cudaStreamSynchronize(c->stream));
            mark.add_to(c->sbreak + 5);   // the upload, the summaries
            c->h2d_bytes += 4ull * h_rows.size() + 8ull * (nf + 1);
            c->multi_stats[0] += groups; c->multi_stats[1] += nf;
            // this set's queries: those that walk, then those whose filter takes the shortcut, each in call order
            order.clear();
            for (int pass = 0; pass < 2; ++pass)
                for (uint32_t q = 0; q < nq; ++q) {
                    const uint32_t u = slot[query_filter[q]];
                    if (u < u0 || u >= u0 + nf) continue;
                    const bool sc = shortcut_ok && ftotal[u - u0] <= S.search_k;
                    if (sc == (pass == 1)) order.push_back(q);
                }
            const uint32_t m = (uint32_t)order.size();
            BatchFilter bf;
            bf.mode = FM_MULTI;
            bf.n_walk = 0;
            for (uint32_t q : order) bf.n_walk += !(shortcut_ok && ftotal[slot[query_filter[q]] - u0] <= S.search_k);
            h_qf.resize(m);
            for (uint32_t i = 0; i < m; ++i) h_qf[i] = slot[query_filter[order[i]]] - u0;
            c->w_mqf.ensure(4ull * m);
            CK(cudaMemcpyAsync(c->w_mqf.p, h_qf.data(), 4ull * m, cudaMemcpyHostToDevice, c->stream));
            if (query_rows) { s_qrows.resize(m); for (uint32_t i = 0; i < m; ++i) s_qrows[i] = query_rows[order[i]]; }
            else { s_q.resize((size_t)m * d); for (uint32_t i = 0; i < m; ++i) memcpy(&s_q[(size_t)i * d], queries + (size_t)order[i] * d, 4ull * d); }
            if (qhdr0) { s_qh0.resize(m); for (uint32_t i = 0; i < m; ++i) s_qh0[i] = qhdr0[order[i]]; }
            bf.rows = c->w_mrows.as<uint32_t>(); bf.offs = c->w_moffs.as<uint64_t>();
            WalkFilter& Fl = bf.Fl;
            Fl.pops = c->w_pops.as<uint32_t>(); Fl.qfilter = c->w_mqf.as<uint32_t>();
            Fl.summary = G.sum; Fl.group_words = G.group_words; Fl.live_off = G.live_off; Fl.count_off = G.count_off;
            o_rows.resize((size_t)m * k); o_dist.resize((size_t)m * k); o_len.resize(m); o_status.resize(m);
            run_batch(c, m, query_rows ? s_qrows.data() : nullptr, query_rows ? nullptr : s_q.data(), qhdr0 ? s_qh0.data() : nullptr, S, bf,
                      o_rows.data(), o_dist.data(), o_len.data(), o_status.data());
            for (uint32_t i = 0; i < m; ++i) {
                const uint32_t q = order[i];
                memcpy(out_rows + (size_t)q * k, &o_rows[(size_t)i * k], 4ull * k);
                memcpy(out_dist + (size_t)q * k, &o_dist[(size_t)i * k], 4ull * k);
                out_len[q] = o_len[i];
                if (out_status) out_status[q] = o_status[i];
            }
        }
}

}  // namespace
}  // extern "C++"

int32_t arroy_b200_search_batch(arroy_ctx* c, uint32_t nq, const uint32_t* query_rows, const float* queries, const float* qhdr0,
                                uint64_t count, uint64_t search_k, uint32_t* out_rows, float* out_dist, uint32_t* out_len, int32_t* out_status) {
    return guarded(c, [&] { search_batch_body(c, nq, query_rows, queries, qhdr0, count, search_k, nullptr, out_rows, out_dist, out_len, out_status); });
}

int32_t arroy_b200_search_batch_filtered(arroy_ctx* c, uint32_t nq, const uint32_t* query_rows, const float* queries, const float* qhdr0,
                                         uint64_t count, uint64_t search_k, const uint32_t* filter_bits, uint32_t* out_rows, float* out_dist,
                                         uint32_t* out_len, int32_t* out_status) {
    return guarded(c, [&] {
        if (!filter_bits) throw ArgError("null filter");
        search_batch_body(c, nq, query_rows, queries, qhdr0, count, search_k, filter_bits, out_rows, out_dist, out_len, out_status);
    });
}

int32_t arroy_b200_search_batch_multi_filtered(arroy_ctx* c, uint32_t nq, const uint32_t* query_rows, const float* queries, const float* qhdr0,
                                               uint64_t count, uint64_t search_k, uint32_t n_filters, const uint64_t* filter_offsets,
                                               const uint32_t* filter_rows, const uint32_t* query_filter, uint32_t* out_rows, float* out_dist,
                                               uint32_t* out_len, int32_t* out_status) {
    return guarded(c, [&] {
        multi_filter_body(c, nq, query_rows, queries, qhdr0, count, search_k, n_filters, filter_offsets, filter_rows, query_filter, out_rows, out_dist,
                          out_len, out_status);
    });
}

int32_t arroy_b200_multi_filter_stats(arroy_ctx* c, uint64_t out[2]) {
    return guarded(c, [&] {
        if (!out) throw ArgError("null argument");
        out[0] = c->multi_stats[0]; out[1] = c->multi_stats[1];
    });
}

int32_t arroy_b200_search_stats(arroy_ctx* c, uint64_t out[4]) {
    return guarded(c, [&] {
        if (!out) throw ArgError("null argument");
        for (int i = 0; i < 4; ++i) out[i] = c->filter_stats[i];
    });
}

int32_t arroy_b200_synth_device(arroy_ctx* c, const uint8_t seed[32], uint32_t dim, uint64_t row0, uint64_t rows, float centre, void* device_out) {
    return guarded(c, [&] {
        set_device(c);
        if (!seed || !device_out) throw ArgError("null argument");
        uint32_t key[8];
        for (int i = 0; i < 8; ++i) key[i] = (uint32_t)seed[4 * i] | ((uint32_t)seed[4 * i + 1] << 8) | ((uint32_t)seed[4 * i + 2] << 16) | ((uint32_t)seed[4 * i + 3] << 24);
        c->s_misc.ensure(64);
        CK(cudaMemcpyAsync(c->s_misc.p, key, 32, cudaMemcpyHostToDevice, c->stream));
        uint64_t blocks = (rows * dim + 15) / 16 + 1;
        int grid = (int)std::min<uint64_t>((blocks + 255) / 256, (uint64_t)c->sm_count * 32);
        synth_kernel<<<std::max(grid, 1), 256, 0, c->stream>>>(c->s_misc.as<uint32_t>(), dim, row0, rows, centre, static_cast<float*>(device_out));
        CK(cudaGetLastError());
        CK(cudaStreamSynchronize(c->stream));
    });
}

int32_t arroy_b200_time_scan(arroy_ctx* c, const float* normal, float hdr0, float hdr1, const uint32_t* rows, uint64_t n_rows, int32_t variant, int32_t iters,
                             int32_t flush_l2, float* out_ms_avg, uint64_t* out_left_count) {
    return guarded(c, [&] {
        require_staged(c); set_device(c);
        if (!normal || !out_ms_avg || n_rows == 0 || n_rows > c->n || iters <= 0 || (variant != 0 && variant != 1)) throw ArgError("bad argument");
        const bool planes = variant == 1;
        if (planes && (is_bq(c->metric) || c->dim < 64 || c->dim > PLANES_MAX_D)) throw ArgError("time_scan variant 1 needs a float metric and 64 <= dim <= PLANES_MAX_D");
        if (planes) planes_prepare(c);
        upload_normal(c, normal, hdr0, hdr1);
        CK(cudaStreamSynchronize(c->stream));
        c->s_flags.ensure(n_rows);
        uint64_t units = (n_rows + SCAN_UNIT - 1) / SCAN_UNIT;
        c->s_unit.ensure(units * 4);
        c->s_job.ensure(sizeof(Job));
        Job jb{};
        jb.kind = JOB_SCAN; jb.len = (uint32_t)n_rows; jb.rows = nullptr; jb.normal = c->s_normal.as<float>();
        jb.flags = c->s_flags.as<uint8_t>(); jb.margins = nullptr; jb.unit_left = c->s_unit.as<uint32_t>();
        if (rows) {
            c->s_rows.ensure(n_rows * 4);
            CK(cudaMemcpyAsync(c->s_rows.p, rows, n_rows * 4, cudaMemcpyHostToDevice, c->stream));
            jb.rows = c->s_rows.as<uint32_t>();
        }
        CK(cudaMemcpyAsync(c->s_job.p, &jb, sizeof(Job), cudaMemcpyHostToDevice, c->stream));
        int grid = (int)std::min<uint64_t>(units, (uint64_t)c->sm_count * 3);
        const size_t flush_bytes = 256ull << 20;
        // variant 1: work_kernel_planes on the one job with every unit through the 8-bit pre-filter (scan_claim_planes), two CTAs
        // per SM as in the build; the stage counts of its last launch are what build_prefilter_stats reports afterwards
        const size_t stats_off = flush_l2 ? flush_bytes : 0;
        c->s_misc.ensure(stats_off + 32);
        unsigned long long* pstats = reinterpret_cast<unsigned long long*>(c->s_misc.as<uint8_t>() + stats_off);
        const ScanPlanes all{0u, pstats};
        auto launch = [&] {
            launch_scan(c, c->stream, c->s_job.as<Job>(), 1, planes ? c->sm_count * 2 : grid, planes ? &all : nullptr);
            CK(cudaGetLastError());
            if (!planes) c->n_launches += 1;
        };
        launch();  // warm-up
        CK(cudaStreamSynchronize(c->stream));
        double total_ms = 0;
        for (int it = 0; it < iters; ++it) {
            if (flush_l2) CK(cudaMemsetAsync(c->s_misc.p, it & 0xff, flush_bytes, c->stream));
            if (planes) CK(cudaMemsetAsync(pstats, 0, 24, c->stream));
            CK(cudaEventRecord(c->ev0, c->stream));
            launch();
            CK(cudaEventRecord(c->ev1, c->stream));
            CK(cudaEventSynchronize(c->ev1));
            float ms = 0;
            CK(cudaEventElapsedTime(&ms, c->ev0, c->ev1));
            total_ms += ms;
        }
        *out_ms_avg = (float)(total_ms / iters);
        if (planes) {
            unsigned long long hs[3] = {0, 0, 0};
            CK(cudaMemcpyAsync(hs, pstats, 24, cudaMemcpyDeviceToHost, c->stream));
            CK(cudaStreamSynchronize(c->stream));
            c->shadow_rows = hs[0]; c->shadow_rescored = hs[1]; c->shadow_stage2 = hs[2]; c->fused_root_rows = 0; c->fused_root_read = 0;
        }
        if (out_left_count) {
            std::vector<uint32_t> ul(units);
            CK(cudaMemcpyAsync(ul.data(), c->s_unit.p, units * 4, cudaMemcpyDeviceToHost, c->stream));
            CK(cudaStreamSynchronize(c->stream));
            uint64_t s = 0;
            for (auto v : ul) s += v;
            *out_left_count = s;
        }
    });
}

struct arroy_b200_arena {
    static constexpr int SHARDS = 64;
    std::mutex mu[SHARDS];
    std::vector<uint8_t> bytes[SHARDS];
    std::vector<std::pair<uint32_t, std::pair<uint64_t, uint64_t>>> index[SHARDS];  // node id -> (offset, len) in its shard
};
arroy_b200_arena* arroy_b200_arena_new(void) { return new arroy_b200_arena(); }
void arroy_b200_arena_free(arroy_b200_arena* a) { delete a; }
void arroy_b200_arena_clear(arroy_b200_arena* a) { for (int i = 0; i < arroy_b200_arena::SHARDS; ++i) { a->bytes[i].clear(); a->index[i].clear(); } }
int32_t arroy_b200_arena_sink(void* arg, uint32_t node_id, const uint8_t* bytes, uint64_t len) {
    auto* a = static_cast<arroy_b200_arena*>(arg);
    const int sh = (int)(std::hash<std::thread::id>()(std::this_thread::get_id()) % arroy_b200_arena::SHARDS);
    std::lock_guard<std::mutex> lk(a->mu[sh]);
    uint64_t off = a->bytes[sh].size();
    a->bytes[sh].insert(a->bytes[sh].end(), bytes, bytes + len);
    a->index[sh].push_back({node_id, {off, len}});
    return 0;
}
uint64_t arroy_b200_arena_stats(arroy_b200_arena* a, uint64_t* out_total_bytes) {
    uint64_t n = 0, b = 0;
    for (int i = 0; i < arroy_b200_arena::SHARDS; ++i) { n += a->index[i].size(); b += a->bytes[i].size(); }
    if (out_total_bytes) *out_total_bytes = b;
    return n;
}
int32_t arroy_b200_arena_get(arroy_b200_arena* a, uint32_t node_id, const uint8_t** out_bytes, uint64_t* out_len) {
    for (int i = 0; i < arroy_b200_arena::SHARDS; ++i)
        for (auto& e : a->index[i]) if (e.first == node_id) { *out_bytes = a->bytes[i].data() + e.second.first; *out_len = e.second.second; return 0; }
    return ARROY_B200_ERR_INVALID;
}

int32_t arroy_b200_build_breakdown(arroy_ctx* c, double out[8]) {
    return guarded(c, [&] { for (int i = 0; i < 8; ++i) out[i] = c->breakdown[i]; });
}

int32_t arroy_b200_counters(arroy_ctx* c, uint64_t out[4]) {
    return guarded(c, [&] { out[0] = c->n_launches; out[1] = c->h2d_bytes; out[2] = c->d2h_bytes; out[3] = (c->fr_batches[FR_BF16] << 32) | (c->fr_fallbacks[FR_BF16] & 0xffffffffull); });
}

int32_t arroy_b200_plane_rerank_stats(arroy_ctx* c, uint64_t out[4]) {
    return guarded(c, [&] {
        if (!out) throw ArgError("null argument");
        uint64_t rows[2] = {0, 0};
        if (c->pr_counts.p) {
            set_device(c);
            CK(cudaStreamSynchronize(c->stream));
            CK(cudaMemcpy(rows, c->pr_counts.p, 16, cudaMemcpyDeviceToHost));
        }
        out[0] = c->fr_batches[FR_PLANES]; out[1] = c->fr_fallbacks[FR_PLANES]; out[2] = rows[0]; out[3] = rows[1];
    });
}

int32_t arroy_b200_prefilter_scores(arroy_ctx* c, uint32_t nq, const float* queries, const uint32_t* rows, uint64_t n_rows, int32_t engine, float* out_scores) {
    return guarded(c, [&] {
        require_staged(c); set_device(c);
        if (nq == 0 || n_rows == 0) return;
        if (!queries || !rows || !out_scores) throw ArgError("null argument");
        if (is_bq(c->metric)) throw ArgError("prefilter_scores needs a float metric (binary-quantized items are bit strings)");
        if (c->dim < 32) throw ArgError("prefilter_scores needs dim >= 32");
        if (n_rows > 0x7fffffffull || (uint64_t)nq * n_rows > (1ull << 29)) throw ArgError("prefilter_scores: problem too large");
        for (uint64_t i = 0; i < n_rows; ++i) if (rows[i] >= c->n) throw ArgError("row index out of range");
        const uint32_t nc = (uint32_t)n_rows, lds = (nc + 3u) & ~3u;
        c->s_rows.ensure(4ull * nc);
        CK(cudaMemcpyAsync(c->s_rows.p, rows, 4ull * nc, cudaMemcpyHostToDevice, c->stream));
        const float* cand = xf_candidates(c, rows, nc);
        c->x_S.ensure(4ull * nq * lds);
        const DevQueries Q = upload_queries(c, 0, nq, nullptr, queries, nullptr);
        xf_scores(c, Q.vecs, nq, cand, nc, c->x_S.as<float>(), lds, TgEpilogue{TG_RAW, nullptr, nullptr, nullptr, nullptr}, engine);
        CK(cudaMemcpy2DAsync(out_scores, 4ull * nc, c->x_S.p, 4ull * lds, 4ull * nc, nq, cudaMemcpyDeviceToHost, c->stream));
        CK(cudaStreamSynchronize(c->stream));
    });
}

int32_t arroy_b200_search_breakdown(arroy_ctx* c, double out[8]) {
    return guarded(c, [&] { for (int i = 0; i < 8; ++i) out[i] = c->sbreak[i]; });
}

int32_t arroy_b200_rerank_breakdown(arroy_ctx* c, double out[8]) {
    return guarded(c, [&] { for (int i = 0; i < 8; ++i) out[i] = c->xbreak[i]; });
}

int32_t arroy_b200_rerank_stats(arroy_ctx* c, uint64_t out[4]) {
    return guarded(c, [&] { out[0] = c->xf_calls; out[1] = c->xf_fallbacks; out[2] = c->xf_selected; out[3] = c->xf_queries; });
}

int32_t arroy_b200_timer_start(arroy_ctx* c) {
    return guarded(c, [&] { set_device(c); CK(cudaStreamSynchronize(c->stream)); CK(cudaEventRecord(c->tev0, c->stream)); });
}
int32_t arroy_b200_timer_stop(arroy_ctx* c, float* out_ms) {
    return guarded(c, [&] {
        set_device(c);
        CK(cudaEventRecord(c->tev1, c->stream));
        CK(cudaEventSynchronize(c->tev1));
        CK(cudaEventElapsedTime(out_ms, c->tev0, c->tev1));
    });
}

// ---- self-test of UDiv (exact.cuh) against div.rn.f32 -------------------------------------------------------------
namespace {
__device__ __forceinline__ uint32_t st_mix(uint64_t x) { x ^= x >> 33; x *= 0xff51afd7ed558ccdull; x ^= x >> 33; x *= 0xc4ceb9fe1a85ec53ull; x ^= x >> 33; return (uint32_t)x; }
__global__ void udiv_selftest_kernel(uint64_t n_groups, uint64_t seed, unsigned long long* mismatches, unsigned long long* fallbacks) {
    const uint64_t g = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (g >= n_groups) return;
    // divisor classes: the counts 2..11 of two_means, random norms around 1, random positive floats of any exponent
    const uint32_t r0 = st_mix(seed + 5 * g);
    float b;
    switch (r0 & 3u) {
        case 0: b = (float)(2 + (r0 >> 8) % 10); break;
        case 1: b = __uint_as_float(0x3f000000u + ((r0 >> 2) & 0x00ffffffu)); break;             // [0.5, 2)
        case 2: b = __uint_as_float(0x30000000u + ((r0 >> 2) % 0x20000000u)); break;             // 2^-31 .. 2^33
        default: b = __uint_as_float((r0 >> 1) & 0x7fffffffu); if (!(b > 0.0f) || b > 3.0e38f) b = 1.5f; break;   // anything positive (denormals included)
    }
    float a[4];
    for (int u = 0; u < 4; ++u) {
        const uint32_t r = st_mix(seed + 5 * g + 1 + u);
        const uint32_t cls = st_mix(r) & 7u;
        if (cls < 5) a[u] = __uint_as_float((r & 0x80ffffffu) | ((100u + (r >> 24) % 56u) << 23));   // 2^-27 .. 2^28
        else if (cls == 5) a[u] = __uint_as_float(r);                                                  // any bit pattern
        else if (cls == 6) a[u] = __uint_as_float(r & 0x80000000u);                                    // +-0
        else a[u] = __uint_as_float((r & 0x807fffffu) | ((r >> 23 & 1u) ? 0x7f000000u : 0x00000000u)); // huge / denormal
    }
    const ab::UDiv D(b);
    float q[4];
    bool bad = !D.ok;
    for (int u = 0; u < 4; ++u) q[u] = D.fast(a[u], bad);
    if (bad) { for (int u = 0; u < 4; ++u) q[u] = __fdiv_rn(a[u], b); atomicAdd(fallbacks, 1ull); }
    for (int u = 0; u < 4; ++u) {
        const float want = __fdiv_rn(a[u], b);
        const bool same = __float_as_uint(want) == __float_as_uint(q[u]) || (want != want && q[u] != q[u]);
        if (!same) atomicAdd(mismatches, 1ull);
        if (D.ok && !ab::UDiv::suspect(a[u]) && __float_as_uint(D.quot(a[u])) != __float_as_uint(want)) atomicAdd(mismatches, 1ull);   // the bare quotient where it is trusted
    }
}
}  // namespace
int32_t arroy_b200_selftest_udiv(arroy_ctx* c, uint64_t n_groups, uint64_t seed, uint64_t* out_mismatches, uint64_t* out_fallbacks) {
    return guarded(c, [&] {
        if (!out_mismatches || !out_fallbacks) throw ArgError("null argument");
        set_device(c);
        c->s_misc.ensure(64);
        CK(cudaMemsetAsync(c->s_misc.p, 0, 16, c->stream));
        unsigned long long* d = c->s_misc.as<unsigned long long>();
        if (n_groups) udiv_selftest_kernel<<<(unsigned)((n_groups + 255) / 256), 256, 0, c->stream>>>(n_groups, seed, d, d + 1);
        CK(cudaGetLastError());
        unsigned long long h[2];
        CK(cudaMemcpyAsync(h, d, 16, cudaMemcpyDeviceToHost, c->stream));
        CK(cudaStreamSynchronize(c->stream));
        *out_mismatches = h[0]; *out_fallbacks = h[1];
    });
}

uint32_t arroy_b200_bq_quantize(const float* in, uint32_t dims, float* out) {
    const uint32_t dp = (dims + 63u) / 64u * 64u;
    if (in && out) for (uint32_t i = 0; i < dp; ++i) { uint32_t bits = 0x80000000u; if (i < dims) memcpy(&bits, in + i, 4); out[i] = (bits >> 31) ? -1.0f : 1.0f; }
    return dp;
}

int32_t arroy_b200_epochs(arroy_ctx* c, uint64_t out[2]) {
    return guarded(c, [&] { if (!out) throw ArgError("null argument"); out[0] = c->staged ? c->stage_epoch : 0; out[1] = c->forest_loaded ? c->forest_epoch : 0; });
}

int32_t arroy_b200_device_ptrs(arroy_ctx* c, void* out[3], uint32_t* out_ld) {
    return guarded(c, [&] {
        if (!c->staging_open) require_staged(c);
        if (c->host_items) throw ArgError("device_ptrs: the item rows of this context are placed in host memory (arroy_b200_item_placement), not on the device");
        out[0] = c->items.p; out[1] = c->h0.p; out[2] = c->h1.p;
        if (out_ld) *out_ld = c->row_bytes / 4;
    });
}

}  // extern "C"

// several GPUs behind one handle (in-library NCCL broadcast of the item buffer)
#include "group.hpp"

// C++ host mirror of the reference's Writer / Reader (client of the C ABI above)
#include "host.hpp"
