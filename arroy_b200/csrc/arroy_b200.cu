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
#include <mutex>
#include <stdexcept>
#include <string>
#include <thread>
#include <vector>

#include "../../include/arroy_b200.h"
#include "build.cuh"
#include "search.cuh"
#include <cublas_v2.h>

#include "xrerank.cuh"
#include "tcgemm.cuh"
#include "frerank.cuh"

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

struct DevBuf {
    void* p = nullptr;
    size_t cap = 0;
    void ensure(size_t bytes) {
        if (bytes <= cap) return;
        if (p) cudaFree(p);
        p = nullptr; cap = 0;
        size_t want = bytes + bytes / 4 + 256;
        CK(cudaMalloc(&p, want));
        cap = want;
    }
    void release() { if (p) cudaFree(p); p = nullptr; cap = 0; }
    template <class T> T* as() { return static_cast<T*>(p); }
};
struct PinBuf {
    void* p = nullptr;
    size_t cap = 0;
    void ensure(size_t bytes) {
        if (bytes <= cap) return;
        if (p) cudaFreeHost(p);
        p = nullptr; cap = 0;
        CK(cudaMallocHost(&p, bytes));
        cap = bytes;
    }
    void release() { if (p) cudaFreeHost(p); p = nullptr; cap = 0; }
    template <class T> T* as() { return static_cast<T*>(p); }
};

struct Wave {  // device buffers of one wave of trees; kept across builds
    DevBuf st, frames, recs, perm0, perm1, flags, unit_left, pool, pool_counter, jobs, scratch, active, error, final_ids, keys, sub_rows, sub_off, slots, abort, cur_normal, start_pos, root, shadow_stats;
    void release() {
        sub_rows.release(); sub_off.release(); slots.release(); abort.release(); cur_normal.release(); start_pos.release(); root.release(); shadow_stats.release();
        st.release(); frames.release(); recs.release(); perm0.release(); perm1.release(); flags.release(); unit_left.release();
        pool.release(); pool_counter.release(); jobs.release(); scratch.release(); active.release(); error.release(); final_ids.release(); keys.release();
    }
};
struct BuiltTreeView {  // views into the pinned HostWave buffers of the context
    const void* recs = nullptr;
    uint32_t n_recs = 0;
    const uint32_t* final_rows = nullptr;  // n entries
    const float* pool = nullptr;
};
struct StageWorker {  // one H2D lane of the staging pipeline: own stream, two pinned bounce buffers
    cudaStream_t st = nullptr;
    PinBuf pin[2];
    cudaEvent_t ev[2] = {nullptr, nullptr};
};
struct HostWave {  // pinned host copies of one wave's results; kept across builds
    PinBuf recs, final_rows, pool;
    void release() { recs.release(); final_rows.release(); pool.release(); }
};

}  // namespace

struct arroy_ctx {
    int device = 0;
    int sm_count = 132;
    cudaStream_t stream = nullptr;
    std::mutex mu;
    std::string err;
    // staged items
    bool staged = false;
    int metric = 0;
    uint32_t dim = 0, ld = 0;   // dim = the vectors' length on the device (binary-quantized metrics: the padded bit count)
    uint32_t user_dim = 0;      // the index' dimensions (what normalized_distance of the binary-quantized metrics divides by)
    uint64_t n = 0;
    DevBuf items, h0, h1, norms, maxbits;
    std::vector<uint32_t> ids;
    // scratch
    DevBuf s_rows, s_flags, s_margins, s_normal, s_unit, s_job, s_keys, s_keys2, s_dists, s_q, s_qh0, s_off, s_orows, s_odist, s_olen, s_misc;
    PinBuf pin;
    cudaEvent_t ev0 = nullptr, ev1 = nullptr;
    cudaStream_t side_stream = nullptr;   // host -> device flags while the persistent build kernel occupies `stream`
    cudaEvent_t ev_done = nullptr, ev_p0 = nullptr, ev_p1 = nullptr;   // ev_p0 / ev_p1 bracket the persistent build kernel
    double stats[8] = {0, 0, 0, 0, 0, 0, 0, 0};
    uint64_t shadow_rows = 0, shadow_rescored = 0, shadow_stage2 = 0, fused_root_rows = 0, fused_root_read = 0;
    uint64_t wave_key[4] = {0, 0, 0, 0}, wave_max = 0, wave_trees_ok = 0; bool wave_key_valid = false;   // shapes of the last successful build (do_build_begin)   // last build: rows scanned through the bf16 shadow / re-scored from f32
    uint64_t n_launches = 0, h2d_bytes = 0, d2h_bytes = 0;  // since create (arroy_b200_counters)
    cudaEvent_t tev0 = nullptr, tev1 = nullptr;
    std::vector<StageWorker> stage_workers;
    bool staging_open = false;             // between arroy_b200_stage_begin and arroy_b200_stage_end
    std::vector<float> stage_h0, stage_h1;  // headers decoded from the leaf values staged so far
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
    cudaGraph_t cached_graph = nullptr;
    cudaGraphExec_t cached_exec = nullptr;
    std::vector<uint8_t> cached_graph_key;  // BuildParams bytes + schedule the cached graph was captured for
    std::vector<HostWave> host_waves;
    double breakdown[8] = {0, 0, 0, 0, 0, 0, 0, 0};
    std::vector<cudaStream_t> tree_streams;   // one per tree of a wave (asynchronous per-tree chains)
    std::vector<cudaEvent_t> tree_events;     // join events, [0] = fork
    // tensor-core pre-filter of rerank_shared
    cublasHandle_t blas = nullptr;
    DevBuf x_gather, x_cnorm, x_ca, x_cb, x_gmax, x_qa, x_qb, x_twoe, x_qnorm, x_S, x_sel, x_beg, x_end, x_flag;
    uint64_t xf_calls = 0, xf_fallbacks = 0, xf_selected = 0, xf_queries = 0;
    cudaEvent_t xev[8] = {nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr};
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
    uint64_t fr_batches = 0, fr_fallbacks = 0;   // last search_batch call, ms: bitmap clear + tree walk, candidate sort, distances, top-k   // last rerank_shared call, ms: prep, score GEMM, select, re-score, top-k, exact dense path
};

namespace {

int metric_header_floats(int m) { return m == DOT_PRODUCT ? 2 : 1; }

void set_device(arroy_ctx* c) { CK(cudaSetDevice(c->device)); }

void require_staged(arroy_ctx* c) { if (!c->staged) throw NotStaged("items have not been staged on this context"); }

size_t work_smem(uint32_t ld, int njobs) { return (size_t)ld * 4 + (size_t)(njobs + 1) * 4 + 16; }

void launch_work(arroy_ctx* c, const Job* jobs, int njobs, int grid) {
    size_t smem = work_smem(c->ld, njobs);
    static std::atomic<size_t> configured{0};
    if (smem > 48 * 1024 && smem > configured.load()) {
        CK(cudaFuncSetAttribute(work_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        configured = smem;
    }
    work_kernel<<<grid, WORK_THREADS, smem, c->stream>>>(jobs, njobs, c->items.as<float>(), c->h0.as<float>(), c->dim, c->ld, c->metric);
    CK(cudaGetLastError());
    c->n_launches += 1;
}

void compute_norms(arroy_ctx* c, bool with_max) {
    c->norms.ensure(c->n * 4);
    c->maxbits.ensure(4);
    if (with_max) CK(cudaMemsetAsync(c->maxbits.p, 0, 4, c->stream));
    uint64_t warps = (c->n + 3) / 4;
    int grid = (int)std::min<uint64_t>((warps + 7) / 8, (uint64_t)c->sm_count * 16);
    if (grid < 1) grid = 1;
    norms_kernel<<<grid, 256, 0, c->stream>>>(c->items.as<float>(), c->n, c->dim, c->ld, c->norms.as<float>(), with_max ? c->maxbits.as<uint32_t>() : nullptr);
    CK(cudaGetLastError());
    c->n_launches += 1;
}

void alloc_items(arroy_ctx* c, int metric, uint32_t dim, uint64_t n, const uint32_t* ids) {
    if (metric < 0 || metric > BQ_MANHATTAN) throw ArgError("unknown metric");
    if (dim == 0) throw ArgError("dim must be > 0");
    c->user_dim = dim;
    if (is_bq(metric)) dim = (dim + 63u) / 64u * 64u;   // the bit string's length (binary_quantized.rs:80-92)
    if (n > 0xffffffffull) throw ArgError("too many items");
    for (uint64_t i = 1; i < n; ++i) if (ids[i] <= ids[i - 1]) throw ArgError("ids must be strictly ascending");
    // a restage invalidates everything derived from the previous items: the bf16 shadow, the 8-bit planes and the device forest
    // (its descendant rows were validated against the previous item count)
    c->staged = false; c->fr_valid = false; c->shadow_valid = false; c->planes_valid = false; c->forest_loaded = false; c->staging_open = false;
    c->stage_epoch += 1;
    c->metric = metric; c->dim = dim; c->ld = (dim + 31u) & ~31u; c->n = n;
    c->ids.assign(ids, ids + n);
    c->items.ensure(std::max<size_t>(16, (size_t)n * c->ld * 4));
    c->h0.ensure(std::max<size_t>(16, n * 4));
    c->h1.ensure(std::max<size_t>(16, n * 4));
    CK(cudaMemsetAsync(c->h0.p, 0, std::max<size_t>(16, n * 4), c->stream));
    CK(cudaMemsetAsync(c->h1.p, 0, std::max<size_t>(16, n * 4), c->stream));
}

// headers as Writer::add_item stores them: D::new_header(vector) (src/writer.rs:388-390)
void default_headers(arroy_ctx* c) {
    if ((c->metric == COSINE || c->metric == BQ_COSINE) && c->n > 0) {   // BQ cosine: sqrt(popcount-dot(v, v)) = sqrt(dim), exact in f32
        compute_norms(c, false);
        CK(cudaMemcpyAsync(c->h0.p, c->norms.p, c->n * 4, cudaMemcpyDeviceToDevice, c->stream));
    }
}

// Staging pipeline: W host threads, each decoding row chunks into its own pinned bounce buffers and
// issuing its own cudaMemcpyAsync on its own stream, so decode (host memcpy of unaligned values)
// and PCIe transfers of different chunks overlap. row_src(i) = address of the dim floats of row i.
// mode 0: row_src(i) = dim f32 (byte aligned only); mode 1 (binary quantized): row_src(i) = src_dim f32 to be quantized to +-1;
// mode 2 (binary quantized): row_src(i) = the stored bit string (dim / 8 bytes) to be expanded to +-1
template <class RowSrc>
void stage_rows_pipeline(arroy_ctx* c, uint64_t n, uint32_t dim, uint32_t ld, RowSrc row_src, float* dst_override = nullptr, size_t chunk_mb_override = 0, bool count_bytes = true,
                         int mode = 0, uint32_t src_dim = 0) {
    if (n == 0) return;
    // 8 lanes x 4 MB chunks: decode of one chunk overlaps the PCIe copies of the others
    unsigned W = std::min(8u, std::max(1u, std::thread::hardware_concurrency()));
    const size_t chunk_mb = chunk_mb_override ? chunk_mb_override : 4;
    const uint64_t chunk_rows = std::max<uint64_t>(1, (chunk_mb << 20) / ((size_t)ld * 4));
    const uint64_t n_chunks = (n + chunk_rows - 1) / chunk_rows;
    W = (unsigned)std::min<uint64_t>(W, n_chunks);
    if (c->stage_workers.size() < W) c->stage_workers.resize(W);
    for (unsigned w = 0; w < W; ++w) {
        StageWorker& sw = c->stage_workers[w];
        if (!sw.st) CK(cudaStreamCreateWithFlags(&sw.st, cudaStreamNonBlocking));
        for (int k = 0; k < 2; ++k) { sw.pin[k].ensure(chunk_rows * ld * 4); if (!sw.ev[k]) CK(cudaEventCreateWithFlags(&sw.ev[k], cudaEventDisableTiming)); }
    }
    CK(cudaStreamSynchronize(c->stream));  // the destination buffer must not be in use
    std::mutex emu;
    std::string err;
    float* dst = dst_override ? dst_override : c->items.as<float>();
    auto worker = [&](unsigned w) {
        try {
            CK(cudaSetDevice(c->device));
            StageWorker& sw = c->stage_workers[w];
            bool used[2] = {false, false};
            int k = 0;
            for (uint64_t ch = w; ch < n_chunks; ch += W, k ^= 1) {
                const uint64_t r0 = ch * chunk_rows, rows = std::min<uint64_t>(chunk_rows, n - r0);
                if (used[k]) CK(cudaEventSynchronize(sw.ev[k]));
                float* b = sw.pin[k].as<float>();
                for (uint64_t i = 0; i < rows; ++i) {
                    float* o = b + i * ld;
                    if (mode == 0) memcpy(o, row_src(r0 + i), 4ull * dim);
                    else if (mode == 1) {
                        const uint8_t* sp = row_src(r0 + i);
                        for (uint32_t t = 0; t < src_dim; ++t) { uint32_t bits; memcpy(&bits, sp + 4ull * t, 4); o[t] = (bits >> 31) ? -1.0f : 1.0f; }
                        for (uint32_t t = src_dim; t < dim; ++t) o[t] = -1.0f;
                    } else {
                        const uint8_t* sp = row_src(r0 + i);
                        for (uint32_t t = 0; t < dim; ++t) o[t] = ((sp[t >> 3] >> (t & 7)) & 1) ? 1.0f : -1.0f;   // little-endian words: bit t of the string
                    }
                    for (uint32_t t = dim; t < ld; ++t) o[t] = 0.f;
                }
                CK(cudaMemcpyAsync(dst + r0 * ld, b, rows * ld * 4, cudaMemcpyHostToDevice, sw.st));
                CK(cudaEventRecord(sw.ev[k], sw.st));
                used[k] = true;
            }
            CK(cudaStreamSynchronize(sw.st));
        } catch (const std::exception& e) { std::lock_guard<std::mutex> lk(emu); if (err.empty()) err = e.what(); }
    };
    if (W == 1) worker(0);
    else { std::vector<std::thread> th; for (unsigned w = 0; w < W; ++w) th.emplace_back(worker, w); for (auto& x : th) x.join(); }
    if (!err.empty()) throw CudaError(err);
    if (count_bytes) c->h2d_bytes += n * (uint64_t)ld * 4;
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

// The control kernel is compiled once per metric (and per cluster size): it is bound by instruction fetch, so every
// instantiation only carries its own metric's code.
template <bool SMEM_WS, int CS>
const void* control_fn(int metric) {
    switch (metric) {
        case EUCLIDEAN: return reinterpret_cast<const void*>(&control_kernel<SMEM_WS, CS, EUCLIDEAN>);
        case COSINE: return reinterpret_cast<const void*>(&control_kernel<SMEM_WS, CS, COSINE>);
        case DOT_PRODUCT: return reinterpret_cast<const void*>(&control_kernel<SMEM_WS, CS, DOT_PRODUCT>);
        case MANHATTAN: return reinterpret_cast<const void*>(&control_kernel<SMEM_WS, CS, MANHATTAN>);
        default: break;
    }
    // binary-quantized metrics: persistent, single-CTA and global-workspace variants only (no cluster variants)
    if constexpr (CS <= 1) {
        switch (metric) {
            case BQ_EUCLIDEAN: return reinterpret_cast<const void*>(&control_kernel<SMEM_WS, CS, BQ_EUCLIDEAN>);
            case BQ_COSINE: return reinterpret_cast<const void*>(&control_kernel<SMEM_WS, CS, BQ_COSINE>);
            default: return reinterpret_cast<const void*>(&control_kernel<SMEM_WS, CS, BQ_MANHATTAN>);
        }
    }
    return nullptr;
}
inline const void* control_fn(bool smem_ws, int cs, int metric) {
    if (!smem_ws) return control_fn<false, 1>(metric);
    if (cs == 0) return control_fn<true, 0>(metric);   // persistent schedule
    return cs == 16 ? control_fn<true, 16>(metric) : (cs == 8 ? control_fn<true, 8>(metric) : control_fn<true, 1>(metric));
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
    size_t ws_bytes = (size_t)WS_VECS * ld * 4;
    int use_smem = ws_bytes <= 200 * 1024 ? 1 : 0;
    if (!use_smem) W.scratch.ensure(ws_bytes * tw);
    // speculative two_means (build.cuh): needs the 24-vector workspace in shared memory
    const int spec = (use_smem && (size_t)WS_VECS_SPEC * ld * 4 <= 200 * 1024) ? 1 : 0;
    if (spec) ws_bytes = (size_t)WS_VECS_SPEC * ld * 4;

    BuildParams P{};
    P.items = c->items.as<float>(); P.ih0 = c->h0.as<float>(); P.ih1 = c->h1.as<float>();
    P.n = (uint32_t)n; P.d = c->dim; P.ld = ld; P.metric = c->metric; P.K = K; P.n_trees = tw;
    P.st = W.st.as<TreeState>(); P.frames = W.frames.as<Frame>(); P.recs = W.recs.as<Record>(); P.rec_cap = rec_cap;
    P.perm[0] = W.perm0.as<uint32_t>(); P.perm[1] = W.perm1.as<uint32_t>();
    P.flags = W.flags.as<uint8_t>(); P.unit_left = W.unit_left.as<uint32_t>(); P.units_per_tree = units;
    P.pool = W.pool.as<float>(); P.pool_stride = pool_stride; P.pool_cap = pool_cap; P.pool_counter = W.pool_counter.as<uint32_t>();
    P.jobs = W.jobs.as<Job>(); P.scratch = W.scratch.as<float>(); P.use_smem_ws = use_smem; P.spec = spec;
    P.active = W.active.as<uint32_t>(); P.error = W.error.as<int32_t>();
    P.sub_rows = nullptr; P.sub_off = nullptr;
    // cluster-resident nodes: up to ~6 MB of item rows per scan (2048 rows at d = 768, every node of a 10k x 64 index)
    P.small_max = (uint32_t)std::max<uint64_t>(2048, (6ull << 20) / (4ull * ld));
    P.max_inner = 1024u;   // attempts per launch; `cancel` is polled between launches
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
    c->n_launches += 2;  // + finalize_kernel below

    const size_t ctrl_smem = use_smem ? ws_bytes : 0;
    if (ctrl_smem > 48 * 1024) CK(cudaFuncSetAttribute(control_fn(true, 1, c->metric), cudaFuncAttributeMaxDynamicSharedMemorySize, (int)ctrl_smem));
    const size_t wsmem = work_smem(ld, (int)tw);
    if (wsmem > 48 * 1024) CK(cudaFuncSetAttribute(work_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)wsmem));
    const size_t limb_smem = (size_t)PLANES_LIMBS * ld;   // work_kernel_shadow's limbs of the normal
    if (wsmem + limb_smem > 48 * 1024) CK(cudaFuncSetAttribute(work_kernel_shadow, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(wsmem + limb_smem)));
    const int work_grid = c->sm_count * 3;

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
    const void* ctrl1 = control_fn(use_smem != 0, 1, c->metric);
    // Few trees on this GPU = the chain of attempts of each tree is the critical path: the async schedule runs the control kernel
    // as a thread-block cluster that scans small nodes itself (build.cuh control_kernel<.., CS = 8 | 16>).
    // measured: d = 64, 1-10 trees: 24 -> 20 us per attempt; d = 768: 38 -> 37 us for one tree but slower from ~6 trees on
    const int cluster = (!lockstep && use_smem && c->dim <= 256 && !is_bq(c->metric)) ? (tw <= 8 ? 16 : (tw <= 16 ? 8 : 1)) : 1;
    const void* ctrlc = control_fn(use_smem != 0, cluster, c->metric);
    if (cluster > 1) {
        CK(cudaFuncSetAttribute(ctrlc, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)ctrl_smem));
        if (cluster == 16) CK(cudaFuncSetAttribute(ctrlc, cudaFuncAttributeNonPortableClusterSizeAllowed, 1));
    }

    // Persistent schedule (default): ONE cooperative launch per wave — a control CTA per tree plus worker CTAs on every SM
    // (build.cuh control_kernel<.., CS = 0>). Needs two CTAs per SM to have enough workers next to the control CTAs; with
    // a big workspace (d > 1152) that means giving up the speculative two_means.
    bool persist = false;
    int pgrid = 0;
    size_t psmem = ctrl_smem;
    const void* ctrlp = nullptr;
    // It wins where the chain of attempts is the critical path (few trees per GPU, small indexes); a wave that is bandwidth-bound
    // from start to end (10M x 100 trees) runs a little faster on work_kernel's three scanning CTAs per SM.
    if ((double)n * (double)tw <= 2.0e8 && !lockstep && use_smem && ld <= 8u * CTRL_THREADS && n < (1ull << 29)) {
        ctrlp = control_fn(true, 0, c->metric);
        const size_t cand[2] = {ctrl_smem, (size_t)WS_VECS * ld * 4};
        for (int k = 0; k < 2 && !persist; ++k) {
            if (k == 1 && !P.spec) break;
            CK(cudaFuncSetAttribute(ctrlp, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)cand[k]));
            int nb = 0;
            CK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&nb, ctrlp, CTRL_THREADS, cand[k]));
            const int cap = nb * c->sm_count;
            if ((nb >= 2 || k == 1) && cap >= (int)tw + std::max(16, c->sm_count / 2)) { persist = true; pgrid = cap; psmem = cand[k]; if (k == 1) P.spec = 0; }
        }
    }
    // scans through the 8-bit planes of the items (kernels.cuh scan_claim_planes): nodes of more than shadow_min_units units
    if (!is_bq(c->metric) && P.d >= 64 && P.d <= PLANES_MAX_D && n * (uint64_t)ld >= (1ull << 22)) {
        planes_prepare(c);
        P.planes = PlaneRows{c->pl_hi.as<int8_t>(), c->pl_lo.as<int8_t>(), c->pl_scale.as<float>()};
        W.shadow_stats.ensure(24);
        CK(cudaMemsetAsync(W.shadow_stats.p, 0, 24, c->stream));
        P.shadow_stats = W.shadow_stats.as<unsigned long long>();
        // many trees per GPU: bandwidth decides, every node goes through the shadow; few: the chain of attempts decides and
        // small nodes keep the one-unit claims of the exact scan (more CTAs per node)
        P.shadow_min_units = (!persist || tw >= 32) ? 12u : (tw >= 12 ? 64u : 128u);
    }
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
        // 8-lanes-per-row path, and a batch of normals fits next to nothing else in the workers' shared memory
        P.root_fused = (!sub.rows && tw >= 2 && P.d >= 32 && (size_t)ROOT_TB * ld * 4 <= psmem) ? 1 : 0;
        W.root.ensure(8);
        CK(cudaMemsetAsync(W.root.p, 0, 8, c->stream));
        P.root_ready = W.root.as<uint32_t>(); P.root_ticket = W.root.as<uint32_t>() + 1;
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
            if (c->cached_exec) { cudaGraphExecDestroy(c->cached_exec); c->cached_exec = nullptr; }
            if (c->cached_graph) { cudaGraphDestroy(c->cached_graph); c->cached_graph = nullptr; }
            c->cached_graph_key.clear();
            while (c->tree_streams.size() < tw) { cudaStream_t st; CK(cudaStreamCreateWithFlags(&st, cudaStreamNonBlocking)); c->tree_streams.push_back(st); }
            while (c->tree_events.size() < (size_t)tw + 1) { cudaEvent_t ev; CK(cudaEventCreateWithFlags(&ev, cudaEventDisableTiming)); c->tree_events.push_back(ev); }
            const size_t wsmem1 = work_smem(ld, 1);
            cudaGraph_t graph = nullptr;
            CK(cudaStreamBeginCapture(c->stream, cudaStreamCaptureModeThreadLocal));
            CK(cudaEventRecord(c->tree_events[0], c->stream));
            for (uint32_t t = 0; t < tw; ++t) {   // one tree (one cluster) per control launch, sm_count work CTAs per work launch
                cudaStream_t st = c->tree_streams[t];
                CK(cudaStreamWaitEvent(st, c->tree_events[0], 0));
                for (int i = 0; i < ASYNC_BATCH; ++i) {
                    launch_control(ctrlc, 1, cluster, ctrl_smem, st, P, t);
                    if (P.planes.hi) work_kernel_shadow<<<c->sm_count, WORK_THREADS, wsmem1 + limb_smem, st>>>(P.jobs + t, 1, P.items, P.planes, P.ih0, P.d, P.ld, P.metric, P.shadow_min_units, P.shadow_stats);
                    else work_kernel<<<c->sm_count, WORK_THREADS, wsmem1, st>>>(P.jobs + t, 1, P.items, P.ih0, P.d, P.ld, P.metric);
                }
                CK(cudaEventRecord(c->tree_events[1 + t], st));
                CK(cudaStreamWaitEvent(c->stream, c->tree_events[1 + t], 0));
            }
            CK(cudaStreamEndCapture(c->stream, &graph));
            c->cached_graph = graph;
            CK(cudaGraphInstantiate(&gexec, graph, 0));
            c->cached_exec = gexec;
            c->cached_graph_key = key;
        }
    }

    c->breakdown[1] += ms_since(t_graph);
    auto t_loop = std::chrono::steady_clock::now();
    c->pin.ensure(64);
    volatile uint32_t* h_active = c->pin.as<uint32_t>();
    volatile int32_t* h_error = reinterpret_cast<volatile int32_t*>(c->pin.as<uint32_t>() + 1);
    std::vector<cudaEvent_t> pev;
    struct EvGuard { std::vector<cudaEvent_t>& v; ~EvGuard() { for (auto e : v) cudaEventDestroy(e); } } evg{pev};
    if (profile) { pev.resize(2 * LOCKSTEP_BATCH); for (auto& e : pev) CK(cudaEventCreate(&e)); }
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
                if (P.planes.hi) work_kernel_shadow<<<c->sm_count * 2, WORK_THREADS, wsmem + limb_smem, c->stream>>>(P.jobs, (int)tw, P.items, P.planes, P.ih0, P.d, P.ld, P.metric, P.shadow_min_units, P.shadow_stats);
                else work_kernel<<<work_grid, WORK_THREADS, wsmem, c->stream>>>(P.jobs, (int)tw, P.items, P.ih0, P.d, P.ld, P.metric);
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

    // results: merge the ping-pong id buffers, then bring everything to (pinned) host memory
    W.final_ids.ensure(4ull * n * tw);
    finalize_kernel<<<dim3(64, tw), 256, 0, c->stream>>>(P, W.final_ids.as<uint32_t>());
    CK(cudaGetLastError());
    std::vector<TreeState> st(tw);
    uint32_t pool_used = 0;
    CK(cudaMemcpyAsync(st.data(), W.st.p, sizeof(TreeState) * tw, cudaMemcpyDeviceToHost, c->stream));
    CK(cudaMemcpyAsync(&pool_used, W.pool_counter.p, 4, cudaMemcpyDeviceToHost, c->stream));
    CK(cudaStreamSynchronize(c->stream));
    if (c->host_waves.size() <= wave_no) c->host_waves.resize(wave_no + 1);
    HostWave& H = c->host_waves[wave_no];
    uint64_t total_recs = 0;
    for (uint32_t t = 0; t < tw; ++t) total_recs += st[t].n_recs;
    H.pool.ensure(std::max<size_t>(16, (size_t)pool_used * pool_stride * 4));
    H.recs.ensure(std::max<size_t>(16, sizeof(Record) * total_recs));
    H.final_rows.ensure(std::max<size_t>(16, 4ull * n * tw));
    if (pool_used) CK(cudaMemcpyAsync(H.pool.p, W.pool.p, (size_t)pool_used * pool_stride * 4, cudaMemcpyDeviceToHost, c->stream));
    CK(cudaMemcpyAsync(H.final_rows.p, W.final_ids.p, 4ull * n * tw, cudaMemcpyDeviceToHost, c->stream));
    out_pool_stride = pool_stride;
    out_trees.resize(tw);
    uint64_t rec_off = 0;
    for (uint32_t t = 0; t < tw; ++t) {
        out_trees[t].recs = static_cast<const void*>(H.recs.as<Record>() + rec_off);
        out_trees[t].n_recs = st[t].n_recs;
        out_trees[t].final_rows = H.final_rows.as<uint32_t>() + (size_t)t * n;
        out_trees[t].pool = H.pool.as<float>();
        CK(cudaMemcpyAsync(H.recs.as<Record>() + rec_off, W.recs.as<Record>() + (size_t)t * rec_cap, sizeof(Record) * st[t].n_recs, cudaMemcpyDeviceToHost, c->stream));
        rec_off += st[t].n_recs;
        c->stats[0] += (double)st[t].scanned;
        c->stats[2] += (double)st[t].n_splits_tried;
        c->stats[3] += (double)st[t].n_random;
        c->stats[7] += (double)st[t].n_misspec;
        if (sub.end_pos) sub.end_pos[t0 + t] = st[t].pos;
    }
    if (persist && P.root_fused) { c->fused_root_rows += (uint64_t)tw * n; c->fused_root_read += n; }
    if (P.shadow_stats) {
        unsigned long long hs[3] = {0, 0, 0};
        CK(cudaMemcpyAsync(hs, P.shadow_stats, 24, cudaMemcpyDeviceToHost, c->stream));
        CK(cudaStreamSynchronize(c->stream));
        c->shadow_rows += hs[0]; c->shadow_rescored += hs[1]; c->shadow_stage2 += hs[2];
    }
    CK(cudaStreamSynchronize(c->stream));
    c->d2h_bytes += (uint64_t)pool_used * pool_stride * 4 + sizeof(TreeState) * tw + sizeof(Record) * total_recs + 4ull * n * tw;
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
    const uint64_t per_tree = n * (4 + 4 + 1 + 4) + (n / SCAN_UNIT + 1) * 4 + sizeof(Frame) * (uint64_t)MAX_DEPTH + 16ull * 8 * leaves_est +
                              4ull * (c->ld + NORMAL_HDR) * 4 * leaves_est + 4096;
    uint64_t reusable = c->wave.perm0.cap + c->wave.perm1.cap + c->wave.flags.cap + c->wave.final_ids.cap + c->wave.pool.cap + c->wave.recs.cap;
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
    int grid = (int)std::min<uint64_t>(units, (uint64_t)c->sm_count * 3);
    launch_work(c, c->s_job.as<Job>(), 1, grid);
    CK(cudaMemcpyAsync(out_side, c->s_flags.p, n_rows, cudaMemcpyDeviceToHost, c->stream));
    if (out_margin) CK(cudaMemcpyAsync(out_margin, c->s_margins.p, n_rows * 4, cudaMemcpyDeviceToHost, c->stream));
    CK(cudaStreamSynchronize(c->stream));
}

// ---- tensor-core pre-filter helpers (rerank_shared) ---------------------------------------------
// candidate matrix for the score GEMM: the item matrix in place when `rows` is a contiguous range,
// else a gathered copy
const float* xf_candidates(arroy_ctx* c, const uint32_t* rows, uint32_t nc) {
    bool contiguous = true;
    for (uint64_t i = 1; i < nc && contiguous; ++i) contiguous = rows[i] == rows[0] + i;
    if (contiguous) return c->items.as<float>() + (size_t)rows[0] * c->ld;
    c->x_gather.ensure(4ull * nc * c->ld);
    xf_gather_kernel<<<c->sm_count * 8, 256, 0, c->stream>>>(c->x_gather.as<float4>(), c->items.as<float4>(), c->s_rows.as<uint32_t>(), nc, c->ld / 4);
    CK(cudaGetLastError());
    c->n_launches += 1;
    return c->x_gather.as<float>();
}

// S (m x nc, pitch lds) = Q . cand^T with TF32 inputs and FP32 accumulation. engine 0: the wgmma
// kernel of tcgemm.cuh; engine 1: cuBLAS (kept as the cross-check of the hand-written kernel)
void xf_scores(arroy_ctx* c, const float* q, uint32_t m, const float* cand, uint32_t nc, float* S, uint32_t lds, TgEpilogue ep, int engine) {
    if (engine == 0) {
        const int mc = (getenv("ARROY_B200_XGEMM_MC") && atoi(getenv("ARROY_B200_XGEMM_MC")) == 1) ? 1 : 2;
        if (!tcgemm_tf32(q, m, cand, nc, c->ld, S, lds, ep, c->sm_count, c->stream, mc)) throw CudaError(std::string("tcgemm_tf32 launch failed: ") + cudaGetErrorString(cudaGetLastError()));
        c->n_launches += 1;
        return;
    }
    if (!c->blas) { if (cublasCreate(&c->blas) != CUBLAS_STATUS_SUCCESS) throw CudaError("cublasCreate failed"); }
    if (cublasSetStream(c->blas, c->stream) != CUBLAS_STATUS_SUCCESS) throw CudaError("cublasSetStream failed");
    const float one = 1.0f, zero = 0.0f;
    cublasStatus_t st = cublasGemmEx(c->blas, CUBLAS_OP_T, CUBLAS_OP_N, (int)nc, (int)m, (int)c->ld, &one, cand, CUDA_R_32F, (int)c->ld,
                                     q, CUDA_R_32F, (int)c->ld, &zero, S, CUDA_R_32F, (int)lds, CUBLAS_COMPUTE_32F_FAST_TF32, CUBLAS_GEMM_DEFAULT);
    if (st != CUBLAS_STATUS_SUCCESS) throw CudaError("cublasGemmEx failed with status " + std::to_string((int)st));
    if (ep.mode != TG_RAW) { tg_finish_kernel<<<c->sm_count * 8, 256, 0, c->stream>>>(S, m, nc, lds, ep); CK(cudaGetLastError()); }
    c->n_launches += 2;
}

int xf_engine() { const char* e = getenv("ARROY_B200_XGEMM"); return (e && strcmp(e, "cublas") == 0) ? 1 : 0; }

// ---- fused re-rank (frerank.cuh) -------------------------------------------------------------------
bool frerank_enabled(arroy_ctx* c, uint32_t k) {
    const char* e = getenv("ARROY_B200_FRERANK");
    const bool off = e != nullptr && atoi(e) == 0;
    return !off && c->metric != MANHATTAN && !is_bq(c->metric) && k <= (uint32_t)FR_SURV && frerank_smem(c->ld) <= 200 * 1024;
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
    planes_encode_kernel<<<(unsigned)blocks, 256, 0, c->stream>>>(c->items.as<float>(), c->n, c->ld, c->pl_hi.as<int8_t>(), c->pl_lo.as<int8_t>(), c->pl_scale.as<float>());
    CK(cudaGetLastError());
    c->n_launches += 1;
    c->planes_valid = true;
}

void frerank_prepare(arroy_ctx* c) {
    if (c->fr_valid) return;
    shadow_prepare(c);
    c->fr_norm.ensure(std::max<size_t>(16, c->n * 4));
    c->fr_gmax.ensure(4);
    { uint64_t warps = (c->n + 3) / 4; int g = (int)std::max<uint64_t>(1, std::min<uint64_t>((warps + 7) / 8, (uint64_t)c->sm_count * 16));
      norms_kernel<<<g, 256, 0, c->stream>>>(c->items.as<float>(), c->n, c->dim, c->ld, c->fr_norm.as<float>(), nullptr); CK(cudaGetLastError()); }
    CK(cudaMemsetAsync(c->fr_gmax.p, 0, 4, c->stream));
    fr_gmax_kernel<<<(unsigned)((c->n + 255) / 256), 256, 0, c->stream>>>(c->fr_norm.as<float>(), c->h0.as<float>(), c->n, c->metric, c->fr_gmax.as<uint32_t>());
    CK(cudaGetLastError());
    c->n_launches += 2;
    c->fr_valid = true;
}

// launches the fused kernel for m queries whose sorted candidate rows are rows[beg[q] .. end[q]); results in s_orows / s_odist /
// s_olen, per-query status in fr_status (0 = done, 1 = needs the plain kernels)
void frerank_launch(arroy_ctx* c, uint32_t m, const float* d_q, const uint32_t* d_qrows, const float* d_qh0, const uint32_t* d_rows,
                    const uint64_t* d_beg, const uint64_t* d_end, uint32_t k) {
    frerank_prepare(c);
    c->fr_status.ensure(4ull * m);
    FrParams P{};
    P.items = c->items.as<float>(); P.shadow = c->fr_shadow.as<__nv_bfloat16>(); P.ih0 = c->h0.as<float>(); P.cnorm = c->fr_norm.as<float>();
    P.d = c->dim; P.ld = c->ld; P.metric = c->metric;
    P.queries = d_q; P.qrows = d_qrows; P.qh0 = d_qh0;
    P.rows = d_rows; P.seg_beg = d_beg; P.seg_end = d_end;
    P.k = k; P.rel = fr_rel(c->dim); P.sub = fr_sub(c->dim); P.hmin = cos_header_min(c->dim); P.gmax_bits = c->fr_gmax.as<uint32_t>();
    P.out_rows = c->s_orows.as<uint32_t>(); P.out_dist = c->s_odist.as<float>(); P.out_len = c->s_olen.as<uint32_t>(); P.status = c->fr_status.as<int32_t>();
    const size_t smem = frerank_smem(c->ld);
    static std::atomic<size_t> configured{0};
    if (smem > 48 * 1024 && smem > configured.load()) { CK(cudaFuncSetAttribute(frerank_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem)); configured = smem; }
    frerank_kernel<<<m, FR_THREADS, smem, c->stream>>>(P);
    CK(cudaGetLastError());
    c->n_launches += 1;
    c->fr_batches += 1;
}

bool frerank_ok(arroy_ctx* c, uint32_t m) {   // after the stream is idle: did every query finish in the fused kernel?
    std::vector<int32_t> st(m);
    CK(cudaMemcpy(st.data(), c->fr_status.p, 4ull * m, cudaMemcpyDeviceToHost));
    for (int32_t x : st) if (x != 0) { c->fr_fallbacks += 1; return false; }
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
    void operator()() { if (!c->xev[n]) CK(cudaEventCreate(&c->xev[n])); CK(cudaEventRecord(c->xev[n], c->stream)); ++n; }
    void add_to(double* b) const { for (int i = 0; i + 1 < n; ++i) { float ms = 0; CK(cudaEventElapsedTime(&ms, c->xev[i], c->xev[i + 1])); b[i] += ms; } }
};

// A call's queries on the device: by item their rows (vecs == nullptr), by vector their vectors (rows == nullptr), and their
// first header.
struct DevQueries {
    const float* vecs = nullptr;
    const uint32_t* rows = nullptr;
    const float* h0 = nullptr;
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
    return Q;
}

// The re-rank of m queries whose sorted candidate rows are rows[beg[q] .. end[q]): at most max_len rows per query, n_keys rows
// in the whole array (s_keys / s_dists hold as many). Results in s_orows / s_odist / s_olen. With try_fused the fused kernel
// goes first, and the plain kernels run only if a query needs them: distance_kernel, then topk_kernel, or for k beyond the
// top-k buffer a full segmented sort of the keys and take_sorted_kernel. `mark`, when given, is recorded after the distances.
// (beg / end are not const: the key sort stays the CUB instantiation with uint64_t* offsets, as the walk's candidate sort)
void rerank_segments(arroy_ctx* c, uint32_t m, const DevQueries& Q, const uint32_t* rows, uint64_t* beg, uint64_t* end,
                     uint64_t n_keys, uint64_t max_len, uint32_t k, bool try_fused, Marks* mark) {
    if (try_fused && frerank_enabled(c, k)) {   // one fused kernel per query: bf16 pre-filter + exact re-score + top-k (frerank.cuh)
        frerank_launch(c, m, Q.vecs, Q.rows, Q.h0, rows, beg, end, k);
        CK(cudaStreamSynchronize(c->stream));
        if (frerank_ok(c, m)) { if (mark) (*mark)(); return; }
    }
    if (max_len) {   // Manhattan sums one row per lane, the other metrics four rows per warp
        const uint64_t per = (c->metric == MANHATTAN || c->metric == BQ_MANHATTAN) ? 32 : 4;
        const uint64_t warps = (max_len + per - 1) / per;
        const uint32_t gx = (uint32_t)std::max<uint64_t>(1, std::min<uint64_t>((warps + 7) / 8, std::max<uint64_t>(1, ((uint64_t)c->sm_count * 8) / std::min<uint32_t>(m, c->sm_count * 8u))));
        distance_kernel<<<dim3(gx, m), 256, 0, c->stream>>>(c->items.as<float>(), c->h0.as<float>(), c->dim, c->ld, c->metric, Q.vecs, Q.rows, Q.h0, m,
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
        topk_kernel<<<m, TOPK_THREADS, 0, c->stream>>>(c->s_keys.as<unsigned long long>(), c->s_dists.as<float>(), rows, beg, end, k, c->metric,
                                                       c->s_orows.as<uint32_t>(), c->s_odist.as<float>(), c->s_olen.as<uint32_t>());
    CK(cudaGetLastError());
}

// The results of queries q0 .. q0 + m (k slots each) to the caller's arrays, with the walk status when out_status is given.
void copy_results(arroy_ctx* c, uint32_t q0, uint32_t m, uint32_t k, uint32_t* out_rows, float* out_dist, uint32_t* out_len, int32_t* out_status = nullptr) {
    CK(cudaMemcpyAsync(out_rows + (size_t)q0 * k, c->s_orows.p, 4ull * m * k, cudaMemcpyDeviceToHost, c->stream));
    CK(cudaMemcpyAsync(out_dist + (size_t)q0 * k, c->s_odist.p, 4ull * m * k, cudaMemcpyDeviceToHost, c->stream));
    CK(cudaMemcpyAsync(out_len + q0, c->s_olen.p, 4ull * m, cudaMemcpyDeviceToHost, c->stream));
    if (out_status) CK(cudaMemcpyAsync(out_status + q0, c->w_status.p, 4ull * m, cudaMemcpyDeviceToHost, c->stream));
    CK(cudaStreamSynchronize(c->stream));
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

int32_t arroy_b200_create(int32_t device, arroy_ctx** out) {
    if (!out) return ARROY_B200_ERR_INVALID;
    *out = nullptr;
    int count = 0;
    if (cudaGetDeviceCount(&count) != cudaSuccess || count <= 0 || device < 0 || device >= count) { cudaGetLastError(); return ARROY_B200_ERR_CUDA; }
    arroy_ctx* c = nullptr;
    try {
        c = new arroy_ctx();
        c->device = device;
        CK(cudaSetDevice(device));
        cudaDeviceProp prop;
        CK(cudaGetDeviceProperties(&prop, device));
        c->sm_count = prop.multiProcessorCount;
        CK(cudaStreamCreateWithFlags(&c->stream, cudaStreamNonBlocking));
        CK(cudaEventCreate(&c->ev0));
        CK(cudaEventCreate(&c->ev1));
        CK(cudaStreamCreateWithFlags(&c->side_stream, cudaStreamNonBlocking));
        CK(cudaEventCreateWithFlags(&c->ev_done, cudaEventDisableTiming));
        CK(cudaEventCreate(&c->ev_p0));
        CK(cudaEventCreate(&c->ev_p1));
        CK(cudaEventCreate(&c->tev0));
        CK(cudaEventCreate(&c->tev1));
        // fail loudly if the kernels were not built for this device
        cudaFuncAttributes fa;
        CK(cudaFuncGetAttributes(&fa, work_kernel));
    } catch (const std::exception& e) {
        fprintf(stderr, "arroy_b200_create: %s\n", e.what());
        delete c;
        cudaGetLastError();
        return ARROY_B200_ERR_CUDA;
    }
    *out = c;
    return ARROY_B200_OK;
}

void arroy_b200_destroy(arroy_ctx* c) {
    if (!c) return;
    cudaSetDevice(c->device);
    if (c->stream) cudaStreamSynchronize(c->stream);
    DevBuf* bufs[] = {&c->items, &c->h0, &c->h1, &c->norms, &c->maxbits, &c->s_rows, &c->s_flags, &c->s_margins, &c->s_normal, &c->s_unit, &c->s_job,
                      &c->s_keys, &c->s_keys2, &c->s_dists, &c->s_q, &c->s_qh0, &c->s_off, &c->s_orows, &c->s_odist, &c->s_olen, &c->s_misc};
    for (auto* b : bufs) b->release();
    { DevBuf* xb[] = {&c->pl_hi, &c->pl_lo, &c->pl_scale, &c->fr_shadow, &c->fr_norm, &c->fr_gmax, &c->fr_status, &c->x_gather, &c->x_cnorm, &c->x_ca, &c->x_cb, &c->x_gmax, &c->x_qa, &c->x_qb, &c->x_twoe, &c->x_qnorm, &c->x_S, &c->x_sel, &c->x_beg, &c->x_end, &c->x_flag}; for (auto* b : xb) b->release(); }
    if (c->blas) cublasDestroy(c->blas);
    for (auto& e : c->xev) if (e) cudaEventDestroy(e);
    if (c->cached_exec) cudaGraphExecDestroy(c->cached_exec);
    if (c->cached_graph) cudaGraphDestroy(c->cached_graph);
    for (auto& sw : c->stage_workers) { sw.pin[0].release(); sw.pin[1].release(); if (sw.ev[0]) cudaEventDestroy(sw.ev[0]); if (sw.ev[1]) cudaEventDestroy(sw.ev[1]); if (sw.st) cudaStreamDestroy(sw.st); }
    { DevBuf* fb[] = {&c->f_kind, &c->f_left, &c->f_right, &c->f_nidx, &c->f_nh0, &c->f_doff, &c->f_dlen, &c->f_normals, &c->f_desc, &c->f_roots, &c->f_rec, &c->f_nofn,
                      &c->w_heaps, &c->w_cand, &c->w_cand2, &c->w_count, &c->w_bitmap, &c->w_status, &c->w_beg, &c->w_end, &c->w_qrows, &c->w_tmp, &c->w_pre};
      for (auto* b : fb) b->release(); }
    c->pin.release();
    c->wave.release(); c->wave_key_valid = false;
    for (auto& hw : c->host_waves) hw.release();
    if (c->ev0) cudaEventDestroy(c->ev0);
    if (c->ev1) cudaEventDestroy(c->ev1);
    if (c->ev_done) cudaEventDestroy(c->ev_done);
    if (c->ev_p0) cudaEventDestroy(c->ev_p0);
    if (c->ev_p1) cudaEventDestroy(c->ev_p1);
    if (c->side_stream) cudaStreamDestroy(c->side_stream);
    if (c->tev0) cudaEventDestroy(c->tev0);
    if (c->tev1) cudaEventDestroy(c->tev1);
    for (auto st : c->tree_streams) cudaStreamDestroy(st);
    for (auto ev : c->tree_events) cudaEventDestroy(ev);
    if (c->stream) cudaStreamDestroy(c->stream);
    delete c;
}

const char* arroy_b200_last_error(arroy_ctx* c) { return c ? c->err.c_str() : "null context"; }

int32_t arroy_b200_stage_items(arroy_ctx* c, int32_t metric, uint32_t dim, uint64_t n, const uint32_t* ids, const uint8_t* const* leaf_values) {
    return guarded(c, [&] {
        set_device(c);
        if (n && (!ids || !leaf_values)) throw ArgError("null ids / leaf_values");
        alloc_items(c, metric, dim, n, ids);
        const uint32_t ld = c->ld;
        const int hf = metric_header_floats(metric);
        std::vector<float> h0(n), h1(n, 0.f);
        // decode the unaligned LMDB values: [tag][Header][dim x f32]
        {
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
        const size_t voff = 1 + 4 * (size_t)hf;
        // binary-quantized leaves store the bit string (node.rs:224-228 with VectorCodec = BinaryQuantized)
        stage_rows_pipeline(c, n, c->dim, ld, [&](uint64_t i) { return leaf_values[i] + voff; }, nullptr, 0, true, is_bq(metric) ? 2 : 0);
        if (n) {
            CK(cudaMemcpyAsync(c->h0.p, h0.data(), n * 4, cudaMemcpyHostToDevice, c->stream));
            CK(cudaMemcpyAsync(c->h1.p, h1.data(), n * 4, cudaMemcpyHostToDevice, c->stream));
        }
        CK(cudaStreamSynchronize(c->stream));
        c->h2d_bytes += 8 * n;
        c->staged = true;
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
        stage_rows_pipeline(c, n_rows, c->dim, c->ld, [&](uint64_t i) { return leaf_values[i] + voff; }, c->items.as<float>() + (size_t)row0 * c->ld, 0, true, is_bq(c->metric) ? 2 : 0);
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
        alloc_items(c, metric, dim, n, ids);
        if (n) {
            const uint8_t* base = reinterpret_cast<const uint8_t*>(vectors);
            const size_t stride = 4ull * dim;
            // binary-quantized metrics: the f32 vectors are quantized on the way (Writer::add_item -> UnalignedVector::from_slice)
            stage_rows_pipeline(c, n, c->dim, c->ld, [&](uint64_t i) { return base + i * stride; }, nullptr, 0, true, is_bq(metric) ? 1 : 0, dim);
            if (hdr0) CK(cudaMemcpyAsync(c->h0.p, hdr0, n * 4, cudaMemcpyHostToDevice, c->stream));
            else default_headers(c);
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
            bq_sign_rows_kernel<<<c->sm_count * 8, 256, 0, c->stream>>>(static_cast<const float*>(device_vectors), c->items.as<float>(), n, dim, c->dim, c->ld);
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
        // jobs per launch bounded by the shared-memory unit-prefix table of work_kernel
        const uint32_t max_jobs = 40000;
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
            int grid = (int)std::max<uint64_t>(1, std::min<uint64_t>(units, (uint64_t)c->sm_count * 3));
            launch_work(c, c->s_job.as<Job>(), (int)m, grid);
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
        P.items = c->items.as<float>(); P.ih0 = c->h0.as<float>(); P.ih1 = c->h1.as<float>();
        P.n = (uint32_t)c->n; P.d = c->dim; P.ld = ld; P.metric = c->metric;
        size_t ws_bytes = (size_t)WS_VECS * ld * 4;
        P.use_smem_ws = ws_bytes <= 200 * 1024;
        P.spec = (P.use_smem_ws && (size_t)WS_VECS_SPEC * ld * 4 <= 200 * 1024) ? 1 : 0;
        if (P.spec) ws_bytes = (size_t)WS_VECS_SPEC * ld * 4;
        P.scratch = reinterpret_cast<float*>(c->s_misc.as<uint8_t>() + 64);
        size_t smem = P.use_smem_ws ? ws_bytes : 0;
        const void* fn = nullptr;
        switch (c->metric) {
            case EUCLIDEAN: fn = P.use_smem_ws ? (const void*)&create_split_kernel<true, EUCLIDEAN> : (const void*)&create_split_kernel<false, EUCLIDEAN>; break;
            case COSINE: fn = P.use_smem_ws ? (const void*)&create_split_kernel<true, COSINE> : (const void*)&create_split_kernel<false, COSINE>; break;
            case DOT_PRODUCT: fn = P.use_smem_ws ? (const void*)&create_split_kernel<true, DOT_PRODUCT> : (const void*)&create_split_kernel<false, DOT_PRODUCT>; break;
            case MANHATTAN: fn = P.use_smem_ws ? (const void*)&create_split_kernel<true, MANHATTAN> : (const void*)&create_split_kernel<false, MANHATTAN>; break;
            case BQ_EUCLIDEAN: fn = P.use_smem_ws ? (const void*)&create_split_kernel<true, BQ_EUCLIDEAN> : (const void*)&create_split_kernel<false, BQ_EUCLIDEAN>; break;
            case BQ_COSINE: fn = P.use_smem_ws ? (const void*)&create_split_kernel<true, BQ_COSINE> : (const void*)&create_split_kernel<false, BQ_COSINE>; break;
            default: fn = P.use_smem_ws ? (const void*)&create_split_kernel<true, BQ_MANHATTAN> : (const void*)&create_split_kernel<false, BQ_MANHATTAN>; break;
        }
        if (smem > 48 * 1024) CK(cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
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
            { uint64_t warps = ((uint64_t)nc + 3) / 4; int g = (int)std::max<uint64_t>(1, std::min<uint64_t>((warps + 7) / 8, (uint64_t)c->sm_count * 16));
              norms_kernel<<<g, 256, 0, c->stream>>>(cand, nc, c->dim, ld, c->x_cnorm.as<float>(), nullptr); CK(cudaGetLastError()); }
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
                { uint64_t warps = ((uint64_t)m + 3) / 4; int g = (int)std::max<uint64_t>(1, std::min<uint64_t>((warps + 7) / 8, (uint64_t)c->sm_count * 16));
                  norms_kernel<<<g, 256, 0, c->stream>>>(Q.vecs, m, c->dim, ld, c->x_qnorm.as<float>(), nullptr); CK(cudaGetLastError()); }
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
                dim3 grid((nc + XCB - 1) / XCB, (m + XQB - 1) / XQB);
                if (c->metric == EUCLIDEAN)
                    xrerank_kernel<true><<<grid, XTHREADS, 0, c->stream>>>(c->items.as<float>(), c->h0.as<float>(), c->dim, ld, c->metric, Q.vecs, Q.h0, m,
                                                                          c->s_rows.as<uint32_t>(), nc, c->s_dists.as<float>());
                else
                    xrerank_kernel<false><<<grid, XTHREADS, 0, c->stream>>>(c->items.as<float>(), c->h0.as<float>(), c->dim, ld, c->metric, Q.vecs, Q.h0, m,
                                                                           c->s_rows.as<uint32_t>(), nc, c->s_dists.as<float>());
                CK(cudaGetLastError());
                topk_dense_kernel<<<m, TOPK_THREADS, 0, c->stream>>>(c->s_dists.as<float>(), c->s_rows.as<uint32_t>(), nc, k, c->metric,
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

template <bool FILTER, bool MULTI = false> void configure_walk_kernels() {
    static bool configured = false;
    if (configured) return;
    CK(cudaFuncSetAttribute(walk_kernel<FILTER, MULTI>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)((size_t)WALK_WARPS * WALK_SHEAP * 8)));
    CK(cudaFuncSetAttribute(walk1_kernel<FILTER, MULTI>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)walk1_smem<FILTER>(W1_MAX_LD)));
    configured = true;
}

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
        if (search_k == 0) search_k = count * F.n_roots;  // reader.rs:330
        // (filtered: saturating, so that search_k near 2^64 still leaves room for every filtered row the shortcut may take)
        const uint64_t sk_plus = filtered && search_k > UINT64_MAX - c->forest_max_desc ? UINT64_MAX : search_k + c->forest_max_desc;
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
                        forest_dots_kernel<<<dim3(gx, m), 256, (size_t)ld * 4, c->stream>>>(F, c->f_n_normals, c->items.as<float>(), c->dim, ld, Q.rows, Q.vecs, c->w_pre.as<float>());
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
                walk1<<<m_walk, W1_THREADS, w1smem, c->stream>>>(F, c->items.as<float>(), c->dim, ld, c->metric, m_walk, Q.rows, Q.vecs, Q.h0, d_pre, c->f_n_normals, w1debug,
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
                walk<<<(m_walk + WALK_WARPS - 1) / WALK_WARPS, WALK_WARPS * 32, walk_smem, c->stream>>>(F, c->items.as<float>(), c->dim, ld, c->metric, m_walk, Q.rows, Q.vecs, Q.h0,
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
        if (filtered) configure_walk_kernels<true>(); else configure_walk_kernels<false>();
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
        configure_walk_kernels<true, true>();
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
        // variant 1: work_kernel_shadow on the one job with every unit through the 8-bit pre-filter (scan_claim_planes), two CTAs
        // per SM as in the build; the stage counts of its last launch are what build_prefilter_stats reports afterwards
        const size_t stats_off = flush_l2 ? flush_bytes : 0;
        c->s_misc.ensure(stats_off + 32);
        unsigned long long* pstats = reinterpret_cast<unsigned long long*>(c->s_misc.as<uint8_t>() + stats_off);
        const size_t psmem = work_smem(c->ld, 1) + (size_t)PLANES_LIMBS * c->ld;
        if (planes && psmem > 48 * 1024) CK(cudaFuncSetAttribute(work_kernel_shadow, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)psmem));
        auto launch = [&] {
            if (!planes) { launch_work(c, c->s_job.as<Job>(), 1, grid); return; }
            work_kernel_shadow<<<c->sm_count * 2, WORK_THREADS, psmem, c->stream>>>(c->s_job.as<Job>(), 1, c->items.as<float>(),
                PlaneRows{c->pl_hi.as<int8_t>(), c->pl_lo.as<int8_t>(), c->pl_scale.as<float>()}, c->h0.as<float>(), c->dim, c->ld, c->metric, 0u, pstats);
            CK(cudaGetLastError());
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
    return guarded(c, [&] { out[0] = c->n_launches; out[1] = c->h2d_bytes; out[2] = c->d2h_bytes; out[3] = (c->fr_batches << 32) | (c->fr_fallbacks & 0xffffffffull); });
}

int32_t arroy_b200_prefilter_scores(arroy_ctx* c, uint32_t nq, const float* queries, const uint32_t* rows, uint64_t n_rows, int32_t engine, float* out_scores) {
    return guarded(c, [&] {
        require_staged(c); set_device(c);
        if (nq == 0 || n_rows == 0) return;
        if (!queries || !rows || !out_scores) throw ArgError("null argument");
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
        out[0] = c->items.p; out[1] = c->h0.p; out[2] = c->h1.p;
        if (out_ld) *out_ld = c->ld;
    });
}

}  // extern "C"

// several GPUs behind one handle (in-library NCCL broadcast of the item buffer)
#include "group.hpp"

// C++ host mirror of the reference's Writer / Reader (client of the C ABI above)
#include "host.hpp"
