// group.hpp — several GPUs of one node behind one handle (SURVEY.md §8b / §8e): the item buffer is uploaded once, on the
// first device, in chunks, and every chunk is handed to ncclBroadcast while the next one is still crossing PCIe; the trees
// are then sharded t mod n_dev and built by all devices at the same time, their nodes numbered exactly as a single-GPU
// build numbers them. Single process, one NCCL communicator per device (ncclCommInitAll). NCCL is bound at run time
// (dlopen): a host without it still loads the library, only arroy_b200_create_group fails.
#pragma once
#include <dlfcn.h>

#include <array>

namespace {

struct NcclApi {
    void* lib = nullptr;
    int (*CommInitAll)(void** comms, int ndev, const int* devlist) = nullptr;
    int (*CommDestroy)(void* comm) = nullptr;
    int (*Broadcast)(const void* send, void* recv, size_t count, int dtype, int root, void* comm, cudaStream_t stream) = nullptr;
    int (*GroupStart)() = nullptr;
    int (*GroupEnd)() = nullptr;
    const char* (*GetErrorString)(int) = nullptr;
    std::string err;
    bool load() {
        if (lib) return true;
        const char* names[] = {"libnccl.so.2", "libnccl.so"};
        for (const char* n : names) { lib = dlopen(n, RTLD_NOW | RTLD_GLOBAL); if (lib) break; }
        if (!lib) { err = std::string("NCCL not found (dlopen libnccl.so.2): ") + (dlerror() ? dlerror() : ""); return false; }
        auto sym = [&](const char* n) { void* p = dlsym(lib, n); if (!p) err = std::string("NCCL symbol missing: ") + n; return p; };
        CommInitAll = reinterpret_cast<decltype(CommInitAll)>(sym("ncclCommInitAll"));
        CommDestroy = reinterpret_cast<decltype(CommDestroy)>(sym("ncclCommDestroy"));
        Broadcast = reinterpret_cast<decltype(Broadcast)>(sym("ncclBroadcast"));
        GroupStart = reinterpret_cast<decltype(GroupStart)>(sym("ncclGroupStart"));
        GroupEnd = reinterpret_cast<decltype(GroupEnd)>(sym("ncclGroupEnd"));
        GetErrorString = reinterpret_cast<decltype(GetErrorString)>(sym("ncclGetErrorString"));
        return CommInitAll && CommDestroy && Broadcast && GroupStart && GroupEnd && GetErrorString;
    }
};
constexpr int NCCL_UINT8 = 1;   // ncclUint8 (nccl.h ncclDataType_t)

}  // namespace

struct arroy_group {
    std::vector<arroy_ctx*> ctx;
    std::vector<int> dev;
    std::vector<void*> comm;
    std::vector<Stream> bstream;   // broadcast streams, one per device
    NcclApi nccl;
    std::string err;
    std::mutex mu;
    double stage_ms[4] = {0, 0, 0, 0};   // last group_stage_items: [0] total wall, [1] waiting for the last broadcast after the last H2D

    ~arroy_group() {   // communicators, then the broadcast streams, then the member contexts
        for (void* cm : comm) if (cm) nccl.CommDestroy(cm);
        for (size_t r = 0; r < bstream.size(); ++r) { cudaSetDevice(dev[r]); bstream[r].reset(); }
        for (auto* c : ctx) delete c;
    }
};

namespace {

template <class F>
int32_t gguarded(arroy_group* g, F&& f) {
    if (!g) return ARROY_B200_ERR_INVALID;
    std::lock_guard<std::mutex> lk(g->mu);
    try { f(); return ARROY_B200_OK; }
    catch (const CudaError& e) { g->err = e.what(); cudaGetLastError(); return ARROY_B200_ERR_CUDA; }
    catch (const ArgError& e) { g->err = e.what(); return ARROY_B200_ERR_INVALID; }
    catch (const CapacityError& e) { g->err = e.what(); return ARROY_B200_ERR_CAPACITY; }
    catch (const Cancelled& e) { g->err = e.what(); return ARROY_B200_ERR_CANCELLED; }
    catch (const NotStaged& e) { g->err = e.what(); return ARROY_B200_ERR_NOT_STAGED; }
    catch (const std::exception& e) { g->err = std::string("internal error: ") + e.what(); return ARROY_B200_ERR_INTERNAL; }
}

void nccl_ck(arroy_group* g, int rc, const char* what) {
    if (rc != 0) throw CudaError(std::string(what) + ": " + g->nccl.GetErrorString(rc));
}

// one ncclBroadcast (root = device 0) of [ptr_r + off, + bytes) on every device, in place
void group_bcast(arroy_group* g, const std::vector<uint8_t*>& base, size_t off, size_t bytes) {
    if (bytes == 0 || g->ctx.size() < 2) return;
    nccl_ck(g, g->nccl.GroupStart(), "ncclGroupStart");
    for (size_t r = 0; r < g->ctx.size(); ++r)
        nccl_ck(g, g->nccl.Broadcast(base[r] + off, base[r] + off, bytes, NCCL_UINT8, 0, g->comm[r], g->bstream[r]), "ncclBroadcast");
    nccl_ck(g, g->nccl.GroupEnd(), "ncclGroupEnd");
}

}  // namespace

extern "C" {

int32_t arroy_b200_create_group(int32_t n_dev, const int32_t* devices, arroy_group** out) {
    if (!out) return ARROY_B200_ERR_INVALID;
    *out = nullptr;
    if (n_dev <= 0 || !devices) return ARROY_B200_ERR_INVALID;
    auto* g = new arroy_group();
    try {
        for (int i = 0; i < n_dev; ++i)
            for (int j = 0; j < i; ++j) if (devices[i] == devices[j]) throw ArgError("duplicate device in group");
        for (int i = 0; i < n_dev; ++i) {
            arroy_ctx* c = nullptr;
            if (arroy_b200_create(devices[i], &c) != ARROY_B200_OK) throw CudaError("arroy_b200_create failed for device " + std::to_string(devices[i]));
            g->ctx.push_back(c); g->dev.push_back(devices[i]);
            CK(cudaSetDevice(devices[i]));
            g->bstream.push_back(new_stream());
        }
        if (n_dev > 1) {
            if (!g->nccl.load()) throw CudaError(g->nccl.err);
            std::vector<void*> comm(n_dev, nullptr);   // kept only once all of them exist
            nccl_ck(g, g->nccl.CommInitAll(comm.data(), n_dev, g->dev.data()), "ncclCommInitAll");
            g->comm = std::move(comm);
        }
    } catch (const std::exception& e) {
        fprintf(stderr, "arroy_b200_create_group: %s\n", e.what());
        delete g;
        cudaGetLastError();
        return ARROY_B200_ERR_CUDA;
    }
    *out = g;
    return ARROY_B200_OK;
}

void arroy_b200_destroy_group(arroy_group* g) { delete g; }

const char* arroy_b200_group_last_error(arroy_group* g) { return g ? g->err.c_str() : "null group"; }
int32_t arroy_b200_group_size(arroy_group* g) { return g ? (int32_t)g->ctx.size() : 0; }
arroy_ctx* arroy_b200_group_ctx(arroy_group* g, int32_t rank) { return (g && rank >= 0 && (size_t)rank < g->ctx.size()) ? g->ctx[rank] : nullptr; }

int32_t arroy_b200_group_stage_items(arroy_group* g, int32_t metric, uint32_t dim, uint64_t n, const uint32_t* ids, const uint8_t* const* leaf_values) {
    return gguarded(g, [&] {
        if (n && (!ids || !leaf_values)) throw ArgError("null ids / leaf_values");
        auto t0 = std::chrono::steady_clock::now();
        const size_t R = g->ctx.size();
        auto ck = [&](size_t r, int32_t rc) { if (rc != ARROY_B200_OK) throw CudaError(std::string("device ") + std::to_string(g->dev[r]) + ": " + arroy_b200_last_error(g->ctx[r])); };
        for (size_t r = 0; r < R; ++r) ck(r, arroy_b200_stage_begin(g->ctx[r], metric, dim, n, ids));
        std::vector<uint8_t*> items(R), h0(R), h1(R);
        for (size_t r = 0; r < R; ++r) { items[r] = static_cast<uint8_t*>(g->ctx[r]->items.p); h0[r] = static_cast<uint8_t*>(g->ctx[r]->h0.p); h1[r] = static_cast<uint8_t*>(g->ctx[r]->h1.p); }
        const size_t row_bytes = g->ctx[0]->row_bytes;
        // chunks of ~256 MB: big enough for NCCL to run at line rate, small enough that the last broadcast (the only one that is
        // not hidden behind an H2D copy) is short
        const uint64_t chunk_rows = std::max<uint64_t>(1, (256ull << 20) / row_bytes);
        for (uint64_t a = 0; a < n; a += chunk_rows) {
            const uint64_t rows = std::min<uint64_t>(chunk_rows, n - a);
            ck(0, arroy_b200_stage_rows(g->ctx[0], a, rows, leaf_values + a));   // returns when the chunk is in device 0's memory
            group_bcast(g, items, (size_t)a * row_bytes, (size_t)rows * row_bytes);   // asynchronous on the broadcast streams
        }
        auto t1 = std::chrono::steady_clock::now();
        ck(0, arroy_b200_stage_end(g->ctx[0], 0));          // headers of device 0 from the leaf values
        group_bcast(g, h0, 0, (size_t)n * 4);
        group_bcast(g, h1, 0, (size_t)n * 4);
        for (size_t r = 0; r < R; ++r) { CK(cudaSetDevice(g->dev[r])); CK(cudaStreamSynchronize(g->bstream[r])); }
        for (size_t r = 1; r < R; ++r) ck(r, arroy_b200_stage_end(g->ctx[r], 1));
        auto t2 = std::chrono::steady_clock::now();
        g->stage_ms[0] = std::chrono::duration<double, std::milli>(t2 - t0).count();
        g->stage_ms[1] = std::chrono::duration<double, std::milli>(t2 - t1).count();
    });
}

int32_t arroy_b200_group_dot_preprocess(arroy_group* g, float* out_extra_dim, float* out_norm) {
    return gguarded(g, [&] {
        for (size_t r = 0; r < g->ctx.size(); ++r) {
            const int32_t rc = arroy_b200_dot_preprocess(g->ctx[r], r == 0 ? out_extra_dim : nullptr, r == 0 ? out_norm : nullptr);
            if (rc != ARROY_B200_OK) throw CudaError(std::string("device ") + std::to_string(g->dev[r]) + ": " + arroy_b200_last_error(g->ctx[r]));
        }
    });
}

int32_t arroy_b200_group_build_trees(arroy_group* g, uint32_t n_trees, const uint8_t (*tree_seeds)[32], const uint32_t* root_ids, uint32_t first_free_node_id,
                                     uint32_t split_after, arroy_b200_cancel_fn cancel, void* cancel_arg, arroy_b200_node_sink sink, void* sink_arg, uint64_t* out_n_nodes) {
    return gguarded(g, [&] {
        if (n_trees && (!tree_seeds || !root_ids)) throw ArgError("null seeds / root ids");
        const uint32_t R = (uint32_t)g->ctx.size();
        // tree t -> device t mod R (trees are independent given the items and their seed, src/writer.rs:795)
        std::vector<std::vector<uint32_t>> mine(R);
        for (uint32_t t = 0; t < n_trees; ++t) mine[t % R].push_back(t);
        std::vector<std::vector<std::array<uint8_t, 32>>> seeds(R);
        std::vector<std::vector<uint32_t>> counts(R);
        for (uint32_t r = 0; r < R; ++r) {
            seeds[r].resize(mine[r].size()); counts[r].assign(mine[r].size(), 0);
            for (size_t i = 0; i < mine[r].size(); ++i) memcpy(seeds[r][i].data(), tree_seeds[mine[r][i]], 32);
        }
        std::vector<int32_t> rc(R, ARROY_B200_OK);
        auto run = [&](auto&& fn) {
            std::vector<std::thread> th;
            for (uint32_t r = 1; r < R; ++r) th.emplace_back([&, r] { rc[r] = fn(r); });
            rc[0] = fn(0);
            for (auto& x : th) x.join();
            for (uint32_t r = 0; r < R; ++r) {
                if (rc[r] == ARROY_B200_ERR_CANCELLED) throw Cancelled("The corresponding build process has been cancelled");
                if (rc[r] != ARROY_B200_OK) throw CudaError(std::string("device ") + std::to_string(g->dev[r]) + ": " + arroy_b200_last_error(g->ctx[r]));
            }
        };
        run([&](uint32_t r) { return arroy_b200_build_trees_begin(g->ctx[r], (uint32_t)mine[r].size(), reinterpret_cast<const uint8_t(*)[32]>(seeds[r].data()), split_after, cancel, cancel_arg, counts[r].data()); });
        // ids: roots pre-allocated; the rest numbered as a 1-thread rayon pool would (last tree first, post-order inside a tree)
        std::vector<uint64_t> cnt(n_trees, 0), base(n_trees, 0);
        for (uint32_t r = 0; r < R; ++r) for (size_t i = 0; i < mine[r].size(); ++i) cnt[mine[r][i]] = counts[r][i];
        uint64_t counter = first_free_node_id, total = 0;
        for (uint32_t k = 0; k < n_trees; ++k) { const uint32_t t = n_trees - 1 - k; base[t] = counter; counter += cnt[t] - 1; total += cnt[t]; }
        if (counter > 0xffffffffull) throw CapacityError("node ids exceed u32 (Error::DatabaseFull)");
        if (out_n_nodes) *out_n_nodes = total;
        std::vector<std::vector<uint32_t>> roots(R);
        std::vector<std::vector<uint64_t>> bases(R);
        for (uint32_t r = 0; r < R; ++r) for (uint32_t t : mine[r]) { roots[r].push_back(root_ids[t]); bases[r].push_back(base[t]); }
        run([&](uint32_t r) { return arroy_b200_build_trees_emit(g->ctx[r], roots[r].data(), bases[r].data(), sink, sink_arg); });
    });
}

int32_t arroy_b200_group_stage_breakdown(arroy_group* g, double out[4]) {
    return gguarded(g, [&] { for (int i = 0; i < 4; ++i) out[i] = g->stage_ms[i]; });
}

}  // extern "C"
