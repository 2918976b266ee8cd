// host.hpp — C++ host mirror of arroy's Writer / ArroyBuilder / Reader / QueryBuilder above the
// device boundary (include/arroy_b200.h). See include/arroy_b200_host.h for the interface map.
// It is a *client* of the C ABI exactly as a fork of the Rust crate would be: every O(N*d) loop
// (item staging, preprocess, side() scans inside the forest build, re-rank) goes through
// arroy_b200_* calls; what stays here is the reference's host control flow:
//   key/value byte formats     src/key.rs:56-83, src/node.rs:218-282, src/metadata.rs:21-61, src/version.rs:39-49
//   Writer::build              src/writer.rs:487-629 (fresh-build path; see DESIGN.md for the incremental path)
//   target_n_trees             src/writer.rs:1358-1394
//   seed chain                 src/writer.rs:575, :795
//   Reader::open / nns_by_leaf src/reader.rs:138-176, :317-401 (the priority-queue tree walk, :338-374)
#pragma once
#include <array>
#include <chrono>
#include <cmath>
#include <functional>
#include <map>
#include <memory>
#include <queue>
#include <set>
#include <unordered_map>

#include "../../include/arroy_b200_host.h"

namespace arroy_host {

using Key8 = std::array<uint8_t, 8>;
enum : uint8_t { MODE_METADATA = 0, MODE_UPDATED = 1, MODE_TREE = 2, MODE_ITEM = 3 };  // src/node_id.rs:11-21

inline Key8 make_key(uint16_t index, uint8_t mode, uint32_t item) {  // src/key.rs:56-68
    return Key8{(uint8_t)(index >> 8), (uint8_t)index, mode, (uint8_t)(item >> 24), (uint8_t)(item >> 16), (uint8_t)(item >> 8), (uint8_t)item, 0};
}
inline uint32_t key_item(const Key8& k) { return ((uint32_t)k[3] << 24) | ((uint32_t)k[4] << 16) | ((uint32_t)k[5] << 8) | k[6]; }

inline const char* metric_name(int m) {
    switch (m) {
        case 0: return "euclidean";
        case 1: return "cosine";
        case 2: return "dot-product";
        default: return "manhattan";
    }
}
inline int header_floats(int m) { return m == 2 ? 2 : 1; }

struct HostError : std::runtime_error {
    int code;
    HostError(int c, const std::string& m) : std::runtime_error(m), code(c) {}
};

inline std::string& tls_error() { static thread_local std::string e; return e; }

// ---- exact host arithmetic for the tree walk (one D::margin per popped split node) --------------
// Same summation orders as the device code (exact.cuh), written as portable scalar C++; compiled
// with -ffp-contract=off so only the explicit fmaf fuses.
inline float host_dot(const float* a, const float* b, size_t n) {
    if (n >= 32) {
        size_t m = n - (n % 32);
        float acc[32];
        for (int l = 0; l < 32; ++l) acc[l] = 0.f;
        for (size_t i = 0; i < m; i += 32)
            for (int l = 0; l < 32; ++l) acc[l] = __builtin_fmaf(a[i + l], b[i + l], acc[l]);
        float h[4];
        for (int k = 0; k < 4; ++k) {
            const float* x = acc + 8 * k;
            float x0 = x[4] + x[0], x1 = x[5] + x[1], x2 = x[6] + x[2], x3 = x[7] + x[3];
            h[k] = (x0 + x2) + (x1 + x3);
        }
        float r = ((h[0] + h[1]) + h[2]) + h[3];
        for (size_t i = m; i < n; ++i) r += a[i] * b[i];
        return r;
    }
    if (n >= 16) {
        size_t m = n - (n % 16);
        float acc[16];
        for (int l = 0; l < 16; ++l) acc[l] = 0.f;
        for (size_t i = 0; i < m; i += 16)
            for (int l = 0; l < 16; ++l) acc[l] = a[i + l] * b[i + l] + acc[l];
        float h[4];
        for (int k = 0; k < 4; ++k) { const float* x = acc + 4 * k; h[k] = (x[0] + x[2]) + (x[1] + x[3]); }
        float r = ((h[0] + h[1]) + h[2]) + h[3];
        for (size_t i = m; i < n; ++i) r += a[i] * b[i];
        return r;
    }
    float s = 0.0f;
    for (size_t i = 0; i < n; ++i) s += a[i] * b[i];
    return s;
}
inline float host_margin(int metric, const float* nv, float nh0, const float* qv, float qh0, size_t d) {
    float dot = host_dot(nv, qv, d);
    if (metric == 1) return dot;                    // cosine.rs:87-89
    if (metric == 2) return dot + nh0 * qh0;        // dot_product.rs:115-117
    return nh0 + dot;                               // euclidean.rs:79-81, manhattan.rs:82-84
}
inline float f32_min(float a, float b) { if (a != a) return b; if (b != b) return a; return a < b ? a : b; }

inline uint64_t target_n_trees(int64_t n_trees_opt, uint64_t dimensions, uint64_t n_items, uint64_t n_roots) {  // writer.rs:1358-1394
    if (n_trees_opt >= 0) return (uint64_t)n_trees_opt;
    double nb_vec = (double)n_items, nb_trees;
    if (nb_vec < 10000.0) nb_trees = std::pow(2.0, std::log2(nb_vec) - 6.0);
    else nb_trees = std::pow(2.0, std::log10(nb_vec) + std::log10((double)dimensions) + std::pow(768.0 / (double)dimensions, 4.0));
    double c = std::ceil(nb_trees);
    uint64_t n = (!(c == c) || c <= 0.0) ? 0 : (c >= 18446744073709551615.0 ? UINT64_MAX : (uint64_t)c);
    if (n_roots > n) {
        uint64_t rm = n_roots - n;
        if ((double)rm / (double)n < 0.20) n = n_roots;
    }
    return n;
}

// RoaringBitmap::deserialize_from for the no-run-container portable format
inline void roaring_deserialize(const uint8_t* b, size_t len, std::vector<uint32_t>& out) {
    auto r32 = [&](size_t o) { uint32_t v; memcpy(&v, b + o, 4); return v; };
    auto r16 = [&](size_t o) { uint16_t v; memcpy(&v, b + o, 2); return v; };
    if (len < 8 || r32(0) != 12346u) throw HostError(ARROY_ERR_PANIC, "unsupported roaring cookie");
    uint32_t n = r32(4);
    size_t off = 8 + 8 * (size_t)n;
    for (uint32_t i = 0; i < n; ++i) {
        uint32_t key = r16(8 + 4 * i), card = (uint32_t)r16(8 + 4 * i + 2) + 1;
        if (card > 4096) {
            for (uint32_t w = 0; w < 8192; ++w) { uint8_t byte = b[off + w]; while (byte) { int bit = __builtin_ctz(byte); out.push_back((key << 16) | (w * 8 + bit)); byte &= byte - 1; } }
            off += 8192;
        } else {
            for (uint32_t k = 0; k < card; ++k) out.push_back((key << 16) | r16(off + 2 * k));
            off += 2 * (size_t)card;
        }
    }
}

}  // namespace arroy_host

struct arroy_env {
    std::map<arroy_host::Key8, std::string> kv;
    std::mutex mu;
    uint64_t generation = 0;                  // bumped on every write
    std::map<uint16_t, uint64_t> index_gen;   // per index: bumped by every committed write to that index. A Reader remembers the
                                              // value it was opened at (the table has no RoTxn snapshots: a reader that outlives a
                                              // write to its index fails with NeedBuild instead of mixing two states)
    void touch(uint16_t index) { generation++; index_gen[index]++; }
    uint64_t gen_of(uint16_t index) const { auto it = index_gen.find(index); return it == index_gen.end() ? 0 : it->second; }
};
struct arroy_rng {
    ab::Rng r;
};
struct arroy_writer {
    arroy_env* env;
    uint16_t index;
    uint32_t dims;
    int metric;
    double timings[8] = {0, 0, 0, 0, 0, 0, 0, 0};
};
struct arroy_reader {
    arroy_env* env;
    arroy_ctx* ctx;
    uint16_t index;
    uint32_t dims;
    int metric;
    std::vector<uint32_t> roots;
    std::vector<uint32_t> items;   // ascending ids (metadata.items)
    // decoded tree nodes, indexed by node id
    struct Node { uint8_t kind = 0; bool has_normal = false; uint32_t left = 0, right = 0; uint32_t normal_off = 0; float h0 = 0, h1 = 0; uint32_t desc_off = 0, desc_len = 0; };
    std::vector<Node> nodes;
    std::vector<float> normals;     // d floats per split node with a normal
    std::vector<uint32_t> desc;     // concatenated descendant id lists
    std::vector<float> hdr0, hdr1;  // item headers (query by item)
    // The device context is shared by every Reader / Writer of the Env, so "I staged my items" is not a fact that stays
    // true: the epochs of the context's resident items / forest this reader produced (arroy_b200_epochs); anything else
    // there belongs to somebody else and is replaced before use.
    uint64_t stage_epoch = 0, forest_epoch = 0;
    uint64_t gen_at_open = 0;
};

namespace arroy_host {

using clk = std::chrono::steady_clock;
inline double ms_since(clk::time_point t0) { return std::chrono::duration<double, std::milli>(clk::now() - t0).count(); }

template <class F>
int32_t hguard(F&& f) {
    try { f(); return 0; }
    catch (const HostError& e) { tls_error() = e.what(); return e.code; }
    catch (const std::exception& e) { tls_error() = std::string("Unexpected panic in: ") + e.what(); return ARROY_ERR_PANIC; }
    catch (...) { tls_error() = "Unexpected panic in: unknown"; return ARROY_ERR_PANIC; }
}
inline void dev_ck(arroy_ctx* ctx, int32_t rc) {
    if (rc == ARROY_B200_OK) return;
    std::string msg = arroy_b200_last_error(ctx);
    if (rc == ARROY_B200_ERR_CANCELLED) throw HostError(ARROY_ERR_BUILD_CANCELLED, "The corresponding build process has been cancelled");
    throw HostError(rc, msg);
}

inline std::string encode_leaf(int metric, const float* v, uint32_t d, float h0, float h1) {  // src/node.rs:224-228
    std::string s;
    s.resize(1 + 4 * header_floats(metric) + 4ull * d);
    s[0] = 0;
    memcpy(&s[1], &h0, 4);
    if (header_floats(metric) == 2) memcpy(&s[5], &h1, 4);
    memcpy(&s[1 + 4 * header_floats(metric)], v, 4ull * d);
    return s;
}

// D::new_header (cosine.rs:39-41: norm; others zero). The cosine norm is left 0 here and filled in
// by the device at build time? No: the stored header must be right at add_item time, so compute it
// with the exact host dot.
inline void new_header(int metric, const float* v, uint32_t d, float& h0, float& h1) {
    h0 = 0.f; h1 = 0.f;
    if (metric == 1) h0 = std::sqrt(host_dot(v, v, d));
}

inline void put_item(arroy_writer* w, uint32_t item, const float* v) {  // Writer::add_item — src/writer.rs:380-395
    float h0, h1;
    new_header(w->metric, v, w->dims, h0, h1);
    w->env->kv[make_key(w->index, MODE_ITEM, item)] = encode_leaf(w->metric, v, w->dims, h0, h1);
    w->env->kv[make_key(w->index, MODE_UPDATED, item)] = std::string();
    w->env->touch(w->index);
}

struct ItemView { std::vector<uint32_t> ids; std::vector<const uint8_t*> ptrs; std::vector<size_t> sizes; };
inline ItemView collect_items(arroy_env* env, uint16_t index) {
    ItemView v;
    auto it = env->kv.lower_bound(make_key(index, MODE_ITEM, 0));
    for (; it != env->kv.end() && it->first[0] == (uint8_t)(index >> 8) && it->first[1] == (uint8_t)index && it->first[2] == MODE_ITEM; ++it) {
        v.ids.push_back(key_item(it->first));
        v.ptrs.push_back(reinterpret_cast<const uint8_t*>(it->second.data()));
        v.sizes.push_back(it->second.size());
    }
    return v;
}
inline void erase_mode(arroy_env* env, uint16_t index, uint8_t mode) {
    auto b = env->kv.lower_bound(make_key(index, mode, 0));
    auto e = b;
    while (e != env->kv.end() && e->first[0] == (uint8_t)(index >> 8) && e->first[1] == (uint8_t)index && e->first[2] == mode) ++e;
    env->kv.erase(b, e);
}
inline std::string encode_metadata(int metric, uint32_t dims, const std::vector<uint32_t>& items, const std::vector<uint32_t>& roots) {  // metadata.rs:21-44
    std::vector<uint8_t> bm;
    ::roaring_serialize(items.data(), items.size(), bm);
    std::string out = metric_name(metric);
    out.push_back('\0');
    uint8_t be[4] = {(uint8_t)(dims >> 24), (uint8_t)(dims >> 16), (uint8_t)(dims >> 8), (uint8_t)dims};
    out.append(reinterpret_cast<char*>(be), 4);
    uint32_t sz = (uint32_t)bm.size();
    uint8_t bs[4] = {(uint8_t)(sz >> 24), (uint8_t)(sz >> 16), (uint8_t)(sz >> 8), (uint8_t)sz};
    out.append(reinterpret_cast<char*>(bs), 4);
    out.append(reinterpret_cast<char*>(bm.data()), bm.size());
    out.append(reinterpret_cast<const char*>(roots.data()), 4 * roots.size());  // native endian (ItemIds::from_slice)
    return out;
}
struct Metadata { std::string distance; uint32_t dims = 0; std::vector<uint32_t> items, roots; };
inline bool read_metadata(arroy_env* env, uint16_t index, Metadata& m) {
    auto it = env->kv.find(make_key(index, MODE_METADATA, 0));
    if (it == env->kv.end()) return false;
    const std::string& s = it->second;
    size_t z = s.find('\0');
    m.distance = s.substr(0, z);
    const uint8_t* b = reinterpret_cast<const uint8_t*>(s.data()) + z + 1;
    m.dims = ((uint32_t)b[0] << 24) | ((uint32_t)b[1] << 16) | ((uint32_t)b[2] << 8) | b[3];
    uint32_t sz = ((uint32_t)b[4] << 24) | ((uint32_t)b[5] << 16) | ((uint32_t)b[6] << 8) | b[7];
    roaring_deserialize(b + 8, sz, m.items);
    size_t rest = s.size() - (z + 1 + 8 + sz);
    m.roots.resize(rest / 4);
    memcpy(m.roots.data(), b + 8 + sz, rest);
    return true;
}
inline void write_version(arroy_env* env, uint16_t index) {  // version.rs:39-49, Version::current() = 0.7.0
    const uint8_t v[12] = {0, 0, 0, 0, 0, 0, 0, 7, 0, 0, 0, 0};
    env->kv[make_key(index, MODE_METADATA, 1)] = std::string(reinterpret_cast<const char*>(v), 12);
}


// ---- pieces of the incremental build (src/writer.rs:632-653, :846-889, :978-1160, :1398-1459) ----------

// std HashMap<u32, _, BuildNoHashHasher> as nohash::IntMap gives it to the reference: the order in
// which `descendants` is iterated decides which seed and which node ids every rebuilt subtree gets
// (writer.rs:778-795), so the insertion / growth / iteration order of hashbrown's SwissTable is
// restated here (identity hash: slot = first free bucket at or after id & mask; capacity 3, 7, then
// buckets / 8 * 7; growth re-inserts in iteration order; iteration = ascending bucket).
struct IntMapOrder {
    std::vector<int64_t> keys;
    std::vector<std::vector<uint32_t>> vals;
    size_t items = 0;
    static size_t capacity_of(size_t buckets) { return buckets < 8 ? buckets - 1 : buckets / 8 * 7; }
    size_t find(uint32_t k) const {
        if (keys.empty()) return SIZE_MAX;
        size_t mask = keys.size() - 1, pos = k & mask;
        for (size_t i = 0; i < keys.size(); ++i) { size_t b = (pos + i) & mask; if (keys[b] == (int64_t)k) return b; if (keys[b] < 0) return SIZE_MAX; }
        return SIZE_MAX;
    }
    void raw_insert(uint32_t k, std::vector<uint32_t>&& v) {
        size_t mask = keys.size() - 1, pos = k & mask;
        for (size_t i = 0;; ++i) { size_t b = (pos + i) & mask; if (keys[b] < 0) { keys[b] = k; vals[b] = std::move(v); return; } }
    }
    std::vector<uint32_t>& entry(uint32_t k) {
        size_t f = find(k);
        if (f != SIZE_MAX) return vals[f];
        if (keys.empty() || items == capacity_of(keys.size())) {
            size_t cap = std::max(items + 1, keys.empty() ? (size_t)0 : capacity_of(keys.size()) + 1);
            size_t nb = cap < 4 ? 4 : (cap < 8 ? 8 : 1);
            if (nb == 1) { size_t adj = cap * 8 / 7; while (nb < adj) nb <<= 1; }
            std::vector<int64_t> ok = std::move(keys);
            std::vector<std::vector<uint32_t>> ov = std::move(vals);
            keys.assign(nb, -1); vals.assign(nb, {});
            for (size_t b = 0; b < ok.size(); ++b) if (ok[b] >= 0) raw_insert((uint32_t)ok[b], std::move(ov[b]));
        }
        raw_insert(k, {});
        ++items;
        return vals[find(k)];
    }
    void merge_from(IntMapOrder& src) {   // for (k, v) in src { self.entry(k).or_default().extend(v) }; src is consumed
        for (size_t b = 0; b < src.keys.size(); ++b) {
            if (src.keys[b] < 0) continue;
            std::vector<uint32_t>& dv = entry((uint32_t)src.keys[b]);
            if (dv.empty()) { dv = std::move(src.vals[b]); continue; }   // the usual case: the two maps hold different nodes
            std::vector<uint32_t> merged;
            std::set_union(dv.begin(), dv.end(), src.vals[b].begin(), src.vals[b].end(), std::back_inserter(merged));
            dv.swap(merged);
        }
    }
};

struct HNode {  // a decoded tree node (src/node.rs:246-282); the normal stays as raw bytes [header | vector]
    uint8_t kind = 0;
    uint32_t left = 0, right = 0;
    std::string normal;             // empty = "normal: none"
    std::vector<uint32_t> desc;
};
inline HNode decode_tree_node(const std::string& v) {
    HNode n;
    const uint8_t* b = reinterpret_cast<const uint8_t*>(v.data());
    if (b[0] == 1) { n.kind = 1; roaring_deserialize(b + 1, v.size() - 1, n.desc); }
    else if (b[0] == 2) {
        n.kind = 2;
        n.left = ((uint32_t)b[1] << 24) | ((uint32_t)b[2] << 16) | ((uint32_t)b[3] << 8) | b[4];
        n.right = ((uint32_t)b[5] << 24) | ((uint32_t)b[6] << 16) | ((uint32_t)b[7] << 8) | b[8];
        n.normal.assign(v.data() + 9, v.size() - 9);
    } else throw HostError(ARROY_ERR_PANIC, "Did not recognize node tag type");
    return n;
}
inline std::string encode_tree_node(const HNode& n) {   // NodeCodec::bytes_encode — src/node.rs:229-241
    std::string out;
    if (n.kind == 1) {
        std::vector<uint8_t> buf;
        buf.push_back(1);
        ::roaring_serialize(n.desc.data(), n.desc.size(), buf);
        out.assign(reinterpret_cast<char*>(buf.data()), buf.size());
    } else {
        out.push_back(2);
        for (int k = 3; k >= 0; --k) out.push_back((char)(n.left >> (8 * k)));
        for (int k = 3; k >= 0; --k) out.push_back((char)(n.right >> (8 * k)));
        out += n.normal;
    }
    return out;
}

struct NodeIdAlloc {  // ConcurrentNodeIds — src/parallel.rs:207-255
    std::vector<uint32_t> available;
    size_t select = 0;
    bool look = false;
    uint64_t current = 0;
    explicit NodeIdAlloc(const std::map<uint32_t, HNode>& used) {
        uint32_t last_id = used.empty() ? 0 : used.rbegin()->first + 1;
        for (uint32_t i = 0; i < last_id; ++i) if (!used.count(i)) available.push_back(i);
        current = last_id;
        look = !available.empty();
    }
    uint32_t next() {
        if (look) { if (select < available.size()) return available[select++]; look = false; }
        if (current > 0xffffffffull) throw HostError(ARROY_ERR_DATABASE_FULL, "Database full. Arroy cannot generate enough internal IDs for your items");
        return (uint32_t)current++;
    }
};

struct IncCtx {
    arroy_env* env; arroy_ctx* ctx; uint16_t index; int metric; uint32_t d; size_t K;
    std::map<uint32_t, HNode> tree;                 // the index' tree nodes as this build sees them
    // the build's writes to the tree keys: node id -> (present, NodeCodec bytes). Applied to env->kv only when the whole build
    // has succeeded — the reference works inside a RwTxn that is dropped on error (writer.rs:487-629)
    std::map<uint32_t, std::pair<bool, std::string>> pending;
    const std::vector<uint32_t>* item_ids;          // ascending ids of the staged items (row = rank)
    // O(1) lookups for the routing loops (millions of them per update): node id -> decoded node (std::map nodes do
    // not move), item id -> row when the ids are small enough for a dense table
    std::vector<const HNode*> by_id;
    std::vector<uint32_t> dense_row;
    void index_lookups() {
        by_id.clear();
        if (!tree.empty()) { by_id.assign((size_t)tree.rbegin()->first + 1, nullptr); for (auto& kv : tree) by_id[kv.first] = &kv.second; }
        dense_row.clear();
        if (!item_ids->empty() && item_ids->back() < (1u << 26)) {
            dense_row.assign((size_t)item_ids->back() + 1, 0xffffffffu);
            for (size_t i = 0; i < item_ids->size(); ++i) dense_row[(*item_ids)[i]] = (uint32_t)i;
        }
    }
    const HNode& node(uint32_t id) const { if (id < by_id.size() && by_id[id]) return *by_id[id]; return tree.at(id); }
    void put(uint32_t id, HNode&& n) {
        pending[id] = {true, encode_tree_node(n)};
        HNode& slot = tree[id];
        slot = std::move(n);
        if (id >= by_id.size()) by_id.resize((size_t)id + 1, nullptr);
        by_id[id] = &slot;
    }
    void erase(uint32_t id) { pending[id] = {false, std::string()}; tree.erase(id); if (id < by_id.size()) by_id[id] = nullptr; }
    void commit() {
        for (auto& kv : pending) {
            if (kv.second.first) env->kv[make_key(index, MODE_TREE, kv.first)] = std::move(kv.second.second);
            else env->kv.erase(make_key(index, MODE_TREE, kv.first));
        }
        pending.clear();
    }
    uint32_t row_of(uint32_t id) const {
        if (id < dense_row.size() && dense_row[id] != 0xffffffffu) return dense_row[id];
        return (uint32_t)(std::lower_bound(item_ids->begin(), item_ids->end(), id) - item_ids->begin());
    }
};

inline void inc_delete_tree(IncCtx& C, uint32_t node) {   // writer.rs:1263-1277
    auto it = C.tree.find(node);
    if (it == C.tree.end()) return;
    if (it->second.kind == 2) { uint32_t l = it->second.left, r = it->second.right; inc_delete_tree(C, l); inc_delete_tree(C, r); }
    C.erase(node);
}

struct TmpOps { std::vector<std::pair<uint32_t, HNode>> puts; std::set<uint32_t> deleted; };   // TmpNodes put / remove

struct IdSet {  // membership test for the updated item ids: dense marker table when ids are small, else a set
    std::vector<uint8_t> mark;
    std::set<uint32_t> sparse;
    bool dense = false;
    explicit IdSet(const std::vector<uint32_t>& ids) {
        uint32_t mx = 0;
        for (uint32_t i : ids) mx = std::max(mx, i);
        if (!ids.empty() && mx < (1u << 28)) { dense = true; mark.assign((size_t)mx + 1, 0); for (uint32_t i : ids) mark[i] = 1; }
        else sparse.insert(ids.begin(), ids.end());
    }
    bool count(uint32_t id) const { return dense ? (id < mark.size() && mark[id]) : sparse.count(id) > 0; }
};

// delete_items_in_file — writer.rs:1021-1114. second.first = "Some(items)"
inline std::pair<uint32_t, std::pair<bool, std::vector<uint32_t>>> inc_delete_items(IncCtx& C, uint32_t current, TmpOps& tmp, const IdSet& to_delete) {
    const HNode& nd = C.node(current);
    if (nd.kind == 1) {
        std::vector<uint32_t> nw;
        for (uint32_t id : nd.desc) if (!to_delete.count(id)) nw.push_back(id);
        if (nw.size() != nd.desc.size()) { HNode t; t.kind = 1; t.desc = nw; tmp.puts.push_back({current, std::move(t)}); }
        return {current, {true, nw}};
    }
    const uint32_t left = nd.left, right = nd.right;
    auto L = inc_delete_items(C, left, tmp, to_delete);
    auto R = inc_delete_items(C, right, tmp, to_delete);
    const uint32_t nl = L.first, nr = R.first;
    auto put_split = [&]() { if (nl != left || nr != right) { HNode t = C.tree.at(current); t.left = nl; t.right = nr; tmp.puts.push_back({current, std::move(t)}); } };
    if (L.second.first && L.second.second.empty()) { tmp.deleted.insert(nl); tmp.deleted.insert(current); return {nr, R.second}; }
    if (R.second.first && R.second.second.empty()) { tmp.deleted.insert(nr); tmp.deleted.insert(current); return {nl, L.second}; }
    if (L.second.first && R.second.first) {
        if (L.second.second.size() + R.second.second.size() <= C.K) {
            std::vector<uint32_t> all;
            std::set_union(L.second.second.begin(), L.second.second.end(), R.second.second.begin(), R.second.second.end(), std::back_inserter(all));
            tmp.deleted.insert(nl); tmp.deleted.insert(nr);
            HNode t; t.kind = 1; t.desc = all;
            tmp.puts.push_back({current, std::move(t)});
            return {current, {true, all}};
        }
        put_split();
        return {current, {false, {}}};
    }
    put_split();
    return {current, {false, {}}};
}

// insert_items_in_descendants_from_frozen_reader — writer.rs:1398-1459; the side() loop runs on the device
inline void inc_route(IncCtx& C, ab::Rng& rng, uint32_t node, const std::vector<uint32_t>& to_insert, IntMapOrder& out) {
    const HNode& nd = C.tree.at(node);
    if (nd.kind == 1) {
        std::vector<uint32_t> merged;
        std::set_union(nd.desc.begin(), nd.desc.end(), to_insert.begin(), to_insert.end(), std::back_inserter(merged));
        out.entry(node) = merged;
        return;
    }
    std::vector<uint32_t> left, right;
    if (nd.normal.empty()) {   // randomly_split_children: Side::random = rng.gen::<bool>() ? Left : Right
        for (uint32_t id : to_insert) { if ((int32_t)rng.next_u32() < 0) left.push_back(id); else right.push_back(id); }
    } else {
        const int hf = header_floats(C.metric);
        float h0 = 0.f, h1 = 0.f;
        memcpy(&h0, nd.normal.data(), 4);
        if (hf == 2) memcpy(&h1, nd.normal.data() + 4, 4);
        std::vector<float> nv(C.d);
        memcpy(nv.data(), nd.normal.data() + 4 * hf, 4ull * C.d);
        std::vector<uint32_t> rows(to_insert.size());
        for (size_t i = 0; i < rows.size(); ++i) rows[i] = C.row_of(to_insert[i]);
        std::vector<uint8_t> side(rows.size());
        dev_ck(C.ctx, arroy_b200_side_batch(C.ctx, nv.data(), h0, h1, rows.data(), rows.size(), side.data(), nullptr));
        for (size_t i = 0; i < rows.size(); ++i) { if (side[i]) right.push_back(to_insert[i]); else left.push_back(to_insert[i]); }
    }
    const uint32_t l = nd.left, r = nd.right;
    if (!left.empty()) inc_route(C, rng, l, left, out);
    if (!right.empty()) inc_route(C, rng, r, right, out);
}

// Level-batched version of the same routing for many roots at once: one arroy_b200_side_multi launch
// per tree depth. The per-root results are then replayed depth-first so that the insertion order
// into the IntMap (which the node ids depend on) is the reference's. Roots whose paths meet a
// "normal: none" node keep the depth-first routine above (its random sides consume the root's rng
// in depth-first order). Returns, per root, whether it was handled here.
struct Routed { std::vector<uint32_t> left, right; };
inline std::vector<char> inc_route_batched(IncCtx& C, const std::vector<uint32_t>& roots, const std::vector<uint32_t>& to_insert,
                                          std::unordered_map<uint32_t, Routed>& routed, std::unordered_map<uint32_t, std::vector<uint32_t>>& leaf_ins) {
    struct Front { uint32_t root_idx, node; std::vector<uint32_t> ids; };
    std::vector<char> ok(roots.size(), 1);
    std::vector<Front> front;
    for (uint32_t r = 0; r < roots.size(); ++r) front.push_back({r, roots[r], to_insert});
    const int hf = header_floats(C.metric);
    while (!front.empty()) {
        std::vector<float> normals, h0;
        std::vector<uint32_t> rows;
        std::vector<uint64_t> off(1, 0);
        std::vector<size_t> job_front;
        for (size_t i = 0; i < front.size(); ++i) {
            Front& f = front[i];
            if (!ok[f.root_idx]) continue;
            const HNode& nd = C.node(f.node);
            if (nd.kind == 1) { leaf_ins[f.node] = std::move(f.ids); continue; }
            if (nd.normal.empty()) { ok[f.root_idx] = 0; continue; }
            float hh = 0.f;
            memcpy(&hh, nd.normal.data(), 4);
            h0.push_back(hh);
            size_t o = normals.size();
            normals.resize(o + C.d);
            memcpy(normals.data() + o, nd.normal.data() + 4 * hf, 4ull * C.d);
            for (uint32_t id : f.ids) rows.push_back(C.row_of(id));
            off.push_back(rows.size());
            job_front.push_back(i);
        }
        std::vector<Front> next;
        if (!job_front.empty()) {
            std::vector<uint8_t> side(rows.size());
            dev_ck(C.ctx, arroy_b200_side_multi(C.ctx, (uint32_t)job_front.size(), normals.data(), h0.data(), nullptr, rows.data(), off.data(), side.data()));
            for (size_t j = 0; j < job_front.size(); ++j) {
                Front& f = front[job_front[j]];
                const HNode& nd = C.node(f.node);
                Routed rt;
                for (size_t i = 0; i < f.ids.size(); ++i) { if (side[off[j] + i]) rt.right.push_back(f.ids[i]); else rt.left.push_back(f.ids[i]); }
                if (!rt.left.empty()) next.push_back({f.root_idx, nd.left, rt.left});
                if (!rt.right.empty()) next.push_back({f.root_idx, nd.right, rt.right});   // (copies: `routed` keeps its own for the replay)
                routed[f.node] = std::move(rt);
            }
        }
        front.swap(next);
    }
    return ok;
}
inline void inc_replay(IncCtx& C, uint32_t node, const std::unordered_map<uint32_t, Routed>& routed, std::unordered_map<uint32_t, std::vector<uint32_t>>& leaf_ins, IntMapOrder& out) {
    const HNode& nd = C.node(node);
    if (nd.kind == 1) {
        const std::vector<uint32_t>& ins = leaf_ins.at(node);
        std::vector<uint32_t> merged;
        std::set_union(nd.desc.begin(), nd.desc.end(), ins.begin(), ins.end(), std::back_inserter(merged));
        out.entry(node) = merged;
        return;
    }
    const Routed& rt = routed.at(node);
    if (!rt.left.empty()) inc_replay(C, nd.left, routed, leaf_ins, out);
    if (!rt.right.empty()) inc_replay(C, nd.right, routed, leaf_ins, out);
}

inline ab::Rng rng_seed_from_u64(uint64_t state) {   // rand_core 0.6 SeedableRng::seed_from_u64
    const uint64_t MUL = 6364136223846793005ull, INC = 11634580027462260723ull;
    uint32_t key[8];
    for (int c = 0; c < 8; ++c) {
        state = state * MUL + INC;
        uint32_t xs = (uint32_t)(((state >> 18) ^ state) >> 27), rot = (uint32_t)(state >> 59);
        key[c] = (xs >> rot) | (xs << ((32 - rot) & 31));
    }
    ab::Rng r;
    r.init(key, 0);
    return r;
}

// The library calls the sink concurrently from its encoder threads; nodes are parked in shards and
// moved into the ordered table once the build is over (TmpNodes files -> LMDB, writer.rs:597-607).
struct SinkArg {
    static constexpr int SHARDS = 64;
    std::mutex mu[SHARDS];
    std::vector<std::pair<uint32_t, std::string>> nodes[SHARDS];
    std::atomic<uint64_t> bytes{0};
};
inline int32_t tree_sink(void* arg, uint32_t node_id, const uint8_t* bytes, uint64_t len) {
    auto* a = static_cast<SinkArg*>(arg);
    const int sh = (int)(std::hash<std::thread::id>()(std::this_thread::get_id()) % SinkArg::SHARDS);
    std::string v(reinterpret_cast<const char*>(bytes), len);
    std::lock_guard<std::mutex> lk(a->mu[sh]);
    a->nodes[sh].emplace_back(node_id, std::move(v));
    a->bytes += len;
    return 0;
}

// ---- memory-limited builds (ArroyBuilder::available_memory) ---------------------------------------------------------
// The reference indexes a large descendant in pieces when the items do not fit in the memory it was given
// (incremental_index_large_descendant, writer.rs:660-739): a random sample that fits is turned into a tree, the rest is routed
// through that tree chunk by chunk (insert_items_in_descendants_from_tmpfile, :1463-1531), and every leaf that ended up larger
// than split_after becomes a new task with its own forked rng (insert_descendants_in_file_and_spawn_tasks, :744-844). The item
// matrix of this library is resident in HBM either way; what is reproduced is the SHAPE of the forest that such a build
// produces — the same draws from the same StdRng streams, the same node ids — so that an index built here with a given
// available_memory equals the reference's. One subtree per device call: arroy_b200_build_subtrees_begin_at continues the
// task's rng at the word position the host reached and hands back the position the tree ended at.
struct LmTask { ab::Rng rng; uint32_t id; std::vector<uint32_t> items; };

inline ab::Rng rng_fork(ab::Rng& r) {   // StdRng::from_seed(rng.gen())
    uint8_t s[32];
    r.gen_seed(s);
    uint32_t key[8];
    for (int i = 0; i < 8; ++i) key[i] = (uint32_t)s[4 * i] | ((uint32_t)s[4 * i + 1] << 8) | ((uint32_t)s[4 * i + 2] << 16) | ((uint32_t)s[4 * i + 3] << 24);
    ab::Rng out;
    out.init(key, 0);
    return out;
}
inline uint64_t rng_below_u64(ab::Rng& r, uint64_t high) {   // rng.gen_range(0..high) for usize: UniformInt<u64>::sample_single (rand 0.8.5)
    const uint64_t range = high;
    if (range == 0) return r.next_u64();
    const uint64_t zone = (range << __builtin_clzll(range)) - 1ull;
    for (;;) {
        uint64_t v = r.next_u64();
        unsigned __int128 m = (unsigned __int128)v * (unsigned __int128)range;
        if ((uint64_t)m <= zone) return (uint64_t)(m >> 64);
    }
}
// how many items fit_in_memory lets through at once — writer.rs:1536-1566 (page_size = 4096, D::size_of_item)
inline uint64_t lm_items_that_fit(int metric, uint32_t d, uint64_t memory) {
    const uint64_t page_size = 4096;
    const uint64_t nb_page_allowed = (uint64_t)std::floor((double)memory / (double)page_size);
    const uint64_t largest_item_size = 4ull * header_floats(metric) + 4ull * d;
    const uint64_t nb_items_per_page = page_size / largest_item_size;
    const uint64_t nb_page_per_item = (uint64_t)std::ceil((double)largest_item_size / (double)page_size);
    uint64_t nb_items = nb_items_per_page > 1 ? nb_page_allowed * nb_items_per_page : (nb_page_per_item > 1 ? nb_page_allowed / nb_page_per_item : nb_page_allowed);
    if (nb_items <= d) nb_items = (uint64_t)d + 1;
    return nb_items;
}

struct LmMachine {
    IncCtx& C; NodeIdAlloc& alloc;
    uint64_t memory; uint32_t split_after;
    arroy_b200_cancel_fn cancel; void* cancel_arg;
    std::vector<LmTask> stack;              // the 1-thread rayon pool's local deque: popped LIFO
    std::map<uint32_t, HNode> tmp;          // the split nodes make_tree_in_file wrote to the thread's TmpNodes
    uint64_t emitted_bytes = 0;

    // fit_in_memory — writer.rs:1536-1584. `to_insert` ascending ids (RoaringBitmap::select(idx) = idx-th smallest)
    bool fit_in_memory(std::vector<uint32_t>& to_insert, ab::Rng& rng, std::vector<uint32_t>& out) {
        out.clear();
        if (to_insert.empty()) return false;
        if (to_insert.size() <= C.d) { out.swap(to_insert); return true; }
        const uint64_t nb_items = lm_items_that_fit(C.metric, C.d, memory);
        if (nb_items >= to_insert.size()) { out.swap(to_insert); return true; }
        for (uint64_t i = 0; i < nb_items; ++i) {
            const uint64_t idx = rng_below_u64(rng, to_insert.size());
            const uint32_t item = to_insert[idx];
            out.insert(std::lower_bound(out.begin(), out.end(), item), item);
            to_insert.erase(to_insert.begin() + idx);
        }
        return true;
    }
    // make_tree_in_file — writer.rs:1586-1668, on the device, continuing `rng`
    void make_tree(ab::Rng& rng, const std::vector<uint32_t>& items, uint32_t root_id, IntMapOrder& descendants) {
        if (items.size() <= C.K) { descendants.entry(root_id) = items; return; }
        std::vector<uint32_t> rows(items.size());
        for (size_t i = 0; i < rows.size(); ++i) rows[i] = C.row_of(items[i]);
        uint8_t seed[32];
        for (int i = 0; i < 8; ++i) for (int b = 0; b < 4; ++b) seed[4 * i + b] = (uint8_t)(rng.key[i] >> (8 * b));
        const uint64_t start = rng.pos, off[2] = {0, rows.size()};
        uint64_t end = 0;
        uint32_t count = 0;
        dev_ck(C.ctx, arroy_b200_build_subtrees_begin_at(C.ctx, 1, reinterpret_cast<const uint8_t(*)[32]>(seed), &start, rows.data(), off, split_after,
                                                        cancel, cancel_arg, &count, &end));
        uint32_t key[8];
        memcpy(key, rng.key, sizeof key);
        rng.init(key, end);
        std::vector<uint32_t> node_ids(count ? count - 1 : 0);
        for (auto& id : node_ids) id = alloc.next();   // post-order, the order the recursion takes them in
        SinkArg sa;
        dev_ck(C.ctx, arroy_b200_build_trees_emit_mapped(C.ctx, &root_id, node_ids.data(), tree_sink, &sa));
        emitted_bytes += sa.bytes.load();
        std::unordered_map<uint32_t, std::string> got;
        for (int sh = 0; sh < SinkArg::SHARDS; ++sh) for (auto& e : sa.nodes[sh]) got.emplace(e.first, std::move(e.second));
        node_ids.push_back(root_id);
        for (uint32_t id : node_ids) {
            HNode h = decode_tree_node(got.at(id));
            if (h.kind == 1) descendants.entry(id) = std::move(h.desc);   // pending: it may still grow and become a task
            else { tmp[id] = h; C.put(id, std::move(h)); }
        }
    }
    // insert_items_in_descendants_from_tmpfile — writer.rs:1463-1531
    void route(ab::Rng& rng, uint32_t node, const std::vector<uint32_t>& to_insert, IntMapOrder& descendants) {
        auto it = tmp.find(node);
        if (it == tmp.end()) {   // not in the tmp file: a pending descendants entry of this task
            std::vector<uint32_t>& dst = descendants.entry(node);
            std::vector<uint32_t> merged;
            std::set_union(dst.begin(), dst.end(), to_insert.begin(), to_insert.end(), std::back_inserter(merged));
            dst.swap(merged);
            return;
        }
        const HNode& nd = it->second;
        std::vector<uint32_t> left, right;
        if (nd.normal.empty()) {
            for (uint32_t id : to_insert) { if ((int32_t)rng.next_u32() < 0) left.push_back(id); else right.push_back(id); }
        } else {
            const int hf = header_floats(C.metric);
            float h0 = 0.f, h1 = 0.f;
            memcpy(&h0, nd.normal.data(), 4);
            if (hf == 2) memcpy(&h1, nd.normal.data() + 4, 4);
            std::vector<float> nv(C.d);
            memcpy(nv.data(), nd.normal.data() + 4 * hf, 4ull * C.d);
            std::vector<uint32_t> rows(to_insert.size());
            for (size_t i = 0; i < rows.size(); ++i) rows[i] = C.row_of(to_insert[i]);
            std::vector<uint8_t> side(rows.size());
            dev_ck(C.ctx, arroy_b200_side_batch(C.ctx, nv.data(), h0, h1, rows.data(), rows.size(), side.data(), nullptr));
            for (size_t i = 0; i < rows.size(); ++i) { if (side[i]) right.push_back(to_insert[i]); else left.push_back(to_insert[i]); }
        }
        const uint32_t l = nd.left, r = nd.right;
        if (!left.empty()) route(rng, l, left, descendants);
        if (!right.empty()) route(rng, r, right, descendants);
    }
    // insert_descendants_in_file_and_spawn_tasks — writer.rs:744-844, in hashbrown iteration order
    void process_descendants(ab::Rng& rng, IntMapOrder& descendants) {
        for (size_t b = 0; b < descendants.keys.size(); ++b) {
            if (descendants.keys[b] < 0) continue;
            const uint32_t id = (uint32_t)descendants.keys[b];
            std::vector<uint32_t>& ids_v = descendants.vals[b];
            if (ids_v.size() <= C.K) { HNode t; t.kind = 1; t.desc = ids_v; C.put(id, std::move(t)); }
            else stack.push_back(LmTask{rng_fork(rng), id, std::move(ids_v)});
        }
    }
    // incremental_index_large_descendant — writer.rs:660-739
    void run_task(LmTask& task) {
        if (cancel && cancel(cancel_arg)) throw HostError(ARROY_ERR_BUILD_CANCELLED, "The corresponding build process has been cancelled");
        IntMapOrder descendants;
        std::vector<uint32_t> to_insert = std::move(task.items), chunk;
        fit_in_memory(to_insert, task.rng, chunk);
        make_tree(task.rng, chunk, task.id, descendants);
        while (fit_in_memory(to_insert, task.rng, chunk)) route(task.rng, task.id, chunk, descendants);
        process_descendants(task.rng, descendants);
    }
    void run() { while (!stack.empty()) { LmTask t = std::move(stack.back()); stack.pop_back(); run_task(t); } }
};

inline void writer_build(arroy_writer* w, arroy_ctx* ctx, arroy_rng* rng, int64_t n_trees_opt, uint64_t split_after, uint64_t available_memory,
                         arroy_b200_cancel_fn cancel, void* cancel_arg, arroy_progress_fn progress, void* progress_arg) {
    arroy_env* env = w->env;
    std::lock_guard<std::mutex> lk(env->mu);
    for (auto& t : w->timings) t = 0;
    auto t_all = clk::now();
    const bool trace_steps = getenv("ARROY_B200_TRACE") != nullptr;
    auto t_step = clk::now();
    const char* last_step = "start";
    auto step = [&](const char* name) {
        if (trace_steps) { fprintf(stderr, "[trace] build step %-36s %.2f ms\n", last_step, ms_since(t_step)); t_step = clk::now(); last_step = name; }
        if (progress) progress(progress_arg, name);
    };
    auto cancelled = [&]() { if (cancel && cancel(cancel_arg)) throw HostError(ARROY_ERR_BUILD_CANCELLED, "The corresponding build process has been cancelled"); };
    const uint16_t index = w->index;
    const uint32_t d = w->dims;
    const int hf = header_floats(w->metric);

    // pre_process_items — writer.rs:964-976 (DotProduct only: needs the items on the device)
    step("PreProcessingTheItems");
    cancelled();
    ItemView items = collect_items(env, index);
    const uint64_t n = items.ids.size();
    const size_t leaf_len = 1 + 4 * hf + 4ull * d;
    for (uint64_t i = 0; i < n; ++i)
        if (items.sizes[i] != leaf_len) throw HostError(ARROY_ERR_PANIC, "items of different sizes in one index");
    auto t0 = clk::now();
    // Nothing below touches env->kv until commit(): a cancelled or failed build leaves the table exactly as it was (the
    // reference's RwTxn is dropped on error), Updated markers included, so need_build() stays true.
    std::vector<float> dot_extra, dot_norm;   // DotProduct::preprocess results, written back at commit (dot_product.rs:154-160)
    std::vector<uint32_t> updated;
    auto commit_common = [&]() {
        for (uint64_t i = 0; i < dot_extra.size(); ++i) {  // cursor.put_current
            std::string& v = env->kv[make_key(index, MODE_ITEM, items.ids[i])];
            memcpy(&v[1], &dot_extra[i], 4);
            memcpy(&v[5], &dot_norm[i], 4);
        }
        erase_mode(env, index, MODE_UPDATED);
    };
    const uint64_t K_early = split_after ? split_after : d;
    const bool needs_device = n > K_early || (w->metric == ARROY_B200_DOT_PRODUCT && n > 0);
    if (needs_device) {
        if (!ctx) throw HostError(ARROY_B200_ERR_CUDA, "no CUDA device context: arroy_b200 has no CPU fallback");
        dev_ck(ctx, arroy_b200_stage_items(ctx, w->metric, d, n, items.ids.data(), items.ptrs.data()));
        w->timings[0] = ms_since(t0);
        w->timings[5] = (double)n * (((d + 31) & ~31u) * 4.0 + 8.0);
    }
    if (w->metric == ARROY_B200_DOT_PRODUCT && n > 0) {
        t0 = clk::now();
        dot_extra.resize(n); dot_norm.resize(n);
        dev_ck(ctx, arroy_b200_dot_preprocess(ctx, dot_extra.data(), dot_norm.data()));
        w->timings[1] = ms_since(t0);
    }
    step("RetrievingTheItemsIds");
    cancelled();
    step("RetrieveTheUpdatedItems");
    {
        auto e = env->kv.lower_bound(make_key(index, MODE_UPDATED, 0));
        while (e != env->kv.end() && e->first[0] == (uint8_t)(index >> 8) && e->first[1] == (uint8_t)index && e->first[2] == MODE_UPDATED) { updated.push_back(key_item(e->first)); ++e; }
    }
    const uint64_t K = split_after ? split_after : d;
    if (n <= K) {  // clear_db_and_create_a_single_leaf — writer.rs:916-962
        step("WritingTheDescendantsAndMetadata");
        cancelled();
        commit_common();
        erase_mode(env, index, MODE_TREE);
        std::vector<uint32_t> roots;
        if (n > 0) {
            std::vector<uint8_t> buf;
            buf.push_back(1);
            ::roaring_serialize(items.ids.data(), items.ids.size(), buf);
            env->kv[make_key(index, MODE_TREE, 0)] = std::string(reinterpret_cast<char*>(buf.data()), buf.size());
            roots.push_back(0);
        }
        env->kv[make_key(index, MODE_METADATA, 0)] = encode_metadata(w->metric, d, items.ids, roots);
        write_version(env, index);
        env->touch(index);
        w->timings[4] = ms_since(t_all);
        return;
    }
    Metadata old;
    bool had = read_metadata(env, index, old);
    std::vector<uint32_t> roots = had ? old.roots : std::vector<uint32_t>();
    const uint64_t target = target_n_trees(n_trees_opt, d, n, roots.size());
    // available_memory (UINT64_MAX = not set; the reference divides it by the number of threads of its pool, 1 here): when the
    // items of one tree do not fit, the whole build goes through the task machine of the update path, as in the reference
    const uint64_t fit = available_memory == UINT64_MAX ? UINT64_MAX : lm_items_that_fit(w->metric, d, available_memory);
    if (!roots.empty() || n > fit) {
        // ---- an index that already has trees: update it in place --------------------------------------
        IncCtx C{env, ctx, index, w->metric, d, (size_t)K, {}, {}, &items.ids};
        {
            // decode every tree node of the index (threads: the leaves' bitmaps are most of the work)
            std::vector<std::pair<uint32_t, const std::string*>> raw;
            auto it = env->kv.lower_bound(make_key(index, MODE_TREE, 0));
            for (; it != env->kv.end() && it->first[0] == (uint8_t)(index >> 8) && it->first[1] == (uint8_t)index && it->first[2] == MODE_TREE; ++it)
                raw.push_back({key_item(it->first), &it->second});
            std::vector<HNode> dec(raw.size());
            const unsigned nt = (unsigned)std::max<size_t>(1, std::min<size_t>({(size_t)16, (size_t)std::thread::hardware_concurrency(), raw.size() / 4096 + 1}));
            std::string derr; std::mutex dmu;
            auto dwork = [&](unsigned t) {
                try { for (size_t i = t; i < raw.size(); i += nt) dec[i] = decode_tree_node(*raw[i].second); }
                catch (const std::exception& e) { std::lock_guard<std::mutex> lk(dmu); derr = e.what(); }
            };
            if (nt == 1) dwork(0);
            else { std::vector<std::thread> th; for (unsigned t = 0; t < nt; ++t) th.emplace_back(dwork, t); for (auto& x : th) x.join(); }
            if (!derr.empty()) throw HostError(ARROY_ERR_PANIC, derr);
            for (size_t i = 0; i < raw.size(); ++i) C.tree.emplace_hint(C.tree.end(), raw[i].first, std::move(dec[i]));
            C.index_lookups();
        }
        step("RetrievingTheUsedTreeNodes");
        NodeIdAlloc alloc(C.tree);
        step("DeletingExtraTrees");
        {   // writer.rs:632-653
            size_t extraneous = roots.size() > target ? roots.size() - (size_t)target : 0;
            for (size_t i = 0; i < extraneous && !roots.empty(); ++i) { cancelled(); uint32_t r0 = roots[0]; roots[0] = roots.back(); roots.pop_back(); inc_delete_tree(C, r0); }
        }
        step("RemoveItemsFromExistingTrees");
        const IdSet to_delete(updated);
        {   // writer.rs:978-1015
            // one recursion per root; they only read the decoded tree, so they run on threads and their puts / removals are
            // merged afterwards (the final state does not depend on the order)
            TmpOps tmp;
            cancelled();
            std::vector<TmpOps> per(roots.size());
            const unsigned nt = (unsigned)std::max<size_t>(1, std::min<size_t>({(size_t)16, (size_t)std::thread::hardware_concurrency(), roots.size()}));
            std::atomic<size_t> next_root{0};
            std::string derr; std::mutex dmu;
            auto rwork = [&] {
                try { for (;;) { size_t i = next_root.fetch_add(1); if (i >= roots.size()) return; roots[i] = inc_delete_items(C, roots[i], per[i], to_delete).first; } }
                catch (const std::exception& e) { std::lock_guard<std::mutex> lk(dmu); derr = e.what(); }
            };
            if (nt == 1) rwork();
            else { std::vector<std::thread> th; for (unsigned t = 0; t < nt; ++t) th.emplace_back(rwork); for (auto& x : th) x.join(); }
            if (!derr.empty()) throw HostError(ARROY_ERR_PANIC, derr);
            for (auto& p : per) { for (auto& pr : p.puts) tmp.puts.push_back(std::move(pr)); tmp.deleted.insert(p.deleted.begin(), p.deleted.end()); }
            std::sort(roots.begin(), roots.end());
            for (uint32_t id : tmp.deleted) C.erase(id);
            for (auto& pr : tmp.puts) if (!tmp.deleted.count(pr.first)) C.put(pr.first, HNode(pr.second));
        }
        step("InsertItemsInCurrentTrees");
        std::vector<uint32_t> to_insert;
        for (uint32_t id : updated) if (std::binary_search(items.ids.begin(), items.ids.end(), id)) to_insert.push_back(id);
        IntMapOrder top;
        if (!roots.empty() && !to_insert.empty()) {   // writer.rs:846-889, :1119-1160 (rayon reduce on a 1-thread pool: one split at len / 2)
            const uint64_t seed = rng->r.next_u64();
            std::unordered_map<uint32_t, Routed> routed;
            std::unordered_map<uint32_t, std::vector<uint32_t>> leaf_ins;
            const std::vector<char> batched = inc_route_batched(C, roots, to_insert, routed, leaf_ins);   // all side() loops, one launch per depth
            auto fold = [&](size_t a, size_t b) {
                IntMapOrder acc;
                for (size_t i = a; i < b; ++i) {
                    cancelled();
                    IntMapOrder per_root;
                    if (batched[i]) inc_replay(C, roots[i], routed, leaf_ins, per_root);
                    else { ab::Rng rr = rng_seed_from_u64(seed + (uint64_t)roots[i]); inc_route(C, rr, roots[i], to_insert, per_root); }
                    acc.merge_from(per_root);
                }
                return acc;
            };
            IntMapOrder reduced;
            if (roots.size() >= 2) { size_t mid = roots.size() / 2; reduced = fold(0, mid); IntMapOrder right = fold(mid, roots.size()); reduced.merge_from(right); }
            else reduced = fold(0, roots.size());
            top.merge_from(reduced);
        }
        step("RetrieveTheLargeDescendants");
        const uint64_t nb_missing = target > roots.size() ? target - roots.size() : 0;
        for (uint64_t i = 0; i < nb_missing; ++i) { uint32_t nid = alloc.next(); roots.push_back(nid); top.entry(nid) = items.ids; }
        // writer.rs:575 + insert_descendants_in_file_and_spawn_tasks (:744-844) in hashbrown order
        uint8_t s1[32];
        rng->r.gen_seed(s1);
        uint32_t key1[8];
        for (int i = 0; i < 8; ++i) key1[i] = (uint32_t)s1[4 * i] | ((uint32_t)s1[4 * i + 1] << 8) | ((uint32_t)s1[4 * i + 2] << 16) | ((uint32_t)s1[4 * i + 3] << 24);
        ab::Rng rng1;
        rng1.init(key1, 0);
        std::vector<std::array<uint8_t, 32>> task_seeds;
        std::vector<uint32_t> task_ids, sub_rows;
        std::vector<uint64_t> sub_off(1, 0);
        bool limited = false;
        for (size_t b = 0; b < top.keys.size(); ++b) if (top.keys[b] >= 0 && top.vals[b].size() > fit) limited = true;
        SinkArg sa;
        if (limited) {
            step("CreateTreesForItems");
            t0 = clk::now();
            LmMachine M{C, alloc, available_memory, (uint32_t)split_after, cancel, cancel_arg, {}, {}, 0};
            M.process_descendants(rng1, top);
            M.run();
            sa.bytes += M.emitted_bytes;
        } else {
        for (size_t b = 0; b < top.keys.size(); ++b) {
            if (top.keys[b] < 0) continue;
            cancelled();
            const uint32_t id = (uint32_t)top.keys[b];
            std::vector<uint32_t>& ids_v = top.vals[b];
            if (ids_v.size() <= K) { HNode t; t.kind = 1; t.desc = ids_v; C.put(id, std::move(t)); }
            else {
                task_seeds.emplace_back();
                rng1.gen_seed(task_seeds.back().data());
                task_ids.push_back(id);
                for (uint32_t iid : ids_v) sub_rows.push_back(C.row_of(iid));
                sub_off.push_back(sub_rows.size());
            }
        }
        step("CreateTreesForItems");
        t0 = clk::now();
        if (!task_ids.empty()) {
            const uint32_t ns = (uint32_t)task_ids.size();
            std::vector<uint32_t> counts(ns, 0);
            dev_ck(ctx, arroy_b200_build_subtrees_begin(ctx, ns, reinterpret_cast<const uint8_t(*)[32]>(task_seeds.data()), sub_rows.data(), sub_off.data(),
                                                       (uint32_t)split_after, cancel, cancel_arg, counts.data()));
            // the spawned tasks run LIFO on a 1-thread pool; each takes its ids from the allocator in post-order
            std::vector<uint64_t> id_off(ns + 1, 0);
            for (uint32_t sidx = 0; sidx < ns; ++sidx) id_off[sidx + 1] = id_off[sidx] + counts[sidx] - 1;
            std::vector<uint32_t> node_ids(id_off[ns]);
            for (uint32_t k2 = 0; k2 < ns; ++k2) { uint32_t sidx = ns - 1 - k2; for (uint64_t j = 0; j + 1 < counts[sidx]; ++j) node_ids[id_off[sidx] + j] = alloc.next(); }
            dev_ck(ctx, arroy_b200_build_trees_emit_mapped(ctx, task_ids.data(), node_ids.data(), tree_sink, &sa));
            std::vector<std::pair<uint32_t, std::string>> all;
            for (int sh = 0; sh < SinkArg::SHARDS; ++sh) { for (auto& e : sa.nodes[sh]) all.emplace_back(std::move(e)); sa.nodes[sh].clear(); }
            for (auto& e : all) C.pending[e.first] = {true, std::move(e.second)};
        }
        }
        w->timings[2] = ms_since(t0);
        w->timings[6] = (double)sa.bytes.load();
        step("WriteTheMetadata");
        cancelled();
        commit_common();
        C.commit();
        env->kv[make_key(index, MODE_METADATA, 0)] = encode_metadata(w->metric, d, items.ids, roots);
        write_version(env, index);
        env->touch(index);
        w->timings[4] = ms_since(t_all);
        return;
    }
    step("RetrievingTheItems");
    step("RetrieveTheLargeDescendants");
    if (target > 0xffffffffull) throw HostError(ARROY_ERR_DATABASE_FULL, "Database full. Arroy cannot generate enough internal IDs for your items");
    for (uint64_t t = 0; t < target; ++t) roots.push_back((uint32_t)t);  // concurrent_node_ids.next() — writer.rs:556-561
    // seed chain — writer.rs:575 (rng1 = from_seed(rng.gen())), :795 (one from_seed(rng1.gen()) per tree)
    uint8_t s1[32];
    rng->r.gen_seed(s1);
    uint32_t key1[8];
    for (int i = 0; i < 8; ++i) key1[i] = (uint32_t)s1[4 * i] | ((uint32_t)s1[4 * i + 1] << 8) | ((uint32_t)s1[4 * i + 2] << 16) | ((uint32_t)s1[4 * i + 3] << 24);
    ab::Rng rng1;
    rng1.init(key1, 0);
    std::vector<std::array<uint8_t, 32>> seeds(target);
    for (uint64_t t = 0; t < target; ++t) rng1.gen_seed(seeds[t].data());
    step("CreateTreesForItems");
    t0 = clk::now();
    SinkArg sa;
    uint64_t n_nodes = 0;
    dev_ck(ctx, arroy_b200_build_trees(ctx, (uint32_t)target, reinterpret_cast<const uint8_t(*)[32]>(seeds.data()), roots.data(), (uint32_t)target,
                                       (uint32_t)split_after, cancel, cancel_arg, tree_sink, &sa, &n_nodes));
    commit_common();
    {   // move the parked nodes into the ordered table, ascending by id
        std::vector<std::pair<uint32_t, std::string>> all;
        for (int sh = 0; sh < SinkArg::SHARDS; ++sh) { for (auto& e : sa.nodes[sh]) all.emplace_back(std::move(e)); sa.nodes[sh].clear(); }
        std::sort(all.begin(), all.end(), [](const std::pair<uint32_t, std::string>& a, const std::pair<uint32_t, std::string>& b) { return a.first < b.first; });
        auto hint = env->kv.lower_bound(make_key(index, MODE_TREE, 0));
        for (auto& e : all) hint = std::next(env->kv.insert_or_assign(hint, make_key(index, MODE_TREE, e.first), std::move(e.second)));
    }
    w->timings[2] = ms_since(t0);
    w->timings[6] = (double)sa.bytes.load();
    step("WriteTheMetadata");
    t0 = clk::now();
    env->kv[make_key(index, MODE_METADATA, 0)] = encode_metadata(w->metric, d, items.ids, roots);
    write_version(env, index);
    env->touch(index);
    w->timings[3] = ms_since(t0);
    w->timings[4] = ms_since(t_all);
}

// ---- Reader ---------------------------------------------------------------------------------------
inline void reader_open(arroy_env* env, uint16_t index, int metric, arroy_ctx* ctx, arroy_reader** out) {
    std::lock_guard<std::mutex> lk(env->mu);
    Metadata md;
    if (!read_metadata(env, index, md))
        throw HostError(ARROY_ERR_MISSING_METADATA, "Metadata are missing on index " + std::to_string(index) + ", You must build your database before attempting to read it");
    if (md.distance != metric_name(metric))
        throw HostError(ARROY_ERR_UNMATCHING_DISTANCE, "Invalid distance provided. Got " + std::string(metric_name(metric)) + " but expected " + md.distance);
    {
        auto it = env->kv.lower_bound(make_key(index, MODE_UPDATED, 0));
        if (it != env->kv.end() && it->first[0] == (uint8_t)(index >> 8) && it->first[1] == (uint8_t)index && it->first[2] == MODE_UPDATED)
            throw HostError(ARROY_ERR_NEED_BUILD, "The trees have not been built after an update on index " + std::to_string(index));
    }
    auto r = std::unique_ptr<arroy_reader>(new arroy_reader());
    r->env = env; r->ctx = ctx; r->index = index; r->metric = metric; r->dims = md.dims;
    r->roots = md.roots; r->items = md.items;
    r->gen_at_open = env->gen_of(index);
    const uint32_t d = md.dims;
    const int hf = header_floats(metric);
    // decode the tree nodes once (the reference decodes per access from the LMDB page)
    auto it = env->kv.lower_bound(make_key(index, MODE_TREE, 0));
    for (; it != env->kv.end() && it->first[0] == (uint8_t)(index >> 8) && it->first[1] == (uint8_t)index && it->first[2] == MODE_TREE; ++it) {
        uint32_t id = key_item(it->first);
        if (r->nodes.size() <= id) r->nodes.resize((size_t)id + 1);
        arroy_reader::Node& nd = r->nodes[id];
        const uint8_t* b = reinterpret_cast<const uint8_t*>(it->second.data());
        size_t len = it->second.size();
        if (b[0] == 1) {
            nd.kind = 1;
            nd.desc_off = (uint32_t)r->desc.size();
            roaring_deserialize(b + 1, len - 1, r->desc);
            nd.desc_len = (uint32_t)r->desc.size() - nd.desc_off;
        } else if (b[0] == 2) {
            nd.kind = 2;
            nd.left = ((uint32_t)b[1] << 24) | ((uint32_t)b[2] << 16) | ((uint32_t)b[3] << 8) | b[4];
            nd.right = ((uint32_t)b[5] << 24) | ((uint32_t)b[6] << 16) | ((uint32_t)b[7] << 8) | b[8];
            if (len > 9) {
                nd.has_normal = true;
                memcpy(&nd.h0, b + 9, 4);
                if (hf == 2) memcpy(&nd.h1, b + 13, 4);
                nd.normal_off = (uint32_t)(r->normals.size() / d);
                size_t o = r->normals.size();
                r->normals.resize(o + d);
                memcpy(&r->normals[o], b + 9 + 4 * hf, 4ull * d);
            }
        } else throw HostError(ARROY_ERR_PANIC, "Did not recognize node tag type");
    }
    // items: keep the headers for by_item; the vectors are staged on the device lazily, at the first
    // query that has candidates to re-rank
    ItemView iv = collect_items(env, index);
    if (iv.ids != r->items) throw HostError(ARROY_ERR_NEED_BUILD, "The trees have not been built after an update on index " + std::to_string(index));
    r->hdr0.resize(iv.ids.size());
    r->hdr1.assign(iv.ids.size(), 0.f);
    for (size_t i = 0; i < iv.ids.size(); ++i) { memcpy(&r->hdr0[i], iv.ptrs[i] + 1, 4); if (hf == 2) memcpy(&r->hdr1[i], iv.ptrs[i] + 5, 4); }
    *out = r.release();
}

// A reader is a snapshot of its index at open time. The in-memory table has no RoTxn, so a reader that outlives a committed
// write to ITS index (rebuild, add / delete, clear) is refused instead of mixing old tree nodes with new items.
inline void check_fresh_locked(const arroy_reader* r) {
    if (r->env->gen_of(r->index) != r->gen_at_open)
        throw HostError(ARROY_ERR_NEED_BUILD, "index " + std::to_string(r->index) + " was modified after this reader was opened; open a new Reader");
}
inline void check_fresh(const arroy_reader* r) { std::lock_guard<std::mutex> lk(r->env->mu); check_fresh_locked(r); }

inline void ensure_staged(arroy_reader* r) {
    if (!r->ctx) throw HostError(ARROY_B200_ERR_CUDA, "no CUDA device context: arroy_b200 has no CPU fallback");
    uint64_t ep[2] = {0, 0};
    dev_ck(r->ctx, arroy_b200_epochs(r->ctx, ep));
    if (r->stage_epoch != 0 && ep[0] == r->stage_epoch) return;   // the resident items are still the ones this reader staged
    std::lock_guard<std::mutex> lk(r->env->mu);
    check_fresh_locked(r);
    ItemView iv = collect_items(r->env, r->index);
    if (iv.ids != r->items) throw HostError(ARROY_ERR_NEED_BUILD, "The trees have not been built after an update on index " + std::to_string(r->index));
    dev_ck(r->ctx, arroy_b200_stage_items(r->ctx, r->metric, r->dims, iv.ids.size(), iv.ids.data(), iv.ptrs.data()));
    dev_ck(r->ctx, arroy_b200_epochs(r->ctx, ep));
    r->stage_epoch = ep[0];
    r->forest_epoch = 0;   // staging drops whatever forest was resident
}

inline int64_t row_of(const arroy_reader* r, uint32_t item);

// Upload the decoded forest for the batched device search (arroy_b200_load_forest); descendants
// are converted from item ids to rows once.
inline void ensure_forest(arroy_reader* r) {
    ensure_staged(r);
    {
        uint64_t ep[2] = {0, 0};
        dev_ck(r->ctx, arroy_b200_epochs(r->ctx, ep));
        if (r->forest_epoch != 0 && ep[1] == r->forest_epoch) return;   // still this reader's forest, over this reader's items
    }
    const size_t nn = r->nodes.size();
    std::vector<uint8_t> kind(nn);
    std::vector<uint32_t> left(nn), right(nn), nidx(nn), doff(nn), dlen(nn);
    std::vector<float> nh0(nn);
    for (size_t i = 0; i < nn; ++i) {
        const arroy_reader::Node& nd = r->nodes[i];
        kind[i] = nd.kind; left[i] = nd.left; right[i] = nd.right; nidx[i] = nd.has_normal ? nd.normal_off : 0xffffffffu;
        nh0[i] = nd.h0; doff[i] = nd.desc_off; dlen[i] = nd.desc_len;
    }
    std::vector<uint32_t> rows(r->desc.size());
    const bool dense = !r->items.empty() && r->items.front() == 0 && r->items.back() == r->items.size() - 1;
    if (dense) rows = r->desc;
    else {
        unsigned nt = std::max(1u, std::min(32u, std::thread::hardware_concurrency()));
        if (rows.size() < 100000) nt = 1;
        auto conv = [&](size_t a, size_t b) { for (size_t i = a; i < b; ++i) rows[i] = (uint32_t)(std::lower_bound(r->items.begin(), r->items.end(), r->desc[i]) - r->items.begin()); };
        if (nt == 1) conv(0, rows.size());
        else { std::vector<std::thread> th; for (unsigned t = 0; t < nt; ++t) th.emplace_back(conv, rows.size() * t / nt, rows.size() * (t + 1) / nt); for (auto& x : th) x.join(); }
    }
    dev_ck(r->ctx, arroy_b200_load_forest(r->ctx, (uint32_t)nn, kind.data(), left.data(), right.data(), nidx.data(), nh0.data(), doff.data(), dlen.data(),
                                          (uint32_t)(r->normals.size() / std::max<uint32_t>(r->dims, 1)), r->normals.data(), rows.size(), rows.data(),
                                          (uint32_t)r->roots.size(), r->roots.data()));
    uint64_t ep[2] = {0, 0};
    dev_ck(r->ctx, arroy_b200_epochs(r->ctx, ep));
    r->forest_epoch = ep[1];
}

inline int64_t row_of(const arroy_reader* r, uint32_t item) {
    auto it = std::lower_bound(r->items.begin(), r->items.end(), item);
    if (it == r->items.end() || *it != item) return -1;
    return it - r->items.begin();
}

struct QE { float dist; uint32_t node; };
struct QLess {  // max-heap on (OrderedFloat(dist), NodeId): NaN greatest, -0 == +0 — reader.rs:338-342
    bool operator()(const QE& a, const QE& b) const {
        bool an = a.dist != a.dist, bn = b.dist != b.dist;
        if (an || bn) { if (an && bn) return a.node < b.node; return bn; }
        if (a.dist < b.dist) return true;
        if (a.dist > b.dist) return false;
        return a.node < b.node;
    }
};

// the candidate-collecting walk of nns_by_leaf — reader.rs:328-379. Returns sorted unique ROW indices.
inline void tree_walk(const arroy_reader* r, const float* qv, float qh0, uint64_t count, uint64_t search_k_opt, uint64_t oversampling_opt,
                      const std::vector<uint32_t>* candidates, std::vector<uint32_t>& out_rows) {
    out_rows.clear();
    if (r->items.empty()) return;
    unsigned __int128 sk = search_k_opt ? (unsigned __int128)search_k_opt : (unsigned __int128)count * r->roots.size();
    sk *= oversampling_opt ? oversampling_opt : 1;  // D::DEFAULT_OVERSAMPLING = 1
    const uint64_t search_k = sk > (unsigned __int128)UINT64_MAX ? UINT64_MAX : (uint64_t)sk;
    std::priority_queue<QE, std::vector<QE>, QLess> queue;
    for (uint32_t root : r->roots) queue.push(QE{INFINITY, root});
    std::vector<uint32_t> nns;
    const size_t d = r->dims;
    while (nns.size() < search_k) {
        if (queue.empty()) break;
        QE top = queue.top();
        queue.pop();
        if (top.node >= r->nodes.size() || r->nodes[top.node].kind == 0)
            throw HostError(ARROY_ERR_MISSING_KEY, "Internal error: Tree(" + std::to_string(top.node) + ") is missing in index `" + std::to_string(r->index) + "`");
        const arroy_reader::Node& nd = r->nodes[top.node];
        if (nd.kind == 1) {
            const uint32_t* ids = r->desc.data() + nd.desc_off;
            if (candidates) { for (uint32_t i = 0; i < nd.desc_len; ++i) if (std::binary_search(candidates->begin(), candidates->end(), ids[i])) nns.push_back(ids[i]); }
            else nns.insert(nns.end(), ids, ids + nd.desc_len);
        } else {
            float mg = nd.has_normal ? host_margin(r->metric, r->normals.data() + (size_t)nd.normal_off * d, nd.h0, qv, qh0, d) : 0.0f;
            queue.push(QE{f32_min(-mg, top.dist), nd.left});   // D::pq_distance — mod.rs:63-68
            queue.push(QE{f32_min(mg, top.dist), nd.right});
        }
    }
    std::sort(nns.begin(), nns.end());
    nns.erase(std::unique(nns.begin(), nns.end()), nns.end());
    out_rows.reserve(nns.size());
    for (uint32_t id : nns) {
        int64_t row = row_of(r, id);
        if (row < 0) throw HostError(ARROY_ERR_MISSING_KEY, "Internal error: Item(" + std::to_string(id) + ") is missing in index `" + std::to_string(r->index) + "`");
        out_rows.push_back((uint32_t)row);
    }
}

// QueryBuilder::candidates as the device takes it: bit r set when row r (= r->items[r]) is a candidate. Ids that are not in
// the index drop out, as `descendants & candidates` drops them in the reference. `sorted_ids` ascending.
inline std::vector<uint32_t> candidate_row_bits(const arroy_reader* r, const std::vector<uint32_t>& sorted_ids) {
    const size_t n = r->items.size();
    std::vector<uint32_t> bits((n + 31) / 32, 0u);
    if (n && r->items.front() == 0 && r->items.back() == n - 1) {   // ids 0..n-1: row = id
        for (uint32_t id : sorted_ids) { if (id >= n) break; bits[id >> 5] |= 1u << (id & 31); }
        return bits;
    }
    size_t j = 0;
    for (uint32_t id : sorted_ids) {
        while (j < r->items.size() && r->items[j] < id) ++j;
        if (j == r->items.size()) break;
        if (r->items[j] == id) bits[j >> 5] |= 1u << (j & 31);
    }
    return bits;
}

// The same filter as ascending, unique rows (arroy_b200_search_batch_multi_filtered takes row lists).
inline std::vector<uint32_t> candidate_rows(const arroy_reader* r, const std::vector<uint32_t>& sorted_ids) {
    const size_t n = r->items.size();
    std::vector<uint32_t> rows;
    if (n && r->items.front() == 0 && r->items.back() == n - 1) {   // ids 0..n-1: row = id
        for (uint32_t id : sorted_ids) { if (id >= n) break; if (rows.empty() || rows.back() != id) rows.push_back(id); }
        return rows;
    }
    size_t j = 0;
    for (uint32_t id : sorted_ids) {
        while (j < n && r->items[j] < id) ++j;
        if (j == n) break;
        if (r->items[j] == id && (rows.empty() || rows.back() != j)) rows.push_back((uint32_t)j);
    }
    return rows;
}

// Where the host walk of one filtered query beats the device on an H100 (tools/bench_filtered_search.py on C2, DESIGN §7.1):
//   - the filter holds at least 1/20 of the items: few leaves reach search_k, so the host walk is short and the device's fixed
//     cost per filtered call (the bitmap upload and the summary pass over every leaf) dominates;
//   - the filter is a dense row range (at least half of the rows between its first and last row pass) of at least 1/1000 of the
//     items and at least 1000 rows: the host walk's per-row binary searches stay in cache and its walk is as short as for a
//     random filter of that size.
inline bool filter_prefers_host_walk(const std::vector<uint32_t>& bits, uint64_t n) {
    uint64_t in_filter = 0, first = UINT64_MAX, last = 0;
    for (size_t w = 0; w < bits.size(); ++w) {
        if (!bits[w]) continue;
        in_filter += __builtin_popcount(bits[w]);
        if (first == UINT64_MAX) first = 32 * w + __builtin_ctz(bits[w]);
        last = 32 * w + 31 - __builtin_clz(bits[w]);
    }
    if (in_filter * 20 >= n) return true;
    return in_filter >= 1000 && in_filter * 1000 >= n && in_filter * 2 >= last - first + 1;
}

inline uint64_t effective_search_k(const arroy_reader* r, uint64_t count, uint64_t search_k, uint64_t oversampling) {
    unsigned __int128 sk = search_k ? (unsigned __int128)search_k : (unsigned __int128)count * r->roots.size();   // reader.rs:330-335
    sk *= oversampling ? oversampling : 1;
    return sk > (unsigned __int128)UINT64_MAX ? UINT64_MAX : std::max<uint64_t>((uint64_t)sk, 1);
}

inline void nns_by_leaf(arroy_reader* r, const float* qv, float qh0, float qh1, uint64_t count, uint64_t search_k, uint64_t oversampling,
                        const uint32_t* cand, int64_t n_cand, uint32_t* out_ids, float* out_dist, uint64_t* out_len, int64_t qrow = -1) {
    *out_len = 0;
    std::vector<uint32_t> cv, rows;
    if (n_cand >= 0) { cv.assign(cand, cand + n_cand); std::sort(cv.begin(), cv.end()); }
    // One query, whole search on the device (the forest stays resident after the first call): the priority-queue walk, the
    // candidate sort and the re-rank are one arroy_b200_search_batch(_filtered) call with nq = 1 — no host walk over 50 trees, no
    // candidate list crossing PCIe. count > 2048, a device walk that gives up (nonzero status), or a filter whose host walk is
    // cheaper (filter_prefers_host_walk) keeps the host walk below.
    std::vector<uint32_t> fbits;
    const bool device = count > 0 && count <= 2048 && !r->items.empty() && r->ctx && getenv("ARROY_B200_HOST_WALK") == nullptr;
    if (device && n_cand >= 0) fbits = candidate_row_bits(r, cv);
    if (device && (n_cand < 0 || !filter_prefers_host_walk(fbits, r->items.size()))) {
        ensure_forest(r);
        const uint64_t eff = effective_search_k(r, count, search_k, oversampling);
        std::vector<uint32_t> orow(count);
        uint32_t olen = 0, qr = (uint32_t)qrow;
        int32_t status = 0;
        const uint32_t* qrp = qrow >= 0 ? &qr : nullptr;
        const float* qvp = qrow >= 0 ? nullptr : qv;
        const float* qhp = qrow >= 0 ? nullptr : &qh0;
        if (n_cand >= 0) dev_ck(r->ctx, arroy_b200_search_batch_filtered(r->ctx, 1, qrp, qvp, qhp, count, eff, fbits.data(), orow.data(), out_dist, &olen, &status));
        else dev_ck(r->ctx, arroy_b200_search_batch(r->ctx, 1, qrp, qvp, qhp, count, eff, orow.data(), out_dist, &olen, &status));
        if (status == 0) {
            for (uint32_t i = 0; i < olen; ++i) out_ids[i] = r->items[orow[i]];
            *out_len = olen;
            return;
        }
    }
    tree_walk(r, qv, qh0, count, search_k, oversampling, n_cand >= 0 ? &cv : nullptr, rows);
    *out_len = 0;
    if (rows.empty() || count == 0) return;
    const uint32_t k = (uint32_t)std::min<uint64_t>(count, rows.size());
    ensure_staged(r);
    std::vector<uint32_t> orow(k);
    uint32_t olen = 0;
    dev_ck(r->ctx, arroy_b200_rerank(r->ctx, qv, qh0, qh1, rows.data(), rows.size(), k, orow.data(), out_dist, &olen));
    for (uint32_t i = 0; i < olen; ++i) out_ids[i] = r->items[orow[i]];
    *out_len = olen;
}

}  // namespace arroy_host

// ====================================================================================================
extern "C" {
using namespace arroy_host;

const char* arroy_host_last_error(void) { return tls_error().c_str(); }

arroy_env* arroy_env_new(void) { return new arroy_env(); }
void arroy_env_free(arroy_env* e) { delete e; }
uint64_t arroy_env_len(arroy_env* e) { std::lock_guard<std::mutex> lk(e->mu); return e->kv.size(); }
int32_t arroy_env_iter(arroy_env* e, arroy_kv_sink sink, void* arg) {
    return hguard([&] {
        std::lock_guard<std::mutex> lk(e->mu);
        for (auto& kv : e->kv)
            if (sink(arg, kv.first.data(), 8, reinterpret_cast<const uint8_t*>(kv.second.data()), kv.second.size()) != 0) break;
    });
}

// Raw access to the table (tests: importing the key/value pairs of a real LMDB file; exporting ours).
int32_t arroy_env_put_raw(arroy_env* e, const uint8_t* key, uint64_t key_len, const uint8_t* val, uint64_t val_len) {
    return hguard([&] {
        if (key_len != 8) throw HostError(ARROY_ERR_PANIC, "arroy keys are 8 bytes (src/key.rs:56-68)");
        std::lock_guard<std::mutex> lk(e->mu);
        Key8 k;
        memcpy(k.data(), key, 8);
        e->kv[k] = std::string(reinterpret_cast<const char*>(val), val_len);
        e->touch((uint16_t)(((uint16_t)key[0] << 8) | key[1]));
    });
}

// Decode a stored value with the product's decoders and encode it again with the product's encoders (what = 0: a tree node,
// NodeCodec src/node.rs:218-282; 1: Metadata, src/metadata.rs:21-61). A faithful codec returns the input bytes.
int32_t arroy_host_reencode(int32_t what, const uint8_t* in, uint64_t len, uint8_t* out, uint64_t cap, uint64_t* out_len) {
    return hguard([&] {
        std::string res;
        const std::string v(reinterpret_cast<const char*>(in), len);
        if (what == 0) res = encode_tree_node(decode_tree_node(v));
        else {
            arroy_env tmp;
            tmp.kv[make_key(0, MODE_METADATA, 0)] = v;
            Metadata m;
            read_metadata(&tmp, 0, m);
            int metric = -1;
            for (int k = 0; k < 4; ++k) if (m.distance == metric_name(k)) metric = k;
            if (metric < 0) throw HostError(ARROY_ERR_UNMATCHING_DISTANCE, "unknown distance name " + m.distance);
            res = encode_metadata(metric, m.dims, m.items, m.roots);
        }
        *out_len = res.size();
        if (res.size() > cap) throw HostError(ARROY_ERR_PANIC, "output buffer too small");
        memcpy(out, res.data(), res.size());
    });
}

arroy_rng* arroy_rng_from_seed(const uint8_t seed[32]) {
    auto* r = new arroy_rng();
    uint32_t key[8];
    for (int i = 0; i < 8; ++i) key[i] = (uint32_t)seed[4 * i] | ((uint32_t)seed[4 * i + 1] << 8) | ((uint32_t)seed[4 * i + 2] << 16) | ((uint32_t)seed[4 * i + 3] << 24);
    r->r.init(key, 0);
    return r;
}
arroy_rng* arroy_rng_seed_from_u64(uint64_t state) {  // rand_core 0.6 SeedableRng::seed_from_u64 (PCG32 expansion)
    const uint64_t MUL = 6364136223846793005ull, INC = 11634580027462260723ull;
    uint8_t seed[32];
    for (int c = 0; c < 8; ++c) {
        state = state * MUL + INC;
        uint32_t xs = (uint32_t)(((state >> 18) ^ state) >> 27), rot = (uint32_t)(state >> 59);
        uint32_t x = (xs >> rot) | (xs << ((32 - rot) & 31));
        memcpy(seed + 4 * c, &x, 4);
    }
    return arroy_rng_from_seed(seed);
}
arroy_rng* arroy_rng_clone(const arroy_rng* r) { return new arroy_rng(*r); }
void arroy_rng_free(arroy_rng* r) { delete r; }
uint32_t arroy_rng_next_u32(arroy_rng* r) { return r->r.next_u32(); }
float arroy_rng_gen_f32(arroy_rng* r) { return (float)(r->r.next_u32() >> 8) * (1.0f / 16777216.0f); }
void arroy_rng_fill_f32(arroy_rng* r, float* out, uint64_t n) { for (uint64_t i = 0; i < n; ++i) out[i] = arroy_rng_gen_f32(r); }

arroy_writer* arroy_writer_new(arroy_env* env, uint16_t index, uint32_t dimensions, int32_t metric) {
    auto* w = new arroy_writer();
    w->env = env; w->index = index; w->dims = dimensions; w->metric = metric;
    return w;
}
void arroy_writer_free(arroy_writer* w) { delete w; }

static void check_dim(arroy_writer* w, uint32_t len) {
    if (len != w->dims) throw HostError(ARROY_ERR_INVALID_VEC_DIMENSION, "Invalid vector dimensions. Got " + std::to_string(len) + " but expected " + std::to_string(w->dims));
}
int32_t arroy_writer_add_item(arroy_writer* w, uint32_t item, const float* vector, uint32_t len) {
    return hguard([&] { check_dim(w, len); std::lock_guard<std::mutex> lk(w->env->mu); put_item(w, item, vector); });
}
int32_t arroy_writer_add_items(arroy_writer* w, uint64_t n, const uint32_t* items, const float* vectors) {
    return hguard([&] { std::lock_guard<std::mutex> lk(w->env->mu); for (uint64_t i = 0; i < n; ++i) put_item(w, items[i], vectors + i * w->dims); });
}
int32_t arroy_writer_append_item(arroy_writer* w, uint32_t item, const float* vector, uint32_t len) {  // writer.rs:403-425
    return hguard([&] {
        check_dim(w, len);
        std::lock_guard<std::mutex> lk(w->env->mu);
        // PutFlags::APPEND: the key must be greater than every key of the database
        if (!w->env->kv.empty() && !(w->env->kv.rbegin()->first < make_key(w->index, MODE_ITEM, item)))
            throw HostError(ARROY_ERR_INVALID_ITEM_APPEND, "Item cannot be appended into the database");
        put_item(w, item, vector);
    });
}
int32_t arroy_writer_del_item(arroy_writer* w, uint32_t item, int32_t* out_existed) {  // writer.rs:428-441
    return hguard([&] {
        std::lock_guard<std::mutex> lk(w->env->mu);
        bool ex = w->env->kv.erase(make_key(w->index, MODE_ITEM, item)) > 0;
        if (ex) { w->env->kv[make_key(w->index, MODE_UPDATED, item)] = std::string(); w->env->touch(w->index); }
        if (out_existed) *out_existed = ex ? 1 : 0;
    });
}
int32_t arroy_writer_clear(arroy_writer* w) {  // writer.rs:444-457
    return hguard([&] {
        std::lock_guard<std::mutex> lk(w->env->mu);
        for (uint8_t m = 0; m < 4; ++m) erase_mode(w->env, w->index, m);
        w->env->touch(w->index);
    });
}
int32_t arroy_writer_need_build(arroy_writer* w, int32_t* out) {  // writer.rs:343-357
    return hguard([&] {
        std::lock_guard<std::mutex> lk(w->env->mu);
        auto it = w->env->kv.lower_bound(make_key(w->index, MODE_UPDATED, 0));
        bool upd = it != w->env->kv.end() && it->first[0] == (uint8_t)(w->index >> 8) && it->first[1] == (uint8_t)w->index && it->first[2] == MODE_UPDATED;
        *out = (upd || w->env->kv.find(make_key(w->index, MODE_METADATA, 0)) == w->env->kv.end()) ? 1 : 0;
    });
}
int32_t arroy_writer_contains_item(arroy_writer* w, uint32_t item, int32_t* out) {
    return hguard([&] { std::lock_guard<std::mutex> lk(w->env->mu); *out = w->env->kv.count(make_key(w->index, MODE_ITEM, item)) ? 1 : 0; });
}
int32_t arroy_writer_is_empty(arroy_writer* w, int32_t* out) {
    return hguard([&] { std::lock_guard<std::mutex> lk(w->env->mu); *out = collect_items(w->env, w->index).ids.empty() ? 1 : 0; });
}
int32_t arroy_writer_item_vector(arroy_writer* w, uint32_t item, float* out, int32_t* out_found) {
    return hguard([&] {
        std::lock_guard<std::mutex> lk(w->env->mu);
        auto it = w->env->kv.find(make_key(w->index, MODE_ITEM, item));
        *out_found = it != w->env->kv.end();
        if (*out_found) memcpy(out, it->second.data() + 1 + 4 * header_floats(w->metric), 4ull * w->dims);
    });
}
int32_t arroy_writer_build(arroy_writer* w, arroy_ctx* ctx, arroy_rng* rng, int64_t n_trees, uint64_t split_after, uint64_t available_memory,
                           arroy_b200_cancel_fn cancel, void* cancel_arg, arroy_progress_fn progress, void* progress_arg) {
    return hguard([&] { writer_build(w, ctx, rng, n_trees, split_after, available_memory, cancel, cancel_arg, progress, progress_arg); });
}
int32_t arroy_writer_build_timings(arroy_writer* w, double out[8]) { for (int i = 0; i < 8; ++i) out[i] = w->timings[i]; return 0; }

int32_t arroy_reader_open(arroy_env* env, uint16_t index, int32_t metric, arroy_ctx* ctx, arroy_reader** out) {
    *out = nullptr;
    return hguard([&] { reader_open(env, index, metric, ctx, out); });
}
void arroy_reader_free(arroy_reader* r) { delete r; }
uint32_t arroy_reader_dimensions(arroy_reader* r) { return r->dims; }
uint64_t arroy_reader_n_trees(arroy_reader* r) { return r->roots.size(); }
uint64_t arroy_reader_n_items(arroy_reader* r) { return r->items.size(); }
uint64_t arroy_reader_item_ids(arroy_reader* r, uint32_t* out, uint64_t cap) {
    if (out) memcpy(out, r->items.data(), 4 * std::min<uint64_t>(cap, r->items.size()));
    return r->items.size();
}
int32_t arroy_reader_item_vector(arroy_reader* r, uint32_t item, float* out, int32_t* out_found) {
    return hguard([&] {
        std::lock_guard<std::mutex> lk(r->env->mu);
        check_fresh_locked(r);
        auto it = r->env->kv.find(make_key(r->index, MODE_ITEM, item));
        *out_found = it != r->env->kv.end();
        if (*out_found) memcpy(out, it->second.data() + 1 + 4 * header_floats(r->metric), 4ull * r->dims);
    });
}
int32_t arroy_reader_stats(arroy_reader* r, uint64_t* out) {  // reader.rs:210-252
    return hguard([&] {
        struct TS { uint64_t depth, dummy, split, desc; };
        std::function<TS(uint32_t)> rec = [&](uint32_t id) -> TS {
            const arroy_reader::Node& nd = r->nodes.at(id);
            if (nd.kind == 1) return TS{1, 0, 0, 1};
            TS l = rec(nd.left), rr = rec(nd.right);
            return TS{1 + std::max(l.depth, rr.depth), l.dummy + rr.dummy + (nd.has_normal ? 0u : 1u), l.split + rr.split + 1, l.desc + rr.desc};
        };
        for (size_t t = 0; t < r->roots.size(); ++t) { TS s = rec(r->roots[t]); out[4 * t] = s.depth; out[4 * t + 1] = s.dummy; out[4 * t + 2] = s.split; out[4 * t + 3] = s.desc; }
    });
}
int32_t arroy_reader_nns_by_item(arroy_reader* r, uint32_t item, uint64_t count, uint64_t search_k, uint64_t oversampling, const uint32_t* cand, int64_t n_cand,
                                 uint32_t* out_ids, float* out_dist, uint64_t* out_len, int32_t* out_found) {
    return hguard([&] {
        *out_len = 0;
        int64_t row = row_of(r, item);
        *out_found = row >= 0;
        if (row < 0) return;  // Ok(None) — reader.rs:46-51
        std::vector<float> q(r->dims);
        int32_t found = 0;
        { std::lock_guard<std::mutex> lk(r->env->mu); check_fresh_locked(r); auto it = r->env->kv.find(make_key(r->index, MODE_ITEM, item)); found = it != r->env->kv.end(); if (found) memcpy(q.data(), it->second.data() + 1 + 4 * header_floats(r->metric), 4ull * r->dims); }
        if (!found) { *out_found = 0; return; }
        nns_by_leaf(r, q.data(), r->hdr0[row], r->hdr1[row], count, search_k, oversampling, cand, n_cand, out_ids, out_dist, out_len, row);
    });
}
int32_t arroy_reader_nns_by_vector(arroy_reader* r, const float* vector, uint32_t len, uint64_t count, uint64_t search_k, uint64_t oversampling,
                                   const uint32_t* cand, int64_t n_cand, uint32_t* out_ids, float* out_dist, uint64_t* out_len) {
    return hguard([&] {
        *out_len = 0;
        if (len != r->dims) throw HostError(ARROY_ERR_INVALID_VEC_DIMENSION, "Invalid vector dimensions. Got " + std::to_string(len) + " but expected " + std::to_string(r->dims));
        float h0, h1;
        check_fresh(r);
        new_header(r->metric, vector, r->dims, h0, h1);  // reader.rs:72-73
        nns_by_leaf(r, vector, h0, h1, count, search_k, oversampling, cand, n_cand, out_ids, out_dist, out_len);
    });
}
}  // extern "C"

namespace arroy_host {

// The filters of a batched call, as id lists sorted ascending: none (`sorted` empty), one for every query, or one per query
// (`of_query`: the query's index into `sorted`).
struct BatchFilters {
    std::vector<std::vector<uint32_t>> sorted;
    std::vector<uint32_t> of_query;
    bool per_query() const { return !of_query.empty(); }
    const std::vector<uint32_t>* of(uint32_t q) const { return sorted.empty() ? nullptr : &sorted[per_query() ? of_query[q] : 0]; }
};

// arroy_reader_nns_batch and arroy_reader_nns_batch_multi
inline void nns_batch_body(arroy_reader* r, uint32_t nq, const uint32_t* items, const float* vectors, uint64_t count, uint64_t search_k,
                           uint64_t oversampling, const BatchFilters& bf, uint32_t* out_ids, float* out_dist, uint32_t* out_len, double* out_ms) {
        const uint32_t d = r->dims;
        const int hf = header_floats(r->metric);
        if ((items == nullptr) == (vectors == nullptr)) throw HostError(ARROY_ERR_PANIC, "exactly one of items / vectors must be given");
        check_fresh(r);
        std::vector<float> q, qh0, qh1;
        std::vector<std::vector<uint32_t>> rows;
        std::vector<uint32_t> fbits;
        if (items)
            for (uint32_t i = 0; i < nq; ++i)
                if (row_of(r, items[i]) < 0) throw HostError(ARROY_ERR_MISSING_KEY, "Internal error: Item(" + std::to_string(items[i]) + ") is missing in index `" + std::to_string(r->index) + "`");
        // by_item: the query vectors are only needed by the host walk (the device path addresses the staged rows);
        // by_vector: their headers come from new_header, as in nns_by_vector (reader.rs:72-73)
        auto load_queries = [&] {
            qh0.resize(nq); qh1.resize(nq); rows.resize(nq);
            if (vectors) {
                q.assign(vectors, vectors + (size_t)nq * d);
                for (uint32_t i = 0; i < nq; ++i) new_header(r->metric, vectors + (size_t)i * d, d, qh0[i], qh1[i]);
                return;
            }
            q.resize((size_t)nq * d);
            std::lock_guard<std::mutex> lk(r->env->mu);
            for (uint32_t i = 0; i < nq; ++i) {
                int64_t row = row_of(r, items[i]);
                const std::string& v = r->env->kv.at(make_key(r->index, MODE_ITEM, items[i]));
                memcpy(&q[(size_t)i * d], v.data() + 1 + 4 * hf, 4ull * d);
                qh0[i] = r->hdr0[row]; qh1[i] = r->hdr1[row];
            }
        };
        if (vectors) load_queries();
        const uint32_t k_dev = (uint32_t)count;
        std::vector<int32_t> status(nq, 0);
        std::vector<uint32_t> orow_dev;
        const bool host_walk = getenv("ARROY_B200_HOST_WALK") != nullptr || count > 2048 || r->items.empty();
        if (!host_walk) {
            // whole search on the device: walk + dedup/sort + re-rank in one call
            ensure_forest(r);
            auto t0d = clk::now();
            std::vector<uint32_t> qrows;
            if (items) { qrows.resize(nq); for (uint32_t i = 0; i < nq; ++i) qrows[i] = (uint32_t)row_of(r, items[i]); }
            orow_dev.resize((size_t)nq * std::max<uint32_t>(k_dev, 1));
            const uint64_t eff_search_k = effective_search_k(r, count, search_k, oversampling);
            const uint32_t* qrp = items ? qrows.data() : nullptr;
            const float* qvp = items ? nullptr : q.data();
            const float* qhp = items ? nullptr : qh0.data();
            if (bf.per_query()) {   // each used filter as ascending rows, CSR (unused ones empty)
                std::vector<uint64_t> offs(bf.sorted.size() + 1, 0);
                std::vector<uint32_t> frows;
                std::vector<uint8_t> used(bf.sorted.size(), 0);
                for (uint32_t f : bf.of_query) used[f] = 1;
                for (size_t f = 0; f < bf.sorted.size(); ++f) {
                    if (used[f]) { const std::vector<uint32_t> fr = candidate_rows(r, bf.sorted[f]); frows.insert(frows.end(), fr.begin(), fr.end()); }
                    offs[f + 1] = frows.size();
                }
                dev_ck(r->ctx, arroy_b200_search_batch_multi_filtered(r->ctx, nq, qrp, qvp, qhp, count, eff_search_k, (uint32_t)bf.sorted.size(), offs.data(), frows.data(),
                                                                      bf.of_query.data(), orow_dev.data(), out_dist, out_len, status.data()));
            } else if (bf.of(0)) {
                fbits = candidate_row_bits(r, *bf.of(0));
                dev_ck(r->ctx, arroy_b200_search_batch_filtered(r->ctx, nq, qrp, qvp, qhp, count, eff_search_k, fbits.data(), orow_dev.data(), out_dist, out_len, status.data()));
            } else
                dev_ck(r->ctx, arroy_b200_search_batch(r->ctx, nq, qrp, qvp, qhp, count, eff_search_k, orow_dev.data(), out_dist, out_len, status.data()));
            bool all_ok = true;
            for (uint32_t i = 0; i < nq; ++i) {
                if (status[i] != 0) { all_ok = false; continue; }
                for (uint32_t j = 0; j < out_len[i]; ++j) out_ids[(size_t)i * k_dev + j] = r->items[orow_dev[(size_t)i * k_dev + j]];
            }
            if (out_ms) { out_ms[0] = 0.0; out_ms[1] = ms_since(t0d); }
            if (all_ok) return;
        }
        // host walk (all queries, or only the ones the device walk gave up on)
        if (items) load_queries();
        auto t0 = clk::now();
        std::atomic<uint32_t> next{0};
        std::string err; std::mutex emu;
        const bool only_failed = !host_walk;
        auto worker = [&] {
            try { for (;;) { uint32_t i = next.fetch_add(1); if (i >= nq) return; if (only_failed && status[i] == 0) continue; tree_walk(r, &q[(size_t)i * d], qh0[i], count, search_k, oversampling, bf.of(i), rows[i]); } }
            catch (const std::exception& e) { std::lock_guard<std::mutex> lk(emu); err = e.what(); }
        };
        unsigned nt = std::max(1u, std::min<unsigned>(nq, std::thread::hardware_concurrency()));
        std::vector<std::thread> th;
        for (unsigned t = 0; t < nt; ++t) th.emplace_back(worker);
        for (auto& x : th) x.join();
        if (!err.empty()) throw HostError(ARROY_ERR_PANIC, err);
        if (out_ms) out_ms[0] = ms_since(t0);
        ensure_staged(r);
        t0 = clk::now();
        std::vector<uint32_t> keep_len(out_len, out_len + nq);
        std::vector<float> keep_dist;
        std::vector<uint32_t> keep_ids;
        if (only_failed) { keep_dist.assign(out_dist, out_dist + (size_t)nq * k_dev); keep_ids.assign(out_ids, out_ids + (size_t)nq * k_dev); }
        std::vector<uint64_t> offs(nq + 1, 0);
        for (uint32_t i = 0; i < nq; ++i) offs[i + 1] = offs[i] + rows[i].size();
        std::vector<uint32_t> flat(offs[nq]);
        for (uint32_t i = 0; i < nq; ++i) memcpy(flat.data() + offs[i], rows[i].data(), 4 * rows[i].size());
        const uint32_t k = (uint32_t)count;
        std::vector<uint32_t> orow((size_t)nq * std::max<uint32_t>(k, 1));
        const bool trace = getenv("ARROY_B200_TRACE") != nullptr;
        if (trace) fprintf(stderr, "[trace] nns_batch: %u queries, %llu candidates, flatten %.2f ms\n", nq, (unsigned long long)offs[nq], ms_since(t0));
        for (uint32_t base = 0; base < nq; base += 32768) {
            uint32_t m = std::min<uint32_t>(32768, nq - base);
            std::vector<uint64_t> lo(m + 1);
            for (uint32_t i = 0; i <= m; ++i) lo[i] = offs[base + i] - offs[base];
            dev_ck(r->ctx, arroy_b200_rerank_batch(r->ctx, m, &q[(size_t)base * d], &qh0[base], &qh1[base], flat.data() + offs[base], lo.data(), k,
                                                   orow.data() + (size_t)base * k, out_dist + (size_t)base * k, out_len + base));
        }
        if (trace) fprintf(stderr, "[trace] nns_batch: device re-rank done at %.2f ms\n", ms_since(t0));
        for (uint32_t i = 0; i < nq; ++i) for (uint32_t j = 0; j < out_len[i]; ++j) out_ids[(size_t)i * k + j] = r->items[orow[(size_t)i * k + j]];
        if (only_failed)
            for (uint32_t i = 0; i < nq; ++i) if (status[i] == 0) {
                out_len[i] = keep_len[i];
                memcpy(out_dist + (size_t)i * k, keep_dist.data() + (size_t)i * k, 4ull * k);
                memcpy(out_ids + (size_t)i * k, keep_ids.data() + (size_t)i * k, 4ull * k);
            }
        if (out_ms) out_ms[1] += ms_since(t0);
}

}  // namespace arroy_host

extern "C" {

int32_t arroy_reader_nns_batch(arroy_reader* r, uint32_t nq, const uint32_t* items, const float* vectors, uint64_t count, uint64_t search_k,
                               uint64_t oversampling, const uint32_t* cand, int64_t n_cand, uint32_t* out_ids, float* out_dist, uint32_t* out_len,
                               double* out_ms) {
    return hguard([&] {
        BatchFilters bf;
        if (n_cand >= 0) { bf.sorted.emplace_back(cand, cand + n_cand); std::sort(bf.sorted[0].begin(), bf.sorted[0].end()); }
        nns_batch_body(r, nq, items, vectors, count, search_k, oversampling, bf, out_ids, out_dist, out_len, out_ms);
    });
}
int32_t arroy_reader_nns_batch_multi(arroy_reader* r, uint32_t nq, const uint32_t* items, const float* vectors, uint64_t count, uint64_t search_k,
                                     uint64_t oversampling, uint32_t n_filters, const uint64_t* cand_offsets, const uint32_t* cand_ids,
                                     const uint32_t* query_filter, uint32_t* out_ids, float* out_dist, uint32_t* out_len, double* out_ms) {
    return hguard([&] {
        if (nq > 0 && n_filters == 0) throw HostError(ARROY_ERR_PANIC, "no filters for the queries");
        if (nq > 0 && (!cand_offsets || !query_filter)) throw HostError(ARROY_ERR_PANIC, "null filter argument");
        for (uint32_t f = 0; f < n_filters; ++f) if (cand_offsets[f + 1] < cand_offsets[f]) throw HostError(ARROY_ERR_PANIC, "filter offsets must not decrease");
        for (uint32_t i = 0; i < nq; ++i) if (query_filter[i] >= n_filters) throw HostError(ARROY_ERR_PANIC, "query_filter out of range");
        BatchFilters bf;
        bf.sorted.resize(n_filters);
        bf.of_query.assign(query_filter, query_filter + nq);
        std::vector<uint8_t> used(n_filters, 0);
        for (uint32_t f : bf.of_query) used[f] = 1;
        for (uint32_t f = 0; f < n_filters; ++f)   // (an unused filter stays empty: nothing reads it)
            if (used[f]) {
                std::vector<uint32_t>& v = bf.sorted[f];
                v.assign(cand_ids + cand_offsets[f], cand_ids + cand_offsets[f + 1]);
                if (!std::is_sorted(v.begin(), v.end())) std::sort(v.begin(), v.end());
            }
        nns_batch_body(r, nq, items, vectors, count, search_k, oversampling, bf, out_ids, out_dist, out_len, out_ms);
    });
}
int32_t arroy_reader_nns_batch_by_item(arroy_reader* r, uint32_t nq, const uint32_t* items, uint64_t count, uint64_t search_k, uint64_t oversampling,
                                       uint32_t* out_ids, float* out_dist, uint32_t* out_len, double* out_ms) {
    return arroy_reader_nns_batch(r, nq, items, nullptr, count, search_k, oversampling, nullptr, -1, out_ids, out_dist, out_len, out_ms);
}

}  // extern "C"
