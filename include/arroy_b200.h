/*
 * arroy_b200.h — C ABI of the H100-native (sm_90a) distance / split / re-rank path of arroy.
 *
 * This is the drop-in boundary (SURVEY.md §8b): a fork of the reference binds these
 * entry points over Rust FFI (`extern "C"`, see INTEGRATION.md) and calls them where
 * it iterates over items today. Plain pointers and sizes only; no C++/torch types.
 *
 * Conventions
 *   - every call returns an int32 status: 0 = ARROY_B200_OK, otherwise an error code;
 *     arroy_b200_last_error(ctx) returns a message for the last failing call on ctx
 *     (mirrors arroy::Error, src/error.rs:7-86; nothing unwinds across the boundary,
 *     the way build tasks turn panics into Error::Panic, src/writer.rs:799-827).
 *   - the caller owns every host buffer passed in or out; the library owns device
 *     memory and pinned staging inside the context.
 *   - entry points are thread-safe per context (internally serialised), like the
 *     reference's Distance trait functions that rayon workers call concurrently.
 *   - "row" = rank of an item id in the ascending id list given to stage_items
 *     (RoaringBitmap iteration order of src/writer.rs:1201).
 *   - header floats per metric (src/node.rs:68-73): Euclidean/Manhattan {bias},
 *     Cosine {norm}, DotProduct {extra_dim, norm}; passed as hdr0, hdr1.
 *   - there is no CPU fallback: without a CUDA device every compute call fails with
 *     ARROY_B200_ERR_CUDA.
 */
#ifndef ARROY_B200_H
#define ARROY_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct arroy_ctx arroy_ctx;

enum {
    ARROY_B200_OK = 0,
    ARROY_B200_ERR_CUDA = 1,          /* CUDA runtime / driver failure, no device */
    ARROY_B200_ERR_INVALID = 2,       /* bad argument (cf. Error::InvalidVecDimension) */
    ARROY_B200_ERR_CANCELLED = 3,     /* cancel callback returned non-zero (Error::BuildCancelled) */
    ARROY_B200_ERR_CAPACITY = 4,      /* internal table overflow (node records / normals / DFS stack) */
    ARROY_B200_ERR_NOT_STAGED = 5,    /* items have not been staged on this context */
    ARROY_B200_ERR_INTERNAL = 6       /* caught C++ exception (cf. Error::Panic) */
};

/* Distance implementations of src/distance/{euclidean,cosine,dot_product,manhattan}.rs */
enum {
    ARROY_B200_EUCLIDEAN = 0,
    ARROY_B200_COSINE = 1,
    ARROY_B200_DOT_PRODUCT = 2,
    ARROY_B200_MANHATTAN = 3,
    /* src/distance/binary_quantized_{euclidean,cosine,manhattan}.rs. Their vectors are bit strings (BinaryQuantized,
     * src/unaligned_vector/binary_quantized.rs); across this boundary — normals, queries, split results — they travel
     * DEQUANTIZED, as the +-1.0 values BinaryQuantized::iter yields, 64 * ceil(dims / 64) of them (padding bits are 0 = -1.0;
     * the reference's byte-wise popcount kernels count them). Staging quantizes: arroy_b200_stage_items takes the stored
     * bit strings, _flat / _device take f32 vectors of `dim` = the index' dimensions. arroy_b200_bq_quantize makes a query. */
    ARROY_B200_BQ_EUCLIDEAN = 4,
    ARROY_B200_BQ_COSINE = 5,
    ARROY_B200_BQ_MANHATTAN = 6
};

/* ---- context ----------------------------------------------------------------------- */

/* process start / end. `device` is the CUDA ordinal. */
int32_t arroy_b200_create(int32_t device, arroy_ctx** out);
void arroy_b200_destroy(arroy_ctx* ctx);
const char* arroy_b200_last_error(arroy_ctx* ctx);
/* library version string and the SM architecture the kernels were compiled for */
const char* arroy_b200_version(void);
/* What the library holds now, in the whole process (no context, no CUDA call): out[0] = live device buffers, out[1] = their
 * bytes, out[2] = live pinned host buffers, out[3] = their bytes, out[4] = live CUDA streams, events, graphs, graph execs and
 * cuBLAS handles. Destroying every context and group brings all five back to where they were before they were created. */
int32_t arroy_b200_allocations(uint64_t out[5]);

/* ---- item staging: replaces ImmutableLeafs::new (src/parallel.rs:271-293) ------------- */

/* `leaf_values[i]` points at the raw stored value of item ids_ascending[i]:
 * [tag 0x00][Header POD][dim x f32 native endian], byte aligned only
 * (src/node.rs:224-228, src/unaligned_vector/f32.rs). The library decodes the unaligned
 * bytes into pinned host memory and uploads them once into float[n][ld] (ld = dim
 * rounded up to 32 floats, zero padded) plus header arrays; binary-quantized values are
 * bit strings and stay bit strings on the device (arroy_b200_device_ptrs).
 * Placement: this call and arroy_b200_stage_items_flat let arroy_b200_item_placement_plan decide, with cudaMemGetInfo's free
 * bytes plus the bytes the context already holds for items, their planes, the bf16 shadow and the wave buffers (a staging with
 * the metric, dim and n of the last device-placed one that asked takes its answer again). Host placement keeps float[n][ld] in
 * library-owned mapped pinned host memory: the rows are decoded straight into it and cross PCIe once, in chunks, to a device
 * bounce buffer where the build's 8-bit planes and scales (and, for _flat's Cosine default headers, the norms) are written; the
 * device then holds 2 ld + 4 bytes per item plus headers, and no f32 rows. Builds scan through the planes and read the f32 rows
 * they cannot decide from host memory. Batched queries and re-ranks estimate their candidates from the planes and read only
 * the rows that can still reach the top-k from host memory (arroy_b200_plane_rerank_stats); single queries and
 * arroy_b200_rerank_shared read all their candidates' host rows. Results are identical either way. A failed
 * pinned allocation is ARROY_B200_ERR_CUDA and leaves nothing staged. ARROY_B200_HOST_ITEMS=1 forces host placement for
 * eligible indexes (tests and measurements). */
int32_t arroy_b200_stage_items(arroy_ctx* ctx, int32_t metric, uint32_t dim, uint64_t n,
                               const uint32_t* ids_ascending, const uint8_t* const* leaf_values);

/* Where arroy_b200_stage_items / _flat put the f32 rows (host only, no device): 0 = device memory, 1 = mapped pinned host
 * memory. Device when the f32 rows, both 8-bit planes, the scales, the headers and the wave buffers of one tree (split_after =
 * dim) fit in 0.7 x free_bytes, the factor the build's wave sizing uses. Otherwise host, but only for a float metric (0-3) with
 * 64 <= dim <= 8192 (the planes' range); every other index is placed on the device, and fails there as before if it does not
 * fit. Monotone in free_bytes. */
uint32_t arroy_b200_item_placement_plan(int32_t metric, uint32_t dim, uint64_t n, uint64_t free_bytes);
/* The placement of the staged items: out[0] = 0 device / 1 host, out[1] = device bytes held for item data (the f32 rows, or for
 * host placement the planes and scales), out[2] = pinned host bytes of the f32 rows (0 on the device). */
int32_t arroy_b200_item_placement(arroy_ctx* ctx, uint64_t out[3]);

/* The same staging for a caller that knows which items it has written since the resident ones were staged: same arguments and
 * the same postcondition as arroy_b200_stage_items (the context holds exactly the n items given, row = rank of the id, headers
 * from the leaf values, a new stage epoch; the bf16 shadow, the 8-bit planes and the loaded forest are invalid), but the rows
 * that are resident already stay on the device and only move to their new place (csrc/restage.cuh).
 * The caller's promise: for every id that is resident (given to the last staging call) and in ids_ascending and NOT in
 * changed_ids, the resident row equals the vector in leaf_values. changed_ids ascends strictly; ids in it that are not in
 * ids_ascending (deleted items) are ignored; ids of ids_ascending that are not resident are uploaded whether listed or not.
 * Headers are small and DotProduct::preprocess rewrites all of them, so h0 / h1 of all n leaf values are read and uploaded.
 * The library stages in full, exactly as arroy_b200_stage_items, when one of these holds (arroy_b200_stage_stats tells):
 *   - nothing is staged, or a staging is open (arroy_b200_stage_begin without _end), or n or the resident count is 0;
 *   - the resident items are placed in host memory (arroy_b200_item_placement);
 *   - metric or dim differ from the resident ones (the row size follows from the two);
 *   - n rows do not fit the capacity of the resident buffer (it is allocated with 25 % of slack, so repeated small appends
 *     stay in place);
 *   - more than a quarter of the n rows would be uploaded;
 *   - the scratch buffer of the move (at most 240 MB, released before the call returns) cannot be allocated. */
int32_t arroy_b200_stage_items_delta(arroy_ctx* ctx, int32_t metric, uint32_t dim, uint64_t n,
                                     const uint32_t* ids_ascending, const uint8_t* const* leaf_values,
                                     uint64_t n_changed, const uint32_t* changed_ids);
/* Of the last arroy_b200_stage_items / arroy_b200_stage_items_delta call: out[0] = rows uploaded from the host, out[1] = rows
 * moved on the device, out[2] = 1 if the delta path ran, 0 for a full staging, out[3] = bytes it copied host -> device: the
 * uploaded rows, 8 n of headers and, on the delta path, 16 bytes per piece of its copy plan (a run of consecutive rows that
 * moves or is uploaded, cut at 64 KB). */
int32_t arroy_b200_stage_stats(arroy_ctx* ctx, uint64_t out[4]);
/* The raw resident rows `rows` (row size as arroy_b200_device_ptrs reports it, padding included) copied to `out`; for tests,
 * next to arroy_b200_item_headers and arroy_b200_prefilter_planes. */
int32_t arroy_b200_read_items(arroy_ctx* ctx, const uint32_t* rows, uint64_t n_rows, uint8_t* out);
/* The plan of the delta staging (host only, no device): out_src[r] = the row of old_ids that row r of new_ids keeps, -1 when
 * its vector is uploaded (the id is not in old_ids, or is in changed_ids). All three lists ascend strictly. Returns the number
 * of -1 entries. */
uint64_t arroy_b200_stage_delta_plan(const uint32_t* old_ids, uint64_t n_old, const uint32_t* new_ids, uint64_t n_new,
                                     const uint32_t* changed_ids, uint64_t n_changed, int64_t* out_src);

/* The same staging in pieces: _begin sizes the device buffers for n items, _rows decodes + uploads the leaf values of rows
 * [row0, row0 + n_rows) (leaf_values[i] belongs to row row0 + i) and returns when they are in device memory, _end uploads the
 * headers collected from the leaf values and marks the items staged (headers_on_device != 0: the caller has filled the header
 * arrays of arroy_b200_device_ptrs itself, e.g. by a broadcast). Between _begin and _end arroy_b200_device_ptrs is valid, so a
 * multi-GPU host can broadcast chunk k while chunk k + 1 is crossing PCIe (arroy_b200_group_stage_items does exactly that). */
int32_t arroy_b200_stage_begin(arroy_ctx* ctx, int32_t metric, uint32_t dim, uint64_t n, const uint32_t* ids_ascending);
int32_t arroy_b200_stage_rows(arroy_ctx* ctx, uint64_t row0, uint64_t n_rows, const uint8_t* const* leaf_values);
int32_t arroy_b200_stage_end(arroy_ctx* ctx, int32_t headers_on_device);

/* Same, from a dense host matrix (n x dim, row-major f32) and optional header arrays
 * (NULL = header as Writer::add_item would store it, i.e. D::new_header(vector),
 * src/writer.rs:388-390). Copies straight from the caller's buffer (pin it for full PCIe rate). */
int32_t arroy_b200_stage_items_flat(arroy_ctx* ctx, int32_t metric, uint32_t dim, uint64_t n,
                                    const uint32_t* ids_ascending, const float* vectors,
                                    const float* hdr0, const float* hdr1);

/* Same, but the matrix already lives in device memory of ctx's device (n x dim f32,
 * row-major, dense). Used by the multi-GPU path after the NCCL broadcast and by
 * benchmarks whose inputs are resident in HBM. The data is copied into the library's
 * padded layout (device to device). Always places the items on the device, as do
 * arroy_b200_stage_begin / _rows / _end and the group API. */
int32_t arroy_b200_stage_items_device(arroy_ctx* ctx, int32_t metric, uint32_t dim, uint64_t n,
                                      const uint32_t* ids_ascending, const void* device_vectors);

/* Read back the item headers as the build sees them (n floats each; hdr1 may be NULL). */
int32_t arroy_b200_item_headers(arroy_ctx* ctx, float* out_hdr0, float* out_hdr1);

/* ---- D::preprocess: replaces DotProduct::preprocess (src/distance/dot_product.rs:119-165,
 *      called from src/writer.rs:964-976). Updates the staged headers in place and
 *      returns them so the caller can write them back to storage. No-op for other metrics. */
int32_t arroy_b200_dot_preprocess(arroy_ctx* ctx, float* out_extra_dim /* n or NULL */,
                                  float* out_norm /* n or NULL */);

/* ---- side() loops (src/writer.rs:1201-1207, 1424-1430, 1494-1500) ---------------------- */

/* For each row: margin = D::margin(normal, item) bit-exact with the reference's x86_64
 * AVX+FMA / SSE / scalar summation order; side = margin.is_sign_positive() ? 1 (Right)
 * : 0 (Left) (src/distance/mod.rs:103-110). out_margin may be NULL. Binary-quantized metrics:
 * the normal is a bit string in the reference, so only the sign of each element counts
 * (is_sign_positive: +0.0 -> +1, -0.0 -> -1); the margin is hdr0 + dot of the +-1 vectors
 * (Cosine: the dot). The same holds for arroy_b200_side_multi. */
int32_t arroy_b200_side_batch(arroy_ctx* ctx, const float* normal, float hdr0, float hdr1,
                              const uint32_t* rows, uint64_t n_rows,
                              uint8_t* out_side, float* out_margin);

/* Many side() loops in one launch (level-batched routing of new items down existing trees,
 * src/writer.rs:1398-1459): job j tests rows[row_offsets[j] .. row_offsets[j+1]) against
 * normals[j] (dim floats) with header hdr0[j] (bias / extra_dim). out_side has the layout of rows. Items placed in host memory
 * are tested through the build's 8-bit planes first (the same sides; only undecided rows read the f32 row). */
int32_t arroy_b200_side_multi(arroy_ctx* ctx, uint32_t n_jobs, const float* normals, const float* hdr0, const float* hdr1,
                              const uint32_t* rows, const uint64_t* row_offsets, uint8_t* out_side);

/* ---- D::create_split (two_means + normal) on a row subset — src/distance/mod.rs:126-171
 *      and the four create_split impls. `rng_key` (8 LE words of the 32-byte StdRng seed)
 *      and `*rng_word_pos` (how many u32 words of the ChaCha12 stream have been consumed)
 *      describe the caller's StdRng; *rng_word_pos is advanced exactly as the reference
 *      would advance it. Rows must be ascending. */
int32_t arroy_b200_create_split(arroy_ctx* ctx, const uint32_t rng_key[8], uint64_t* rng_word_pos,
                                const uint32_t* rows, uint64_t n_rows,
                                float* out_normal /* dim */, float* out_hdr /* 2 */);

/* ---- whole forest: replaces the per-tree tasks of src/writer.rs:568-591 / :660-739 ----- */

/* Called once per produced tree node, in no particular order, with the exact bytes
 * NodeCodec::bytes_encode would produce (src/node.rs:229-241) — what TmpNodes::put
 * receives in the reference (src/parallel.rs:130-147). Like TmpNodes::put, which every rayon
 * worker calls on its own thread-local file, the sink may be called CONCURRENTLY from several
 * host threads (never twice for the same node id); it must be thread-safe. Return non-zero to
 * abort the build. */
typedef int32_t (*arroy_b200_node_sink)(void* arg, uint32_t node_id, const uint8_t* bytes, uint64_t len);
/* Polled between device steps; non-zero cancels (BuildOption::cancel, src/writer.rs:116-124). */
typedef int32_t (*arroy_b200_cancel_fn)(void* arg);

/* Build `n_trees` trees over all staged items. tree_seeds[t] is the 32-byte seed of tree
 * t's StdRng (src/writer.rs:795); root_ids[t] its pre-allocated root node id
 * (src/writer.rs:556-561). Non-root node ids are numbered from first_free_node_id in the
 * order a 1-thread rayon pool produces (last tree first, post-order inside a tree), so the
 * result is deterministic and equal to the reference's single-thread snapshots.
 * split_after = max items per Descendants node (src/writer.rs:474-477; 0 = dim).
 * `out_n_nodes` (optional) receives the number of emitted nodes. */
int32_t arroy_b200_build_trees(arroy_ctx* ctx, uint32_t n_trees, const uint8_t (*tree_seeds)[32],
                               const uint32_t* root_ids, uint32_t first_free_node_id,
                               uint32_t split_after,
                               arroy_b200_cancel_fn cancel, void* cancel_arg,
                               arroy_b200_node_sink sink, void* sink_arg,
                               uint64_t* out_n_nodes);

/* The same build in two phases, for forests sharded over several GPUs / processes (trees are
 * independent given the item matrix and their seed, src/writer.rs:795): every rank calls _begin
 * for ITS trees (the device work; out_node_counts[t] = number of nodes of local tree t, root
 * included), the ranks exchange the counts and derive the id bases, then _emit encodes the nodes:
 * non-root node number li (post-order) of local tree t gets id base_ids[t] + li, its root gets
 * root_ids[t]. With base_ids following the last-tree-first rule the union of all ranks' nodes is
 * byte-identical to a single arroy_b200_build_trees call over all trees. */
int32_t arroy_b200_build_trees_begin(arroy_ctx* ctx, uint32_t n_trees, const uint8_t (*tree_seeds)[32],
                                     uint32_t split_after, arroy_b200_cancel_fn cancel, void* cancel_arg,
                                     uint32_t* out_node_counts /* n_trees */);
int32_t arroy_b200_build_trees_emit(arroy_ctx* ctx, const uint32_t* root_ids, const uint64_t* base_ids,
                                    arroy_b200_node_sink sink, void* sink_arg);

/* Incremental builds (src/writer.rs:778-829): after new items were routed down the existing trees,
 * every Descendants node that outgrew split_after is rebuilt as a subtree over ITS items only.
 * subtree s is built over the ascending rows rows[row_offsets[s] .. row_offsets[s+1]) (more than
 * split_after of them) with its own seed; counts as for arroy_b200_build_trees_begin. The nodes are
 * then emitted with caller-chosen ids (the reference takes them from ConcurrentNodeIds, which
 * re-uses freed ids first, src/parallel.rs:238-254): the subtree's root gets root_ids[s] (the id of
 * the descendant it replaces), its other nodes node_ids[...] in post-order, all subtrees
 * concatenated (subtree s contributes counts[s] - 1 ids). */
int32_t arroy_b200_build_subtrees_begin(arroy_ctx* ctx, uint32_t n_subtrees, const uint8_t (*seeds)[32],
                                        const uint32_t* rows, const uint64_t* row_offsets, uint32_t split_after,
                                        arroy_b200_cancel_fn cancel, void* cancel_arg, uint32_t* out_node_counts);
/* The same for hosts that keep using a task's StdRng before and after its tree (memory-limited builds, src/writer.rs:660-739:
 * fit_in_memory draws from the task rng, make_tree_in_file continues the same stream, the routing and the spawned sub-tasks
 * continue it again): seeds[s] is the KEY of subtree s' StdRng, start_pos[s] the number of u32 words already consumed (NULL = 0),
 * out_end_pos[s] (optional) the number consumed when the subtree is finished. */
int32_t arroy_b200_build_subtrees_begin_at(arroy_ctx* ctx, uint32_t n_subtrees, const uint8_t (*seeds)[32], const uint64_t* start_pos,
                                           const uint32_t* rows, const uint64_t* row_offsets, uint32_t split_after,
                                           arroy_b200_cancel_fn cancel, void* cancel_arg, uint32_t* out_node_counts, uint64_t* out_end_pos);
int32_t arroy_b200_build_trees_emit_mapped(arroy_ctx* ctx, const uint32_t* root_ids, const uint32_t* node_ids,
                                           arroy_b200_node_sink sink, void* sink_arg);

/* Statistics of the last build on this context (for roofline accounting):
 * stats[0] = rows that went through side() (sum over scans, retries included)
 * stats[1] = device steps, stats[2] = create_split calls, stats[3] = random-fallback splits,
 * stats[4] = device milliseconds of the build loop (CUDA events), stats[5] = ms in scan kernels (persistent schedule: the
 * duration of the one kernel that holds every scan and partition of the wave; per-attempt launches: only measured with
 * ARROY_B200_PROFILE=1), stats[6] = tree nodes emitted, stats[7] = create_split calls whose
 * speculative two_means was redone sequentially (a mis-predicted branch; results are identical either way). */
int32_t arroy_b200_build_stats(arroy_ctx* ctx, double stats[8]);
/* Of the rows counted in stats[0], how many went through side()'s 8-bit pre-filter (out[0]: the two-plane encoding of the items,
 * one or two bytes per element) and how many of those could not be decided by its error bounds and were scored from the f32
 * row (out[1]). The
 * other rows took the plain f32 scan. out[2]: rows of stats[0] that were covered by the fused root pass (trees x items), which
 * read out[3] rows from the item matrix for all of them. Flags are identical either way. */
int32_t arroy_b200_build_shadow_stats(arroy_ctx* ctx, uint64_t out[4]);
/* The same accounting with the stages of the pre-filter apart: out[0] = rows that went through it (its first stage reads the
 * hi plane, one byte per element), out[1] = of them, rows its first stage could not decide (second stage: the lo plane),
 * out[2] = of them, rows the second stage could not decide either (scored from the f32 row), out[3], out[4] = out[2], out[3] of
 * arroy_b200_build_shadow_stats. */
int32_t arroy_b200_build_prefilter_stats(arroy_ctx* ctx, uint64_t out[5]);
/* The pre-filter's encoding of the staged items (built here if no build has built it since staging): hi and lo receive
 * n x ld int8 each (ld = dim rounded up to 32, padding zero), scale n floats; see kernels.cuh planes_encode_kernel. */
int32_t arroy_b200_prefilter_planes(arroy_ctx* ctx, int8_t* hi, int8_t* lo, float* scale);

/* ---- re-rank: replaces the loop of src/reader.rs:381-399 ------------------------------- */

/* distance = D::built_distance(query, item) for every row, k smallest by
 * (OrderedFloat(distance), item id) ascending (NaN greatest, -0 == +0), then
 * D::normalized_distance. `rows` must be ascending and unique (the reference sorts and
 * dedups first, src/reader.rs:378-379). Writes min(k, n_rows) results. */
int32_t arroy_b200_rerank(arroy_ctx* ctx, const float* query, float qhdr0, float qhdr1,
                          const uint32_t* rows, uint64_t n_rows, uint32_t k,
                          uint32_t* out_rows, float* out_dist, uint32_t* out_len);

/* nq queries in one launch; query q re-ranks rows[row_offsets[q] .. row_offsets[q+1]).
 * Results for query q are written at out_*[q*k ..], out_len[q] entries valid; the slots past them are set to 0. */
int32_t arroy_b200_rerank_batch(arroy_ctx* ctx, uint32_t nq, const float* queries /* nq x dim */,
                                const float* qhdr0 /* nq or NULL */, const float* qhdr1 /* nq or NULL */,
                                const uint32_t* rows, const uint64_t* row_offsets /* nq+1 */, uint32_t k,
                                uint32_t* out_rows, float* out_dist, uint32_t* out_len);

/* nq queries against ONE shared candidate list (BASELINE config 5: 4096 x 100k, d = 768).
 * Large problems (nq * n_rows >= 2^22, d >= 32, not Manhattan) run in two stages: a TF32
 * tensor-core contraction bounds every pair's distance, which discards all candidates that
 * provably cannot reach a query's top-k; the survivors are then re-scored in the reference's exact
 * summation order. Small problems (or ARROY_B200_XRERANK=exact) use a register-tiled exact FP32
 * kernel for every pair. Either way ids and distances are identical to nq calls of
 * arroy_b200_rerank. `rows` ascending and unique. */
int32_t arroy_b200_rerank_shared(arroy_ctx* ctx, uint32_t nq, const float* queries /* nq x dim */,
                                 const float* qhdr0 /* nq or NULL */, const uint32_t* rows, uint64_t n_rows, uint32_t k,
                                 uint32_t* out_rows, float* out_dist, uint32_t* out_len);

/* ---- batched search on the device: candidate walk + re-rank (src/reader.rs:317-401) --------- */

/* Upload a built forest once (after a build / when a reader opens): node arrays indexed by
 * tree node id — kind 0 = missing, 1 = Descendants (desc_rows[desc_off .. +desc_len], ROW indices,
 * ascending), 2 = SplitPlaneNormal (left / right child ids, normal_idx into `normals`
 * (n_normals x dim, row-major) or 0xffffffff for "normal: none", normal_hdr0 = bias / extra_dim). */
int32_t arroy_b200_load_forest(arroy_ctx* ctx, uint32_t n_nodes, const uint8_t* kind, const uint32_t* left,
                               const uint32_t* right, const uint32_t* normal_idx, const float* normal_hdr0,
                               const uint32_t* desc_off, const uint32_t* desc_len,
                               uint32_t n_normals, const float* normals, uint64_t n_desc, const uint32_t* desc_rows,
                               uint32_t n_roots, const uint32_t* roots);

/* nq complete searches in one call: the priority-queue walk of Reader::nns_by_leaf
 * (reader.rs:338-374, one warp per query, identical pop order and margins), dedup + sort of the
 * candidates (reader.rs:378-379), then the re-rank + top-k above. Queries are either stored items
 * (query_rows != NULL: QueryBuilder::by_item) or vectors (queries: nq x dim, qhdr0 = their header:
 * Cosine norm; 0 for the other metrics: QueryBuilder::by_vector). search_k = 0 means
 * count * n_trees * D::DEFAULT_OVERSAMPLING (reader.rs:330-335, saturating), where DEFAULT_OVERSAMPLING
 * is 3 for the three binary-quantized metrics and 1 for the others. A nonzero search_k is the walk's
 * stop count as given: the reference multiplies QueryBuilder::search_k(s) by the oversampling too, so
 * a binding passes s * oversampling (3 * s for a binary-quantized index without one). Query q's
 * results are at out_*[q*count ..], out_len[q] of them; the slots past out_len[q] are set to 0.
 * out_status[q] (optional): 0 ok, 1 candidate buffer overflow,
 * 2 heap overflow, 3 missing node — the caller falls back to its own walk for those queries.
 * The same search_k rule holds for the two filtered variants below. */
int32_t arroy_b200_search_batch(arroy_ctx* ctx, uint32_t nq, const uint32_t* query_rows, const float* queries,
                                const float* qhdr0, uint64_t count, uint64_t search_k,
                                uint32_t* out_rows, float* out_dist, uint32_t* out_len, int32_t* out_status);

/* arroy_b200_search_batch with one QueryBuilder::candidates filter shared by every query of the call (reader.rs:350-357):
 * filter_bits holds ceil(n / 32) words, bit r (word r / 32, bit r % 32) set when staged row r passes. A walk keeps only the
 * filtered rows of each Descendants node and counts only those towards search_k, as the reference does; it never enters a
 * subtree without a filtered row (or a missing node). When the filtered rows of the whole forest number at most search_k, the
 * walk is skipped and they are re-ranked directly. Results and out_status as arroy_b200_search_batch. */
int32_t arroy_b200_search_batch_filtered(arroy_ctx* ctx, uint32_t nq, const uint32_t* query_rows, const float* queries,
                                         const float* qhdr0, uint64_t count, uint64_t search_k, const uint32_t* filter_bits,
                                         uint32_t* out_rows, float* out_dist, uint32_t* out_len, int32_t* out_status);

/* Filtered-search counters since create: out[0] = filtered queries completed on the device, out[1] = of those, answered
 * without a walk (the filter's rows in the forest numbered at most search_k), out[2] = filtered queries returned with a
 * nonzero status (the caller falls back to its own walk), out[3] = nodes popped by filtered walks. */
int32_t arroy_b200_search_stats(arroy_ctx* ctx, uint64_t out[4]);

/* arroy_b200_search_batch_filtered with one filter per query: query q uses filter query_filter[q] (< n_filters).
 * Filter f is the ascending, unique staged rows filter_rows[filter_offsets[f] .. filter_offsets[f+1]).
 * Several queries may share a filter; unused filters are allowed. Row q of the outputs equals
 * arroy_b200_search_batch_filtered(..., bitmap of filter query_filter[q], ...) for that query alone, and out_status keeps
 * its meaning. The filters the queries use are summarised 32 per pass over the forest's descendant lists; a filter whose rows
 * in the forest number at most search_k answers its queries without a walk. Counted in arroy_b200_search_stats like the
 * one-filter queries. A query_filter >= n_filters, n_filters == 0 with nq > 0, decreasing offsets, a row >= n or rows not
 * strictly ascending within a filter are argument errors. */
int32_t arroy_b200_search_batch_multi_filtered(arroy_ctx* ctx, uint32_t nq, const uint32_t* query_rows, const float* queries,
                                               const float* qhdr0, uint64_t count, uint64_t search_k, uint32_t n_filters,
                                               const uint64_t* filter_offsets, const uint32_t* filter_rows, const uint32_t* query_filter,
                                               uint32_t* out_rows, float* out_dist, uint32_t* out_len, int32_t* out_status);
/* out[0] = filter-summary passes run by multi-filter calls since create, out[1] = filters summarised */
int32_t arroy_b200_multi_filter_stats(arroy_ctx* ctx, uint64_t out[2]);

/* ---- synthetic data + timing helpers (bench / tests; not part of the reference seam) ---- */

/* Fill a device matrix (rows x dim f32, dense) with element (i,j) = n-th gen::<f32>() of
 * StdRng::from_seed(seed), n = (row0+i)*dim + j, minus `centre` (SURVEY.md §8d). */
int32_t arroy_b200_synth_device(arroy_ctx* ctx, const uint8_t seed[32], uint32_t dim, uint64_t row0,
                                uint64_t rows, float centre, void* device_out);

/* Time `iters` launches of the side()/margin scan kernel over `n_rows` staged rows
 * (rows == NULL: rows 0..n_rows-1) with CUDA events on the library's stream; optional
 * L2 flush between launches. Returns the average milliseconds per launch. Results stay on
 * the device (this measures the kernel, not the boundary). variant 0: the f32 scan
 * (work_kernel); variant 1: the build's 8-bit pre-filter (work_kernel_planes, every unit
 * through the planes; float metrics, 64 <= dim <= 8192), whose stage counts of the last
 * launch arroy_b200_build_prefilter_stats then reports. */
int32_t arroy_b200_time_scan(arroy_ctx* ctx, const float* normal, float hdr0, float hdr1,
                             const uint32_t* rows, uint64_t n_rows, int32_t variant, int32_t iters,
                             int32_t flush_l2, float* out_ms_avg, uint64_t* out_left_count);

/* A ready-made thread-safe node sink: an append-only arena, the in-memory counterpart of the
 * reference's per-thread TmpNodes files (src/parallel.rs:22-147). Pass arroy_b200_arena_sink
 * as `sink` and the arena as `sink_arg`. */
typedef struct arroy_b200_arena arroy_b200_arena;
arroy_b200_arena* arroy_b200_arena_new(void);
void arroy_b200_arena_free(arroy_b200_arena* arena);
void arroy_b200_arena_clear(arroy_b200_arena* arena);
int32_t arroy_b200_arena_sink(void* arena, uint32_t node_id, const uint8_t* bytes, uint64_t len);
/* returns the number of nodes held; *out_total_bytes = sum of their lengths */
uint64_t arroy_b200_arena_stats(arroy_b200_arena* arena, uint64_t* out_total_bytes);
int32_t arroy_b200_arena_get(arroy_b200_arena* arena, uint32_t node_id, const uint8_t** out_bytes, uint64_t* out_len);

/* Host-side wall-clock breakdown of the last build (ms): [0] buffer setup + tree init,
 * [1] CUDA graph capture + instantiate, [2] device step loop, [3] read-back after the kernels (tree states, pool fill,
 * pre-filter counters; the results themselves reach host memory while the wave builds),
 * [4] NodeCodec encoding + sink calls, [5] graph launches (count), [6] the schedules the build's
 * waves ran, one bit each, OR-ed over the waves: 1 persistent (one cooperative launch per wave),
 * 2 lockstep, 4 async CUDA graph with one control CTA per tree, 8 / 16 async with a thread-block
 * cluster of 8 / 16 control CTAs per tree, 32 two_means workspace in global memory (rows wider
 * than 3648 floats), 64 speculative two_means; [7] normal pool slots copied after the kernels because
 * the host pool had no room for them (count; ARROY_B200_EXPORT_SLOTS). */
int32_t arroy_b200_build_breakdown(arroy_ctx* ctx, double out[8]);

/* Counters since arroy_b200_create: out[0] = kernel launches issued by this library,
 * out[1] = bytes copied host->device, out[2] = bytes copied device->host (builds: including what the kernels write to
 * host memory), out[3] = (query batches re-ranked by
 * the fused bf16-pre-filter kernel << 32) | batches that fell back to the plain distance + top-k kernels. */
int32_t arroy_b200_counters(arroy_ctx* ctx, uint64_t out[4]);

/* The plane pre-filter of host-placed indexes' re-rank, counted since arroy_b200_create. Batched searches and re-ranks of an
 * index whose f32 rows are in host memory (arroy_b200_item_placement) estimate every candidate from the build's 8-bit planes on
 * the device, with a proven error bound, and re-score only the rows that can still reach the top-k from the host rows (in the
 * reference's order: results are identical). out[0] = query batches that went through it, out[1] = of those, batches that fell
 * back to the plain kernels (a query with more than 8192 candidates or 2048 survivors; such a batch reads all its candidates
 * from host memory again), out[2] = candidate rows estimated from the planes, out[3] = rows it re-scored from the f32 rows, i.e.
 * read from host memory. ARROY_B200_FRERANK=0 turns it off. Device-placed indexes leave all four at 0. */
int32_t arroy_b200_plane_rerank_stats(arroy_ctx* ctx, uint64_t out[4]);

/* The score matrix of the pre-filter, for tests and profiling: out_scores[q * n_rows + i] ~ dot(query q,
 * item rows[i]) computed with TF32 inputs and FP32 accumulation on the tensor cores; guaranteed within
 * 2^-8 * |q| * |item| of the exact dot product. engine 0 = the library's wgmma kernel, 1 = cuBLAS.
 * Needs dim >= 32. */
int32_t arroy_b200_prefilter_scores(arroy_ctx* ctx, uint32_t nq, const float* queries /* nq x dim */,
                                    const uint32_t* rows, uint64_t n_rows, int32_t engine, float* out_scores);

/* Pre-filter statistics of arroy_b200_rerank_shared since create: out[0] = query chunks that went
 * through the tensor-core pre-filter, out[1] = chunks that fell back to the exact dense kernel
 * (more survivors than the per-query cap), out[2] = survivors re-scored exactly (sum over
 * queries), out[3] = queries pre-filtered. */
int32_t arroy_b200_rerank_stats(arroy_ctx* ctx, uint64_t out[4]);

/* CUDA-event breakdown of the last arroy_b200_search_batch call (ms, summed over its query chunks):
 * [0] bitmap clear + tree walk, [1] candidate sort, [2] distances, [3] top-k, [4] reserved; after a multi-filter call also
 * [5] filter upload + row masks, [6] filter summaries (both summed over its filter sets); [7] reserved. */
int32_t arroy_b200_search_breakdown(arroy_ctx* ctx, double out[8]);

/* CUDA-event breakdown of the last arroy_b200_rerank_shared call (ms, summed over its query chunks):
 * [0] norms + bound constants, [1] score contraction on the tensor cores (tcgemm_tf32_kernel),
 * [2] threshold selection, [3] exact re-score of the survivors, [4] top-k, [5] exact dense kernel +
 * top-k (chunks that did not go through the pre-filter), [6..7] reserved. */
int32_t arroy_b200_rerank_breakdown(arroy_ctx* ctx, double out[8]);

/* CUDA-event stopwatch on the library's own stream (the stream every kernel above is launched
 * on): start records an event after draining the stream, stop records a second one, waits for
 * it and returns the elapsed milliseconds between the two. */
int32_t arroy_b200_timer_start(arroy_ctx* ctx);
int32_t arroy_b200_timer_stop(arroy_ctx* ctx, float* out_ms);

/* Self-test of the library's branch-free f32 division (used inside create_split / two_means for x / norm and x / count, which
 * the reference computes with IEEE division — src/distance/mod.rs:86-94, :76-82): n_groups x 4 quotients over every operand
 * class against div.rn.f32; *out_mismatches must come back 0. out_fallbacks = groups that took the div.rn path. */
int32_t arroy_b200_selftest_udiv(arroy_ctx* ctx, uint64_t n_groups, uint64_t seed, uint64_t* out_mismatches, uint64_t* out_fallbacks);

/* BinaryQuantized::from_slice + ::iter of one vector (host helper, no device): out[i] = is_sign_positive(in[i]) ? 1 : -1 for
 * i < dims, -1 up to the next multiple of 64. Returns that padded length; in / out may be NULL to query it. */
uint32_t arroy_b200_bq_quantize(const float* in, uint32_t dims, float* out);

/* Ownership tokens of the device-resident state, for callers that share one context between several
 * readers / writers (the host keeps one context per heed::Env): out[0] = epoch of the staged items,
 * out[1] = epoch of the loaded forest; each is bumped by every arroy_b200_stage_items* /
 * arroy_b200_load_forest call and reads 0 while nothing valid is resident (stage epochs are not reused by another context of
 * the process). A caller remembers the
 * epochs it produced and re-stages / re-loads when they differ, instead of trusting state another
 * owner has replaced. */
int32_t arroy_b200_epochs(arroy_ctx* ctx, uint64_t out[2]);

/* Raw device pointers of the staged items (for the NCCL broadcast of the multi-GPU path):
 * out[0] = float[n][ld] matrix, out[1] = hdr0[n], out[2] = hdr1[n] (may be 0); *out_ld = ld. Binary-quantized metrics: the
 * rows are bit strings of 16 * ceil(dims / 128) bytes and *out_ld is that byte count / 4. Items placed in host memory
 * (arroy_b200_item_placement) have no device matrix: ARROY_B200_ERR_INVALID. */
int32_t arroy_b200_device_ptrs(arroy_ctx* ctx, void* out[3], uint32_t* out_ld);

/* ---- several GPUs of one node behind one handle (SURVEY.md §8b / §8e) -------------------------------------------------
 * Replaces the rayon scope of src/writer.rs:568-591 for hosts with more than one device: one process, one context per
 * device, NCCL (bound at run time) for the single data-path collective.
 *   create_group      one context per listed device + ncclCommInitAll; fails with ERR_CUDA if a device or NCCL is missing
 *   group_stage_items ImmutableLeafs::new for all devices: the leaf values are decoded and uploaded to devices[0] in ~256 MB
 *                     chunks and every chunk is handed to ncclBroadcast (root = devices[0]) while the next one is still
 *                     crossing PCIe; headers follow the same way
 *   group_build_trees arroy_b200_build_trees with tree t built by device t mod n_dev, all devices at the same time; node ids
 *                     and bytes are identical to a single-device build; the sink is called concurrently
 *   group_ctx         the member context of one device (for arroy_b200_build_stats, arroy_b200_rerank, ... on that device) */
typedef struct arroy_group arroy_group;
int32_t arroy_b200_create_group(int32_t n_dev, const int32_t* devices, arroy_group** out);
void arroy_b200_destroy_group(arroy_group* group);
const char* arroy_b200_group_last_error(arroy_group* group);
int32_t arroy_b200_group_size(arroy_group* group);
arroy_ctx* arroy_b200_group_ctx(arroy_group* group, int32_t rank);
int32_t arroy_b200_group_stage_items(arroy_group* group, int32_t metric, uint32_t dim, uint64_t n,
                                     const uint32_t* ids_ascending, const uint8_t* const* leaf_values);
int32_t arroy_b200_group_dot_preprocess(arroy_group* group, float* out_extra_dim /* n or NULL */, float* out_norm /* n or NULL */);
int32_t arroy_b200_group_build_trees(arroy_group* group, uint32_t n_trees, const uint8_t (*tree_seeds)[32],
                                     const uint32_t* root_ids, uint32_t first_free_node_id, uint32_t split_after,
                                     arroy_b200_cancel_fn cancel, void* cancel_arg,
                                     arroy_b200_node_sink sink, void* sink_arg, uint64_t* out_n_nodes);
/* wall-clock of the last group_stage_items (ms): [0] total, [1] tail after the last H2D chunk (headers + the one broadcast
 * that nothing hides), [2..3] reserved */
int32_t arroy_b200_group_stage_breakdown(arroy_group* group, double out[4]);

#ifdef __cplusplus
}
#endif
#endif /* ARROY_B200_H */
