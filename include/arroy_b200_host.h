/*
 * arroy_b200_host.h — C view of the C++ host mirror of arroy's public interface.
 *
 * The reference's host is Rust (Writer / ArroyBuilder / Reader / QueryBuilder over LMDB via
 * heed). Neither rustc nor liblmdb exist in this image, so the host side that sits above
 * the device boundary (include/arroy_b200.h) is restated in C++ inside the same shared
 * library, with the same names, argument meaning and error behaviour:
 *   Writer      src/writer.rs:268-485   (new, add_item, append_item, del_item, clear,
 *                                        need_build, contains_item, is_empty, item_vector, builder)
 *   ArroyBuilder src/writer.rs:126-265  (n_trees, split_after, available_memory, cancel, progress, build)
 *   Reader      src/reader.rs:138-298   (open, dimensions, n_trees, n_items, item_ids, item_vector, nns, stats)
 *   QueryBuilder src/reader.rs:26-124   (by_item, by_vector, search_k, oversampling, candidates)
 * LMDB is replaced by an ordered in-memory key/value table that stores the reference's
 * exact key and value BYTES (src/key.rs:56-83, src/node.rs:218-282, src/metadata.rs:21-61,
 * src/version.rs:39-49), so its content can be diffed against (or exported to) a real arroy
 * database. A maintainer of the Rust crate does NOT bind this file; it exists so that tests
 * and benchmarks exercise the path through the same operations a user of arroy performs.
 */
#ifndef ARROY_B200_HOST_H
#define ARROY_B200_HOST_H

#include <stddef.h>
#include <stdint.h>

#include "arroy_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

typedef struct arroy_env arroy_env;        /* stands in for heed::Env + Database<D> */
typedef struct arroy_writer arroy_writer;  /* arroy::Writer<D> */
typedef struct arroy_reader arroy_reader;  /* arroy::Reader<D> */
typedef struct arroy_rng arroy_rng;        /* rand::rngs::StdRng (ChaCha12) */

/* arroy::Error (src/error.rs:7-86); values < 100 are the device codes of arroy_b200.h */
enum {
    ARROY_ERR_INVALID_VEC_DIMENSION = 100,
    ARROY_ERR_DATABASE_FULL = 101,
    ARROY_ERR_INVALID_ITEM_APPEND = 102,
    ARROY_ERR_UNMATCHING_DISTANCE = 103,
    ARROY_ERR_MISSING_METADATA = 104,
    ARROY_ERR_NEED_BUILD = 105,
    ARROY_ERR_BUILD_CANCELLED = 106,
    ARROY_ERR_MISSING_KEY = 107,
    ARROY_ERR_UNKNOWN_VERSION = 108,
    ARROY_ERR_PANIC = 109
};

/* message of the last failing host call on this thread (Display of arroy::Error) */
const char* arroy_host_last_error(void);

/* ---- environment -------------------------------------------------------------------------- */
arroy_env* arroy_env_new(void);
void arroy_env_free(arroy_env* env);
uint64_t arroy_env_len(arroy_env* env);
/* iterate all (key, value) pairs in key order — what `database.iter()` yields in the tests */
typedef int32_t (*arroy_kv_sink)(void* arg, const uint8_t* key, uint64_t key_len, const uint8_t* val, uint64_t val_len);
int32_t arroy_env_iter(arroy_env* env, arroy_kv_sink sink, void* arg);

/* raw put of one (key, value) pair — importing the content of a real arroy LMDB file (keys are the 8 bytes of src/key.rs:56-68) */
int32_t arroy_env_put_raw(arroy_env* env, const uint8_t* key, uint64_t key_len, const uint8_t* val, uint64_t val_len);
/* decode a stored value with the library's decoders and encode it again with its encoders (what = 0: tree node, 1: Metadata);
 * used to pin the codecs (RoaringBitmap bytes included) against files written by the reference */
int32_t arroy_host_reencode(int32_t what, const uint8_t* in, uint64_t len, uint8_t* out, uint64_t cap, uint64_t* out_len);

/* ---- StdRng -------------------------------------------------------------------------------- */
arroy_rng* arroy_rng_from_seed(const uint8_t seed[32]);
arroy_rng* arroy_rng_seed_from_u64(uint64_t state);
arroy_rng* arroy_rng_clone(const arroy_rng* rng);
void arroy_rng_free(arroy_rng* rng);
uint32_t arroy_rng_next_u32(arroy_rng* rng);
float arroy_rng_gen_f32(arroy_rng* rng);
void arroy_rng_fill_f32(arroy_rng* rng, float* out, uint64_t n);

/* ---- Writer -------------------------------------------------------------------------------- */
arroy_writer* arroy_writer_new(arroy_env* env, uint16_t index, uint32_t dimensions, int32_t metric);
void arroy_writer_free(arroy_writer* w);
int32_t arroy_writer_add_item(arroy_writer* w, uint32_t item, const float* vector, uint32_t len);
/* add_item in a loop over a dense matrix (n x dimensions) */
int32_t arroy_writer_add_items(arroy_writer* w, uint64_t n, const uint32_t* items, const float* vectors);
int32_t arroy_writer_append_item(arroy_writer* w, uint32_t item, const float* vector, uint32_t len);
int32_t arroy_writer_del_item(arroy_writer* w, uint32_t item, int32_t* out_existed);
int32_t arroy_writer_clear(arroy_writer* w);
int32_t arroy_writer_need_build(arroy_writer* w, int32_t* out);
int32_t arroy_writer_contains_item(arroy_writer* w, uint32_t item, int32_t* out);
int32_t arroy_writer_is_empty(arroy_writer* w, int32_t* out);
int32_t arroy_writer_item_vector(arroy_writer* w, uint32_t item, float* out /* dimensions */, int32_t* out_found);

/* ArroyBuilder::build. n_trees < 0 = not set (target_n_trees formula, src/writer.rs:1358-1394);
 * split_after 0 = not set; available_memory UINT64_MAX = not set. With a value, trees whose items do not "fit"
 * (fit_in_memory, src/writer.rs:1536-1584) are built the way the reference builds them — a sampled chunk becomes a tree, the
 * rest is routed through it, oversized leaves become new tasks (src/writer.rs:660-844) — so the forest equals the one the
 * reference produces with the same setting on a 1-thread pool; the items stay resident in HBM regardless. progress receives
 * the MainStep name (src/writer.rs:44-70). */
typedef void (*arroy_progress_fn)(void* arg, const char* main_step);
int32_t arroy_writer_build(arroy_writer* w, arroy_ctx* ctx, arroy_rng* rng, int64_t n_trees, uint64_t split_after,
                           uint64_t available_memory, arroy_b200_cancel_fn cancel, void* cancel_arg,
                           arroy_progress_fn progress, void* progress_arg);
/* timing breakdown of the last build (ms): [0] stage (decode + H2D) [1] preprocess [2] device build
 * + node emission [3] metadata [4] total; [5] bytes H2D; [6] bytes D2H-ish (node bytes emitted) */
int32_t arroy_writer_build_timings(arroy_writer* w, double out[8]);

/* ---- Reader -------------------------------------------------------------------------------- */
int32_t arroy_reader_open(arroy_env* env, uint16_t index, int32_t metric, arroy_ctx* ctx, arroy_reader** out);
void arroy_reader_free(arroy_reader* r);
uint32_t arroy_reader_dimensions(arroy_reader* r);
uint64_t arroy_reader_n_trees(arroy_reader* r);
uint64_t arroy_reader_n_items(arroy_reader* r);
/* out may be NULL to query the count */
uint64_t arroy_reader_item_ids(arroy_reader* r, uint32_t* out, uint64_t cap);
int32_t arroy_reader_item_vector(arroy_reader* r, uint32_t item, float* out, int32_t* out_found);
/* TreeStats per root: depth, dummy_normals, split_nodes, descendants (src/reader.rs:210-252) */
int32_t arroy_reader_stats(arroy_reader* r, uint64_t* out /* 4 x n_trees */);

/* QueryBuilder. search_k / oversampling 0 = not set; candidates NULL (n_candidates < 0) = none.
 * by_item: *out_found = 0 mirrors Ok(None). Results: (item id, normalized distance) ascending. */
int32_t arroy_reader_nns_by_item(arroy_reader* r, uint32_t item, uint64_t count, uint64_t search_k, uint64_t oversampling,
                                 const uint32_t* candidates, int64_t n_candidates,
                                 uint32_t* out_ids, float* out_dist, uint64_t* out_len, int32_t* out_found);
int32_t arroy_reader_nns_by_vector(arroy_reader* r, const float* vector, uint32_t len, uint64_t count, uint64_t search_k,
                                   uint64_t oversampling, const uint32_t* candidates, int64_t n_candidates,
                                   uint32_t* out_ids, float* out_dist, uint64_t* out_len);
/* Many queries in one call (not in the reference, which has no batching API): exactly one of items (by_item, nq ids) and
 * vectors (by_vector, nq x dimensions) is given, and one optional candidates filter (NULL / n_candidates < 0 = none) applies to
 * every query. The walks, candidate sort and re-rank run on the device (arroy_b200_search_batch / _filtered); queries the
 * device walk gives up on, count > 2048 or ARROY_B200_HOST_WALK=1 take the host walk and one batched device re-rank.
 * out_* are nq x count; each row equals the single query with the same settings. */
int32_t arroy_reader_nns_batch(arroy_reader* r, uint32_t nq, const uint32_t* items, const float* vectors, uint64_t count,
                               uint64_t search_k, uint64_t oversampling, const uint32_t* candidates, int64_t n_candidates,
                               uint32_t* out_ids, float* out_dist, uint32_t* out_len,
                               double* out_ms /* [0] tree walk [1] re-rank, may be NULL */);
/* arroy_reader_nns_batch with one candidates filter per query: query i uses filter query_filter[i] (< n_filters), the item ids
 * cand_ids[cand_offsets[f] .. cand_offsets[f+1]) (any order; duplicates and ids outside the index drop out, as in
 * QueryBuilder::candidates). Several queries may share a filter and unused filters are allowed. The device walks every query
 * with its own filter (arroy_b200_search_batch_multi_filtered); the host walk takes over as in arroy_reader_nns_batch, each query
 * with its own filter. Each row equals the single query with that filter. */
int32_t arroy_reader_nns_batch_multi(arroy_reader* r, uint32_t nq, const uint32_t* items, const float* vectors, uint64_t count,
                                     uint64_t search_k, uint64_t oversampling, uint32_t n_filters, const uint64_t* cand_offsets,
                                     const uint32_t* cand_ids, const uint32_t* query_filter, uint32_t* out_ids, float* out_dist,
                                     uint32_t* out_len, double* out_ms /* [0] tree walk [1] re-rank, may be NULL */);
/* arroy_reader_nns_batch with items and no filter */
int32_t arroy_reader_nns_batch_by_item(arroy_reader* r, uint32_t nq, const uint32_t* items, uint64_t count, uint64_t search_k,
                                       uint64_t oversampling, uint32_t* out_ids, float* out_dist, uint32_t* out_len,
                                       double* out_ms /* [0] tree walk [1] re-rank, may be NULL */);

#ifdef __cplusplus
}
#endif
#endif
