/*
 * wax_vs_cuda.h -- C-ABI of libwaxvs_cuda.so: the H100 (sm_90a) brute-force vector scan + top-k
 * that replaces WaxVectorSearch's Metal compute pipeline and CPU fallback behind the
 * `VectorSearchEngine` Swift protocol.
 *
 * Shape of the boundary.  Wax has no C-ABI for vector search; the seam is the Swift protocol
 *   Sources/WaxVectorSearch/VectorSearchEngine.swift:10-18
 * plus the concrete-type extras callers use (MetalVectorEngine.swift: init :153, isAvailable :144,
 * serialize :682, deserialize :716, addBatchStreaming :404).  Every entry point below is what a
 * `CUDAVectorEngine` Swift actor binds for one of those members; the cited line is the reference
 * member it replaces.  Conventions follow the repo's only FFI precedent, WaxCoreCompressionC
 * (Sources/WaxCoreCompressionC/include/wax_compression_shims.h:7-34): int32_t return code (0 = ok,
 * negative = distinct failure), caller-owned plain pointers + sizes, every pointer NULL-checked,
 * no ownership transfer.  INTEGRATION.md shows the Swift binding.
 *
 * Threading (mirrors the actor's AsyncReadWriteLock, MetalVectorEngine.swift:56-80): any number of
 * concurrent wax_vs_search* calls XOR one mutator (add/remove/reserve/deserialize/destroy).  The
 * library also enforces this internally with a reader/writer lock, so misuse blocks instead of racing.
 * search calls block the calling thread until results are in the caller's buffers.
 *
 * All arithmetic is IEEE fp32; ids are uint64; the corpus lives row-major in HBM.
 */
#ifndef WAX_VS_CUDA_H
#define WAX_VS_CUDA_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct wax_vs_engine wax_vs_engine; /* opaque: owns HBM, streams, scratch pool */

/* Return codes.  The Swift side maps them onto the WaxError cases the Metal engine throws. */
enum {
    WAX_VS_OK = 0,
    WAX_VS_ERR_NULL = -1,          /* NULL argument                         -> WaxError.invalidToc       */
    WAX_VS_ERR_DIMENSION = -2,     /* vector length != dimensions           -> WaxError.encodingError
                                      (MetalVectorEngine.swift:830-833, :360-370)                       */
    WAX_VS_ERR_CAPACITY = -3,      /* dims > 1 000 000 / rows > UInt32.max  -> WaxError.capacityExceeded
                                      (MetalVectorEngine.swift:157-162, :858-860)                       */
    WAX_VS_ERR_CUDA = -4,          /* device / allocation / launch failure  -> WaxError.invalidToc(reason:) */
    WAX_VS_ERR_FORMAT = -5,        /* malformed MV2V blob                   -> WaxError.invalidToc(reason:)
                                      (MetalVectorEngine.swift:718-808)                                 */
    WAX_VS_ERR_ARGUMENT = -6,      /* dims == 0, unknown similarity, ...    -> WaxError.invalidToc       */
    WAX_VS_ERR_BUFFER = -7,        /* caller buffer too small                                           */
    WAX_VS_ERR_UNSUPPORTED = -8    /* feature not available in this build                                */
};

/* VecSimilarity raw values (Sources/WaxCore/FileFormat/MV2SEnums.swift:34-38). */
enum { WAX_VS_COSINE = 0, WAX_VS_DOT = 1, WAX_VS_L2 = 2 };

#define WAX_VS_MAX_RESULTS 10000      /* MetalVectorEngine.swift:18 */
#define WAX_VS_MAX_DIMENSIONS 1000000 /* Sources/WaxCore/Constants.swift:51 */

/* One candidate of the device-side result list (sharded search: what a rank contributes to the
   NCCL all-gather, SURVEY.md section 8e).  24 bytes, naturally aligned. */
typedef struct wax_vs_candidate {
    float distance;     /* USearch-convention distance (ascending = better)                        */
    uint32_t valid;     /* 1 = real candidate, 0 = padding (fewer than k finite candidates)        */
    uint64_t row;       /* global row = row_offset + local row or row key: the cross-shard tie-break */
    uint64_t frame_id;
} wax_vs_candidate;

/* ---- availability / lifetime ---------------------------------------------------------------- */

/* MetalVectorEngine.isAvailable (MetalVectorEngine.swift:144-146): available <=> rc == 0 && *out > 0. */
int32_t wax_vs_device_count(int32_t *out);

/* MetalVectorEngine.init(metric:dimensions:) (MetalVectorEngine.swift:153-274).  Unlike the Metal
   engine (cosine only, :163-165) all three metrics are supported, with USearchVectorEngine's
   semantics (USearchVectorEngine.swift:44-67; VectorMetric.swift:21-30).  `devices`/`n_devices`: the
   CUDA ordinals to use; NULL/0 = current device, 1 = that device.
   n_devices >= 2 returns a MULTI-DEVICE handle: the corpus sharded by rows over n_devices shards, shard r on devices[r]
   (DESIGN.md section 4.16).  Every answer it gives equals that of one engine with the same call history, bit for bit:
   ids, order, score bits, counts, MV2V bytes, error codes and reasons.  It serves wax_vs_dimensions, _similarity,
   _count, _reserve, _add, _add_batch, _remove, _remove_batch, _rebalance, _search, _search_batch, _search_filtered,
   _search_batch_filtered, _search_batch_multi_filtered, _set_attributes, _set_locations, _set_terms,
   _search_batch_where, _where_near, _where_terms, _where_groups, _where_roots, _set_groups, _set_root_tags, _search_grouped,
   _search_batch_grouped, _grouped_where, _grouped_where_near, _grouped_multi_where, _grouped_multi_where_groups,
   _grouped_multi_where_roots, _serialized_length, _serialize, _deserialize, wax_vs_debug_set_option
   (applied to every shard) and wax_vs_debug_counter (summed over the shards, plus "shard_rows.<r>": shard r's rows);
   every other entry point (the rank-level shard_*, *_device, keyed, export, absorb and merge entries, the other debug_*) returns
   WAX_VS_ERR_UNSUPPORTED naming itself.  Grouped search with clamp(top_groups) > WAX_VS_SHARD_MAX_GROUPS is refused as
   the sharded grouped form refuses it.  An ordinal
   may repeat ({0, 0, 0}): the shards then share that device, a test and debug configuration.  Checked before any
   device query: n_devices > WAX_VS_SHARD_MAX_RANKS or a negative ordinal -> WAX_VS_ERR_ARGUMENT, NULL devices ->
   WAX_VS_ERR_NULL.  Two distinct devices that cannot access each other's memory -> WAX_VS_ERR_UNSUPPORTED.
   Multi-process and multi-node sharding is one engine per rank + wax_vs_search_device + one all-gather
   (wax_b200/sharded.py). */
int32_t wax_vs_create(uint32_t dimensions, uint8_t similarity, const int32_t *devices, int32_t n_devices,
                      wax_vs_engine **out);
void wax_vs_destroy(wax_vs_engine *engine);

/* `dimensions` property of the protocol (VectorSearchEngine.swift:11). */
int32_t wax_vs_dimensions(const wax_vs_engine *engine, uint32_t *out);
int32_t wax_vs_similarity(const wax_vs_engine *engine, uint8_t *out);
/* vectorCount (MetalVectorEngine.swift:50). */
int32_t wax_vs_count(wax_vs_engine *engine, uint64_t *out);

/* ---- corpus mutation -------------------------------------------------------------------------- */

/* reserveIfNeeded (MetalVectorEngine.swift:857-871): make room for `rows` rows in HBM. */
int32_t wax_vs_reserve(wax_vs_engine *engine, uint64_t rows);

/* add(frameId:vector:) (MetalVectorEngine.swift:330-357): upsert one row. `vector_len` must equal
   dimensions (validate, :830-833). */
int32_t wax_vs_add(wax_vs_engine *engine, uint64_t frame_id, const float *vector, uint32_t vector_len);

/* Bulk transfers (add_batch, deserialize, serialize) move caller memory through two pinned staging buffers with the
   host-side copy of one chunk overlapping the DMA of the other, so PAGEABLE caller buffers still reach PCIe speed;
   caller memory that is already pinned is handed to the DMA engine directly. */
/* addBatch(frameIds:vectors:) (MetalVectorEngine.swift:359-402): upsert n rows, `rows` is n x dims
   row-major (the Swift side flattens [[Float]]).  An id already present is overwritten in place
   (:385-389), a new id is appended at row N (:390-397); later duplicates inside one batch overwrite
   earlier ones, as the reference's sequential loop does.  n == 0 is a no-op (:360). */
int32_t wax_vs_add_batch(wax_vs_engine *engine, const uint64_t *frame_ids, const float *rows, uint64_t n,
                         uint32_t vector_len);

/* remove(frameId:) (MetalVectorEngine.swift:423-444): unknown id / empty engine = no-op rc 0 (:425-426);
   known id: row deleted, later rows keep their relative order (:431-441). */
int32_t wax_vs_remove(wax_vs_engine *engine, uint64_t frame_id);

/* remove(frameId:) for n frames in ONE pass (SURVEY.md section 8f-3; the reference memmoves the whole tail once per id,
   MetalVectorEngine.swift:431-441): same result as n calls of wax_vs_remove in any order -- unknown / repeated ids
   are ignored, surviving rows keep their relative order -- with one compaction of the matrix in HBM, one compaction
   of the id array and one id->row hash rebuild.  *out_removed (optional) = rows actually deleted. */
int32_t wax_vs_remove_batch(wax_vs_engine *engine, const uint64_t *frame_ids, uint64_t n, uint64_t *out_removed);

/* Even out the rows of a multi-device handle's shards, in place.  *out_moved (optional) = rows moved.
   A mutator (DESIGN.md section 4.16): every shard ends with T / R or T / R + 1 of the T rows, the extra ones on the shards
   that held the most, and each moved row takes its key, group, attributes, location and terms with it.  Nothing the
   handle serves changes except "shard_rows.<r>": every answer still equals one engine's with the same call history, and
   a later upsert or remove of a moved frame finds it where it now lives.  A balanced handle (max - min <= 1) moves
   nothing and touches no shard.  One engine (n_devices <= 1) returns WAX_VS_OK with *out_moved = 0.  A failed
   allocation (a receiving shard's growth, the staging) is found before that shard's rows change: WAX_VS_ERR_CUDA, every
   earlier move complete, no row held twice or lost.  The merge works in slabs of the option "rebalance_slab_bytes"
   (wax_vs_debug_set_option, default 256 MiB). */
int32_t wax_vs_rebalance(wax_vs_engine *engine, uint64_t *out_moved);

/* ---- row keys: the rank-local store of the row-sharded engine (DESIGN.md section 4.15) ------------------------------
   A keyed engine holds one u64 key per row, the row's insertion sequence number in the whole sharded corpus; keys
   strictly increase with the row.  The device entry points (wax_vs_search_device and every entry below it that takes a
   row_offset or reports global rows) report row r as row_offset + key[r], so the ranks' candidates merge in the single
   engine's position order wherever each row lives.  An engine becomes keyed by wax_vs_add_batch_keyed or
   wax_vs_deserialize_rows; until then row r's key is r and everything behaves as before.  wax_vs_deserialize and
   wax_vs_debug_fill_synthetic drop the keys.  On a keyed engine wax_vs_add_batch gives appended rows the keys after the
   last one, an upsert keeps its row's key and wax_vs_remove_batch keeps the survivors' keys. */
/* wax_vs_add_batch whose appended rows take the keys first_key, first_key + 1, ... in order of first appearance.
   first_key not above the last row's key -> WAX_VS_ERR_ARGUMENT, before anything changes.  *out_appended (optional) =
   rows appended (the batch's distinct new ids). */
int32_t wax_vs_add_batch_keyed(wax_vs_engine *engine, const uint64_t *frame_ids, const float *rows, uint64_t n,
                               uint32_t vector_len, uint64_t first_key, uint64_t *out_appended);
/* out[i] = 1 when the engine holds frame_ids[i], else 0. */
int32_t wax_vs_contains(wax_vs_engine *engine, const uint64_t *frame_ids, uint64_t n, uint8_t *out);
/* Replace the contents with rows [first, first + n) of an MV2V blob, keyed first, first + 1, ...  The blob is checked
   exactly as wax_vs_deserialize checks it (same codes and reasons); a row range outside it -> WAX_VS_ERR_ARGUMENT. */
int32_t wax_vs_deserialize_rows(wax_vs_engine *engine, const uint8_t *src, uint64_t len, uint64_t first, uint64_t n);
/* Copy rows [first, first + n) out: frame ids, vectors (n x dims) and keys (r for an engine without keys).  Each output
   may be NULL.  A range outside the rows -> WAX_VS_ERR_ARGUMENT. */
int32_t wax_vs_export_rows(wax_vs_engine *engine, uint64_t first, uint64_t n, uint64_t *out_ids, float *out_vectors,
                           uint64_t *out_keys);

/* The rank-level halves of a rebalance of the multi-process engine (ShardedVectorEngine.rebalance, DESIGN.md section
   4.15): a donor exports a run of its rows with their side columns, the receiver merges them by key.  The donor then
   drops the rows with wax_vs_remove_batch of their ids. */
/* Copy the vectors of rows [first, first + n) device-to-device into d_out (n x dims fp32 on the engine's device),
   enqueued on cuda_stream (NULL = the legacy default stream): NCCL can send them from there without a host bounce.  A
   later mutator of the engine waits for the copy.  A range outside the rows -> WAX_VS_ERR_ARGUMENT (as
   wax_vs_export_rows); n == 0 is a no-op; d_out NULL -> WAX_VS_ERR_NULL. */
int32_t wax_vs_export_rows_device(wax_vs_engine *engine, uint64_t first, uint64_t n, float *d_out, void *cuda_stream);

/* One row's side columns (32 bytes): its group, its attributes and its location bins (lat_bin == WAX_VS_NO_LOCATION:
   none, lon_bin 0). */
typedef struct wax_vs_row_columns {
    uint64_t group;
    int64_t timestamp;
    uint64_t tags;
    int32_t lat_bin;
    int32_t lon_bin;
} wax_vs_row_columns;
#define WAX_VS_NO_LOCATION (-2147483647 - 1)
/* Bits of the columns an engine holds (set_groups, set_attributes, set_locations, set_terms have been called). */
#define WAX_VS_COLUMN_GROUPS 1u
#define WAX_VS_COLUMN_ATTRIBUTES 2u
#define WAX_VS_COLUMN_LOCATIONS 4u
#define WAX_VS_COLUMN_TERMS 8u

/* The side columns of rows [first, first + n): out_columns[n] each row's group, attributes and location; the term
   lists as out_term_offsets[n + 1] (from 0) into out_terms; *out_terms_len = the number of term ids in the rows (call
   with out_terms NULL to size the buffer first); *out_set = the WAX_VS_COLUMN_* bits of the columns this engine holds.
   A column the engine does not hold is exported as the defaults its rows answer with: group = own frame id,
   attributes {0, 0}, no location, no terms.  Every output may be NULL.  Ids and keys come from wax_vs_export_rows.
   A range outside the rows -> WAX_VS_ERR_ARGUMENT (as wax_vs_export_rows); out_terms with terms_cap below the term
   ids -> WAX_VS_ERR_BUFFER. */
int32_t wax_vs_export_columns(wax_vs_engine *engine, uint64_t first, uint64_t n, wax_vs_row_columns *out_columns,
                              uint64_t *out_term_offsets, uint64_t *out_terms, uint64_t terms_cap, uint64_t *out_terms_len,
                              uint32_t *out_set);

/* Merge n rows into the engine by key: frame_ids[n], keys[n] (strictly increasing), d_vectors (n x dims fp32 on the
   engine's device, complete when the call is made) and the side columns as wax_vs_export_columns gives them:
   columns_set = the WAX_VS_COLUMN_* bits the source held, columns[n] (needed with the group, attribute or location
   bit), term_offsets[n + 1] and terms (needed with the terms bit).  Every answer afterwards is that of an engine whose
   rows, in key order, are its own and the incoming ones.  A column set on one side only is filled with the defaults
   the other side's rows answered with; term lists are appended to the engine's term pool.  The merge works in slabs of
   the option "rebalance_slab_bytes" written top-down, so it rewrites the rows above the first incoming key; every
   allocation comes before a row changes (a failed one -> WAX_VS_ERR_CUDA, the engine untouched).  The row caches from
   the first incoming key on are rebuilt by the next search that needs them.  Checked before anything changes, ->
   WAX_VS_ERR_ARGUMENT with a reason: keys that do not strictly increase, a key or a frame id the engine already holds,
   a frame id given twice, an engine that holds rows without keys, unknown column bits, term offsets that decrease or
   a row's terms that do not strictly increase, d_vectors not device memory on the engine's device.  NULL pointers ->
   WAX_VS_ERR_NULL.  n == 0 is a no-op. */
int32_t wax_vs_absorb_rows(wax_vs_engine *engine, const uint64_t *frame_ids, const uint64_t *keys, const float *d_vectors,
                           uint64_t n, uint32_t columns_set, const wax_vs_row_columns *columns,
                           const uint64_t *term_offsets, const uint64_t *terms);

/* ---- search ------------------------------------------------------------------------------------- */

/* search(vector:topK:) (VectorSearchEngine.swift:13; MetalVectorEngine.swift:446-627;
   USearchVectorEngine.swift:201-216).
     - empty engine: *out_n = 0, rc 0 (:448)
     - query_len != dimensions: WAX_VS_ERR_DIMENSION before any work (:449)
     - top_k clamped to [1, 10000] (:450, :842-846); returns min(k, N) rows minus non-finite (:597)
     - best first: ascending distance, ties by ascending row (the reference leaves ties unspecified)
     - out_scores[i] = VectorMetric.score(fromDistance:) (VectorMetric.swift:32-43):
         cosine 1 - d with d = 1 - q.v/(|q||v|), ALWAYS divided by the in-kernel |q|;
         dot -(1 - q.v);  l2 -sum (q-v)^2
   out_ids / out_scores need room for out_cap entries, out_cap >= min(clamp(top_k), N) else
   WAX_VS_ERR_BUFFER.
   Cosine / dot with k <= 32 on a corpus of at least 512 MiB (fp32) first nominate on the engine's bf16 copy of the
   corpus (half the bytes), re-score the nominees exactly and prove the result; the fp32 scan answers only when that
   proof fails.  Results are the fp32 scan's either way. */
int32_t wax_vs_search(wax_vs_engine *engine, const float *query, uint32_t query_len, int64_t top_k,
                      uint64_t *out_ids, float *out_scores, uint32_t out_cap, uint32_t *out_n);

/* n_queries independent searches (batched form of the above; results of query i start at out_ids[i*out_stride],
   count out_n[i]).  out_stride >= min(clamp(top_k), N).  Eligible batches share one tensor-core pass over the corpus
   (results identical to n_queries calls of wax_vs_search): cosine and dot, and l2 when the option "batch_l2" is 1
   (wax_vs_debug_set_option; default 0 for now), with dims % 32 == 0 and dims <= 8192, at least "batch_min" queries
   (default 4) and k <= 128 (up to 1024 when the corpus holds at least 64 x k rows).  Other batches run one exact scan
   per query. */
int32_t wax_vs_search_batch(wax_vs_engine *engine, const float *queries, uint32_t n_queries,
                            uint32_t query_len, int64_t top_k, uint64_t *out_ids, float *out_scores,
                            uint32_t out_stride, uint32_t *out_n);

/* Filtered search -- SURVEY.md section 8(f) rank 4, an API EXTENSION over the reference: Wax filters frames
   after the engine call and over-fetches 3 x topK to compensate (UnifiedSearch.swift:58, :371-442, :1195-1200,
   :1241-1258).  Here the filter is applied below the top-k, so exactly min(clamp(top_k), #allowed) best
   allowed rows come back.  mode 0: only rows whose frameId is in frame_ids[] may be returned (allow-list);
   mode 1: rows whose frameId is in frame_ids[] are excluded (deny-list, e.g. deleted / superseded frames).
   Unknown ids are ignored.  Same ordering, scoring and error behaviour as wax_vs_search. */
int32_t wax_vs_search_filtered(wax_vs_engine *engine, const float *query, uint32_t query_len, int64_t top_k,
                               const uint64_t *frame_ids, uint64_t n_ids, int32_t mode, uint64_t *out_ids,
                               float *out_scores, uint32_t out_cap, uint32_t *out_n);

/* The batched form: ONE filter, n_queries queries, one pass over the corpus (results of query i start at
   out_ids[i*out_stride], count out_n[i]; out_stride >= min(clamp(top_k), #allowed)).  Allow-lists of <= 16 384 rows
   score only the listed rows; otherwise the row filter rides below the top-k of the tensor-core levels (nominations,
   filter level and the exact fall-back consult the same bitset) or of the fused scan.  Results are identical to
   n_queries calls of wax_vs_search_filtered. */
int32_t wax_vs_search_batch_filtered(wax_vs_engine *engine, const float *queries, uint32_t n_queries,
                                     uint32_t query_len, int64_t top_k, const uint64_t *frame_ids, uint64_t n_ids,
                                     int32_t mode, uint64_t *out_ids, float *out_scores, uint32_t out_stride,
                                     uint32_t *out_n);

/* The batched form with one filter PER QUERY (a server batching requests that each carry their own frame filter):
   query i searches under filter query_filter[i], or unfiltered for WAX_VS_NO_FILTER.  Filter f is the ids
   frame_ids[filter_offsets[f] .. filter_offsets[f+1]) with mode filter_modes[f] (0 allow-list, 1 deny-list);
   filters no query references are not resolved.  Results of query i start at out_ids[i*out_stride], count out_n[i];
   out_stride >= max_i min(clamp(top_k), #allowed_i) (else WAX_VS_ERR_BUFFER).  Query i's answer is identical to
   wax_vs_search_filtered under its filter (wax_vs_search when unfiltered): same ids, same order, same score bits.
   Routing: allow-lists of <= 16 384 rows score only their listed rows (one batched gather for all such queries);
   queries whose filter allows at least clamp(top_k) rows share the tensor-core levels (or a masked fused scan each),
   every query consulting its own row bitset; the rest (deny-lists leaving fewer than k rows) scan one by one.  The
   bitsets are built on the device from the resolved rows; one tensor pass holds at most the option
   "filter_bitset_bytes" of them (default 2 GiB, one bitset is ceil(N/32) * 4 bytes), more filters run in several
   sub-batches (counter "filter_bitset_passes").  Arguments are checked before the empty-engine early return:
   WAX_VS_ERR_ARGUMENT for a mode other than 0 / 1, filter_offsets[0] != 0, decreasing offsets, or a query_filter
   entry >= n_filters other than WAX_VS_NO_FILTER; WAX_VS_ERR_NULL for a NULL array (frame_ids may be NULL when
   filter_offsets[n_filters] == 0, filter_modes when n_filters == 0).  Unknown and repeated ids are ignored. */
#define WAX_VS_NO_FILTER 0xFFFFFFFFu
int32_t wax_vs_search_batch_multi_filtered(wax_vs_engine *engine, const float *queries, uint32_t n_queries,
                                           uint32_t query_len, int64_t top_k, const uint64_t *frame_ids,
                                           const uint64_t *filter_offsets, const int32_t *filter_modes,
                                           uint32_t n_filters, const uint32_t *query_filter, uint64_t *out_ids,
                                           float *out_scores, uint32_t out_stride, uint32_t *out_n);

/* ---- grouped search: the best frames of the best groups (API EXTENSION over the reference) -------------------------
   Wax's PhotoRAG and VideoRAG answer with the best PHOTOS / VIDEOS, each a root frame plus derived frames (regions, OCR,
   captions, segments) with their own embeddings.  They over-fetch frames and group the hits on the host:
   PhotoRAG searches topK = max(resultLimit, searchTopK = 200) (PhotoRAGOrchestrator.swift:244-257, PhotoRAGConfig.swift:74,78)
   and keeps the best score per parentId ?? id (:264-308); VideoRAG fetches max(400, resultLimit x segmentLimitPerVideo x 8)
   frames (VideoRAGOrchestrator.swift:252), groups them by root (:273-350) and keeps segmentLimitPerVideo segments per
   video (VideoRAGTypes.swift:64-65; :406-440).  That over-fetch can return fewer groups than asked, or miss a group's
   rows.  wax_vs_search_grouped is exact.

   Groups: a row's group id is the id last given to its frame by wax_vs_set_groups, else the frame's own id -- so a root
   frame left unset and its derived frames set to the root's id form one group (Wax's parentId ?? id).  Groups follow
   their rows: an appended frame is its own group, an upsert keeps the frame's group, removes drop it.  MV2V has no place
   for groups: wax_vs_deserialize and wax_vs_debug_fill_synthetic reset every row to its own group, and the caller
   re-applies the grouping from its frame metadata (parentId) after loading. */
#define WAX_VS_MAX_PER_GROUP 128
/* Assign frames to groups (upsert): frame_ids[i] -> group_ids[i]; unknown frame ids are ignored, a later entry for the
   same frame wins; *out_assigned (optional) = rows whose group was written.  A mutator (write lock). */
int32_t wax_vs_set_groups(wax_vs_engine *engine, const uint64_t *frame_ids, const uint64_t *group_ids, uint64_t n,
                          uint64_t *out_assigned);
/* The best min(per_group, ...) frames of each of the clamp(top_groups) best groups, group-major.  The rows that take
   part are the allowed rows with a finite distance, ranked by (distance, row); a group ranks by its best row (ties
   between groups go to the lower row); the answer is the first min(clamp(top_groups), #groups taking part) groups, each
   with its min(per_group, its rows taking part) best rows, best first.  Scores as wax_vs_search, bit for bit.
   Filter as wax_vs_search_filtered; n_ids == 0 with mode 1 (deny nothing) = unfiltered.  out_groups[i] = group id of
   entry i.  out_cap >= min(clamp(top_groups) * per_group, N) else WAX_VS_ERR_BUFFER.  Checked before the empty-engine
   early return: per_group == 0, per_group > WAX_VS_MAX_PER_GROUP, clamp(top_groups) * per_group > WAX_VS_MAX_RESULTS or
   a mode other than 0 / 1 -> WAX_VS_ERR_ARGUMENT; a NULL output, or NULL frame_ids with n_ids > 0 -> WAX_VS_ERR_NULL.
   The first grouped search after a mutation or wax_vs_set_groups builds a device group index (at most 20 bytes per row,
   counter "group_index_builds"); later ones reuse it. */
int32_t wax_vs_search_grouped(wax_vs_engine *engine, const float *query, uint32_t query_len, int64_t top_groups,
                              uint32_t per_group, const uint64_t *frame_ids, uint64_t n_ids, int32_t mode,
                              uint64_t *out_ids, float *out_scores, uint64_t *out_groups, uint32_t out_cap,
                              uint32_t *out_n);

/* The batched form (a server batching PhotoRAG / VideoRAG requests): n_queries queries under ONE filter (as
   wax_vs_search_batch_filtered; n_ids == 0 with mode 1 = unfiltered).  Query i's answer is identical to
   wax_vs_search_grouped for that query alone -- same frame ids, group ids, order and score bits -- group-major at
   out_*[i * out_stride], count out_n[i]; out_stride >= min(clamp(top_groups) * per_group, N) else WAX_VS_ERR_BUFFER.
   Same argument checks as wax_vs_search_grouped, before the empty-engine early return; n_queries == 0 returns OK.
   How: each query's exact top-k_c rows, k_c = min(1024, max(128, 4 * clamp(top_groups))), come from the batched
   filtered search (the tensor-core levels, or the gather of a small allow-list).  A group ranks by its best row, so the
   first clamp(top_groups) distinct groups of that list are the top groups and their listed rows their best rows; a
   selected group with fewer listed rows than per_group is scored exactly over its own rows.  A query whose list names
   too few groups (one video's segments fill it) runs the single-query pipeline, as do whole batches the tensor-core
   levels do not take (small batches, dims % 32 != 0, l2 without the option "batch_l2", clamp(top_groups) > 256,
   deny-lists leaving fewer than k_c rows).  Counters: "grouped_batch_covered_queries", "grouped_batch_expanded_groups"
   ((query, group) pairs scored over the group's rows), "grouped_batch_fallback_queries". */
int32_t wax_vs_search_batch_grouped(wax_vs_engine *engine, const float *queries, uint32_t n_queries,
                                    uint32_t query_len, int64_t top_groups, uint32_t per_group,
                                    const uint64_t *frame_ids, uint64_t n_ids, int32_t mode, uint64_t *out_ids,
                                    float *out_scores, uint64_t *out_groups, uint32_t out_stride, uint32_t *out_n);

/* ---- frame attributes: time-range and tag predicates below the top-k (API EXTENSION over the reference) -------------
   Wax post-filters every hit in UnifiedSearch.passesFrameFilter (UnifiedSearch.swift:1241-1258): a timeRange
   (SearchRequest.swift:90-105; TimeRange.contains: after inclusive, before exclusive) and the includeDeleted /
   includeSuperseded / includeSurrogates flags; PhotoRAG and VideoRAG pass a timeRange into the same request
   (PhotoRAGOrchestrator.swift:238-252, VideoRAGOrchestrator.swift:226-261) and skip superseded and deleted frames by hand
   (:286, :318, :758).  Here each row carries a timestamp and a 64-bit tag mask, and a predicate over them is evaluated on
   the device; the caller assigns the tag bits (INTEGRATION.md maps FrameMeta onto them).

   A row never given attributes has timestamp 0 and tags 0.  Attributes follow their rows as groups do: an appended frame
   gets the defaults, an upsert keeps the frame's attributes, removes drop them; MV2V has no place for them, so
   wax_vs_deserialize and wax_vs_debug_fill_synthetic reset every row and the caller re-applies them after loading.  The
   first where search after a mutation or wax_vs_set_attributes uploads a device copy (16 bytes per row, counter
   "attribute_uploads"); later ones reuse it. */
typedef struct wax_vs_where {
    int64_t after;      /* timestamp >= after;  INT64_MIN = no lower bound                                  */
    int64_t before;     /* timestamp <  before; INT64_MAX = no upper bound (a timestamp of INT64_MAX passes) */
    uint64_t all_tags;  /* (tags & all_tags) == all_tags                                                    */
    uint64_t no_tags;   /* (tags & no_tags)  == 0                                                           */
} wax_vs_where;
/* Set frames' attributes (upsert, as wax_vs_set_groups): frame_ids[i] -> timestamps[i], tags[i]; unknown frame ids are
   ignored, a later entry for the same frame wins; timestamps or tags may be NULL to leave that column unchanged.
   *out_assigned (optional) = distinct known frames named.  A mutator (write lock). */
int32_t wax_vs_set_attributes(wax_vs_engine *engine, const uint64_t *frame_ids, const int64_t *timestamps,
                              const uint64_t *tags, uint64_t n, uint64_t *out_assigned);
/* wax_vs_search_batch_multi_filtered plus a predicate per query: query i searches the rows that pass
   wheres[query_where[i]] AND its id filter query_filter[i] (either may be WAX_VS_NO_FILTER).  A predicate that admits
   nothing (after >= before, all_tags overlapping no_tags) is valid and yields empty answers.  Query i's answer is
   identical to wax_vs_search_batch_multi_filtered with an allow-list of exactly the frames passing both: same ids, same
   order, same score bits.  The argument checks of multi_filtered run before the empty-engine early return, and a
   query_where entry >= n_wheres other than WAX_VS_NO_FILTER -> WAX_VS_ERR_ARGUMENT; NULL wheres (n_wheres > 0) or
   query_where (n_queries > 0) -> WAX_VS_ERR_NULL.  A single query is the batch of one.
   How: the unit that gets a row filter is each distinct (where, id filter) pair.  An allow-list is tested against the
   attributes on the host (O(listed)); otherwise one device pass counts the rows passing every predicate of the call,
   windows of <= 16 384 rows (nothing of the deny-list among them) are listed by the device and scored as a gather, and
   wider ones get a row bitset (the deny-list's, the predicate ANDed in on the device) for the tensor-core levels or the
   masked scan, exactly as an id filter's. */
int32_t wax_vs_search_batch_where(wax_vs_engine *engine, const float *queries, uint32_t n_queries, uint32_t query_len,
                                  int64_t top_k, const uint64_t *frame_ids, const uint64_t *filter_offsets,
                                  const int32_t *filter_modes, uint32_t n_filters, const uint32_t *query_filter,
                                  const wax_vs_where *wheres, uint32_t n_wheres, const uint32_t *query_where,
                                  uint64_t *out_ids, float *out_scores, uint32_t out_stride, uint32_t *out_n);
/* wax_vs_search_batch_grouped with ONE predicate for the batch, ANDed with its id filter; NULL where ->
   WAX_VS_ERR_NULL, otherwise the checks of wax_vs_search_batch_grouped.  Each answer is identical to
   wax_vs_search_grouped under the allow-list of the passing frames: same frame ids, group ids, order and score bits.
   n_queries == 1 runs the single-query grouped pipeline. */
int32_t wax_vs_search_batch_grouped_where(wax_vs_engine *engine, const float *queries, uint32_t n_queries,
                                          uint32_t query_len, int64_t top_groups, uint32_t per_group,
                                          const uint64_t *frame_ids, uint64_t n_ids, int32_t mode,
                                          const wax_vs_where *where, uint64_t *out_ids, float *out_scores,
                                          uint64_t *out_groups, uint32_t out_stride, uint32_t *out_n);

/* ---- frame locations: PhotoRAG's location radius as a predicate below the top-k (API EXTENSION) ---------------------
   PhotoRAG answers a location query with an allow-list (PhotoRAGOrchestrator.buildLocationAllowlist,
   PhotoRAGOrchestrator.swift:788-854): the frames of every 0.01-degree bin (locationBins, :766-771, binned by
   locationBin(from:), :868-875) in a box around the centre, passed as frameFilter beside the request's timeRange
   (:238-257).  Here each row may carry its bins and the box is one more clause of a where, evaluated on the device.

   Frame side: a row has a location, stored as its bins (Int(floor(lat * 100)), Int(floor(lon * 100)) in fp64, not
   clamped; bins beyond int32 are stored saturated, and no box reaches past +-36 000), or has none, and then never passes
   a location clause.  Locations follow their rows as attributes do: an appended frame has none, an upsert keeps the
   frame's, removes drop them, wax_vs_deserialize and wax_vs_debug_fill_synthetic reset every row (MV2V has no place for
   them).  The first where_near search after a mutation or wax_vs_set_locations uploads a device copy (8 bytes per row,
   counter "location_uploads").

   Query side, in fp64 as buildLocationAllowlist computes it: the centre clamped as PhotoCoordinate.init and the radius as
   PhotoLocationQuery.init (PhotoRAGTypes.swift:33-57) with Swift's min / max (a NaN latitude becomes -90, a NaN radius
   0); latDelta = r / 111000, lonDelta = min(180, r / max(1e-6, 111000 * cos(lat * pi / 180))); lat bins
   floor((lat -+ latDelta) * 100) clamped to [-9000, 9000], lon bins floor((lon -+ lonDelta) * 100) not clamped; when
   minLonBin > maxLonBin the lon bins are [minLonBin, 18000] and [-18000, maxLonBin].  There is no location clause where
   Swift returns nil: radius <= 0, a bin count <= 0, or latBinCount * lonBinCount >= 100 000.  A row passes the clause
   when its lat bin is in range and its lon bin in one of the lon ranges: exactly membership in the union of
   locationBins[bin] over the box.
   Two host-arithmetic notes: where Swift's Int(_:) would trap (a non-finite or out-of-range bin, e.g. an infinite
   radius) the library returns WAX_VS_ERR_ARGUMENT; cos is the C library's, which Foundation uses on Linux too (on Darwin
   it may differ in the last ulp, which moves a box edge only when lon +- lonDelta falls within an ulp of a bin edge). */
typedef struct wax_vs_where_near {
    wax_vs_where where;     /* the time and tag clauses                                  */
    double latitude;        /* the centre, degrees                                       */
    double longitude;
    double radius_m;        /* metres; <= 0 or NaN: no location clause                   */
} wax_vs_where_near;
/* Set frames' locations (upsert, as wax_vs_set_attributes): frame_ids[i] -> (latitudes[i], longitudes[i]) in degrees; a
   NaN pair clears the frame's location; any other non-finite coordinate -> WAX_VS_ERR_ARGUMENT and nothing is written.
   Unknown frame ids are ignored, a later entry for the same frame wins; *out_assigned (optional) = distinct known frames
   named.  A mutator (write lock). */
int32_t wax_vs_set_locations(wax_vs_engine *engine, const uint64_t *frame_ids, const double *latitudes,
                             const double *longitudes, uint64_t n, uint64_t *out_assigned);
/* The query-side arithmetic above, on the host (no engine, no device): *out_active = 1 and out_box = {minLatBin,
   maxLatBin, minLonBin, maxLonBin} for a box, *out_active = 0 and zeros for "no location clause"; WAX_VS_ERR_ARGUMENT
   where Swift would trap. */
int32_t wax_vs_location_box(double latitude, double longitude, double radius_m, int32_t out_box[4], int32_t *out_active);
/* The frame-side rule, on the host, as wax_vs_set_locations stores it: *out_has = 0 (and zeros) for a NaN pair, else
   out_bin = {latBin, lonBin}; WAX_VS_ERR_ARGUMENT for any other non-finite coordinate. */
int32_t wax_vs_location_bin(double latitude, double longitude, int32_t out_bin[2], int32_t *out_has);
/* wax_vs_search_batch_where with a location box in each predicate.  Query i's answer is identical to
   wax_vs_search_batch_multi_filtered under an allow-list of exactly the frames that pass its time and tag clauses, lie in
   its box and pass its id filter: same ids, order and score bits.  The argument checks of wax_vs_search_batch_where, and
   the boxes' (WAX_VS_ERR_ARGUMENT), run before the empty-engine early return.  How: as wax_vs_search_batch_where, with
   the box tested next to the time and tag clauses on the host (allow-lists) and in the location forms of the device
   passes (count, listing, bitset AND); a call none of whose predicates has a box runs wax_vs_search_batch_where. */
int32_t wax_vs_search_batch_where_near(wax_vs_engine *engine, const float *queries, uint32_t n_queries,
                                       uint32_t query_len, int64_t top_k, const uint64_t *frame_ids,
                                       const uint64_t *filter_offsets, const int32_t *filter_modes, uint32_t n_filters,
                                       const uint32_t *query_filter, const wax_vs_where_near *wheres, uint32_t n_wheres,
                                       const uint32_t *query_where, uint64_t *out_ids, float *out_scores,
                                       uint32_t out_stride, uint32_t *out_n);
/* wax_vs_search_batch_grouped_where with ONE where_near predicate for the batch; each answer is identical to
   wax_vs_search_grouped under the allow-list of the frames passing it and the id filter: same frame ids, group ids,
   order and score bits. */
int32_t wax_vs_search_batch_grouped_where_near(wax_vs_engine *engine, const float *queries, uint32_t n_queries,
                                               uint32_t query_len, int64_t top_groups, uint32_t per_group,
                                               const uint64_t *frame_ids, uint64_t n_ids, int32_t mode,
                                               const wax_vs_where_near *where, uint64_t *out_ids, float *out_scores,
                                               uint64_t *out_groups, uint32_t out_stride, uint32_t *out_n);
/* wax_vs_search_batch_grouped with a where and an id filter of its own for each query (a server batching PhotoRAG /
   VideoRAG requests from many sessions): query i searches the frames that pass the time, tag and location clauses of
   wheres[query_where[i]] AND id filter query_filter[i] (either may be WAX_VS_NO_FILTER; both: unfiltered; filters as
   wax_vs_search_batch_multi_filtered).  Its answer is identical to wax_vs_search_grouped for that query alone under an
   allow-list of exactly those frames -- same frame ids, group ids, group-major order and score bits -- at
   out_*[i * out_stride], count out_n[i].  top_groups and per_group hold for the whole batch.  A where whose box is "no
   location clause" is a time and tag predicate; a where that admits nothing is valid and gives out_n[i] = 0.  There is no
   term clause: grouped search takes none.  Checked before the empty-engine early return: the checks of
   wax_vs_search_batch_where_near (filters, query_filter and query_where ranges, NULL arrays, the boxes) and the grouped
   ones of wax_vs_search_batch_grouped (per_group, clamp(top_groups) * per_group, NULL outputs; out_stride >=
   min(clamp(top_groups) * per_group, N) else WAX_VS_ERR_BUFFER).  n_queries == 0 returns OK; n_queries == 1 runs the
   single-query grouped pipeline.
   How: the (where, id filter) pairs are the units of wax_vs_search_batch_where, each query's exact top-k_c rows come from
   that batched search, and the coverage level is wax_vs_search_batch_grouped's.  A selected group that must be scored
   over its own rows is scored under its query's row bitset, rebuilt on the device in passes of at most
   "filter_bitset_bytes" of distinct units (counter "grouped_batch_expansion_passes").  Crowded queries, and batches the
   coverage level does not take (a mix of gather and tensor classes among them), run the single-query pipeline, each
   under its own pair.  wax_vs_search_batch_grouped, _grouped_where and _grouped_where_near are the case of one pair for
   every query. */
int32_t wax_vs_search_batch_grouped_multi_where(wax_vs_engine *engine, const float *queries, uint32_t n_queries,
                                                uint32_t query_len, int64_t top_groups, uint32_t per_group,
                                                const uint64_t *frame_ids, const uint64_t *filter_offsets,
                                                const int32_t *filter_modes, uint32_t n_filters,
                                                const uint32_t *query_filter, const wax_vs_where_near *wheres,
                                                uint32_t n_wheres, const uint32_t *query_where, uint64_t *out_ids,
                                                float *out_scores, uint64_t *out_groups, uint32_t out_stride,
                                                uint32_t *out_n);

/* ---- frame terms: Wax's metadataFilter as term clauses below the top-k (API EXTENSION) --------------------------------
   MetadataFilter (SearchRequest.swift:130-145) requires exact key = value entries of meta.metadata.entries, TagPairs of
   meta.tags and strings of meta.labels (UnifiedSearch.matches(metadataFilter:meta:), UnifiedSearch.swift:1215-1239).
   Here each row may carry a set of 64-bit term ids, assigned by the caller (the bindings intern Wax's three kinds of
   requirement exactly), and a where may require up to 32 of them.

   Frame side: terms follow their rows as locations do: an appended frame has none, an upsert keeps the frame's set,
   removes drop them, wax_vs_deserialize and wax_vs_debug_fill_synthetic reset every row (MV2V has no place for them, and
   nothing is stored until the first wax_vs_set_terms).  The first where_terms search after a mutation or
   wax_vs_set_terms builds a device inverted index (counters "term_index_builds", "term_index_bytes").

   Query side: a row passes a where's term clause when its set holds every required id; an empty list is no clause, and
   a row without terms passes no non-empty clause (Swift's answer for a nil meta.metadata). */
/* Replace the whole term set of each named frame (upsert by frame id, as wax_vs_set_attributes): frame_ids[i] ->
   terms[term_offsets[i] .. term_offsets[i + 1]).  Duplicate ids in a list are kept once, an empty list clears the set,
   unknown frame ids are ignored and a later entry for the same frame wins; *out_assigned (optional) = distinct known
   frames named.  NULL term_offsets, frame_ids (n > 0) or terms (a non-empty list) -> WAX_VS_ERR_NULL; offsets that do
   not start at 0 or decrease -> WAX_VS_ERR_ARGUMENT, and nothing is written.  A mutator (write lock). */
int32_t wax_vs_set_terms(wax_vs_engine *engine, const uint64_t *frame_ids, const uint64_t *term_offsets,
                         const uint64_t *terms, uint64_t n, uint64_t *out_assigned);
/* wax_vs_search_batch_where_near with a term clause in each where: where w requires
   where_terms[where_term_offsets[w] .. where_term_offsets[w + 1]) (0 to 32 ids, duplicates allowed).  Query i's answer
   is identical to wax_vs_search_batch_multi_filtered under an allow-list of exactly the frames that hold every required
   id and pass the time, tag and location clauses and the id filter: same ids, order and score bits.  The argument checks
   of wax_vs_search_batch_where_near, and NULL where_term_offsets or where_terms (some where has a term) ->
   WAX_VS_ERR_NULL, offsets that do not start at 0 or decrease, or more than 32 ids in a where -> WAX_VS_ERR_ARGUMENT,
   run before the empty-engine early return.  A call in which no where has a term runs wax_vs_search_batch_where_near.
   How: wheres with terms and equal contents are one unit.  A (where, id filter) pair with terms is tested on the host
   against an allow-list; otherwise the device resolves each required id's posting list, takes the rarest one's rows as
   candidates (O(its length), never a pass over the corpus), checks the other terms, the where's clauses and a
   deny-list on each, and counts the rows that pass: <= 16 384 rows are listed and scored as a gather, wider units get
   their bits set in a row bitset under the filter_bitset_bytes split.  A call whose listed rows would pass 2^32 - 1
   -> WAX_VS_ERR_CAPACITY.  Grouped search takes no term clause. */
int32_t wax_vs_search_batch_where_terms(wax_vs_engine *engine, const float *queries, uint32_t n_queries,
                                        uint32_t query_len, int64_t top_k, const uint64_t *frame_ids,
                                        const uint64_t *filter_offsets, const int32_t *filter_modes, uint32_t n_filters,
                                        const uint32_t *query_filter, const wax_vs_where_near *wheres, uint32_t n_wheres,
                                        const uint32_t *query_where, const uint64_t *where_term_offsets,
                                        const uint64_t *where_terms, uint64_t *out_ids, float *out_scores,
                                        uint32_t out_stride, uint32_t *out_n);

/* ---- group clauses: VideoRAG's video filter below the top-k (API EXTENSION) -----------------------------------------
   VideoRAGQuery.videoIDs (VideoRAGTypes.swift:53) becomes FrameFilter(frameIds:), the union of segmentIdsByVideoID[v]
   over the chosen videos, built in Swift on every request (VideoRAGOrchestrator.swift:239-247) and resolved id by id on
   the host.  Here a where may name the groups instead: a row passes a where's group clause when its group is one of
   the where's group ids.  A row's group is the one grouped search uses: the id last given to the frame by
   wax_vs_set_groups, else the frame's own id (so with no set_groups the clause is a clause on frame ids); it follows the
   frame through every mutator.  A clause lists 0 to 65 536 ids; duplicates are allowed, an id no row carries matches
   nothing, and an empty list is no clause.  The clause is ANDed with the where's other clauses and the query's id
   filter.  VideoRAG maps videoIDs to the roots of the chosen videos (the parentId its hits are grouped by).
   How: wheres with equal contents are one unit.  A (where, id filter) pair with groups is tested on the host against an
   allow-list; otherwise the device resolves each distinct group id of the call in the group index of grouped search
   (built as grouped search builds it, counter "group_index_builds") and walks the rows of the unit's groups, or the
   postings of its rarest term when that list is shorter than the group union -- O(rows of those groups), never a pass
   over the corpus.  Each candidate is checked against the other clauses and a deny-list.  The rows that pass are counted:
   <= 16 384 are listed and scored as a gather, wider units get their bits set in a row bitset under the
   filter_bitset_bytes split.  Counters "where_group_units" (units planned on the device) and "where_group_rows_walked"
   (the candidate positions their walks visit, once per unit and call). */
/* wax_vs_search_batch_where_terms with a group clause in each where: where w requires one of
   where_groups[where_group_offsets[w] .. where_group_offsets[w + 1]).  where_term_offsets may be NULL (no where has a
   term).  Query i's answer is identical to wax_vs_search_batch_multi_filtered under an allow-list of exactly the frames
   that pass every clause and the id filter: same ids, order and score bits.  Before the empty-engine early return: the
   checks of wax_vs_search_batch_where_near, then NULL where_group_offsets, or NULL where_groups when some where has a
   group -> WAX_VS_ERR_NULL, group offsets that do not start at 0 or decrease, or more than 65 536 ids in a where ->
   WAX_VS_ERR_ARGUMENT, then the term checks of wax_vs_search_batch_where_terms.  A call in which no where has a group
   runs wax_vs_search_batch_where_terms (term offsets given) or wax_vs_search_batch_where_near.  A call whose listed rows
   would pass 2^32 - 1 -> WAX_VS_ERR_CAPACITY. */
int32_t wax_vs_search_batch_where_groups(wax_vs_engine *engine, const float *queries, uint32_t n_queries,
                                         uint32_t query_len, int64_t top_k, const uint64_t *frame_ids,
                                         const uint64_t *filter_offsets, const int32_t *filter_modes, uint32_t n_filters,
                                         const uint32_t *query_filter, const wax_vs_where_near *wheres, uint32_t n_wheres,
                                         const uint32_t *query_where, const uint64_t *where_term_offsets,
                                         const uint64_t *where_terms, const uint64_t *where_group_offsets,
                                         const uint64_t *where_groups, uint64_t *out_ids, float *out_scores,
                                         uint32_t out_stride, uint32_t *out_n);
/* wax_vs_search_batch_grouped_multi_where with a group clause in each where, as wax_vs_search_batch_where_groups takes
   it (grouped search takes no term clause): VideoRAG's request -- the best segments of the best videos, among these
   videos, inside this time window -- for many queries at once.  Query i's answer is identical to wax_vs_search_grouped
   under an allow-list of exactly the frames that pass: same frame ids, group ids, group-major order and score bits.  The
   checks of wax_vs_search_batch_grouped_multi_where, then the group checks of wax_vs_search_batch_where_groups, before
   the empty-engine early return.  A call in which no where has a group runs wax_vs_search_batch_grouped_multi_where.
   A selected group scored over its own rows, and a crowded query, is scored under its unit's row bitset, rebuilt on the
   device. */
int32_t wax_vs_search_batch_grouped_multi_where_groups(wax_vs_engine *engine, const float *queries, uint32_t n_queries,
                                                       uint32_t query_len, int64_t top_groups, uint32_t per_group,
                                                       const uint64_t *frame_ids, const uint64_t *filter_offsets,
                                                       const int32_t *filter_modes, uint32_t n_filters,
                                                       const uint32_t *query_filter, const wax_vs_where_near *wheres,
                                                       uint32_t n_wheres, const uint32_t *query_where,
                                                       const uint64_t *where_group_offsets, const uint64_t *where_groups,
                                                       uint64_t *out_ids, float *out_scores, uint64_t *out_groups,
                                                       uint32_t out_stride, uint32_t *out_n);

/* ---- root clauses: PhotoRAG's and VideoRAG's test on each hit's root below the top-k (API EXTENSION) -----------------
   After ranking, both orchestrators drop every hit whose root (parentId ?? id) has no meta, is not kind == root, is
   deleted or has supersededBy set (PhotoRAGOrchestrator.swift:280-286, VideoRAGOrchestrator.swift:314-318).  Re-ingesting
   a photo or video supersedes the old root while its segments keep their embeddings, so a grouped search filtered that
   way afterwards comes back short.  Here each group id may hold a 64-bit root-tag word, and a where may carry a root
   clause on it, evaluated on the device below the top-k.

   Group side: wax_vs_set_root_tags keeps a word per group id; a group never given one has the word 0.  A row's group is
   the one grouped search and the group clause use (its wax_vs_set_groups id, else its frame id).  The words are keyed
   by group, not by row: adds, upserts, removes, set_groups and rebalance leave them alone (a row that moves to another
   group takes that group's word), and an id no row carries yet is kept for the rows that take it later.
   wax_vs_deserialize clears them (MV2V has no place for them; the caller re-applies them).  The word is the caller's;
   the bindings set bits such as IS_ROOT, DELETED and SUPERSEDED from the root's FrameMeta.

   Query side: a row passes the clause when its group's word holds every bit of all_tags and none of no_tags; {0, 0} is
   no clause.  The clause passes or fails all the rows of a group together, so grouped search returns the exact top
   groups among the groups that pass.  PhotoRAG's test is all_tags = IS_ROOT, no_tags = DELETED | SUPERSEDED (a root
   without meta never got IS_ROOT).
   How: the first search with a root clause after a mutation, wax_vs_set_groups or wax_vs_set_root_tags builds a device
   column of each row's word (8 bytes per row, from the group index of grouped search; counter "root_column_builds");
   nothing is allocated before.  Every pass that tests a where (the count, listing and bitset passes, the term and group
   units) has a rooted form that loads the row's word beside its attributes.  Listed rows are tested on the host. */
typedef struct wax_vs_root_clause {
    uint64_t all_tags;  /* (word & all_tags) == all_tags */
    uint64_t no_tags;   /* (word & no_tags)  == 0        */
} wax_vs_root_clause;
/* Set groups' root-tag words (upsert by group id): group_ids[i] -> tags[i]; a later entry for the same id wins, and any
   id is accepted, carried by a row or not.  *out_assigned (optional) = distinct group ids named.  NULL group_ids or tags
   (n > 0) -> WAX_VS_ERR_NULL.  A mutator (write lock).  A multi-device handle keeps the whole table on every shard and
   reports one engine's *out_assigned. */
int32_t wax_vs_set_root_tags(wax_vs_engine *engine, const uint64_t *group_ids, const uint64_t *tags, uint64_t n,
                             uint64_t *out_assigned);
/* wax_vs_search_batch_where_groups with a root clause in each where: where w's is where_roots[w] (NULL: no where has
   one).  Query i's answer is identical to wax_vs_search_batch_multi_filtered under an allow-list of exactly the frames
   that pass every clause and the id filter: same ids, order and score bits.  The argument checks of
   wax_vs_search_batch_where_groups (its term offsets when given, and the boxes) run before the empty-engine early
   return.  A call in which no where has a root clause runs wax_vs_search_batch_where_groups. */
int32_t wax_vs_search_batch_where_roots(wax_vs_engine *engine, const float *queries, uint32_t n_queries,
                                        uint32_t query_len, int64_t top_k, const uint64_t *frame_ids,
                                        const uint64_t *filter_offsets, const int32_t *filter_modes, uint32_t n_filters,
                                        const uint32_t *query_filter, const wax_vs_where_near *wheres, uint32_t n_wheres,
                                        const uint32_t *query_where, const uint64_t *where_term_offsets,
                                        const uint64_t *where_terms, const uint64_t *where_group_offsets,
                                        const uint64_t *where_groups, const wax_vs_root_clause *where_roots,
                                        uint64_t *out_ids, float *out_scores, uint32_t out_stride, uint32_t *out_n);
/* wax_vs_search_batch_grouped_multi_where_groups with a root clause in each where, as
   wax_vs_search_batch_where_roots takes it: PhotoRAG's and VideoRAG's request -- the best frames of the best photos or
   videos whose root is live -- with no over-fetch.  Query i's answer is identical to wax_vs_search_grouped under an
   allow-list of exactly the frames that pass: same frame ids, group ids, group-major order and score bits; whenever at
   least clamp(top_groups) groups pass, that many come back.  The checks of
   wax_vs_search_batch_grouped_multi_where_groups (and the boxes) run before the empty-engine early return.  A call in
   which no where has a root clause runs wax_vs_search_batch_grouped_multi_where_groups. */
int32_t wax_vs_search_batch_grouped_multi_where_roots(wax_vs_engine *engine, const float *queries, uint32_t n_queries,
                                                      uint32_t query_len, int64_t top_groups, uint32_t per_group,
                                                      const uint64_t *frame_ids, const uint64_t *filter_offsets,
                                                      const int32_t *filter_modes, uint32_t n_filters,
                                                      const uint32_t *query_filter, const wax_vs_where_near *wheres,
                                                      uint32_t n_wheres, const uint32_t *query_where,
                                                      const uint64_t *where_group_offsets, const uint64_t *where_groups,
                                                      const wax_vs_root_clause *where_roots, uint64_t *out_ids,
                                                      float *out_scores, uint64_t *out_groups, uint32_t out_stride,
                                                      uint32_t *out_n);

/* Device-resident form used by the row-sharded engine: `d_queries` (n_queries x dims) and
   `d_candidates` (n_queries x k_eff entries, k_eff = min(clamp(top_k), 10000) -- NOT clipped to N, padding
   has valid = 0) are DEVICE pointers on the engine's device; the work is enqueued on `cuda_stream`
   (a cudaStream_t; NULL = legacy default stream) and the call returns without synchronising.
   candidate.row = row_offset + local row (row_offset + the row's key on a keyed engine).
   Ordering against mutators: the library remembers that device-path work was enqueued and every mutator
   (add / remove / reserve / deserialize / fill) drains the DEVICE (cudaDeviceSynchronize) under its write lock
   before it touches the corpus, so an in-flight scan never reads rows that are being moved. */
int32_t wax_vs_search_device(wax_vs_engine *engine, const float *d_queries, uint32_t n_queries,
                             int64_t top_k, uint64_t row_offset, wax_vs_candidate *d_candidates,
                             void *cuda_stream);

/* Batched device-resident form (the row-sharded engine's search_batch): same pointers and candidate layout as
   wax_vs_search_device, but the queries go through the batched tensor-core levels (bf16-shadow nominations ->
   TF32 retry -> exact scan; results identical to n_queries single-query calls) whenever the batch is eligible
   (wax_vs_search_batch's rules).  Those levels read their proof flags back, so this call MAY synchronise
   `cuda_stream` before it returns; d_candidates is complete in `cuda_stream` order. */
int32_t wax_vs_search_batch_device(wax_vs_engine *engine, const float *d_queries, uint32_t n_queries,
                                   int64_t top_k, uint64_t row_offset, wax_vs_candidate *d_candidates,
                                   void *cuda_stream);

/* ---- row-sharded search across the GPUs of one node (SURVEY.md section 8e; no reference counterpart) -------------
   One engine per GPU holds a contiguous row range of the corpus; the query is replicated; every rank scans its shard
   and the per-shard top-k lists are exchanged and merged under the total order (distance, GLOBAL row).  The exchange is
   fused into the scan launch: the kernel's last CTA writes its k candidates straight into every rank's mailbox over
   NVLink / NVSwitch peer memory, raises a flag, waits for the others' flags and merges world x k candidates -- no
   collective launch, no D2H copy, no host merge (wax_b200/csrc/waxvs_shard.cuh).  Every rank gets the same result.

   Setup: each rank calls wax_vs_shard_open (allocates its mailbox, returns a WAX_VS_SHARD_HANDLE_BYTES blob), the
   blobs are exchanged by any out-of-band means (the Python mirror uses one torch.distributed all-gather; a single
   process driving several GPUs just passes them along), then every rank calls wax_vs_shard_connect with all `world`
   blobs in rank order (CUDA IPC between processes, peer access inside one process).
   Searches are COLLECTIVE: every rank must issue the same searches in the same order (same query, same top_k).
   top_k is clamped to [1, 10000] as usual but must not exceed WAX_VS_SHARD_MAX_K (the fused top-k range);
   larger k -> WAX_VS_ERR_UNSUPPORTED (gather wax_vs_search_device candidates instead).  A rank whose peers never
   arrive gets WAX_VS_ERR_CUDA after the exchange timeout (20 s; option "shard_timeout_ms") instead of hanging. */
#define WAX_VS_SHARD_HANDLE_BYTES 128
#define WAX_VS_SHARD_MAX_RANKS 16
#define WAX_VS_SHARD_MAX_K 128
int32_t wax_vs_shard_open(wax_vs_engine *engine, int32_t rank, int32_t world, uint64_t row_offset,
                          uint8_t *out_handle /* WAX_VS_SHARD_HANDLE_BYTES */);
int32_t wax_vs_shard_connect(wax_vs_engine *engine, const uint8_t *handles /* n_handles x HANDLE_BYTES, rank order */,
                             int32_t n_handles);
/* Leave the group: unmaps the peers' mailboxes.  This rank's own mailbox stays allocated until wax_vs_destroy or the
   next wax_vs_shard_open, because other processes may still have it mapped -- close on every rank, synchronise the
   ranks (a barrier), then destroy. */
int32_t wax_vs_shard_close(wax_vs_engine *engine);
/* search(vector:topK:) over the whole sharded corpus; host query in, host ids / scores out (best first, as
   wax_vs_search); blocks until the merged result is in the caller's buffers.  out_cap >= clamp(top_k). */
int32_t wax_vs_shard_search(wax_vs_engine *engine, const float *query, uint32_t query_len, int64_t top_k,
                            uint64_t *out_ids, float *out_scores, uint32_t out_cap, uint32_t *out_n);
/* Device-side merge for the sharded search_batch: d_gathered = [world][n_queries][k] candidates exactly as an
   all-gather of the ranks' wax_vs_search_batch_device outputs leaves them (rank-major; every per-query list sorted, padding
   valid = 0 last); d_out = [n_queries][k_out] (k_out <= k), the k_out best of each query under (distance, GLOBAL row),
   whichever rows each rank holds (contiguous ranges or keyed rows).  Enqueued on cuda_stream, no synchronisation. */
int32_t wax_vs_merge_candidates_device(wax_vs_engine *engine, const wax_vs_candidate *d_gathered, uint32_t world,
                                       uint32_t n_queries, uint32_t k, uint32_t k_out, wax_vs_candidate *d_out,
                                       void *cuda_stream);
/* wax_vs_search_filtered over the whole sharded corpus: every rank passes the SAME frame_ids / mode; a rank resolves
   the ids its own shard holds (the rest are unknown to it and ignored), plans its shard as wax_vs_search_filtered
   does (a short allow-list is gathered, anything else is a row filter in the fused scan) and the exchange merges the
   ranks' lists.  Exactly one exchange per query per rank.  The no-clause case of wax_vs_shard_search_where. */
int32_t wax_vs_shard_search_filtered(wax_vs_engine *engine, const float *query, uint32_t query_len, int64_t top_k,
                                     const uint64_t *frame_ids, uint64_t n_ids, int32_t mode, uint64_t *out_ids,
                                     float *out_scores, uint32_t out_cap, uint32_t *out_n);
/* Collective, fused transport, top_k <= WAX_VS_SHARD_MAX_K: one query under one where (time, tag and location clauses
   of `where`, plus terms[0 .. n_terms) required, 0..32 ids) AND the id filter (frame_ids, n_ids, mode as
   wax_vs_shard_search_filtered; n_ids == 0 with mode 1 = none).  Every rank passes the same arguments.  The answer is
   the same on every rank and identical (ids, order, score bits) to wax_vs_search_batch_where_terms for that query on
   one engine holding the whole corpus.  NULL where, out_n, frame_ids (n_ids > 0) or terms (n_terms > 0) ->
   WAX_VS_ERR_NULL; a mode other than 0 / 1, more than 32 terms or a non-finite box -> WAX_VS_ERR_ARGUMENT; these checks
   run before the engine is locked, so every rank fails alike before any rank joins the exchange.  top_k above
   WAX_VS_SHARD_MAX_K -> WAX_VS_ERR_UNSUPPORTED.
   How: each rank plans its shard as the where entry points do.  A unit of at most 16 384 rows is gathered, scored and
   sorted, then exchanged by a one-CTA launch; a wider one is a row bitset in the fused scan, whose last CTA exchanges;
   a shard where nothing passes exchanges padding.  A collective call never frees device memory or waits for the whole
   device (a peer's exchange may be waiting for this rank on the same GPU): the rank's scratch is sized for its whole
   shard, and superseded mirrors are released by the mutators, under the write lock. */
int32_t wax_vs_shard_search_where(wax_vs_engine *engine, const float *query, uint32_t query_len, int64_t top_k,
                                  const uint64_t *frame_ids, uint64_t n_ids, int32_t mode,
                                  const wax_vs_where_near *where, const uint64_t *terms, uint32_t n_terms,
                                  uint64_t *out_ids, float *out_scores, uint32_t out_cap, uint32_t *out_n);
/* The rank-local half of a batched sharded where search, for any transport and any k up to 10 000.  Arguments are those
   of wax_vs_search_batch_where_terms; where_term_offsets may be NULL when no where has a term.  d_queries is a device
   pointer, as in wax_vs_search_batch_device.  Output: d_candidates [n_queries][clamp(top_k)] on the device.  Each list is
   sorted by (distance, global row), and padding has valid = 0 and comes last.  This is exactly the layout
   that wax_vs_merge_candidates_device takes after an all-gather.  A query with no allowed row on this shard, and every
   query of an empty shard, is all padding.  The argument checks of wax_vs_search_batch_where_terms, and NULL d_queries
   or d_candidates -> WAX_VS_ERR_NULL, run before the empty-engine early return.  The call may synchronise cuda_stream,
   as wax_vs_search_batch_device does. */
int32_t wax_vs_search_batch_where_device(wax_vs_engine *engine, const float *d_queries, uint32_t n_queries, int64_t top_k,
                                         const uint64_t *frame_ids, const uint64_t *filter_offsets,
                                         const int32_t *filter_modes, uint32_t n_filters, const uint32_t *query_filter,
                                         const wax_vs_where_near *wheres, uint32_t n_wheres, const uint32_t *query_where,
                                         const uint64_t *where_term_offsets, const uint64_t *where_terms,
                                         uint64_t row_offset, wax_vs_candidate *d_candidates, void *cuda_stream);

/* ---- sharded grouped search: wax_vs_search_batch_grouped_multi_where over the row-sharded engine ------------------
   Exact, in two exchanges of any transport (wax_b200/sharded.py).  G = clamp(top_groups), P = per_group.
   Round 1: every rank's own grouped answer (wax_vs_shard_grouped_heads_device), all-gathered.
   Merge 1: the global top G groups by their best rows (wax_vs_merge_group_heads_device).  P == 1 ends here.
   Round 2: every rank's P best rows of each chosen group (wax_vs_shard_grouped_expand_device), all-gathered and merged
   per (query, group) by wax_vs_merge_candidates_device(world, n_queries * G, P, P).
   Each entry point uses the caller's stream and may synchronise it. */
typedef struct wax_vs_group_candidate {   /* 32 bytes, naturally aligned */
    float distance;     /* as wax_vs_candidate                                   */
    uint32_t valid;     /* 1 = real row, 0 = padding (all fields zero)           */
    uint64_t row;       /* global row = row_offset + local row or row key        */
    uint64_t frame_id;
    uint64_t group_id;
} wax_vs_group_candidate;
#define WAX_VS_SHARD_MAX_GROUPS 256        /* clamp(top_groups) of the sharded grouped form */
/* Round 1.  d_heads = [n_queries][G][P] on the device: query i's answer of wax_vs_search_batch_grouped_multi_where on
   this engine alone (same batch, wheres and id filters), group-major, groups best first, rows best first, with global
   rows.  Padding has valid = 0 and is zeroed; an empty shard writes only padding.  Checked before the empty-engine early
   return: the checks of wax_vs_search_batch_grouped_multi_where; clamp(top_groups) > WAX_VS_SHARD_MAX_GROUPS ->
   WAX_VS_ERR_UNSUPPORTED; NULL d_queries or d_heads -> WAX_VS_ERR_NULL.  n_queries == 0 returns OK. */
int32_t wax_vs_shard_grouped_heads_device(wax_vs_engine *engine, const float *d_queries, uint32_t n_queries,
                                          int64_t top_groups, uint32_t per_group, const uint64_t *frame_ids,
                                          const uint64_t *filter_offsets, const int32_t *filter_modes, uint32_t n_filters,
                                          const uint32_t *query_filter, const wax_vs_where_near *wheres, uint32_t n_wheres,
                                          const uint32_t *query_where, uint64_t row_offset, wax_vs_group_candidate *d_heads,
                                          void *cuda_stream);
/* Merge 1.  d_gathered = [world][n_queries][G][P], the ranks' d_heads in rank order as an all-gather leaves them (any
   placement of rows on ranks).  d_chosen = [n_queries][G]: per query the union of the ranks' group heads (a group's first
   row), the best head kept per group id, the first G by (distance, global row); padding (valid = 0, zeroed) last.  These
   are the global top G groups, each as its best row.  world outside 1..WAX_VS_SHARD_MAX_RANKS, per_group outside
   1..WAX_VS_MAX_PER_GROUP -> WAX_VS_ERR_ARGUMENT; clamp(top_groups) > WAX_VS_SHARD_MAX_GROUPS -> WAX_VS_ERR_UNSUPPORTED;
   NULL pointers -> WAX_VS_ERR_NULL. */
int32_t wax_vs_merge_group_heads_device(wax_vs_engine *engine, const wax_vs_group_candidate *d_gathered, uint32_t world,
                                        uint32_t n_queries, int64_t top_groups, uint32_t per_group,
                                        wax_vs_group_candidate *d_chosen, void *cuda_stream);
/* Round 2.  d_rows = [n_queries][G][P] wax_vs_candidate: slot (i, s) holds this shard's best min(P, rows) rows of group
   d_chosen[i][s] under query i's where and id filter, sorted by (distance, global row), padding last and zeroed.  A
   group this rank listed in round 1 (d_own_heads, its own d_heads) is copied from there; a group it holds but did not
   list is scored over its rows (counter "shard_grouped_expanded_groups"); any other slot is padding.  The filters and
   wheres must be those of round 1.  The checks of wax_vs_shard_grouped_heads_device, and NULL d_chosen, d_own_heads or
   d_rows -> WAX_VS_ERR_NULL, run before the empty-engine early return. */
int32_t wax_vs_shard_grouped_expand_device(wax_vs_engine *engine, const float *d_queries, uint32_t n_queries,
                                           int64_t top_groups, uint32_t per_group, const uint64_t *frame_ids,
                                           const uint64_t *filter_offsets, const int32_t *filter_modes, uint32_t n_filters,
                                           const uint32_t *query_filter, const wax_vs_where_near *wheres,
                                           uint32_t n_wheres, const uint32_t *query_where,
                                           const wax_vs_group_candidate *d_chosen,
                                           const wax_vs_group_candidate *d_own_heads, uint64_t row_offset,
                                           wax_vs_candidate *d_rows, void *cuda_stream);

/* Device-resident form: d_query (dims floats) and d_candidates (clamp(top_k) merged entries, padding valid = 0) are
   device pointers; enqueued on `cuda_stream`, returns without synchronising. */
int32_t wax_vs_shard_search_device(wax_vs_engine *engine, const float *d_query, int64_t top_k,
                                   wax_vs_candidate *d_candidates, void *cuda_stream);

/* ---- persistence: "MV2V" v1 encoding = 2, byte-identical to MetalVectorEngine.serialize ---------- */

/* serialize() (MetalVectorEngine.swift:682-714). */
int32_t wax_vs_serialized_length(wax_vs_engine *engine, uint64_t *out);
int32_t wax_vs_serialize(wax_vs_engine *engine, uint8_t *dst, uint64_t cap, uint64_t *out_len);
/* deserialize(_:) (MetalVectorEngine.swift:716-815; VectorSerializer.swift:84-157): replaces the
   engine's contents.  Any violation -> WAX_VS_ERR_FORMAT with the reference's reason string in
   wax_vs_last_error(). */
int32_t wax_vs_deserialize(wax_vs_engine *engine, const uint8_t *src, uint64_t len);

/* Thread-local, NUL-terminated reason for the last non-zero return on this thread (the `reason:` of
   the WaxError the Swift side throws). Never NULL. */
const char *wax_vs_last_error(void);

/* ---- instrumentation (not part of the reference surface) -------------------------------------------- */

/* debugBufferPoolStats (MetalVectorEngine.swift:119-121; MetalVectorEnginePoolTests.swift:7-20):
   how many per-search scratch contexts were ever allocated / reused. */
int32_t wax_vs_debug_pool_stats(wax_vs_engine *engine, uint64_t *allocations, uint64_t *reuses);

/* Replace the contents with `rows` synthetic rows generated ON DEVICE (100 M x 384 does not fit a host):
   row r holds generator row (first_row + r) of stream `seed` (bit-identical to
   oracle wax_oracle_synth_row), frameId = id_base + r. */
int32_t wax_vs_debug_fill_synthetic(wax_vs_engine *engine, uint64_t seed, uint64_t first_row,
                                    uint64_t rows, uint64_t id_base, int32_t normalize);
/* Copy rows [first, first+n) back to the host (tests). */
int32_t wax_vs_debug_read_rows(wax_vs_engine *engine, uint64_t first, uint64_t n, float *dst);

/* Kernel-only timing with everything resident in HBM: generates `n_queries` distinct unit queries on device
   (generator stream `seed`), runs `warmup` + `iters` single-query searches back to back on one stream (step i
   uses query i mod n_queries), brackets the `iters` with CUDA events on that stream and returns the total
   milliseconds plus the number of kernel launches inside the bracket. */
int32_t wax_vs_debug_time_search(wax_vs_engine *engine, uint32_t n_queries, int64_t top_k, uint64_t seed,
                                 uint32_t warmup, uint32_t iters, float *out_ms_total,
                                 uint64_t *out_launches);

/* wax_vs_debug_time_search for the sharded path: warmup + iters collective searches strictly one at a time on one
   stream, CUDA events around the `iters` (every rank makes the same call; queries are generated on device from
   `seed`, identical on every rank). */
int32_t wax_vs_debug_time_shard_search(wax_vs_engine *engine, uint32_t n_queries, int64_t top_k, uint64_t seed,
                                       uint32_t warmup, uint32_t iters, float *out_ms_total, uint64_t *out_launches);

/* Host <-> device transfer rates on this box (GB/s) for `bytes` of pageable host memory: out7 = {one-thread staging
   memcpy, staging memcpy with the worker threads, DMA pinned->HBM, DMA HBM->pinned, upload pipeline pageable->HBM,
   download pipeline HBM->pageable, worker threads}.  Explains what bounds wax_vs_add_batch / wax_vs_serialize. */
int32_t wax_vs_debug_transfer_probe(wax_vs_engine *engine, uint64_t bytes, float *out7);

/* Where one fused search spends its time, from %globaltimer stamps inside the kernel (averages over `iters` searches,
   microseconds): out5 = {kernel start -> last warp leaves the scan loop, -> last CTA has selected its k, -> the last CTA
   starts the grid stage, -> result written, CUDA-event duration of the launch on its stream}. */
int32_t wax_vs_debug_phase_trace(wax_vs_engine *engine, int64_t top_k, uint32_t iters, float *out5);

/* Batched-path instrumentation: how many queries were answered by the tensor-core nomination path with a
   completed exactness proof, and how many had to be re-run on the exact single-query path. */
int32_t wax_vs_debug_batch_stats(wax_vs_engine *engine, uint64_t *tensor_queries, uint64_t *fallback_queries);

/* Named instrumentation counters: "batch_tensor_queries", "batch_fallback_queries", "batch_bf16_queries" (queries
   nominated from the bf16 shadow), "batch_retry_queries" (bf16-unproven queries retried on the TF32 nominations),
   "shadow_bytes" (HBM held by the bf16 shadow), "shadow_unavailable" (1 = the shadow did not fit in HBM, batches
   nominate in TF32 at about half the rate), "batch_tf32_queries", "filter_bitset_passes" (sub-batches of per-query
   filtered queries on the tensor-core class, wax_vs_search_batch_multi_filtered), "group_index_builds" (device group
   index builds of wax_vs_search_grouped), "attribute_uploads" (device attribute copies of the where searches),
   "term_index_builds" / "term_index_bytes" (term index builds of the where_terms searches / HBM the index holds),
   "where_group_units" / "where_group_rows_walked" (units of the where_groups searches planned on the device / the
   candidate positions they walk), "root_column_builds" (root column builds of the where_roots searches), "pool_allocs", "pool_reuses", "single_shadow_queries" / "single_shadow_fallbacks"
   (single queries the shadow route answered / that the fp32 scan answered after a failed proof, either shadow; read them
   while no search is running), "single_int8_queries" (single queries whose route nominated from the int8 shadow),
   "int8_shadow_bytes" / "int8_shadow_rows" (HBM held by the int8 shadow's live rows, codes and scales / rows it covers),
   "single_u4_queries", "u4_shadow_bytes" / "u4_shadow_rows" (the same for the 4-bit shadow). */
int32_t wax_vs_debug_counter(wax_vs_engine *engine, const char *name, uint64_t *out);

/* The form of the last fp32 scan this engine launched (the exact scan every search path ends in; tests): out[10] =
   {kernel: 1 = TMA-staged, 2 = direct-load; C (rows of C x 128 elements, 0 = generic length), rows per step, warps,
   stages (0 for the direct-load kernel); grid; chunk_steps (0 = static claims); mode: 0 = k <= 32 list, 1 = k <= 128
   list, 2 = emit distance keys + radix select; tail: 0 = list merges (or none: emit), 1 = radix select over the grid's
   keys staged in shared memory, 2 = radix select reading them from L2; query: 1 = in the kernel parameters, 0 = in
   device memory}.  All zero before the first scan.  Read it while no search runs.  WAX_VS_ERR_UNSUPPORTED on a
   multi-device handle. */
int32_t wax_vs_debug_last_scan(wax_vs_engine *engine, uint32_t out[10]);

/* Device-only timing of the batched path (n_queries synthetic unit queries per step, everything resident):
   total milliseconds of `iters` steps (CUDA events on the launching stream), kernel launches in the bracket and
   the number of queries of the last step whose proof did not complete (they would be re-run exactly). */
int32_t wax_vs_debug_time_search_batch(wax_vs_engine *engine, uint32_t n_queries, int64_t top_k, uint64_t seed,
                                       uint32_t warmup, uint32_t iters, float *out_ms_total,
                                       uint64_t *out_launches, uint32_t *out_unproven);

/* Read-out of the batched path's nomination stage (tests): runs the tensor-core nomination + exact finish for
   `n_queries` host queries and top_k <= 128 in the form the options select (batch_bf16, batch_ares, batch_pair,
   batch_heap), optionally with a row filter (`allow_bits`: one bit per row, set = allowed; NULL = all rows).
   out_scores [n_queries][count] receives every nomination score' the epilogue compared against its threshold (after
   the cosine row scale; l2: score' = q.v - |v|^2 / 2, larger = nearer); out_ok [n_queries] the proof flags; out_heaps [slices * groups][kprime][128] the nominee heaps
   as dumped (key = (orderable(-score') << 32) | row); out_shape[7] = {bf16, resident queries, CTA pair, ring stages,
   kprime, slices, groups}.  A batch that needs more than one launch -> WAX_VS_ERR_ARGUMENT; heaps_cap below the
   heap entries -> WAX_VS_ERR_BUFFER with everything but the heaps written. */
int32_t wax_vs_debug_batch_nominations(wax_vs_engine *engine, const float *queries, uint32_t n_queries, int64_t top_k,
                                       const uint32_t *allow_bits, float *out_scores, uint32_t *out_ok,
                                       uint64_t *out_heaps, uint64_t heaps_cap, uint32_t *out_shape);

/* Read-out of the single-query bf16-shadow route's first two launches (tests): for one host query and top_k <= 32, the
   SHADOW form of the scan nominates 128 rows from the bf16 shadow and the finish re-scores them exactly and proves the
   result -- the route's own launch code, in the shape the options select (shadow_rows_per_step, shadow_warps,
   shadow_stages, grid, chunk_steps, tail_select), whatever "shadow_scan", "shadow_scan_min_bytes" and the skip window
   after a failed proof say; the proof counters are not touched.  `allow_bits`: optional row filter (one bit per row,
   set = allowed).  out_keys[128] receives the nominee keys in the layout the finish reads (entry 0 = the worst of the
   128, entries 1..127 = the best first; key = (orderable(-score') << 32) | row, padding 0xFFFFFFFFFFFFFFFF);
   out_ok[1] the proof flag; out_result[min(top_k, count)] the finish's candidates (frame_id resolved); out_shape[7] =
   {rows per 128-dim chunk C, rows per step, warps, stages, grid, chunk_steps (0 = static), tail_select}.
   WAX_VS_ERR_UNSUPPORTED when the route cannot run: l2, dims not a multiple of 128 up to 1536, top_k > 32, no
   shadow, an empty corpus or a requested shape whose ring does not fit. */
int32_t wax_vs_debug_shadow_nominations(wax_vs_engine *engine, const float *query, int64_t top_k, const uint32_t *allow_bits,
                                        uint64_t *out_keys, uint32_t *out_ok, wax_vs_candidate *out_result,
                                        uint32_t *out_shape);

/* The bf16 shadow of rows [first, first + n) (brought up to date first): dims bf16 bit patterns per row, cosine rows
   pre-scaled by 1/|v|.  WAX_VS_ERR_UNSUPPORTED when the engine keeps no shadow (batch_bf16 = 0, dims % 64 != 0, or it
   did not fit in device memory). */
int32_t wax_vs_debug_read_shadow(wax_vs_engine *engine, uint64_t first, uint64_t n, uint16_t *dst);

/* The int8 form of wax_vs_debug_shadow_nominations: the same read-out with the INT8 form of the scan nominating from the
   int8 shadow, in the shape the options select (int8_rows_per_step, int8_warps, int8_stages, grid, chunk_steps,
   tail_select), and the finish proving with that shadow's measured bound -- whatever "int8_scan_min_bytes" and the
   bound's size say (a corpus whose bound is coarser than the bf16 one is read out too: the search would take the bf16
   route).  Nominee keys carry score' = s * (q . c).  WAX_VS_ERR_UNSUPPORTED as for the bf16 read-out, or when the int8
   shadow does not fit in device memory. */
int32_t wax_vs_debug_int8_nominations(wax_vs_engine *engine, const float *query, int64_t top_k, const uint32_t *allow_bits,
                                      uint64_t *out_keys, uint32_t *out_ok, wax_vs_candidate *out_result,
                                      uint32_t *out_shape);

/* The int8 shadow of rows [first, first + n) (brought up to date first): dst_codes[n][dims] the stored bytes (code + 128;
   cosine rows pre-scaled by 1/|v| before coding), dst_scales[n] each row's scale s, *out_rho_max the measured bound:
   >= ||v^ - s (byte - 128)||_2 for every row, +inf when a row is not finite.  WAX_VS_ERR_UNSUPPORTED for l2, dims not a
   multiple of 128 up to 1536, or when the int8 shadow does not fit in device memory. */
int32_t wax_vs_debug_read_int8_shadow(wax_vs_engine *engine, uint64_t first, uint64_t n, uint8_t *dst_codes,
                                      float *dst_scales, float *out_rho_max);

/* The 4-bit form of wax_vs_debug_shadow_nominations: the U4 form of the scan nominates from the 4-bit shadow in the shape
   the options select (u4_rows_per_step, u4_warps, u4_stages, grid, chunk_steps) and the grid-wide re-score proves --
   whatever "u4_scan_min_bytes" and the demotion say.  Every CTA of the scan writes its best 256 keys: out_keys takes
   out_shape[4] * 256 of them (unordered, padding 0xFFFF...; WAX_VS_ERR_BUFFER when keys_cap is smaller), score' =
   fl(fl(s_q h) (2 sum c_q u - 15 sum c_q)).  out_bound[3] = {rho_max of the shadow, rho_q of this query's int8 coding,
   tau_excl: the score' no left-out row exceeds, -inf when no row was left out}. */
int32_t wax_vs_debug_u4_nominations(wax_vs_engine *engine, const float *query, int64_t top_k, const uint32_t *allow_bits,
                                    uint64_t *out_keys, uint64_t keys_cap, uint32_t *out_ok, wax_vs_candidate *out_result,
                                    uint32_t *out_shape, float *out_bound);

/* The 4-bit shadow of rows [first, first + n) (brought up to date first): dst_codes[n][dims / 2] the stored bytes (byte b of
   word w: element 8w + b in the low nibble, 8w + 4 + b in the high one; cosine rows pre-scaled by 1/|v| before coding),
   dst_half_steps[n] each row's half step h (the row decodes to h (2u - 15)), *out_rho_max the measured bound as for int8.
   WAX_VS_ERR_UNSUPPORTED as for the int8 read-out. */
int32_t wax_vs_debug_read_u4_shadow(wax_vs_engine *engine, uint64_t first, uint64_t n, uint8_t *dst_codes,
                                    float *dst_half_steps, float *out_rho_max);

/* Streaming-read ceiling on the same box: a plain coalesced LDG.128 read of the live corpus bytes, best of
   `iters` (milliseconds, and the bytes read).  Context for the roofline fraction (SURVEY.md section 8d). */
int32_t wax_vs_debug_stream_read(wax_vs_engine *engine, uint32_t iters, float *out_best_ms, uint64_t *out_bytes);

/* Tuning knobs for experiments ("variant", "ctas_per_sm", ...).  Unknown key -> WAX_VS_ERR_ARGUMENT.
   "batch_l2" (default 0): 1 lets l2 batches take the tensor-core levels of wax_vs_search_batch, _batch_filtered and
   _batch_device (and wax_vs_debug_time_search_batch / wax_vs_debug_batch_nominations); 0 loops the exact scan.  The
   default is to flip once the l2 levels have been measured on the H100.
   "filter_bitset_bytes" (default 2 GiB): device memory the row bitsets of one tensor pass of
   wax_vs_search_batch_multi_filtered may use; at least one bitset always fits.
   "shadow_scan" (default 1): 0 sends every single query to the fp32 scan (the bf16-shadow route off);
   "shadow_scan_min_bytes" (default 512 MiB): the smallest fp32 corpus that takes that route;
   "shadow_rows_per_step" / "shadow_warps" / "shadow_stages" (0 = auto): the shape of its nominating scan;
   "int8_scan_min_bytes" (default 512 MiB): the smallest fp32 corpus whose route nominates from the int8 shadow (when it
   fits and its measured bound is no coarser than the bf16 one); setting it also retries an int8 shadow that did not fit;
   "int8_rows_per_step" / "int8_warps" / "int8_stages" (0 = auto): the shape of the INT8 nominating scan;
   "u4_scan_min_bytes" (default 2 GiB): the smallest fp32 corpus whose route nominates from the 4-bit shadow (when it
   fits with a finite bound; a failed 4-bit proof sends the next 16 eligible queries, doubling, to the int8 form); setting
   it also retries a 4-bit shadow that did not fit and ends a demotion;
   "u4_rows_per_step" / "u4_warps" / "u4_stages" (0 = auto): the shape of the U4 nominating scan. */
int32_t wax_vs_debug_set_option(wax_vs_engine *engine, const char *key, int64_t value);

/* Library build info: "waxvs_cuda <version> sm_90a ...". */
const char *wax_vs_version(void);

#ifdef __cplusplus
}
#endif
#endif /* WAX_VS_CUDA_H */
