/*
 * wax_oracle.h -- CPU ORACLE for Wax's brute-force vector scan + top-k.
 *
 * THIS IS TEST INFRASTRUCTURE, NOT PRODUCT CODE.  Only tests/, __graft_entry__.smoke()
 * and bench.py's cpu_baseline / --impl reference legs may load it.  The product path
 * (wax_b200/, libwaxvs_cuda.so) never links, imports or falls back to anything here.
 *
 * Parity status: "parity unpinned" beyond the reference's own known-answer tests.
 *   The reference (christopherkarani/Wax) is Swift 6.2 / Apple-only; neither engine can be built
 *   here (no Swift toolchain, no Metal, USearch 2.23.0 is an un-vendored SwiftPM dependency --
 *   Package.resolved:113-120).  The oracle is therefore a *restatement*, pinned against every
 *   known-answer the reference's tests hold for this path (tests/golden/reference_kats.json,
 *   transcribed with file:line) and nothing stronger exists upstream (SURVEY.md section 8c).
 *
 * What is restated (all paths relative to the root of the Wax repository):
 *   - USearch metric formulas reached through VectorMetric.toUSearchMetric()
 *     (Sources/WaxVectorSearch/VectorMetric.swift:21-30): cos / ip / l2sq, as published in
 *     unum-cloud/USearch 2.23.0 include/usearch/index_plugins.hpp (metric_cos_gt, metric_ip_gt,
 *     metric_l2sq_gt):  cos = 1 - ab/(sqrt(a2)*sqrt(b2)) with {one zero norm -> 1, both -> 0};
 *     ip = 1 - ab;  l2sq = sum (a-b)^2.
 *   - VectorMetric.score(fromDistance:)      VectorMetric.swift:32-43
 *   - engine search semantics (empty -> [], dim check, clamp k to [1,10000], min(k,N) rows,
 *     ascending distance, non-finite candidates dropped)
 *                                            MetalVectorEngine.swift:446-455,595-603,842-846
 *                                            USearchVectorEngine.swift:201-216,331-335
 *   - VectorMath.normalizeL2 / isNormalizedL2 Sources/Wax/Utilities/VectorMath.swift:15-33,123-127
 *   - Metal kernel cosine (assumes |q|=1, guard 1e-6)   Shaders/CosineDistance.metal:233-328
 *   - Metal CPU-fallback heap top-k          MetalVectorEngine.swift:630-680
 *   - "MV2V" encoding=2 blob                 MetalVectorEngine.swift:682-815,
 *                                            VectorSerializer.swift:84-157,175-251
 *   - the benchmark embedder's value generator (FNV-1a -> 64-bit LCG -> [-1,1] -> L2 normalise)
 *                                            Tests/WaxIntegrationTests/RAGBenchmarkSupport.swift:130-156
 *
 * Ordering: the reference leaves ties unspecified (unstable bitonic/heap,
 * TopKReduction.metal:84-101, MetalVectorEngine.swift:671,678).  The oracle (and the CUDA kernels)
 * fix the total order (distance ascending, row ascending).
 */
#ifndef WAX_ORACLE_H
#define WAX_ORACLE_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

/* VecSimilarity raw values (Sources/WaxCore/FileFormat/MV2SEnums.swift:34-38). */
enum { WAX_ORACLE_COSINE = 0, WAX_ORACLE_DOT = 1, WAX_ORACLE_L2 = 2 };

/* Accumulation modes. */
enum {
    /* fp32, one running sum per quantity, element order 0..D-1, separate multiply and add:
       the scalar loop of USearch's metric_*_gt / the reference's in-test cosine
       (MiniLMEmbeddingQualityTests.swift:37-52).  This is the "reference order". */
    WAX_ORACLE_ACC_F32_SEQ = 0,
    /* fp64 accumulation of the fp32 inputs, result rounded to fp32 once: ground truth for
       tolerance and tie analysis. */
    WAX_ORACLE_ACC_F64 = 1,
    /* fp32 FMA with 128 interleaved accumulators (element i -> accumulator i mod 128), combined
       ((a0+a1)+(a2+a3)) per group of four and then by a 32-leaf xor-butterfly tree (16,8,4,2,1).
       Same real-number formula, different rounding order: this is exactly the order the CUDA
       kernels use, so CUDA-vs-oracle in this mode must be BIT-EXACT.  It is also the order that
       vectorises on the host, so it is the mode timed as cpu_baseline. */
    WAX_ORACLE_ACC_F32_TREE = 2
};

#define WAX_ORACLE_MAX_RESULTS 10000   /* MetalVectorEngine.swift:18, USearchVectorEngine.swift:6 */
#define WAX_ORACLE_MAX_DIMS 1000000    /* Sources/WaxCore/Constants.swift:51 */

/* ---- scalar pieces ---------------------------------------------------------------------- */

/* VectorMetric.score(fromDistance:)  (VectorMetric.swift:32-43). */
float wax_oracle_score_from_distance(int metric, float d);

/* clampTopK (MetalVectorEngine.swift:842-846; USearchVectorEngine.swift:331-335). */
int64_t wax_oracle_clamp_topk(int64_t top_k);

/* USearch distance between query a and document b under `metric`, accumulation `mode`. */
float wax_oracle_distance(int metric, int mode, const float *a, const float *b, uint32_t dims);

/* Metal kernel cosine distance: 1 - dot/sqrt(sum v^2), NOT divided by |q|; |v| <= 1e-6 -> distance 1
   (CosineDistance.metal:233-328).  fp32 sequential.  Used only to document the deviation. */
float wax_oracle_metal_cosine_distance(const float *q, const float *v, uint32_t dims);

/* VectorMath.normalizeL2 (VectorMath.swift:15-33): s = sum x^2, m = sqrt(s), m > 0 -> x * (1/m),
   else copy.  fp32 sequential sum. */
void wax_oracle_normalize_l2(const float *in, float *out, uint32_t n);
/* VectorMath.isNormalizedL2 (VectorMath.swift:123-127): n > 0 && |sqrt(sum x^2) - 1| <= tol. */
int wax_oracle_is_normalized_l2(const float *v, uint32_t n, float tol);

/* ---- exact scan + top-k ------------------------------------------------------------------- */

/* Scan `n_rows` row-major fp32 rows of `dims` floats, return the min(clamp(top_k), #finite) best.
   out_* need room for min(clamp(top_k), n_rows).  Rows are reported as row + row_base.
   threads <= 1: single host thread; else that many pthreads (row partition + merge).
   Returns 0, or -1 on bad arguments. */
int wax_oracle_search(int metric, int mode, const float *corpus, uint64_t n_rows, uint32_t dims,
                      const float *query, int64_t top_k, uint64_t row_base, int threads,
                      uint64_t *out_rows, float *out_distances, float *out_scores, uint32_t *out_n);

/* Same scan over the synthetic corpus rows [first_row, first_row+n_rows) of generator `seed`,
   generated on the fly (no N*D host buffer). */
int wax_oracle_search_synth(int metric, int mode, uint64_t seed, uint64_t first_row, uint64_t n_rows,
                            uint32_t dims, int normalize, const float *query, int64_t top_k,
                            int threads, uint64_t *out_rows, float *out_distances,
                            float *out_scores, uint32_t *out_n);

/* Multi-query forms: the same scan for n_queries queries (row-major [n_queries][dims]) in ONE pass over the rows
   (a synthetic row is generated once for all queries).  Outputs are [n_queries][k] with
   k = min(clamp(top_k), n_rows); out_n[q] = results of query q.  Identical arithmetic, identical total order. */
int wax_oracle_search_multi(int metric, int mode, const float *corpus, uint64_t n_rows, uint32_t dims,
                            const float *queries, uint32_t n_queries, int64_t top_k, uint64_t row_base, int threads,
                            uint64_t *out_rows, float *out_distances, float *out_scores, uint32_t *out_n);
int wax_oracle_search_synth_multi(int metric, int mode, uint64_t seed, uint64_t first_row, uint64_t n_rows,
                                  uint32_t dims, int normalize, const float *queries, uint32_t n_queries,
                                  int64_t top_k, int threads, uint64_t *out_rows, float *out_distances,
                                  float *out_scores, uint32_t *out_n);

/* MetalVectorEngine.topK CPU heap (MetalVectorEngine.swift:630-680): k smallest of `distances`,
   boundary ties keep the earlier row (value >= heap[0] -> skip); final order here is made total
   (distance, row) because Swift's sort is not stable.  Returns count written. */
uint32_t wax_oracle_metal_cpu_topk(const float *distances, uint64_t count, uint32_t k,
                                   uint64_t *out_rows, float *out_distances);

/* ---- synthetic corpus (bit-exact twin of the CUDA generator) --------------------------------- */

/* Row `row` of stream `seed`: state0 = splitmix64_mix(fnv1a64(seed LE || row LE)); per component
   state = state*6364136223846793005 + 1442695040888963407; x = float(int64(state)) / float(INT64_MAX)
   (RAGBenchmarkSupport.swift:130-143); if normalize: s = fma-sequential sum x^2, x *= 1/sqrt(s). */
void wax_oracle_synth_row(uint64_t seed, uint64_t row, uint32_t dims, int normalize, float *out);
void wax_oracle_synth_rows(uint64_t seed, uint64_t first_row, uint64_t n_rows, uint32_t dims,
                           int normalize, int threads, float *out);

/* ---- MV2V encoding=2 blob ------------------------------------------------------------------ */

/* 36-byte header + count*dims LE f32 + u64 idBytes + count LE u64 (MetalVectorEngine.swift:682-714). */
uint64_t wax_oracle_mv2v_length(uint32_t dims, uint64_t count);
int wax_oracle_mv2v_encode(uint8_t similarity, uint32_t dims, uint64_t count, const float *vectors,
                           const uint64_t *frame_ids, uint8_t *dst, uint64_t cap, uint64_t *out_len);
/* Validates exactly as MetalVectorEngine.deserialize (:716-815) + VectorSerializer.decodeVecSegment
   (:84-157).  On success sets *out_count and pointers into `src`.  Returns 0 or a negative code:
   -1 too small, -2 magic, -3 version, -4 encoding, -5 similarity, -6 dims, -7 reserved bytes,
   -8 vector length, -9 missing id length, -10 id length, -11 total length. */
int wax_oracle_mv2v_decode(const uint8_t *src, uint64_t len, uint8_t expect_similarity,
                           uint32_t expect_dims, uint64_t *out_count, const uint8_t **out_vectors,
                           const uint8_t **out_ids);

#ifdef __cplusplus
}
#endif
#endif
