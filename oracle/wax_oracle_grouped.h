/*
 * wax_oracle_grouped.h -- CPU ORACLE for grouped search (wax_vs_search_grouped).
 *
 * THIS IS TEST INFRASTRUCTURE, NOT PRODUCT CODE (see wax_oracle.h).  It is compiled together with wax_oracle.c into
 * libwax_oracle_grouped.so and restates, in plain C and with the distances of wax_oracle_distance, what Wax's
 * PhotoRAG / VideoRAG callers compute on the host after an over-fetching search: the hits mapped to their root
 * (parentId ?? id) and the best rows kept per root (PhotoRAGOrchestrator.swift:264-308,
 * VideoRAGOrchestrator.swift:273-350,406-440) -- made exact and total:
 *   - rows that take part: allowed (mask NULL = all) and with a finite distance;
 *   - ranked by (distance ascending, row ascending);
 *   - a group's rank is the position of its best row in that order (ties between groups go to the lower row);
 *   - the answer is the first min(clamp(top_groups), #groups taking part) groups, each with its
 *     min(per_group, its rows taking part) best rows;
 *   - group-major output: groups best first, rows best first within a group.
 */
#ifndef WAX_ORACLE_GROUPED_H
#define WAX_ORACLE_GROUPED_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

/* row_group[r] = group id of row r; allowed[r] != 0 = row r may take part (NULL = every row).  Outputs need room for
   min(clamp(top_groups) * per_group, n_rows) entries: rows (+ row_base), distances, scores, group ids.  per_group must
   be >= 1.  threads <= 1: one host thread for the distances.  Returns 0, or -1 on bad arguments. */
int wax_oracle_search_grouped(int metric, int mode, const float *corpus, uint64_t n_rows, uint32_t dims,
                              const float *query, const uint64_t *row_group, const uint8_t *allowed, int64_t top_groups,
                              uint32_t per_group, uint64_t row_base, int threads, uint64_t *out_rows,
                              float *out_distances, float *out_scores, uint64_t *out_groups, uint32_t *out_n);

/* The same over the synthetic rows [first_row, first_row + n_rows) of generator `seed`, for n_queries queries in one
   streamed pass (a row is generated once for all queries; no n_rows x dims host buffer).  Outputs are
   [n_queries][cap] with cap = min(clamp(top_groups) * per_group, n_rows); out_n[q] = entries of query q.  Rows are
   reported relative to first_row. */
int wax_oracle_search_grouped_synth(int metric, int mode, uint64_t seed, uint64_t first_row, uint64_t n_rows,
                                    uint32_t dims, int normalize, const float *queries, uint32_t n_queries,
                                    const uint64_t *row_group, const uint8_t *allowed, int64_t top_groups,
                                    uint32_t per_group, int threads, uint64_t *out_rows, float *out_distances,
                                    float *out_scores, uint64_t *out_groups, uint32_t *out_n);

#ifdef __cplusplus
}
#endif
#endif
