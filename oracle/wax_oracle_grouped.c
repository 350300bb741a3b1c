/* wax_oracle_grouped.c -- CPU oracle for grouped search (see wax_oracle_grouped.h).  Test infrastructure only. */
#include "wax_oracle_grouped.h"

#include <math.h>
#include <pthread.h>
#include <stdlib.h>
#include <string.h>

#include "wax_oracle.h"

typedef struct {
    float d;
    uint64_t row;
} Hit;

static int hit_cmp(const void *pa, const void *pb) {
    const Hit *a = (const Hit *)pa, *b = (const Hit *)pb;
    if (a->d < b->d) return -1;
    if (a->d > b->d) return 1;
    return (a->row > b->row) - (a->row < b->row);
}

static uint64_t mix64(uint64_t x) {
    x ^= x >> 30; x *= 0xbf58476d1ce4e5b9ull; x ^= x >> 27; x *= 0x94d049bb133111ebull; x ^= x >> 31;
    return x;
}

/* The selection of the semantics above over one query's distances dist[0 .. n_rows). */
static int grouped_select(int metric, const float *dist, uint64_t n_rows, const uint64_t *row_group,
                          const uint8_t *allowed, int64_t top_groups, uint32_t per_group, uint64_t row_base,
                          uint64_t *out_rows, float *out_distances, float *out_scores, uint64_t *out_groups,
                          uint32_t *out_n) {
    const uint64_t g_max = (uint64_t)wax_oracle_clamp_topk(top_groups);
    Hit *hits = (Hit *)malloc((n_rows ? n_rows : 1) * sizeof(Hit));
    if (!hits) return -1;
    uint64_t m = 0;
    for (uint64_t r = 0; r < n_rows; ++r)
        if ((!allowed || allowed[r]) && isfinite(dist[r])) { hits[m].d = dist[r]; hits[m].row = r; ++m; }
    qsort(hits, m, sizeof(Hit), hit_cmp);
    /* group id -> slot (selected group index), or -1 once the answer is full and the group was not selected */
    uint64_t cap = 64;
    while (cap < 2 * m + 16) cap <<= 1;
    uint64_t *keys = (uint64_t *)malloc(cap * sizeof(uint64_t));
    int64_t *slot = (int64_t *)malloc(cap * sizeof(int64_t));
    uint8_t *used = (uint8_t *)calloc(cap, 1);
    uint64_t *lists = (uint64_t *)malloc((g_max * per_group ? g_max * per_group : 1) * sizeof(uint64_t));
    uint32_t *counts = (uint32_t *)calloc(g_max, sizeof(uint32_t));
    uint64_t *gids = (uint64_t *)malloc(g_max * sizeof(uint64_t));
    if (!keys || !slot || !used || !lists || !counts || !gids) {
        free(hits); free(keys); free(slot); free(used); free(lists); free(counts); free(gids);
        return -1;
    }
    uint64_t n_sel = 0;
    for (uint64_t i = 0; i < m; ++i) {
        const uint64_t g = row_group[hits[i].row];
        uint64_t h = mix64(g) & (cap - 1);
        while (used[h] && keys[h] != g) h = (h + 1) & (cap - 1);
        if (!used[h]) {
            used[h] = 1; keys[h] = g;
            if (n_sel < g_max) { slot[h] = (int64_t)n_sel; gids[n_sel] = g; ++n_sel; }
            else slot[h] = -1;
        }
        if (slot[h] < 0) continue;
        const uint64_t s = (uint64_t)slot[h];
        if (counts[s] < per_group) lists[s * per_group + counts[s]++] = hits[i].row;
    }
    uint32_t k = 0;
    for (uint64_t s = 0; s < n_sel; ++s)
        for (uint32_t j = 0; j < counts[s]; ++j) {
            const uint64_t r = lists[s * per_group + j];
            out_rows[k] = r + row_base;
            out_distances[k] = dist[r];
            out_scores[k] = wax_oracle_score_from_distance(metric, dist[r]);
            out_groups[k] = gids[s];
            ++k;
        }
    *out_n = k;
    free(hits); free(keys); free(slot); free(used); free(lists); free(counts); free(gids);
    return 0;
}

/* ---- distances, partitioned over threads ------------------------------------------------------------------------ */
typedef struct {
    int metric, mode, normalize;
    const float *corpus;           /* NULL: synthetic rows */
    uint64_t seed, first_row;
    uint32_t dims;
    const float *queries;
    uint32_t n_queries;
    uint64_t n_rows, lo, hi;
    float *dist;                   /* [n_queries][n_rows] */
} Job;

static void *dist_worker(void *arg) {
    Job *j = (Job *)arg;
    float *row = j->corpus ? NULL : (float *)malloc((size_t)j->dims * sizeof(float));
    for (uint64_t r = j->lo; r < j->hi; ++r) {
        const float *v = row;
        if (j->corpus) v = j->corpus + r * j->dims;
        else wax_oracle_synth_row(j->seed, j->first_row + r, j->dims, j->normalize, row);
        for (uint32_t q = 0; q < j->n_queries; ++q)
            j->dist[(uint64_t)q * j->n_rows + r] =
                wax_oracle_distance(j->metric, j->mode, j->queries + (uint64_t)q * j->dims, v, j->dims);
    }
    free(row);
    return NULL;
}

static int distances(Job base, int threads, float *dist) {
    if (threads < 1) threads = 1;
    if ((uint64_t)threads > base.n_rows) threads = base.n_rows ? (int)base.n_rows : 1;
    Job *jobs = (Job *)malloc((size_t)threads * sizeof(Job));
    pthread_t *tid = (pthread_t *)malloc((size_t)threads * sizeof(pthread_t));
    if (!jobs || !tid) { free(jobs); free(tid); return -1; }
    const uint64_t per = (base.n_rows + threads - 1) / threads;
    for (int t = 0; t < threads; ++t) {
        jobs[t] = base;
        jobs[t].dist = dist;
        jobs[t].lo = per * t < base.n_rows ? per * t : base.n_rows;
        jobs[t].hi = per * (t + 1) < base.n_rows ? per * (t + 1) : base.n_rows;
    }
    for (int t = 1; t < threads; ++t) pthread_create(&tid[t], NULL, dist_worker, &jobs[t]);
    dist_worker(&jobs[0]);
    for (int t = 1; t < threads; ++t) pthread_join(tid[t], NULL);
    free(jobs); free(tid);
    return 0;
}

static int check_args(int metric, int mode, uint32_t dims, int64_t top_groups, uint32_t per_group) {
    (void)top_groups;
    if (metric < 0 || metric > 2 || mode < 0 || mode > 2 || dims == 0 || per_group == 0) return -1;
    return 0;
}

int wax_oracle_search_grouped(int metric, int mode, const float *corpus, uint64_t n_rows, uint32_t dims,
                              const float *query, const uint64_t *row_group, const uint8_t *allowed, int64_t top_groups,
                              uint32_t per_group, uint64_t row_base, int threads, uint64_t *out_rows,
                              float *out_distances, float *out_scores, uint64_t *out_groups, uint32_t *out_n) {
    if (!out_n || check_args(metric, mode, dims, top_groups, per_group)) return -1;
    *out_n = 0;
    if (n_rows == 0) return 0;
    if (!corpus || !query || !row_group) return -1;
    float *dist = (float *)malloc(n_rows * sizeof(float));
    if (!dist) return -1;
    Job base;
    memset(&base, 0, sizeof base);
    base.metric = metric; base.mode = mode; base.corpus = corpus; base.dims = dims;
    base.queries = query; base.n_queries = 1; base.n_rows = n_rows;
    int rc = distances(base, threads, dist);
    if (!rc)
        rc = grouped_select(metric, dist, n_rows, row_group, allowed, top_groups, per_group, row_base, out_rows,
                            out_distances, out_scores, out_groups, out_n);
    free(dist);
    return rc;
}

int wax_oracle_search_grouped_synth(int metric, int mode, uint64_t seed, uint64_t first_row, uint64_t n_rows,
                                    uint32_t dims, int normalize, const float *queries, uint32_t n_queries,
                                    const uint64_t *row_group, const uint8_t *allowed, int64_t top_groups,
                                    uint32_t per_group, int threads, uint64_t *out_rows, float *out_distances,
                                    float *out_scores, uint64_t *out_groups, uint32_t *out_n) {
    if (!out_n || check_args(metric, mode, dims, top_groups, per_group)) return -1;
    for (uint32_t q = 0; q < n_queries; ++q) out_n[q] = 0;
    if (n_rows == 0 || n_queries == 0) return 0;
    if (!queries || !row_group) return -1;
    uint64_t cap = (uint64_t)wax_oracle_clamp_topk(top_groups) * per_group;
    if (cap > n_rows) cap = n_rows;
    float *dist = (float *)malloc((uint64_t)n_queries * n_rows * sizeof(float));
    if (!dist) return -1;
    Job base;
    memset(&base, 0, sizeof base);
    base.metric = metric; base.mode = mode; base.normalize = normalize; base.seed = seed; base.first_row = first_row;
    base.dims = dims; base.queries = queries; base.n_queries = n_queries; base.n_rows = n_rows;
    int rc = distances(base, threads, dist);
    for (uint32_t q = 0; q < n_queries && !rc; ++q)
        rc = grouped_select(metric, dist + (uint64_t)q * n_rows, n_rows, row_group, allowed, top_groups, per_group, 0,
                            out_rows + q * cap, out_distances + q * cap, out_scores + q * cap, out_groups + q * cap,
                            out_n + q);
    free(dist);
    return rc;
}
