// waxvs_roots.cuh -- root clauses of a where (wax_vs_search_batch_where_roots,
// wax_vs_search_batch_grouped_multi_where_roots): PhotoRAG's and VideoRAG's test on each hit's root frame
// (PhotoRAGOrchestrator.swift:280-286, VideoRAGOrchestrator.swift:314-318: the root has meta, is kind == root, is not
// deleted and not superseded) as a predicate on a 64-bit tag word kept per group, evaluated on the device.
//
// The caller keeps the words by group id (wax_vs_set_root_tags); the host holds them as a table sorted by id.  A search
// with a root clause reads them through a per-row column, col[row] = the word of row's group (8 bytes per row), built from
// the group index of grouped search (waxvs_group.cuh: ids[G] ascending, CSR starts[G+1] / perm[N]) by root_column_kernel
// and kept until the rows, the grouping or the table change.  A per-row column, not a gather through row_group[row] into
// a per-group table, so that the where passes stream it beside the AttrRows even when every row is its own group.
#pragma once
#include <cstdint>

namespace waxvs {

// col[row] = the word of row's group, for every row of the group index.  Warp w takes the dense groups
// [32 w', 32 w' + 32) for w' = w, w + warps, ...: lane j finds group 32 w' + j's id in the sorted table root_ids[0, n_roots)
// (a group not in it has word 0), then the warp writes each of those groups' rows perm[starts[g], starts[g + 1]) in turn.
__global__ void root_column_kernel(const uint64_t *__restrict__ group_ids, const uint32_t *__restrict__ starts,
                                   const uint32_t *__restrict__ perm, uint32_t n_groups,
                                   const uint64_t *__restrict__ root_ids, const uint64_t *__restrict__ root_tags,
                                   uint32_t n_roots, uint64_t *__restrict__ col) {
    const uint32_t lane = threadIdx.x & 31u;
    const uint32_t warps = (gridDim.x * blockDim.x) >> 5;
    for (uint32_t g0 = ((blockIdx.x * blockDim.x + threadIdx.x) >> 5) << 5; g0 < n_groups; g0 += warps << 5) {  // warp-uniform
        const uint32_t g = g0 + lane;
        uint64_t word = 0;
        uint32_t begin = 0, end = 0;
        if (g < n_groups) {
            const uint64_t id = group_ids[g];
            uint32_t lo = 0, hi = n_roots;             // first table id >= the group's
            while (lo < hi) {
                const uint32_t mid = (lo + hi) >> 1;
                if (root_ids[mid] < id) lo = mid + 1u; else hi = mid;
            }
            if (lo < n_roots && root_ids[lo] == id) word = root_tags[lo];
            begin = starts[g];
            end = starts[g + 1];
        }
        const uint32_t n_here = min(32u, n_groups - g0);
        for (uint32_t k = 0; k < n_here; ++k) {
            const uint64_t w = __shfl_sync(0xFFFFFFFFu, word, k);
            const uint32_t b = __shfl_sync(0xFFFFFFFFu, begin, k), e = __shfl_sync(0xFFFFFFFFu, end, k);
            for (uint32_t j = b + lane; j < e; j += 32u) col[perm[j]] = w;
        }
    }
}

}  // namespace waxvs
