// waxvs_group_batch.cuh -- batched grouped search (wax_vs_search_batch_grouped): the top groups of many queries from
// each query's exact top-k_c rows.
//
// A group ranks by its best row in the total order (distance, row), so in ANY prefix of that order -- here the exact
// top-k_c rows the batched (filtered) search already computes -- the groups appear, by first occurrence, in rank order,
// every group missing from the prefix ranks below all that appear, and a group's rows in the prefix are its best rows.
//   group_cover_kernel: per query, the first clamp(top_groups) distinct groups of the list and their listed rows; a query
//     whose list names too few groups (and does not hold every allowed row) is crowded and takes the single-query path;
//     a selected group with fewer listed rows than per_group whose CSR span holds more rows needs an expansion;
//   group_score_tile_kernel: expansion level 0 -- scores a tile of a group's CSR positions exactly for one query and
//     keeps the per_group best; later levels merge the tiles' lists with group_expand_kernel, as the single query does.
#pragma once
#include "waxvs_batch.cuh"
#include "waxvs_group.cuh"

namespace waxvs {

// |q|^2 of one query, computed by every lane of the warp in the order of gather_score_kernel's prelude (the a2 that
// exact_row_distance takes; gather_score_kernel inlines the same loop).
__device__ __forceinline__ float query_sq_norm(const float *query, uint32_t dims, int lane) {
    float s0 = 0.f, s1 = 0.f, s2 = 0.f, s3 = 0.f;
    for (uint32_t base = 4u * lane; base < dims; base += 128u) {
        const float x = __ldg(query + base); s0 = __fmaf_rn(x, x, s0);
        if (base + 1 < dims) { const float y = __ldg(query + base + 1); s1 = __fmaf_rn(y, y, s1); }
        if (base + 2 < dims) { const float z = __ldg(query + base + 2); s2 = __fmaf_rn(z, z, s2); }
        if (base + 3 < dims) { const float w = __ldg(query + base + 3); s3 = __fmaf_rn(w, w, s3); }
    }
    return warp_butterfly_sum(__fadd_rn(__fadd_rn(s0, s1), __fadd_rn(s2, s3)));
}

constexpr uint32_t kCoverMax = 1024;          // longest coverage list: one list entry per thread of the cover kernel

// A selected group whose best rows must be scored exactly: query (staged index), its rank among the query's groups,
// its CSR span.
struct CoverExpand {
    uint32_t query, slot, begin, count;
};

// Level-0 expansion work item: score CSR positions [begin, begin + count) (<= kExpandTile) for query `query` and keep
// the per_group smallest keys at dst_off of the result (final_out = 1) or of the next level's input.  mask_slot: the
// bitset of the query's row filter in the pass's masks, or WAX_VS_NO_FILTER (unfiltered).
struct ScoreItem {
    uint32_t query, begin, count, dst_off, final_out, mask_slot;
};

// One CTA of kCoverMax threads per query.  cands + q * k_list: the query's exact top-k_list rows, best first (invalid
// entries = fewer allowed finite rows).  out + q * n_top * per_group receives [n_top][per_group] keys (dist_key << 32 |
// row), padded with WAXVS_KEY_NONE; status[q] = 1 covered, 0 crowded; groups to expand are appended to expand[].
__global__ void __launch_bounds__(kCoverMax) group_cover_kernel(const wax_vs_candidate *__restrict__ cands, uint32_t k_list,
                                                                 uint32_t k_c, const uint32_t *__restrict__ row_group,
                                                                 const uint32_t *__restrict__ starts, uint32_t n_top,
                                                                 uint32_t per_group, uint64_t *__restrict__ out,
                                                                 uint32_t *__restrict__ status,
                                                                 CoverExpand *__restrict__ expand,
                                                                 uint32_t *__restrict__ n_expand) {
    __shared__ uint64_t sk[kCoverMax];         // (dense group << 32 | list index), sorted: a group's entries form a run
    __shared__ uint32_t s_rank[kCoverMax];     // per list index: its rank among its group's listed rows
    __shared__ uint32_t s_cnt[kCoverMax];      // per list index: its group's listed rows
    __shared__ uint32_t s_first[kCoverMax];    // per list index: the list index of its group's first occurrence
    __shared__ uint32_t s_grank[kCoverMax];    // per first occurrence: the group's rank
    __shared__ uint32_t s_warp[kCoverMax / 32];
    const uint32_t t = threadIdx.x, q = blockIdx.x, lane = t & 31u, warp = t >> 5;
    const wax_vs_candidate *cq = cands + static_cast<size_t>(q) * k_list;
    bool valid = false;
    uint32_t row = 0, g = 0;
    float dist = 0.0f;
    if (t < k_list && cq[t].valid) {
        valid = true;
        row = static_cast<uint32_t>(cq[t].row);
        dist = cq[t].distance;
        g = row_group[row];
    }
    sk[t] = valid ? ((static_cast<uint64_t>(g) << 32) | t) : WAXVS_KEY_NONE;
    const uint32_t n_valid = __syncthreads_count(valid);    // the valid entries are the list's first n_valid
    block_bitonic_sort(sk, kCoverMax);
    if (t < n_valid) {
        const uint64_t key = sk[t];
        const uint64_t g_lo = key & 0xFFFFFFFF00000000ull, g_hi = g_lo + (1ull << 32);
        uint32_t lo = 0, hi = t;                              // first sorted position of the group
        while (lo < hi) { const uint32_t mid = (lo + hi) >> 1; if (sk[mid] < g_lo) lo = mid + 1; else hi = mid; }
        const uint32_t run0 = lo;
        hi = n_valid;                                         // first sorted position past the group
        lo = t + 1;
        while (lo < hi) { const uint32_t mid = (lo + hi) >> 1; if (sk[mid] < g_hi) lo = mid + 1; else hi = mid; }
        const uint32_t idx = static_cast<uint32_t>(key);
        s_rank[idx] = t - run0;
        s_cnt[idx] = lo - run0;
        s_first[idx] = static_cast<uint32_t>(sk[run0]);
    }
    __syncthreads();
    // group ranks: first occurrences counted in list order
    const bool first = valid && s_rank[t] == 0;
    const uint32_t ballot = __ballot_sync(WAXVS_FULL_MASK, first);
    if (lane == 0) s_warp[warp] = __popc(ballot);
    __syncthreads();
    uint32_t before = 0, n_groups = 0;
    for (uint32_t w = 0; w < kCoverMax / 32; ++w) {
        before += w < warp ? s_warp[w] : 0u;
        n_groups += s_warp[w];
    }
    if (first) s_grank[t] = before + __popc(ballot & ((1u << lane) - 1u));
    const bool complete = n_valid < k_c;                     // the list holds every allowed row with a finite distance
    const bool covered = complete || n_groups >= n_top;
    if (t == 0) status[q] = covered ? 1u : 0u;
    if (!covered) return;                                    // block-uniform
    uint64_t *oq = out + static_cast<size_t>(q) * n_top * per_group;
    for (uint32_t i = t; i < n_top * per_group; i += blockDim.x) oq[i] = WAXVS_KEY_NONE;
    __syncthreads();
    if (!valid) return;
    const uint32_t gr = s_grank[s_first[t]], rank = s_rank[t], cnt = s_cnt[t];
    if (gr >= n_top) return;
    if (rank < per_group) oq[gr * per_group + rank] = (static_cast<uint64_t>(orderable_u32(dist)) << 32) | row;
    if (first && cnt < per_group && !complete) {
        const uint32_t begin = starts[g], count = starts[g + 1] - begin;
        if (count > cnt) expand[atomicAdd(n_expand, 1u)] = CoverExpand{q, gr, begin, count};
    }
}

// Expansion level 0 for a batch: item `blockIdx.x` scores its CSR positions for its query, exactly (warp per row, the
// kernels' operation order, so the bits equal the scan's); rows outside the item's filter (bit clear in bitset
// mask_slot of `masks`, `words` words each) or with a non-finite distance drop out.  The tile is sorted in shared memory
// and its per_group best are kept.
template <int METRIC>
__global__ void __launch_bounds__(256) group_score_tile_kernel(const ScoreItem *__restrict__ items, const float *corpus,
                                                                const float *queries, uint32_t dims,
                                                                const uint32_t *__restrict__ perm,
                                                                const uint32_t *__restrict__ masks, uint32_t words,
                                                                uint32_t per_group,
                                                                uint64_t *__restrict__ scratch_out,
                                                                uint64_t *__restrict__ result) {
    __shared__ uint64_t sk[kExpandTile];
    const ScoreItem it = items[blockIdx.x];
    const int lane = threadIdx.x & 31;
    const float *query = queries + static_cast<size_t>(it.query) * dims;
    const uint32_t *mask = it.mask_slot == WAX_VS_NO_FILTER ? nullptr : masks + static_cast<size_t>(it.mask_slot) * words;
    float a2 = 0.0f, sqrt_a2 = 0.0f;
    if (METRIC == kCosine) {
        a2 = query_sq_norm(query, dims, lane);
        sqrt_a2 = __fsqrt_rn(a2);
    }
    uint32_t pow2 = 32;
    while (pow2 < it.count || pow2 < per_group) pow2 <<= 1;
    for (uint32_t i = it.count + threadIdx.x; i < pow2; i += blockDim.x) sk[i] = WAXVS_KEY_NONE;
    const uint32_t warps = blockDim.x >> 5;
    for (uint32_t i0 = threadIdx.x >> 5; i0 < it.count; i0 += 4u * warps) {
        uint32_t rr[4];
        const float *vp[4];
        float d[4];
#pragma unroll
        for (uint32_t r = 0; r < 4; ++r) {
            const uint32_t i = i0 + r * warps;
            rr[r] = perm[it.begin + (i < it.count ? i : i0)];
            vp[r] = corpus + static_cast<size_t>(rr[r]) * dims;
        }
        exact_row_distance_x4<METRIC>(query, vp, dims, a2, sqrt_a2, lane, d);
        if (lane == 0) {
#pragma unroll
            for (uint32_t r = 0; r < 4; ++r) {
                const uint32_t i = i0 + r * warps;
                if (i >= it.count) continue;
                const bool allowed = !mask || ((mask[rr[r] >> 5] >> (rr[r] & 31u)) & 1u);
                sk[i] = (allowed && finite_f32(d[r])) ? make_key(d[r], rr[r]) : WAXVS_KEY_NONE;
            }
        }
    }
    __syncthreads();
    block_bitonic_sort(sk, pow2);
    uint64_t *dst = (it.final_out ? result : scratch_out) + it.dst_off;
    for (uint32_t i = threadIdx.x; i < per_group; i += blockDim.x) dst[i] = sk[i];
}

// ---- sharded grouped search (wax_vs_shard_grouped_heads_device / _expand_device) --------------------------------------
// A rank's rows as the records the ranks exchange: global row, frame id (ids[row] or id_base + row) and group id
// (group_ids[row_group[row]]).  key = dist_key << 32 | local row; WAXVS_KEY_NONE is padding (all zero).
struct ShardRowInfo {
    uint64_t row_offset, id_base;
    const uint64_t *ids;                     // nullptr: identity ids
    const uint64_t *row_keys;                // keyed shard: global row = row_offset + row_keys[row] (nullptr: + row)
    const uint32_t *row_group;
    const uint64_t *group_ids;
};
__device__ __forceinline__ wax_vs_group_candidate shard_group_record(uint64_t key, const ShardRowInfo &ri) {
    wax_vs_group_candidate c{};
    if (key != WAXVS_KEY_NONE) {
        const uint32_t row = static_cast<uint32_t>(key);
        c.distance = from_orderable_u32(static_cast<uint32_t>(key >> 32));
        c.valid = 1u;
        c.row = ri.row_offset + (ri.row_keys ? ri.row_keys[row] : row);
        c.frame_id = ri.ids ? ri.ids[row] : ri.id_base + row;
        c.group_id = ri.group_ids[ri.row_group[row]];
    }
    return c;
}

// Round 1: the covered staged queries' result keys ([staged][slots]) -> their caller slots of heads ([query][slots]);
// staged query j is query order[j], covered when status[j] != 0 (the others are delivered by the host).
__global__ void __launch_bounds__(256) shard_group_heads_kernel(const uint64_t *__restrict__ keys, uint32_t n_staged,
                                                                uint32_t slots, const uint32_t *__restrict__ order,
                                                                const uint32_t *__restrict__ status, const ShardRowInfo ri,
                                                                wax_vs_group_candidate *__restrict__ heads) {
    const size_t total = static_cast<size_t>(n_staged) * slots;
    for (size_t i = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < total;
         i += static_cast<size_t>(gridDim.x) * blockDim.x) {
        const uint32_t j = static_cast<uint32_t>(i / slots), s = static_cast<uint32_t>(i % slots);
        if (status[j]) heads[static_cast<size_t>(order[j]) * slots + s] = shard_group_record(keys[i], ri);
    }
}

// Round 2, one warp per chosen (query, slot) of [n_queries][n_top]: a group this rank listed for the query in round 1
// (own heads) is copied into rows ([query][slot][per_group]); a group the shard holds (its id found among the index's
// sorted group ids) is appended to `expand` with its CSR span; anything else stays padding (the caller zeroed `rows`).
__global__ void __launch_bounds__(256) shard_group_lookup_kernel(const wax_vs_group_candidate *__restrict__ chosen,
                                                                 const wax_vs_group_candidate *__restrict__ own,
                                                                 uint32_t n_queries, uint32_t n_top, uint32_t per_group,
                                                                 const uint64_t *__restrict__ group_ids, uint32_t n_groups,
                                                                 const uint32_t *__restrict__ starts,
                                                                 wax_vs_candidate *__restrict__ rows,
                                                                 CoverExpand *__restrict__ expand,
                                                                 uint32_t *__restrict__ n_expand) {
    const uint32_t lane = threadIdx.x & 31u;
    const uint64_t slot = (static_cast<uint64_t>(blockIdx.x) * blockDim.x + threadIdx.x) >> 5;
    if (slot >= static_cast<uint64_t>(n_queries) * n_top) return;      // warp-uniform
    const wax_vs_group_candidate ch = chosen[slot];
    if (!ch.valid) return;
    const uint32_t q = static_cast<uint32_t>(slot / n_top), s = static_cast<uint32_t>(slot % n_top);
    const wax_vs_group_candidate *oq = own + static_cast<size_t>(q) * n_top * per_group;
    uint32_t listed = 0xFFFFFFFFu;
    for (uint32_t g0 = 0; g0 < n_top && listed == 0xFFFFFFFFu; g0 += 32) {
        const uint32_t g = g0 + lane;
        const bool hit = g < n_top && oq[static_cast<size_t>(g) * per_group].valid &&
                         oq[static_cast<size_t>(g) * per_group].group_id == ch.group_id;
        const uint32_t b = __ballot_sync(WAXVS_FULL_MASK, hit);
        if (b) listed = g0 + __ffs(b) - 1;
    }
    if (listed != 0xFFFFFFFFu) {                                        // copy: already this shard's best rows
        for (uint32_t j = lane; j < per_group; j += 32) {
            const wax_vs_group_candidate h = oq[static_cast<size_t>(listed) * per_group + j];
            if (h.valid) rows[slot * per_group + j] = wax_vs_candidate{h.distance, 1u, h.row, h.frame_id};
        }
        return;
    }
    if (lane) return;
    uint32_t lo = 0, hi = n_groups;                                     // expansion: the group's rows on this shard
    while (lo < hi) {
        const uint32_t mid = (lo + hi) >> 1;
        if (group_ids[mid] < ch.group_id) lo = mid + 1; else hi = mid;
    }
    if (lo < n_groups && group_ids[lo] == ch.group_id)
        expand[atomicAdd(n_expand, 1u)] = CoverExpand{q, s, starts[lo], starts[lo + 1] - starts[lo]};
}

// Round 2: the expanded slots' keys ([query][slot][per_group] in keys) -> their candidate records in rows.
__global__ void __launch_bounds__(128) shard_group_expanded_kernel(const CoverExpand *__restrict__ expand,
                                                                   const uint64_t *__restrict__ keys, uint32_t n_top,
                                                                   uint32_t per_group, const ShardRowInfo ri,
                                                                   wax_vs_candidate *__restrict__ rows) {
    const CoverExpand x = expand[blockIdx.x];
    const size_t base = (static_cast<size_t>(x.query) * n_top + x.slot) * per_group;
    for (uint32_t j = threadIdx.x; j < per_group; j += blockDim.x) {
        const wax_vs_group_candidate c = shard_group_record(keys[base + j], ri);
        rows[base + j] = wax_vs_candidate{c.distance, c.valid, c.row, c.frame_id};
    }
}

}  // namespace waxvs
