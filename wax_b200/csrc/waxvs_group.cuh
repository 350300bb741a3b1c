// waxvs_group.cuh -- grouped search: the best rows of the best groups (wax_vs_search_grouped).
//
// Wax's PhotoRAG / VideoRAG callers want the best k PHOTOS or VIDEOS, each a root frame plus many derived frames with
// their own embeddings (PhotoRAGOrchestrator.swift:244-308, VideoRAGOrchestrator.swift:252-350,406-440).  They over-fetch
// frames and group the hits on the host; here the grouping runs below the top-k, over the per-row distance keys the
// large-k scan already emits (scan_*_kernel<..., EMIT = true>):
//   group index (cached per corpus version): the rows sorted by (group id, row) -- perm[pos] = row, starts[g] = the first
//     position of dense group g -- and row_group[row] = g;
//   group_reduce_kernel: each group's best (key, row) over its CSR positions -> best[g] (64-bit atomicMin after a per-lane
//     run and a per-warp combine, so one group holding half the corpus costs a few atomics per 512 positions);
//   group_keys_kernel: a row-indexed key array holding best[g]'s key at best[g]'s row and WAXVS_UKEY_NONE elsewhere, fed
//     unchanged to the radix select (waxvs_select.cuh): its k smallest are the top groups' best rows in the total order;
//   group_expand_kernel (per_group > 1): per selected group, the per_group best rows; a group is cut into tiles of
//     kExpandTile positions, one CTA sorts a tile and keeps its per_group best, further levels merge those lists
//     kExpandTile keys at a time -- the work is spread over the whole grid however skewed the groups are.
#pragma once
#include "waxvs_common.cuh"
#include "waxvs_scan.cuh"

namespace waxvs {

constexpr uint32_t kExpandTile = 2048;        // keys one expansion CTA sorts in shared memory
constexpr uint32_t kReduceRun = 16;           // consecutive CSR positions one lane reduces

// ---- group index build ----------------------------------------------------------------------------------------------
// Sort input: key = group id of row r (explicit array, else the frame id: ids[r] or id_base + r), value = r.
__global__ void group_sort_input_kernel(uint64_t *__restrict__ keys, uint32_t *__restrict__ vals, uint32_t n,
                                        const uint64_t *__restrict__ groups, const uint64_t *__restrict__ ids,
                                        uint64_t id_base) {
    for (uint32_t r = blockIdx.x * blockDim.x + threadIdx.x; r < n; r += gridDim.x * blockDim.x) {
        keys[r] = groups ? groups[r] : (ids ? ids[r] : id_base + r);
        vals[r] = r;
    }
}

// heads[pos] = 1 where a new group starts in the sorted keys.
__global__ void group_heads_kernel(const uint64_t *__restrict__ sorted, uint32_t n, uint32_t *__restrict__ heads) {
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x)
        heads[i] = (i == 0 || sorted[i] != sorted[i - 1]) ? 1u : 0u;
}

// incl[pos] = inclusive prefix sum of heads = dense group index + 1.  starts[n_groups] = n is written by the host.
__global__ void group_finish_kernel(const uint32_t *__restrict__ perm, const uint32_t *__restrict__ incl, uint32_t n,
                                    uint32_t *__restrict__ row_group, uint32_t *__restrict__ starts) {
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        const uint32_t g = incl[i] - 1u;
        row_group[perm[i]] = g;
        if (i == 0 || incl[i - 1] != incl[i]) starts[g] = i;
    }
}

// ids[g] = the group id of dense group g (its run head in the sorted keys): ascending, so a group id's dense index is a
// binary search away, and row r's group id is ids[row_group[r]].
__global__ void group_ids_kernel(const uint64_t *__restrict__ sorted, const uint32_t *__restrict__ starts,
                                 uint32_t n_groups, uint64_t *__restrict__ ids) {
    for (uint32_t g = blockIdx.x * blockDim.x + threadIdx.x; g < n_groups; g += gridDim.x * blockDim.x)
        ids[g] = sorted[starts[g]];
}

// ---- per query --------------------------------------------------------------------------------------------------------
// best[g] (initialised to WAXVS_KEY_NONE) = min over g's rows of (dist_key << 32 | row); dropped rows do not take part.
// Lane L of a warp reduces positions [base + 16 L, base + 16 L + 16): a finished run is flushed with one atomicMin, the
// open run at the end is first combined across the lanes that share its group (one atomic per group per warp).
__global__ void __launch_bounds__(256) group_reduce_kernel(const uint32_t *__restrict__ perm,
                                                           const uint32_t *__restrict__ row_group,
                                                           const uint32_t *__restrict__ dist_keys, uint32_t n,
                                                           unsigned long long *__restrict__ best) {
    const uint32_t lane = threadIdx.x & 31u;
    const uint64_t warp = (static_cast<uint64_t>(blockIdx.x) * blockDim.x + threadIdx.x) >> 5;
    const uint64_t warps = (static_cast<uint64_t>(gridDim.x) * blockDim.x) >> 5;
    for (uint64_t base = warp * 32u * kReduceRun; base < n; base += warps * 32u * kReduceRun) {
        uint32_t cur_g = 0xFFFFFFFFu;
        uint64_t cur = WAXVS_KEY_NONE;
        const uint64_t p0 = base + static_cast<uint64_t>(lane) * kReduceRun;
        for (uint32_t j = 0; j < kReduceRun; ++j) {
            const uint64_t pos = p0 + j;
            if (pos >= n) break;
            const uint32_t row = perm[pos];
            const uint32_t g = row_group[row];
            if (g != cur_g) {
                if (cur != WAXVS_KEY_NONE) atomicMin(best + cur_g, static_cast<unsigned long long>(cur));
                cur_g = g;
                cur = WAXVS_KEY_NONE;
            }
            const uint32_t uk = dist_keys[row];
            if (uk != WAXVS_UKEY_NONE) {
                const uint64_t key = (static_cast<uint64_t>(uk) << 32) | row;
                cur = key < cur ? key : cur;
            }
        }
        // open runs: lanes with the same group combine first (hi word, then the row among the lanes holding the min)
        const uint32_t peers = __match_any_sync(WAXVS_FULL_MASK, cur_g);
        const uint32_t hi = static_cast<uint32_t>(cur >> 32);
        const uint32_t min_hi = __reduce_min_sync(peers, hi);
        const uint32_t lo = (hi == min_hi) ? static_cast<uint32_t>(cur) : 0xFFFFFFFFu;
        const uint32_t min_lo = __reduce_min_sync(peers, lo);
        const uint64_t m = (static_cast<uint64_t>(min_hi) << 32) | min_lo;
        if (lane == static_cast<uint32_t>(__ffs(peers) - 1) && m != WAXVS_KEY_NONE)
            atomicMin(best + cur_g, static_cast<unsigned long long>(m));
    }
}

// gkeys[r] = the distance key of row r if r is its group's best row, else WAXVS_UKEY_NONE.
__global__ void group_keys_kernel(const uint32_t *__restrict__ row_group, const unsigned long long *__restrict__ best,
                                  uint32_t n, uint32_t *__restrict__ gkeys) {
    for (uint32_t r = blockIdx.x * blockDim.x + threadIdx.x; r < n; r += gridDim.x * blockDim.x) {
        const uint64_t b = best[row_group[r]];
        gkeys[r] = (b != WAXVS_KEY_NONE && static_cast<uint32_t>(b) == r) ? static_cast<uint32_t>(b >> 32) : WAXVS_UKEY_NONE;
    }
}

// The selected groups' CSR spans: spans[i] = (first position, rows) of the group of candidate i (valid = 0: (0, 0)).
__global__ void group_spans_kernel(const wax_vs_candidate *__restrict__ cands, uint32_t n_sel,
                                   const uint32_t *__restrict__ row_group, const uint32_t *__restrict__ starts,
                                   uint2 *__restrict__ spans) {
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n_sel; i += gridDim.x * blockDim.x) {
        uint2 s = make_uint2(0u, 0u);
        if (cands[i].valid) {
            const uint32_t g = row_group[cands[i].row];
            s = make_uint2(starts[g], starts[g + 1] - starts[g]);
        }
        spans[i] = s;
    }
}

// One expansion work item: sort `count` (<= kExpandTile) keys and keep the `per_group` smallest at dst[dst_off ...].
// Level 0 reads CSR positions [begin, begin + count) (key = dist_key << 32 | row, dropped rows = WAXVS_KEY_NONE);
// later levels read `count` keys at src[begin] (earlier lists of per_group keys each, padded with WAXVS_KEY_NONE).
struct ExpandItem {
    uint32_t begin, count, dst_off, final_out;   // final_out: 1 = write to the result, 0 = to the next level's input
};

__global__ void __launch_bounds__(1024) group_expand_kernel(const ExpandItem *__restrict__ items, uint32_t level0,
                                                            const uint32_t *__restrict__ perm,
                                                            const uint32_t *__restrict__ dist_keys,
                                                            const uint64_t *__restrict__ src, uint32_t per_group,
                                                            uint64_t *__restrict__ scratch_out, uint64_t *__restrict__ result) {
    __shared__ uint64_t sk[kExpandTile];
    const ExpandItem it = items[blockIdx.x];
    uint32_t pow2 = 32;
    while (pow2 < it.count || pow2 < per_group) pow2 <<= 1;
    for (uint32_t i = threadIdx.x; i < pow2; i += blockDim.x) {
        uint64_t key = WAXVS_KEY_NONE;
        if (i < it.count) {
            if (level0) {
                const uint32_t row = perm[it.begin + i];
                const uint32_t uk = dist_keys[row];
                if (uk != WAXVS_UKEY_NONE) key = (static_cast<uint64_t>(uk) << 32) | row;
            } else {
                key = src[it.begin + i];
            }
        }
        sk[i] = key;
    }
    __syncthreads();
    for (uint32_t size = 2; size <= pow2; size <<= 1) {
        for (uint32_t stride = size >> 1; stride > 0; stride >>= 1) {
            for (uint32_t i = threadIdx.x; i < pow2 / 2; i += blockDim.x) {
                const uint32_t lo = (i / stride) * (2 * stride) + (i % stride);
                const uint32_t hi = lo + stride;
                const bool asc = ((lo & size) == 0);
                const uint64_t a = sk[lo], b = sk[hi];
                if ((a > b) == asc) { sk[lo] = b; sk[hi] = a; }
            }
            __syncthreads();
        }
    }
    uint64_t *dst = (it.final_out ? result : scratch_out) + it.dst_off;
    for (uint32_t i = threadIdx.x; i < per_group; i += blockDim.x) dst[i] = sk[i];
}

}  // namespace waxvs
