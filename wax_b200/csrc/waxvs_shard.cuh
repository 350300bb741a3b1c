// waxvs_shard.cuh -- the row-sharded search's ONE exchange, fused into the scan launch.
//
// SURVEY.md section 8(e): the corpus shards row-wise across the GPUs of a node, every rank scans its shard for the
// replicated query and the per-shard top-k lists (k x 24 B per rank) are exchanged and merged under the same total
// order (distance ascending, GLOBAL row ascending).  The reference has no distributed code.  An all-gather of the lists
// + D2H + a host merge costs a sizeable part of a small shard's scan, so here the exchange is part of the scan kernel
// itself:
//
//   * every rank owns a MAILBOX in its HBM (ShardMailbox); peers map it (CUDA IPC between the one-process-per-GPU
//     ranks, plain peer access inside one process) and WRITE into it over NVLink / NVSwitch -- nobody ever reads
//     remote memory (a remote read is a round trip, a remote write is posted);
//   * the last CTA of the scan (the one that already merges the grid's block lists) pushes its k candidates into
//     slot [seq % depth][rank] of EVERY rank's mailbox, fences at system scope, raises flag[slot][rank] = seq on every
//     rank, then spins on its OWN mailbox until all `world` flags carry seq;
//   * it merges the world x k candidates (every list is sorted: a candidate's final position is its index plus, for
//     every other rank, a binary search of its (distance, global row) pair in that rank's list; the rows are read only
//     when distances tie, and padding is ordered by rank), writes the k best to the result buffer and, for the host
//     entry point, straight into mapped
//     pinned host memory followed by a host-visible flag: no collective launch, no D2H copy, no host merge;
//   * slot reuse is guarded by acknowledgements (acks[r] = last seq rank r has finished reading from its own mailbox),
//     so any number of queries may be in flight on any streams.
//
// Every rank computes the same merge from the same bytes, so all ranks return identical results (what an all-gather
// followed by a merge on every rank gives).  Spins carry a timeout (a rank that never arrives must not hang the GPU).
#pragma once
#include "waxvs_common.cuh"
#include "../../include/wax_vs_cuda.h"

namespace waxvs {

constexpr int kShardMaxRanks = 16;
constexpr int kShardDepth = 8;       // queries whose candidates a mailbox can hold at once
constexpr int kShardKCap = 128;      // = the fused top-k range

struct ShardMailbox {
    unsigned long long flags[kShardDepth][kShardMaxRanks];   // flags[s][r] = seq: rank r's candidates for seq are in cands[s][r]
    unsigned long long acks[kShardMaxRanks];                  // acks[r] = last seq rank r finished reading from ITS OWN mailbox
    wax_vs_candidate cands[kShardDepth][kShardMaxRanks][kShardKCap];
};

struct ShardParams {
    ShardMailbox *box[kShardMaxRanks];   // [rank] = own mailbox, others = peers' (device-accessible)
    uint32_t rank, world;                // world == 0: not sharded
    unsigned long long seq;              // 1, 2, 3, ... identical on every rank for the same query
    unsigned long long timeout_ns;
    wax_vs_candidate *final_out;         // [k] merged result (device)
    wax_vs_candidate *host_out;          // [k] merged result in mapped pinned host memory, or nullptr
    unsigned long long *host_flag;       // mapped pinned: seq when host_out is complete (bit 63 = exchange timed out)
};

constexpr unsigned long long kShardErrorBit = 1ull << 63;

__device__ __forceinline__ unsigned long long ld_acquire_sys_u64(const unsigned long long *p) {
    unsigned long long v;
    asm volatile("ld.acquire.sys.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ void st_release_sys_u64(unsigned long long *p, unsigned long long v) {
    asm volatile("st.release.sys.global.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}
__device__ __forceinline__ unsigned long long global_timer_ns() {
    unsigned long long t;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
    return t;
}

// Called by EVERY thread of one CTA.  `local` = this rank's sorted candidate list ([k], padding valid = 0 last), written
// to global memory by this CTA before the call.  `skeys` = shared-memory scratch of world * k uint32.
__device__ __noinline__ void shard_exchange_cta(const ShardParams &sh, const wax_vs_candidate *local, uint32_t k,
                                                uint32_t *skeys) {
    const uint32_t tid = threadIdx.x, nthr = blockDim.x;
    const uint32_t slot = static_cast<uint32_t>(sh.seq % kShardDepth);
    ShardMailbox *mine = sh.box[sh.rank];
    __shared__ uint32_t s_err;
    if (tid == 0) s_err = 0;
    __syncthreads();   // also: the caller's writes of local[] are visible to the whole CTA

    // 1. the slot is free once every rank has finished reading what it held `depth` queries ago
    if (tid < sh.world && sh.seq > kShardDepth) {
        const unsigned long long need = sh.seq - kShardDepth, t0 = global_timer_ns();
        while (ld_acquire_sys_u64(&mine->acks[tid]) < need)
            if (global_timer_ns() - t0 > sh.timeout_ns) { s_err = 1; break; }
    }
    __syncthreads();

    // 2. push the local list into every rank's mailbox (posted NVLink writes; own mailbox included)
    for (uint32_t i = tid; i < sh.world * k; i += nthr) {
        const uint32_t r = i / k, j = i % k;
        const unsigned long long *src = reinterpret_cast<const unsigned long long *>(local + j);
        unsigned long long *dst = reinterpret_cast<unsigned long long *>(&sh.box[r]->cands[slot][sh.rank][j]);
        dst[0] = src[0]; dst[1] = src[1]; dst[2] = src[2];
    }
    __threadfence_system();
    __syncthreads();
    if (tid < sh.world) st_release_sys_u64(&sh.box[tid]->flags[slot][sh.rank], sh.seq);

    // 3. wait for every rank's list
    if (tid < sh.world) {
        const unsigned long long t0 = global_timer_ns();
        while (ld_acquire_sys_u64(&mine->flags[slot][tid]) < sh.seq)
            if (global_timer_ns() - t0 > sh.timeout_ns) { s_err = 1; break; }
    }
    __syncthreads();
    const bool failed = s_err != 0;

    // 4. merge: distance keys of all lists in shared memory, final position by binary searches
    const uint32_t total = sh.world * k;
    for (uint32_t i = tid; i < total; i += nthr) {
        const unsigned long long w0 = ld_cg_u64(reinterpret_cast<const uint64_t *>(&mine->cands[slot][i / k][i % k]));
        const uint32_t valid = static_cast<uint32_t>(w0 >> 32);
        skeys[i] = (valid == 1u && !failed) ? orderable_u32(__uint_as_float(static_cast<uint32_t>(w0))) : WAXVS_UKEY_NONE;
    }
    __syncthreads();
    for (uint32_t i = tid; i < total; i += nthr) {
        const uint32_t r = i / k, j = i % k, key = skeys[i];
        const unsigned long long row = key == WAXVS_UKEY_NONE ? 0ull : ld_cg_u64(reinterpret_cast<const uint64_t *>(&mine->cands[slot][r][j]) + 1);
        uint32_t pos = j;
        for (uint32_t r2 = 0; r2 < sh.world && pos < k; ++r2) {
            if (r2 == r) continue;
            const uint32_t *lst = skeys + r2 * k;
            uint32_t lo = 0, hi = k;
            while (lo < hi) {                       // entries before (key, row); equal distances read the rows
                const uint32_t mid = (lo + hi) >> 1, v = lst[mid];
                bool before = v < key;
                if (v == key)
                    before = key == WAXVS_UKEY_NONE ? r2 < r
                                                    : ld_cg_u64(reinterpret_cast<const uint64_t *>(&mine->cands[slot][r2][mid]) + 1) < row;
                if (before) lo = mid + 1; else hi = mid;
            }
            pos += lo;
        }
        if (pos < k) {
            const uint64_t *src = reinterpret_cast<const uint64_t *>(&mine->cands[slot][r][j]);
            unsigned long long w0 = ld_cg_u64(src), w1 = ld_cg_u64(src + 1), w2 = ld_cg_u64(src + 2);
            if (key == WAXVS_UKEY_NONE) { w0 = 0; w1 = 0; w2 = 0; }        // padding: valid = 0
            unsigned long long *dst = reinterpret_cast<unsigned long long *>(sh.final_out + pos);
            dst[0] = w0; dst[1] = w1; dst[2] = w2;
            if (sh.host_out) {
                unsigned long long *hd = reinterpret_cast<unsigned long long *>(sh.host_out + pos);
                hd[0] = w0; hd[1] = w1; hd[2] = w2;
            }
        }
    }
    __threadfence_system();
    __syncthreads();

    // 5. tell every rank this mailbox slot has been read; tell the host the result is complete
    if (tid < sh.world) st_release_sys_u64(&sh.box[tid]->acks[sh.rank], sh.seq);
    if (tid == 0 && sh.host_flag) st_release_sys_u64(sh.host_flag, failed ? (sh.seq | kShardErrorBit) : sh.seq);
}

// Stand-alone form (one CTA): the local list was produced by earlier work on the stream (an empty shard, a scan
// configuration whose shared-memory lists are too small for the fused form).
__global__ void __launch_bounds__(256) shard_exchange_kernel(const ShardParams sh, const wax_vs_candidate *local, uint32_t k) {
    __shared__ uint32_t skeys[kShardMaxRanks * kShardKCap];
    shard_exchange_cta(sh, local, k, skeys);
}

// ------------------------------------------------------------------------------------------------------------
// Batched form of the same merge (sharded search_batch): `gathered` = [world][n_queries][k] candidates as an all-gather
// of the ranks' per-query lists leaves them (every list sorted, padding valid = 0 last); out = [n_queries][k_out], the
// k_out best of each query under (distance, GLOBAL row) -- the position rule of shard_exchange_cta, binary searches in
// global memory.  One CTA per query.  Replaces a host-side numpy merge, which costs more than a shard's tensor-core
// pass.  The rule needs no order between the ranks' rows, so it holds for keyed shards, whose rows interleave.
__device__ __forceinline__ uint32_t cand_dist_key(const wax_vs_candidate &c) {
    return c.valid ? orderable_u32(c.distance) : WAXVS_UKEY_NONE;
}
// Candidate (km, m) of rank o comes before candidate (key, c) of rank r: by distance, then global row; padding by rank.
__device__ __forceinline__ bool cand_before(uint32_t km, const wax_vs_candidate &m, uint32_t o, uint32_t key,
                                            const wax_vs_candidate &c, uint32_t r) {
    if (km != key) return km < key;
    return key == WAXVS_UKEY_NONE ? o < r : m.row < c.row;
}
// How a merge finds rank r's records: one rank-major gathered buffer, as an all-gather leaves it ...
template <class T>
struct GatheredLists {
    const T *base;
    size_t rank_stride;                    // the records of one rank
    __device__ __forceinline__ const T *operator()(uint32_t r) const { return base + r * rank_stride; }
};
// ... or a table of per-rank buffers, each on its rank's device and read here over peer memory (the multi-device handle,
// waxvs_multi.cuh).  The table rides in the kernel parameters.
template <class T>
struct PeerLists {
    const T *list[kShardMaxRanks];
    __device__ __forceinline__ const T *operator()(uint32_t r) const { return list[r]; }
};
template <class Lists>
__global__ void __launch_bounds__(128) merge_gathered_kernel(const Lists lists, uint32_t world, uint32_t n_queries, uint32_t k,
                                                             uint32_t k_out, wax_vs_candidate *__restrict__ out) {
    const uint32_t q = blockIdx.x;
    const size_t at = static_cast<size_t>(q) * k;                    // this query's list in every rank's buffer
    for (uint32_t t = threadIdx.x; t < world * k; t += blockDim.x) {
        const uint32_t r = t / k, j = t % k;
        const wax_vs_candidate c = lists(r)[at + j];
        const uint32_t key = cand_dist_key(c);
        uint32_t pos = j;
        for (uint32_t o = 0; o < world; ++o) {
            if (o == r) continue;
            const wax_vs_candidate *lst = lists(o) + at;
            uint32_t lo = 0, hi = k;
            while (lo < hi) {
                const uint32_t mid = (lo + hi) >> 1;
                if (cand_before(cand_dist_key(lst[mid]), lst[mid], o, key, c, r)) lo = mid + 1; else hi = mid;
            }
            pos += lo;
        }
        if (pos < k_out) out[static_cast<size_t>(q) * k_out + pos] = c;
    }
}

// ------------------------------------------------------------------------------------------------------------
// Sharded grouped search, merge 1 (wax_vs_merge_group_heads_device): the ranks' round-1 answers gathered as
// [world][n_queries][G][P] -> per query the global top G groups, each as its best row.  A group's head on a rank is its
// best row there, so its global head is the best of its heads; a group is ranked by that head in (distance, GLOBAL row).
// The heads are sorted by their rows first, and then by (distance key, row rank), which is (distance, global row) for any
// placement of rows on ranks.
constexpr uint32_t kShardMaxGroups = 256;   // = WAX_VS_SHARD_MAX_GROUPS: world * G <= 4 096 heads in shared memory

// Sorts (key[i], val[i]) pairs ascending by key, then val (pow2 entries, every thread of the CTA).
__device__ __forceinline__ void block_bitonic_sort_pairs(uint64_t *key, uint32_t *val, uint32_t pow2) {
    for (uint32_t size = 2; size <= pow2; size <<= 1) {
        for (uint32_t stride = size >> 1; stride > 0; stride >>= 1) {
            for (uint32_t i = threadIdx.x; i < pow2 / 2; i += blockDim.x) {
                const uint32_t lo = (i / stride) * (2 * stride) + (i % stride), hi = lo + stride;
                const bool asc = ((lo & size) == 0);
                const uint64_t ka = key[lo], kb = key[hi];
                const uint32_t va = val[lo], vb = val[hi];
                const bool greater = ka > kb || (ka == kb && va > vb);
                if (greater == asc) { key[lo] = kb; key[hi] = ka; val[lo] = vb; val[hi] = va; }
            }
            __syncthreads();
        }
    }
}

// One CTA per query; dynamic shared memory: pow2 * 20 bytes, pow2 = the power of two >= max(world * G, 32).
// `lists` finds rank r's [n_queries][G][P] records (GatheredLists or PeerLists).
template <class Lists>
__global__ void __launch_bounds__(1024) merge_group_heads_kernel(const Lists lists, uint32_t world, uint32_t n_queries,
                                                                 uint32_t n_top, uint32_t per_group, uint32_t pow2,
                                                                 wax_vs_group_candidate *__restrict__ chosen) {
    extern __shared__ uint64_t heads_smem[];
    uint64_t *s_key = heads_smem;                                      // [pow2]
    uint32_t *s_val = reinterpret_cast<uint32_t *>(heads_smem + pow2); // [pow2]
    uint32_t *s_head = s_val + pow2;                                   // [pow2] head index at each ordered position
    uint32_t *s_keep = s_head + pow2;                                  // [pow2] 1: the position is its group's best head
    __shared__ uint32_t s_warp[32], s_total;
    const uint32_t q = blockIdx.x, t = threadIdx.x, heads = world * n_top;
    auto head = [&](uint32_t i) -> const wax_vs_group_candidate & {
        return lists(i / n_top)[(static_cast<size_t>(q) * n_top + i % n_top) * per_group];
    };
    // 1. every rank's heads in (distance, global row) order: the rank of each head's row, then (distance key, row rank)
    uint32_t mine = 0;
    for (uint32_t i = t; i < pow2; i += blockDim.x) {
        const bool v = i < heads && head(i).valid;
        s_key[i] = v ? head(i).row : ~0ull;
        s_val[i] = i;
        mine += v;
    }
    for (uint32_t i = t; i < pow2; i += blockDim.x) s_keep[i] = 0;
    if (t == 0) s_total = 0;
    __syncthreads();
    atomicAdd(&s_total, mine);
    block_bitonic_sort_pairs(s_key, s_val, pow2);                       // ends in __syncthreads
    for (uint32_t p = t; p < pow2; p += blockDim.x) s_head[s_val[p]] = p;
    __syncthreads();
    for (uint32_t i = t; i < pow2; i += blockDim.x) {
        const bool v = i < heads && head(i).valid;
        s_key[i] = v ? (static_cast<uint64_t>(orderable_u32(head(i).distance)) << 32 | s_head[i]) : ~0ull;
        s_val[i] = v ? i : 0xFFFFFFFFu;
    }
    __syncthreads();
    block_bitonic_sort_pairs(s_key, s_val, pow2);
    const uint32_t valid = s_total;
    // 2. by (group id, position): the first position of each group id is its best head
    for (uint32_t p = t; p < pow2; p += blockDim.x) {
        s_head[p] = s_val[p];
        s_key[p] = p < valid ? head(s_val[p]).group_id : ~0ull;
        s_val[p] = p < valid ? p : 0xFFFFFFFFu;
    }
    __syncthreads();
    block_bitonic_sort_pairs(s_key, s_val, pow2);
    for (uint32_t j = t; j < valid; j += blockDim.x)
        if (j == 0 || s_key[j - 1] != s_key[j]) s_keep[s_val[j]] = 1u;
    __syncthreads();
    // 3. the kept heads' ranks: an exclusive scan over the ordered positions, each thread a run of `per` of them
    const uint32_t per = (pow2 + blockDim.x - 1) / blockDim.x, lane = t & 31u, warp = t >> 5;
    uint32_t local = 0;
    for (uint32_t e = 0; e < per; ++e) {
        const uint32_t p = t * per + e;
        if (p < valid) local += s_keep[p];
    }
    uint32_t incl = local;
    for (uint32_t o = 1; o < 32; o <<= 1) {
        const uint32_t y = __shfl_up_sync(WAXVS_FULL_MASK, incl, o);
        if (lane >= o) incl += y;
    }
    if (lane == 31) s_warp[warp] = incl;
    __syncthreads();
    if (warp == 0) {
        const uint32_t nw = blockDim.x >> 5;
        uint32_t w = lane < nw ? s_warp[lane] : 0u;
        for (uint32_t o = 1; o < 32; o <<= 1) {
            const uint32_t y = __shfl_up_sync(WAXVS_FULL_MASK, w, o);
            if (lane >= o) w += y;
        }
        if (lane < nw) s_warp[lane] = w;                               // inclusive per warp
    }
    __syncthreads();
    uint32_t rank = (warp ? s_warp[warp - 1] : 0u) + incl - local;
    const uint32_t kept = s_warp[(blockDim.x >> 5) - 1];
    wax_vs_group_candidate *out = chosen + static_cast<size_t>(q) * n_top;
    for (uint32_t e = 0; e < per; ++e) {
        const uint32_t p = t * per + e;
        if (p < valid && s_keep[p]) {
            if (rank < n_top) out[rank] = head(s_head[p]);
            ++rank;
        }
    }
    for (uint32_t s = kept + t; s < n_top; s += blockDim.x) out[s] = wax_vs_group_candidate{};
}

// ------------------------------------------------------------------------------------------------------------
// The device form of a batched where search (wax_vs_search_batch_where_device) stages and answers its queries in the
// plan's order.  order[j] = the caller's query that staged query j is; k_of[j] = the slots of its list that were written.
__global__ void __launch_bounds__(256) stage_query_rows_kernel(const float *__restrict__ queries,
                                                               const uint32_t *__restrict__ order, uint32_t n,
                                                               uint32_t dims, float *__restrict__ staged) {
    const size_t total = static_cast<size_t>(n) * dims;
    for (size_t i = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < total;
         i += static_cast<size_t>(gridDim.x) * blockDim.x) {
        const uint32_t j = static_cast<uint32_t>(i / dims), d = static_cast<uint32_t>(i % dims);
        staged[i] = queries[static_cast<size_t>(order[j]) * dims + d];
    }
}
// Staged query j's first k_of[j] candidates (at staged + j * k_max) -> out[order[j]][0, k_of[j]) of k_out slots each.
// The caller zeroed `out`, so every other slot is padding (valid = 0).  k_of[j] <= k_max <= k_out.
__global__ void __launch_bounds__(256) scatter_candidates_kernel(const wax_vs_candidate *__restrict__ staged, uint32_t k_max,
                                                                 const uint32_t *__restrict__ order,
                                                                 const uint32_t *__restrict__ k_of, uint32_t n,
                                                                 uint32_t k_out, wax_vs_candidate *__restrict__ out) {
    const size_t total = static_cast<size_t>(n) * k_max;
    for (size_t i = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < total;
         i += static_cast<size_t>(gridDim.x) * blockDim.x) {
        const uint32_t j = static_cast<uint32_t>(i / k_max), s = static_cast<uint32_t>(i % k_max);
        if (s < k_of[j]) out[static_cast<size_t>(order[j]) * k_out + s] = staged[i];
    }
}

}  // namespace waxvs
