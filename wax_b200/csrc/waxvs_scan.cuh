// waxvs_scan.cuh -- the fused single-pass scan: query L2-norm + distance + top-k in ONE launch.
//
// Replaces, for the CUDA engine, the reference's two-dispatch pipeline
//   cosineDistanceKernelSIMD8/SIMD4  (Shaders/CosineDistance.metal:233-328, :152-229)  -> N*4 B distances
//   topKReduceDistances/Entries loop (Shaders/TopKReduction.metal:103-167; MetalVectorEngine.swift:511-575)
// and the host-side query normalisation (VectorSearchSession.swift:70-76).  The corpus is the only HBM
// stream: no distance array, no second pass.
//
// Data layout: corpus row-major [n_rows][dims] fp32 in HBM (as MetalVectorEngine.swift:134,345-349).
//
// Work split (HBM-bound, ~1 flop/byte -- deliberately NOT a GEMM):
//   * persistent grid, one CTA per SM; every warp owns a private ring of `stages` shared-memory tiles of
//     R rows and streams "steps" (R consecutive rows = R*dims*4 contiguous bytes) with 1-D TMA bulk copies
//     (cp.async.bulk -> SASS UBLKCP) completing on the warp's own mbarriers -- no block-wide barrier in
//     the main loop, (stages-1)*R*dims*4 bytes in flight per warp;
//   * a lane reads its 16-byte chunks (lane + 32c) of a row with conflict-free LDS.128, FMAs them against
//     the query chunks it keeps in registers into 4 accumulators per quantity (element i -> accumulator
//     i mod 128: the order oracle ACC_F32_TREE mirrors, so results are bit-exact against it);
//   * R rows are reduced together with a shuffle reduce-scatter (warp_reduce_scatter) and finished by the
//     lane that owns the row (IEEE sqrt/div, USearch zero-norm rules);
//   * each warp keeps a sorted k<=32 list in registers; a row is compared against the list's k-th key
//     (one 64-bit compare) and inserted by shuffles only when it wins (rare after warm-up);
//   * per-CTA merge in shared memory, per-grid merge by the last CTA to finish (atomic ticket): still the
//     same launch.
#pragma once
#include "waxvs_common.cuh"
#include "waxvs_shard.cuh"
#include "../../include/wax_vs_cuda.h"

namespace waxvs {

constexpr int kInlineQueryFloats = 512;

struct ScanParams {
    const float *corpus;        // [n_rows][dims]
    const float *query;         // [dims]
    uint32_t n_rows;
    uint32_t dims;
    uint32_t k;                 // entries to produce (<= 128 for the fused list kernels)
    uint32_t stages;            // ring depth per warp (TMA kernels)
    uint64_t *block_keys;       // [grid][32*E] scratch
    uint32_t *ticket;           // zero on entry, zero again on exit
    wax_vs_candidate *out;      // [k] results, best first
    uint32_t *dist_keys;        // emit mode: [n_rows] orderable distance keys (WAXVS_UKEY_NONE = dropped)
    const uint64_t *frame_ids;  // device ids or nullptr (then id = id_base + row)
    uint64_t id_base;
    uint64_t row_offset;        // added to the reported row (shard offset)
    const uint64_t *row_keys;   // keyed shard: row r is reported as row_offset + row_keys[r] (nullptr = row_offset + r)
    uint32_t use_l2_hint;       // 1: evict-first policy on the corpus stream
    uint32_t chunk_steps;       // > 0: dynamic scheduling, warps claim chunks of this many steps from work_counter
    uint32_t *work_counter;     // zero on entry, zero again on exit (reset by the last CTA)
    const uint32_t *mask;       // optional row filter: bit r of mask[r / 32] set = row r may be returned (nullptr = all)
    // Host delivery (the synchronous single-query entry point): the last CTA also stores the result into mapped pinned
    // host memory and then raises a host-visible flag, so the caller needs neither a D2H copy nor a stream
    // synchronisation; and a short query travels in the kernel parameters instead of through an H2D copy.
    wax_vs_candidate *host_out;         // [k] mapped pinned, or nullptr
    unsigned long long *host_flag;      // mapped pinned: set to host_seq once host_out is complete
    unsigned long long host_seq;
    alignas(16) float query_inline[kInlineQueryFloats];   // used when query == nullptr (TMA-staged kernels, dims <= kInlineQueryFloats)
    // Tail of the launch: 0 = pairwise bitonic merges of sorted lists (warp lists -> block list -> last CTA merges the
    // grid's block lists), 1 = exact radix SELECTION (finish_topk_select): block-wide k-th-smallest over the keys, the
    // last CTA selects over grid x k keys staged in `tail_smem_bytes` of the (by then idle) ring.  Same result bits.
    uint32_t tail_select;
    uint32_t tail_smem_bytes;
    unsigned long long *trace;  // instrumentation (wax_vs_debug_phase_trace) or nullptr: [0] min kernel start, [1] max end of a
                                // warp's scan loop, [2] max end of a CTA's selection, [3] start and [4] end of the last CTA's
                                // grid stage -- %globaltimer nanoseconds
    ShardParams shard;          // shard.world > 0: `out` is this rank's local list and the last CTA goes on to exchange it
                                // with the other ranks over NVLink and to merge (waxvs_shard.cuh): still the same launch
    // The bf16-shadow route of a single query (DESIGN 4.1): the SHADOW form nominates, batch_finish_kernel re-scores and
    // proves, then the fp32 form runs guarded by the proof.
    uint64_t *nominees;         // SHADOW: [k][kNomineeStride] the nominee keys, laid out as batch_finish_kernel's heaps of
                                // one query and one slice (entry 0 = the worst nominee, real only when all k are)
    float *query_store;         // SHADOW, query in the parameters: CTA 0 also stores it here for the launches that follow
    const uint32_t *proof_ok;   // fp32 cosine / dot, E = 1: non-null = guarded by the proof flag batch_finish_kernel wrote: when set
                                // every CTA returns at entry (CTA 0 first delivers `out` to the host), else a plain scan
    uint32_t *proof_count;      // guarded: [0] proofs that held, [1] that failed -- running counts on the device ...
    uint32_t *proof_count_host; // ... mirrored into mapped pinned memory, read by the host without synchronising
    const float *row_scale;     // INT8: [rows, padded to whole steps] the scale s of each int8 shadow row; U4: the half step h
    uint32_t *u4_aux;           // U4: [0] the smallest (key >> 32) any warp list or CTA selection cut rows at (every row left
                                // out has a key at or above it; 0xFFFFFFFF on entry = nothing cut), [1] rho_q (fp32 bits)
};

constexpr uint32_t kU4CtaNominees = 256;    // U4: nominees every CTA writes (the best of its warps' lists)

// batch_finish_kernel reads entry e of query 0's heap of slice 0 at e * kBatchM (static_assert in waxvs_batch.cuh).
constexpr int kNomineeStride = 128;

__device__ __forceinline__ bool row_allowed(const ScanParams &p, uint32_t row) {
    return p.mask == nullptr || ((__ldg(p.mask + (row >> 5)) >> (row & 31u)) & 1u) != 0u;
}

__device__ __forceinline__ void write_candidate(const ScanParams &p, int slot, uint64_t key) {
    wax_vs_candidate c;
    if (key == WAXVS_KEY_NONE) {
        c.distance = 0.0f; c.valid = 0; c.row = 0; c.frame_id = 0;
    } else {
        const uint32_t row = static_cast<uint32_t>(key);
        c.distance = from_orderable_u32(static_cast<uint32_t>(key >> 32));
        c.valid = 1;
        c.row = p.row_offset + (p.row_keys ? p.row_keys[row] : row);
        c.frame_id = p.frame_ids ? p.frame_ids[row] : p.id_base + row;
    }
    p.out[slot] = c;
    if (p.host_out) p.host_out[slot] = c;
}

// The tails' output: result slot `slot` (0 = best) -- a candidate, or (SHADOW) a nominee key, the worst of the k in
// entry 0 and slot i < k-1 in entry i+1.
template <bool SHADOW>
__device__ __forceinline__ void write_slot(const ScanParams &p, int slot, uint64_t key) {
    if constexpr (SHADOW) p.nominees[static_cast<size_t>(slot == static_cast<int>(p.k) - 1 ? 0 : slot + 1) * kNomineeStride] = key;
    else write_candidate(p, slot, key);
}

// bf16 x 4 (one uint2 of the shadow, element 0 in the low half) -> fp32, exactly.
__device__ __forceinline__ float4 bf16x4_to_float4(uint2 u) {
    return make_float4(__uint_as_float(u.x << 16), __uint_as_float(u.x & 0xFFFF0000u),
                       __uint_as_float(u.y << 16), __uint_as_float(u.y & 0xFFFF0000u));
}

// 4 biased int8 (one uint32 of the int8 shadow, byte b = c + 128, element 0 in the low byte) -> fp32 c, exactly: PRMT the
// byte under the exponent of 2^23 (0x4B0000bb = 2^23 + b), then subtract 2^23 + 128.
__device__ __forceinline__ float4 int8x4_to_float4(uint32_t u) {
    constexpr float kBias = 8388736.0f;     // 2^23 + 128
    return make_float4(__fsub_rn(__uint_as_float(__byte_perm(u, 0x4B000000u, 0x7650)), kBias),
                       __fsub_rn(__uint_as_float(__byte_perm(u, 0x4B000000u, 0x7651)), kBias),
                       __fsub_rn(__uint_as_float(__byte_perm(u, 0x4B000000u, 0x7652)), kBias),
                       __fsub_rn(__uint_as_float(__byte_perm(u, 0x4B000000u, 0x7653)), kBias));
}

// Reduce-scatter of H integer partial sums over each half-warp (the U4 form: 16 lanes share a row): on exit v[0] of lane
// L holds the 16-lane sum of entry (L & 15) / (16 / H) of its half.  Integer sums: exact in any order.
template <int H>
__device__ __forceinline__ void half_warp_reduce_scatter(int (&v)[H], int lane) {
    static_assert(H == 1 || H == 2 || H == 4 || H == 8, "H must be a power of two <= 8");
    int off = 8;
#pragma unroll
    for (int half = H / 2; half >= 1; half >>= 1, off >>= 1) {
        const bool upper = (lane & off) != 0;
#pragma unroll
        for (int j = 0; j < half; ++j) {
            const int send = upper ? v[j] : v[j + half];
            const int keep = upper ? v[j + half] : v[j];
            v[j] = keep + __shfl_xor_sync(WAXVS_FULL_MASK, send, off);
        }
    }
#pragma unroll
    for (; off >= 1; off >>= 1) v[0] += __shfl_xor_sync(WAXVS_FULL_MASK, v[0], off);
}

// CTA merge + grid merge + output.  Called by every thread of the CTA after the scan loop.
// lists: shared [warps][E*32] u64;  block_keys: global [grid][E*32].
template <int E, bool SHADOW = false>
__device__ __forceinline__ void finish_topk(const ScanParams &p, WarpTopK<E> &tk, uint64_t *lists, int warp,
                                            int lane, int warps) {
    const int k = static_cast<int>(p.k);
    constexpr int W = E * 32;
    __shared__ uint32_t s_last;
    auto load_list = [&](const uint64_t *src, uint64_t (&dst)[E]) {
#pragma unroll
        for (int j = 0; j < E; ++j) dst[j] = src[j * 32 + lane];
    };
#pragma unroll
    for (int j = 0; j < E; ++j) lists[warp * W + j * 32 + lane] = tk.key[j];
    __syncthreads();
    if (warp == 0) {
#pragma unroll 1
        for (int w = 1; w < warps; ++w) {
            uint64_t other[E];
            load_list(lists + w * W, other);
            tk.merge_sorted(other, lane, k);
        }
#pragma unroll
        for (int j = 0; j < E; ++j) p.block_keys[static_cast<size_t>(blockIdx.x) * W + j * 32 + lane] = tk.key[j];
        __threadfence();
        __syncwarp();
        if (lane == 0) s_last = (atomicAdd(p.ticket, 1u) == gridDim.x - 1) ? 1u : 0u;
    }
    __syncthreads();
    if (!s_last) return;
    __threadfence();
    tk.init();
    // Block lists come from L2 (a round trip each if loaded one by one): fetch four at a time, then merge.
    // (the merge loops are kept rolled: every inlined merge is ~150 instructions and this code runs once, so unrolled
    // copies only buy instruction-cache misses)
    constexpr int U = (E == 1) ? 4 : 2;
#pragma unroll 1
    for (uint32_t b0 = warp; b0 < gridDim.x; b0 += warps * U) {
        uint64_t other[U][E];
#pragma unroll
        for (int u = 0; u < U; ++u) {
            const uint32_t b = b0 + u * warps;
#pragma unroll
            for (int j = 0; j < E; ++j)
                other[u][j] = (b < gridDim.x) ? ld_cg_u64(p.block_keys + static_cast<size_t>(b) * W + j * 32 + lane)
                                              : WAXVS_KEY_NONE;
        }
#pragma unroll
        for (int u = 0; u < U; ++u) tk.merge_sorted(other[u], lane, k);
    }
    __syncthreads();  // everyone is done reading lists from the CTA merge
#pragma unroll
    for (int j = 0; j < E; ++j) lists[warp * W + j * 32 + lane] = tk.key[j];
    __syncthreads();
    if (warp == 0) {
#pragma unroll 1
        for (int w = 1; w < warps; ++w) {
            uint64_t other[E];
            load_list(lists + w * W, other);
            tk.merge_sorted(other, lane, k);
        }
#pragma unroll
        for (int j = 0; j < E; ++j)
            if (j * 32 + lane < k) write_slot<SHADOW>(p, j * 32 + lane, tk.key[j]);
        if (lane == 0) { *p.ticket = 0u; if (p.work_counter) *p.work_counter = 0u; }
        if (p.host_flag && !p.shard.world) {          // result complete in host memory: tell the waiting caller
            __threadfence_system();
            __syncwarp();
            if (lane == 0) st_release_sys_u64(p.host_flag, p.host_seq);
        }
    }
    // Row-sharded search: push the local list to every rank, wait for theirs, merge -- the block lists are done with,
    // their shared memory holds the distance keys of the merge (the host checks that world * k * 4 bytes fit).
    if (p.shard.world) shard_exchange_cta(p.shard, p.out, p.k, reinterpret_cast<uint32_t *>(lists));
}

// ------------------------------------------------------------------------------------------------------------
// Selection tail.  The merge tail above costs one ~150-instruction bitonic merge per pair of lists: 7 per CTA plus one
// per CTA of the grid in the last CTA -- a serial tail that is a large part of a search over a real (<= 174 K-row) Wax
// index.  Selection does not care about order: a block-wide MSB-first radix select (8 bits a
// pass, it stops as soon as the bin holding the k-th key holds one key) finds the k-th smallest key exactly, the keys
// at or below it are the answer; only the final k are ranked (k x k compares) to come out sorted.
struct SelectScratch {
    uint32_t hist[256];
    uint64_t sel[128];          // the selected keys of the final stage
    uint32_t digit, k_rem, in_bin, n_sel;
    unsigned long long found;
};

// All threads of the CTA call.  for_each(f): f(key) for every key the calling thread owns (WAXVS_KEY_NONE = absent; it
// is the largest key, so it only matters when fewer than k real keys exist).  Returns the k-th smallest key of the CTA's
// keys (WAXVS_KEY_NONE when there are fewer than k real ones): the selection is {key <= result, key != NONE}.
template <typename ForEach>
__device__ __forceinline__ uint64_t block_select_kth(ForEach for_each, uint32_t k, SelectScratch *ss) {
    const uint32_t tid = threadIdx.x;
    uint64_t prefix = 0;
    uint32_t k_rem = k;
#pragma unroll 1
    for (int shift = 56; shift >= 0; shift -= 8) {
        for (uint32_t i = tid; i < 256u; i += blockDim.x) ss->hist[i] = 0;
        __syncthreads();
        const uint64_t want = (shift == 56) ? 0ull : (prefix >> (shift + 8));
        for_each([&](uint64_t key) {
            if (shift == 56 || (key >> (shift + 8)) == want) atomicAdd(&ss->hist[(key >> shift) & 255u], 1u);
        });
        __syncthreads();
        if (tid < 32) {             // the digit whose cumulative count reaches k_rem: 8 bins per lane + a warp scan
            uint32_t c[8], sum = 0;
#pragma unroll
            for (int i = 0; i < 8; ++i) { c[i] = ss->hist[tid * 8 + i]; sum += c[i]; }
            uint32_t incl = sum;
#pragma unroll
            for (int off = 1; off < 32; off <<= 1) {
                const uint32_t up = __shfl_up_sync(WAXVS_FULL_MASK, incl, off);
                if (static_cast<int>(tid) >= off) incl += up;
            }
            const uint32_t excl = incl - sum;
            if (excl < k_rem && k_rem <= incl) {      // exactly one lane
                uint32_t run = excl;
#pragma unroll
                for (int i = 0; i < 8; ++i) {
                    if (run < k_rem && k_rem <= run + c[i]) { ss->digit = tid * 8 + i; ss->k_rem = k_rem - run; ss->in_bin = c[i]; }
                    run += c[i];
                }
            }
        }
        __syncthreads();
        prefix |= static_cast<uint64_t>(ss->digit) << shift;
        k_rem = ss->k_rem;
        if (ss->in_bin == 1u && shift > 0) {          // one key carries this prefix: it is the k-th smallest -- fetch it
            const uint64_t top = prefix >> shift;
            for_each([&](uint64_t key) { if ((key >> shift) == top) ss->found = key; });
            __syncthreads();
            const uint64_t x = ss->found;
            __syncthreads();
            return x;
        }
    }
    return prefix;
}

// The selection tail: called by every thread of the CTA after the scan loop (the warps' register lists need not be
// merged, or even sorted, for this).  scratch = the dynamic shared memory (the idle ring), p.tail_smem_bytes of it.
// Returns true in the CTA that finished the grid stage (its threads have written the result, not yet synchronised).
template <int E, bool SHADOW = false>
__device__ __forceinline__ bool finish_topk_select(const ScanParams &p, WarpTopK<E> &tk, unsigned char *scratch) {
    __shared__ SelectScratch ss;
    __shared__ uint32_t s_last2;
    const uint32_t tid = threadIdx.x, nthr = blockDim.x, k = p.k;
    // ---- stage A: this CTA's k smallest keys -> block_keys[blockIdx][0..k) (unordered, NONE-padded)
    auto own_keys = [&](auto f) {
#pragma unroll
        for (int j = 0; j < E; ++j) f(tk.key[j]);
    };
    const uint64_t xa = block_select_kth(own_keys, k, &ss);
    if (tid == 0) ss.n_sel = 0;
    __syncthreads();
    uint64_t *mine = p.block_keys + static_cast<size_t>(blockIdx.x) * k;
#pragma unroll
    for (int j = 0; j < E; ++j)
        if (tk.key[j] != WAXVS_KEY_NONE && tk.key[j] <= xa) mine[atomicAdd(&ss.n_sel, 1u)] = tk.key[j];
    __syncthreads();
    for (uint32_t i = ss.n_sel + tid; i < k; i += nthr) mine[i] = WAXVS_KEY_NONE;
    __threadfence();
    __syncthreads();
    if (p.trace && tid == 0) atomicMax(p.trace + 2, global_timer_ns());
    if (tid == 0) s_last2 = (atomicAdd(p.ticket, 1u) == gridDim.x - 1) ? 1u : 0u;
    __syncthreads();
    if (!s_last2) return false;
    __threadfence();
    if (p.trace && tid == 0) p.trace[3] = global_timer_ns();
    // ---- stage B (last CTA): the k smallest of the grid's gridDim.x * k keys, ranked, written out
    const uint32_t total = gridDim.x * k;
    const bool staged = static_cast<size_t>(total) * sizeof(uint64_t) <= p.tail_smem_bytes;
    uint64_t *sk = reinterpret_cast<uint64_t *>(scratch);
    if (staged) {
        for (uint32_t i = tid; i < total; i += nthr) sk[i] = ld_cg_u64(p.block_keys + i);
        __syncthreads();
    }
    auto grid_keys = [&](auto f) {
        if (staged) { for (uint32_t i = tid; i < total; i += nthr) f(sk[i]); }
        else { for (uint32_t i = tid; i < total; i += nthr) f(ld_cg_u64(p.block_keys + i)); }
    };
    const uint64_t xb = block_select_kth(grid_keys, k, &ss);
    if (tid == 0) ss.n_sel = 0;
    __syncthreads();
    grid_keys([&](uint64_t key) { if (key != WAXVS_KEY_NONE && key <= xb) ss.sel[atomicAdd(&ss.n_sel, 1u)] = key; });
    __syncthreads();
    const uint32_t n_sel = ss.n_sel;                  // == k, or every real key when there are fewer than k
    for (uint32_t i = tid; i < k; i += nthr) {
        if (i < n_sel) {
            const uint64_t key = ss.sel[i];
            uint32_t rank = 0;
            for (uint32_t j = 0; j < n_sel; ++j) rank += ss.sel[j] < key ? 1u : 0u;
            write_slot<SHADOW>(p, static_cast<int>(rank), key);
        } else {
            write_slot<SHADOW>(p, static_cast<int>(i), WAXVS_KEY_NONE);   // padding after the n_sel ranked entries
        }
    }
    if (p.host_flag && !p.shard.world) __threadfence_system();
    __syncthreads();
    if (tid == 0) {
        *p.ticket = 0u;
        if (p.work_counter) *p.work_counter = 0u;
        if (p.host_flag && !p.shard.world) st_release_sys_u64(p.host_flag, p.host_seq);
        if (p.trace) p.trace[4] = global_timer_ns();
    }
    if (p.shard.world) shard_exchange_cta(p.shard, p.out, p.k, reinterpret_cast<uint32_t *>(scratch));
    return true;
}

// The U4 form's tail: no grid stage.  Every CTA selects the kU4CtaNominees smallest keys of its warps' lists and writes
// them to p.nominees[blockIdx.x * kU4CtaNominees ..] (unordered, NONE-padded); shadow_rescore_kernel re-scores them all.
// A row that is not written was cut either by its warp's full list (key >= the list's last key) or by this selection
// (key > the CTA's cut key): the smallest such key over the grid, in p.u4_aux[0], bounds the score' of every row left out.
template <int E>
__device__ __forceinline__ void finish_u4_nominees(const ScanParams &p, WarpTopK<E> &tk) {
    __shared__ SelectScratch ss;
    __shared__ uint32_t s_cut;
    const uint32_t tid = threadIdx.x, nthr = blockDim.x;
    if (tid == 0) s_cut = WAXVS_UKEY_NONE;
    auto own_keys = [&](auto f) {
#pragma unroll
        for (int j = 0; j < E; ++j) f(tk.key[j]);
    };
    // block_select_kth needs at least kU4CtaNominees keys in the CTA, NONE included; one warp holds only 32 E: then
    // every real key is selected (the barrier below publishes s_cut)
    const uint64_t xa = nthr * E >= kU4CtaNominees ? block_select_kth(own_keys, kU4CtaNominees, &ss) : WAXVS_KEY_NONE;
    if (tid == 0) ss.n_sel = 0;
    __syncthreads();
    uint64_t *mine = p.nominees + static_cast<size_t>(blockIdx.x) * kU4CtaNominees;
#pragma unroll
    for (int j = 0; j < E; ++j)
        if (tk.key[j] != WAXVS_KEY_NONE && tk.key[j] <= xa) mine[atomicAdd(&ss.n_sel, 1u)] = tk.key[j];
    if ((tid & 31u) == 0 && tk.thresh != WAXVS_KEY_NONE) atomicMin(&s_cut, static_cast<uint32_t>(tk.thresh >> 32));
    __syncthreads();
    for (uint32_t i = ss.n_sel + tid; i < kU4CtaNominees; i += nthr) mine[i] = WAXVS_KEY_NONE;
    if (tid == 0) {
        uint32_t cut = s_cut;
        if (xa != WAXVS_KEY_NONE) cut = min(cut, static_cast<uint32_t>(xa >> 32));
        if (cut != WAXVS_UKEY_NONE) atomicMin(p.u4_aux, cut);
    }
}

// ------------------------------------------------------------------------------------------------------------
// TMA-staged kernel.  C > 0: dims == 128*C, query chunks in registers, loops fully unrolled (the hot shapes
// 128..1024).  C == 0: any dims % 4 == 0 whose rows fit a stage (1536, 3072, 1000, ...): same algorithm with the
// chunk count at run time and the query chunks read from a shared-memory copy.
//   R      rows per step (power of two)
//   E      register-list slots per lane: fused top-k for k <= 32*E (E = 1: k <= 32, E = 4: k <= 128 -- the production
//          candidateLimit of 72, UnifiedSearch.swift:1195-1200, stays in the single launch)
//   EMIT   false: fused top-k;  true: write orderable distance keys for the large-k select path
//   SHADOW true (C > 0, cosine / dot, E = 4, fused): the nominating pass of the bf16-shadow route.  p.corpus is the
//          shadow (bf16 rows, cosine rows pre-scaled by 1/|v|): a lane reads chunk lane + 32c as one uint2 of 4 bf16
//          where the fp32 form reads a float4, widens it exactly and FMAs it against the fp32 query -- one quantity per
//          row, score' = q.v~ for both metrics, key make_key(-score', row) (= nominee_key).  Only the row is rounded,
//          so kBf16Eps bounds |score' - score|.  Every warp keeps k (= 128) nominees, so the grid's k-th bounds every
//          row left out; the tails write them for batch_finish_kernel (write_slot).  A non-finite score' counts as +inf.
//   INT8   (with SHADOW) the nominating pass of the int8-shadow route: p.corpus holds the rows as biased int8 codes c (one
//          byte per element, ROW_BYTES = 128 C) and p.row_scale each row's scale s.  A lane reads chunk lane + 32c as one
//          uint32 of 4 codes, widens them exactly (int8x4_to_float4) and FMAs them against the same fp32 query registers;
//          the row's sum is multiplied once by s: score' = s (q.c).  The R scales of a step ride in the same stage behind
//          the rows (a second bulk copy on the same mbarrier), so R >= 4 keeps that copy 16-byte aligned.
//   U4     (with SHADOW, not INT8) the nominating pass of the 4-bit-shadow route: p.corpus holds the rows as 16-level
//          codes u, two per byte (ROW_BYTES = 64 C; byte b of word w: element 8w + b in the low nibble, 8w + 4 + b in the
//          high one), p.row_scale each row's half step h: the row decodes to h (2u - 15).  The query is coded once per
//          launch to int8 (c_q = rne(q / s_q), s_q = max|q_i| / 127) and the row's sum is integer, two dp4a per word:
//          score' = fl(fl(s_q h) (2 sum c_q u - 15 sum c_q)), exact but for those two roundings.  16 lanes share a row (C
//          words each), the half-warps take the even and the odd rows of a step; for even C the odd half swaps its word
//          pairs so that the two halves never read the same banks.  CTA 0 stores rho_q = ||q - s_q c_q|| (measured in
//          fp64, rounded up; +inf for a non-finite query) in p.u4_aux[1]; the tail is finish_u4_nominees.
template <int C, int R, int METRIC, int E, bool EMIT, bool SHADOW = false, bool INT8 = false, bool U4 = false>
__global__ void __launch_bounds__(512, 1) scan_tma_kernel(const __grid_constant__ ScanParams p) {
    static_assert(!SHADOW || (C > 0 && METRIC != kL2 && !EMIT), "the shadow form covers the unrolled cosine / dot shapes");
    static_assert(!INT8 || (SHADOW && R >= 4), "the int8 form is a shadow form with 16-byte scale copies");
    static_assert(!U4 || (SHADOW && !INT8 && R >= 4 && E == 4), "the 4-bit form is a shadow form with 16-byte scale copies");
    constexpr bool SCALED = INT8 || U4;     // the step's row scales ride behind its rows
    if constexpr (!SHADOW && !EMIT && E == 1 && METRIC != kL2) {
        if (p.proof_ok) {               // guarded launch after a shadow proof (batch_finish_kernel, same stream; k <= 32)
            const bool proven = *p.proof_ok != 0u;
            if (blockIdx.x == 0) {
                if (threadIdx.x == 0) {
                    const uint32_t n = ++p.proof_count[proven ? 0 : 1];
                    *static_cast<volatile uint32_t *>(p.proof_count_host + (proven ? 0 : 1)) = n;
                }
                if (proven && p.host_flag) {      // the delivery the last CTA would otherwise do
                    for (uint32_t i = threadIdx.x; i < p.k; i += blockDim.x) p.host_out[i] = p.out[i];
                    __threadfence_system();
                    __syncthreads();
                    if (threadIdx.x == 0) st_release_sys_u64(p.host_flag, p.host_seq);
                }
            }
            if (proven) return;
        }
    }
    const int D4 = C > 0 ? 32 * C : static_cast<int>(p.dims / 4u);          // float4 (SHADOW: uint2, INT8: uint32) per row
    const int CN = C > 0 ? C : (D4 + 31) / 32;                               // chunks per lane
    const uint32_t ROW_BYTES = C > 0 ? (U4 ? 64u : INT8 ? 128u : SHADOW ? 256u : 512u) * C : p.dims * 4u;
    const uint32_t STAGE_BYTES = ROW_BYTES * R + (SCALED ? R * 4u : 0u);     // SCALED: the step's scales behind its rows
    constexpr int LANES_PER_ROW = 32 / R;

    extern __shared__ __align__(128) unsigned char smem[];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, warps = blockDim.x >> 5;
    const uint32_t stages = p.stages;
    unsigned char *ring = smem + static_cast<size_t>(warp) * stages * STAGE_BYTES;
    uint64_t *bars = reinterpret_cast<uint64_t *>(smem + static_cast<size_t>(warps) * stages * STAGE_BYTES) +
                     warp * stages;
    uint64_t *lists = reinterpret_cast<uint64_t *>(smem + static_cast<size_t>(warps) * stages * STAGE_BYTES) +
                      warps * stages;
    uint32_t *stage_step = reinterpret_cast<uint32_t *>(lists + warps * 32 * E) + warp * stages;  // step held by each stage
    float4 *qs = reinterpret_cast<float4 *>(reinterpret_cast<uint32_t *>(lists + warps * 32 * E) + warps * stages + 4);  // C == 0

    // ---- query chunks in registers (C > 0) or shared memory (C == 0) + fused |q|^2 ----
    float4 q[C > 0 ? C : 1];
    const float4 *q4 = reinterpret_cast<const float4 *>(p.query);
    const float4 *qp = reinterpret_cast<const float4 *>(p.query_inline);     // kernel-parameter copy (query == nullptr)
    auto load_q = [&](int i) -> float4 { return q4 ? __ldg(q4 + i) : qp[i]; };
    if (C > 0) {
#pragma unroll
        for (int c = 0; c < (C > 0 ? C : 1); ++c) q[c] = load_q(lane + 32 * c);
    } else {
        qs = reinterpret_cast<float4 *>((reinterpret_cast<uintptr_t>(qs) + 15) & ~uintptr_t(15));
        for (int i = threadIdx.x; i < CN * 32; i += blockDim.x) qs[i] = (i < D4) ? load_q(i) : make_float4(0.f, 0.f, 0.f, 0.f);
        __syncthreads();
    }
    auto qchunk = [&](int c) -> float4 { return C > 0 ? q[C > 0 ? c : 0] : qs[lane + 32 * c]; };
    if constexpr (SHADOW) {             // the finish and the guarded scan read the query from device memory
        if (p.query_store && p.query == nullptr && blockIdx.x == 0)
            for (uint32_t i = threadIdx.x; i < p.dims; i += blockDim.x) p.query_store[i] = p.query_inline[i];
    }
    // U4: the query as int8 codes, in the words this lane reads of every row
    constexpr int CU = U4 ? (C > 0 ? C : 1) : 1;
    constexpr int H = U4 ? R / 2 : 1;                 // rows of a step per half-warp
    const int hl = lane & 15, hh = lane >> 4;
    int qlo[CU], qhi[CU], word_of[CU];
    int q_code_sum = 0;
    float s_q = 0.0f;
    if constexpr (U4) {
        float m = 0.0f;
        bool bad = false;
#pragma unroll
        for (int c = 0; c < CU; ++c) {
            bad |= !finite_f32(q[c].x) || !finite_f32(q[c].y) || !finite_f32(q[c].z) || !finite_f32(q[c].w);
            m = fmaxf(m, fmaxf(fmaxf(fabsf(q[c].x), fabsf(q[c].y)), fmaxf(fabsf(q[c].z), fabsf(q[c].w))));
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(WAXVS_FULL_MASK, m, o));
        bad = __any_sync(WAXVS_FULL_MASK, bad);
        s_q = __fdiv_rn(m, 127.0f);
        const bool code_it = !bad && s_q > 0.0f && finite_f32(s_q);
        double r2 = 0.0;
#pragma unroll
        for (int c = 0; c < CU; ++c) {
            word_of[c] = hl + 16 * ((C % 2 == 0) ? (c ^ hh) : c);
            int packed[2];
#pragma unroll
            for (int half = 0; half < 2; ++half) {
                const float4 x4 = load_q(2 * word_of[c] + half);
                const float xs[4] = {x4.x, x4.y, x4.z, x4.w};
                uint32_t w = 0;
#pragma unroll
                for (int j = 0; j < 4; ++j) {
                    const int code = code_it ? max(-127, min(127, __float2int_rn(__fdiv_rn(xs[j], s_q)))) : 0;
                    w |= static_cast<uint32_t>(code & 0xFF) << (8 * j);
                    const double e = static_cast<double>(xs[j]) - static_cast<double>(s_q) * static_cast<double>(code);
                    r2 = fma(e, e, r2);
                }
                packed[half] = static_cast<int>(w);
                q_code_sum = __dp4a(packed[half], 0x01010101, q_code_sum);
            }
            qlo[c] = packed[0]; qhi[c] = packed[1];
        }
#pragma unroll
        for (int o = 8; o > 0; o >>= 1) {       // a half-warp holds every word of the query once
            q_code_sum += __shfl_xor_sync(WAXVS_FULL_MASK, q_code_sum, o);
            r2 += __shfl_xor_sync(WAXVS_FULL_MASK, r2, o);
        }
        if (blockIdx.x == 0 && threadIdx.x == 0) {
            float rho_q = __double2float_ru(sqrt(r2) * (1.0 + 0x1p-40));
            if (bad || !finite_f32(s_q) || !finite_f32(rho_q)) rho_q = INFINITY;
            p.u4_aux[1] = __float_as_uint(rho_q);
        }
    }
    float a2 = 0.0f, sqrt_a2 = 0.0f;
    if (METRIC == kCosine && !SHADOW) {
        float s0 = 0.f, s1 = 0.f, s2 = 0.f, s3 = 0.f;
#pragma unroll
        for (int c = 0; c < CN; ++c) {
            const float4 qc = qchunk(c);
            s0 = __fmaf_rn(qc.x, qc.x, s0); s1 = __fmaf_rn(qc.y, qc.y, s1);
            s2 = __fmaf_rn(qc.z, qc.z, s2); s3 = __fmaf_rn(qc.w, qc.w, s3);
        }
        a2 = warp_butterfly_sum(__fadd_rn(__fadd_rn(s0, s1), __fadd_rn(s2, s3)));
        sqrt_a2 = __fsqrt_rn(a2);
    }

    if (p.trace && threadIdx.x == 0) atomicMin(p.trace + 0, global_timer_ns());
    const uint32_t total_warps = gridDim.x * warps;
    const uint32_t gwarp = blockIdx.x * warps + warp;
    const uint32_t n_steps = (p.n_rows + R - 1) / R;
    uint64_t policy = 0;
    if (p.use_l2_hint) policy = l2_policy_evict_first();

    auto issue = [&](uint32_t step, uint32_t s) {   // lane 0 only
        const uint32_t row0 = step * R;
        const uint32_t rows = min(static_cast<uint32_t>(R), p.n_rows - row0);
        const uint32_t bytes = rows * ROW_BYTES;
        stage_step[s] = step;                        // released to the warp by the mbarrier arrive below
        mbar_arrive_expect_tx(&bars[s], bytes + (SCALED ? R * 4u : 0u));
        const void *src = SHADOW ? static_cast<const void *>(reinterpret_cast<const unsigned char *>(p.corpus) +
                                                             static_cast<size_t>(row0) * ROW_BYTES)
                                 : static_cast<const void *>(p.corpus + static_cast<size_t>(row0) * p.dims);
        if (p.use_l2_hint) bulk_copy_g2s_hint(ring + s * STAGE_BYTES, src, bytes, &bars[s], policy);
        else bulk_copy_g2s(ring + s * STAGE_BYTES, src, bytes, &bars[s]);
        // the scale array is padded to whole steps: a ragged last step still copies R scales
        if constexpr (SCALED) bulk_copy_g2s(ring + s * STAGE_BYTES + R * ROW_BYTES, p.row_scale + row0, R * 4u, &bars[s]);
    };

    // Step sequence of this warp.  Static: gwarp, gwarp + total_warps, ...  Dynamic (chunk_steps > 0, fused
    // top-k only): chunks of `chunk_steps` consecutive steps claimed from a global counter, the next claim
    // always in flight, so SMs that stream faster simply take more chunks (no tail imbalance).
    const bool dynamic = !EMIT && p.chunk_steps > 0 && p.work_counter != nullptr;
    const uint32_t chunk = p.chunk_steps;
    uint32_t cur = gwarp, cur_end = 0, claim_l0 = 0;
    if (dynamic) {
        if (lane == 0) { cur = atomicAdd(p.work_counter, chunk); claim_l0 = atomicAdd(p.work_counter, chunk); }
        cur = __shfl_sync(WAXVS_FULL_MASK, cur, 0);
        cur_end = min(cur + chunk, n_steps);
    }
    auto next_step = [&]() -> uint32_t {             // warp-uniform; >= n_steps when the warp is out of work
        if (!dynamic) { const uint32_t st = cur; cur = (cur < n_steps) ? cur + total_warps : cur; return st; }
        if (cur < cur_end) return cur++;
        if (cur >= n_steps) return n_steps;
        const uint32_t start = __shfl_sync(WAXVS_FULL_MASK, claim_l0, 0);
        if (lane == 0 && start < n_steps) claim_l0 = atomicAdd(p.work_counter, chunk);
        cur = start;
        cur_end = min(start + chunk, n_steps);
        if (cur >= n_steps) return n_steps;
        return cur++;
    };

    if (lane == 0) {
        for (uint32_t s = 0; s < stages; ++s) mbar_init(&bars[s], 1);
        mbar_fence_init();
    }
    __syncwarp();
    uint32_t issued = 0, consumed = 0;
    for (uint32_t s = 0; s < stages; ++s) {
        const uint32_t step = next_step();
        if (step >= n_steps) break;
        if (lane == 0) issue(step, s);
        ++issued;
    }

    WarpTopK<E> tk;
    tk.init();
    const int k = static_cast<int>(p.k);

    uint32_t s = 0, parity = 0;
    while (consumed < issued) {
        mbar_wait_parity(&bars[s], parity);
        const uint32_t step = stage_step[s];
        const float4 *tile = reinterpret_cast<const float4 *>(ring + s * STAGE_BYTES);
        // INT8: the scale of the row this lane finishes after the reduce-scatter, read before the stage is refilled
        // U4: a lane finishes row 2 (hl / (16 / H)) + hh of the step
        const int my_in_step = U4 ? 2 * (hl / (16 / H)) + hh : lane / LANES_PER_ROW;
        const float row_s = SCALED ? reinterpret_cast<const float *>(ring + s * STAGE_BYTES + R * ROW_BYTES)[my_in_step] : 1.0f;

        float sum0[R], sum1[R];
        int isum[H] = {};
        if constexpr (U4) {
            const uint32_t *tw = reinterpret_cast<const uint32_t *>(tile) + hh * 16 * C;
#pragma unroll
            for (int j = 0; j < H; ++j) {
                int a = 0;
#pragma unroll
                for (int c = 0; c < CU; ++c) {
                    const uint32_t w = tw[j * 32 * C + word_of[c]];
                    a = __dp4a(static_cast<int>(w & 0x0F0F0F0Fu), qlo[c], a);
                    a = __dp4a(static_cast<int>((w >> 4) & 0x0F0F0F0Fu), qhi[c], a);
                }
                isum[j] = a;
            }
        } else if (C == 0) {
            // Generic rows (dims < 128 or not one of the unrolled multiples of 128), several rows per step: chunk-outer /
            // row-inner, so a query chunk is read from shared memory once for the R rows (the row-outer form read it per row:
            // twice the shared-memory traffic).  Each row still sees its chunks in ascending
            // order on its own accumulators: the same operations in the same order as the row-outer loop below.
            float a[R][4], b[R][4];
#pragma unroll
            for (int r = 0; r < R; ++r)
#pragma unroll
                for (int j = 0; j < 4; ++j) { a[r][j] = 0.f; b[r][j] = 0.f; }
            // (a few chunks in flight per lane: with one or two rows per step the loads of consecutive chunks must overlap)
#pragma unroll (R >= 8 ? 1 : 8 / R)
            for (int c = 0; c < CN; ++c) {
                if (lane + 32 * c >= D4) break;
                const float4 qc = qchunk(c);
#pragma unroll
                for (int r = 0; r < R; ++r) {
                    const float4 v = tile[r * D4 + lane + 32 * c];
                    if (METRIC == kL2) {
                        const float dx = __fsub_rn(qc.x, v.x), dy = __fsub_rn(qc.y, v.y);
                        const float dz = __fsub_rn(qc.z, v.z), dw = __fsub_rn(qc.w, v.w);
                        a[r][0] = __fmaf_rn(dx, dx, a[r][0]); a[r][1] = __fmaf_rn(dy, dy, a[r][1]);
                        a[r][2] = __fmaf_rn(dz, dz, a[r][2]); a[r][3] = __fmaf_rn(dw, dw, a[r][3]);
                    } else {
                        a[r][0] = __fmaf_rn(qc.x, v.x, a[r][0]); a[r][1] = __fmaf_rn(qc.y, v.y, a[r][1]);
                        a[r][2] = __fmaf_rn(qc.z, v.z, a[r][2]); a[r][3] = __fmaf_rn(qc.w, v.w, a[r][3]);
                        if (METRIC == kCosine) {
                            b[r][0] = __fmaf_rn(v.x, v.x, b[r][0]); b[r][1] = __fmaf_rn(v.y, v.y, b[r][1]);
                            b[r][2] = __fmaf_rn(v.z, v.z, b[r][2]); b[r][3] = __fmaf_rn(v.w, v.w, b[r][3]);
                        }
                    }
                }
            }
#pragma unroll
            for (int r = 0; r < R; ++r) {
                sum0[r] = __fadd_rn(__fadd_rn(a[r][0], a[r][1]), __fadd_rn(a[r][2], a[r][3]));
                sum1[r] = __fadd_rn(__fadd_rn(b[r][0], b[r][1]), __fadd_rn(b[r][2], b[r][3]));
            }
        } else
#pragma unroll
        for (int r = 0; r < R; ++r) {
            float a0 = 0.f, a1 = 0.f, a2_ = 0.f, a3 = 0.f, b0 = 0.f, b1 = 0.f, b2 = 0.f, b3 = 0.f;
#pragma unroll
            for (int c = 0; c < CN; ++c) {
                if (C == 0 && lane + 32 * c >= D4) break;   // ragged last chunk (dims % 128 != 0): this lane has no element
                const float4 v = INT8 ? int8x4_to_float4(reinterpret_cast<const uint32_t *>(tile)[r * D4 + lane + 32 * c])
                               : SHADOW ? bf16x4_to_float4(reinterpret_cast<const uint2 *>(tile)[r * D4 + lane + 32 * c])
                                        : tile[r * D4 + lane + 32 * c];
                const float4 qc = qchunk(c);
                if (METRIC == kL2) {
                    const float dx = __fsub_rn(qc.x, v.x), dy = __fsub_rn(qc.y, v.y);
                    const float dz = __fsub_rn(qc.z, v.z), dw = __fsub_rn(qc.w, v.w);
                    a0 = __fmaf_rn(dx, dx, a0); a1 = __fmaf_rn(dy, dy, a1);
                    a2_ = __fmaf_rn(dz, dz, a2_); a3 = __fmaf_rn(dw, dw, a3);
                } else {
                    a0 = __fmaf_rn(qc.x, v.x, a0); a1 = __fmaf_rn(qc.y, v.y, a1);
                    a2_ = __fmaf_rn(qc.z, v.z, a2_); a3 = __fmaf_rn(qc.w, v.w, a3);
                    if (METRIC == kCosine && !SHADOW) {
                        b0 = __fmaf_rn(v.x, v.x, b0); b1 = __fmaf_rn(v.y, v.y, b1);
                        b2 = __fmaf_rn(v.z, v.z, b2); b3 = __fmaf_rn(v.w, v.w, b3);
                    }
                }
            }
            sum0[r] = __fadd_rn(__fadd_rn(a0, a1), __fadd_rn(a2_, a3));
            sum1[r] = __fadd_rn(__fadd_rn(b0, b1), __fadd_rn(b2, b3));
        }
        __syncwarp();  // every lane has consumed this stage (and read stage_step): safe to refill it
        {
            const uint32_t next = next_step();
            if (next < n_steps) {
                if (lane == 0) issue(next, s);
                ++issued;
            }
        }
        ++consumed;
        if (++s == stages) { s = 0; parity ^= 1u; }

        if constexpr (U4) half_warp_reduce_scatter<H>(isum, lane);
        else warp_reduce_scatter<R>(sum0, lane);
        if (METRIC == kCosine && !SHADOW) warp_reduce_scatter<R>(sum1, lane);

        const uint32_t my_row = step * R + my_in_step;
        float d;
        if constexpr (U4) d = -__fmul_rn(__fmul_rn(s_q, row_s), static_cast<float>(2 * isum[0] - 15 * q_code_sum));   // -score'
        else if (INT8) d = -__fmul_rn(row_s, sum0[0]);   // -score' = -s (q.c)
        else if (SHADOW) d = -sum0[0];     // -score': the nominee key's distance
        else if (METRIC == kCosine) d = finish_cos(sum0[0], a2, sqrt_a2, sum1[0]);
        else if (METRIC == kDot) d = finish_dot(sum0[0]);
        else d = finish_l2(sum0[0]);
        // SHADOW: a non-finite score' bounds nothing -- a product q_i v~_i can overflow where q_i v_i does not (v~ rounded
        // up), giving +-inf or inf - inf = NaN for a row whose exact score is finite.  Such a row is nominated first
        // (score' = +inf), so the finish re-scores it; and as entry 0 it refuses the proof.
        if (SHADOW && !finite_f32(d)) d = -INFINITY;
        const bool leader = U4 ? (hl % (16 / H)) == 0 : (lane % LANES_PER_ROW) == 0;
        const bool ok = (my_row < p.n_rows) && (SHADOW || finite_f32(d));

        if (EMIT) {
            if (leader && my_row < p.n_rows)
                p.dist_keys[my_row] = (ok && row_allowed(p, my_row)) ? orderable_u32(d) : WAXVS_UKEY_NONE;
        } else {
            const uint64_t key = ok ? make_key(d, my_row) : WAXVS_KEY_NONE;
            // the filter is consulted only for rows that would enter the list (rare once the list is warm)
            const bool cand = leader && key < tk.thresh && row_allowed(p, my_row);
            uint32_t m = __ballot_sync(WAXVS_FULL_MASK, cand);
            if (E == 1) {
                while (m) {
                    const int src = __ffs(m) - 1;
                    m &= m - 1;
                    const uint64_t x = shfl_u64(key, src);
                    if (x < tk.thresh) tk.insert(x, lane, k);
                }
            } else if (m) {                             // batched insertion (WarpTopK::flush)
                if (tk.npend + __popc(m) > 32) tk.flush(lane, k);
                while (m) {
                    const int src = __ffs(m) - 1;
                    m &= m - 1;
                    tk.park(shfl_u64(key, src), lane);
                }
            }
        }
    }

    if (p.trace && lane == 0) atomicMax(p.trace + 1, global_timer_ns());
    if (!EMIT) {
        if (E > 1) tk.flush(lane, k);
        if constexpr (U4) finish_u4_nominees<E>(p, tk);
        else if (p.tail_select) finish_topk_select<E, SHADOW>(p, tk, smem);
        else finish_topk<E, SHADOW>(p, tk, lists, warp, lane, warps);
    }
}

// ------------------------------------------------------------------------------------------------------------
// Generic kernel: any dims (including dims % 4 != 0 and rows too large for a shared-memory tile).
// One warp per row, coalesced direct global loads (LDG.128 when dims % 4 == 0), same accumulation order.
template <int METRIC, int E, bool EMIT>
__global__ void __launch_bounds__(256, 4) scan_ldg_kernel(const __grid_constant__ ScanParams p) {
    __shared__ uint64_t lists[8 * 32 * E];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, warps = blockDim.x >> 5;
    const uint32_t dims = p.dims;
    const bool vec4 = (dims % 4u) == 0u;
    const uint32_t d4 = dims / 4u;

    float a2 = 0.0f, sqrt_a2 = 0.0f;
    if (METRIC == kCosine) {
        float s0 = 0.f, s1 = 0.f, s2 = 0.f, s3 = 0.f;
        for (uint32_t base = 4u * lane; base < dims; base += 128u) {
            const float x = __ldg(p.query + base);
            const float y = (base + 1 < dims) ? __ldg(p.query + base + 1) : 0.0f;
            const float z = (base + 2 < dims) ? __ldg(p.query + base + 2) : 0.0f;
            const float w = (base + 3 < dims) ? __ldg(p.query + base + 3) : 0.0f;
            s0 = __fmaf_rn(x, x, s0);
            if (base + 1 < dims) s1 = __fmaf_rn(y, y, s1);
            if (base + 2 < dims) s2 = __fmaf_rn(z, z, s2);
            if (base + 3 < dims) s3 = __fmaf_rn(w, w, s3);
        }
        a2 = warp_butterfly_sum(__fadd_rn(__fadd_rn(s0, s1), __fadd_rn(s2, s3)));
        sqrt_a2 = __fsqrt_rn(a2);
    }

    WarpTopK<E> tk;
    tk.init();
    const int k = static_cast<int>(p.k);
    const uint32_t total_warps = gridDim.x * warps;

    for (uint32_t row = blockIdx.x * warps + warp; row < p.n_rows; row += total_warps) {
        const float *v = p.corpus + static_cast<size_t>(row) * dims;
        float a0 = 0.f, a1 = 0.f, a2_ = 0.f, a3 = 0.f, b0 = 0.f, b1 = 0.f, b2 = 0.f, b3 = 0.f;
        auto acc = [&](float qx, float vx, float &a, float &b) {
            if (METRIC == kL2) { const float dd = __fsub_rn(qx, vx); a = __fmaf_rn(dd, dd, a); }
            else {
                a = __fmaf_rn(qx, vx, a);
                if (METRIC == kCosine) b = __fmaf_rn(vx, vx, b);
            }
        };
        if (vec4) {
            const float4 *v4 = reinterpret_cast<const float4 *>(v);
            const float4 *q4 = reinterpret_cast<const float4 *>(p.query);
            // the row is read once: streaming loads (evict-first, no L1 residency) leave L1 to the query, which every row
            // re-reads; eight 16-byte loads in flight per lane
#pragma unroll 8
            for (uint32_t c = lane; c < d4; c += 32u) {
                const float4 x = __ldcs(v4 + c);
                const float4 y = __ldg(q4 + c);
                acc(y.x, x.x, a0, b0); acc(y.y, x.y, a1, b1); acc(y.z, x.z, a2_, b2); acc(y.w, x.w, a3, b3);
            }
        } else {
            for (uint32_t base = 4u * lane; base < dims; base += 128u) {
                acc(__ldg(p.query + base), __ldg(v + base), a0, b0);
                if (base + 1 < dims) acc(__ldg(p.query + base + 1), __ldg(v + base + 1), a1, b1);
                if (base + 2 < dims) acc(__ldg(p.query + base + 2), __ldg(v + base + 2), a2_, b2);
                if (base + 3 < dims) acc(__ldg(p.query + base + 3), __ldg(v + base + 3), a3, b3);
            }
        }
        const float s0 = warp_butterfly_sum(__fadd_rn(__fadd_rn(a0, a1), __fadd_rn(a2_, a3)));
        float d;
        if (METRIC == kCosine) {
            const float s1 = warp_butterfly_sum(__fadd_rn(__fadd_rn(b0, b1), __fadd_rn(b2, b3)));
            d = finish_cos(s0, a2, sqrt_a2, s1);
        } else if (METRIC == kDot) d = finish_dot(s0);
        else d = finish_l2(s0);
        const bool ok = finite_f32(d);
        if (EMIT) {
            if (lane == 0) p.dist_keys[row] = (ok && row_allowed(p, row)) ? orderable_u32(d) : WAXVS_UKEY_NONE;
        } else if (ok) {
            const uint64_t key = make_key(d, row);
            if (key < tk.thresh && row_allowed(p, row)) {
                if (E == 1) tk.insert(key, lane, k);
                else {
                    if (tk.npend == 32) tk.flush(lane, k);
                    tk.park(key, lane);
                }
            }
        }
    }
    if (!EMIT) {
        if (E > 1) tk.flush(lane, k);
        finish_topk<E>(p, tk, lists, warp, lane, warps);
    }
}

}  // namespace waxvs
