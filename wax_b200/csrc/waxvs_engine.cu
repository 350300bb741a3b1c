// waxvs_engine.cu -- host side of libwaxvs_cuda.so: the engine object behind include/wax_vs_cuda.h.
//
// What it mirrors (paths relative to the Wax repository root): the state and behaviour of
//   actor MetalVectorEngine            Sources/WaxVectorSearch/MetalVectorEngine.swift:17-893
// with USearchVectorEngine's metric coverage (USearchVectorEngine.swift:44-67) -- the corpus matrix resident
// on the device (here: HBM, row-major fp32), a frameIds side array, a pool of per-search scratch contexts
// (the transient buffer pool, :84-121), upsert/ordered-remove mutation semantics (:330-444), the MV2V
// encoding=2 blob (:682-815) -- re-designed for a discrete 180 GB GPU: id->row hash instead of the O(N)
// firstIndex(of:) scan, explicit pinned staging, one fused kernel launch per query.
//
// There is NO CPU fallback in this file or anywhere in the product path: without a CUDA device every entry
// point that needs one returns WAX_VS_ERR_CUDA.
#include <cuda_runtime.h>

#include <algorithm>
#include <atomic>
#include <cstdarg>
#include <cstdio>
#include <cstring>
#include <limits>
#include <map>
#include <mutex>
#include <new>
#include <shared_mutex>
#include <string>
#include <unordered_map>
#include <chrono>
#include <random>
#include <thread>
#include <unistd.h>
#include <cmath>
#include <vector>

#include "../../include/wax_vs_cuda.h"
#include "waxvs_common.cuh"
#include "waxvs_scan.cuh"
#include "waxvs_select.cuh"
#include "waxvs_synth.cuh"
#include "waxvs_batch.cuh"

#include "waxvs_group.cuh"
#include "waxvs_group_batch.cuh"
#include "waxvs_where.cuh"
#include "waxvs_terms.cuh"
#include "waxvs_where_groups.cuh"
#include "waxvs_roots.cuh"

#include <cub/cub.cuh>
#include <cudaTypedefs.h>

using namespace waxvs;

// The where items and the term and group-clause units as the host plans them: every clause, the root clause included.
// Each launch stages the form its kernels take (where_pass, launch_term_filter, launch_group_filter).
using WhereFull = Rooted<WhereNearItem>;
using TermUnitR = Rooted<TermUnit>;
using GroupUnitR = Rooted<GroupUnit>;

// ---------------------------------------------------------------------------------------------------------
// errors
static thread_local char g_last_error[512] = "";

static int32_t fail(int32_t code, const char *fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_last_error, sizeof g_last_error, fmt, ap);
    va_end(ap);
    return code;
}
#define CUDA_TRY(expr)                                                                            \
    do {                                                                                          \
        cudaError_t _e = (expr);                                                                  \
        if (_e != cudaSuccess)                                                                    \
            return fail(WAX_VS_ERR_CUDA, "%s failed: %s", #expr, cudaGetErrorString(_e));         \
    } while (0)

struct DeviceGuard {
    int prev = -1, dev;
    bool ok = true;
    explicit DeviceGuard(int device) : dev(device) {
        if (cudaGetDevice(&prev) != cudaSuccess) { prev = -1; }
        if (prev != dev) ok = (cudaSetDevice(dev) == cudaSuccess);
    }
    ~DeviceGuard() { if (prev >= 0) cudaSetDevice(prev); }
    int32_t error() const { return fail(WAX_VS_ERR_CUDA, "failed to select CUDA device %d", dev); }   // when !ok
};

// An owned allocation of `cap` elements: device memory, or (PINNED) mapped + portable host memory that kernels may write
// results straight into (host delivery) from any device.  ensure(n) grows it without keeping the contents; the memory
// goes back on release() or destruction, which must run while the owner's device is current.
template <typename T, bool PINNED>
struct Buf {
    T *p = nullptr;
    size_t cap = 0;     // elements
    Buf() = default;
    Buf(const Buf &) = delete;
    Buf &operator=(const Buf &) = delete;
    ~Buf() { release(); }
    operator T *() const { return p; }
    void release() {
        if (p) PINNED ? cudaFreeHost(p) : cudaFree(p);
        p = nullptr;
        cap = 0;
    }
    int32_t ensure(size_t n, const char *what) {
        if (n <= cap) return WAX_VS_OK;
        release();
        const cudaError_t err = PINNED ? cudaHostAlloc(reinterpret_cast<void **>(&p), n * sizeof(T), cudaHostAllocMapped | cudaHostAllocPortable)
                                       : cudaMalloc(&p, n * sizeof(T));
        if (err != cudaSuccess)
            return fail(WAX_VS_ERR_CUDA, PINNED ? "failed to allocate pinned %s (%zu bytes): %s" : "failed to allocate %s (%zu bytes): %s",
                        what, n * sizeof(T), cudaGetErrorString(cudaGetLastError()));
        cap = n;
        return WAX_VS_OK;
    }
};
template <typename T> using DevBuf = Buf<T, false>;
template <typename T> using PinnedBuf = Buf<T, true>;

// ---------------------------------------------------------------------------------------------------------
// id -> row: open addressing, linear probing.  Replaces frameIds.firstIndex(of:) (MetalVectorEngine.swift:334,385,426).
struct IdMap {
    std::vector<uint64_t> keys;
    std::vector<uint32_t> vals;
    size_t mask = 0, used = 0;
    static uint64_t mix(uint64_t x) {
        x ^= x >> 30; x *= 0xbf58476d1ce4e5b9ull; x ^= x >> 27; x *= 0x94d049bb133111ebull; x ^= x >> 31;
        return x;
    }
    void reset(size_t expect) {
        size_t cap = 64;
        while (cap < expect * 2 + 16) cap <<= 1;
        keys.assign(cap, 0);
        vals.assign(cap, 0xFFFFFFFFu);
        mask = cap - 1;
        used = 0;
    }
    void prefetch(uint64_t id) const {
        if (vals.empty()) return;
        const size_t i = mix(id) & mask;
        __builtin_prefetch(&keys[i]);
        __builtin_prefetch(&vals[i]);
    }
    uint32_t find(uint64_t id) const {
        if (vals.empty()) return 0xFFFFFFFFu;
        for (size_t i = mix(id) & mask;; i = (i + 1) & mask) {
            if (vals[i] == 0xFFFFFFFFu) return 0xFFFFFFFFu;
            if (keys[i] == id) return vals[i];
        }
    }
    void put(uint64_t id, uint32_t row) {
        if (vals.empty() || (used + 1) * 2 > keys.size()) grow();
        for (size_t i = mix(id) & mask;; i = (i + 1) & mask) {
            if (vals[i] == 0xFFFFFFFFu) { keys[i] = id; vals[i] = row; ++used; return; }
            if (keys[i] == id) { vals[i] = row; return; }
        }
    }
    void grow() {
        std::vector<uint64_t> ok; std::vector<uint32_t> ov;
        ok.swap(keys); ov.swap(vals);
        reset(std::max<size_t>(used * 2, 32));
        for (size_t i = 0; i < ov.size(); ++i) if (ov[i] != 0xFFFFFFFFu) put(ok[i], ov[i]);
    }
};

// ---------------------------------------------------------------------------------------------------------
// The shadows the single-query route nominates from (DESIGN 4.1), in the order of their bytes per row: bf16 (the SHADOW
// form of the scan), int8 (INT8) and 4-bit (U4).  Indexes the per-form tables, options, shadows and counters.
enum RouteForm : int { kRouteBf16, kRouteInt8, kRouteU4, kRouteForms };

struct Tuning {
    int variant = 0;      // 0 auto, 1 TMA-staged, 2 direct LDG
    int rows_per_step = 0;  // 0 auto
    int stages = 0;       // 0 auto
    int warps = 0;        // 0 auto
    int grid = 0;         // 0 = one CTA per SM
    int l2_hint = 0;
    int ldg_ctas_per_sm = 4;
    int chunk_steps = -1;   // dynamic scheduling granularity of the TMA kernel: -1 auto (8 steps, fewer when the corpus gives
                            // each warp only a few steps, e.g. 10 K rows x 4 rows per step = 2 500 steps over 1 056 warps), 0 = static round-robin
    int fused_k_max = 128;  // k <= this stays in the single fused launch (register lists); larger k: emit + radix select
    int batch_tensor = 1;   // 1: batches take the wgmma TF32 nominate + exact re-score path when eligible
    int batch_min = 4;      // smallest batch routed to the tensor path
    int time_overlap = 0;   // wax_vs_debug_time_search: alternate consecutive queries over two streams
    int batch_pair = 0;     // 1: CTA pairs of a cluster share each corpus tile through a TMA multicast (needs >= 2 groups)
    uint32_t tma_max_dims = 4096;   // generic TMA shape up to this row length, the direct-load kernel above
    int batch_large_k = 1;  // batches with 128 < k <= 1024 take the tensor-core levels (0: loop the single-query emit + select path)
    int batch_heap = 0;     // 0 auto (cost model + adaptive bump), 16 / 24 / 32 / 64: nominee heap size per (slice, query) = kernel shape
    int batch_noinsert = 0; // instrumentation: GEMM pipeline only (results meaningless)
    int batch_bf16 = 1;     // 1: nominate from a bf16 shadow of the corpus when HBM allows (bf16 wgmma, 2x the TF32 rate; +dims*2 B/row)
    int batch_ares = 1;     // with batch_bf16: keep the CTA's queries resident in shared memory when a 2-stage ring still fits
    int batch_rescore = 0;  // 0 auto; else nominees re-scored exactly per query (256, 512 or 1024)
    int batch_retry = 1;    // queries level 1 cannot prove go through the filter level (TF32, complete by construction) before an exact scan
    int filter_bf16 = 1;    // unproven queries first get a filter pass over the bf16 shadow (half the bytes of an exact scan)
    int filter_cap = 8192;  // candidates per query the filter level may collect (power of two <= 16384); overflow -> exact scan
    int inline_query = 1;   // host entry points: a query of <= 512 floats travels in the kernel parameters (no H2D copy)
    int host_delivery = 1;  // host entry points: the kernel stores the result in mapped host memory + flag (no D2H copy / sync)
    int tail_select = 1;    // TMA-staged kernels: radix-selection tail instead of pairwise list merges (same results)
    int shard_fused = 1;    // sharded search: exchange + merge inside the scan launch (0: separate 1-CTA launch)
    int batch_l2 = 0;       // 1: l2 batches take the tensor-core levels too (off: they loop the single-query path).  A staging
                            // switch: the default flips once the l2 levels have H100 figures behind them
    int single_shadow = 0;  // 1: single queries / batches below batch_min take the tensor-core bf16-shadow nominations
                            // (one query in a 128-query wgmma tile) instead of the shadow route of `shadow_scan`
    uint64_t filter_bitset_bytes = 2ull << 30;   // per-query filters: row bitsets one tensor pass may hold
    uint64_t rebalance_slab_bytes = 256ull << 20;   // a rebalance merge's slab and staging chunk (absorb_rows), each
    int shadow_scan = 1;    // single queries (cosine / dot, k <= 32) nominate on the bf16 shadow with the streaming scan, then
                            // an exact re-score + proof, the fp32 scan only when the proof fails (0: always the fp32 scan)
    // Each form of the route, by RouteForm (options "<shadow|int8|u4>_scan_min_bytes", "_rows_per_step", "_warps",
    // "_stages"): the smallest fp32 corpus it takes, and the shape of its nominating scan (0 auto).
    struct Route { uint64_t min_bytes; int rows_per_step = 0, warps = 0, stages = 0; };
    Route route[kRouteForms] = {
        {512ull << 20},    // bf16: smaller corpora are latency-bound: two more launches and a shadow do not pay; on H100
                           // at 384 dims the route breaks even near 380 MB (DESIGN 5)
        {512ull << 20},    // int8 (half the bytes of the bf16 shadow), for corpora whose measured int8 bound is no coarser
                           // than the bf16 one (DESIGN 4.1, 5)
        {2048ull << 20},   // 4-bit (half the bytes again), while its proofs hold (DESIGN 4.1, 5): its re-score of
                           // thousands of nominees is a fixed cost, measured only at 15 GB, so corpora of a GB or two
                           // stay on the int8 form
    };
};

// Per-search scratch: the analogue of TransientBuffers (MetalVectorEngine.swift:36-41, :84-117).
struct SearchCtx {
    cudaStream_t stream = nullptr;
    bool own_stream = false;
    const uint64_t *row_keys = nullptr;            // the engine's device row keys while a call that reports global rows
                                                   // (device and shard entry points) holds this context; else nullptr
    DevBuf<float> d_queries;
    DevBuf<wax_vs_candidate> d_out;
    PinnedBuf<float> h_queries;
    PinnedBuf<wax_vs_candidate> h_out;
    DevBuf<uint64_t> d_block_keys;
    DevBuf<uint32_t> d_ticket;
    DevBuf<uint32_t> d_dist_keys;                  // large-k path
    DevBuf<SelectState> d_select;
    DevBuf<uint64_t> d_sel_keys;                   // 16384 u64
    cudaEvent_t ev0 = nullptr, ev1 = nullptr;
    DevBuf<uint64_t> d_heaps;                      // batched path: nominee heaps
    DevBuf<uint32_t> d_ok;                         // batched path: per-query proof flags
    PinnedBuf<uint32_t> h_ok;
    DevBuf<uint32_t> d_tau;                        // batched path: shared per-query thresholds
    DevBuf<__nv_bfloat16> d_queries_bf16;          // batched bf16 path: converted queries
    DevBuf<float> d_retry_q;                       // bf16 -> TF32 retry: compacted queries
    DevBuf<wax_vs_candidate> d_retry_out;
    DevBuf<uint32_t> d_retry_ok;
    DevBuf<float> d_tau_star;                      // level 1 -> filter level: per-query thresholds
    PinnedBuf<float> h_tau_star;
    DevBuf<float> d_filter_tau;                    // compacted thresholds of the unproven queries
    PinnedBuf<float> h_filter_tau;
    DevBuf<uint32_t> d_cand_count;
    DevBuf<uint32_t> d_cand_rows;
    DevBuf<uint64_t> d_cand_keys;
    DevBuf<uint32_t> d_mask;                       // filtered search: row bitsets [filters][words]
    DevBuf<uint32_t> d_filter_rows;                // filtered search: the filters' resolved rows, concatenated
    DevBuf<uint64_t> d_filter_spec;                // filtered search: bitset builder spec (filter_bits_init_kernel)
    DevBuf<uint32_t> d_query_filter;               // filtered search: each query's bitset index
    DevBuf<uint32_t> d_retry_filter;               // filter level: bitset indices of the compacted queries
    DevBuf<uint2> d_gather_span;                   // filtered search: each gathered query's span of d_filter_rows
    DevBuf<uint64_t> d_gather_keys;                // filtered search: keys of the listed rows
    DevBuf<uint32_t> d_order;                      // device-form where search: staged order, then each staged query's k
    DevBuf<wax_vs_candidate> d_shard_local;        // sharded search: this rank's list before the exchange [kShardKCap]
    DevBuf<unsigned long long> d_group_best;       // grouped search: each group's best (key, row)
    DevBuf<uint32_t> d_group_keys;                 // grouped search: row-indexed keys of the groups' best rows
    DevBuf<uint2> d_group_spans;                   // grouped search: CSR span of each selected group
    PinnedBuf<uint2> h_group_spans;
    DevBuf<ExpandItem> d_expand_items;             // grouped search: expansion work items, all levels
    DevBuf<uint64_t> d_expand[3];                  // grouped search: expansion lists (two level buffers, the result)
    PinnedBuf<uint64_t> h_expand;
    DevBuf<uint64_t> d_bg_keys;                    // batched grouped search: [query][top_groups][per_group] result keys
    PinnedBuf<uint64_t> h_bg_keys;
    DevBuf<uint32_t> d_bg_status;                  // batched grouped search: covered flag per query, then the expansion count
    PinnedBuf<uint32_t> h_bg_status;
    DevBuf<CoverExpand> d_bg_expand;               // batched grouped search: the groups to expand
    PinnedBuf<CoverExpand> h_bg_expand;
    DevBuf<ScoreItem> d_score_items;               // batched grouped search: expansion tiles (level 0)
    PinnedBuf<unsigned long long> h_flag;          // host-delivery completion flag
    unsigned long long host_seq = 0;               // last value the flag was asked to take
    DevBuf<WhereFull> d_where_items;               // where search: predicates of the count / compaction / bitset launches
                                                   // (in the launch's form: WhereItemOf<located, rooted>)
    DevBuf<uint32_t> d_where_counts;               // where search: rows passing each predicate, then compaction cursors
    DevBuf<uint64_t> d_term_ids;                   // where_terms search: the call's distinct required term ids ...
    DevBuf<TermSpan> d_term_spans;                 // ... their posting spans
    DevBuf<TermUnitR> d_term_units;                // ... the units of term_filter_kernel (in the launch's form)
    DevBuf<uint32_t> d_term_counts;                // ... their counts, then listing cursors
    DevBuf<uint32_t> d_term_deny;                  // ... and their deny-lists' rows, each list ascending
    DevBuf<uint64_t> d_gw_ids;                     // where_groups search: the call's distinct group ids ...
    DevBuf<GroupSpan> d_gw_resolved;               // ... their dense groups and CSR spans
    DevBuf<GroupSpan> d_gw_spans;                  // ... each unit's groups, with their prefix
    DevBuf<GroupUnitR> d_gw_units;                 // ... the units of where_group_filter_kernel (in the launch's form)
    DevBuf<uint32_t> d_gw_counts;                  // ... their counts, then listing cursors
    DevBuf<uint32_t> d_gw_deny;                    // ... and their deny-lists' rows, each list ascending
    DevBuf<uint32_t> d_proof_count;                // shadow route: [0] proofs that held, [1] that failed (guarded scan) ...
    PinnedBuf<uint32_t> h_proof_count;             // ... and their mapped host mirror
    uint32_t seen_failed = 0;                      // h_proof_count[1] when the host last looked
    bool last_u4 = false;                          // the last route query enqueued here nominated from the 4-bit shadow
    DevBuf<uint32_t> d_u4_aux;                     // 4-bit route: [0] cut key of the rows left out, [1] rho_q (ScanParams::u4_aux),
                                                   // [2] the cut key the last re-score proved with (read-out)
    ~SearchCtx() {                                 // the buffers release themselves
        if (ev0) cudaEventDestroy(ev0);
        if (ev1) cudaEventDestroy(ev1);
        if (own_stream && stream) cudaStreamDestroy(stream);
    }
};

struct MultiEngine;   // waxvs_multi.cuh

struct wax_vs_engine {
    MultiEngine *multi = nullptr;   // a multi-device handle (n_devices >= 2): its shards and state, else nullptr
    int device = 0;
    int sm_count = 132;
    size_t smem_optin = 0;
    uint32_t dims = 0;
    uint8_t similarity = 0;

    float *d_corpus = nullptr;
    uint64_t cap_rows = 0, n_rows = 0;

    // frame ids: implicit (id_base + row) after fill_synthetic until the first mutation, else explicit.
    bool ids_identity = true;
    uint64_t id_base = 0;
    std::vector<uint64_t> ids;
    IdMap map;
    bool map_valid = true;
    // Frame ids are handed out in increasing order by the store, so the id array is normally SORTED: then a lookup is a
    // binary search in it and bulk appends touch no hash table at all; the table is built only once an out-of-order id
    // arrives (and kept from then on).  Order-preserving removes and in-place upserts keep the array sorted.
    bool ids_sorted = true;
    DevBuf<uint64_t> d_ids;
    bool d_ids_dirty = true;
    std::mutex ids_mu;
    // Row keys of a keyed shard (DESIGN 4.15): keys[r] is row r's insertion sequence number in the sharded corpus, strictly
    // increasing with r, and the device entry points report row r as row_offset + keys[r].  Absent (keys_set false, a row
    // is reported as row_offset + r) until wax_vs_add_batch_keyed or wax_vs_deserialize_rows runs.  Every mutator keeps
    // keys aligned with `ids` and d_keys current.
    bool keys_set = false;
    std::vector<uint64_t> keys;
    DevBuf<uint64_t> d_keys;

    std::shared_mutex rw;  // readers: search / serialize; writer: mutators (AsyncReadWriteLock, :56-80)
    std::mutex pool_mu;
    std::vector<SearchCtx *> pool;
    std::unordered_map<void *, SearchCtx *> stream_ctx;  // wax_vs_search_device: one ctx per caller stream
    uint64_t pool_allocs = 0, pool_reuses = 0;
    Tuning tune;

    // cached per corpus version for the batched path: 1/|v| per row and max |v|; l2 engines also |v|^2 / 2 per row
    DevBuf<float> d_inv_norm;
    DevBuf<uint32_t> d_max_norm;
    DevBuf<float> d_half_sq;
    uint64_t norms_rows = 0;       // rows [0, norms_rows) of d_inv_norm (and d_half_sq) are valid (appends extend it, other
                                   // mutations reset it)
    std::mutex norms_mu;
    // Shadows of the corpus, by RouteForm (cached per corpus version, guarded by norms_mu): bf16 (two values per word;
    // also the batched bf16 nominations), int8 (four biased codes per word) and 4-bit (16 levels, eight codes per word)
    // for the single-query route (DESIGN 4.1).  The coded two also hold one scale per row (the 4-bit one: a half step;
    // padded to whole scan steps) and the measured bound rho_max (fp32 bits on the device; read back once per build
    // together with max|v|, giving the bound the finish uses).
    struct Shadow {
        DevBuf<uint32_t> codes;
        DevBuf<float> scale;
        DevBuf<uint32_t> rho;
        uint64_t rows = 0;             // rows [0, rows) are valid; valid = covers every live row
        bool valid = false, unavailable = false;
        bool coarse = false;           // the last build measured a bound too coarse for the route: none is built again until
                                       // the rows are rewritten (invalidate_row_caches with no prefix) or its min_bytes option is set
        float rho_max = 0.0f, eps_rel = INFINITY;   // rho_max, and rho_max / M rounded up (M = 1 cosine, max|v| dot);
                                                    // bf16: eps_rel = kBf16Eps once built
        void release() { codes.release(); scale.release(); rows = 0; valid = false; }
        // A kept prefix keeps rho_max too: still an upper bound.  A shadow with a measured bound is no longer valid, so
        // that its next use reads rho_max and max|v| back again; the bf16 one stays valid over a kept prefix
        // (shadow_bytes reports the prefix).
        void invalidate(uint64_t keep_prefix, bool measured_bound) {
            rows = std::min(rows, keep_prefix);
            if (measured_bound || rows == 0) valid = false;
            if (keep_prefix == 0) coarse = false;
        }
    } shadows[kRouteForms];
    // The 4-bit bound is 16 times the int8 one, so whether its nominees prove depends on the scores: a failed 4-bit proof
    // sends the next u4_demote_window eligible queries to the int8 form (u4_demoted counts them down), and the window
    // doubles when the first 4-bit query after it fails again.
    uint32_t u4_demoted = 0, u4_demote_window = 16;
    bool u4_probing = false;                              // the next 4-bit proof decides whether the window doubles
    uint64_t single_route_queries[kRouteForms] = {};      // single queries nominated from each shadow (pool_mu)
    uint32_t last_scan[10] = {};                          // the form of the last fp32 scan launched (wax_vs_debug_last_scan; pool_mu)
    uint64_t batch_tensor_queries = 0, batch_fallback_queries = 0;   // instrumentation
    uint64_t batch_bf16_queries = 0, batch_retry_queries = 0, batch_tf32_queries = 0, batch_filter_bf16_queries = 0;
    uint64_t filter_bitset_passes = 0;
    // Groups (wax_vs_set_groups): groups[r] = row r's group id, kept aligned with `ids` by every mutator.  Empty while
    // groups_set is false: then every row is its own group (group id = frame id) and nothing is stored.
    bool groups_set = false;
    std::vector<uint64_t> groups;
    // Device group index for grouped search (waxvs_group.cuh), cached per corpus version and grouping: rows sorted by
    // (group id, row) as perm + starts, each row's dense group and each dense group's id (ascending: the sharded grouped
    // search looks groups up by id).  Every mutator and set_groups invalidate it; the first grouped search after that
    // rebuilds it under group_mu (concurrent readers hold only the read lock).
    struct GroupIndex {
        DevBuf<uint32_t> perm, row_group, starts;
        DevBuf<uint64_t> ids;
        uint32_t n_groups = 0;
        bool valid = false;
    } gindex;
    std::mutex group_mu;
    uint64_t group_index_builds = 0;   // instrumentation (pool_mu)
    uint64_t where_group_units = 0;        // where_groups search: units with a group clause planned on the device ...
    uint64_t where_group_rows_walked = 0;  // ... and the candidate positions their walks visit (pool_mu)
    // Root tags (wax_vs_set_root_tags): the caller's 64-bit word per group id, ids ascending with their words, keyed by
    // group and not by row, so no row mutator touches them; deserialize clears them.  The device column col[r] = the word
    // of row r's group (waxvs_roots.cuh) is a cache like the group index: every mutator, set_groups and set_root_tags
    // invalidate it; the first search with a root clause after that rebuilds it under root_mu.  Nothing is allocated
    // until then.
    struct RootTags {
        std::vector<uint64_t> ids, tags;
        DevBuf<uint64_t> col;
        bool col_valid = false;
    } roots;
    std::mutex root_mu;
    uint64_t root_column_builds = 0;       // instrumentation (pool_mu)
    // Frame attributes (wax_vs_set_attributes): attrs[r] = row r's (timestamp, tags), kept aligned with `ids` by every
    // mutator exactly as `groups` is.  Empty while attrs_set is false: then every row has timestamp 0 and tags 0.
    bool attrs_set = false;
    std::vector<AttrRow> attrs;
    // Device mirror (16 bytes per row) for the where predicates, a cache like the group index: every mutator and
    // set_attributes invalidate it; the first search that needs it rebuilds it under attrs_mu and publishes it complete.
    DevBuf<AttrRow> d_attrs;
    bool attrs_dev_valid = false;
    std::mutex attrs_mu;
    uint64_t attribute_uploads = 0;    // instrumentation (pool_mu)
    // Frame locations (wax_vs_set_locations): locs[r] = row r's PhotoRAG bins, kept aligned with `ids` by every mutator
    // exactly as `attrs` is.  Empty while locs_set is false: then no row has a location.  The device mirror (8 bytes
    // per row) is the attribute mirror's twin: invalidated with it, rebuilt under attrs_mu by the first launch that tests a
    // box.
    bool locs_set = false;
    std::vector<LocRow> locs;
    DevBuf<LocRow> d_locs;
    bool locs_dev_valid = false;
    uint64_t location_uploads = 0;     // instrumentation (pool_mu)
    // Frame terms (wax_vs_set_terms): row r's sorted, distinct term ids are term_pool[term_refs[r].off, + .n), kept
    // aligned with `ids` by every mutator exactly as `attrs` is.  A set_terms appends to the pool and repoints the row;
    // term_garbage counts the pool entries no row points at, and the pool is compacted when they pass half of it.  Empty
    // while terms_set is false: then no row has a term.
    struct TermRef {
        uint64_t off;
        uint32_t n;
    };
    bool terms_set = false;
    std::vector<TermRef> term_refs;
    std::vector<uint64_t> term_pool;
    uint64_t term_garbage = 0;
    // Device inverted index for the term clauses (waxvs_terms.cuh), a cache like the group index: every mutator and
    // set_terms invalidate it; the first where_terms search after that rebuilds it under term_mu.
    // Invalidation releases it (under the write lock), so a build only allocates: a build inside a sharded where search
    // must not free device memory (reserve_shard_scratch).  For the same reason a shard rank keeps the build's scratch
    // until then; other engines release it at the end of the build.
    struct TermIndex {
        DevBuf<uint64_t> keys, start;
        DevBuf<uint32_t> postings;
        DevBuf<uint64_t> sort_keys, sorted_keys;   // build scratch
        DevBuf<uint32_t> sort_rows, heads, numbering;
        DevBuf<uint8_t> temp;
        uint32_t n_terms = 0;
        uint64_t n_postings = 0;
        bool valid = false;
        void release_scratch() {
            sort_keys.release(); sorted_keys.release(); sort_rows.release(); heads.release(); numbering.release();
            temp.release();
        }
        void release() {
            keys.release(); start.release(); postings.release();
            release_scratch();
            n_terms = 0;
            n_postings = 0;
            valid = false;
        }
    } tindex;
    std::mutex term_mu;
    uint64_t term_index_builds = 0;    // instrumentation (pool_mu)
    uint64_t grouped_batch_covered_queries = 0, grouped_batch_expanded_groups = 0, grouped_batch_fallback_queries = 0;
    uint64_t grouped_batch_expansion_passes = 0;
    uint64_t shard_grouped_expanded_groups = 0;
    // Adaptive level choice: when more than a quarter of a batch fails the coarse bf16 bound (tightly clustered
    // neighbours), the next 16 batches nominate in TF32 straight away, then bf16 is probed again.
    uint32_t bf16_skip_batches = 0;
    // Single queries: after a failed shadow proof the next kShadowSkipQueries eligible queries take the fp32 scan directly
    uint32_t shadow_scan_skip = 0;
    // adaptive nominee-heap size (bf16 level 1): a batch that left queries unproven makes the next `heap_bump_ttl` batches
    // use one size more than the model picks; a failure right after probing back down doubles the time-out
    uint32_t heap_bump = 0, heap_bump_ttl = 0, heap_backoff = 256;
    bool heap_probing = false;
    uint32_t last_heap = 0;
    // Bulk ingest / export staging (SURVEY 8f-3): two pinned buffers so that the host-side copy of chunk i+1 overlaps
    // the DMA of chunk i, one copy stream, a device staging area for upserts and for the compaction of removes.
    struct Ingest {
        cudaStream_t stream = nullptr;
        cudaEvent_t ev[2] = {nullptr, nullptr};
        uint8_t *pin[2] = {nullptr, nullptr};
        size_t pin_bytes = 0;
        DevBuf<float> d_stage;
        DevBuf<uint32_t> d_index;
        int threads = 1;
        ~Ingest() {
            for (int i = 0; i < 2; ++i) {
                if (pin[i]) cudaFreeHost(pin[i]);
                if (ev[i]) cudaEventDestroy(ev[i]);
            }
            if (stream) cudaStreamDestroy(stream);
        }
    } ing;
    uint64_t ingest_h2d_bytes = 0, ingest_d2h_bytes = 0;         // instrumentation
    std::mutex ingest_mu;                                        // readers that use the staging (serialize)
    // Device-path searches (wax_vs_search_device & co.) return while their kernels are still in flight on the
    // caller's stream.  Mutators must not touch the corpus under them: every mutator drains the device first when
    // this flag says something was enqueued since the last drain.
    std::atomic<bool> async_pending{false};
    unsigned long long *debug_trace = nullptr;   // wax_vs_debug_phase_trace: device buffer the scan kernels stamp (else nullptr)

    // Row-sharded search (wax_vs_shard_*): this engine is rank `rank` of `world`; box[r] = rank r's mailbox.
    struct Shard {
        bool open = false, connected = false;
        int rank = 0, world = 0;
        uint64_t row_offset = 0;
        ShardMailbox *box[kShardMaxRanks] = {};
        bool ipc[kShardMaxRanks] = {};            // mapped with cudaIpcOpenMemHandle (closed in shard_close)
        unsigned long long seq = 0;               // collective calls issued so far (same on every rank)
        unsigned long long timeout_ns = 20ull * 1000 * 1000 * 1000;
        std::mutex mu;                            // one collective call at a time per rank: seq order = issue order
        SearchCtx *ctx = nullptr;                 // host entry point: stream + scratch
        DevBuf<wax_vs_candidate> d_final;         // [kShardKCap]
        PinnedBuf<wax_vs_candidate> h_final;      // [kShardKCap]: the kernel writes the merged result here
        PinnedBuf<unsigned long long> h_flag;     // seq when h_final is complete
    } shard;
};

extern "C" { static void shard_teardown(wax_vs_engine *e, bool free_own); }

static const uint64_t *device_row_keys(const wax_vs_engine *e) { return e->keys_set ? e->d_keys.p : nullptr; }

// Called by every mutator after it has taken the write lock (and selected the device).
static void drain_device_path(wax_vs_engine *e) {
    if (e->async_pending.exchange(false)) cudaDeviceSynchronize();
}
// Derived per-row caches (1/|v|, bf16 shadow) after a mutation.  keep_prefix: rows [0, keep_prefix) are untouched (a pure
// append keeps everything it had); 0 = rebuild from scratch on the next batched search.
static void invalidate_row_caches(wax_vs_engine *e, uint64_t keep_prefix) {
    e->norms_rows = std::min(e->norms_rows, keep_prefix);
    for (int f = 0; f < kRouteForms; ++f) e->shadows[f].invalidate(keep_prefix, f != kRouteBf16);
    e->gindex.valid = false;           // appends too: the new rows need index entries
    e->roots.col_valid = false;        // and the root column, read through it
    e->attrs_dev_valid = false;        // likewise the attribute mirror
    e->locs_dev_valid = false;         // and the location mirror
    e->tindex.release();               // and the term index
    // The row-sized device buffers of the where mirrors and of the collective scratch go too, here under the write lock
    // with the device drained: a sharded where search then only allocates them for the new row count, and never frees
    // (reserve_shard_scratch).
    e->d_attrs.release();
    e->d_locs.release();
    if (SearchCtx *c = e->shard.ctx) {
        c->d_filter_rows.release();
        c->d_mask.release();
        c->d_term_deny.release();
    }
}

// The term pool rewritten in row order once more than half of it is garbage (set_terms, remove_batch).
static void compact_term_pool(wax_vs_engine *e) {
    if (e->term_garbage * 2 <= e->term_pool.size()) return;
    std::vector<uint64_t> pool;
    pool.reserve(e->term_pool.size() - e->term_garbage);
    for (auto &t : e->term_refs) {
        const uint64_t off = pool.size();
        pool.insert(pool.end(), e->term_pool.begin() + t.off, e->term_pool.begin() + t.off + t.n);
        t.off = t.n ? off : 0;
    }
    e->term_pool.swap(pool);
    e->term_garbage = 0;
}
// No row has terms (deserialize, fill_synthetic): MV2V has no place for them.
static void clear_terms(wax_vs_engine *e) {
    e->terms_set = false;
    e->term_refs.clear(); e->term_refs.shrink_to_fit();
    e->term_pool.clear(); e->term_pool.shrink_to_fit();
    e->term_garbage = 0;
    e->tindex.release();               // the index goes with them
}

// ---------------------------------------------------------------------------------------------------------
// scratch contexts
static int32_t ctx_new(wax_vs_engine *e, SearchCtx **out, bool with_stream) {
    SearchCtx *c = new (std::nothrow) SearchCtx();
    if (!c) return fail(WAX_VS_ERR_CUDA, "out of host memory");
    auto bail = [&](int32_t rc) { delete c; return rc; };
    if (with_stream) {
        if (cudaStreamCreateWithFlags(&c->stream, cudaStreamNonBlocking) != cudaSuccess)
            return bail(fail(WAX_VS_ERR_CUDA, "cudaStreamCreate failed"));
        c->own_stream = true;
    }
    const size_t block_keys = static_cast<size_t>(std::max(e->sm_count * 8, 2048)) * 128;
    if (cudaMalloc(&c->d_block_keys.p, block_keys * sizeof(uint64_t)) != cudaSuccess ||
        cudaMalloc(&c->d_ticket.p, 4 * sizeof(uint32_t)) != cudaSuccess ||      // [0] ticket, [1] work counter
        cudaMemset(c->d_ticket, 0, 4 * sizeof(uint32_t)) != cudaSuccess ||
        cudaEventCreate(&c->ev0) != cudaSuccess || cudaEventCreate(&c->ev1) != cudaSuccess)
        return bail(fail(WAX_VS_ERR_CUDA, "failed to allocate search scratch: %s",
                         cudaGetErrorString(cudaGetLastError())));
    c->d_block_keys.cap = block_keys;
    c->d_ticket.cap = 4;
    *out = c;
    return WAX_VS_OK;
}

static int32_t ctx_acquire(wax_vs_engine *e, SearchCtx **out) {
    {
        std::lock_guard<std::mutex> g(e->pool_mu);
        if (!e->pool.empty()) {
            *out = e->pool.back();
            e->pool.pop_back();
            ++e->pool_reuses;
            (*out)->row_keys = nullptr;
            return WAX_VS_OK;
        }
        ++e->pool_allocs;
    }
    return ctx_new(e, out, true);
}
static void ctx_release(wax_vs_engine *e, SearchCtx *c) {
    std::lock_guard<std::mutex> g(e->pool_mu);
    e->pool.push_back(c);
}
// A pooled context held for the length of one call.  clears_trace: also detach the phase-trace buffer on the way out.
struct CtxLease {
    wax_vs_engine *e;
    SearchCtx *c = nullptr;
    bool clears_trace = false;
    explicit CtxLease(wax_vs_engine *eng, bool clear_trace = false) : e(eng), clears_trace(clear_trace) {}
    CtxLease(const CtxLease &) = delete;
    CtxLease &operator=(const CtxLease &) = delete;
    ~CtxLease() {
        if (c) ctx_release(e, c);
        if (clears_trace) e->debug_trace = nullptr;
    }
    int32_t acquire() { return ctx_acquire(e, &c); }
};
// The scratch context bound to a caller-owned stream (device-path entry points): find-or-create in ONE critical
// section, so two threads that first use the same stream cannot both insert (and leak) a context.  These calls report
// global rows, so the context carries the row keys.
static int32_t ctx_for_stream(wax_vs_engine *e, void *cuda_stream, SearchCtx **out) {
    std::lock_guard<std::mutex> pg(e->pool_mu);
    auto it = e->stream_ctx.find(cuda_stream);
    if (it != e->stream_ctx.end()) {
        *out = it->second;
        (*out)->row_keys = device_row_keys(e);
        return WAX_VS_OK;
    }
    SearchCtx *c = nullptr;
    int32_t rc = ctx_new(e, &c, false);
    if (rc) return rc;
    c->stream = static_cast<cudaStream_t>(cuda_stream);
    c->row_keys = device_row_keys(e);
    e->stream_ctx[cuda_stream] = c;
    ++e->pool_allocs;
    *out = c;
    return WAX_VS_OK;
}

// ---------------------------------------------------------------------------------------------------------
// kernel dispatch
struct TmaConfig { int C, R, warps, stages; size_t smem; };

// The unrolled shapes of the TMA scan: rows of C x 128 elements (12: the 1536-dim embeddings).
constexpr int kUnrolledC[7] = {1, 2, 3, 4, 6, 8, 12};
// Index in kUnrolledC of rows of d elements, -1 when no unrolled shape has them.
static int unrolled_index(uint32_t d) {
    for (int i = 0; i < 7; ++i)
        if (d == 128u * kUnrolledC[i]) return i;
    return -1;
}
// Dynamic shared memory a TMA-staged scan may take: the opt-in limit minus the kernels' static shared memory.
static size_t tma_smem_budget(const wax_vs_engine *e) { return (e->smem_optin ? e->smem_optin : 232448) - 4096; }
// ... and what a ring of `stages` steps of stage_bytes per warp takes (with each warp's barriers and list).
static size_t tma_ring_smem(int warps, int stages, size_t stage_bytes) {
    return static_cast<size_t>(warps) * stages * (stage_bytes + 8 + 4) + static_cast<size_t>(warps) * 1024 + 16;
}

// The fp32 scan's shape (the route's forms: pick_route_config).
static bool pick_tma_config(const wax_vs_engine *e, TmaConfig *cfg, int mode = 0) {
    const uint32_t d = e->dims;
    if (d % 4u != 0) return false;                      // rows must be 16-byte multiples for the bulk copy
    const size_t budget = tma_smem_budget(e);
    const int ci = unrolled_index(d);
    const int C = ci < 0 ? 0 : kUnrolledC[ci];
    if (C == 0 && d < 32) return false;                  // a few floats per row: the direct-load kernel
    if (C == 0 && d > e->tune.tma_max_dims) return false;   // very long rows: too few warps fit beside two stages, the
                                                             // direct-load kernel takes them
    // Rows per step / warps per CTA by row length: keep a step at >= 4-12 KB and give short rows more warps (their bound
    // is per-row instruction latency, not bytes in flight).  These defaults were chosen on B200, not re-tuned on H100; the
    // `rows_per_step` / `warps` / `stages` options override them.
    int R, warps_default = 8;
    if (C == 0) {                                      // generic shape: run-time chunk count, query in shared memory
        // keep a step at >= 2-8 KB: short generic rows (dims < 128, 160, 300, 400, ...) take 8 or 4 rows per step and
        // more warps, like the unrolled C <= 2 shapes
        // (long rows: as many rows as keep a step at <= 32 KB -- the few warps that then fit still hold ~190 KB in flight)
        int auto_r = d > 256 ? 4 : 8;
        if (d > 640) { auto_r = 8; while (auto_r > 1 && static_cast<size_t>(auto_r) * d * 4 > 32768) auto_r >>= 1; }
        if (d > 3072) auto_r = 1;       // 12-16 KB rows: one per step keeps six warps in flight
        const int want_r = e->tune.rows_per_step;
        R = (want_r == 1 || want_r == 2 || want_r == 4 || want_r == 8) ? want_r : auto_r;
        if (R == 8) warps_default = 16;
        else if (R == 4) warps_default = 12;
    } else if (C == 12) {
        R = e->tune.rows_per_step == 1 || e->tune.rows_per_step == 2 ? e->tune.rows_per_step : 2;
    } else if (C >= 6) {
        R = e->tune.rows_per_step == 2 || e->tune.rows_per_step == 4 ? e->tune.rows_per_step : 2;
    } else {
        R = e->tune.rows_per_step == 4 || e->tune.rows_per_step == 8 ? e->tune.rows_per_step : (C <= 2 ? 8 : 4);
        if (C == 1) warps_default = 16;
        else if (C == 2) warps_default = 12;
        // wide lists (33 <= k <= 128, four keys per lane): 16 warps per CTA spread the list upkeep; below 8 GB of corpus
        // that won over 8 warps on B200, above it the 8-warp shape's 48 KB in flight did (chosen on B200, not re-tuned on H100)
        else if (mode == 1 && static_cast<uint64_t>(e->n_rows) * d * 4 < (8ull << 30)) warps_default = 16;
    }
    // Default ring depth 2: ~48 KB in flight per SM for the 8-warp shapes (the `stages` option overrides it).  The route's
    // forms have options of their own: they run right before a guarded fp32 scan that keeps the fp32 shape.
    const int stages = e->tune.stages > 0 ? e->tune.stages : 2;
    const size_t stage_bytes = static_cast<size_t>(R) * d * sizeof(float);
    const size_t query_bytes = C == 0 ? (static_cast<size_t>(d) * 4 + 512 + 32) : 0;
    auto smem_for = [&](int w) { return tma_ring_smem(w, stages, stage_bytes) + query_bytes; };
    int warps = std::max(1, std::min(16, e->tune.warps ? e->tune.warps : warps_default));
    if (!e->tune.warps) while (warps > 2 && smem_for(warps) > budget) --warps;   // long rows: fewer warps per CTA
    if (smem_for(warps) > budget) return false;
    cfg->C = C; cfg->R = R; cfg->warps = warps; cfg->stages = stages; cfg->smem = smem_for(warps);
    return true;
}

// The opt-in shared-memory limit is per function and per device: set it once per engine (= per device), and again
// only if a larger ring is requested, instead of on every launch -- it costs more host time than a 10 K-row scan.
// The opt-in dynamic shared memory of `kernel` on e's device, raised to at least `bytes`.  The attribute belongs to the
// function on the device, not to an engine, so the grants are kept per (device, kernel) for the whole process: engines
// that share a device (the ranks of a shard group in one process) only ever raise it, never lower it under another.
template <typename K>
static cudaError_t grant_smem(wax_vs_engine *e, K kernel, size_t bytes) {
    static std::mutex mu;
    static std::map<std::pair<int, const void *>, int> granted;
    std::lock_guard<std::mutex> g(mu);
    int &have = granted[{e->device, reinterpret_cast<const void *>(kernel)}];
    if (have >= static_cast<int>(bytes)) return cudaSuccess;
    cudaError_t err = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(bytes));
    if (err == cudaSuccess) have = static_cast<int>(bytes);
    return err;
}

template <int C, int R, int M, int E, bool EMIT, bool SHADOW = false, bool INT8 = false, bool U4 = false>
static cudaError_t launch_tma_inst(wax_vs_engine *e, const ScanParams &p, int grid, const TmaConfig &cfg, cudaStream_t s) {
    cudaError_t err = grant_smem(e, scan_tma_kernel<C, R, M, E, EMIT, SHADOW, INT8, U4>, cfg.smem);
    if (err != cudaSuccess) return err;
    scan_tma_kernel<C, R, M, E, EMIT, SHADOW, INT8, U4><<<grid, cfg.warps * 32, cfg.smem, s>>>(p);
    return cudaGetLastError();
}
// mode: 0 = fused list k <= 32, 1 = fused list k <= 128, 2 = emit distance keys
template <int C, int R>
static cudaError_t launch_tma_cr(wax_vs_engine *e, const ScanParams &p, int grid, const TmaConfig &cfg, int metric, int mode,
                                 cudaStream_t s) {
    switch (metric * 3 + mode) {
        case 0: return launch_tma_inst<C, R, kCosine, 1, false>(e, p, grid, cfg, s);
        case 1: return launch_tma_inst<C, R, kCosine, 4, false>(e, p, grid, cfg, s);
        case 2: return launch_tma_inst<C, R, kCosine, 1, true>(e, p, grid, cfg, s);
        case 3: return launch_tma_inst<C, R, kDot, 1, false>(e, p, grid, cfg, s);
        case 4: return launch_tma_inst<C, R, kDot, 4, false>(e, p, grid, cfg, s);
        case 5: return launch_tma_inst<C, R, kDot, 1, true>(e, p, grid, cfg, s);
        case 6: return launch_tma_inst<C, R, kL2, 1, false>(e, p, grid, cfg, s);
        case 7: return launch_tma_inst<C, R, kL2, 4, false>(e, p, grid, cfg, s);
        default: return launch_tma_inst<C, R, kL2, 1, true>(e, p, grid, cfg, s);
    }
}
static cudaError_t launch_tma(wax_vs_engine *e, const ScanParams &p, int grid, const TmaConfig &cfg, int metric, int mode,
                              cudaStream_t s) {
#define WAXVS_CASE(Cv, Rv) if (cfg.C == Cv && cfg.R == Rv) return launch_tma_cr<Cv, Rv>(e, p, grid, cfg, metric, mode, s)
    WAXVS_CASE(1, 4); WAXVS_CASE(1, 8); WAXVS_CASE(2, 4); WAXVS_CASE(2, 8);
    WAXVS_CASE(3, 4); WAXVS_CASE(3, 8); WAXVS_CASE(4, 4); WAXVS_CASE(4, 8);
    WAXVS_CASE(6, 2); WAXVS_CASE(6, 4); WAXVS_CASE(8, 2); WAXVS_CASE(8, 4);
    WAXVS_CASE(12, 1); WAXVS_CASE(12, 2);
    WAXVS_CASE(0, 1); WAXVS_CASE(0, 2); WAXVS_CASE(0, 4); WAXVS_CASE(0, 8);
#undef WAXVS_CASE
    return cudaErrorInvalidValue;
}
// The nominating pass of the route (SHADOW form, INT8 / U4 for the coded shadows): cosine / dot, k' nominees (E = 4).
// The 4-bit score' does not depend on the metric (cosine rows are pre-scaled in the shadow): one instantiation serves both.
template <RouteForm F, int C, int R>
static cudaError_t launch_route_cr(wax_vs_engine *e, const ScanParams &p, int grid, const TmaConfig &cfg, int metric,
                                   cudaStream_t s) {
    if constexpr (F == kRouteU4) {
        return launch_tma_inst<C, R, kDot, 4, false, true, false, true>(e, p, grid, cfg, s);
    } else {
        return metric == kCosine ? launch_tma_inst<C, R, kCosine, 4, false, true, F == kRouteInt8>(e, p, grid, cfg, s)
                                 : launch_tma_inst<C, R, kDot, 4, false, true, F == kRouteInt8>(e, p, grid, cfg, s);
    }
}
// The (C, R) shapes compiled for each form of the route, listed once: launch_<form>_scan launches the form's scan in the
// shape `cfg`, and with p = nullptr only tells whether that shape is compiled (cudaSuccess; pick_route_config takes a
// rows_per_step option by it).
#define WAXVS_CASE(Cv, Rv) \
    if (cfg.C == Cv && cfg.R == Rv) return p ? launch_route_cr<F, Cv, Rv>(e, *p, grid, cfg, metric, s) : cudaSuccess
static cudaError_t launch_shadow_scan(wax_vs_engine *e, const ScanParams *p, int grid, const TmaConfig &cfg, int metric,
                                      cudaStream_t s) {
    constexpr RouteForm F = kRouteBf16;
    WAXVS_CASE(1, 8); WAXVS_CASE(1, 16); WAXVS_CASE(2, 8); WAXVS_CASE(2, 16);
    WAXVS_CASE(3, 4); WAXVS_CASE(3, 8); WAXVS_CASE(3, 16); WAXVS_CASE(4, 4); WAXVS_CASE(4, 8);
    WAXVS_CASE(6, 2); WAXVS_CASE(6, 4); WAXVS_CASE(8, 2); WAXVS_CASE(8, 4); WAXVS_CASE(12, 2); WAXVS_CASE(12, 4);
    return cudaErrorInvalidValue;
}
static cudaError_t launch_int8_scan(wax_vs_engine *e, const ScanParams *p, int grid, const TmaConfig &cfg, int metric,
                                   cudaStream_t s) {
    constexpr RouteForm F = kRouteInt8;
    WAXVS_CASE(1, 8); WAXVS_CASE(1, 16); WAXVS_CASE(2, 8); WAXVS_CASE(2, 16);
    WAXVS_CASE(3, 4); WAXVS_CASE(3, 8); WAXVS_CASE(3, 16); WAXVS_CASE(4, 4); WAXVS_CASE(4, 8);
    WAXVS_CASE(6, 4); WAXVS_CASE(6, 8); WAXVS_CASE(8, 4); WAXVS_CASE(12, 4);
    return cudaErrorInvalidValue;
}
static cudaError_t launch_u4_scan(wax_vs_engine *e, const ScanParams *p, int grid, const TmaConfig &cfg, int metric,
                                  cudaStream_t s) {
    constexpr RouteForm F = kRouteU4;
    WAXVS_CASE(1, 8); WAXVS_CASE(1, 16); WAXVS_CASE(2, 8); WAXVS_CASE(2, 16); WAXVS_CASE(3, 8); WAXVS_CASE(3, 16);
    WAXVS_CASE(4, 4); WAXVS_CASE(4, 8); WAXVS_CASE(6, 4); WAXVS_CASE(6, 8); WAXVS_CASE(8, 4); WAXVS_CASE(12, 4);
    return cudaErrorInvalidValue;
}
#undef WAXVS_CASE

// What differs between the forms of the single-query route (DESIGN 4.1), by RouteForm.
struct RouteFormSpec {
    const char *name;
    uint32_t bits;            // per element of a shadow row
    bool scaled;              // rows carry a scale (in the scan's stages too), and the shadow a measured bound
    cudaError_t (*launch)(wax_vs_engine *, const ScanParams *, int, const TmaConfig &, int, cudaStream_t);   // its scan
    int default_r[7];         // rows per step without the option, by C of kUnrolledC
    int warps, stages;        // without the options
    bool keep_warps;          // without the warps option the default is kept and a ring that does not fit refused (else
                              // fewer warps until it fits)
    bool grid_rescore;        // nominees: kU4CtaNominees per CTA, re-scored and proven on the whole grid by
                              // shadow_rescore_kernel (else the kShadowNominees x kNomineeStride warp lists of one query,
                              // re-scored and proven by batch_finish_kernel)
    uint32_t tail_bytes;      // per element of the ring, the staging the scan's selection tail may use (the 4-bit form
                              // has no selection tail and keeps the bf16 figure)
    float max_eps_rel;        // the coarsest bound whose nominees the route takes
};
constexpr RouteFormSpec kRouteSpec[kRouteForms] = {
    // bf16: 16 warps, 3 stages of 2-6 KB: on H100 at 10 M x 384 (C = 3) rows 4 / warps 16 / stages 3 took 2.503 ms per
    // query against 2.545 for the fp32 shape's bytes (rows 8 / warps 8 / stages 2), the best of eight shapes alternated
    // in one run (DESIGN 4.1); the other C take the same ring, not measured separately.
    {"bf16", 16, false, launch_shadow_scan, {8, 8, 4, 4, 2, 2, 2}, 16, 3, false, false, 2, kBf16Eps},
    // int8: steps of ~3 KB like the best bf16 shape, 16 warps, 3 stages (DESIGN 4.1)
    {"int8", 8, true, launch_int8_scan, {8, 8, 8, 4, 4, 4, 4}, 16, 3, false, false, 1, kBf16Eps},
    // 4-bit: steps of ~3 KB (16 rows at 384 dims), 16 warps, 3 stages; its bound is coarser than the bf16 one by design,
    // so any finite one is taken
    {"4-bit", 4, true, launch_u4_scan, {16, 16, 16, 8, 8, 4, 4}, 16, 3, true, true, 2, std::numeric_limits<float>::max()},
};

// The nominating scan's shape for a form of the route: the unrolled shapes only, its options or its defaults.
static bool pick_route_config(const wax_vs_engine *e, RouteForm f, TmaConfig *cfg) {
    const RouteFormSpec &fs = kRouteSpec[f];
    const Tuning::Route &t = e->tune.route[f];
    const int ci = unrolled_index(e->dims);
    if (ci < 0) return false;
    const int C = kUnrolledC[ci];
    const bool listed = fs.launch(nullptr, nullptr, 0, TmaConfig{C, t.rows_per_step, 0, 0, 0}, 0, nullptr) == cudaSuccess;
    const int R = listed ? t.rows_per_step : fs.default_r[ci];
    const int stages = t.stages > 0 ? t.stages : fs.stages;
    const size_t stage_bytes = static_cast<size_t>(R) * (e->dims * fs.bits / 8 + (fs.scaled ? sizeof(float) : 0));
    const size_t budget = tma_smem_budget(e);
    int warps = std::max(1, std::min(16, t.warps ? t.warps : fs.warps));
    if (!t.warps && !fs.keep_warps) while (warps > 2 && tma_ring_smem(warps, stages, stage_bytes) > budget) --warps;
    const size_t smem = tma_ring_smem(warps, stages, stage_bytes);
    if (smem > budget) return false;
    *cfg = TmaConfig{C, R, warps, stages, smem};
    return true;
}

static cudaError_t launch_ldg(const ScanParams &p, int grid, int metric, int mode, cudaStream_t s) {
    switch (metric * 3 + mode) {
        case 0: scan_ldg_kernel<kCosine, 1, false><<<grid, 256, 0, s>>>(p); break;
        case 1: scan_ldg_kernel<kCosine, 4, false><<<grid, 256, 0, s>>>(p); break;
        case 2: scan_ldg_kernel<kCosine, 1, true><<<grid, 256, 0, s>>>(p); break;
        case 3: scan_ldg_kernel<kDot, 1, false><<<grid, 256, 0, s>>>(p); break;
        case 4: scan_ldg_kernel<kDot, 4, false><<<grid, 256, 0, s>>>(p); break;
        case 5: scan_ldg_kernel<kDot, 1, true><<<grid, 256, 0, s>>>(p); break;
        case 6: scan_ldg_kernel<kL2, 1, false><<<grid, 256, 0, s>>>(p); break;
        case 7: scan_ldg_kernel<kL2, 4, false><<<grid, 256, 0, s>>>(p); break;
        default: scan_ldg_kernel<kL2, 1, true><<<grid, 256, 0, s>>>(p); break;
    }
    return cudaGetLastError();
}

// Enqueue one query's scan + top-k on `stream`.  k_eff <= 10000.  Adds the number of kernels launched.
// Wait for a kernel's host-visible completion flag (mapped pinned memory): the result is usable a few microseconds
// after the kernel stored it, without an event / stream synchronisation.  The stream is polled now and then so that a
// launch failure surfaces.  Returns WAX_VS_OK, 1 when the flag carries the error bit, or a negative code.
static int32_t wait_host_flag(cudaStream_t stream, unsigned long long *flag_ptr, unsigned long long seq,
                              unsigned long long timeout_ns) {
    volatile unsigned long long *flag = flag_ptr;
    const auto t0 = std::chrono::steady_clock::now();
    uint32_t spins = 0;
    for (;;) {
        const unsigned long long v = *flag;
        if ((v & ~kShardErrorBit) == seq) {
            std::atomic_thread_fence(std::memory_order_acquire);
            return (v & kShardErrorBit) ? 1 : WAX_VS_OK;
        }
        if ((++spins & 0x3FFu) == 0) {
            const cudaError_t q = cudaStreamQuery(stream);
            if (q != cudaSuccess && q != cudaErrorNotReady)
                return fail(WAX_VS_ERR_CUDA, "search failed on the device: %s", cudaGetErrorString(q));
            if (q == cudaSuccess && ((*flag) & ~kShardErrorBit) != seq)
                return fail(WAX_VS_ERR_CUDA, "search finished without publishing its result");
            if (std::chrono::steady_clock::now() - t0 > std::chrono::nanoseconds(timeout_ns) + std::chrono::seconds(5))
                return fail(WAX_VS_ERR_CUDA, "search did not complete");
        }
    }
}

// n host queries -> pinned staging (c->h_queries) -> c->d_queries, on `stream`; order (optional): staged query j is
// queries[order[j]]
static int32_t stage_queries(wax_vs_engine *e, SearchCtx *c, const float *queries, uint32_t n, cudaStream_t stream,
                             const uint32_t *order = nullptr) {
    const size_t qfloats = static_cast<size_t>(n) * e->dims;
    int32_t rc = c->d_queries.ensure(qfloats, "query buffer");
    if (!rc) rc = c->h_queries.ensure(qfloats, "query staging");
    if (rc) return rc;
    if (order) {
        for (uint32_t j = 0; j < n; ++j)
            memcpy(c->h_queries + static_cast<size_t>(j) * e->dims, queries + static_cast<size_t>(order[j]) * e->dims,
                   e->dims * sizeof(float));
    } else {
        memcpy(c->h_queries, queries, qfloats * sizeof(float));
    }
    CUDA_TRY(cudaMemcpyAsync(c->d_queries, c->h_queries, qfloats * sizeof(float), cudaMemcpyHostToDevice, stream));
    return WAX_VS_OK;
}

// Host delivery (the synchronous host entry points, fused top-k only): h_query travels in the kernel parameters when the
// kernel can take it (else it is copied H2D here), and the kernel stores the result into host_out + raises host_flag.
struct HostDelivery {
    const float *h_query;               // host query (dims floats); d_query is ignored when set
    wax_vs_candidate *host_out;         // mapped pinned [k], or nullptr
    unsigned long long *host_flag;      // mapped pinned
    unsigned long long seq;
    bool delivered = false;             // out: the launched kernel will raise host_flag (else: copy d_out back yourself)
};

// Exact radix select (waxvs_select.cuh) of the k smallest (key << 32 | row) over a row-indexed key array of n entries
// (WAXVS_UKEY_NONE = absent); p.k = k candidates go to p.out, best first, padding valid = 0.
static int32_t enqueue_select(wax_vs_engine *e, SearchCtx *c, const uint32_t *keys, uint32_t n, uint32_t k,
                              const ScanParams &p, cudaStream_t stream, uint64_t *launches) {
    int32_t rc = c->d_select.ensure(1, "selection state");
    if (!rc) rc = c->d_sel_keys.ensure(16384, "selected keys");
    if (rc) return rc;
    const int sgrid = std::max(1, std::min<int>(e->sm_count * 4, static_cast<int>((n + 511) / 512)));
    select_init_kernel<<<1, 256, 0, stream>>>(c->d_select, k);
    for (int pass = 0; pass < kSelectPasses; ++pass) {
        select_hist_kernel<<<sgrid, 512, 0, stream>>>(keys, n, c->d_select, pass);
        select_scan_kernel<<<1, 1024, 0, stream>>>(c->d_select, pass);
    }
    select_compact_kernel<<<sgrid, 512, 0, stream>>>(keys, n, c->d_select, c->d_sel_keys, 16384);
    uint32_t pow2 = 64;
    while (pow2 < k) pow2 <<= 1;
    CUDA_TRY(grant_smem(e, select_sort_kernel, pow2 * sizeof(uint64_t)));
    select_sort_kernel<<<1, 1024, pow2 * sizeof(uint64_t), stream>>>(c->d_select, c->d_sel_keys, pow2, p);
    CUDA_TRY(cudaGetLastError());
    *launches += 3 + 2 * kSelectPasses;
    return WAX_VS_OK;
}

// Persistent grid of a TMA-staged scan over n_rows rows in the shape `cfg`; sets the ring depth and (auto) the dynamic
// chunk size in p.
static int tma_grid(const wax_vs_engine *e, const SearchCtx *c, const TmaConfig &cfg, ScanParams &p) {
    p.stages = static_cast<uint32_t>(cfg.stages);
    const uint64_t steps = (e->n_rows + cfg.R - 1) / cfg.R;
    const int max_grid = e->tune.grid > 0 ? e->tune.grid : e->sm_count;
    int grid = static_cast<int>(std::min<uint64_t>(max_grid, (steps + cfg.warps - 1) / cfg.warps));
    grid = std::max(std::min(grid, static_cast<int>(c->d_block_keys.cap / 128)), 1);
    if (e->tune.chunk_steps < 0)     // auto: about two claims per warp at least, at most 8 steps
        p.chunk_steps = static_cast<uint32_t>(std::max<uint64_t>(1, std::min<uint64_t>(8, steps / (static_cast<uint64_t>(grid) * cfg.warps * 2))));
    return grid;
}

static bool batch_bf16_wanted(const wax_vs_engine *e);
static int32_t ensure_shadow(wax_vs_engine *e, cudaStream_t stream);
static int32_t ensure_coded_shadow(wax_vs_engine *e, RouteForm f, cudaStream_t stream, bool keep_coarse);
// The shadow of form f, brought up to date when it fits (keep_coarse: see ensure_coded_shadow).
static int32_t ensure_route_shadow(wax_vs_engine *e, RouteForm f, cudaStream_t stream, bool keep_coarse = false) {
    return f == kRouteBf16 ? ensure_shadow(e, stream) : ensure_coded_shadow(e, f, stream, keep_coarse);
}

// ---- the shadow route of a single query (DESIGN 4.1) ----
// The fp32 scan reads dims * 4 bytes per row and runs at the HBM read ceiling; a shadow holds the same rows in fewer
// bytes (bf16, int8 or 4-bit).  Three launches on `stream`, no host round trip: the form's nominating scan picks the best
// rows by score', a re-score (the batched path's finish kernel, one query, one slice; the 4-bit form: a grid-wide one)
// re-scores them exactly in the scan's own order and proves that no other row can beat or tie the k-th (DESIGN 4.5), and
// `p` -- the query's fp32 scan, launched next by the caller -- is guarded by that proof: it returns at entry when the
// proof held, else it answers the query as it always does.
constexpr uint32_t kShadowNominees = 128;     // k': every warp list of the SHADOW and INT8 forms holds this many
constexpr uint32_t kShadowRescore = 256;
constexpr uint32_t kShadowSkipQueries = 16;   // after a failed proof: eligible queries that take the fp32 scan directly
// Nothing is enqueued (and p stays unguarded) when the route does not apply to this engine and query; the caller has
// already checked the rest: one unsharded fused query with k <= 32 on an unrolled TMA shape.
// (batch_bf16 and dims % 64 == 0 as for the bf16 nominations, but not whether the bf16 shadow fitted: when it did not,
// the coded forms still run on their own shadows, and the bf16 form finds no shadow and leaves the query to the fp32 scan)
static bool shadow_route_applies(const wax_vs_engine *e) {
    return e->tune.shadow_scan && (e->similarity == WAX_VS_COSINE || e->similarity == WAX_VS_DOT) && !e->debug_trace &&
           e->tune.batch_bf16 != 0 && e->dims % kBatchKBlockBf16 == 0 &&
           e->n_rows * e->dims * sizeof(float) >= e->tune.route[kRouteBf16].min_bytes;
}
// The form the route takes for the next query, from what the engine observes: the first of the 4-bit, int8 and bf16
// forms (each the fastest that proves on some corpus) whose min_bytes the fp32 corpus reaches, whose shape fits (*cfg)
// and whose shadow fits with a bound no coarser than the form's max_eps_rel -- a corpus with outlier dimensions coarsens
// the int8 rows' scales and keeps the bf16 form, which proves for it.  The 4-bit form is skipped while a failed 4-bit
// proof has demoted the route (`demoted`: the caller's reading of u4_demoted).  Call with the route applying; builds the
// shadows it tries (a corpus found too coarse builds none until its rows are rewritten, see ensure_coded_shadow).
// *use = false: no form applies, the fp32 scan answers.
static int32_t select_route_form(wax_vs_engine *e, cudaStream_t stream, bool demoted, bool *use, RouteForm *form,
                                 TmaConfig *cfg) {
    *use = false;
    for (const RouteForm f : {kRouteU4, kRouteInt8, kRouteBf16}) {
        if ((f == kRouteU4 && demoted) || e->n_rows * e->dims * sizeof(float) < e->tune.route[f].min_bytes ||
            !pick_route_config(e, f, cfg))
            continue;
        if (const int32_t rc = ensure_route_shadow(e, f, stream)) return rc;
        if (e->shadows[f].valid && e->shadows[f].eps_rel <= kRouteSpec[f].max_eps_rel) {
            *use = true;
            *form = f;
            return WAX_VS_OK;
        }
    }
    return WAX_VS_OK;
}

// Launches 1 and 2 of the route for the query of `p` (the fp32 scan's parameters: query, filter, k, out, ids) in form f
// and its shape `cfg`, over a valid shadow: the nominating scan writes its keys to c->d_heaps, the re-score writes the
// exact result to p.out and its proof flag to c->d_ok.  shape (optional, the read-outs wax_vs_debug_*_nominations):
// {C, R, warps, stages, grid, chunk_steps, tail_select} of the nominating launch.
static int32_t enqueue_shadow_nominations(wax_vs_engine *e, SearchCtx *c, const ScanParams &p, const TmaConfig &cfg,
                                          cudaStream_t stream, uint64_t *launches, uint32_t *shape, RouteForm f) {
    const RouteFormSpec &fs = kRouteSpec[f];
    const wax_vs_engine::Shadow &sh = e->shadows[f];
    int32_t rc;
    if (fs.grid_rescore && !c->d_u4_aux) {           // the cut word starts at "nothing cut"; every re-score leaves it so
        if ((rc = c->d_u4_aux.ensure(3, "4-bit route state"))) return rc;
        CUDA_TRY(cudaMemsetAsync(c->d_u4_aux, 0xFF, 3 * sizeof(uint32_t), stream));
    }
    // grid_rescore: up to kU4CtaNominees keys per CTA of the grid (tma_grid never exceeds sm_count or the grid option)
    const size_t cta_keys = static_cast<size_t>(std::max(e->tune.grid, e->sm_count)) * kU4CtaNominees;
    if ((rc = c->d_heaps.ensure(std::max(static_cast<size_t>(kShadowNominees) * kNomineeStride, fs.grid_rescore ? cta_keys : 0), "nominee keys")) ||
        (rc = c->d_ok.ensure(1, "proof flags")) || (!p.query && (rc = c->d_queries.ensure(e->dims, "query buffer"))))
        return rc;

    ScanParams sp = p;
    sp.corpus = reinterpret_cast<const float *>(sh.codes.p);
    sp.row_scale = fs.scaled ? sh.scale.p : nullptr;
    sp.u4_aux = fs.grid_rescore ? c->d_u4_aux.p : nullptr;
    sp.k = kShadowNominees;
    sp.out = nullptr; sp.host_out = nullptr; sp.host_flag = nullptr;
    sp.nominees = c->d_heaps;
    sp.query_store = p.query ? nullptr : c->d_queries.p;
    sp.tail_select = e->tune.tail_select ? 1u : 0u;
    sp.tail_smem_bytes = static_cast<uint32_t>(static_cast<size_t>(cfg.warps) * cfg.stages * cfg.R * e->dims * fs.tail_bytes);
    const int grid = tma_grid(e, c, cfg, sp);
    CUDA_TRY(fs.launch(e, &sp, grid, cfg, e->similarity, stream));

    if (fs.grid_rescore) {           // every CTA's nominees, re-scored and proven on the whole grid
        RescoreParams rp{};
        rp.corpus = e->d_corpus; rp.query = p.query ? p.query : c->d_queries.p;
        rp.dims = e->dims; rp.k = p.k; rp.n_nominees = static_cast<uint32_t>(grid) * kU4CtaNominees;
        rp.nominees = c->d_heaps; rp.aux = c->d_u4_aux; rp.max_norm_bits = e->d_max_norm; rp.rho_max = sh.rho_max;
        rp.block_keys = c->d_block_keys; rp.ticket = c->d_ticket; rp.work_counter = sp.work_counter; rp.out = p.out; rp.ok = c->d_ok;
        rp.frame_ids = p.frame_ids; rp.id_base = p.id_base; rp.row_offset = p.row_offset; rp.row_keys = p.row_keys;
        rp.tail_smem_bytes = static_cast<uint32_t>(grid) * p.k * sizeof(uint64_t);      // <= 132 x 32 keys: no opt-in needed
        if (rp.tail_smem_bytes > 48u * 1024u) rp.tail_smem_bytes = 0;                    // (a wider grid reads them from L2)
        const auto kernel = e->similarity == WAX_VS_COSINE ? shadow_rescore_kernel<kCosine> : shadow_rescore_kernel<kDot>;
        kernel<<<grid, 512, rp.tail_smem_bytes, stream>>>(rp);
        CUDA_TRY(cudaGetLastError());
    } else {
        FinishParams fp{};
        fp.corpus = e->d_corpus; fp.queries = p.query ? p.query : c->d_queries.p;
        fp.n_rows = p.n_rows; fp.dims = e->dims; fp.n_queries = 1; fp.groups = 1; fp.slices = 1;
        fp.kprime = kShadowNominees; fp.k = p.k; fp.metric = e->similarity;
        fp.heaps = c->d_heaps; fp.max_norm_bits = e->d_max_norm;
        fp.out = p.out; fp.ok = c->d_ok;
        fp.frame_ids = p.frame_ids; fp.id_base = p.id_base; fp.row_offset = p.row_offset; fp.row_keys = p.row_keys;
        fp.pow2_all = 512; fp.rescore = kShadowRescore; fp.eps_rel = sh.eps_rel;
        const size_t fsmem = static_cast<size_t>(fp.pow2_all + fp.rescore) * sizeof(uint64_t);
        const auto kernel = e->similarity == WAX_VS_COSINE ? batch_finish_kernel<kCosine> : batch_finish_kernel<kDot>;
        CUDA_TRY(grant_smem(e, kernel, fsmem));
        kernel<<<1, 512, fsmem, stream>>>(fp);
        CUDA_TRY(cudaGetLastError());
    }
    *launches += 2;
    if (shape) {
        const uint32_t s[7] = {static_cast<uint32_t>(cfg.C), static_cast<uint32_t>(cfg.R), static_cast<uint32_t>(cfg.warps),
                               static_cast<uint32_t>(cfg.stages), static_cast<uint32_t>(grid), sp.chunk_steps, sp.tail_select};
        std::copy(s, s + 7, shape);
    }
    return WAX_VS_OK;
}

static int32_t enqueue_shadow_route(wax_vs_engine *e, SearchCtx *c, ScanParams &p, cudaStream_t stream, uint64_t *launches) {
    if (!shadow_route_applies(e)) return WAX_VS_OK;
    int32_t rc;
    if (!c->h_proof_count) {
        if ((rc = c->d_proof_count.ensure(2, "proof counts")) || (rc = c->h_proof_count.ensure(2, "proof count mirror"))) return rc;
        CUDA_TRY(cudaMemsetAsync(c->d_proof_count, 0, 2 * sizeof(uint32_t), stream));
        c->h_proof_count[0] = c->h_proof_count[1] = 0;
        c->seen_failed = 0;
    }
    bool demoted;
    {
        std::lock_guard<std::mutex> pg(e->pool_mu);
        const uint32_t failed = *static_cast<volatile uint32_t *>(c->h_proof_count + 1);   // no synchronisation: may lag
        if (failed != c->seen_failed) {
            c->seen_failed = failed;
            if (c->last_u4) {           // a 4-bit proof failed (the fp32 scan answered): the int8 form for a while
                if (e->u4_probing) e->u4_demote_window = std::min(e->u4_demote_window * 2, 1u << 20);
                e->u4_demoted = e->u4_demote_window;
            } else {
                e->shadow_scan_skip = kShadowSkipQueries;
            }
        } else if (c->last_u4 && e->u4_probing) {        // the probe after a demotion held
            e->u4_demote_window = 16;
        }
        if (c->last_u4) e->u4_probing = false;
        c->last_u4 = false;
        if (e->shadow_scan_skip > 0) { --e->shadow_scan_skip; return WAX_VS_OK; }
        demoted = e->u4_demoted > 0;
        if (demoted && --e->u4_demoted == 0) e->u4_probing = true;
    }
    bool use = false;
    RouteForm form = kRouteBf16;
    TmaConfig cfg{};
    if ((rc = select_route_form(e, stream, demoted, &use, &form, &cfg)) || !use) return rc;
    if ((rc = enqueue_shadow_nominations(e, c, p, cfg, stream, launches, nullptr, form))) return rc;
    c->last_u4 = form == kRouteU4;
    {
        std::lock_guard<std::mutex> pg(e->pool_mu);
        ++e->single_route_queries[form];
    }
    p.proof_ok = c->d_ok;
    p.proof_count = c->d_proof_count;
    p.proof_count_host = c->h_proof_count;
    return WAX_VS_OK;
}

// The scan parameters of one query (`d_query` on the device, or nullptr when place_host_query sets it); the caller sets
// the tail, the delivery and the shard exchange.  Auto chunk_steps (0 here) is set by tma_grid.
static ScanParams scan_params(const wax_vs_engine *e, SearchCtx *c, const float *d_query, uint32_t k_eff, uint64_t row_offset,
                              wax_vs_candidate *d_out, const uint64_t *d_ids, const uint32_t *d_mask) {
    ScanParams p{};
    p.corpus = e->d_corpus; p.query = d_query;
    p.n_rows = static_cast<uint32_t>(e->n_rows); p.dims = e->dims; p.k = k_eff;
    p.block_keys = c->d_block_keys; p.ticket = c->d_ticket; p.out = d_out;
    p.frame_ids = d_ids; p.id_base = e->id_base; p.row_offset = row_offset; p.row_keys = c->row_keys;
    p.use_l2_hint = e->tune.l2_hint ? 1u : 0u;
    p.chunk_steps = e->tune.chunk_steps > 0 ? static_cast<uint32_t>(e->tune.chunk_steps) : 0u;
    p.work_counter = c->d_ticket + 1;
    p.mask = d_mask;
    p.trace = e->debug_trace;
    return p;
}

// A host query: in the kernel parameters when the kernel can take it (inline_ok: a fused TMA-staged scan), else copied
// to c->d_queries on `stream`.
static int32_t place_host_query(wax_vs_engine *e, SearchCtx *c, ScanParams &p, const float *h_query, bool inline_ok,
                                cudaStream_t stream) {
    if (inline_ok && e->tune.inline_query != 0 && e->dims <= static_cast<uint32_t>(kInlineQueryFloats)) {
        memcpy(p.query_inline, h_query, e->dims * sizeof(float));
        p.query = nullptr;
        return WAX_VS_OK;
    }
    int32_t rc = stage_queries(e, c, h_query, 1, stream);
    if (rc) return rc;
    p.query = c->d_queries;
    return WAX_VS_OK;
}

// The stand-alone exchange of this rank's `local` list of k candidates (sorted, padding last), merged into sp.final_out.
static int32_t enqueue_exchange(const ShardParams &sp, const wax_vs_candidate *local, uint32_t k, cudaStream_t stream,
                                uint64_t *launches) {
    shard_exchange_kernel<<<1, 256, 0, stream>>>(sp, local, k);
    CUDA_TRY(cudaGetLastError());
    ++*launches;
    return WAX_VS_OK;
}

// `shard` (optional): the row-sharded form -- d_out receives the result MERGED over all ranks; the exchange runs inside
// the scan launch when the kernel's shared-memory lists can hold the merge keys, else as one extra 1-CTA launch.
// keys_only: run the emitting scan alone -- c->d_dist_keys receives every row's distance key (the masked rows'
// WAXVS_UKEY_NONE) and the caller does its own selection (grouped search); d_out and k_eff are not used.
// shadow_route: the query may take the bf16-shadow route when it applies (enqueue_shadow_route) -- the single-query entry
// points; the batched levels' exact fall-backs (queries a bf16 proof already refused) and the sharded search do not.
static int32_t enqueue_search(wax_vs_engine *e, SearchCtx *c, const float *d_query, uint32_t k_eff,
                              uint64_t row_offset, wax_vs_candidate *d_out, const uint64_t *d_ids,
                              cudaStream_t stream, uint64_t *launches, const uint32_t *d_mask = nullptr,
                              const ShardParams *shard = nullptr, const HostDelivery *host = nullptr,
                              bool keys_only = false, bool shadow_route = false) {
    wax_vs_candidate *d_merged = nullptr;
    if (shard) {
        if (k_eff > static_cast<uint32_t>(kShardKCap))
            return fail(WAX_VS_ERR_UNSUPPORTED, "sharded search supports top_k <= %d (got %u)", kShardKCap, k_eff);
        int32_t rc = c->d_shard_local.ensure(kShardKCap, "shard candidates");
        if (rc) return rc;
        d_merged = d_out;
        d_out = c->d_shard_local;           // the scan produces the LOCAL list; the exchange writes d_merged
    }
    auto exchange_standalone = [&]() -> int32_t {
        ShardParams sp = *shard;
        sp.final_out = d_merged;
        return enqueue_exchange(sp, d_out, k_eff, stream, launches);
    };
    if (e->n_rows == 0) {
        CUDA_TRY(cudaMemsetAsync(d_out, 0, static_cast<size_t>(k_eff) * sizeof(wax_vs_candidate), stream));
        return shard ? exchange_standalone() : WAX_VS_OK;
    }
    ScanParams p = scan_params(e, c, d_query, k_eff, row_offset, d_out, d_ids, d_mask);
    const bool emit = keys_only || k_eff > static_cast<uint32_t>(e->tune.fused_k_max);
    const int mode = emit ? 2 : (k_eff <= 32 ? 0 : 1);
    if (emit) {
        int32_t rc = c->d_dist_keys.ensure(static_cast<size_t>(e->n_rows), "distance keys");
        if (rc) return rc;
        p.dist_keys = c->d_dist_keys;
    }

    TmaConfig cfg{};
    bool use_tma = (e->tune.variant != 2) && pick_tma_config(e, &cfg, mode);
    if (e->tune.variant == 1 && !use_tma)
        return fail(WAX_VS_ERR_UNSUPPORTED, "TMA-staged kernel does not support dims=%u", e->dims);
    if (host && host->h_query) {
        int32_t rc = place_host_query(e, c, p, host->h_query, use_tma && !emit, stream);
        if (rc) return rc;
    }
    if (host && host->host_out && !emit && !shard) {
        p.host_out = host->host_out; p.host_flag = host->host_flag; p.host_seq = host->seq;
        const_cast<HostDelivery *>(host)->delivered = true;
    }
    if (use_tma && !emit && e->tune.tail_select) {   // selection tail: the idle ring is its staging area
        p.tail_select = 1u;
        p.tail_smem_bytes = static_cast<uint32_t>(static_cast<size_t>(cfg.warps) * cfg.stages * cfg.R * e->dims * sizeof(float));
    }
    bool fused_exchange = false;
    if (shard && !emit) {     // the merge keys (world * k uint32) live in the kernel's block-list shared memory
        const size_t list_bytes = p.tail_select ? p.tail_smem_bytes
                                                : static_cast<size_t>(use_tma ? cfg.warps : 8) * 32 * (mode == 0 ? 1 : 4) * sizeof(uint64_t);
        fused_exchange = e->tune.shard_fused != 0 && static_cast<size_t>(shard->world) * k_eff * sizeof(uint32_t) <= list_bytes;
        if (fused_exchange) { p.shard = *shard; p.shard.final_out = d_merged; }
    }
    if (shadow_route && !shard && mode == 0 && use_tma && cfg.C > 0) {
        int32_t rc = enqueue_shadow_route(e, c, p, stream, launches);
        if (rc) return rc;
    }
    int grid;
    const int grid_cap = static_cast<int>(c->d_block_keys.cap / 128);
    if (use_tma) {
        grid = tma_grid(e, c, cfg, p);
        CUDA_TRY(launch_tma(e, p, grid, cfg, e->similarity, mode, stream));
    } else {
        const int max_grid = e->tune.grid > 0 ? e->tune.grid : e->sm_count * e->tune.ldg_ctas_per_sm;
        grid = static_cast<int>(std::min<uint64_t>(max_grid, (e->n_rows + 7) / 8));
        grid = std::max(std::min(grid, grid_cap), 1);
        CUDA_TRY(launch_ldg(p, grid, e->similarity, mode, stream));
    }
    ++*launches;
    {   // the form just launched, for wax_vs_debug_last_scan (the tail test is finish_topk_select's own)
        const bool staged = static_cast<size_t>(grid) * k_eff * sizeof(uint64_t) <= p.tail_smem_bytes;
        const uint32_t form[10] = {use_tma ? 1u : 2u, use_tma ? static_cast<uint32_t>(cfg.C) : 0u,
                                   use_tma ? static_cast<uint32_t>(cfg.R) : 1u, use_tma ? static_cast<uint32_t>(cfg.warps) : 8u,
                                   use_tma ? static_cast<uint32_t>(cfg.stages) : 0u, static_cast<uint32_t>(grid),
                                   use_tma && !emit ? p.chunk_steps : 0u, static_cast<uint32_t>(mode),
                                   p.tail_select ? (staged ? 1u : 2u) : 0u, p.query == nullptr ? 1u : 0u};
        std::lock_guard<std::mutex> pg(e->pool_mu);
        memcpy(e->last_scan, form, sizeof form);
    }

    if (emit && !keys_only) {
        int32_t rc = enqueue_select(e, c, c->d_dist_keys, static_cast<uint32_t>(e->n_rows), k_eff, p, stream, launches);
        if (rc) return rc;
    }
    if (shard && !fused_exchange) return exchange_standalone();
    return WAX_VS_OK;
}

// ---------------------------------------------------------------------------------------------------------
// batched path: wgmma TF32 / bf16 nomination + exact re-score (waxvs_batch.cuh)
static PFN_cuTensorMapEncodeTiled_v12000 tensor_map_encoder() {
    static PFN_cuTensorMapEncodeTiled_v12000 fn = nullptr;
    static std::once_flag once;
    std::call_once(once, [] {
        void *ptr = nullptr;
        cudaDriverEntryPointQueryResult q;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &ptr, cudaEnableDefault, &q) == cudaSuccess &&
            q == cudaDriverEntryPointSuccess)
            fn = reinterpret_cast<PFN_cuTensorMapEncodeTiled_v12000>(ptr);
    });
    return fn;
}

// Row-major [rows][dims] matrix (fp32, or bf16 for the shadow path), box = box_rows x 128 bytes (32 floats / 64 bf16),
// 128-byte swizzle, OOB -> zeros.
static int32_t make_tensor_map(CUtensorMap *map, const void *base, uint64_t rows, uint32_t dims, uint32_t box_rows,
                               bool bf16 = false) {
    auto enc = tensor_map_encoder();
    if (!enc) return fail(WAX_VS_ERR_CUDA, "cuTensorMapEncodeTiled is not available from this driver");
    const size_t esize = bf16 ? sizeof(__nv_bfloat16) : sizeof(float);
    const cuuint64_t gdim[2] = {dims, rows};
    const cuuint64_t gstride[1] = {static_cast<cuuint64_t>(dims) * esize};
    const cuuint32_t box[2] = {static_cast<cuuint32_t>(bf16 ? kBatchKBlockBf16 : kBatchKBlock), box_rows};
    const cuuint32_t estr[2] = {1, 1};
    const CUresult r = enc(map, bf16 ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2,
                           const_cast<void *>(base), gdim, gstride, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                           CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) return fail(WAX_VS_ERR_CUDA, "cuTensorMapEncodeTiled failed (CUresult %d)", static_cast<int>(r));
    return WAX_VS_OK;
}

static bool batch_bf16_wanted(const wax_vs_engine *e);
static bool batch_tensor_eligible(const wax_vs_engine *e, uint32_t n_queries, uint32_t k_eff) {
    const uint32_t min_batch = (e->tune.single_shadow && batch_bf16_wanted(e)) ? 1u : static_cast<uint32_t>(std::max(e->tune.batch_min, 1));
    return e->tune.batch_tensor && n_queries >= min_batch &&
           (e->similarity == WAX_VS_COSINE || e->similarity == WAX_VS_DOT || (e->similarity == WAX_VS_L2 && e->tune.batch_l2)) &&
           e->dims % kBatchKBlock == 0 &&
           e->dims <= 8192 &&        // the proof's accumulation slack (dims * 2^-23) stays below the operand bound
           k_eff >= 1 && e->n_rows >= 1 &&
           // 128 < k <= 1024 (the production candidate limit reaches 1 000, UnifiedSearch.swift:1195-1200): real batches
           // only.  Level 1 can rarely PROVE such a k (64 nominees per slice barely cover it) but its exactly re-scored
           // nominees give the filter level its threshold, and that level is complete by construction.
           (k_eff <= 128 || (k_eff <= static_cast<uint32_t>(kBatchRescoreMax) && e->tune.batch_large_k &&
                             n_queries >= static_cast<uint32_t>(std::max(e->tune.batch_min, 4)) &&
                             e->n_rows >= 64ull * k_eff));   // smaller corpora: too few row slices to nominate k rows
}

// 1/|v| per row + max |v| (l2 engines: and |v|^2 / 2 per row, in the same pass), cached per corpus version.  Appends only
// extend the cache (rows [norms_rows, n_rows) are computed, the running max only grows); anything that moves or
// overwrites rows resets norms_rows to 0.
static int32_t ensure_norms_locked(wax_vs_engine *e, cudaStream_t stream) {
    const bool l2 = e->similarity == WAX_VS_L2;
    if (e->norms_rows == e->n_rows && e->d_inv_norm && (!l2 || e->d_half_sq)) return WAX_VS_OK;
    if (static_cast<size_t>(e->n_rows) > e->d_inv_norm.cap || !e->d_inv_norm ||
        (l2 && (static_cast<size_t>(e->n_rows) > e->d_half_sq.cap || !e->d_half_sq))) {
        e->norms_rows = 0;                                       // ensure re-allocates: the cached prefix is gone
        const size_t want = static_cast<size_t>(std::max<uint64_t>(e->cap_rows, std::max<uint64_t>(e->n_rows, 1)));
        int32_t rc = e->d_inv_norm.ensure(want, "row norms");
        if (!rc && l2) rc = e->d_half_sq.ensure(want, "row half squared norms");
        if (rc) return rc;
    }
    if (!e->d_max_norm) {
        int32_t rc = e->d_max_norm.ensure(1, "max row norm");
        if (rc) return rc;
        e->norms_rows = 0;
    }
    if (e->norms_rows > e->n_rows) e->norms_rows = 0;
    if (e->norms_rows == 0) CUDA_TRY(cudaMemsetAsync(e->d_max_norm, 0, sizeof(uint32_t), stream));
    const uint64_t first = e->norms_rows, count = e->n_rows - first;
    if (count) {
        const int grid = static_cast<int>(std::min<uint64_t>(static_cast<uint64_t>(e->sm_count) * 8, (count + 7) / 8));
        if (l2)
            row_norms_kernel<true><<<std::max(grid, 1), 256, 0, stream>>>(e->d_corpus + first * e->dims, static_cast<uint32_t>(count),
                                                                          e->dims, e->d_inv_norm + first, e->d_max_norm,
                                                                          e->d_half_sq + first);
        else
            row_norms_kernel<<<std::max(grid, 1), 256, 0, stream>>>(e->d_corpus + first * e->dims, static_cast<uint32_t>(count), e->dims,
                                                                    e->d_inv_norm + first, e->d_max_norm);
        CUDA_TRY(cudaGetLastError());
    }
    CUDA_TRY(cudaStreamSynchronize(stream));
    e->norms_rows = e->n_rows;
    return WAX_VS_OK;
}
static int32_t ensure_norms(wax_vs_engine *e, cudaStream_t stream) {
    std::lock_guard<std::mutex> g(e->norms_mu);
    return ensure_norms_locked(e, stream);
}

// The bf16 nominations want dims % 64 == 0 (whole 128-byte k-blocks of bf16).
static bool batch_bf16_wanted(const wax_vs_engine *e) {
    return e->tune.batch_bf16 != 0 && e->dims % kBatchKBlockBf16 == 0 && !e->shadows[kRouteBf16].unavailable;
}

// 32-bit words per row of the form-f shadow, one scale per row padded to whole scan steps (R <= 16), and the bytes of
// `rows` rows.
static size_t shadow_words(const wax_vs_engine *e, RouteForm f) { return e->dims * kRouteSpec[f].bits / 32; }
static size_t shadow_scale_entries(uint64_t rows) { return static_cast<size_t>((rows + 15) / 16 * 16); }
static size_t shadow_bytes(const wax_vs_engine *e, RouteForm f, uint64_t rows) {
    return rows * shadow_words(e, f) * sizeof(uint32_t) + (kRouteSpec[f].scaled ? shadow_scale_entries(rows) * sizeof(float) : 0);
}
// Room in the form-f shadow for the live rows (what it held is given back when it is too small).  Sized for the corpus
// CAPACITY so that appends extend it in place; if only the live rows fit, that.  It must leave max(2 GiB, 10 % of the
// device) free for scratch and growth, and a coded shadow also what the bf16 shadow will take (see ensure_coded_shadow).
// Allocated by hand, not through ensure(): running out here is not an error and sets no last error; the shadow is
// marked unavailable instead.
static int32_t alloc_shadow(wax_vs_engine *e, RouteForm f, cudaStream_t stream) {
    wax_vs_engine::Shadow &sh = e->shadows[f];
    const bool scaled = kRouteSpec[f].scaled;
    const size_t words = shadow_words(e, f);
    const uint64_t need = e->n_rows, pref = std::max<uint64_t>(e->cap_rows, e->n_rows);
    if (sh.codes.cap >= need * words && (!scaled || sh.scale.cap >= shadow_scale_entries(need))) return WAX_VS_OK;
    sh.release();
    size_t free_b = 0, total_b = 0;
    const bool info = cudaMemGetInfo(&free_b, &total_b) == cudaSuccess;
    const size_t headroom = std::max<size_t>(size_t(2) << 30, total_b / 10);
    size_t reserve = 0;                    // the bf16 shadow's allocation to come
    if (f != kRouteBf16 && batch_bf16_wanted(e) && e->shadows[kRouteBf16].codes.cap < need * shadow_words(e, kRouteBf16)) {
        const size_t b_need = shadow_bytes(e, kRouteBf16, need), b_pref = shadow_bytes(e, kRouteBf16, pref);
        reserve = free_b >= b_pref + headroom ? b_pref : (free_b >= b_need + headroom ? b_need : 0);
    }
    uint64_t want = pref;
    if (info && free_b < shadow_bytes(e, f, want) + reserve + headroom) want = need;
    if (!info || free_b < shadow_bytes(e, f, want) + reserve + headroom ||
        cudaMalloc(&sh.codes.p, want * words * sizeof(uint32_t)) != cudaSuccess ||
        (scaled && cudaMalloc(&sh.scale.p, shadow_scale_entries(want) * sizeof(float)) != cudaSuccess)) {
        cudaGetLastError();
        sh.release();
        sh.unavailable = true;             // stays off until its option is set again (bf16: batch_bf16)
        return WAX_VS_OK;
    }
    sh.codes.cap = want * words;
    if (scaled) {
        sh.scale.cap = shadow_scale_entries(want);
        CUDA_TRY(cudaMemsetAsync(sh.scale, 0, sh.scale.cap * sizeof(float), stream));   // the step padding
    }
    return WAX_VS_OK;
}

// bf16 shadow of the corpus (cosine: rows pre-scaled by 1/|v|), cached per corpus version and extended incrementally
// by appends like the norms.  Returns WAX_VS_OK with valid == false when the extra dims*2 bytes per row do not fit in
// HBM (the caller then nominates in TF32 from the fp32 corpus; counter "shadow_unavailable").
static int32_t ensure_shadow(wax_vs_engine *e, cudaStream_t stream) {
    std::lock_guard<std::mutex> g(e->norms_mu);
    wax_vs_engine::Shadow &sh = e->shadows[kRouteBf16];
    if ((sh.valid && sh.rows == e->n_rows) || sh.unavailable) return WAX_VS_OK;
    int32_t rc = ensure_norms_locked(e, stream);
    if (rc || (rc = alloc_shadow(e, kRouteBf16, stream)) || sh.unavailable) return rc;
    if (sh.rows > e->n_rows) sh.rows = 0;
    const uint64_t first = sh.rows, count = e->n_rows - first;
    if (count) {
        const int grid = static_cast<int>(std::min<uint64_t>(static_cast<uint64_t>(e->sm_count) * 16, (count * (e->dims / 4) + 255) / 256));
        shadow_bf16_kernel<<<std::max(grid, 1), 256, 0, stream>>>(e->d_corpus + first * e->dims,
                                                                  e->similarity == WAX_VS_COSINE ? e->d_inv_norm + first : nullptr,
                                                                  count, e->dims,
                                                                  reinterpret_cast<__nv_bfloat16 *>(sh.codes.p) + first * e->dims);
        CUDA_TRY(cudaGetLastError());
    }
    CUDA_TRY(cudaStreamSynchronize(stream));
    sh.rows = e->n_rows;
    sh.valid = true;
    sh.eps_rel = kBf16Eps;                 // the bound the finish proves bf16 nominees with
    return WAX_VS_OK;
}

// int8 (f = kRouteInt8, shadow_int8_kernel) or 4-bit (kRouteU4, shadow_u4_kernel) shadow of the corpus for the
// single-query route (cosine rows pre-scaled by 1/|v| as in the bf16 shadow): built lazily, extended by appends (which can
// only raise rho_max), kept over a remove's untouched prefix, rebuilt after overwrites.  Returns WAX_VS_OK with
// valid == false when it does not fit (the route then takes another form; counter "int8_shadow_bytes" /
// "u4_shadow_bytes" = 0).  The build synchronises `stream` and reads rho_max and max|v| back: eps_rel = rho_max / M
// rounded up (M = 1 for cosine, whose rows are pre-scaled, and max|v| for dot), so that the finish's eps_rel * |q| * M
// is at least |q| rho_max.
// Memory: the bf16 shadow comes first.  Unless it already holds the live rows (or was refused), a coded shadow reserves
// what ensure_shadow would allocate next to the same free memory -- its capacity size when that fits the headroom rule,
// else the live rows -- so that it never leaves the bf16 shadow, and with it the route's bf16 form and the batched bf16
// nominations, less room than they would have without it.
// A corpus whose bound is too coarse for the route (above the form's max_eps_rel: for int8, outlier dimensions; the
// 4-bit bound is coarser than the bf16 one by design, so only a non-finite one) gives its shadow back right after the
// build and builds none again (coarse) until its rows are rewritten: appends can only raise rho_max.  keep_coarse (the
// read-outs) keeps such a shadow; the route never uses it.
static int32_t ensure_coded_shadow(wax_vs_engine *e, RouteForm f, cudaStream_t stream, bool keep_coarse) {
    std::lock_guard<std::mutex> g(e->norms_mu);
    wax_vs_engine::Shadow &cs = e->shadows[f];
    if ((cs.valid && cs.rows == e->n_rows) || cs.unavailable || (cs.coarse && !keep_coarse))
        return WAX_VS_OK;
    int32_t rc = ensure_norms_locked(e, stream);
    if (rc) return rc;
    if ((rc = cs.rho.ensure(1, "coded shadow bound"))) return rc;
    if ((rc = alloc_shadow(e, f, stream)) || cs.unavailable) return rc;
    const size_t words = shadow_words(e, f);
    if (cs.rows > e->n_rows) cs.rows = 0;
    if (cs.rows == 0) CUDA_TRY(cudaMemsetAsync(cs.rho, 0, sizeof(uint32_t), stream));
    const uint64_t first = cs.rows, count = e->n_rows - first;
    if (count) {
        const int grid = static_cast<int>(std::min<uint64_t>(static_cast<uint64_t>(e->sm_count) * 8, (count + 7) / 8));
        (f == kRouteU4 ? shadow_u4_kernel : shadow_int8_kernel)<<<std::max(grid, 1), 256, 0, stream>>>(
            e->d_corpus + first * e->dims, e->similarity == WAX_VS_COSINE ? e->d_inv_norm + first : nullptr, count, e->dims,
            cs.codes + first * words, cs.scale + first, cs.rho);
        CUDA_TRY(cudaGetLastError());
    }
    uint32_t bits[2] = {0, 0};
    CUDA_TRY(cudaMemcpyAsync(&bits[0], cs.rho, sizeof(uint32_t), cudaMemcpyDeviceToHost, stream));
    CUDA_TRY(cudaMemcpyAsync(&bits[1], e->d_max_norm, sizeof(uint32_t), cudaMemcpyDeviceToHost, stream));
    CUDA_TRY(cudaStreamSynchronize(stream));
    float rho, m;
    memcpy(&rho, &bits[0], sizeof rho);
    memcpy(&m, &bits[1], sizeof m);
    if (e->similarity == WAX_VS_COSINE) m = 1.0f;
    const float q = rho / m;               // rounded up: one ulp up unless exact
    cs.rho_max = rho;
    // (a non-finite max|v| leaves the finish no finite bound either way: no int8 route then)
    cs.eps_rel = (std::isfinite(q) && std::isfinite(m) && m > 0.0f)
                          ? (static_cast<double>(q) * m >= rho ? q : std::nextafter(q, INFINITY)) : INFINITY;
    cs.rows = e->n_rows;
    cs.valid = true;
    if (cs.eps_rel > kRouteSpec[f].max_eps_rel) {          // too coarse for the route (above)
        cs.coarse = true;
        if (!keep_coarse) {                    // nothing holds it: it was not valid for these rows before this call
            cs.release();
        }
    }
    return WAX_VS_OK;
}

// One launch of the nominate kernel in one form; its opt-in shared memory is granted first.
template <bool BF, bool FI, bool AR, bool PR, bool DUMP, bool L2>
static cudaError_t launch_nominate_inst(wax_vs_engine *e, uint32_t grid, uint32_t smem, cudaStream_t stream,
                                        const CUtensorMap &map_q, const CUtensorMap &map_c, const BatchParams &bp) {
    const auto kernel = batch_nominate_kernel<BF, FI, AR, PR, DUMP, L2>;
    const cudaError_t err = grant_smem(e, kernel, smem);
    if (err != cudaSuccess) return err;
    cudaLaunchConfig_t cfg{};
    cfg.gridDim = dim3(grid); cfg.blockDim = dim3(kBatchThreads); cfg.stream = stream; cfg.dynamicSmemBytes = smem;
    cudaLaunchAttribute attr[1];
    if (PR) {
        attr[0].id = cudaLaunchAttributeClusterDimension;
        attr[0].val.clusterDim.x = 2; attr[0].val.clusterDim.y = 1; attr[0].val.clusterDim.z = 1;
        cfg.attrs = attr; cfg.numAttrs = 1;
    }
    return cudaLaunchKernelEx(&cfg, kernel, map_q, map_c, bp);
}

// The nominate kernel in the form (bf16, filter, resident queries, CTA pair) a pass picked; DUMP: with the score
// read-out (wax_vs_debug_batch_nominations).  These are all the forms there are: the filter level runs neither as CTA
// pairs nor with the read-out, and TF32 queries always stream through the ring.  L2: the same forms with the l2 score.
template <bool DUMP, bool L2>
static cudaError_t launch_nominate_forms(wax_vs_engine *e, bool bf16, bool filter, bool ares, bool pair, uint32_t grid,
                                         uint32_t smem, cudaStream_t stream, const CUtensorMap &map_q,
                                         const CUtensorMap &map_c, const BatchParams &bp) {
#define WAXVS_NOM(BF, FI, AR, PR) return launch_nominate_inst<BF, FI, AR, PR, DUMP, L2>(e, grid, smem, stream, map_q, map_c, bp)
    if constexpr (!DUMP) {
        if (filter) {
            if (!bf16) WAXVS_NOM(false, true, false, false);
            if (ares) WAXVS_NOM(true, true, true, false);
            WAXVS_NOM(true, true, false, false);
        }
    }
    if (!bf16) {
        if (pair) WAXVS_NOM(false, false, false, true);
        WAXVS_NOM(false, false, false, false);
    }
    if (ares) {
        if (pair) WAXVS_NOM(true, false, true, true);
        WAXVS_NOM(true, false, true, false);
    }
    if (pair) WAXVS_NOM(true, false, false, true);
    WAXVS_NOM(true, false, false, false);
#undef WAXVS_NOM
}
template <bool DUMP>
static cudaError_t launch_nominate(wax_vs_engine *e, bool l2, bool bf16, bool filter, bool ares, bool pair, uint32_t grid,
                                   uint32_t smem, cudaStream_t stream, const CUtensorMap &map_q, const CUtensorMap &map_c,
                                   const BatchParams &bp) {
    return l2 ? launch_nominate_forms<DUMP, true>(e, bf16, filter, ares, pair, grid, smem, stream, map_q, map_c, bp)
              : launch_nominate_forms<DUMP, false>(e, bf16, filter, ares, pair, grid, smem, stream, map_q, map_c, bp);
}

// ---- nominee-heap policy (level 1) ----
// P(X >= h) for X ~ Poisson(m): the chance that one row slice holds h or more of a query's "threatening" rows.
static double poisson_tail(double m, int h) {
    double term = std::exp(-m);                      // P(X = 0)
    for (int i = 1; i <= h; ++i) term *= m / i;      // P(X = h)
    double tail = 0.0, t = term;
    for (int i = h + 1; i < h + 200 && t > 1e-300; ++i) { tail += t; t *= m / i; }
    return std::min(1.0, tail + t);
}

// Nominee heap size per (slice, query) = kernel shape, for nq queries over `slices` row slices.  TF32 shapes: 16 entries
// when 16 nominees per slice comfortably cover k (16 * slices >= 8 k), else 64.  bf16 shapes (16 / 24 / 32 / 64): level 1
// can prove a query only if no slice holds `heap` rows scoring within the bf16 bound of the k-th result; with the corpus
// spread over the slices those "threatening" rows (about 2.2 k of them for the bf16 bound on unit-scale embeddings) fall
// ~Poisson(m = 2.2 k / slices) per slice.  ONE unproven query costs its whole batch a second pass, while larger heaps
// cost ring stages (4 / 3 / 3 / 2): the heap that minimises the expected cost is picked, then raised by heap_bump.
static uint32_t pick_heap(wax_vs_engine *e, bool bf16, uint32_t nq, uint32_t slices, uint32_t k_eff) {
    const bool small_heap = e->tune.batch_heap == 16 || (e->tune.batch_heap == 0 && 16u * slices >= 8u * k_eff);
    if (!bf16) return small_heap ? 16u : 64u;
    uint32_t want = static_cast<uint32_t>(std::max(e->tune.batch_heap, 0));
    if (k_eff > 128u && want == 0u) want = 64u;       // large k: level 1 only has to NOMINATE k rows (filter level decides)
    if (want == 16u || want == 24u || want == 32u || want == 64u) return want;
    // expected cost of a batch = the shape's relative time + P(some query of the batch is unproven) x one more
    // pass.  Threatening rows per query: ~2.2 k (cosine, unit rows) / ~2.8 k (dot: the bound scales with the
    // LARGEST row norm).  The relative times of the heap sizes are guesses carried over from B200 (ring depths
    // 4 / 3 / 3 / 2 on H100); they have not been measured on H100.  l2 takes the dot figure: its bound has the same
    // max-norm structure; that figure has not been measured for l2.
    static const uint32_t ladder[4] = {16u, 24u, 32u, 64u};
    static const double rel_time[4] = {1.00, 1.02, 1.10, 1.40};
    const double m = (e->similarity == WAX_VS_COSINE ? 2.2 : 2.8) * k_eff / slices;
    uint32_t bump = 0;
    { std::lock_guard<std::mutex> pg(e->pool_mu); bump = e->heap_bump; }
    double best = 1e30;
    uint32_t pick = 3u;
    for (uint32_t i = 0; i < 4u; ++i) {
        const double p_fail = std::min(1.0, static_cast<double>(nq) * slices * poisson_tail(m, static_cast<int>(ladder[i])));
        if (p_fail >= 1.0 && ladder[i] != 64u) continue;             // hopeless: every batch would pay a second pass
        const double cost = rel_time[i] + 4.0 * p_fail;              // risk-averse: the model can be off
        if (cost < best) { best = cost; pick = i; }
    }
    return ladder[std::min(pick + bump, 3u)];                         // the data overrules the model (below)
}

// After a level-1 batch that nominated from the bf16 shadow with k <= 128 (large k is expected to need the filter
// level).  When more than a quarter of the batch is unproven (tightly clustered neighbours), the next 16 batches
// nominate in TF32.  With the automatic heap size the data has the last word on it: unproven queries -> one size up
// for `heap_backoff` batches; when that time-out ends one size down is probed again, and a failure during the probe
// doubles the time-out.
static void record_level1_outcome(wax_vs_engine *e, uint32_t n_queries, size_t unproven, uint32_t used_heap) {
    std::lock_guard<std::mutex> pg(e->pool_mu);
    if (unproven * 4 > n_queries) e->bf16_skip_batches = 16;
    if (used_heap == 0u || e->tune.batch_heap != 0) return;
    e->last_heap = used_heap;
    if (unproven && used_heap < 64u) {
        if (e->heap_probing) e->heap_backoff = std::min<uint32_t>(e->heap_backoff * 2u, 1u << 16);
        e->heap_bump = std::min<uint32_t>(e->heap_bump + 1u, 3u);
        e->heap_bump_ttl = e->heap_backoff;
    }
    e->heap_probing = false;
    if (!unproven && e->heap_bump > 0 && e->heap_bump_ttl > 0 && --e->heap_bump_ttl == 0) {
        --e->heap_bump;
        e->heap_probing = true;
        e->heap_bump_ttl = e->heap_bump ? e->heap_backoff : 0;
    }
}

// ---- row filters of a batch ----
// Filter f is the bitset bits + f * words (bit set = the row may be returned).  index: each query's filter
// (WAX_VS_NO_FILTER = none), on the device and the same on the host; nullptr = every query uses `bits` (nullptr = none).
struct RowFilter {
    const uint32_t *bits = nullptr;
    uint32_t words = 0;
    const uint32_t *d_index = nullptr, *h_index = nullptr;
    const uint32_t *mask(uint32_t qi) const {
        if (!h_index) return bits;
        return h_index[qi] == WAX_VS_NO_FILTER ? nullptr : bits + static_cast<size_t>(h_index[qi]) * words;
    }
};

// ---- the tensor-core nomination pass of both levels ----
// One launch of a pass: queries [q0, q0 + nq) in `groups` query groups, each over `slices` row slices.
struct NominateChunk {
    uint32_t q0, nq, groups, slices, kprime;
    const float *queries;       // the launch's fp32 queries
    bool ares, pair;
    int stages;
};

// Enqueues one nomination pass over n_queries device queries on `stream`, in launches of at most max_groups query groups,
// and owns what the levels share: the bf16 query conversion, the tensor maps, the ring shape and the common BatchParams.
// The level supplies the heap size (heap(nq, slices) -> kprime), its own BatchParams fields (prepare(chunk, bp)) and
// the launches that follow each nomination launch (finish(chunk)).  pair: CTA pairs when a launch has two query groups
// or more; dump: the score read-out forms.
template <typename Heap, typename Prepare, typename Finish>
static int32_t enqueue_nominate_pass(wax_vs_engine *e, SearchCtx *c, const float *d_queries, uint32_t n_queries, bool bf16,
                                     bool filter, bool pair, bool dump, uint32_t max_groups, const RowFilter &rf,
                                     cudaStream_t stream, uint64_t *launches, Heap heap, Prepare prepare, Finish finish) {
    int32_t rc;
    // bf16 nominations: convert the queries once per call (n_queries x dims, tiny next to the corpus pass)
    if (bf16) {
        const size_t qn = static_cast<size_t>(n_queries) * e->dims;
        if ((rc = c->d_queries_bf16.ensure(qn, "bf16 queries"))) return rc;
        const int g = static_cast<int>(std::min<size_t>((qn / 4 + 255) / 256, static_cast<size_t>(e->sm_count) * 8));
        shadow_bf16_kernel<<<std::max(g, 1), 256, 0, stream>>>(d_queries, nullptr, n_queries, e->dims, c->d_queries_bf16);
        CUDA_TRY(cudaGetLastError());
        ++*launches;
    }
    const uint32_t tiles_total = static_cast<uint32_t>((e->n_rows + kBatchN - 1) / kBatchN);
    const uint32_t num_kb16 = e->dims / kBatchKBlockBf16;
    const bool l2 = e->similarity == WAX_VS_L2;          // the l2 score: the forms subtract the cached |v|^2 / 2
    for (uint32_t q0 = 0; q0 < n_queries; q0 += max_groups * kBatchM) {
        NominateChunk ch{};
        ch.q0 = q0;
        ch.nq = std::min<uint32_t>(n_queries - q0, max_groups * kBatchM);
        ch.queries = d_queries + static_cast<size_t>(q0) * e->dims;
        ch.groups = (ch.nq + kBatchM - 1) / kBatchM;
        // CTA pairs (two query groups, one row slice, each CTA loads half of every corpus tile for both): needs at least
        // two groups; an odd group count is padded with an all-out-of-range group.
        ch.pair = pair && ch.groups >= 2;
        if (ch.pair) ch.groups = (ch.groups + 1u) & ~1u;
        const uint32_t units = ch.pair ? ch.groups / 2u : ch.groups;
        const uint32_t unit_slots = static_cast<uint32_t>(e->sm_count) / (ch.pair ? 2u : 1u);
        ch.slices = std::max<uint32_t>(1, std::min<uint32_t>(unit_slots / units, tiles_total));
        ch.kprime = heap(ch.nq, ch.slices);
        ch.slices = std::max<uint32_t>(1, std::min<uint32_t>(ch.slices, 16384u / ch.kprime));   // union fits the finish sort
        // resident queries (bf16) when a ring of at least two corpus stages still fits beside them
        const int ares_st = (bf16 && e->tune.batch_ares) ? batch_ring_stages(static_cast<int>(ch.kprime), num_kb16) : 0;
        ch.ares = ares_st >= 2;
        ch.stages = ch.ares ? ares_st : batch_ring_stages(static_cast<int>(ch.kprime));
        // bf16: the converted queries against the corpus shadow; TF32: the fp32 queries against the corpus
        const void *qbase = bf16 ? static_cast<const void *>(c->d_queries_bf16 + static_cast<size_t>(q0) * e->dims) : ch.queries;
        const void *cbase = bf16 ? static_cast<const void *>(e->shadows[kRouteBf16].codes.p) : e->d_corpus;
        CUtensorMap map_q, map_c;
        if ((rc = make_tensor_map(&map_q, qbase, ch.nq, e->dims, kBatchM, bf16))) return rc;
        if ((rc = make_tensor_map(&map_c, cbase, e->n_rows, e->dims, ch.pair ? kBatchN / 2 : kBatchN, bf16))) return rc;
        BatchParams bp{};
        bp.n_rows = static_cast<uint32_t>(e->n_rows); bp.dims = e->dims; bp.n_queries = ch.nq; bp.groups = ch.groups;
        bp.slices = ch.slices; bp.tiles_total = tiles_total; bp.kprime = ch.kprime; bp.metric = e->similarity;
        bp.stages = static_cast<uint32_t>(ch.stages);
        // the cosine shadow rows are pre-normalised: no epilogue scaling on the bf16 path
        bp.row_scale = (e->similarity == WAX_VS_COSINE && !bf16) ? e->d_inv_norm.p : nullptr;
        bp.half_sq = l2 ? e->d_half_sq.p : nullptr;
        bp.allow_bits = rf.bits;
        bp.query_filter = rf.d_index ? rf.d_index + ch.q0 : nullptr;     // indexed by the launch's queries
        bp.filter_words = rf.words;
        if ((rc = prepare(ch, bp))) return rc;
        const uint32_t grid = ch.groups * ch.slices;
        const uint32_t smem = batch_smem_bytes(ch.stages, static_cast<int>(ch.kprime), ch.ares ? num_kb16 : 0u);
        const cudaError_t lerr = dump ? launch_nominate<true>(e, l2, bf16, filter, ch.ares, ch.pair, grid, smem, stream, map_q, map_c, bp)
                                      : launch_nominate<false>(e, l2, bf16, filter, ch.ares, ch.pair, grid, smem, stream, map_q, map_c, bp);
        CUDA_TRY(lerr);
        CUDA_TRY(cudaGetLastError());
        ++*launches;
        if ((rc = finish(ch))) return rc;
    }
    return WAX_VS_OK;
}

// Level 1: the tensor-core nomination + exact finish for n_queries device-resident queries.  d_ok[i] = 1 when query i's
// result is proven exact; the caller sends the others to the filter level, then to enqueue_search.  allow_bf16 = false
// forces TF32 nominations (adaptive level choice).  *used_bf16 reports what ran; d_tau_star (optional) receives each
// query's threshold for the filter level.  `dump` (tests only, one launch at most) runs the same shape with the score
// read-out and reports the shape.
struct NominationDump {
    float *d_scores;        // [n_queries][n_rows]
    uint32_t shape[7];      // bf16, ares, pair, stages, kprime, slices, groups
};
static int32_t enqueue_batch_tensor(wax_vs_engine *e, SearchCtx *c, const float *d_queries, uint32_t n_queries,
                                    uint32_t k_eff, uint64_t row_offset, wax_vs_candidate *d_out, uint32_t *d_ok,
                                    const uint64_t *d_ids, cudaStream_t stream, uint64_t *launches,
                                    bool allow_bf16 = true, bool *used_bf16 = nullptr, float *d_tau_star = nullptr,
                                    const RowFilter &rf = RowFilter{}, uint32_t *used_heap = nullptr,
                                    NominationDump *dump = nullptr) {
    int32_t rc = ensure_norms(e, stream);
    if (rc) return rc;
    bool bf16 = allow_bf16 && batch_bf16_wanted(e);
    if (bf16) {
        if ((rc = ensure_shadow(e, stream))) return rc;
        bf16 = e->shadows[kRouteBf16].valid;
    }
    if (used_bf16) *used_bf16 = bf16;
    // k > 128: the union of the slices' 64-entry heaps must hold k nominees with some room (slices >= 1.15 k / 64), so
    // fewer query groups share the SMs and a large batch is split into several launches
    uint32_t max_groups = static_cast<uint32_t>(e->sm_count);
    if (k_eff > 128u) max_groups = std::max<uint32_t>(1u, max_groups / ((k_eff * 115u / 100u + 63u) / 64u));
    if (dump && n_queries > max_groups * kBatchM)
        return fail(WAX_VS_ERR_ARGUMENT, "the nomination read-out covers one launch: at most %u queries", max_groups * kBatchM);
    // how many nominees the finish kernel re-scores exactly: the (rescore+1)-th nominee bounds the rows it skips, and
    // the coarser bf16 bound needs more distance between it and the k-th result (DESIGN 4.5)
    uint32_t rescore = static_cast<uint32_t>(kBatchRescore);
    if (e->tune.batch_rescore > 0) rescore = static_cast<uint32_t>(e->tune.batch_rescore);
    else if (bf16) rescore = k_eff <= 16 ? 256u : (k_eff <= 48 ? 512u : 1024u);
    if (k_eff > 128u) rescore = static_cast<uint32_t>(kBatchRescoreMax);   // the finish kernel writes k re-scored nominees
    rescore = rescore <= 256u ? 256u : (rescore <= 512u ? 512u : static_cast<uint32_t>(kBatchRescoreMax));

    auto heap = [&](uint32_t nq, uint32_t slices) { return pick_heap(e, bf16, nq, slices, k_eff); };
    auto prepare = [&](const NominateChunk &ch, BatchParams &bp) -> int32_t {
        const size_t slots = static_cast<size_t>(ch.groups) * kBatchM;
        int32_t prc = c->d_heaps.ensure(slots * ch.slices * ch.kprime, "nominee heaps");
        if (!prc) prc = c->d_tau.ensure(slots, "shared thresholds");
        if (prc) return prc;
        CUDA_TRY(cudaMemsetAsync(c->d_tau, 0, slots * sizeof(uint32_t), stream));
        bp.heaps = c->d_heaps;
        bp.tau_global = c->d_tau;
        bp.no_insert = e->tune.batch_noinsert ? 1u : 0u;
        if (bf16 && used_heap) *used_heap = std::max(*used_heap, ch.kprime);
        if (dump) {
            bp.dump_scores = dump->d_scores;
            const uint32_t shape[7] = {bf16, ch.ares, ch.pair, static_cast<uint32_t>(ch.stages), ch.kprime, ch.slices, ch.groups};
            std::copy(shape, shape + 7, dump->shape);
        }
        return WAX_VS_OK;
    };
    auto finish = [&](const NominateChunk &ch) -> int32_t {
        FinishParams fp{};
        fp.corpus = e->d_corpus; fp.queries = ch.queries; fp.n_rows = static_cast<uint32_t>(e->n_rows); fp.dims = e->dims;
        fp.n_queries = ch.nq; fp.groups = ch.groups; fp.slices = ch.slices; fp.kprime = ch.kprime; fp.k = k_eff;
        fp.metric = e->similarity; fp.heaps = c->d_heaps; fp.max_norm_bits = e->d_max_norm;
        fp.out = d_out + static_cast<size_t>(ch.q0) * k_eff; fp.ok = d_ok + ch.q0;
        fp.frame_ids = d_ids; fp.id_base = e->id_base; fp.row_offset = row_offset; fp.row_keys = c->row_keys;
        uint32_t pow2 = 512;
        while (pow2 < ch.slices * ch.kprime) pow2 <<= 1;
        fp.pow2_all = pow2;
        fp.rescore = rescore;
        fp.eps_rel = bf16 ? kBf16Eps : kTf32Eps;
        fp.tau_star = d_tau_star ? d_tau_star + ch.q0 : nullptr;
        fp.tau_stride = n_queries;
        const size_t fsmem = static_cast<size_t>(pow2 + rescore) * sizeof(uint64_t);
        const auto kernel = e->similarity == WAX_VS_COSINE ? batch_finish_kernel<kCosine>
                            : e->similarity == WAX_VS_DOT  ? batch_finish_kernel<kDot>
                                                           : batch_finish_kernel<kL2>;
        CUDA_TRY(grant_smem(e, kernel, fsmem));
        kernel<<<ch.nq, 512, fsmem, stream>>>(fp);
        CUDA_TRY(cudaGetLastError());
        ++*launches;
        return WAX_VS_OK;
    };
    return enqueue_nominate_pass(e, c, d_queries, n_queries, bf16, false, e->tune.batch_pair != 0, dump != nullptr,
                                 max_groups, rf, stream, launches, heap, prepare, finish);
}

static uint32_t clamp_topk(int64_t k) {  // MetalVectorEngine.swift:842-846
    if (k < 1) return 1;
    if (k > WAX_VS_MAX_RESULTS) return WAX_VS_MAX_RESULTS;
    return static_cast<uint32_t>(k);
}

// VectorMetric.score(fromDistance:) (VectorMetric.swift:32-43)
static float score_from_distance(uint8_t sim, float d) {
    if (!finite_f32(d)) return 0.0f;
    return sim == WAX_VS_COSINE ? 1.0f - d : -d;
}

// ---------------------------------------------------------------------------------------------------------
// corpus storage
static int32_t set_capacity(wax_vs_engine *e, uint64_t rows) {
    if (rows <= e->cap_rows) return WAX_VS_OK;
    float *n = nullptr;
    const size_t bytes = static_cast<size_t>(rows) * e->dims * sizeof(float);
    if (cudaMalloc(&n, bytes) != cudaSuccess) {
        // the shadows are derived data: give their HBM back before giving up (mutators hold the write lock)
        cudaGetLastError();
        for (auto &sh : e->shadows)
            if (sh.codes) { sh.release(); sh.unavailable = true; }
        if (cudaMalloc(&n, bytes) != cudaSuccess)
            return fail(WAX_VS_ERR_CUDA, "Failed to resize vectors buffer (%zu bytes): %s", bytes,
                        cudaGetErrorString(cudaGetLastError()));
    }
    if (e->n_rows) {
        cudaError_t err = cudaMemcpy(n, e->d_corpus, static_cast<size_t>(e->n_rows) * e->dims * sizeof(float),
                                     cudaMemcpyDeviceToDevice);
        if (err != cudaSuccess) { cudaFree(n); return fail(WAX_VS_ERR_CUDA, "corpus copy failed: %s", cudaGetErrorString(err)); }
    }
    if (e->d_corpus) cudaFree(e->d_corpus);
    e->d_corpus = n;
    e->cap_rows = rows;
    return WAX_VS_OK;
}

// reserveIfNeeded (MetalVectorEngine.swift:857-871): doubling from 64.
static int32_t grow_for(wax_vs_engine *e, uint64_t required) {
    if (required > 0xFFFFFFFFull)
        return fail(WAX_VS_ERR_CAPACITY, "capacity exceeded: limit %llu, requested %llu", 0xFFFFFFFFull,
                    static_cast<unsigned long long>(required));
    if (required <= e->cap_rows) return WAX_VS_OK;
    uint64_t next = e->cap_rows ? e->cap_rows : 64;
    while (next < required) next = std::min<uint64_t>(next * 2, 0xFFFFFFFFull);
    return set_capacity(e, next);
}

static void materialize_ids(wax_vs_engine *e) {
    if (!e->ids_identity) return;
    e->ids.resize(e->n_rows);
    for (uint64_t r = 0; r < e->n_rows; ++r) e->ids[r] = e->id_base + r;
    e->ids_identity = false;
    e->map_valid = false;
    e->ids_sorted = true;            // id_base + row
    e->d_ids_dirty = true;
}
static void ensure_map(wax_vs_engine *e) {
    if (e->map_valid) return;
    e->map.reset(e->ids.size());
    for (size_t r = 0; r < e->ids.size(); ++r) e->map.put(e->ids[r], static_cast<uint32_t>(r));
    e->map_valid = true;
}
// frameId -> row (0xFFFFFFFF = absent) for explicit ids: binary search while the id array is sorted, else the hash table.
static uint32_t find_row(wax_vs_engine *e, uint64_t id) {
    if (e->ids_sorted) {
        const auto it = std::lower_bound(e->ids.begin(), e->ids.end(), id);
        return (it != e->ids.end() && *it == id) ? static_cast<uint32_t>(it - e->ids.begin()) : 0xFFFFFFFFu;
    }
    ensure_map(e);
    return e->map.find(id);
}
// frameId -> row (0xFFFFFFFF = absent) for implicit and explicit ids.  May build the hash table: the caller holds the
// write lock or ids_mu.
static uint32_t row_of(wax_vs_engine *e, uint64_t id) {
    if (!e->ids_identity) return find_row(e, id);
    return id >= e->id_base && id - e->id_base < e->n_rows ? static_cast<uint32_t>(id - e->id_base) : 0xFFFFFFFFu;
}
static uint64_t frame_id_of(const wax_vs_engine *e, uint64_t row) { return e->ids_identity ? e->id_base + row : e->ids[row]; }
// A keyed engine's device key column after a mutation (write lock held): rows [from, n_rows) changed.  A column that has
// to grow is uploaded whole.
static int32_t upload_row_keys(wax_vs_engine *e, uint64_t from) {
    if (!e->keys_set || e->n_rows == 0) return WAX_VS_OK;
    if (e->d_keys.cap < e->n_rows) {
        int32_t rc = e->d_keys.ensure(std::max<size_t>(e->n_rows, e->cap_rows), "row keys");
        if (rc) return rc;
        from = 0;
    }
    if (from < e->n_rows)
        CUDA_TRY(cudaMemcpy(e->d_keys + from, e->keys.data() + from, (e->n_rows - from) * sizeof(uint64_t),
                            cudaMemcpyHostToDevice));
    return WAX_VS_OK;
}
// From implicit keys (row r has key r) to an explicit column, before the first keyed mutation.
static int32_t materialize_row_keys(wax_vs_engine *e) {
    if (e->keys_set) return WAX_VS_OK;
    e->keys.resize(e->n_rows);
    for (uint64_t r = 0; r < e->n_rows; ++r) e->keys[r] = r;
    e->keys_set = true;
    return upload_row_keys(e, 0);
}
static int32_t sync_device_ids(wax_vs_engine *e, const uint64_t **out) {
    std::lock_guard<std::mutex> g(e->ids_mu);
    if (e->ids_identity) { *out = nullptr; return WAX_VS_OK; }
    if (e->d_ids_dirty) {
        int32_t rc = e->d_ids.ensure(std::max<size_t>(e->ids.size(), 1), "frame ids");
        if (rc) return rc;
        if (!e->ids.empty())
            CUDA_TRY(cudaMemcpy(e->d_ids, e->ids.data(), e->ids.size() * sizeof(uint64_t), cudaMemcpyHostToDevice));
        e->d_ids_dirty = false;
    }
    *out = e->d_ids;
    return WAX_VS_OK;
}

// A where as the host plans it: the time and tag clauses, the location box (kNoLocBox: no location clause) and the
// sorted, distinct term ids a row must hold (none: no term clause), the group clause and the root clause.
struct Clause {
    WherePred pred;
    LocBox box;
    std::vector<uint64_t> terms;
    std::vector<uint64_t> groups;      // sorted, distinct group ids, one of which the row's group must be (none: no clause)
    RootClause root{0, 0};             // the row's group's root-tag word must pass it ({0, 0}: no clause)
};

// What a filtered, where or grouped search asks for.  Its entry point checks the arguments and builds it once (the
// request_* builders); then it is only read, by one engine or concurrently by every shard of a multi-device handle.
// Query i searches under id filter query_filter[i] and where query_where[i], either of which may be WAX_VS_NO_FILTER.
// The arrays are the caller's, or the request's own storage for the forms with one filter or one where for every query
// and for canonical term wheres, so a request is neither copied nor moved.
struct SearchRequest {
    const float *queries;                   // host memory; the device forms pass their queries beside the request
    uint32_t n_queries, query_len;
    int64_t top_k;                          // grouped search: top_groups
    uint32_t per_group;                     // grouped search only
    bool batched;                           // grouped search: the batch pipeline may take the queries
    const uint64_t *frame_ids = nullptr;
    const uint64_t *filter_offsets = nullptr;
    const int32_t *filter_modes = nullptr;
    uint32_t n_filters = 0;
    const uint32_t *query_filter = nullptr;
    std::vector<Clause> wheres;
    const uint32_t *query_where = nullptr;  // nullptr: no where list, the filtered entry points (plan_request)
    uint64_t one_offsets[2] = {0, 0};
    int32_t one_mode = 0;
    std::vector<uint32_t> filter_of, where_of;
    SearchRequest(const float *q, uint32_t n, uint32_t len, int64_t k, uint32_t groups_of = 0, bool batch = false)
        : queries(q), n_queries(n), query_len(len), top_k(k), per_group(groups_of), batched(batch) {}
    SearchRequest(const SearchRequest &) = delete;
    SearchRequest &operator=(const SearchRequest &) = delete;
};

extern "C" {
static int32_t absorb_rows(wax_vs_engine *e, wax_vs_engine *donor, uint64_t first, uint64_t n);
static int32_t search_where_device(wax_vs_engine *e, const SearchRequest &req, const float *d_queries, uint64_t row_offset,
                                   wax_vs_candidate *d_candidates, void *cuda_stream);
static int32_t grouped_heads_device(wax_vs_engine *e, const SearchRequest &req, const float *d_queries, uint64_t row_offset,
                                    wax_vs_group_candidate *d_heads, void *cuda_stream);
static int32_t grouped_expand_device(wax_vs_engine *e, const SearchRequest &req, const float *d_queries,
                                     const wax_vs_group_candidate *d_chosen, const wax_vs_group_candidate *d_own_heads,
                                     uint64_t row_offset, wax_vs_candidate *d_rows, void *cuda_stream);
}

#include "waxvs_multi.cuh"

// ---------------------------------------------------------------------------------------------------------
// C-ABI
extern "C" {

const char *wax_vs_last_error(void) { return g_last_error; }
const char *wax_vs_version(void) { return "waxvs_cuda 0.1 sm_90a (fused scan+top-k; TMA bulk staging)"; }

int32_t wax_vs_device_count(int32_t *out) {
    if (!out) return fail(WAX_VS_ERR_NULL, "out is NULL");
    int n = 0;
    cudaError_t err = cudaGetDeviceCount(&n);
    if (err != cudaSuccess) { *out = 0; cudaGetLastError(); return fail(WAX_VS_ERR_CUDA, "CUDA device not available: %s", cudaGetErrorString(err)); }
    *out = n;
    return WAX_VS_OK;
}

int32_t wax_vs_create(uint32_t dimensions, uint8_t similarity, const int32_t *devices, int32_t n_devices,
                      wax_vs_engine **out) {
    if (!out) return fail(WAX_VS_ERR_NULL, "out is NULL");
    *out = nullptr;
    if (dimensions == 0) return fail(WAX_VS_ERR_ARGUMENT, "dimensions must be > 0");  // :154-156
    if (dimensions > WAX_VS_MAX_DIMENSIONS)                                           // :157-162
        return fail(WAX_VS_ERR_CAPACITY, "capacity exceeded: limit %d, requested %u", WAX_VS_MAX_DIMENSIONS, dimensions);
    if (similarity > 2) return fail(WAX_VS_ERR_ARGUMENT, "vec similarity must be 0..2 (got %u)", similarity);
    if (n_devices > 1) {               // a multi-device handle (waxvs_multi.cuh): its own checks come before any device query
        if (n_devices > WAX_VS_SHARD_MAX_RANKS)
            return fail(WAX_VS_ERR_ARGUMENT, "%d devices: a multi-device handle takes at most %d", n_devices, WAX_VS_SHARD_MAX_RANKS);
        if (!devices) return fail(WAX_VS_ERR_NULL, "devices is NULL");
        for (int32_t r = 0; r < n_devices; ++r)
            if (devices[r] < 0) return fail(WAX_VS_ERR_ARGUMENT, "device ordinal %d is negative", devices[r]);
        return multi_create(dimensions, similarity, devices, n_devices, out);
    }
    int count = 0;
    if (cudaGetDeviceCount(&count) != cudaSuccess || count <= 0) {
        cudaGetLastError();
        return fail(WAX_VS_ERR_CUDA, "CUDA device not available");  // "Metal device not available" :167-169
    }
    int dev = 0;
    if (devices && n_devices == 1) dev = devices[0];
    else if (cudaGetDevice(&dev) != cudaSuccess) dev = 0;
    if (dev < 0 || dev >= count) return fail(WAX_VS_ERR_ARGUMENT, "device ordinal %d out of range (0..%d)", dev, count - 1);

    wax_vs_engine *e = new (std::nothrow) wax_vs_engine();
    if (!e) return fail(WAX_VS_ERR_CUDA, "out of host memory");
    e->device = dev; e->dims = dimensions; e->similarity = similarity;
    DeviceGuard g(dev);
    int v = 0;
    if (!g.ok || cudaDeviceGetAttribute(&v, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess) {
        delete e;
        return fail(WAX_VS_ERR_CUDA, "failed to select CUDA device %d", dev);
    }
    e->sm_count = v;
    if (cudaDeviceGetAttribute(&v, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev) == cudaSuccess) e->smem_optin = static_cast<size_t>(v);
    int32_t rc = set_capacity(e, 64);  // initialReserve (:19, :225-229)
    if (rc) { delete e; return rc; }
    *out = e;
    return WAX_VS_OK;
}

void wax_vs_destroy(wax_vs_engine *e) {
    if (!e) return;
    if (e->multi) { multi_destroy(e->multi); delete e; return; }
    DeviceGuard g(e->device);      // the engine's own buffers go with `delete e`: on its device too
    {
        std::unique_lock<std::shared_mutex> w(e->rw);
        cudaDeviceSynchronize();
        shard_teardown(e, true);
        for (SearchCtx *c : e->pool) delete c;
        for (auto &kv : e->stream_ctx) delete kv.second;
        if (e->d_corpus) cudaFree(e->d_corpus);
    }
    delete e;
}

int32_t wax_vs_dimensions(const wax_vs_engine *e, uint32_t *out) {
    if (e && e->multi && out) { *out = e->dims; return WAX_VS_OK; }
    if (!e || !out) return fail(WAX_VS_ERR_NULL, "NULL argument");
    *out = e->dims;
    return WAX_VS_OK;
}
int32_t wax_vs_similarity(const wax_vs_engine *e, uint8_t *out) {
    if (!e || !out) return fail(WAX_VS_ERR_NULL, "NULL argument");
    *out = e->similarity;
    return WAX_VS_OK;
}
int32_t wax_vs_count(wax_vs_engine *e, uint64_t *out) {
    if (e && e->multi && out) { std::shared_lock<std::shared_mutex> r(e->multi->rw); *out = e->multi->total(); return WAX_VS_OK; }
    if (!e || !out) return fail(WAX_VS_ERR_NULL, "NULL argument");
    std::shared_lock<std::shared_mutex> r(e->rw);
    *out = e->n_rows;
    return WAX_VS_OK;
}

int32_t wax_vs_reserve(wax_vs_engine *e, uint64_t rows) {
    if (e && e->multi) return multi_reserve(e->multi, rows);
    if (!e) return fail(WAX_VS_ERR_NULL, "engine is NULL");
    if (rows > 0xFFFFFFFFull)
        return fail(WAX_VS_ERR_CAPACITY, "capacity exceeded: limit %llu, requested %llu", 0xFFFFFFFFull,
                    static_cast<unsigned long long>(rows));
    std::unique_lock<std::shared_mutex> w(e->rw);
    DeviceGuard g(e->device);
    drain_device_path(e);
    int32_t rc = set_capacity(e, rows);
    if (rc == WAX_VS_OK && !e->ids_identity && rows > e->ids.capacity()) {
        e->ids.reserve(rows);                       // no id-array / hash-table regrowth during the appends that follow
        if (!e->ids_sorted && e->map_valid && e->map.keys.size() < rows * 2 + 16) {
            IdMap bigger;
            bigger.reset(rows);
            for (size_t r = 0; r < e->ids.size(); ++r) bigger.put(e->ids[r], static_cast<uint32_t>(r));
            e->map = std::move(bigger);
        }
    }
    return rc;
}

// Phase trace of the mutators for performance work: WAXVS_TRACE_INGEST=1 prints "<what>: <phase> <us>" lines to stderr.
struct IngestTrace {
    bool on;
    const char *what;
    std::chrono::steady_clock::time_point t;
    explicit IngestTrace(const char *w) : on(getenv("WAXVS_TRACE_INGEST") != nullptr), what(w), t(std::chrono::steady_clock::now()) {}
    void mark(const char *phase) {
        if (!on) return;
        const auto now = std::chrono::steady_clock::now();
        fprintf(stderr, "[waxvs] %s: %s %.1f us\n", what, phase, std::chrono::duration<double, std::micro>(now - t).count());
        t = now;
    }
};

// ---- bulk ingest / export plumbing (SURVEY.md section 8f-3) ---------------------------------------------------------------
// Host <-> HBM at device speed from PAGEABLE caller memory: the bytes go through two pinned staging buffers; worker
// threads fill (or drain) one buffer while the DMA engine moves the other.  Caller memory that is already pinned
// (cudaHostAlloc / cudaHostRegister) is handed to the DMA engine directly.
static int32_t ingest_init(wax_vs_engine *e) {
    auto &g = e->ing;
    if (g.stream) return WAX_VS_OK;
    CUDA_TRY(cudaStreamCreateWithFlags(&g.stream, cudaStreamNonBlocking));
    for (int i = 0; i < 2; ++i) CUDA_TRY(cudaEventCreateWithFlags(&g.ev[i], cudaEventDisableTiming));
    unsigned hw = std::thread::hardware_concurrency();
    long quota = 0, period = 0;                       // cgroup v2 CPU quota, when there is one
    if (FILE *f = fopen("/sys/fs/cgroup/cpu.max", "r")) {
        char q[32] = "";
        if (fscanf(f, "%31s %ld", q, &period) == 2 && strcmp(q, "max") != 0) quota = atol(q);
        fclose(f);
    }
    if (quota > 0 && period > 0) hw = static_cast<unsigned>(std::max<long>(1, std::min<long>(hw ? hw : 1, (quota + period / 2) / period)));
    g.threads = static_cast<int>(std::max(1u, std::min(8u, hw ? hw : 1u)));
    return WAX_VS_OK;
}
// The two large pinned staging buffers are shared by every engine of the process (pinning 2 x 64 MB costs ~0.1 s, far
// more than most transfers): whoever holds g_staging_mu owns them for the length of one upload / download.  Small
// transfers use the engine's own 1 MB pair.
static std::mutex g_staging_mu;
static uint8_t *g_staging[2] = {nullptr, nullptr};
constexpr size_t kStagingBytes = size_t(64) << 20;
constexpr size_t kSmallStagingBytes = size_t(1) << 20;

static int32_t ingest_staging(wax_vs_engine *e, size_t want_bytes) {
    auto &g = e->ing;
    int32_t rc = ingest_init(e);
    if (rc) return rc;
    (void)want_bytes;
    if (g.pin_bytes >= kSmallStagingBytes) return WAX_VS_OK;
    for (int i = 0; i < 2; ++i) {
        if (cudaHostAlloc(reinterpret_cast<void **>(&g.pin[i]), kSmallStagingBytes, cudaHostAllocPortable) != cudaSuccess)
            return fail(WAX_VS_ERR_CUDA, "failed to allocate pinned ingest staging: %s", cudaGetErrorString(cudaGetLastError()));
    }
    g.pin_bytes = kSmallStagingBytes;
    return WAX_VS_OK;
}
// caller holds g_staging_mu
static int32_t shared_staging() {
    for (int i = 0; i < 2; ++i) {
        if (!g_staging[i] && cudaHostAlloc(reinterpret_cast<void **>(&g_staging[i]), kStagingBytes, cudaHostAllocPortable) != cudaSuccess)
            return fail(WAX_VS_ERR_CUDA, "failed to allocate the shared pinned staging (%zu bytes): %s", kStagingBytes, cudaGetErrorString(cudaGetLastError()));
    }
    return WAX_VS_OK;
}
static void parallel_memcpy(void *dst, const void *src, size_t bytes, int threads) {
    const size_t min_slice = size_t(2) << 20;
    int t = static_cast<int>(std::min<size_t>(static_cast<size_t>(std::max(threads, 1)), std::max<size_t>(1, bytes / min_slice)));
    if (t <= 1) { memcpy(dst, src, bytes); return; }
    std::vector<std::thread> pool;
    pool.reserve(static_cast<size_t>(t - 1));
    const size_t per = ((bytes + t - 1) / t + 63) & ~size_t(63);
    for (int i = 1; i < t; ++i) {
        const size_t off = std::min(bytes, per * i), len = std::min(bytes - off, per);
        if (len) pool.emplace_back([=] { memcpy(static_cast<char *>(dst) + off, static_cast<const char *>(src) + off, len); });
    }
    memcpy(dst, src, std::min(bytes, per));
    for (auto &th : pool) th.join();
}

static bool host_pointer_is_pinned(const void *p) {
    cudaPointerAttributes at{};
    if (cudaPointerGetAttributes(&at, p) != cudaSuccess) { cudaGetLastError(); return false; }
    return at.type == cudaMemoryTypeHost;
}

// host (pageable or pinned) -> device, synchronous on return
static int32_t upload_bytes(wax_vs_engine *e, void *d_dst, const void *h_src, size_t bytes) {
    if (bytes == 0) return WAX_VS_OK;
    int32_t rc = ingest_staging(e, bytes);
    if (rc) return rc;
    auto &g = e->ing;
    e->ingest_h2d_bytes += bytes;
    if (host_pointer_is_pinned(h_src)) {
        CUDA_TRY(cudaMemcpyAsync(d_dst, h_src, bytes, cudaMemcpyHostToDevice, g.stream));
        CUDA_TRY(cudaStreamSynchronize(g.stream));
        return WAX_VS_OK;
    }
    const bool big = bytes > 2 * kSmallStagingBytes;
    std::unique_lock<std::mutex> pool(g_staging_mu, std::defer_lock);
    if (big) { pool.lock(); if ((rc = shared_staging())) return rc; }
    uint8_t *const *pin = big ? g_staging : g.pin;
    const size_t pin_bytes = big ? kStagingBytes : g.pin_bytes;
    size_t off = 0;
    for (int i = 0; off < bytes; ++i) {
        const int b = i & 1;
        const size_t len = std::min(pin_bytes, bytes - off);
        CUDA_TRY(cudaEventSynchronize(g.ev[b]));                 // the DMA that last read this buffer is done
        parallel_memcpy(pin[b], static_cast<const char *>(h_src) + off, len, g.threads);
        CUDA_TRY(cudaMemcpyAsync(static_cast<char *>(d_dst) + off, pin[b], len, cudaMemcpyHostToDevice, g.stream));
        CUDA_TRY(cudaEventRecord(g.ev[b], g.stream));
        off += len;
    }
    CUDA_TRY(cudaStreamSynchronize(g.stream));
    return WAX_VS_OK;
}

// device -> host (pageable or pinned), synchronous on return
static int32_t download_bytes(wax_vs_engine *e, void *h_dst, const void *d_src, size_t bytes) {
    if (bytes == 0) return WAX_VS_OK;
    int32_t rc = ingest_staging(e, bytes);
    if (rc) return rc;
    auto &g = e->ing;
    e->ingest_d2h_bytes += bytes;
    if (host_pointer_is_pinned(h_dst)) {
        CUDA_TRY(cudaMemcpyAsync(h_dst, d_src, bytes, cudaMemcpyDeviceToHost, g.stream));
        CUDA_TRY(cudaStreamSynchronize(g.stream));
        return WAX_VS_OK;
    }
    const bool big = bytes > 2 * kSmallStagingBytes;
    std::unique_lock<std::mutex> pool(g_staging_mu, std::defer_lock);
    if (big) { pool.lock(); if ((rc = shared_staging())) return rc; }
    uint8_t *const *pin = big ? g_staging : g.pin;
    const size_t pin_bytes = big ? kStagingBytes : g.pin_bytes;
    const size_t n_chunks = (bytes + pin_bytes - 1) / pin_bytes;
    auto issue = [&](size_t i) -> cudaError_t {
        const size_t off = i * pin_bytes, len = std::min(pin_bytes, bytes - off);
        cudaError_t err = cudaMemcpyAsync(pin[i & 1], static_cast<const char *>(d_src) + off, len, cudaMemcpyDeviceToHost, g.stream);
        if (err == cudaSuccess) err = cudaEventRecord(g.ev[i & 1], g.stream);
        return err;
    };
    CUDA_TRY(issue(0));
    for (size_t i = 0; i < n_chunks; ++i) {
        if (i + 1 < n_chunks) CUDA_TRY(issue(i + 1));            // its buffer was drained in iteration i-1
        CUDA_TRY(cudaEventSynchronize(g.ev[i & 1]));
        const size_t off = i * pin_bytes, len = std::min(pin_bytes, bytes - off);
        parallel_memcpy(static_cast<char *>(h_dst) + off, pin[i & 1], len, g.threads);
    }
    CUDA_TRY(cudaStreamSynchronize(g.stream));
    return WAX_VS_OK;
}

// addBatch for wax_vs_add_batch (first_key nullptr) and wax_vs_add_batch_keyed.  The appended rows of a keyed engine take
// the keys *first_key, *first_key + 1, ... (nullptr: the keys that follow the last one).
static int32_t add_batch_rows(wax_vs_engine *e, const uint64_t *frame_ids, const float *rows, uint64_t n,
                              uint32_t vector_len, const uint64_t *first_key, uint64_t *out_appended) {
    if (!e) return fail(WAX_VS_ERR_NULL, "engine is NULL");
    if (out_appended) *out_appended = 0;
    if (n == 0) return WAX_VS_OK;  // guard !frameIds.isEmpty (:360)
    if (!frame_ids || !rows) return fail(WAX_VS_ERR_NULL, "NULL argument");
    if (vector_len != e->dims)     // :367-370
        return fail(WAX_VS_ERR_DIMENSION, "vector dimension mismatch: expected %u, got %u", e->dims, vector_len);
    IngestTrace tr("add_batch");
    std::unique_lock<std::shared_mutex> w(e->rw);
    if (first_key && e->n_rows > 0) {
        const uint64_t last = e->keys_set ? e->keys.back() : e->n_rows - 1;
        if (*first_key <= last)
            return fail(WAX_VS_ERR_ARGUMENT, "first key %llu is not above the last row key %llu",
                        static_cast<unsigned long long>(*first_key), static_cast<unsigned long long>(last));
    }
    DeviceGuard g(e->device);
    drain_device_path(e);
    tr.mark("lock+drain");
    int32_t rc = grow_for(e, e->n_rows + n);  // maxNewCount (:379-380)
    if (rc) return rc;
    if (first_key && (rc = materialize_row_keys(e))) return rc;
    tr.mark("grow");
    materialize_ids(e);
    tr.mark("ids");

    // Resolve the destination row of every batch item in order (the sequential loop at :384-398).
    std::vector<uint32_t> target(n);
    const uint64_t n0 = e->n_rows;
    bool pure_append = true;
    bool increasing = e->ids_sorted && (e->ids.empty() || frame_ids[0] > e->ids.back());
    for (uint64_t i = 1; i < n && increasing; ++i) increasing = frame_ids[i] > frame_ids[i - 1];
    if (increasing) {
        // the common bulk-ingest case: every id is new and larger than all stored ones -- no lookups, no hash table
        e->ids.insert(e->ids.end(), frame_ids, frame_ids + n);
        if (e->groups_set) e->groups.insert(e->groups.end(), frame_ids, frame_ids + n);   // a new frame is its own group
        if (e->attrs_set) e->attrs.resize(e->attrs.size() + n, AttrRow{0, 0});               // ... and has no attributes
        if (e->locs_set) e->locs.resize(e->locs.size() + n, LocRow{kNoLocation, 0});         // ... nor a location
        if (e->terms_set) e->term_refs.resize(e->term_refs.size() + n, wax_vs_engine::TermRef{0, 0});   // ... nor terms
        for (uint64_t i = 0; i < n; ++i) target[i] = static_cast<uint32_t>(n0 + i);
        e->n_rows += n;
        e->map_valid = false;
    } else {
        for (uint64_t i = 0; i < n; ++i) {
            if (!e->ids_sorted && i + 8 < n) e->map.prefetch(frame_ids[i + 8]);   // the table is far bigger than the caches
            uint32_t row = find_row(e, frame_ids[i]);
            if (row == 0xFFFFFFFFu) {
                row = static_cast<uint32_t>(e->n_rows);
                if (e->ids_sorted && !e->ids.empty() && frame_ids[i] < e->ids.back()) {
                    e->ids_sorted = false;                   // first out-of-order id: from now on the hash table answers
                    e->map_valid = false;
                    ensure_map(e);
                }
                e->ids.push_back(frame_ids[i]);
                if (e->groups_set) e->groups.push_back(frame_ids[i]);    // an upsert of a known frame keeps its group
                if (e->attrs_set) e->attrs.push_back(AttrRow{0, 0});     // ... and its attributes
                if (e->locs_set) e->locs.push_back(LocRow{kNoLocation, 0});   // ... and its location
                if (e->terms_set) e->term_refs.push_back(wax_vs_engine::TermRef{0, 0});   // ... and its terms
                if (!e->ids_sorted) e->map.put(frame_ids[i], row);
                else e->map_valid = false;
                ++e->n_rows;
            }
            target[i] = row;
            if (row != n0 + i) pure_append = false;
        }
    }
    e->d_ids_dirty = true;
    if (out_appended) *out_appended = e->n_rows - n0;
    if (e->keys_set) {
        const uint64_t base = first_key ? *first_key : (n0 ? e->keys.back() + 1 : 0);
        for (uint64_t r = n0; r < e->n_rows; ++r) e->keys.push_back(base + (r - n0));
        if ((rc = upload_row_keys(e, n0))) return rc;
    }
    const size_t row_bytes = static_cast<size_t>(e->dims) * sizeof(float);
    tr.mark("resolve targets");
    if (pure_append) {
        invalidate_row_caches(e, n0);          // the cached norms / shadow of rows [0, n0) stay valid
        rc = upload_bytes(e, e->d_corpus + n0 * e->dims, rows, n * row_bytes);
        tr.mark("upload");
        return rc;
    }
    invalidate_row_caches(e, 0);
    // Overwrites present: a later item for the same row wins; earlier ones are dropped.
    {
        std::unordered_map<uint32_t, uint64_t> last;
        last.reserve(n * 2);
        for (uint64_t i = 0; i < n; ++i) last[target[i]] = i;
        for (uint64_t i = 0; i < n; ++i) if (last[target[i]] != i) target[i] = 0xFFFFFFFFu;
    }
    // Staged in HBM (persistent staging area, grown on demand) and scattered by one kernel: no per-call allocation.
    auto &ig = e->ing;
    if ((rc = ingest_init(e))) return rc;
    const uint64_t slab_rows = std::max<uint64_t>(1, std::min<uint64_t>(n, (size_t(256) << 20) / row_bytes));
    if ((rc = ig.d_stage.ensure(static_cast<size_t>(slab_rows) * e->dims, "upsert staging"))) return rc;
    if ((rc = ig.d_index.ensure(static_cast<size_t>(slab_rows), "upsert targets"))) return rc;
    for (uint64_t done = 0; done < n; done += slab_rows) {
        const uint64_t m = std::min(slab_rows, n - done);
        if ((rc = upload_bytes(e, ig.d_stage, rows + done * e->dims, m * row_bytes))) return rc;
        CUDA_TRY(cudaMemcpyAsync(ig.d_index, target.data() + done, m * sizeof(uint32_t), cudaMemcpyHostToDevice, ig.stream));
        scatter_rows_kernel<<<static_cast<unsigned>(m), 128, 0, ig.stream>>>(e->d_corpus, ig.d_stage, ig.d_index, m, e->dims);
        CUDA_TRY(cudaGetLastError());
        CUDA_TRY(cudaStreamSynchronize(ig.stream));
    }
    return WAX_VS_OK;
}

int32_t wax_vs_add_batch(wax_vs_engine *e, const uint64_t *frame_ids, const float *rows, uint64_t n,
                         uint32_t vector_len) {
    if (e && e->multi) return multi_add_batch(e->multi, frame_ids, rows, n, e->dims, vector_len);
    return add_batch_rows(e, frame_ids, rows, n, vector_len, nullptr, nullptr);
}

int32_t wax_vs_add_batch_keyed(wax_vs_engine *e, const uint64_t *frame_ids, const float *rows, uint64_t n,
                               uint32_t vector_len, uint64_t first_key, uint64_t *out_appended) {
    WAX_VS_MULTI_REFUSE(e, "wax_vs_add_batch_keyed");
    return add_batch_rows(e, frame_ids, rows, n, vector_len, &first_key, out_appended);
}

int32_t wax_vs_add(wax_vs_engine *e, uint64_t frame_id, const float *vector, uint32_t vector_len) {
    return wax_vs_add_batch(e, &frame_id, vector, 1, vector_len);
}

int32_t wax_vs_contains(wax_vs_engine *e, const uint64_t *frame_ids, uint64_t n, uint8_t *out) {
    WAX_VS_MULTI_REFUSE(e, "wax_vs_contains");
    if (!e) return fail(WAX_VS_ERR_NULL, "engine is NULL");
    if (n == 0) return WAX_VS_OK;
    if (!frame_ids || !out) return fail(WAX_VS_ERR_NULL, "NULL argument");
    std::shared_lock<std::shared_mutex> r(e->rw);
    std::lock_guard<std::mutex> g(e->ids_mu);     // row_of may build the id map
    for (uint64_t i = 0; i < n; ++i) out[i] = row_of(e, frame_ids[i]) != 0xFFFFFFFFu;
    return WAX_VS_OK;
}

// remove(frameId:) for a whole set of frames (MetalVectorEngine.swift:423-444 applied n times, as ONE pass): unknown ids
// are ignored (:426), the surviving rows keep their relative order (:431-441).  The reference memmoves the tail once
// per id; here the survivors' source rows are computed once on the host, the matrix is compacted slab by slab through
// an HBM bounce buffer (gather kernel + copy back: destinations never overtake unread sources because rows only move
// down and slabs go in ascending order), the id array is compacted once and the id->row hash rebuilt once.
int32_t wax_vs_remove_batch(wax_vs_engine *e, const uint64_t *frame_ids, uint64_t n, uint64_t *out_removed) {
    if (e && e->multi) return multi_remove_batch(e->multi, frame_ids, n, out_removed);
    if (!e) return fail(WAX_VS_ERR_NULL, "engine is NULL");
    if (out_removed) *out_removed = 0;
    if (n == 0) return WAX_VS_OK;
    if (!frame_ids) return fail(WAX_VS_ERR_NULL, "frame_ids is NULL");
    IngestTrace tr("remove_batch");
    std::unique_lock<std::shared_mutex> w(e->rw);
    if (e->n_rows == 0) return WAX_VS_OK;  // :425
    // which rows go
    std::vector<uint32_t> gone;
    gone.reserve(n);
    for (uint64_t i = 0; i < n; ++i) {
        const uint32_t r = row_of(e, frame_ids[i]);
        if (r != 0xFFFFFFFFu) gone.push_back(r);                    // :426 unknown id = no-op
    }
    if (gone.empty()) return WAX_VS_OK;
    std::sort(gone.begin(), gone.end());
    gone.erase(std::unique(gone.begin(), gone.end()), gone.end());
    DeviceGuard g(e->device);
    drain_device_path(e);
    materialize_ids(e);
    const uint64_t old_n = e->n_rows, first = gone.front(), new_n = old_n - gone.size();
    // source row of every destination row >= first (rows below the first removed row do not move)
    std::vector<uint32_t> src;
    src.reserve(static_cast<size_t>(new_n - first));
    {
        size_t gi = 0;
        for (uint64_t r = first; r < old_n; ++r) {
            if (gi < gone.size() && gone[gi] == r) { ++gi; continue; }
            src.push_back(static_cast<uint32_t>(r));
        }
    }
    tr.mark("resolve rows + sources");
    int32_t rc = ingest_init(e);
    if (rc) return rc;
    auto &ig = e->ing;
    const size_t row_bytes = static_cast<size_t>(e->dims) * sizeof(float);
    const uint64_t moving = src.size();
    if (moving) {
        const uint64_t slab_rows = std::max<uint64_t>(1, std::min<uint64_t>(moving, (size_t(256) << 20) / row_bytes));
        if ((rc = ig.d_stage.ensure(static_cast<size_t>(slab_rows) * e->dims, "compaction bounce buffer"))) return rc;
        if ((rc = ig.d_index.ensure(static_cast<size_t>(slab_rows), "compaction sources"))) return rc;
        if ((rc = ingest_staging(e, slab_rows * sizeof(uint32_t)))) return rc;
        for (uint64_t done = 0; done < moving; done += slab_rows) {
            const uint64_t m = std::min(slab_rows, moving - done);
            // contiguous runs (nothing removed inside the slab) are a plain device copy; otherwise gather by index
            const bool contiguous = src[done + m - 1] - src[done] == m - 1;
            float *dst = e->d_corpus + (first + done) * e->dims;
            if (contiguous) {
                CUDA_TRY(cudaMemcpyAsync(ig.d_stage, e->d_corpus + static_cast<uint64_t>(src[done]) * e->dims, m * row_bytes,
                                         cudaMemcpyDeviceToDevice, ig.stream));
            } else {
                CUDA_TRY(cudaMemcpyAsync(ig.d_index, src.data() + done, m * sizeof(uint32_t), cudaMemcpyHostToDevice, ig.stream));
                const unsigned grid = static_cast<unsigned>(std::min<uint64_t>(m, static_cast<uint64_t>(e->sm_count) * 32));
                gather_rows_kernel<<<grid, 128, 0, ig.stream>>>(ig.d_stage, e->d_corpus, ig.d_index, m, e->dims);
                CUDA_TRY(cudaGetLastError());
            }
            CUDA_TRY(cudaMemcpyAsync(dst, ig.d_stage, m * row_bytes, cudaMemcpyDeviceToDevice, ig.stream));
            CUDA_TRY(cudaStreamSynchronize(ig.stream));          // src / d_index are reused by the next slab
        }
    }
    tr.mark("compact matrix");
    // ids: one compaction, one hash rebuild (lazily, on the next lookup)
    if (e->terms_set)
        for (const uint32_t r : gone) e->term_garbage += e->term_refs[r].n;   // the removed rows' pool entries
    for (uint64_t j = 0; j < moving; ++j) {
        e->ids[first + j] = e->ids[src[j]];
        if (e->groups_set) e->groups[first + j] = e->groups[src[j]];
        if (e->attrs_set) e->attrs[first + j] = e->attrs[src[j]];
        if (e->locs_set) e->locs[first + j] = e->locs[src[j]];
        if (e->terms_set) e->term_refs[first + j] = e->term_refs[src[j]];
        if (e->keys_set) e->keys[first + j] = e->keys[src[j]];
    }
    e->ids.resize(new_n);
    if (e->keys_set) e->keys.resize(new_n);
    if (e->groups_set) e->groups.resize(new_n);
    if (e->attrs_set) e->attrs.resize(new_n);
    if (e->locs_set) e->locs.resize(new_n);
    if (e->terms_set) {
        e->term_refs.resize(new_n);
        compact_term_pool(e);
    }
    e->n_rows = new_n;
    e->map_valid = false;
    e->d_ids_dirty = true;
    invalidate_row_caches(e, first);           // rows below the first removed row did not move
    if ((rc = upload_row_keys(e, first))) return rc;
    tr.mark("compact ids");
    if (out_removed) *out_removed = gone.size();
    return WAX_VS_OK;
}

int32_t wax_vs_remove(wax_vs_engine *e, uint64_t frame_id) {
    return wax_vs_remove_batch(e, &frame_id, 1, nullptr);
}

// The source of a rebalance merge (absorb_body): n rows in strictly increasing key order, their vectors (n x dims fp32 on
// device()) and their side columns.  set() is the WAX_VS_COLUMN_* bits of the columns the source holds; a column it does
// not hold is answered with the defaults its rows have (group = own frame id, attributes {0, 0}, no location, no terms).
static_assert(sizeof(wax_vs_row_columns) == 32 && WAX_VS_NO_LOCATION == kNoLocation, "wax_vs_row_columns layout");
struct TermList {
    const uint64_t *p;
    uint32_t n;
};
// Rows [first, first + n) of another engine of this process (multi_rebalance), read under its read lock.
struct DonorRows {
    const wax_vs_engine *d;
    uint64_t first, n;
    const float *vectors() const { return d->d_corpus + first * d->dims; }
    int device() const { return d->device; }
    uint32_t set() const {
        return (d->groups_set ? WAX_VS_COLUMN_GROUPS : 0u) | (d->attrs_set ? WAX_VS_COLUMN_ATTRIBUTES : 0u) |
               (d->locs_set ? WAX_VS_COLUMN_LOCATIONS : 0u) | (d->terms_set ? WAX_VS_COLUMN_TERMS : 0u);
    }
    uint64_t key(uint64_t j) const { return d->keys[first + j]; }
    uint64_t id(uint64_t j) const { return frame_id_of(d, first + j); }
    uint64_t group(uint64_t j) const { return d->groups[first + j]; }
    AttrRow attr(uint64_t j) const { return d->attrs[first + j]; }
    LocRow loc(uint64_t j) const { return d->locs[first + j]; }
    TermList terms(uint64_t j) const {
        const wax_vs_engine::TermRef t = d->term_refs[first + j];
        return TermList{d->term_pool.data() + t.off, t.n};
    }
};
// Rows the caller hands over (wax_vs_absorb_rows), already checked.
struct CallerRows {
    const uint64_t *ids, *keys_;
    const float *vecs;
    int dev;
    uint64_t n;
    uint32_t columns_set;
    const wax_vs_row_columns *cols;
    const uint64_t *term_offsets, *term_ids;
    const float *vectors() const { return vecs; }
    int device() const { return dev; }
    uint32_t set() const { return columns_set; }
    uint64_t key(uint64_t j) const { return keys_[j]; }
    uint64_t id(uint64_t j) const { return ids[j]; }
    uint64_t group(uint64_t j) const { return cols[j].group; }
    AttrRow attr(uint64_t j) const { return AttrRow{cols[j].timestamp, cols[j].tags}; }
    LocRow loc(uint64_t j) const { return LocRow{cols[j].lat_bin, cols[j].lon_bin}; }
    TermList terms(uint64_t j) const {
        return TermList{term_ids + term_offsets[j], static_cast<uint32_t>(term_offsets[j + 1] - term_offsets[j])};
    }
};

// The receiving half of a rebalance move (DESIGN.md sections 4.15 and 4.16): the rows of `in` merge into `e` by key
// together with their ids, keys, groups, attributes, locations and terms.  The write lock of `e` is held and the rows
// are checked.  Every allocation (the receiver's growth, the bounce buffer, the staging, the key column) comes before a
// row changes, so a failed allocation leaves `e` as it was.  Destination slabs are written top-down: own rows only move
// up and incoming rows only move down, so a slab's sources lie in it or below it, and each slab is gathered into the
// bounce buffer (merge_rows_kernel) before it is copied in place, as the compaction of remove_batch does.  The incoming
// rows of one slab are one contiguous run of the source's, staged on the receiver's device with cudaMemcpyPeerAsync (a
// device-local copy when the two share a device): no kernel reads peer memory.  The source is only read.
extern "C++" {                                 // the merge body is a template over its source
template <class Src>
static int32_t absorb_body(wax_vs_engine *e, const Src &in) {
    IngestTrace tr("rebalance merge");
    DeviceGuard g(e->device);
    if (!g.ok) return g.error();
    drain_device_path(e);
    const uint64_t n = in.n, n0 = e->n_rows, m = n0 + n;
    // rows below the first incoming key keep their place; every destination row from f on has a tagged source
    const uint64_t f = static_cast<uint64_t>(std::lower_bound(e->keys.begin(), e->keys.end(), in.key(0)) - e->keys.begin());
    const uint64_t total = m - f;
    std::vector<uint64_t> src(total);
    for (uint64_t t = 0, i = f, j = 0; t < total; ++t)
        src[t] = j < n && (i == n0 || in.key(j) < e->keys[i]) ? (kMergeIncoming | j++) : i++;
    tr.mark("lock+drain+merge positions");

    int32_t rc;
    if ((rc = grow_for(e, m)) || (rc = ingest_init(e))) return rc;
    auto &ig = e->ing;
    const size_t row_bytes = static_cast<size_t>(e->dims) * sizeof(float);
    const uint64_t slab_rows = std::max<uint64_t>(1, std::min<uint64_t>(total, e->tune.rebalance_slab_bytes / row_bytes));
    DevBuf<float> incoming;
    DevBuf<uint64_t> d_src;
    if ((rc = ig.d_stage.ensure(static_cast<size_t>(slab_rows) * e->dims, "rebalance bounce buffer")) ||
        (rc = incoming.ensure(static_cast<size_t>(std::min(slab_rows, n)) * e->dims, "rebalance staging")) ||
        (rc = d_src.ensure(static_cast<size_t>(slab_rows), "rebalance sources")))
        return rc;
    uint64_t keys_from = f;
    if (e->d_keys.cap < m) {                   // the last allocation: the whole key column is uploaded below
        if ((rc = e->d_keys.ensure(std::max<size_t>(m, e->cap_rows), "row keys"))) return rc;
        keys_from = 0;
    }
    tr.mark("grow+staging");

    std::vector<uint64_t> tags;
    for (uint64_t hi = total; hi > 0;) {
        const uint64_t lo = hi > slab_rows ? hi - slab_rows : 0, len = hi - lo;
        tags.assign(src.begin() + lo, src.begin() + hi);
        uint64_t jlo = ~0ull, jhi = 0;         // the incoming run this slab takes
        for (const uint64_t t : tags)
            if (t & kMergeIncoming) { jlo = std::min(jlo, t & ~kMergeIncoming); jhi = std::max(jhi, (t & ~kMergeIncoming) + 1); }
        if (jhi > jlo) {
            CUDA_TRY(cudaMemcpyPeerAsync(incoming, e->device, in.vectors() + jlo * e->dims, in.device(),
                                         (jhi - jlo) * row_bytes, ig.stream));
            for (uint64_t &t : tags) if (t & kMergeIncoming) t -= jlo;
        }
        CUDA_TRY(cudaMemcpyAsync(d_src, tags.data(), len * sizeof(uint64_t), cudaMemcpyHostToDevice, ig.stream));
        const unsigned grid = static_cast<unsigned>(std::min<uint64_t>(len, static_cast<uint64_t>(e->sm_count) * 32));
        merge_rows_kernel<<<grid, 128, 0, ig.stream>>>(ig.d_stage, e->d_corpus, incoming, d_src, len, e->dims);
        CUDA_TRY(cudaGetLastError());
        CUDA_TRY(cudaMemcpyAsync(e->d_corpus + (f + lo) * e->dims, ig.d_stage, len * row_bytes, cudaMemcpyDeviceToDevice,
                                 ig.stream));
        CUDA_TRY(cudaStreamSynchronize(ig.stream));          // tags / d_src / incoming are reused by the next slab
        hi = lo;
    }
    tr.mark("merge matrix");

    // The host columns in the same order.  A column set on one side only is materialised with the defaults the other
    // side's rows answered with: group = own frame id, attributes {0, 0}, no location, no terms.
    materialize_ids(e);
    auto merge = [&](auto &col, auto incoming_of) {
        auto tail = std::vector<typename std::decay_t<decltype(col)>::value_type>(total);
        for (uint64_t t = 0; t < total; ++t)
            tail[t] = (src[t] & kMergeIncoming) ? incoming_of(src[t] & ~kMergeIncoming) : col[src[t]];
        col.resize(f);
        col.insert(col.end(), tail.begin(), tail.end());
    };
    const uint32_t set = in.set();
    if ((set & WAX_VS_COLUMN_GROUPS) && !e->groups_set) { e->groups = e->ids; e->groups_set = true; }
    if ((set & WAX_VS_COLUMN_ATTRIBUTES) && !e->attrs_set) { e->attrs.assign(n0, AttrRow{0, 0}); e->attrs_set = true; }
    if ((set & WAX_VS_COLUMN_LOCATIONS) && !e->locs_set) { e->locs.assign(n0, LocRow{kNoLocation, 0}); e->locs_set = true; }
    if ((set & WAX_VS_COLUMN_TERMS) && !e->terms_set) {
        e->term_refs.assign(n0, wax_vs_engine::TermRef{0, 0});
        e->terms_set = true;
    }
    merge(e->ids, [&](uint64_t j) { return in.id(j); });
    merge(e->keys, [&](uint64_t j) { return in.key(j); });
    e->keys_set = true;
    if (e->groups_set) merge(e->groups, [&](uint64_t j) { return (set & WAX_VS_COLUMN_GROUPS) ? in.group(j) : in.id(j); });
    if (e->attrs_set) merge(e->attrs, [&](uint64_t j) { return (set & WAX_VS_COLUMN_ATTRIBUTES) ? in.attr(j) : AttrRow{0, 0}; });
    if (e->locs_set)
        merge(e->locs, [&](uint64_t j) { return (set & WAX_VS_COLUMN_LOCATIONS) ? in.loc(j) : LocRow{kNoLocation, 0}; });
    if (e->terms_set)
        merge(e->term_refs, [&](uint64_t j) {
            if (!(set & WAX_VS_COLUMN_TERMS)) return wax_vs_engine::TermRef{0, 0};
            const TermList t = in.terms(j);
            if (t.n == 0) return wax_vs_engine::TermRef{0, 0};
            const uint64_t off = e->term_pool.size();
            e->term_pool.insert(e->term_pool.end(), t.p, t.p + t.n);
            return wax_vs_engine::TermRef{off, t.n};
        });
    e->n_rows = m;
    e->ids_sorted = std::is_sorted(e->ids.begin(), e->ids.end());   // distinct ids: sorted = increasing
    e->map_valid = false;
    e->d_ids_dirty = true;
    invalidate_row_caches(e, f);
    rc = upload_row_keys(e, keys_from);
    tr.mark("merge columns");
    return rc;
}
}  // extern "C++"

// Rows [first, first + n) of `donor`, another engine of this process, merge into `e` (multi_rebalance).  The donor is
// only read; the caller drops the rows from it afterwards.
static int32_t absorb_rows(wax_vs_engine *e, wax_vs_engine *donor, uint64_t first, uint64_t n) {
    if (n == 0) return WAX_VS_OK;
    std::unique_lock<std::shared_mutex> w(e->rw);
    std::shared_lock<std::shared_mutex> donor_lock(donor->rw);
    if (!donor->keys_set || first + n > donor->n_rows || (!e->keys_set && e->n_rows))
        return fail(WAX_VS_ERR_ARGUMENT, "rebalance: rows [%llu, +%llu) of a keyed shard expected",
                    static_cast<unsigned long long>(first), static_cast<unsigned long long>(n));
    return absorb_body(e, DonorRows{donor, first, n});
}

int32_t wax_vs_absorb_rows(wax_vs_engine *e, const uint64_t *frame_ids, const uint64_t *keys, const float *d_vectors,
                           uint64_t n, uint32_t columns_set, const wax_vs_row_columns *columns,
                           const uint64_t *term_offsets, const uint64_t *terms) {
    WAX_VS_MULTI_REFUSE(e, "wax_vs_absorb_rows");
    if (!e) return fail(WAX_VS_ERR_NULL, "engine is NULL");
    if (n == 0) return WAX_VS_OK;
    if (!frame_ids || !keys || !d_vectors) return fail(WAX_VS_ERR_NULL, "NULL argument");
    const uint32_t all = WAX_VS_COLUMN_GROUPS | WAX_VS_COLUMN_ATTRIBUTES | WAX_VS_COLUMN_LOCATIONS | WAX_VS_COLUMN_TERMS;
    if (columns_set & ~all) return fail(WAX_VS_ERR_ARGUMENT, "absorb_rows: unknown column bits 0x%x", columns_set & ~all);
    if ((columns_set & (WAX_VS_COLUMN_GROUPS | WAX_VS_COLUMN_ATTRIBUTES | WAX_VS_COLUMN_LOCATIONS)) && !columns)
        return fail(WAX_VS_ERR_NULL, "columns is NULL");
    if ((columns_set & WAX_VS_COLUMN_TERMS) && !term_offsets) return fail(WAX_VS_ERR_NULL, "term_offsets is NULL");
    if ((columns_set & WAX_VS_COLUMN_TERMS) && term_offsets[n] && !terms) return fail(WAX_VS_ERR_NULL, "terms is NULL");
    for (uint64_t j = 1; j < n; ++j)
        if (keys[j] <= keys[j - 1])
            return fail(WAX_VS_ERR_ARGUMENT, "absorb_rows: keys must strictly increase (row %llu)",
                        static_cast<unsigned long long>(j));
    if (columns_set & WAX_VS_COLUMN_TERMS) {
        if (term_offsets[0] != 0) return fail(WAX_VS_ERR_ARGUMENT, "absorb_rows: term_offsets[0] must be 0");
        for (uint64_t j = 0; j < n; ++j) {
            if (term_offsets[j + 1] < term_offsets[j] || term_offsets[j + 1] - term_offsets[j] > 0xFFFFFFFFull)
                return fail(WAX_VS_ERR_ARGUMENT, "absorb_rows: term_offsets must not decrease (row %llu)",
                            static_cast<unsigned long long>(j));
            for (uint64_t t = term_offsets[j] + 1; t < term_offsets[j + 1]; ++t)
                if (terms[t] <= terms[t - 1])
                    return fail(WAX_VS_ERR_ARGUMENT, "absorb_rows: row %llu's terms must strictly increase",
                                static_cast<unsigned long long>(j));
        }
    }
    {
        std::vector<uint64_t> sorted(frame_ids, frame_ids + n);
        std::sort(sorted.begin(), sorted.end());
        const auto dup = std::adjacent_find(sorted.begin(), sorted.end());
        if (dup != sorted.end())
            return fail(WAX_VS_ERR_ARGUMENT, "absorb_rows: frame %llu appears twice", static_cast<unsigned long long>(*dup));
    }
    cudaPointerAttributes attr{};
    if (cudaPointerGetAttributes(&attr, d_vectors) != cudaSuccess || attr.type != cudaMemoryTypeDevice ||
        attr.device != e->device) {
        cudaGetLastError();
        return fail(WAX_VS_ERR_ARGUMENT, "absorb_rows: d_vectors is not memory on the engine's device %d", e->device);
    }
    std::unique_lock<std::shared_mutex> w(e->rw);
    if (!e->keys_set && e->n_rows) return fail(WAX_VS_ERR_ARGUMENT, "absorb_rows: the engine holds rows without keys");
    for (uint64_t j = 0; j < n; ++j)
        if (std::binary_search(e->keys.begin(), e->keys.end(), keys[j]))
            return fail(WAX_VS_ERR_ARGUMENT, "absorb_rows: key %llu is already held", static_cast<unsigned long long>(keys[j]));
    for (uint64_t j = 0; j < n; ++j)
        if (row_of(e, frame_ids[j]) != 0xFFFFFFFFu)
            return fail(WAX_VS_ERR_ARGUMENT, "absorb_rows: frame %llu is already held",
                        static_cast<unsigned long long>(frame_ids[j]));
    return absorb_body(e, CallerRows{frame_ids, keys, d_vectors, e->device, n, columns_set, columns, term_offsets, terms});
}

int32_t wax_vs_rebalance(wax_vs_engine *e, uint64_t *out_moved) {
    if (out_moved) *out_moved = 0;
    if (!e) return fail(WAX_VS_ERR_NULL, "engine is NULL");
    return e->multi ? multi_rebalance(e->multi, out_moved) : WAX_VS_OK;   // one engine has nothing to even out
}

// Filter level (level 2 of the batched path): for queries level 1 could not prove.  One TF32 tensor-core pass in
// FILTER form appends EVERY row whose score' beats the query's fixed threshold tau* (= exact k-th score of level 1's
// re-scored nominees - eps_tf32, so no true top-k row can be missing) to the query's candidate list; every candidate
// is re-scored exactly, the k best are the answer.  Complete by construction -- d_ok[i] = 0 only if a list
// overflowed (more than filter_cap rows within 2 eps of the k-th score: near-duplicates en masse).
// bf16 = true: the pass reads the bf16 shadow (half the bytes of the fp32 corpus; d_tau must then be the thresholds built
// with the bf16 bound, which admit more candidates); false: TF32 from the fp32 corpus.
static int32_t enqueue_filter_level(wax_vs_engine *e, SearchCtx *c, const float *d_queries, const float *d_tau,
                                    uint32_t n_queries, uint32_t k_eff, uint64_t row_offset, wax_vs_candidate *d_out,
                                    uint32_t *d_ok, const uint64_t *d_ids, cudaStream_t stream, uint64_t *launches,
                                    bool bf16 = false, const RowFilter &rf = RowFilter{}) {
    int32_t rc = ensure_norms(e, stream);
    if (rc) return rc;
    uint32_t cap = 64;                      // a power of two in [64, 16384], at least k
    while ((cap < static_cast<uint32_t>(std::max(e->tune.filter_cap, 64)) || cap < k_eff) && cap < 16384u) cap <<= 1;
    if ((rc = c->d_cand_count.ensure(static_cast<size_t>(n_queries), "filter counts"))) return rc;
    if ((rc = c->d_cand_rows.ensure(static_cast<size_t>(n_queries) * cap, "filter candidates"))) return rc;
    if ((rc = c->d_cand_keys.ensure(static_cast<size_t>(n_queries) * cap, "filter keys"))) return rc;
    CUDA_TRY(cudaMemsetAsync(c->d_cand_count, 0, static_cast<size_t>(n_queries) * sizeof(uint32_t), stream));
    auto prepare = [&](const NominateChunk &ch, BatchParams &bp) -> int32_t {
        bp.tau_fixed = d_tau + ch.q0;
        bp.cand_count = c->d_cand_count + ch.q0;
        bp.cand_rows = c->d_cand_rows + static_cast<size_t>(ch.q0) * cap;
        bp.cand_cap = cap;
        return WAX_VS_OK;
    };
    auto finish = [&](const NominateChunk &ch) -> int32_t {
        const uint32_t *count = c->d_cand_count + ch.q0;
        uint64_t *keys = c->d_cand_keys + static_cast<size_t>(ch.q0) * cap;
        const auto rescore = e->similarity == WAX_VS_COSINE ? filter_rescore_kernel<kCosine>
                             : e->similarity == WAX_VS_DOT  ? filter_rescore_kernel<kDot>
                                                            : filter_rescore_kernel<kL2>;
        rescore<<<dim3(32, ch.nq), 256, 0, stream>>>(e->d_corpus, ch.queries, e->dims, count,
                                                     c->d_cand_rows + static_cast<size_t>(ch.q0) * cap, cap, keys);
        CUDA_TRY(cudaGetLastError());
        FilterSelectParams sp{};
        sp.cand_count = count; sp.keys = keys; sp.cand_cap = cap; sp.k = k_eff;
        sp.out = d_out + static_cast<size_t>(ch.q0) * k_eff; sp.ok = d_ok + ch.q0;
        sp.frame_ids = d_ids; sp.id_base = e->id_base; sp.row_offset = row_offset; sp.row_keys = c->row_keys;
        const size_t ssmem = static_cast<size_t>(cap) * sizeof(uint64_t);
        CUDA_TRY(grant_smem(e, filter_select_kernel, ssmem));
        filter_select_kernel<<<ch.nq, 1024, ssmem, stream>>>(sp);
        CUDA_TRY(cudaGetLastError());
        *launches += 2;
        return WAX_VS_OK;
    };
    return enqueue_nominate_pass(e, c, d_queries, n_queries, bf16, true, false, false, static_cast<uint32_t>(e->sm_count),
                                 rf, stream, launches, [](uint32_t, uint32_t) { return 16u; }, prepare, finish);
}

// ---- search ---------------------------------------------------------------------------------------------------
// The exact scan for n queries, one enqueue_search each on `stream`: query i (qs[i] when a list is given) reads
// d_queries[i], writes d_out[i] and consults its own row filter.  sync_on_error: drain the stream before a failure is
// returned.  shadow_route: see enqueue_search (never for the exact fall-backs of the batched levels).
static int32_t enqueue_scans(wax_vs_engine *e, SearchCtx *c, const float *d_queries, uint32_t n, const uint32_t *qs,
                             uint32_t k_eff, uint64_t row_offset, wax_vs_candidate *d_out, const uint64_t *d_ids,
                             cudaStream_t stream, uint64_t *launches, const RowFilter &rf, bool sync_on_error,
                             bool shadow_route = false) {
    for (uint32_t i = 0; i < n; ++i) {
        const uint32_t qi = qs ? qs[i] : i;
        const int32_t rc = enqueue_search(e, c, d_queries + static_cast<size_t>(qi) * e->dims, k_eff, row_offset,
                                          d_out + static_cast<size_t>(qi) * k_eff, d_ids, stream, launches, rf.mask(qi),
                                          nullptr, nullptr, false, shadow_route);
        if (rc) {
            if (sync_on_error) cudaStreamSynchronize(stream);
            return rc;
        }
    }
    return WAX_VS_OK;
}

// n_queries device-resident queries -> d_out[n_queries][k_eff] on c->stream: the tensor-core levels (bf16 shadow ->
// TF32 retry -> exact scan, DESIGN 4.5.1) when the batch is eligible, else one fused scan per query.  The tensor
// levels read their proof flags back, so they synchronise c->stream; the scan loop only enqueues.  rf: the queries' row
// filters (every level consults each query's own bitset, so the proof is a statement about its ALLOWED rows).
static int32_t run_queries_on_device(wax_vs_engine *e, SearchCtx *c, const float *d_queries, uint32_t n_queries,
                                     uint32_t k_eff, uint64_t row_offset, wax_vs_candidate *d_out, const uint64_t *d_ids,
                                     uint64_t *launches, const RowFilter &rf = RowFilter{}) {
    int32_t rc = WAX_VS_OK;
    bool tensor_path = batch_tensor_eligible(e, n_queries, k_eff), allow_bf16 = true;
    if (tensor_path) {
        std::lock_guard<std::mutex> pg(e->pool_mu);
        if (e->bf16_skip_batches > 0) { --e->bf16_skip_batches; allow_bf16 = false; }
    }
    // below batch_min the tensor path only pays off through the bf16 shadow (single_shadow): never TF32 for one query
    if (tensor_path && !allow_bf16 && n_queries < static_cast<uint32_t>(std::max(e->tune.batch_min, 1))) tensor_path = false;
    if (!tensor_path)       // one query (or a few): each its own scan, through the shadow route where it applies
        return enqueue_scans(e, c, d_queries, n_queries, nullptr, k_eff, row_offset, d_out, d_ids, c->stream, launches, rf, true,
                             true);
    // Batched: one tensor-core pass over the corpus nominates, the finish kernel re-scores exactly and
    // proves completeness; unproven queries (rare) are re-run on the exact single-query path below.
    if ((rc = c->d_ok.ensure(static_cast<size_t>(n_queries), "proof flags"))) return rc;
    if ((rc = c->h_ok.ensure(static_cast<size_t>(n_queries), "proof flag staging"))) return rc;
    if ((rc = c->d_tau_star.ensure(static_cast<size_t>(n_queries) * 2, "filter thresholds"))) return rc;
    if ((rc = c->h_tau_star.ensure(static_cast<size_t>(n_queries) * 2, "filter threshold staging"))) return rc;
    bool used_bf16 = false;
    uint32_t used_heap = 0;
    rc = enqueue_batch_tensor(e, c, d_queries, n_queries, k_eff, row_offset, d_out, c->d_ok, d_ids, c->stream, launches,
                              allow_bf16, &used_bf16, c->d_tau_star, rf, &used_heap);
    if (rc) { cudaStreamSynchronize(c->stream); return rc; }
    CUDA_TRY(cudaMemcpyAsync(c->h_ok, c->d_ok, n_queries * sizeof(uint32_t), cudaMemcpyDeviceToHost, c->stream));
    CUDA_TRY(cudaMemcpyAsync(c->h_tau_star, c->d_tau_star, 2 * n_queries * sizeof(float), cudaMemcpyDeviceToHost, c->stream));
    CUDA_TRY(cudaStreamSynchronize(c->stream));
    std::vector<uint32_t> unproven;
    for (uint32_t qi = 0; qi < n_queries; ++qi) if (!c->h_ok[qi]) unproven.push_back(qi);
    if (used_bf16 && k_eff <= 128u) record_level1_outcome(e, n_queries, unproven.size(), used_heap);
    uint64_t retried = 0, retried_bf16 = 0;
    // Level 2, the filter levels: the unproven queries that have a finite threshold, as one compacted sub-batch, get
    // ONE more tensor-core pass that keeps no heap -- it lists every row above the query's fixed threshold (complete
    // by construction).  First over the bf16 shadow when level 1 used it (half the bytes of an exact scan, so it pays
    // even for a single query; its wider bound admits more candidates), then -- for the lists that overflowed, and
    // only for sub-batches worth a tensor pass -- in TF32 over the fp32 corpus.  What is left takes the exact scan.
    auto filter_pass = [&](std::vector<uint32_t> &todo, bool bf16lvl) -> int32_t {
        const uint32_t nf = static_cast<uint32_t>(todo.size());
        int32_t frc;
        if ((frc = c->d_retry_q.ensure(static_cast<size_t>(nf) * e->dims, "filter-level queries"))) return frc;
        if ((frc = c->d_retry_out.ensure(static_cast<size_t>(nf) * k_eff, "filter-level results"))) return frc;
        if ((frc = c->d_retry_ok.ensure(static_cast<size_t>(nf), "filter-level flags"))) return frc;
        if ((frc = c->d_filter_tau.ensure(static_cast<size_t>(nf), "filter-level thresholds"))) return frc;
        if ((frc = c->h_filter_tau.ensure(static_cast<size_t>(nf), "filter-level threshold staging"))) return frc;
        const float *taus = c->h_tau_star + (bf16lvl ? n_queries : 0u);      // [0]: TF32 bound, [1]: bf16 bound
        for (uint32_t i = 0; i < nf; ++i) c->h_filter_tau[i] = taus[todo[i]];
        CUDA_TRY(cudaMemcpyAsync(c->d_filter_tau, c->h_filter_tau, nf * sizeof(float), cudaMemcpyHostToDevice, c->stream));
        for (uint32_t i = 0; i < nf; ++i)
            CUDA_TRY(cudaMemcpyAsync(c->d_retry_q + static_cast<size_t>(i) * e->dims,
                                     d_queries + static_cast<size_t>(todo[i]) * e->dims, e->dims * sizeof(float),
                                     cudaMemcpyDeviceToDevice, c->stream));
        // per-query filters: the compacted queries keep their bitsets, in the same order
        RowFilter frf = rf;
        std::vector<uint32_t> retry_index;
        if (rf.h_index) {
            retry_index.resize(nf);
            for (uint32_t i = 0; i < nf; ++i) retry_index[i] = rf.h_index[todo[i]];
            if ((frc = c->d_retry_filter.ensure(nf, "filter-level filter indices"))) return frc;
            CUDA_TRY(cudaMemcpyAsync(c->d_retry_filter, retry_index.data(), nf * sizeof(uint32_t), cudaMemcpyHostToDevice,
                                     c->stream));
            frf.d_index = c->d_retry_filter;
            frf.h_index = retry_index.data();
        }
        frc = enqueue_filter_level(e, c, c->d_retry_q, c->d_filter_tau, nf, k_eff, row_offset, c->d_retry_out,
                                   c->d_retry_ok, d_ids, c->stream, launches, bf16lvl, frf);
        if (frc) { cudaStreamSynchronize(c->stream); return frc; }
        CUDA_TRY(cudaMemcpyAsync(c->h_ok, c->d_retry_ok, nf * sizeof(uint32_t), cudaMemcpyDeviceToHost, c->stream));
        CUDA_TRY(cudaStreamSynchronize(c->stream));
        std::vector<uint32_t> overflowed;
        for (uint32_t i = 0; i < nf; ++i) {
            if (c->h_ok[i])
                CUDA_TRY(cudaMemcpyAsync(d_out + static_cast<size_t>(todo[i]) * k_eff,
                                         c->d_retry_out + static_cast<size_t>(i) * k_eff, k_eff * sizeof(wax_vs_candidate),
                                         cudaMemcpyDeviceToDevice, c->stream));
            else
                overflowed.push_back(todo[i]);
        }
        todo.swap(overflowed);
        return WAX_VS_OK;
    };
    if (e->tune.batch_retry && !unproven.empty()) {
        std::vector<uint32_t> todo, rest;
        for (uint32_t qi : unproven)
            ((std::isfinite(c->h_tau_star[qi]) && std::isfinite(c->h_tau_star[n_queries + qi])) ? todo : rest).push_back(qi);
        if (!todo.empty() && used_bf16 && e->tune.filter_bf16) {
            retried_bf16 = todo.size();
            if ((rc = filter_pass(todo, true))) return rc;
        }
        if (todo.size() >= static_cast<size_t>(std::max(e->tune.batch_min, 1))) {
            retried = todo.size();
            if ((rc = filter_pass(todo, false))) return rc;
        }
        rest.insert(rest.end(), todo.begin(), todo.end());
        std::sort(rest.begin(), rest.end());
        unproven.swap(rest);
    }
    if ((rc = enqueue_scans(e, c, d_queries, static_cast<uint32_t>(unproven.size()), unproven.data(), k_eff, row_offset,
                            d_out, d_ids, c->stream, launches, rf, true)))
        return rc;
    std::lock_guard<std::mutex> pg(e->pool_mu);
    e->batch_tensor_queries += n_queries - unproven.size();
    e->batch_fallback_queries += unproven.size();
    if (used_bf16) e->batch_bf16_queries += n_queries;
    else e->batch_tf32_queries += n_queries;
    e->batch_retry_queries += retried;
    e->batch_filter_bf16_queries += retried_bf16;
    return WAX_VS_OK;
}

// n_queries x k_eff candidates -> frame ids and scores, query qi's at qi * out_stride; out_n[qi] = how many were valid.
// row -> frameId and distance -> score on the host, as MetalVectorEngine.swift:595-603 does.  Optional: order[j] = the
// query candidate list j belongs to, k_of[j] = how many of its k_eff slots were written.
static void deliver_results(const wax_vs_engine *e, const wax_vs_candidate *cands, uint32_t n_queries, uint32_t k_eff,
                            uint64_t *out_ids, float *out_scores, uint32_t out_stride, uint32_t *out_n,
                            const uint32_t *order = nullptr, const uint32_t *k_of = nullptr) {
    for (uint32_t j = 0; j < n_queries; ++j) {
        const uint32_t qi = order ? order[j] : j;
        const uint32_t kq = k_of ? k_of[j] : k_eff;
        uint32_t m = 0;
        for (uint32_t i = 0; i < kq; ++i) {
            const wax_vs_candidate &cd = cands[static_cast<size_t>(j) * k_eff + i];
            if (!cd.valid) continue;
            out_ids[static_cast<size_t>(qi) * out_stride + m] = frame_id_of(e, cd.row);
            out_scores[static_cast<size_t>(qi) * out_stride + m] = score_from_distance(e->similarity, cd.distance);
            ++m;
        }
        out_n[qi] = m;
    }
}

// The query argument of the host-path search entry points (validate, :449, :830-833).
static int32_t check_query(const wax_vs_engine *e, const float *query, uint32_t query_len) {
    if (!query) return fail(WAX_VS_ERR_NULL, "query is NULL");
    if (query_len != e->dims)
        return fail(WAX_VS_ERR_DIMENSION, "vector dimension mismatch: expected %u, got %u", e->dims, query_len);
    return WAX_VS_OK;
}

static int32_t search_host(wax_vs_engine *e, const float *queries, uint32_t n_queries, uint32_t query_len,
                           int64_t top_k, uint64_t *out_ids, float *out_scores, uint32_t out_stride,
                           uint32_t *out_n) {
    if (e && e->multi)
        return multi_search(e->multi, e->dims, e->similarity, queries, n_queries, query_len, top_k, out_ids, out_scores,
                            out_stride, out_n);
    if (!e || !out_n) return fail(WAX_VS_ERR_NULL, "NULL argument");
    std::shared_lock<std::shared_mutex> r(e->rw);
    if (e->n_rows == 0) {  // guard vectorCount > 0 else { return [] } (:448) -- before validation, as the reference
        for (uint32_t i = 0; i < n_queries; ++i) out_n[i] = 0;
        return WAX_VS_OK;
    }
    if (n_queries == 0) return WAX_VS_OK;
    int32_t rc;
    if ((rc = check_query(e, queries, query_len))) return rc;
    const uint32_t limit = clamp_topk(top_k);
    const uint32_t k_eff = static_cast<uint32_t>(std::min<uint64_t>(limit, e->n_rows));  // topKCount (:451)
    if (!out_ids || !out_scores) return fail(WAX_VS_ERR_NULL, "output buffer is NULL");
    if (out_stride < k_eff)
        return fail(WAX_VS_ERR_BUFFER, "output buffers hold %u entries, need %u", out_stride, k_eff);

    DeviceGuard g(e->device);
    if (!g.ok) return g.error();
    CtxLease lease(e);
    if ((rc = lease.acquire())) return rc;
    SearchCtx *c = lease.c;

    const size_t ncand = static_cast<size_t>(n_queries) * k_eff;
    if ((rc = c->d_out.ensure(ncand, "result buffer"))) return rc;
    if ((rc = c->h_out.ensure(ncand, "result staging"))) return rc;
    uint64_t launches = 0;
    bool delivered = false;
    // One query on the fused scan: the query rides in the kernel parameters and the kernel itself stores the result in
    // mapped host memory and raises a flag -- no H2D copy, no D2H copy, no stream synchronisation on the way.
    if (n_queries == 1 && e->tune.host_delivery && k_eff <= static_cast<uint32_t>(e->tune.fused_k_max) &&
        !batch_tensor_eligible(e, 1, k_eff)) {
        if (!c->h_flag) {
            if ((rc = c->h_flag.ensure(1, "completion flag"))) return rc;
            *c->h_flag = 0; c->host_seq = 0;
        }
        HostDelivery hd{queries, c->h_out, c->h_flag, ++c->host_seq};
        if ((rc = enqueue_search(e, c, nullptr, k_eff, 0, c->d_out, nullptr, c->stream, &launches, nullptr, nullptr, &hd,
                                 false, true))) {
            cudaStreamSynchronize(c->stream);
            return rc;
        }
        delivered = hd.delivered;
        if (delivered && (rc = wait_host_flag(c->stream, c->h_flag, hd.seq, 30ull * 1000 * 1000 * 1000)) != WAX_VS_OK) {
            cudaStreamSynchronize(c->stream);
            return rc > 0 ? fail(WAX_VS_ERR_CUDA, "search reported a device-side error") : rc;
        }
    } else {
        if ((rc = stage_queries(e, c, queries, n_queries, c->stream))) return rc;
        if ((rc = run_queries_on_device(e, c, c->d_queries, n_queries, k_eff, 0, c->d_out, nullptr, &launches))) return rc;
    }
    if (!delivered) {
        CUDA_TRY(cudaMemcpyAsync(c->h_out, c->d_out, ncand * sizeof(wax_vs_candidate), cudaMemcpyDeviceToHost, c->stream));
        CUDA_TRY(cudaStreamSynchronize(c->stream));
    }
    deliver_results(e, c->h_out, n_queries, k_eff, out_ids, out_scores, out_stride, out_n);
    return WAX_VS_OK;
}

int32_t wax_vs_search(wax_vs_engine *e, const float *query, uint32_t query_len, int64_t top_k,
                      uint64_t *out_ids, float *out_scores, uint32_t out_cap, uint32_t *out_n) {
    return search_host(e, query, 1, query_len, top_k, out_ids, out_scores, out_cap, out_n);
}

int32_t wax_vs_search_batch(wax_vs_engine *e, const float *queries, uint32_t n_queries, uint32_t query_len,
                            int64_t top_k, uint64_t *out_ids, float *out_scores, uint32_t out_stride,
                            uint32_t *out_n) {
    return search_host(e, queries, n_queries, query_len, top_k, out_ids, out_scores, out_stride, out_n);
}

int32_t wax_vs_search_device(wax_vs_engine *e, const float *d_queries, uint32_t n_queries, int64_t top_k,
                             uint64_t row_offset, wax_vs_candidate *d_candidates, void *cuda_stream) {
    WAX_VS_MULTI_REFUSE(e, "wax_vs_search_device");
    if (!e || !d_queries || !d_candidates) return fail(WAX_VS_ERR_NULL, "NULL argument");
    std::shared_lock<std::shared_mutex> r(e->rw);
    DeviceGuard g(e->device);
    if (!g.ok) return g.error();
    const uint32_t k_eff = clamp_topk(top_k);
    SearchCtx *c = nullptr;
    int32_t rc = ctx_for_stream(e, cuda_stream, &c);
    if (rc) return rc;
    e->async_pending.store(true);
    const uint64_t *d_ids = nullptr;
    if ((rc = sync_device_ids(e, &d_ids))) return rc;
    uint64_t launches = 0;
    return enqueue_scans(e, c, d_queries, n_queries, nullptr, k_eff, row_offset, d_candidates, d_ids,
                         static_cast<cudaStream_t>(cuda_stream), &launches, RowFilter{}, false, true);
}

// Batched form of wax_vs_search_device: the tensor-core levels on the caller's stream for the rank's shard.  Unlike
// the single-query form it may SYNCHRONISE the stream (the proof flags are read back before the unproven queries
// are re-run), so on return d_candidates is complete on `cuda_stream` order and usually already materialised.
int32_t wax_vs_search_batch_device(wax_vs_engine *e, const float *d_queries, uint32_t n_queries, int64_t top_k,
                                   uint64_t row_offset, wax_vs_candidate *d_candidates, void *cuda_stream) {
    WAX_VS_MULTI_REFUSE(e, "wax_vs_search_batch_device");
    if (!e || !d_queries || !d_candidates) return fail(WAX_VS_ERR_NULL, "NULL argument");
    if (n_queries == 0) return WAX_VS_OK;
    std::shared_lock<std::shared_mutex> r(e->rw);
    DeviceGuard g(e->device);
    if (!g.ok) return g.error();
    const uint32_t k_eff = clamp_topk(top_k);
    SearchCtx *c = nullptr;
    int32_t rc = ctx_for_stream(e, cuda_stream, &c);
    if (rc) return rc;
    e->async_pending.store(true);
    const uint64_t *d_ids = nullptr;
    if ((rc = sync_device_ids(e, &d_ids))) return rc;
    uint64_t launches = 0;
    if (k_eff > e->n_rows)     // a shard smaller than k: the scan pads with invalid candidates, the tensor path does not
        return enqueue_scans(e, c, d_queries, n_queries, nullptr, k_eff, row_offset, d_candidates, d_ids, c->stream,
                             &launches, RowFilter{}, false);
    return run_queries_on_device(e, c, d_queries, n_queries, k_eff, row_offset, d_candidates, d_ids, &launches);
}

// ---- filtered search (SURVEY.md section 8f-4) -------------------------------------------------------------------
// The reference filters AFTER the engine call and over-fetches 3 x topK to compensate (UnifiedSearch.swift:58,
// 371-442, 1195-1200, 1241-1258).  Here the filter is pushed below the top-k: a row bitset consulted only for rows
// that would enter the list, or -- for small allow-lists -- a gather that scores only the listed rows.
// frameIds -> the distinct rows of this engine they name, appended to `rows` (unknown and repeated ids are ignored).
// `seen` is a zeroed scratch bitset of ceil(N / 32) words shared by all the filters of a call: only the words this
// filter touched are cleared again, so no list is sorted and no bitset is rebuilt per filter.  Returns the rows appended.
static uint64_t build_row_filter(wax_vs_engine *e, const uint64_t *frame_ids, uint64_t n_ids, std::vector<uint32_t> &seen,
                                 std::vector<uint32_t> &rows) {
    const size_t first = rows.size();
    std::lock_guard<std::mutex> g(e->ids_mu);   // the lazily built id map is shared by concurrent readers
    // (row_of builds the lazily constructed hash table when it is needed: serialised by ids_mu)
    for (uint64_t i = 0; i < n_ids; ++i) {
        const uint32_t row = row_of(e, frame_ids[i]);
        if (row == 0xFFFFFFFFu) continue;
        const uint32_t w = row >> 5, b = 1u << (row & 31u);
        if (!(seen[w] & b)) { seen[w] |= b; rows.push_back(row); }
    }
    for (size_t i = first; i < rows.size(); ++i) seen[rows[i] >> 5] = 0u;
    return rows.size() - first;
}

// The filters of a call, resolved once: filter f's distinct rows are rows[first[f] .. first[f] + count[f]).
struct FilterSet {
    std::vector<uint32_t> rows;
    std::vector<uint64_t> first, count;
    std::vector<uint8_t> referenced;            // filters some query names (the others are not resolved)
    // Where search only (empty otherwise): filter f's bitset is ANDed with preds[where[f]] (its slot unused) unless that
    // is WAX_VS_NO_FILTER, and then allows allowed[f] rows; the rows of the filters in `compact` (device_rows in all) are
    // listed by the device after `rows`, each item's slot being where its rows start.  Every item carries its box.
    std::vector<uint32_t> where;
    std::vector<uint64_t> allowed;
    std::vector<WhereFull> preds, compact;
    uint64_t device_rows = 0;
    // Where_terms search only (plan_term_units): the narrow term units, whose rows the device lists at their slots after
    // the compact rows, and the wide ones, whose rows the device sets in their filter's bitset; term_of[f] = filter f's
    // wide unit in term_wide (empty, or WAX_VS_NO_FILTER, when it has none: its rows are the listed ones).
    std::vector<TermUnitR> term_list, term_wide;
    std::vector<uint32_t> term_of;
    // Where_groups search only (plan_group_units): filter f's group unit is group_units[group_of[f]] (empty, or
    // WAX_VS_NO_FILTER, when it has none).  A unit of <= kWhereGatherRows rows (fs.count[f]) is listed by the device at its
    // slot after the term units' rows; a wider one gets its bits set in its filter's bitset.
    std::vector<GroupUnitR> group_units;
    std::vector<uint32_t> group_of;
};
// query_filter = nullptr: every filter is resolved (the single-filter entry points).
static void resolve_filters(wax_vs_engine *e, const uint64_t *frame_ids, const uint64_t *filter_offsets, uint32_t n_filters,
                            const uint32_t *query_filter, uint32_t n_queries, FilterSet &fs) {
    fs.first.assign(n_filters, 0);
    fs.count.assign(n_filters, 0);
    fs.referenced.assign(n_filters, query_filter ? 0 : 1);
    for (uint32_t i = 0; i < n_queries; ++i)
        if (query_filter[i] != WAX_VS_NO_FILTER) fs.referenced[query_filter[i]] = 1;
    std::vector<uint32_t> seen(static_cast<size_t>((e->n_rows + 31) / 32), 0u);
    for (uint32_t f = 0; f < n_filters; ++f) {
        if (!fs.referenced[f]) continue;
        fs.first[f] = fs.rows.size();
        fs.count[f] = build_row_filter(e, frame_ids + filter_offsets[f], filter_offsets[f + 1] - filter_offsets[f], seen, fs.rows);
    }
}

// n_filters row bitsets of ceil(N / 32) words into c->d_mask on `stream`, from the resolved rows in c->d_filter_rows:
// spec is filter_bits_init_kernel's (running row counts, where each filter's rows start, modes).  The host uploads
// 4 bytes per listed row instead of N / 8 bytes per filter.  c->d_mask must not be reallocated while earlier
// launches on `stream` still read it: callers size it first.
static int32_t build_filter_bits(wax_vs_engine *e, SearchCtx *c, const std::vector<uint64_t> &spec, uint32_t n_filters,
                                 cudaStream_t stream, uint64_t *launches) {
    const uint32_t words = static_cast<uint32_t>((e->n_rows + 31) / 32);
    int32_t rc;
    if ((rc = c->d_filter_spec.ensure(spec.size(), "filter spec"))) return rc;
    if ((rc = c->d_mask.ensure(static_cast<size_t>(n_filters) * words, "row filters"))) return rc;
    CUDA_TRY(cudaMemcpyAsync(c->d_filter_spec, spec.data(), spec.size() * sizeof(uint64_t), cudaMemcpyHostToDevice, stream));
    const size_t total_words = static_cast<size_t>(n_filters) * words;
    const int cap = e->sm_count * 8;
    const int g1 = static_cast<int>(std::min<size_t>(cap, (total_words + 255) / 256));
    filter_bits_init_kernel<<<std::max(g1, 1), 256, 0, stream>>>(c->d_mask, words, static_cast<uint32_t>(e->n_rows),
                                                                 c->d_filter_spec, n_filters);
    CUDA_TRY(cudaGetLastError());
    ++*launches;
    const uint64_t listed = spec[n_filters];
    if (listed) {
        const int g2 = static_cast<int>(std::min<uint64_t>(cap, (listed + 255) / 256));
        filter_bits_apply_kernel<<<g2, 256, 0, stream>>>(c->d_mask, words, c->d_filter_rows, c->d_filter_spec, n_filters);
        CUDA_TRY(cudaGetLastError());
        ++*launches;
    }
    return WAX_VS_OK;
}
// The resolved rows into c->d_filter_rows on `stream`, after growing it to at least `reserve` rows; `rows` must outlive
// the copy.  mode 0 (allow) / 1 (deny): also the bitset of `rows` as the one filter, into c->d_mask.
static int32_t stage_filter_rows(wax_vs_engine *e, SearchCtx *c, const std::vector<uint32_t> &rows, size_t reserve,
                                 int32_t mode, cudaStream_t stream, uint64_t *launches) {
    int32_t rc;
    if ((rc = c->d_filter_rows.ensure(std::max<size_t>(reserve, 1), "filter rows"))) return rc;
    if (!rows.empty())
        CUDA_TRY(cudaMemcpyAsync(c->d_filter_rows, rows.data(), rows.size() * sizeof(uint32_t), cudaMemcpyHostToDevice, stream));
    if (mode < 0) return WAX_VS_OK;
    return build_filter_bits(e, c, {0, rows.size(), 0, static_cast<uint64_t>(mode)}, 1, stream, launches);
}

// ---- row-sharded search: fused scan + NVLink exchange + merge (waxvs_shard.cuh; SURVEY.md section 8e) ---------------
// Handle blob exchanged between the ranks (WAX_VS_SHARD_HANDLE_BYTES): how a peer reaches this rank's mailbox.
struct ShardHandle {
    uint32_t magic, version;
    int32_t pid, device;
    uint64_t nonce;                  // per-process random: same (pid, nonce) = same process -> plain peer access
    uint64_t ptr;                    // mailbox device pointer (valid in the owning process)
    int32_t rank, world;
    cudaIpcMemHandle_t ipc;          // 64 bytes: for other processes on the node
    uint8_t pad[WAX_VS_SHARD_HANDLE_BYTES - 40 - sizeof(cudaIpcMemHandle_t)];
};
static_assert(sizeof(ShardHandle) == WAX_VS_SHARD_HANDLE_BYTES, "handle blob size");
static uint64_t process_nonce() {
    static const uint64_t n = [] { std::random_device rd; return (static_cast<uint64_t>(rd()) << 32) ^ rd() ^ 0x9E3779B97F4A7C15ull; }();
    return n;
}

// Caller holds the write lock, device selected.  Two steps because other PROCESSES may still have this rank's mailbox
// mapped: wax_vs_shard_close only unmaps the peers' mailboxes (free_own = false); the own mailbox is released when the
// engine is destroyed or re-opened, i.e. after the group has agreed (a barrier on the caller's side) that everyone
// has closed.
static void shard_teardown(wax_vs_engine *e, bool free_own) {
    auto &sh = e->shard;
    if (!sh.open) return;
    cudaDeviceSynchronize();
    for (int r = 0; r < sh.world; ++r) {
        if (r != sh.rank && sh.ipc[r] && sh.box[r]) cudaIpcCloseMemHandle(sh.box[r]);
        sh.ipc[r] = false;
        if (r != sh.rank) sh.box[r] = nullptr;
    }
    sh.connected = false;
    cudaGetLastError();
    if (!free_own) return;
    if (sh.box[sh.rank]) cudaFree(sh.box[sh.rank]);
    sh.box[sh.rank] = nullptr;
    delete sh.ctx;             // the result buffers stay with the engine: a re-open reuses them
    sh.ctx = nullptr;
    cudaGetLastError();
    sh.open = false;
    sh.seq = 0;
}

int32_t wax_vs_shard_open(wax_vs_engine *e, int32_t rank, int32_t world, uint64_t row_offset, uint8_t *out_handle) {
    WAX_VS_MULTI_REFUSE(e, "wax_vs_shard_open");
    if (!e || !out_handle) return fail(WAX_VS_ERR_NULL, "NULL argument");
    if (world < 1 || world > kShardMaxRanks || rank < 0 || rank >= world)
        return fail(WAX_VS_ERR_ARGUMENT, "rank %d of %d: world must be 1..%d", rank, world, kShardMaxRanks);
    std::unique_lock<std::shared_mutex> w(e->rw);
    DeviceGuard g(e->device);
    if (!g.ok) return g.error();
    drain_device_path(e);
    shard_teardown(e, true);
    auto &sh = e->shard;
    ShardMailbox *box = nullptr;
    CUDA_TRY(cudaMalloc(&box, sizeof(ShardMailbox)));
    int32_t rc = sh.d_final.ensure(kShardKCap, "shard result");
    if (!rc) rc = sh.h_final.ensure(kShardKCap, "shard result delivery");
    if (!rc) rc = sh.h_flag.ensure(1, "shard completion flag");
    if (rc) { cudaFree(box); return rc; }
    cudaError_t err = cudaMemset(box, 0, sizeof(ShardMailbox));
    if (err == cudaSuccess) err = cudaDeviceSynchronize();
    ShardHandle h{};
    if (err == cudaSuccess) err = cudaIpcGetMemHandle(&h.ipc, box);
    if (err != cudaSuccess) {
        cudaFree(box);
        return fail(WAX_VS_ERR_CUDA, "failed to create the shard mailbox: %s", cudaGetErrorString(err));
    }
    *sh.h_flag = 0;
    if ((rc = ctx_new(e, &sh.ctx, true))) { cudaFree(box); return rc; }
    sh.rank = rank; sh.world = world; sh.row_offset = row_offset;
    sh.box[rank] = box;
    sh.open = true; sh.connected = (world == 1);
    sh.seq = 0;
    h.magic = 0x48535857u; h.version = 1; h.pid = static_cast<int32_t>(getpid()); h.device = e->device;
    h.nonce = process_nonce(); h.ptr = reinterpret_cast<uint64_t>(box); h.rank = rank; h.world = world;
    memcpy(out_handle, &h, sizeof h);
    return WAX_VS_OK;
}

int32_t wax_vs_shard_connect(wax_vs_engine *e, const uint8_t *handles, int32_t n_handles) {
    WAX_VS_MULTI_REFUSE(e, "wax_vs_shard_connect");
    if (!e || !handles) return fail(WAX_VS_ERR_NULL, "NULL argument");
    std::unique_lock<std::shared_mutex> w(e->rw);
    auto &sh = e->shard;
    if (!sh.open) return fail(WAX_VS_ERR_ARGUMENT, "wax_vs_shard_open has not been called");
    if (n_handles != sh.world) return fail(WAX_VS_ERR_ARGUMENT, "expected %d handles, got %d", sh.world, n_handles);
    DeviceGuard g(e->device);
    if (!g.ok) return g.error();
    for (int r = 0; r < sh.world; ++r) {
        ShardHandle h;
        memcpy(&h, handles + static_cast<size_t>(r) * sizeof h, sizeof h);
        if (h.magic != 0x48535857u || h.version != 1 || h.rank != r || h.world != sh.world)
            return fail(WAX_VS_ERR_ARGUMENT, "handle %d is not rank %d of %d", r, r, sh.world);
        if (r == sh.rank) continue;
        if (h.pid == static_cast<int32_t>(getpid()) && h.nonce == process_nonce()) {
            // same process (several engines in one host process): plain peer access to the other device
            if (h.device != e->device) {
                int can = 0;
                CUDA_TRY(cudaDeviceCanAccessPeer(&can, e->device, h.device));
                if (!can) return fail(WAX_VS_ERR_UNSUPPORTED, "device %d cannot access device %d (no P2P path)", e->device, h.device);
                cudaError_t pe = cudaDeviceEnablePeerAccess(h.device, 0);
                if (pe != cudaSuccess && pe != cudaErrorPeerAccessAlreadyEnabled)
                    return fail(WAX_VS_ERR_CUDA, "cudaDeviceEnablePeerAccess(%d) failed: %s", h.device, cudaGetErrorString(pe));
                cudaGetLastError();
            }
            sh.box[r] = reinterpret_cast<ShardMailbox *>(h.ptr);
            sh.ipc[r] = false;
        } else {
            void *ptr = nullptr;
            cudaError_t ie = cudaIpcOpenMemHandle(&ptr, h.ipc, cudaIpcMemLazyEnablePeerAccess);
            if (ie != cudaSuccess) {
                cudaGetLastError();
                return fail(WAX_VS_ERR_UNSUPPORTED, "cudaIpcOpenMemHandle for rank %d failed: %s (no P2P/IPC path between the ranks)",
                            r, cudaGetErrorString(ie));
            }
            sh.box[r] = static_cast<ShardMailbox *>(ptr);
            sh.ipc[r] = true;
        }
    }
    sh.connected = true;
    return WAX_VS_OK;
}

int32_t wax_vs_shard_close(wax_vs_engine *e) {
    WAX_VS_MULTI_REFUSE(e, "wax_vs_shard_close");
    if (!e) return fail(WAX_VS_ERR_NULL, "engine is NULL");
    std::unique_lock<std::shared_mutex> w(e->rw);
    DeviceGuard g(e->device);
    shard_teardown(e, false);
    return WAX_VS_OK;
}

// caller holds e->shard.mu: the next collective sequence number and the parameter block that goes with it
static ShardParams shard_params_next(wax_vs_engine *e) {
    auto &sh = e->shard;
    ShardParams sp{};
    for (int r = 0; r < sh.world; ++r) sp.box[r] = sh.box[r];
    sp.rank = static_cast<uint32_t>(sh.rank); sp.world = static_cast<uint32_t>(sh.world);
    sp.seq = ++sh.seq;
    sp.timeout_ns = sh.timeout_ns;
    return sp;
}

int32_t wax_vs_shard_search_device(wax_vs_engine *e, const float *d_query, int64_t top_k, wax_vs_candidate *d_candidates,
                                   void *cuda_stream) {
    WAX_VS_MULTI_REFUSE(e, "wax_vs_shard_search_device");
    if (!e || !d_query || !d_candidates) return fail(WAX_VS_ERR_NULL, "NULL argument");
    std::shared_lock<std::shared_mutex> r(e->rw);
    if (!e->shard.connected) return fail(WAX_VS_ERR_ARGUMENT, "the shard group is not connected (wax_vs_shard_open / _connect)");
    DeviceGuard g(e->device);
    if (!g.ok) return g.error();
    const uint32_t k_eff = clamp_topk(top_k);
    if (k_eff > static_cast<uint32_t>(kShardKCap))
        return fail(WAX_VS_ERR_UNSUPPORTED, "sharded search supports top_k <= %d (got %u)", kShardKCap, k_eff);
    SearchCtx *c = nullptr;
    int32_t rc = ctx_for_stream(e, cuda_stream, &c);
    if (rc) return rc;
    e->async_pending.store(true);
    const uint64_t *d_ids = nullptr;
    if ((rc = sync_device_ids(e, &d_ids))) return rc;
    std::lock_guard<std::mutex> sg(e->shard.mu);
    ShardParams sp = shard_params_next(e);
    uint64_t launches = 0;
    return enqueue_search(e, c, d_query, k_eff, e->shard.row_offset, d_candidates, d_ids,
                          static_cast<cudaStream_t>(cuda_stream), &launches, nullptr, &sp);
}

static int32_t shard_wait_host(wax_vs_engine *e, unsigned long long seq) {
    int32_t rc = wait_host_flag(e->shard.ctx->stream, e->shard.h_flag, seq, e->shard.timeout_ns);
    if (rc == 1)
        return fail(WAX_VS_ERR_CUDA, "shard exchange timed out: a peer rank did not deliver its candidates for query #%llu", seq);
    return rc;
}

static int32_t shard_search_host(wax_vs_engine *e, const SearchRequest &req, uint64_t *out_ids, float *out_scores,
                                 uint32_t out_cap, uint32_t *out_n);

int32_t wax_vs_shard_search(wax_vs_engine *e, const float *query, uint32_t query_len, int64_t top_k, uint64_t *out_ids,
                            float *out_scores, uint32_t out_cap, uint32_t *out_n) {
    WAX_VS_MULTI_REFUSE(e, "wax_vs_shard_search");
    if (!e || !out_n) return fail(WAX_VS_ERR_NULL, "NULL argument");
    const SearchRequest req(query, 1, query_len, top_k);
    return shard_search_host(e, req, out_ids, out_scores, out_cap, out_n);
}

// Device-timed sharded searches, strictly one query at a time on one stream (the same mode as wax_vs_debug_time_search):
// `n_queries` unit queries generated on device from generator stream `seed` (identical on every rank), warmup + iters
// collective searches back to back, CUDA events around the `iters`.  Every rank must make the same call.
int32_t wax_vs_debug_time_shard_search(wax_vs_engine *e, uint32_t n_queries, int64_t top_k, uint64_t seed, uint32_t warmup,
                                       uint32_t iters, float *out_ms_total, uint64_t *out_launches) {
    WAX_VS_MULTI_REFUSE(e, "wax_vs_debug_time_shard_search");
    if (!e || !out_ms_total) return fail(WAX_VS_ERR_NULL, "NULL argument");
    if (n_queries == 0) n_queries = 1;
    std::shared_lock<std::shared_mutex> r(e->rw);
    if (!e->shard.connected) return fail(WAX_VS_ERR_ARGUMENT, "the shard group is not connected (wax_vs_shard_open / _connect)");
    DeviceGuard g(e->device);
    auto &sh = e->shard;
    std::lock_guard<std::mutex> sg(sh.mu);
    SearchCtx *c = sh.ctx;
    c->row_keys = device_row_keys(e);
    const uint32_t k_eff = clamp_topk(top_k);
    int32_t rc;
    if ((rc = c->d_queries.ensure(static_cast<size_t>(n_queries) * e->dims, "query buffer"))) return rc;
    synth_fill_kernel<<<(n_queries + 255) / 256, 256, 0, c->stream>>>(c->d_queries, n_queries, e->dims, seed, 0, 1);
    CUDA_TRY(cudaGetLastError());
    const uint64_t *d_ids = nullptr;
    if ((rc = sync_device_ids(e, &d_ids))) return rc;
    uint64_t launches = 0;
    for (uint32_t it = 0; it < warmup + iters; ++it) {
        if (it == warmup) { launches = 0; CUDA_TRY(cudaEventRecord(c->ev0, c->stream)); }
        ShardParams sp = shard_params_next(e);
        rc = enqueue_search(e, c, c->d_queries + static_cast<size_t>(it % n_queries) * e->dims, k_eff, sh.row_offset,
                            sh.d_final, d_ids, c->stream, &launches, nullptr, &sp);
        if (rc) { cudaStreamSynchronize(c->stream); return rc; }
    }
    CUDA_TRY(cudaEventRecord(c->ev1, c->stream));
    CUDA_TRY(cudaStreamSynchronize(c->stream));
    CUDA_TRY(cudaEventElapsedTime(out_ms_total, c->ev0, c->ev1));
    if (out_launches) *out_launches = launches;
    return WAX_VS_OK;
}

// Device-side merge of all-gathered per-rank candidate lists (the sharded search_batch): stateless, enqueued on the
// caller's stream, no synchronisation.
int32_t wax_vs_merge_candidates_device(wax_vs_engine *e, const wax_vs_candidate *d_gathered, uint32_t world,
                                       uint32_t n_queries, uint32_t k, uint32_t k_out, wax_vs_candidate *d_out,
                                       void *cuda_stream) {
    WAX_VS_MULTI_REFUSE(e, "wax_vs_merge_candidates_device");
    if (!e || !d_gathered || !d_out) return fail(WAX_VS_ERR_NULL, "NULL argument");
    if (world == 0 || world > 1024u || k == 0 || k_out == 0 || k_out > k)
        return fail(WAX_VS_ERR_ARGUMENT, "merge: world %u, k %u, k_out %u", world, k, k_out);
    if (n_queries == 0) return WAX_VS_OK;
    DeviceGuard g(e->device);
    if (!g.ok) return g.error();
    merge_gathered_kernel<<<n_queries, 128, 0, static_cast<cudaStream_t>(cuda_stream)>>>(
        GatheredLists<wax_vs_candidate>{d_gathered, static_cast<size_t>(n_queries) * k}, world, n_queries, k, k_out, d_out);
    CUDA_TRY(cudaGetLastError());
    return WAX_VS_OK;
}

// ---- frame attributes on the device (waxvs_where.cuh) --------------------------------------------------------------
// The attribute mirror of the current corpus, built on c's stream by the first search after a mutation or
// set_attributes that needs it; with `locations`, the location mirror too (after a mutation or set_locations).  Readers
// hold the read lock; attrs_mu serialises the builds, each of which completes before its mirror is published.
static int32_t ensure_locations(wax_vs_engine *e, SearchCtx *c) {
    if (e->locs_dev_valid) return WAX_VS_OK;
    const size_t n = static_cast<size_t>(e->n_rows);
    int32_t rc;
    if ((rc = e->d_locs.ensure(std::max<size_t>(n, 1), "row locations"))) return rc;
    const std::vector<LocRow> none(e->locs_set ? 0 : n, LocRow{kNoLocation, 0});            // never set: no row has one
    CUDA_TRY(cudaMemcpyAsync(e->d_locs, e->locs_set ? e->locs.data() : none.data(), n * sizeof(LocRow),
                             cudaMemcpyHostToDevice, c->stream));
    CUDA_TRY(cudaStreamSynchronize(c->stream));
    e->locs_dev_valid = true;
    std::lock_guard<std::mutex> pg(e->pool_mu);
    ++e->location_uploads;
    return WAX_VS_OK;
}
static int32_t ensure_attributes(wax_vs_engine *e, SearchCtx *c, bool locations = false) {
    std::lock_guard<std::mutex> lk(e->attrs_mu);
    int32_t rc;
    if (locations && (rc = ensure_locations(e, c))) return rc;
    if (e->attrs_dev_valid) return WAX_VS_OK;
    const size_t n = static_cast<size_t>(e->n_rows);
    if ((rc = e->d_attrs.ensure(std::max<size_t>(n, 1), "row attributes"))) return rc;
    if (e->attrs_set) CUDA_TRY(cudaMemcpyAsync(e->d_attrs, e->attrs.data(), n * sizeof(AttrRow), cudaMemcpyHostToDevice, c->stream));
    else CUDA_TRY(cudaMemsetAsync(e->d_attrs, 0, n * sizeof(AttrRow), c->stream));    // never set: timestamp 0, tags 0
    CUDA_TRY(cudaStreamSynchronize(c->stream));
    e->attrs_dev_valid = true;
    std::lock_guard<std::mutex> pg(e->pool_mu);
    ++e->attribute_uploads;
    return WAX_VS_OK;
}

// The term index of the current corpus and term lists (waxvs_terms.cuh), built on c's stream by the first where_terms
// search after a mutation or set_terms: the (term, row) pairs in row order, radix-sorted by term with CUB (stable, so
// each posting list stays in ascending row order), the heads flagged and prefix-summed into term_keys / term_start.  The
// sort takes an int item count (as the group index's), so more than 2^31 - 1 pairs is refused.  Readers hold the read
// lock; term_mu serialises the build, which completes before the index is published.
static int32_t ensure_term_index(wax_vs_engine *e, SearchCtx *c) {
    std::lock_guard<std::mutex> lk(e->term_mu);
    auto &ti = e->tindex;
    if (ti.valid) return WAX_VS_OK;
    uint64_t n_pairs = 0;
    if (e->terms_set)
        for (const auto &t : e->term_refs) n_pairs += t.n;
    if (n_pairs > static_cast<uint64_t>(INT32_MAX))
        return fail(WAX_VS_ERR_CAPACITY, "term index of %llu (term, row) pairs: at most %d are supported",
                    static_cast<unsigned long long>(n_pairs), INT32_MAX);
    const uint32_t P = static_cast<uint32_t>(n_pairs);
    cudaStream_t s = c->stream;
    int32_t rc;
    uint32_t n_terms = 0;
    if ((rc = ti.postings.ensure(std::max<uint32_t>(P, 1), "term postings"))) return rc;
    if (P) {
        std::vector<uint64_t> h_keys(P);
        std::vector<uint32_t> h_rows(P);
        for (uint64_t r = 0, at = 0; r < e->n_rows; ++r) {
            const auto &t = e->term_refs[r];
            for (uint32_t j = 0; j < t.n; ++j, ++at) {
                h_keys[at] = e->term_pool[t.off + j];
                h_rows[at] = static_cast<uint32_t>(r);
            }
        }
        auto &keys_in = ti.sort_keys, &keys_out = ti.sorted_keys;
        auto &rows_in = ti.sort_rows, &heads = ti.heads, &incl = ti.numbering;
        auto &temp = ti.temp;
        size_t sort_bytes = 0, scan_bytes = 0;
        CUDA_TRY(cub::DeviceRadixSort::SortPairs(nullptr, sort_bytes, keys_in.p, keys_out.p, rows_in.p, ti.postings.p,
                                                 static_cast<int>(P), 0, 64, s));
        CUDA_TRY(cub::DeviceScan::InclusiveSum(nullptr, scan_bytes, heads.p, incl.p, static_cast<int>(P), s));
        if ((rc = keys_in.ensure(P, "term sort keys")) || (rc = keys_out.ensure(P, "sorted term keys")) ||
            (rc = rows_in.ensure(P, "term sort rows")) || (rc = heads.ensure(P, "term heads")) ||
            (rc = incl.ensure(P, "term numbering")) ||
            (rc = temp.ensure(std::max<size_t>(std::max(sort_bytes, scan_bytes), 1), "term index scratch")))
            return rc;
        CUDA_TRY(cudaMemcpyAsync(keys_in, h_keys.data(), static_cast<size_t>(P) * sizeof(uint64_t), cudaMemcpyHostToDevice, s));
        CUDA_TRY(cudaMemcpyAsync(rows_in, h_rows.data(), static_cast<size_t>(P) * sizeof(uint32_t), cudaMemcpyHostToDevice, s));
        CUDA_TRY(cub::DeviceRadixSort::SortPairs(temp.p, sort_bytes, keys_in.p, keys_out.p, rows_in.p, ti.postings.p,
                                                 static_cast<int>(P), 0, 64, s));
        const int grid = static_cast<int>(std::max<uint64_t>(1, std::min<uint64_t>(static_cast<uint64_t>(e->sm_count) * 8, (P + 255) / 256)));
        group_heads_kernel<<<grid, 256, 0, s>>>(keys_out, P, heads);
        CUDA_TRY(cudaGetLastError());
        CUDA_TRY(cub::DeviceScan::InclusiveSum(temp.p, scan_bytes, heads.p, incl.p, static_cast<int>(P), s));
        CUDA_TRY(cudaMemcpyAsync(&n_terms, incl.p + (P - 1), sizeof(uint32_t), cudaMemcpyDeviceToHost, s));
        CUDA_TRY(cudaStreamSynchronize(s));
        if ((rc = ti.keys.ensure(n_terms, "term keys")) || (rc = ti.start.ensure(static_cast<size_t>(n_terms) + 1, "term starts")))
            return rc;
        term_index_finish_kernel<<<grid, 256, 0, s>>>(keys_out, incl, P, ti.keys, ti.start);
        CUDA_TRY(cudaGetLastError());
        CUDA_TRY(cudaStreamSynchronize(s));     // before the scratch goes
        if (!e->shard.open) ti.release_scratch();
    } else if ((rc = ti.keys.ensure(1, "term keys")) || (rc = ti.start.ensure(1, "term starts"))) {
        return rc;
    }
    const uint64_t end = P;
    CUDA_TRY(cudaMemcpyAsync(ti.start.p + n_terms, &end, sizeof(uint64_t), cudaMemcpyHostToDevice, s));
    CUDA_TRY(cudaStreamSynchronize(s));
    ti.n_terms = n_terms;
    ti.n_postings = P;
    ti.valid = true;
    std::lock_guard<std::mutex> pg(e->pool_mu);
    ++e->term_index_builds;
    return WAX_VS_OK;
}

static int where_grid(const wax_vs_engine *e, uint64_t threads) {
    return static_cast<int>(std::max<uint64_t>(1, std::min<uint64_t>(static_cast<uint64_t>(e->sm_count) * 8,
                                                                     (threads + kWhereThreads - 1) / kWhereThreads)));
}

// Whether b is a location clause (kNoLocBox is none; no box location_box builds equals it).
static bool box_active(const LocBox &b) {
    return b.lat_lo != kNoLocBox.lat_lo || b.lat_hi != kNoLocBox.lat_hi || b.lon_lo0 != kNoLocBox.lon_lo0 ||
           b.lon_hi0 != kNoLocBox.lon_hi0 || b.lon_lo1 != kNoLocBox.lon_lo1 || b.lon_hi1 != kNoLocBox.lon_hi1;
}

// Whether c is a root clause ({0, 0} is none).
static bool root_active(const RootClause &c) { return c.all_tags != 0u || c.no_tags != 0u; }

static int32_t ensure_root_column(wax_vs_engine *e, SearchCtx *c);

// One where pass over `items` on `stream`: the items staged in c->d_where_items in the pass's form, then launch(located,
// rooted, d_items, i0, count) for each kWhereChunk of them (and ++*launches unless that is nullptr).  `located` is
// std::true_type when some box is active, the located kernels over the items with their boxes, after the location
// mirror is brought up; otherwise std::false_type, the plain kernels, which read no location.  kNoLocBox admits every
// row, rows without a location included, so the two forms agree wherever both apply.  Likewise `rooted` is
// std::true_type when some item has a root clause, after the root column is brought up, and the clause {0, 0} admits
// every row.
extern "C++" {     // templates, inside the C API's block
template <bool kLocated, bool kRooted, class Launch>
static int32_t where_pass_form(SearchCtx *c, const std::vector<WhereFull> &items, cudaStream_t stream, uint64_t *launches,
                               Launch launch) {
    using Item = WhereItemOf<kLocated, kRooted>;
    const uint32_t m = static_cast<uint32_t>(items.size());
    std::vector<Item> h(m);
    for (uint32_t i = 0; i < m; ++i) {
        h[i].pred = items[i].pred;
        h[i].slot = items[i].slot;
        if constexpr (kLocated) h[i].box = items[i].box;
        if constexpr (kRooted) h[i].root = items[i].root;
    }
    Item *d_items = reinterpret_cast<Item *>(c->d_where_items.p);
    CUDA_TRY(cudaMemcpyAsync(d_items, h.data(), m * sizeof(Item), cudaMemcpyHostToDevice, stream));
    for (uint32_t i0 = 0; i0 < m; i0 += kWhereChunk) {
        launch(std::bool_constant<kLocated>{}, std::bool_constant<kRooted>{}, d_items + i0, i0, std::min(kWhereChunk, m - i0));
        if (launches) ++*launches;
    }
    CUDA_TRY(cudaGetLastError());
    return WAX_VS_OK;
}
template <class Launch>
static int32_t where_pass(wax_vs_engine *e, SearchCtx *c, const std::vector<WhereFull> &items, cudaStream_t stream,
                          uint64_t *launches, Launch launch) {
    const uint32_t m = static_cast<uint32_t>(items.size());
    if (!m) return WAX_VS_OK;
    const bool located = std::any_of(items.begin(), items.end(), [](const WhereFull &it) { return box_active(it.box); });
    const bool rooted = std::any_of(items.begin(), items.end(), [](const WhereFull &it) { return root_active(it.root); });
    int32_t rc;
    if ((rc = ensure_attributes(e, c, located)) || (rooted && (rc = ensure_root_column(e, c))) ||
        (rc = c->d_where_items.ensure(m, "where predicates")))
        return rc;
    if (located)
        return rooted ? where_pass_form<true, true>(c, items, stream, launches, launch)
                      : where_pass_form<true, false>(c, items, stream, launches, launch);
    return rooted ? where_pass_form<false, true>(c, items, stream, launches, launch)
                  : where_pass_form<false, false>(c, items, stream, launches, launch);
}
}  // extern "C++"

// counts[i] = the rows passing items[i]: one streaming pass per kWhereChunk predicates, read back once.
static int32_t where_counts(wax_vs_engine *e, SearchCtx *c, const std::vector<WhereFull> &items,
                            std::vector<uint32_t> &counts) {
    const uint32_t m = static_cast<uint32_t>(items.size()), n = static_cast<uint32_t>(e->n_rows);
    counts.assign(m, 0u);
    if (!m) return WAX_VS_OK;
    int32_t rc;
    if ((rc = c->d_where_counts.ensure(m, "where counts"))) return rc;
    CUDA_TRY(cudaMemsetAsync(c->d_where_counts, 0, m * sizeof(uint32_t), c->stream));
    if ((rc = where_pass(e, c, items, c->stream, nullptr,
                         [&](auto located, auto rooted, const auto *d_items, uint32_t i0, uint32_t count) {
                             where_count_kernel<decltype(located)::value, decltype(rooted)::value>
                                 <<<where_grid(e, n), kWhereThreads, 0, c->stream>>>(e->d_attrs, e->d_locs, n, d_items, count,
                                                                                    c->d_where_counts + i0, e->roots.col);
                         })))
        return rc;
    CUDA_TRY(cudaMemcpyAsync(counts.data(), c->d_where_counts, m * sizeof(uint32_t), cudaMemcpyDeviceToHost, c->stream));
    CUDA_TRY(cudaStreamSynchronize(c->stream));
    return WAX_VS_OK;
}

// ANDs items[i] into bitset items[i].slot of c->d_mask on `stream` (after the filter builders wrote it).
static int32_t apply_where_bits(wax_vs_engine *e, SearchCtx *c, const std::vector<WhereFull> &items, cudaStream_t stream,
                                uint64_t *launches) {
    const uint32_t n = static_cast<uint32_t>(e->n_rows), words = (n + 31u) / 32u;
    return where_pass(e, c, items, stream, launches, [&](auto located, auto rooted, const auto *d_items, uint32_t, uint32_t count) {
        where_bits_kernel<decltype(located)::value, decltype(rooted)::value>
            <<<where_grid(e, static_cast<uint64_t>(words) * 32u), kWhereThreads, 0, stream>>>(
                e->d_attrs, e->d_locs, n, words, c->d_mask, d_items, count, e->roots.col);
    });
}

// The rows of the narrow predicates (fs.compact) into c->d_filter_rows at their slots, on `stream`.
static int32_t list_where_rows(wax_vs_engine *e, SearchCtx *c, const std::vector<WhereFull> &items, cudaStream_t stream,
                               uint64_t *launches) {
    const uint32_t m = static_cast<uint32_t>(items.size()), n = static_cast<uint32_t>(e->n_rows);
    if (!m) return WAX_VS_OK;
    int32_t rc;
    if ((rc = c->d_where_counts.ensure(m, "where cursors"))) return rc;
    CUDA_TRY(cudaMemsetAsync(c->d_where_counts, 0, m * sizeof(uint32_t), stream));
    return where_pass(e, c, items, stream, launches, [&](auto located, auto rooted, const auto *d_items, uint32_t i0, uint32_t count) {
        where_compact_kernel<decltype(located)::value, decltype(rooted)::value><<<where_grid(e, n), kWhereThreads, 0, stream>>>(
            e->d_attrs, e->d_locs, n, d_items, count, c->d_where_counts + i0, c->d_filter_rows, e->roots.col);
    });
}

// The term or group-clause units of a launch staged in `buf` on stream s, in the launch's form: as they are when some
// unit has a root clause (*rooted = true; the root column is brought up first), else without their root clauses, the
// unrooted form's units.
extern "C++" {     // a template, inside the C API's block
template <class Base>
static int32_t stage_units(wax_vs_engine *e, SearchCtx *c, DevBuf<Rooted<Base>> &buf, const std::vector<Rooted<Base>> &units,
                           cudaStream_t s, bool *rooted) {
    const size_t n = units.size();
    *rooted = std::any_of(units.begin(), units.end(), [](const Rooted<Base> &u) { return root_active(u.root); });
    int32_t rc;
    if (*rooted) {
        if ((rc = ensure_root_column(e, c))) return rc;
        CUDA_TRY(cudaMemcpyAsync(buf.p, units.data(), n * sizeof(Rooted<Base>), cudaMemcpyHostToDevice, s));
        return WAX_VS_OK;
    }
    const std::vector<Base> plain(units.begin(), units.end());
    CUDA_TRY(cudaMemcpyAsync(reinterpret_cast<Base *>(buf.p), plain.data(), n * sizeof(Base), cudaMemcpyHostToDevice, s));
    return WAX_VS_OK;
}
}  // extern "C++"

// term_filter_kernel over `units` on `stream` (waxvs_terms.cuh): counting into c->d_term_counts (zeroed here) and, with
// rows_out, listing each unit's rows at its slot; or, with bits, setting them in bitset `slot` of bits.  plan_term_units
// sized c->d_term_units and c->d_term_counts for the call's largest launch, so no buffer an earlier launch reads moves.
static int32_t launch_term_filter(wax_vs_engine *e, SearchCtx *c, const std::vector<TermUnitR> &units, uint32_t *rows_out,
                                  uint32_t *bits, cudaStream_t s, uint64_t *launches) {
    const uint32_t n = static_cast<uint32_t>(units.size());
    if (!n) return WAX_VS_OK;
    int32_t rc;
    bool rooted;
    if ((rc = c->d_term_units.ensure(n, "term units")) || (rc = c->d_term_counts.ensure(n, "term counts"))) return rc;
    if (!bits) CUDA_TRY(cudaMemsetAsync(c->d_term_counts, 0, n * sizeof(uint32_t), s));
    if ((rc = stage_units(e, c, c->d_term_units, units, s, &rooted))) return rc;
    const uint32_t words = static_cast<uint32_t>((e->n_rows + 31) / 32);
    for (uint32_t u0 = 0; u0 < n; u0 += 65535u) {       // grid.y limit
        const uint32_t nu = std::min<uint32_t>(n - u0, 65535u);
        uint32_t longest = 1;
        for (uint32_t j = u0; j < u0 + nu; ++j) longest = std::max(longest, units[j].spans[0].count);
        const uint32_t spread = std::max<uint32_t>(4, static_cast<uint32_t>(e->sm_count) * 16 / nu);
        const dim3 grid(std::min<uint32_t>((longest + kTermThreads - 1) / kTermThreads, spread), nu);
        uint32_t *counts = bits ? nullptr : c->d_term_counts + u0;
        if (rooted)
            term_filter_kernel<true><<<grid, kTermThreads, 0, s>>>(e->tindex.postings, e->d_attrs, e->d_locs, c->d_term_deny,
                                                                   c->d_term_units + u0, counts, rows_out, bits, words,
                                                                   e->roots.col);
        else
            term_filter_kernel<false><<<grid, kTermThreads, 0, s>>>(e->tindex.postings, e->d_attrs, e->d_locs, c->d_term_deny,
                                                                    reinterpret_cast<const TermUnit *>(c->d_term_units.p) + u0,
                                                                    counts, rows_out, bits, words, nullptr);
        CUDA_TRY(cudaGetLastError());
        ++*launches;
    }
    return WAX_VS_OK;
}

constexpr uint64_t kWhereGatherRows = 16384;   // the gather class's largest allow-list (plan_filtered)

// where_group_filter_kernel over `units` on `stream` (waxvs_where_groups.cuh), as launch_term_filter: counting into
// c->d_gw_counts (zeroed here) and, with rows_out, listing each unit's rows at its slot; or, with bits, setting them in
// bitset `slot` of bits.  plan_group_units sized c->d_gw_units and c->d_gw_counts for the call's largest launch and
// staged the units' group spans in c->d_gw_spans and their deny-lists in c->d_gw_deny.
static int32_t launch_group_filter(wax_vs_engine *e, SearchCtx *c, const std::vector<GroupUnitR> &units, uint32_t *rows_out,
                                   uint32_t *bits, cudaStream_t s, uint64_t *launches) {
    const uint32_t n = static_cast<uint32_t>(units.size());
    if (!n) return WAX_VS_OK;
    int32_t rc;
    bool rooted;
    if ((rc = c->d_gw_units.ensure(n, "group units")) || (rc = c->d_gw_counts.ensure(n, "group unit counts"))) return rc;
    if (!bits) CUDA_TRY(cudaMemsetAsync(c->d_gw_counts, 0, n * sizeof(uint32_t), s));
    if ((rc = stage_units(e, c, c->d_gw_units, units, s, &rooted))) return rc;
    const uint32_t words = static_cast<uint32_t>((e->n_rows + 31) / 32);
    for (uint32_t u0 = 0; u0 < n; u0 += 65535u) {       // grid.y limit
        const uint32_t nu = std::min<uint32_t>(n - u0, 65535u);
        uint32_t longest = 1;
        for (uint32_t j = u0; j < u0 + nu; ++j) longest = std::max(longest, units[j].n_cand);
        const uint32_t spread = std::max<uint32_t>(4, static_cast<uint32_t>(e->sm_count) * 16 / nu);
        const dim3 grid(std::min<uint32_t>((longest + kTermThreads - 1) / kTermThreads, spread), nu);
        uint32_t *counts = bits ? nullptr : c->d_gw_counts + u0;
        if (rooted)
            where_group_filter_kernel<true><<<grid, kTermThreads, 0, s>>>(
                e->gindex.perm, e->gindex.row_group, e->tindex.postings, c->d_gw_spans, e->d_attrs, e->d_locs, c->d_gw_deny,
                c->d_gw_units + u0, counts, rows_out, bits, words, e->roots.col);
        else
            where_group_filter_kernel<false><<<grid, kTermThreads, 0, s>>>(
                e->gindex.perm, e->gindex.row_group, e->tindex.postings, c->d_gw_spans, e->d_attrs, e->d_locs, c->d_gw_deny,
                reinterpret_cast<const GroupUnit *>(c->d_gw_units.p) + u0, counts, rows_out, bits, words, nullptr);
        CUDA_TRY(cudaGetLastError());
        ++*launches;
    }
    return WAX_VS_OK;
}

// Filter f's group unit when it is wide (its bits are set in its bitset, it lists nothing), else nullptr.
static const GroupUnitR *wide_group_unit(const FilterSet &fs, uint32_t f) {
    if (fs.group_of.empty() || fs.group_of[f] == WAX_VS_NO_FILTER || fs.count[f] <= kWhereGatherRows) return nullptr;
    return &fs.group_units[fs.group_of[f]];
}

// ---- batched filtered search ------------------------------------------------------------------------------------
// n_queries queries, query i under filter query_filter[i] (WAX_VS_NO_FILTER: unfiltered); the single-filter entry
// points are the case of one filter that every query names.  Every query referenced filter is resolved once; query i
// asks for k_i = min(clamp(top_k), allowed_i) rows and falls in one of three classes:
//  - gather: an allow-list of <= 16 384 rows -- exact scores of the listed rows only, all such queries in one batched
//    gather over the concatenated lists, one CTA per query sorts;
//  - tensor: allowed_i >= clamp(top_k), so the class shares one k -- run_queries_on_device with a bitset per query (the
//    tensor-core levels, whose nominations, filter level and exact fall-back all consult the query's own bitset, so the
//    completeness proof is a statement about ITS allowed rows; or one masked fused scan per query);
//  - scan: the rest (deny-lists that leave fewer than k rows, an unfiltered query on a corpus below k), one masked fused
//    scan each with its own k_i.
// The bitsets are built on the device; a pass holds at most filter_bitset_bytes of them, more filters run in several
// sub-batches (queries sorted by filter, so each filter's bitset is built once).
// Each query's k and class.  Staged query j is query order[j] and fills k_of[j] of its k_max candidate slots; the staged
// order is the tensor class, the gather class, the scan class, the first and last sorted by filter so that a sub-batch
// names a run of consecutive filters (unfiltered queries last).  Queries whose filter allows nothing are not staged.
struct FilteredPlan {
    std::vector<uint32_t> order, k_of;
    uint32_t k_max = 0, n_tensor = 0, n_gather = 0;
};
// What plan_request made of a request: the resolved id filters (`ids`; where lists only), the filters the plan runs
// (`fs`: the request's id filters, or its (where, id filter) pairs) with their modes, query i's filter pair_of[i]
// (WAX_VS_NO_FILTER: unfiltered), and each query's k and class.
struct WherePlan {
    FilterSet ids, fs;
    std::vector<int32_t> modes;
    std::vector<uint32_t> pair_of;
    FilteredPlan plan;
};
static void plan_filtered(const wax_vs_engine *e, int64_t top_k, const int32_t *filter_modes, const uint32_t *query_filter,
                          uint32_t n_queries, const FilterSet &fs, FilteredPlan &plan) {
    const uint64_t n_rows = e->n_rows;
    const uint32_t limit = clamp_topk(top_k);
    std::vector<uint32_t> tensor, gather, scan;                // query indices
    std::vector<uint32_t> k_of_query(n_queries, 0);
    uint32_t k_max = 0;
    for (uint32_t i = 0; i < n_queries; ++i) {
        const uint32_t f = query_filter[i];
        uint64_t allowed = f == WAX_VS_NO_FILTER ? n_rows : (filter_modes[f] == 0 ? fs.count[f] : n_rows - fs.count[f]);
        if (f != WAX_VS_NO_FILTER && !fs.where.empty() && fs.where[f] != WAX_VS_NO_FILTER) allowed = fs.allowed[f];
        const uint32_t k = static_cast<uint32_t>(std::min<uint64_t>(limit, allowed));
        if (k == 0) continue;
        k_of_query[i] = k;
        k_max = std::max(k_max, k);
        if (f != WAX_VS_NO_FILTER && filter_modes[f] == 0 && fs.count[f] <= 16384) gather.push_back(i);
        else if (allowed >= limit) tensor.push_back(i);
        else scan.push_back(i);
    }
    auto by_filter = [&](uint32_t a, uint32_t b) { return query_filter[a] < query_filter[b]; };
    std::stable_sort(tensor.begin(), tensor.end(), by_filter);
    std::stable_sort(scan.begin(), scan.end(), by_filter);
    plan.order = tensor;
    plan.order.insert(plan.order.end(), gather.begin(), gather.end());
    plan.order.insert(plan.order.end(), scan.begin(), scan.end());
    plan.k_of.resize(plan.order.size());
    for (size_t j = 0; j < plan.order.size(); ++j) plan.k_of[j] = k_of_query[plan.order[j]];
    plan.k_max = k_max;
    plan.n_tensor = static_cast<uint32_t>(tensor.size());
    plan.n_gather = static_cast<uint32_t>(gather.size());
}

// The bitsets of the filters `which` (bitset l is filter which[l]'s) into c->d_mask on c->stream, from the rows
// run_filtered staged in c->d_filter_rows: the listed rows in the filter's mode, then where search's predicate and box
// ANDed in, and a wide term or group unit's rows set.  On an error the stream is synchronised.
static int32_t build_pass_bits(wax_vs_engine *e, SearchCtx *c, const WherePlan &wp, const std::vector<uint32_t> &which,
                               uint64_t *launches) {
    const FilterSet &fs = wp.fs;
    const uint32_t nf = static_cast<uint32_t>(which.size());
    std::vector<uint64_t> spec(3u * nf + 1u, 0);
    for (uint32_t l = 0; l < nf; ++l) {
        const bool wide = (!fs.term_of.empty() && fs.term_of[which[l]] != WAX_VS_NO_FILTER) || wide_group_unit(fs, which[l]);
        spec[l + 1] = spec[l] + (wide ? 0 : fs.count[which[l]]);       // a wide term or group unit lists nothing
        spec[nf + 1 + l] = fs.first[which[l]];
        spec[2u * nf + 1u + l] = static_cast<uint64_t>(wp.modes[which[l]]);
    }
    int32_t rc;
    if ((rc = build_filter_bits(e, c, spec, nf, c->stream, launches))) { cudaStreamSynchronize(c->stream); return rc; }
    std::vector<WhereFull> wbits;                               // where search: the predicates ANDed in
    for (uint32_t l = 0; l < nf && !fs.where.empty(); ++l)
        if (fs.where[which[l]] != WAX_VS_NO_FILTER) {
            wbits.push_back(fs.preds[fs.where[which[l]]]);
            wbits.back().slot = l;
        }
    std::vector<TermUnitR> tbits;                               // where_terms search: wide units' rows
    for (uint32_t l = 0; l < nf && !fs.term_of.empty(); ++l)
        if (fs.term_of[which[l]] != WAX_VS_NO_FILTER) {
            tbits.push_back(fs.term_wide[fs.term_of[which[l]]]);
            tbits.back().slot = l;
        }
    std::vector<GroupUnitR> gbits;                              // where_groups search: wide units' rows
    for (uint32_t l = 0; l < nf; ++l)
        if (const GroupUnitR *u = wide_group_unit(fs, which[l])) {
            gbits.push_back(*u);
            gbits.back().slot = l;
        }
    if ((rc = apply_where_bits(e, c, wbits, c->stream, launches)) ||
        (rc = launch_term_filter(e, c, tbits, nullptr, c->d_mask, c->stream, launches)) ||
        (rc = launch_group_filter(e, c, gbits, nullptr, c->d_mask, c->stream, launches))) {
        cudaStreamSynchronize(c->stream);
        return rc;
    }
    return WAX_VS_OK;
}

// The filters' rows into c->d_filter_rows on c->stream, where build_pass_bits and the gather class read them: the
// host-listed rows, then the rows the device lists (narrow where units, narrow term units, narrow group units).
static int32_t stage_pair_rows(wax_vs_engine *e, SearchCtx *c, const FilterSet &fs, uint64_t *launches) {
    int32_t rc;
    if ((rc = stage_filter_rows(e, c, fs.rows, fs.rows.size() + fs.device_rows, -1, c->stream, nullptr))) return rc;
    std::vector<GroupUnitR> glist;
    for (uint32_t f = 0; f < fs.group_of.size(); ++f)
        if (fs.group_of[f] != WAX_VS_NO_FILTER && fs.count[f] && !wide_group_unit(fs, f)) glist.push_back(fs.group_units[fs.group_of[f]]);
    if ((rc = list_where_rows(e, c, fs.compact, c->stream, launches)) ||
        (rc = launch_term_filter(e, c, fs.term_list, c->d_filter_rows, nullptr, c->stream, launches)) ||
        (rc = launch_group_filter(e, c, glist, c->d_filter_rows, nullptr, c->stream, launches))) {
        cudaStreamSynchronize(c->stream);
        return rc;
    }
    return WAX_VS_OK;
}

// What run_filtered's candidates carry and where they go.  The defaults serve the host entry points, which map local rows
// to frame ids themselves.  A shard reports global rows (row_offset + local row) and its frame ids (d_ids, nullptr for
// identity ids); the device form's queries are on the device; the collective form (one query) exchanges its list with
// the other ranks, merged into shard->final_out.
struct FilteredTarget {
    uint64_t row_offset = 0;
    const uint64_t *d_ids = nullptr;
    bool device_queries = false;
    const ShardParams *shard = nullptr;
};

// The planned queries on c->stream: staged query j's candidates land at c->d_out[j * k_max], on the device (with
// tgt.shard: this rank's list there, the merged one at tgt.shard->final_out).  Stages the queries (c->d_queries, staged
// order; for device queries the order goes to c->d_order) and the filters' rows (c->d_filter_rows).  plan.k_max > 0.
static int32_t run_filtered(wax_vs_engine *e, SearchCtx *c, const float *queries, const WherePlan &wp,
                            const FilteredTarget &tgt = FilteredTarget{}) {
    const FilterSet &fs = wp.fs;
    const FilteredPlan &plan = wp.plan;
    const uint32_t *query_filter = wp.pair_of.data();
    const std::vector<uint32_t> &order = plan.order, &k_of = plan.k_of;
    const std::vector<uint64_t> &first = fs.first, &count = fs.count;
    const uint32_t k_max = plan.k_max, n_tensor = plan.n_tensor, n_gather = plan.n_gather;
    const uint32_t n_staged = static_cast<uint32_t>(order.size());
    const uint32_t words = static_cast<uint32_t>((e->n_rows + 31) / 32);
    int32_t rc;
    const size_t ncand = static_cast<size_t>(n_staged) * k_max;       // staged query j's candidates at j * k_max
    if (tgt.device_queries) {
        const size_t qfloats = static_cast<size_t>(n_staged) * e->dims;
        if ((rc = c->d_queries.ensure(qfloats, "query buffer")) || (rc = c->d_order.ensure(2u * n_staged, "query order")))
            return rc;
        CUDA_TRY(cudaMemcpyAsync(c->d_order, order.data(), n_staged * sizeof(uint32_t), cudaMemcpyHostToDevice, c->stream));
        CUDA_TRY(cudaMemcpyAsync(c->d_order + n_staged, k_of.data(), n_staged * sizeof(uint32_t), cudaMemcpyHostToDevice,
                                 c->stream));
        const int grid = static_cast<int>(std::max<size_t>(1, std::min<size_t>(static_cast<size_t>(e->sm_count) * 8, (qfloats + 255) / 256)));
        stage_query_rows_kernel<<<grid, 256, 0, c->stream>>>(queries, c->d_order, n_staged, e->dims, c->d_queries);
        CUDA_TRY(cudaGetLastError());
    } else if ((rc = stage_queries(e, c, queries, n_staged, c->stream, order.data()))) {
        return rc;
    }
    if ((rc = c->d_out.ensure(ncand, "result buffer"))) return rc;
    uint64_t launches = 0;
    if ((rc = stage_pair_rows(e, c, fs, &launches))) return rc;

    // gather class: one concatenated row list, a span per query; the sort grants shared memory for the longest list
    if (n_gather) {
        std::vector<uint2> spans(n_gather);
        uint32_t longest = 1;
        for (uint32_t j = 0; j < n_gather; ++j) {
            const uint32_t f = query_filter[order[n_tensor + j]];
            spans[j] = make_uint2(static_cast<uint32_t>(first[f]), static_cast<uint32_t>(count[f]));
            longest = std::max(longest, spans[j].y);
        }
        if ((rc = c->d_gather_span.ensure(n_gather, "gather spans"))) return rc;
        if ((rc = c->d_gather_keys.ensure(static_cast<size_t>(longest) * n_gather, "gather keys"))) return rc;
        CUDA_TRY(cudaMemcpyAsync(c->d_gather_span, spans.data(), n_gather * sizeof(uint2), cudaMemcpyHostToDevice, c->stream));
        uint32_t pow2 = 64;
        while (pow2 < longest) pow2 <<= 1;
        CUDA_TRY(grant_smem(e, gather_sort_kernel, pow2 * sizeof(uint64_t)));
        const uint32_t gx = std::max<uint32_t>(1, std::min<uint32_t>((longest + 31) / 32, static_cast<uint32_t>(e->sm_count) * 8));
        for (uint32_t q0 = 0; q0 < n_gather; q0 += 32768u) {       // grid.y limit
            const uint32_t nq = std::min<uint32_t>(n_gather - q0, 32768u);
            const dim3 ggrid(gx, nq);
            const float *dq = c->d_queries + static_cast<size_t>(n_tensor + q0) * e->dims;
            const uint2 *span = c->d_gather_span + q0;
            uint64_t *keys = c->d_gather_keys + static_cast<size_t>(q0) * longest;
            switch (e->similarity) {
                case WAX_VS_COSINE: gather_score_kernel<kCosine><<<ggrid, 256, 0, c->stream>>>(e->d_corpus, dq, e->dims, c->d_filter_rows, span, longest, keys); break;
                case WAX_VS_DOT: gather_score_kernel<kDot><<<ggrid, 256, 0, c->stream>>>(e->d_corpus, dq, e->dims, c->d_filter_rows, span, longest, keys); break;
                default: gather_score_kernel<kL2><<<ggrid, 256, 0, c->stream>>>(e->d_corpus, dq, e->dims, c->d_filter_rows, span, longest, keys); break;
            }
            CUDA_TRY(cudaGetLastError());
            ScanParams sp{};
            sp.k = k_max; sp.out = c->d_out + static_cast<size_t>(n_tensor + q0) * k_max; sp.id_base = e->id_base;
            sp.frame_ids = tgt.d_ids; sp.row_offset = tgt.row_offset; sp.row_keys = c->row_keys;
            gather_sort_kernel<<<nq, 1024, pow2 * sizeof(uint64_t), c->stream>>>(keys, span, longest, pow2, sp);
            CUDA_TRY(cudaGetLastError());
            launches += 2;
        }
        if (tgt.shard && (rc = enqueue_exchange(*tgt.shard, c->d_out, k_max, c->stream, &launches))) return rc;
    }

    // tensor and scan classes: sub-batches whose bitsets fit the budget (at least one always does)
    const uint64_t fit = std::max<uint64_t>(1, e->tune.filter_bitset_bytes / (static_cast<uint64_t>(words) * sizeof(uint32_t)));
    uint64_t distinct = 0;
    for (const uint8_t r : fs.referenced) distinct += r;
    const uint32_t per_pass = static_cast<uint32_t>(std::min<uint64_t>(fit, std::max<uint64_t>(distinct, 1)));
    // sized once for the largest pass: a later pass must not reallocate a buffer earlier launches still read
    if ((rc = c->d_mask.ensure(static_cast<size_t>(per_pass) * words, "row filters"))) return rc;
    if ((rc = c->d_filter_spec.ensure(3u * per_pass + 1u, "filter spec"))) return rc;
    if ((rc = c->d_query_filter.ensure(std::max<uint32_t>(n_tensor, 1), "query filters"))) return rc;
    std::vector<uint32_t> index(n_staged, WAX_VS_NO_FILTER);           // staged query -> bitset of its pass
    uint64_t passes = 0;
    auto run_class = [&](uint32_t j0, uint32_t j1, bool tensor_class) -> int32_t {
        for (uint32_t s0 = j0; s0 < j1;) {
            std::vector<uint32_t> which;                                // the pass's filters, in bitset order
            uint32_t s1 = s0;
            for (; s1 < j1; ++s1) {
                const uint32_t f = query_filter[order[s1]];
                if (f != WAX_VS_NO_FILTER && (which.empty() || which.back() != f)) {
                    if (which.size() == per_pass) break;
                    which.push_back(f);
                }
                index[s1] = f == WAX_VS_NO_FILTER ? WAX_VS_NO_FILTER : static_cast<uint32_t>(which.size() - 1);
            }
            int32_t prc;
            if (!which.empty() && (prc = build_pass_bits(e, c, wp, which, &launches))) return prc;
            RowFilter rf{c->d_mask.p, words, nullptr, index.data() + s0};
            const uint32_t nq = s1 - s0;
            const float *dq = c->d_queries + static_cast<size_t>(s0) * e->dims;
            wax_vs_candidate *dout = c->d_out + static_cast<size_t>(s0) * k_max;
            if (tensor_class && nq > 1) {
                CUDA_TRY(cudaMemcpyAsync(c->d_query_filter + s0, index.data() + s0, nq * sizeof(uint32_t), cudaMemcpyHostToDevice,
                                         c->stream));
                rf.d_index = c->d_query_filter + s0;
                if ((prc = run_queries_on_device(e, c, dq, nq, k_max, tgt.row_offset, dout, tgt.d_ids, &launches, rf)))
                    return prc;
            } else {                // single queries (search_filtered) and the scan class: the single-query path
                for (uint32_t j = 0; j < nq; ++j) {
                    prc = enqueue_search(e, c, dq + static_cast<size_t>(j) * e->dims, k_of[s0 + j], tgt.row_offset,
                                         tgt.shard ? tgt.shard->final_out : dout + static_cast<size_t>(j) * k_max, tgt.d_ids,
                                         c->stream, &launches, rf.mask(j), tgt.shard, nullptr, false, true);
                    if (prc) { cudaStreamSynchronize(c->stream); return prc; }
                }
            }
            if (tensor_class) ++passes;
            s0 = s1;
        }
        return WAX_VS_OK;
    };
    if ((rc = run_class(0, n_tensor, true))) return rc;
    if ((rc = run_class(n_tensor + n_gather, n_staged, false))) return rc;
    if (passes) {
        std::lock_guard<std::mutex> pg(e->pool_mu);
        e->filter_bitset_passes += passes;
    }
    return WAX_VS_OK;
}

// The request's per-query id filters: filter f lists frame_ids[filter_offsets[f], filter_offsets[f + 1]) as an
// allow-list (mode 0) or a deny-list (mode 1), and query i names filter query_filter[i].
static int32_t request_filters(SearchRequest &r, const uint64_t *frame_ids, const uint64_t *filter_offsets,
                               const int32_t *filter_modes, uint32_t n_filters, const uint32_t *query_filter) {
    if (!filter_offsets || (n_filters && !filter_modes) || (r.n_queries && !query_filter))
        return fail(WAX_VS_ERR_NULL, "NULL argument");
    for (uint32_t f = 0; f < n_filters; ++f)
        if (filter_modes[f] != 0 && filter_modes[f] != 1)
            return fail(WAX_VS_ERR_ARGUMENT, "filter mode must be 0 (allow-list) or 1 (deny-list)");
    if (filter_offsets[0] != 0) return fail(WAX_VS_ERR_ARGUMENT, "filter_offsets[0] must be 0");
    for (uint32_t f = 0; f < n_filters; ++f)
        if (filter_offsets[f + 1] < filter_offsets[f])
            return fail(WAX_VS_ERR_ARGUMENT, "filter_offsets decrease at filter %u", f);
    if (filter_offsets[n_filters] && !frame_ids) return fail(WAX_VS_ERR_NULL, "frame_ids is NULL");
    for (uint32_t i = 0; i < r.n_queries; ++i)
        if (query_filter[i] != WAX_VS_NO_FILTER && query_filter[i] >= n_filters)
            return fail(WAX_VS_ERR_ARGUMENT, "query %u names filter %u of %u", i, query_filter[i], n_filters);
    r.frame_ids = frame_ids;
    r.filter_offsets = filter_offsets;
    r.filter_modes = filter_modes;
    r.n_filters = n_filters;
    r.query_filter = query_filter;
    return WAX_VS_OK;
}

// One id filter for every query.  With empty_deny_is_none a deny-list of no ids is no filter (the grouped and shard entry
// points); otherwise it is a filter that denies no row (the filtered ones).  The answers are the same.
static int32_t request_one_filter(SearchRequest &r, const uint64_t *frame_ids, uint64_t n_ids, int32_t mode,
                                  bool empty_deny_is_none) {
    if (mode != 0 && mode != 1) return fail(WAX_VS_ERR_ARGUMENT, "filter mode must be 0 (allow-list) or 1 (deny-list)");
    if (n_ids && !frame_ids) return fail(WAX_VS_ERR_NULL, "frame_ids is NULL");
    r.one_offsets[1] = n_ids;
    r.one_mode = mode;
    r.filter_of.assign(r.n_queries, empty_deny_is_none && mode == 1 && n_ids == 0 ? WAX_VS_NO_FILTER : 0u);
    r.frame_ids = frame_ids;
    r.filter_offsets = r.one_offsets;
    r.filter_modes = &r.one_mode;
    r.n_filters = 1;
    r.query_filter = r.filter_of.data();
    return WAX_VS_OK;
}

// The planned queries run on c, their answers delivered to the caller's buffers (plan.k_max > 0).
static int32_t deliver_filtered(wax_vs_engine *e, SearchCtx *c, const float *queries, const WherePlan &wp,
                                uint64_t *out_ids, float *out_scores, uint32_t out_stride, uint32_t *out_n) {
    const FilteredPlan &plan = wp.plan;
    int32_t rc;
    const size_t ncand = static_cast<size_t>(plan.order.size()) * plan.k_max;
    if ((rc = c->h_out.ensure(ncand, "result staging"))) return rc;
    if ((rc = run_filtered(e, c, queries, wp))) return rc;
    CUDA_TRY(cudaMemcpyAsync(c->h_out, c->d_out, ncand * sizeof(wax_vs_candidate), cudaMemcpyDeviceToHost, c->stream));
    CUDA_TRY(cudaStreamSynchronize(c->stream));   // also keeps the host arrays alive until their copies are done
    deliver_results(e, c->h_out, static_cast<uint32_t>(plan.order.size()), plan.k_max, out_ids, out_scores, out_stride,
                    out_n, plan.order.data(), plan.k_of.data());
    return WAX_VS_OK;
}

// ---- where search: attribute predicates below the top-k (waxvs_where.cuh) -------------------------------------------
// Query i searches the rows that pass wheres[query_where[i]] AND its id filter.  The unit that gets a row filter is the
// distinct (where, id filter) pair some query names; a pair without a where is the id filter itself.  A pair with one
// becomes an ordinary filter of the plan above:
//  - allow-list AND where: the listed rows are tested against the host attribute arrays (O(listed)) -> an allow-list;
//  - deny-list AND where, or the where alone: allowed = (rows passing, from one device count pass for all the call's
//    predicates) - (listed rows passing).  When nothing listed passes and at most kWhereGatherRows rows do, the device
//    lists them (the gather class); otherwise the filter's bitset is the deny-list's (mode 1, listing only the rows that
//    pass) with the predicate ANDed in on the device, for the tensor and scan classes.

static WherePred where_pred(const wax_vs_where &w) { return WherePred{w.after, w.before, w.all_tags, w.no_tags}; }

static WhereFull where_item(const Clause &w) {
    WhereFull it{};
    it.pred = w.pred;
    it.box = w.box;
    it.root = w.root;
    return it;
}

// Whether row r lies in box b (a row without a location lies in no active box).
static bool host_loc_passes(const wax_vs_engine *e, const LocBox &b, uint32_t r) {
    const LocRow l = e->locs_set ? e->locs[r] : LocRow{kNoLocation, 0};
    return loc_passes(b, l.lat, l.lon);
}

// Whether row r holds every id of the sorted, distinct list `req` (a row without terms holds none).
static bool host_terms_pass(const wax_vs_engine *e, const std::vector<uint64_t> &req, uint32_t r) {
    if (req.empty()) return true;
    if (!e->terms_set) return false;
    const auto &t = e->term_refs[r];
    const uint64_t *p = e->term_pool.data() + t.off;
    return std::includes(p, p + t.n, req.begin(), req.end());
}

// Whether row r's group (its frame id while no set_groups was made) is one of the sorted, distinct list `groups`.
static bool host_group_passes(const wax_vs_engine *e, const std::vector<uint64_t> &groups, uint32_t r) {
    if (groups.empty()) return true;
    return std::binary_search(groups.begin(), groups.end(), e->groups_set ? e->groups[r] : frame_id_of(e, r));
}

// Whether the root-tag word of row r's group (its frame id while no set_groups was made; 0 for a group never given
// one) passes root clause rc.
static bool host_root_passes(const wax_vs_engine *e, const RootClause &rc, uint32_t r) {
    if (!root_active(rc)) return true;
    const auto &ids = e->roots.ids;
    const uint64_t g = e->groups_set ? e->groups[r] : frame_id_of(e, r);
    const auto it = std::lower_bound(ids.begin(), ids.end(), g);
    return root_passes(rc, it != ids.end() && *it == g ? e->roots.tags[it - ids.begin()] : 0u);
}

// The listed rows that pass every clause of `w`, appended to `out`.
static void host_rows_passing(const wax_vs_engine *e, const Clause &w, const uint32_t *rows, uint64_t n,
                              std::vector<uint32_t> &out) {
    for (uint64_t i = 0; i < n; ++i) {
        const AttrRow a = e->attrs_set ? e->attrs[rows[i]] : AttrRow{0, 0};
        if (where_passes(w.pred, a.ts, a.tags) && host_loc_passes(e, w.box, rows[i]) &&
            host_terms_pass(e, w.terms, rows[i]) && host_group_passes(e, w.groups, rows[i]) &&
            host_root_passes(e, w.root, rows[i]))
            out.push_back(rows[i]);
    }
}

// The posting span of every distinct term id the wheres of pairs[p] (p in units_p) require, into `req` (sorted) and
// `spans` (spans[j] is req[j]'s), on c's stream: the term index brought up, one launch, one read-back.
static int32_t resolve_term_spans(wax_vs_engine *e, SearchCtx *c, const std::vector<Clause> &wheres,
                                  const std::vector<std::pair<uint32_t, uint32_t>> &pairs,
                                  const std::vector<uint32_t> &units_p, std::vector<uint64_t> &req,
                                  std::vector<TermSpan> &spans) {
    int32_t rc;
    if ((rc = ensure_term_index(e, c))) return rc;
    const auto &ti = e->tindex;
    cudaStream_t s = c->stream;
    for (const uint32_t p : units_p) req.insert(req.end(), wheres[pairs[p].first].terms.begin(), wheres[pairs[p].first].terms.end());
    std::sort(req.begin(), req.end());
    req.erase(std::unique(req.begin(), req.end()), req.end());
    const uint32_t n_ids = static_cast<uint32_t>(req.size());
    spans.assign(n_ids, TermSpan{0, 0, 0});
    if ((rc = c->d_term_ids.ensure(n_ids, "required terms")) || (rc = c->d_term_spans.ensure(n_ids, "term spans"))) return rc;
    CUDA_TRY(cudaMemcpyAsync(c->d_term_ids, req.data(), n_ids * sizeof(uint64_t), cudaMemcpyHostToDevice, s));
    term_spans_kernel<<<std::max<uint32_t>(1, std::min<uint32_t>((n_ids + 255) / 256, e->sm_count * 8)), 256, 0, s>>>(
        ti.keys, ti.start, ti.n_terms, c->d_term_ids, n_ids, c->d_term_spans);
    CUDA_TRY(cudaGetLastError());
    CUDA_TRY(cudaMemcpyAsync(spans.data(), c->d_term_spans, n_ids * sizeof(TermSpan), cudaMemcpyDeviceToHost, s));
    CUDA_TRY(cudaStreamSynchronize(s));
    return WAX_VS_OK;
}

// The deny-lists of the units pairs[p] (p in units_p), each sorted, once per list: deny_of[f] = filter f's rows in
// deny_rows.
static void unit_deny_lists(const FilterSet &ids, const std::vector<std::pair<uint32_t, uint32_t>> &pairs,
                            const std::vector<uint32_t> &units_p, std::vector<uint32_t> &deny_rows,
                            std::unordered_map<uint32_t, TermSpan> &deny_of) {
    for (const uint32_t p : units_p) {
        const uint32_t f = pairs[p].second;
        if (f == WAX_VS_NO_FILTER || deny_of.count(f)) continue;
        deny_of[f] = TermSpan{deny_rows.size(), static_cast<uint32_t>(ids.count[f]), 0};
        deny_rows.insert(deny_rows.end(), ids.rows.begin() + ids.first[f], ids.rows.begin() + ids.first[f] + ids.count[f]);
        std::sort(deny_rows.end() - ids.count[f], deny_rows.end());
    }
}

// The term units of a call (pairs[p] for p in units_p, whose where has terms and whose id filter is none or a
// deny-list) on c's stream: the posting span of every distinct required id (one launch, one read-back), then one
// term_filter_kernel launch counts each unit's rows from the postings of its rarest term (another read-back).  A unit
// becomes an allow-list of its fs.count[p] rows: a narrow one (<= kWhereGatherRows) is listed by the device in
// run_filtered at a slot from `at` on, as long as its count; a wide one gets its bits set in its bitset by the device,
// under the sub-batch split of filter_bitset_bytes.  The lists are therefore bounded as the device-listed where rows
// are, and no bitset is held outside that split.  A deny-list is checked by binary search in its rows, sorted, in
// c->d_term_deny.  The location mirror is brought up when some unit has a box.  `at` ends past the last slot.
static int32_t plan_term_units(wax_vs_engine *e, SearchCtx *c, const std::vector<Clause> &wheres, const FilterSet &ids,
                               const std::vector<std::pair<uint32_t, uint32_t>> &pairs, const std::vector<uint32_t> &units_p,
                               FilterSet &fs, uint64_t &at) {
    int32_t rc;
    cudaStream_t s = c->stream;
    std::vector<uint64_t> req;
    std::vector<TermSpan> spans;
    if ((rc = resolve_term_spans(e, c, wheres, pairs, units_p, req, spans))) return rc;

    std::vector<uint32_t> deny_rows;
    std::unordered_map<uint32_t, TermSpan> deny_of;
    unit_deny_lists(ids, pairs, units_p, deny_rows, deny_of);
    if ((rc = c->d_term_deny.ensure(std::max<size_t>(deny_rows.size(), 1), "term deny-lists"))) return rc;
    if (!deny_rows.empty())
        CUDA_TRY(cudaMemcpyAsync(c->d_term_deny, deny_rows.data(), deny_rows.size() * sizeof(uint32_t), cudaMemcpyHostToDevice, s));

    // each unit's candidates are the postings of its rarest term; a term no row holds leaves the unit empty
    std::vector<TermUnitR> units;
    std::vector<uint32_t> unit_pair;
    bool located = false;
    for (const uint32_t p : units_p) {
        const Clause &w = wheres[pairs[p].first];
        const uint32_t f = pairs[p].second;
        fs.first[p] = at;
        fs.count[p] = 0;
        TermUnitR u{};
        u.pred = w.pred;
        u.root = w.root;
        u.box = w.box;
        u.has_box = box_active(w.box);
        u.n_spans = static_cast<uint32_t>(w.terms.size());
        u.deny = f == WAX_VS_NO_FILTER ? TermSpan{0, 0, 0} : deny_of[f];
        uint32_t rarest = 0;
        for (uint32_t j = 0; j < u.n_spans; ++j) {
            u.spans[j] = spans[std::lower_bound(req.begin(), req.end(), w.terms[j]) - req.begin()];
            if (u.spans[j].count < u.spans[rarest].count) rarest = j;
        }
        if (u.spans[rarest].count == 0) continue;
        std::swap(u.spans[0], u.spans[rarest]);
        located = located || u.has_box;
        units.push_back(u);
        unit_pair.push_back(p);
    }
    const uint32_t n_units = static_cast<uint32_t>(units.size());
    if (!n_units) return WAX_VS_OK;
    if ((rc = ensure_attributes(e, c, located))) return rc;
    // sized once for the largest launch of the call (run_filtered launches subsets of these units)
    if ((rc = c->d_term_units.ensure(n_units, "term units")) || (rc = c->d_term_counts.ensure(n_units, "term counts")))
        return rc;
    uint64_t launches = 0;
    if ((rc = launch_term_filter(e, c, units, nullptr, nullptr, s, &launches))) { cudaStreamSynchronize(s); return rc; }
    std::vector<uint32_t> counts(n_units);
    CUDA_TRY(cudaMemcpyAsync(counts.data(), c->d_term_counts, n_units * sizeof(uint32_t), cudaMemcpyDeviceToHost, s));
    CUDA_TRY(cudaStreamSynchronize(s));
    fs.term_of.assign(fs.count.size(), WAX_VS_NO_FILTER);
    for (uint32_t j = 0; j < n_units; ++j) {
        const uint32_t p = unit_pair[j];
        fs.count[p] = counts[j];
        if (counts[j] == 0) continue;
        if (counts[j] <= kWhereGatherRows) {                 // narrow: listed at its slot (the gather class)
            units[j].slot = at;
            fs.first[p] = at;
            at += counts[j];
            fs.term_list.push_back(units[j]);
        } else {                                             // wide: its bitset's bits (tensor class)
            fs.term_of[p] = static_cast<uint32_t>(fs.term_wide.size());
            fs.term_wide.push_back(units[j]);
        }
    }
    if (at > UINT32_MAX)                                     // the gather spans hold 32-bit offsets
        return fail(WAX_VS_ERR_CAPACITY, "the filters of one call list %llu rows, at most %u are supported",
                    static_cast<unsigned long long>(at), UINT32_MAX);
    return WAX_VS_OK;
}

// The group units of a call (pairs[p] for p in units_p, whose where has groups and whose id filter is none or a
// deny-list) on c's stream, planned as plan_term_units plans term units: the device group index brought up, every
// distinct group id of the call resolved to its dense group and CSR span (one launch, one read-back), each unit's
// groups and their prefix staged in c->d_gw_spans, then one where_group_filter_kernel launch counts each unit's rows
// (another read-back).  A unit walks the rows of its groups, or the postings of its rarest term when that list is the
// shorter; a unit none of whose groups (or some of whose terms) any row carries is empty and launches nothing.  A unit
// becomes an allow-list of its fs.count[p] rows, listed by the device from `at` on (<= kWhereGatherRows) or set in its
// bitset (wider).  `at` ends past the last slot.
static int32_t ensure_group_index(wax_vs_engine *e, SearchCtx *c);
static int32_t plan_group_units(wax_vs_engine *e, SearchCtx *c, const std::vector<Clause> &wheres, const FilterSet &ids,
                                const std::vector<std::pair<uint32_t, uint32_t>> &pairs, const std::vector<uint32_t> &units_p,
                                FilterSet &fs, uint64_t &at) {
    int32_t rc;
    if ((rc = ensure_group_index(e, c))) return rc;
    const auto &gi = e->gindex;
    cudaStream_t s = c->stream;
    std::vector<uint64_t> req;
    bool with_terms = false;
    for (const uint32_t p : units_p) {
        const Clause &w = wheres[pairs[p].first];
        req.insert(req.end(), w.groups.begin(), w.groups.end());
        with_terms = with_terms || !w.terms.empty();
    }
    std::sort(req.begin(), req.end());
    req.erase(std::unique(req.begin(), req.end()), req.end());
    const uint32_t n_ids = static_cast<uint32_t>(req.size());
    std::vector<GroupSpan> resolved(n_ids);
    if ((rc = c->d_gw_ids.ensure(n_ids, "where groups")) || (rc = c->d_gw_resolved.ensure(n_ids, "where group spans")))
        return rc;
    CUDA_TRY(cudaMemcpyAsync(c->d_gw_ids, req.data(), n_ids * sizeof(uint64_t), cudaMemcpyHostToDevice, s));
    where_group_spans_kernel<<<std::max<uint32_t>(1, std::min<uint32_t>((n_ids + 255) / 256, e->sm_count * 8)), 256, 0, s>>>(
        gi.ids, gi.starts, gi.n_groups, c->d_gw_ids, n_ids, c->d_gw_resolved);
    CUDA_TRY(cudaGetLastError());
    CUDA_TRY(cudaMemcpyAsync(resolved.data(), c->d_gw_resolved, n_ids * sizeof(GroupSpan), cudaMemcpyDeviceToHost, s));
    CUDA_TRY(cudaStreamSynchronize(s));
    std::vector<uint64_t> treq;
    std::vector<TermSpan> tspans;
    if (with_terms && (rc = resolve_term_spans(e, c, wheres, pairs, units_p, treq, tspans))) return rc;

    std::vector<uint32_t> deny_rows;
    std::unordered_map<uint32_t, TermSpan> deny_of;
    unit_deny_lists(ids, pairs, units_p, deny_rows, deny_of);

    // each unit's groups in ascending dense order (its ids are sorted, and dense groups follow the ids' order), those no
    // row carries dropped, with the exclusive prefix of their row counts
    std::vector<GroupSpan> gspans;
    std::vector<GroupUnitR> units;
    std::vector<uint32_t> unit_pair;
    bool located = false;
    uint64_t walked = 0;
    for (const uint32_t p : units_p) {
        const Clause &w = wheres[pairs[p].first];
        const uint32_t f = pairs[p].second;
        fs.first[p] = at;
        fs.count[p] = 0;
        GroupUnitR u{};
        u.pred = w.pred;
        u.root = w.root;
        u.box = w.box;
        u.has_box = box_active(w.box);
        u.deny = f == WAX_VS_NO_FILTER ? TermSpan{0, 0, 0} : deny_of[f];
        u.gspan0 = gspans.size();
        uint32_t rows = 0;
        for (const uint64_t g : w.groups) {
            GroupSpan gs = resolved[std::lower_bound(req.begin(), req.end(), g) - req.begin()];
            if (gs.count == 0) continue;
            gs.before = rows;
            rows += gs.count;
            gspans.push_back(gs);
        }
        u.n_gspans = static_cast<uint32_t>(gspans.size() - u.gspan0);
        u.n_spans = static_cast<uint32_t>(w.terms.size());
        uint32_t rarest = 0;
        for (uint32_t j = 0; j < u.n_spans; ++j) {
            u.spans[j] = tspans[std::lower_bound(treq.begin(), treq.end(), w.terms[j]) - treq.begin()];
            if (u.spans[j].count < u.spans[rarest].count) rarest = j;
        }
        if (rows == 0 || (u.n_spans && u.spans[rarest].count == 0)) {
            gspans.resize(u.gspan0);
            continue;
        }
        if (u.n_spans) std::swap(u.spans[0], u.spans[rarest]);
        u.walk_terms = u.n_spans && u.spans[0].count < rows;
        u.n_cand = u.walk_terms ? u.spans[0].count : rows;
        walked += u.n_cand;
        located = located || u.has_box;
        units.push_back(u);
        unit_pair.push_back(p);
    }
    {
        std::lock_guard<std::mutex> pg(e->pool_mu);
        e->where_group_units += units_p.size();
        e->where_group_rows_walked += walked;
    }
    const uint32_t n_units = static_cast<uint32_t>(units.size());
    if (!n_units) return WAX_VS_OK;
    if ((rc = ensure_attributes(e, c, located))) return rc;
    // sized once for the largest launch of the call (run_filtered and grouped_one launch subsets of these units)
    if ((rc = c->d_gw_spans.ensure(gspans.size(), "where group unit spans")) ||
        (rc = c->d_gw_deny.ensure(std::max<size_t>(deny_rows.size(), 1), "where group deny-lists")) ||
        (rc = c->d_gw_units.ensure(n_units, "group units")) || (rc = c->d_gw_counts.ensure(n_units, "group unit counts")))
        return rc;
    CUDA_TRY(cudaMemcpyAsync(c->d_gw_spans, gspans.data(), gspans.size() * sizeof(GroupSpan), cudaMemcpyHostToDevice, s));
    if (!deny_rows.empty())
        CUDA_TRY(cudaMemcpyAsync(c->d_gw_deny, deny_rows.data(), deny_rows.size() * sizeof(uint32_t), cudaMemcpyHostToDevice, s));
    uint64_t launches = 0;
    if ((rc = launch_group_filter(e, c, units, nullptr, nullptr, s, &launches))) { cudaStreamSynchronize(s); return rc; }
    std::vector<uint32_t> counts(n_units);
    CUDA_TRY(cudaMemcpyAsync(counts.data(), c->d_gw_counts, n_units * sizeof(uint32_t), cudaMemcpyDeviceToHost, s));
    CUDA_TRY(cudaStreamSynchronize(s));
    fs.group_of.assign(fs.count.size(), WAX_VS_NO_FILTER);
    for (uint32_t j = 0; j < n_units; ++j) {
        const uint32_t p = unit_pair[j];
        fs.count[p] = counts[j];
        if (counts[j] == 0) continue;
        if (counts[j] <= kWhereGatherRows) {                 // narrow: listed at its slot (the gather class)
            units[j].slot = at;
            fs.first[p] = at;
            at += counts[j];
        }                                                    // wide: its bitset's bits (wide_group_unit)
        fs.group_of[p] = static_cast<uint32_t>(fs.group_units.size());
        fs.group_units.push_back(units[j]);
    }
    if (at > UINT32_MAX)                                     // the gather spans hold 32-bit offsets
        return fail(WAX_VS_ERR_CAPACITY, "the filters of one call list %llu rows, at most %u are supported",
                    static_cast<unsigned long long>(at), UINT32_MAX);
    return WAX_VS_OK;
}

// The pairs of a call as the filters of `fs` (modes[p], pair_of[i] = query i's pair or WAX_VS_NO_FILTER), from the
// resolved id filters `ids`.  Runs the count pass on c's stream.  A pair's where is tested whole on the host against an
// allow-list; otherwise a where with groups makes the pair a group unit (plan_group_units), one with terms a term unit
// (plan_term_units), and any other where is tested on the device, its box with it.
static int32_t plan_where_pairs(wax_vs_engine *e, SearchCtx *c, const std::vector<Clause> &wheres,
                                const uint32_t *query_where, const int32_t *filter_modes, const uint32_t *query_filter,
                                uint32_t n_queries, const FilterSet &ids, FilterSet &fs, std::vector<int32_t> &modes,
                                std::vector<uint32_t> &pair_of) {
    pair_of.assign(n_queries, WAX_VS_NO_FILTER);
    std::unordered_map<uint64_t, uint32_t> index;
    std::vector<std::pair<uint32_t, uint32_t>> pairs;              // (where, id filter)
    for (uint32_t i = 0; i < n_queries; ++i) {
        const uint32_t w = query_where[i], f = query_filter[i];
        if (w == WAX_VS_NO_FILTER && f == WAX_VS_NO_FILTER) continue;
        const auto ins = index.emplace((static_cast<uint64_t>(w) << 32) | f, static_cast<uint32_t>(pairs.size()));
        if (ins.second) pairs.emplace_back(w, f);
        pair_of[i] = ins.first->second;
    }
    // the predicates whose count the plan needs: those of pairs without an allow-list
    std::vector<uint32_t> slot(wheres.size(), WAX_VS_NO_FILTER);
    std::vector<WhereFull> counted;
    for (const auto &pr : pairs)
        if (pr.first != WAX_VS_NO_FILTER && (pr.second == WAX_VS_NO_FILTER || filter_modes[pr.second] == 1) &&
            slot[pr.first] == WAX_VS_NO_FILTER && wheres[pr.first].terms.empty() && wheres[pr.first].groups.empty()) {
            slot[pr.first] = static_cast<uint32_t>(counted.size());
            counted.push_back(where_item(wheres[pr.first]));
        }
    std::vector<uint32_t> passing;
    int32_t rc;
    if ((rc = where_counts(e, c, counted, passing))) return rc;
    const uint32_t np = static_cast<uint32_t>(pairs.size());
    fs.first.assign(np, 0);
    fs.count.assign(np, 0);
    fs.referenced.assign(np, 1);
    fs.where.assign(np, WAX_VS_NO_FILTER);
    fs.allowed.assign(np, 0);
    modes.assign(np, 0);
    std::vector<uint32_t> listed_by_device, term_units, group_units;
    for (uint32_t p = 0; p < np; ++p) {
        const uint32_t w = pairs[p].first, f = pairs[p].second;
        const uint32_t *rows = f == WAX_VS_NO_FILTER ? nullptr : ids.rows.data() + ids.first[f];
        const uint64_t n_listed = f == WAX_VS_NO_FILTER ? 0 : ids.count[f];
        fs.first[p] = fs.rows.size();
        if (w == WAX_VS_NO_FILTER) {                               // the id filter as it is
            fs.rows.insert(fs.rows.end(), rows, rows + n_listed);
            fs.count[p] = n_listed;
            modes[p] = filter_modes[f];
            continue;
        }
        if (!wheres[w].groups.empty() && (f == WAX_VS_NO_FILTER || filter_modes[f] == 1)) {  // listed from the group index
            group_units.push_back(p);
            continue;
        }
        if (!wheres[w].terms.empty() && (f == WAX_VS_NO_FILTER || filter_modes[f] == 1)) {   // listed from the postings
            term_units.push_back(p);
            continue;
        }
        host_rows_passing(e, wheres[w], rows, n_listed, fs.rows);
        fs.count[p] = fs.rows.size() - fs.first[p];
        if (f != WAX_VS_NO_FILTER && filter_modes[f] == 0) continue;          // allow-list AND where: an allow-list
        const uint64_t pass = passing[slot[w]];
        if (fs.count[p] == 0 && pass > 0 && pass <= kWhereGatherRows) {       // narrow: the device lists the rows
            fs.count[p] = pass;
            fs.compact.push_back(where_item(wheres[w]));
            listed_by_device.push_back(p);
            continue;
        }
        modes[p] = 1;                                                         // deny the listed rows that pass ...
        fs.where[p] = static_cast<uint32_t>(fs.preds.size());                 // ... within the rows that pass
        fs.preds.push_back(where_item(wheres[w]));
        fs.allowed[p] = pass - fs.count[p];
    }
    uint64_t at = fs.rows.size();                                             // device-listed rows follow the host's
    for (size_t j = 0; j < listed_by_device.size(); ++j) {
        const uint32_t p = listed_by_device[j];
        fs.first[p] = at;
        fs.compact[j].slot = at;
        at += fs.count[p];
    }
    if (!term_units.empty() && (rc = plan_term_units(e, c, wheres, ids, pairs, term_units, fs, at))) return rc;
    if (!group_units.empty() && (rc = plan_group_units(e, c, wheres, ids, pairs, group_units, fs, at))) return rc;
    fs.device_rows = at - fs.rows.size();
    return WAX_VS_OK;
}

// The planning step of every filtered, where and grouped search on this engine: the request's id filters resolved to
// rows, then its (where, id filter) pairs planned as the filters of wp.fs (plan_where_pairs, which runs the count pass
// on c's stream), then each query's k at most clamp(k) and its class (plan_filtered; skipped with plan_queries = false,
// as round 2 of the sharded grouped search needs no classes).  A request without a where list plans its id filters as
// they are, in filter order.
static int32_t plan_request(wax_vs_engine *e, SearchCtx *c, const SearchRequest &req, int64_t k, WherePlan &wp,
                            bool plan_queries = true) {
    if (req.query_where) {
        resolve_filters(e, req.frame_ids, req.filter_offsets, req.n_filters, req.query_filter, req.n_queries, wp.ids);
        if (const int32_t rc = plan_where_pairs(e, c, req.wheres, req.query_where, req.filter_modes, req.query_filter,
                                                req.n_queries, wp.ids, wp.fs, wp.modes, wp.pair_of))
            return rc;
    } else {
        resolve_filters(e, req.frame_ids, req.filter_offsets, req.n_filters, req.query_filter, req.n_queries, wp.fs);
        wp.modes.assign(req.filter_modes, req.filter_modes + req.n_filters);
        wp.pair_of.assign(req.query_filter, req.query_filter + req.n_queries);
    }
    if (plan_queries) plan_filtered(e, k, wp.modes.data(), wp.pair_of.data(), req.n_queries, wp.fs, wp.plan);
    return WAX_VS_OK;
}

// The filtered and where entry points on one engine, after their argument checks.
static int32_t search_where_host(wax_vs_engine *e, const SearchRequest &req, uint64_t *out_ids, float *out_scores,
                                 uint32_t out_stride, uint32_t *out_n) {
    int32_t rc;
    std::shared_lock<std::shared_mutex> r(e->rw);
    for (uint32_t i = 0; i < req.n_queries; ++i) out_n[i] = 0;
    if (e->n_rows == 0 || req.n_queries == 0) return WAX_VS_OK;
    if ((rc = check_query(e, req.queries, req.query_len))) return rc;
    DeviceGuard g(e->device);
    if (!g.ok) return g.error();
    CtxLease lease(e);
    if ((rc = lease.acquire())) return rc;
    WherePlan wp;
    if ((rc = plan_request(e, lease.c, req, req.top_k, wp))) return rc;
    const uint32_t k_max = wp.plan.k_max;
    if (k_max == 0) return WAX_VS_OK;
    if (!out_ids || !out_scores) return fail(WAX_VS_ERR_NULL, "output buffer is NULL");
    if (out_stride < k_max) return fail(WAX_VS_ERR_BUFFER, "output buffers hold %u entries, need %u", out_stride, k_max);
    return deliver_filtered(e, lease.c, req.queries, wp, out_ids, out_scores, out_stride, out_n);
}

// The filtered and where entry points after their argument checks: on one engine, or across the shards of a
// multi-device handle, which first zeroes out_n as one engine does.
static int32_t search_where(wax_vs_engine *e, const SearchRequest &req, uint64_t *out_ids, float *out_scores,
                            uint32_t out_stride, uint32_t *out_n) {
    if (!e->multi) return search_where_host(e, req, out_ids, out_scores, out_stride, out_n);
    for (uint32_t i = 0; i < req.n_queries; ++i) out_n[i] = 0;
    return multi_search_where(e->multi, e->dims, e->similarity, req, out_ids, out_scores, out_stride, out_n);
}

// The request's per-query wheres: query i names where query_where[i] of n_wheres, whose clauses one of the builders
// below makes.
static int32_t request_where_list(SearchRequest &r, const void *wheres, uint32_t n_wheres, const uint32_t *query_where) {
    if ((n_wheres && !wheres) || (r.n_queries && !query_where)) return fail(WAX_VS_ERR_NULL, "NULL argument");
    for (uint32_t i = 0; i < r.n_queries; ++i)
        if (query_where[i] != WAX_VS_NO_FILTER && query_where[i] >= n_wheres)
            return fail(WAX_VS_ERR_ARGUMENT, "query %u names where %u of %u", i, query_where[i], n_wheres);
    r.query_where = query_where;
    return WAX_VS_OK;
}

// The time and tag clauses of wheres[0, n_wheres), no location, no terms.
static void request_plain_clauses(SearchRequest &r, const wax_vs_where *wheres, uint32_t n_wheres) {
    r.wheres.resize(n_wheres);
    for (uint32_t w = 0; w < n_wheres; ++w) r.wheres[w] = Clause{where_pred(wheres[w]), kNoLocBox, {}};
}

// The request's where, if it has one, for every query.
static void request_one_where(SearchRequest &r) {
    r.where_of.assign(r.n_queries, r.wheres.empty() ? WAX_VS_NO_FILTER : 0u);
    r.query_where = r.where_of.data();
}

int32_t wax_vs_search_filtered(wax_vs_engine *e, const float *query, uint32_t query_len, int64_t top_k,
                               const uint64_t *frame_ids, uint64_t n_ids, int32_t mode, uint64_t *out_ids,
                               float *out_scores, uint32_t out_cap, uint32_t *out_n) {
    return wax_vs_search_batch_filtered(e, query, 1, query_len, top_k, frame_ids, n_ids, mode, out_ids, out_scores, out_cap,
                                        out_n);
}

int32_t wax_vs_search_batch_filtered(wax_vs_engine *e, const float *queries, uint32_t n_queries, uint32_t query_len,
                                     int64_t top_k, const uint64_t *frame_ids, uint64_t n_ids, int32_t mode,
                                     uint64_t *out_ids, float *out_scores, uint32_t out_stride, uint32_t *out_n) {
    if (!e || !out_n) return fail(WAX_VS_ERR_NULL, "NULL argument");
    SearchRequest req(queries, n_queries, query_len, top_k);
    const int32_t rc = request_one_filter(req, frame_ids, n_ids, mode, false);
    return rc ? rc : search_where(e, req, out_ids, out_scores, out_stride, out_n);
}

int32_t wax_vs_search_batch_multi_filtered(wax_vs_engine *e, const float *queries, uint32_t n_queries, uint32_t query_len,
                                           int64_t top_k, const uint64_t *frame_ids, const uint64_t *filter_offsets,
                                           const int32_t *filter_modes, uint32_t n_filters, const uint32_t *query_filter,
                                           uint64_t *out_ids, float *out_scores, uint32_t out_stride, uint32_t *out_n) {
    if (!e || !out_n) return fail(WAX_VS_ERR_NULL, "NULL argument");
    SearchRequest req(queries, n_queries, query_len, top_k);
    const int32_t rc = request_filters(req, frame_ids, filter_offsets, filter_modes, n_filters, query_filter);
    return rc ? rc : search_where(e, req, out_ids, out_scores, out_stride, out_n);
}

int32_t wax_vs_search_batch_where(wax_vs_engine *e, const float *queries, uint32_t n_queries, uint32_t query_len,
                                  int64_t top_k, const uint64_t *frame_ids, const uint64_t *filter_offsets,
                                  const int32_t *filter_modes, uint32_t n_filters, const uint32_t *query_filter,
                                  const wax_vs_where *wheres, uint32_t n_wheres, const uint32_t *query_where,
                                  uint64_t *out_ids, float *out_scores, uint32_t out_stride, uint32_t *out_n) {
    if (!e || !out_n) return fail(WAX_VS_ERR_NULL, "NULL argument");
    SearchRequest req(queries, n_queries, query_len, top_k);
    int32_t rc;
    if ((rc = request_filters(req, frame_ids, filter_offsets, filter_modes, n_filters, query_filter)) ||
        (rc = request_where_list(req, wheres, n_wheres, query_where)))
        return rc;
    request_plain_clauses(req, wheres, n_wheres);
    return search_where(e, req, out_ids, out_scores, out_stride, out_n);
}

// ---- location predicates: PhotoRAG's location box beside the time and tag clauses (waxvs_where.cuh) -----------------
constexpr double kSwiftPi = 3.141592653589793;   // Double.pi
// Swift's min / max (the second operand wins only when it compares so; a NaN operand then loses to the first).
static double swift_min(double x, double y) { return y < x ? y : x; }
static double swift_max(double x, double y) { return y >= x ? y : x; }
// Int(x) for x = floor(...): false where Swift traps (NaN, infinite or outside Int64).
static bool swift_int(double x, int64_t *out) {
    if (!(x >= -9223372036854775808.0 && x < 9223372036854775808.0)) return false;
    *out = static_cast<int64_t>(x);
    return true;
}
static int32_t saturate_bin(double x) {          // floor(v * 100) of a finite v; no box reaches past +-36 000
    return x >= 2147483647.0 ? INT32_MAX : (x <= -2147483647.0 ? -INT32_MAX : static_cast<int32_t>(x));
}

// PhotoLocationQuery / PhotoCoordinate (PhotoRAGTypes.swift:33-57) and buildLocationAllowlist
// (PhotoRAGOrchestrator.swift:788-854) in fp64: the box of bins, or *active = false where Swift returns nil (no location
// clause; *box is then kNoLocBox).  out4 (optional) = {minLatBin, maxLatBin, minLonBin, maxLonBin} of an active box.
static int32_t location_box(double lat, double lon, double radius_m, LocBox *box, bool *active, int32_t *out4 = nullptr) {
    *box = kNoLocBox;
    *active = false;
    lat = swift_min(90.0, swift_max(-90.0, lat));
    lon = swift_min(180.0, swift_max(-180.0, lon));
    const double radius = swift_max(0.0, radius_m);
    if (!(radius > 0)) return WAX_VS_OK;
    const double lat_delta = radius / 111000.0;
    const double lon_delta = swift_min(180.0, radius / swift_max(1e-6, 111000.0 * std::cos(lat * kSwiftPi / 180)));
    int64_t b[4];
    if (!swift_int(std::floor((lat - lat_delta) * 100.0), &b[0]) || !swift_int(std::floor((lat + lat_delta) * 100.0), &b[1]) ||
        !swift_int(std::floor((lon - lon_delta) * 100.0), &b[2]) || !swift_int(std::floor((lon + lon_delta) * 100.0), &b[3]))
        return fail(WAX_VS_ERR_ARGUMENT, "location box of (%g, %g, %g m) is not representable", lat, lon, radius_m);
    const int64_t min_lat = std::max<int64_t>(-9000, b[0]), max_lat = std::min<int64_t>(9000, b[1]);
    const int64_t min_lon = b[2], max_lon = b[3];                    // |bin| <= 36 000: lon in [-180, 180], delta <= 180
    const int64_t lat_count = max_lat - min_lat + 1;
    const int64_t lon_count = min_lon <= max_lon ? max_lon - min_lon + 1 : (18000 - min_lon) + (max_lon + 18000) + 1;
    if (lat_count <= 0 || lon_count <= 0 || lat_count * lon_count >= 100000) return WAX_VS_OK;
    const int32_t lo = static_cast<int32_t>(min_lon), hi = static_cast<int32_t>(max_lon);
    *box = min_lon <= max_lon ? LocBox{static_cast<int32_t>(min_lat), static_cast<int32_t>(max_lat), lo, hi, 1, 0}
                              : LocBox{static_cast<int32_t>(min_lat), static_cast<int32_t>(max_lat), lo, 18000, -18000, hi};
    *active = true;
    if (out4) {
        out4[0] = static_cast<int32_t>(min_lat); out4[1] = static_cast<int32_t>(max_lat);
        out4[2] = lo; out4[3] = hi;
    }
    return WAX_VS_OK;
}

int32_t wax_vs_location_box(double latitude, double longitude, double radius_m, int32_t out_box[4], int32_t *out_active) {
    if (!out_box || !out_active) return fail(WAX_VS_ERR_NULL, "NULL argument");
    LocBox box;
    bool active;
    out_box[0] = out_box[1] = out_box[2] = out_box[3] = 0;
    *out_active = 0;
    int32_t rc;
    if ((rc = location_box(latitude, longitude, radius_m, &box, &active, out_box))) return rc;
    *out_active = active ? 1 : 0;
    return WAX_VS_OK;
}

// locationBin(from:) (PhotoRAGOrchestrator.swift:868-875): a NaN pair is "no location"; any other non-finite coordinate
// is an argument error.
static int32_t location_bin(double lat, double lon, LocRow *out) {
    if (std::isnan(lat) && std::isnan(lon)) { *out = LocRow{kNoLocation, 0}; return WAX_VS_OK; }
    if (!std::isfinite(lat) || !std::isfinite(lon))
        return fail(WAX_VS_ERR_ARGUMENT, "location (%g, %g) is not finite (a NaN pair clears a location)", lat, lon);
    *out = LocRow{saturate_bin(std::floor(lat * 100.0)), saturate_bin(std::floor(lon * 100.0))};
    return WAX_VS_OK;
}

int32_t wax_vs_location_bin(double latitude, double longitude, int32_t out_bin[2], int32_t *out_has) {
    if (!out_bin || !out_has) return fail(WAX_VS_ERR_NULL, "NULL argument");
    LocRow l{kNoLocation, 0};
    int32_t rc;
    if ((rc = location_bin(latitude, longitude, &l))) return rc;
    *out_has = l.lat != kNoLocation;
    out_bin[0] = *out_has ? l.lat : 0;
    out_bin[1] = *out_has ? l.lon : 0;
    return WAX_VS_OK;
}

// Upsert by frame id as set_attributes; every coordinate pair is checked before anything is written.
int32_t wax_vs_set_locations(wax_vs_engine *e, const uint64_t *frame_ids, const double *latitudes, const double *longitudes,
                             uint64_t n, uint64_t *out_assigned) {
    if (e && e->multi) return multi_set(e->multi, out_assigned, [&](wax_vs_engine *s, uint64_t *got) { return wax_vs_set_locations(s, frame_ids, latitudes, longitudes, n, got); });
    if (!e) return fail(WAX_VS_ERR_NULL, "engine is NULL");
    if (out_assigned) *out_assigned = 0;
    if (n == 0) return WAX_VS_OK;
    if (!frame_ids || !latitudes || !longitudes) return fail(WAX_VS_ERR_NULL, "NULL argument");
    std::vector<LocRow> bins(n);
    int32_t rc;
    for (uint64_t i = 0; i < n; ++i)
        if ((rc = location_bin(latitudes[i], longitudes[i], &bins[i]))) return rc;
    std::unique_lock<std::shared_mutex> w(e->rw);
    DeviceGuard g(e->device);
    drain_device_path(e);
    if (!e->locs_set) {                // from implicit (no row has a location) to an explicit column
        e->locs.assign(e->n_rows, LocRow{kNoLocation, 0});
        e->locs_set = true;
    }
    std::vector<uint32_t> written(static_cast<size_t>((e->n_rows + 31) / 32), 0u);
    uint64_t assigned = 0;
    for (uint64_t i = 0; i < n; ++i) {
        const uint32_t row = row_of(e, frame_ids[i]);
        if (row == 0xFFFFFFFFu) continue;                // unknown frame: ignored
        e->locs[row] = bins[i];                          // a later entry for the same frame wins
        const uint32_t wd = row >> 5, b = 1u << (row & 31u);
        if (!(written[wd] & b)) { written[wd] |= b; ++assigned; }
    }
    e->locs_dev_valid = false;
    if (out_assigned) *out_assigned = assigned;
    return WAX_VS_OK;
}

// The clauses of wheres[0, n_wheres): the time and tag clauses and the location box of each, no terms.
static int32_t near_clauses(const wax_vs_where_near *wheres, uint32_t n_wheres, std::vector<Clause> &clauses) {
    clauses.resize(n_wheres);
    for (uint32_t i = 0; i < n_wheres; ++i) {
        clauses[i].pred = where_pred(wheres[i].where);
        bool active;
        int32_t rc;
        if ((rc = location_box(wheres[i].latitude, wheres[i].longitude, wheres[i].radius_m, &clauses[i].box, &active)))
            return rc;
    }
    return WAX_VS_OK;
}

int32_t wax_vs_search_batch_where_near(wax_vs_engine *e, const float *queries, uint32_t n_queries, uint32_t query_len,
                                       int64_t top_k, const uint64_t *frame_ids, const uint64_t *filter_offsets,
                                       const int32_t *filter_modes, uint32_t n_filters, const uint32_t *query_filter,
                                       const wax_vs_where_near *wheres, uint32_t n_wheres, const uint32_t *query_where,
                                       uint64_t *out_ids, float *out_scores, uint32_t out_stride, uint32_t *out_n) {
    if (!e || !out_n) return fail(WAX_VS_ERR_NULL, "NULL argument");
    SearchRequest req(queries, n_queries, query_len, top_k);
    int32_t rc;
    if ((rc = request_filters(req, frame_ids, filter_offsets, filter_modes, n_filters, query_filter)) ||
        (rc = request_where_list(req, wheres, n_wheres, query_where)) || (rc = near_clauses(wheres, n_wheres, req.wheres)))
        return rc;
    return search_where(e, req, out_ids, out_scores, out_stride, out_n);
}

// ---- term clauses: Wax's metadataFilter as required term ids, from an inverted index (waxvs_terms.cuh) ---------------
// Offsets of n lists: start at 0, never decrease; with max_len, no list is longer.
static int32_t check_term_offsets(const uint64_t *offsets, uint64_t n, const uint64_t *terms, uint64_t max_len,
                                  const char *what) {
    if (offsets[0] != 0) return fail(WAX_VS_ERR_ARGUMENT, "%s[0] must be 0", what);
    for (uint64_t i = 0; i < n; ++i) {
        if (offsets[i + 1] < offsets[i])
            return fail(WAX_VS_ERR_ARGUMENT, "%s decrease at list %llu", what, static_cast<unsigned long long>(i));
        if (offsets[i + 1] - offsets[i] > max_len)
            return fail(WAX_VS_ERR_ARGUMENT, "%s: list %llu has %llu terms, at most %llu are allowed", what,
                        static_cast<unsigned long long>(i), static_cast<unsigned long long>(offsets[i + 1] - offsets[i]),
                        static_cast<unsigned long long>(max_len));
    }
    if (offsets[n] && !terms) return fail(WAX_VS_ERR_NULL, "term list is NULL");
    return WAX_VS_OK;
}

// Replace each named frame's whole term set (upsert by frame id, as set_locations); every list is checked before anything
// is written.  The new list goes to the end of the pool, the row is repointed, and the pool is compacted when more than
// half of it is garbage.
int32_t wax_vs_set_terms(wax_vs_engine *e, const uint64_t *frame_ids, const uint64_t *term_offsets, const uint64_t *terms,
                         uint64_t n, uint64_t *out_assigned) {
    if (e && e->multi) return multi_set(e->multi, out_assigned, [&](wax_vs_engine *s, uint64_t *got) { return wax_vs_set_terms(s, frame_ids, term_offsets, terms, n, got); });
    if (!e) return fail(WAX_VS_ERR_NULL, "engine is NULL");
    if (out_assigned) *out_assigned = 0;
    if (!term_offsets) return fail(WAX_VS_ERR_NULL, "term_offsets is NULL");
    if (n && !frame_ids) return fail(WAX_VS_ERR_NULL, "frame_ids is NULL");
    int32_t rc;
    if ((rc = check_term_offsets(term_offsets, n, terms, UINT32_MAX, "term_offsets"))) return rc;
    if (n == 0) return WAX_VS_OK;
    std::unique_lock<std::shared_mutex> w(e->rw);
    DeviceGuard g(e->device);
    drain_device_path(e);
    if (!e->terms_set) {               // from implicit (no row has a term) to explicit lists
        e->term_refs.assign(e->n_rows, wax_vs_engine::TermRef{0, 0});
        e->terms_set = true;
    }
    std::vector<uint32_t> written(static_cast<size_t>((e->n_rows + 31) / 32), 0u);
    std::vector<uint64_t> list;
    uint64_t assigned = 0;
    for (uint64_t i = 0; i < n; ++i) {
        const uint32_t row = row_of(e, frame_ids[i]);
        if (row == 0xFFFFFFFFu) continue;                // unknown frame: ignored
        list.assign(terms + term_offsets[i], terms + term_offsets[i + 1]);
        std::sort(list.begin(), list.end());
        list.erase(std::unique(list.begin(), list.end()), list.end());
        auto &ref = e->term_refs[row];                   // a later entry for the same frame wins
        e->term_garbage += ref.n;
        ref = wax_vs_engine::TermRef{list.empty() ? 0 : e->term_pool.size(), static_cast<uint32_t>(list.size())};
        e->term_pool.insert(e->term_pool.end(), list.begin(), list.end());
        const uint32_t wd = row >> 5, b = 1u << (row & 31u);
        if (!(written[wd] & b)) { written[wd] |= b; ++assigned; }
    }
    compact_term_pool(e);
    e->tindex.release();
    if (out_assigned) *out_assigned = assigned;
    return WAX_VS_OK;
}

// lists[offsets[w], offsets[w + 1]) of each where w, sorted and deduplicated, into (r.wheres[w].*field).
static void request_id_lists(SearchRequest &r, uint32_t n_wheres, const uint64_t *offsets, const uint64_t *lists,
                             std::vector<uint64_t> Clause::*field) {
    for (uint32_t w = 0; w < n_wheres; ++w) {
        std::vector<uint64_t> &ids = r.wheres[w].*field;
        ids.assign(lists + offsets[w], lists + offsets[w + 1]);
        std::sort(ids.begin(), ids.end());
        ids.erase(std::unique(ids.begin(), ids.end()), ids.end());
    }
}

// With a where list, wheres with terms or groups and equal contents (clauses, box, root clause, required ids, group ids)
// are one: each query names the first of them, so a batch that scopes 1 024 queries to 16 sessions plans 16 units, not
// 1 024.
static void canonical_wheres(SearchRequest &r) {
    if (!r.query_where) return;
    const uint32_t n_wheres = static_cast<uint32_t>(r.wheres.size());
    std::vector<uint32_t> canon(n_wheres);
    std::unordered_map<std::string, uint32_t> first_of;
    for (uint32_t w = 0; w < n_wheres; ++w) {
        const Clause &cl = r.wheres[w];
        canon[w] = w;
        if (cl.terms.empty() && cl.groups.empty()) continue;
        const uint64_t n_terms = cl.terms.size();
        std::string key(reinterpret_cast<const char *>(&cl.pred), sizeof(WherePred));
        key.append(reinterpret_cast<const char *>(&cl.box), sizeof(LocBox));
        key.append(reinterpret_cast<const char *>(&cl.root), sizeof(RootClause));
        key.append(reinterpret_cast<const char *>(&n_terms), sizeof(n_terms));
        key.append(reinterpret_cast<const char *>(cl.terms.data()), cl.terms.size() * sizeof(uint64_t));
        key.append(reinterpret_cast<const char *>(cl.groups.data()), cl.groups.size() * sizeof(uint64_t));
        canon[w] = first_of.emplace(std::move(key), w).first->second;
    }
    r.where_of.resize(r.n_queries);
    for (uint32_t i = 0; i < r.n_queries; ++i)
        r.where_of[i] = r.query_where[i] == WAX_VS_NO_FILTER ? WAX_VS_NO_FILTER : canon[r.query_where[i]];
    r.query_where = r.where_of.data();
}

// The clauses of wheres[0, n_wheres) with their term lists, equal wheres made one (canonical_wheres).
static int32_t request_term_clauses(SearchRequest &r, const wax_vs_where_near *wheres, uint32_t n_wheres,
                                    const uint64_t *where_term_offsets, const uint64_t *where_terms) {
    int32_t rc;
    if ((rc = check_term_offsets(where_term_offsets, n_wheres, where_terms, kMaxWhereTerms, "where_term_offsets"))) return rc;
    if ((rc = near_clauses(wheres, n_wheres, r.wheres))) return rc;
    request_id_lists(r, n_wheres, where_term_offsets, where_terms, &Clause::terms);
    canonical_wheres(r);
    return WAX_VS_OK;
}

int32_t wax_vs_search_batch_where_terms(wax_vs_engine *e, const float *queries, uint32_t n_queries, uint32_t query_len,
                                        int64_t top_k, const uint64_t *frame_ids, const uint64_t *filter_offsets,
                                        const int32_t *filter_modes, uint32_t n_filters, const uint32_t *query_filter,
                                        const wax_vs_where_near *wheres, uint32_t n_wheres, const uint32_t *query_where,
                                        const uint64_t *where_term_offsets, const uint64_t *where_terms,
                                        uint64_t *out_ids, float *out_scores, uint32_t out_stride, uint32_t *out_n) {
    if (!e || !out_n) return fail(WAX_VS_ERR_NULL, "NULL argument");
    SearchRequest req(queries, n_queries, query_len, top_k);
    int32_t rc;
    if ((rc = request_filters(req, frame_ids, filter_offsets, filter_modes, n_filters, query_filter)) ||
        (rc = request_where_list(req, wheres, n_wheres, query_where)))
        return rc;
    if (!where_term_offsets) return fail(WAX_VS_ERR_NULL, "where_term_offsets is NULL");
    if ((rc = request_term_clauses(req, wheres, n_wheres, where_term_offsets, where_terms))) return rc;
    return search_where(e, req, out_ids, out_scores, out_stride, out_n);
}

// ---- group clauses: VideoRAG's videoIDs as "the row's group is one of these", from the group index -------------------
// (waxvs_where_groups.cuh).  The group offsets of n_wheres wheres: not NULL, start at 0, never decrease, at most
// kMaxWhereGroups ids in a where, and the ids not NULL when some where has one.  *any = some where has a group.
static int32_t check_group_offsets(const uint64_t *offsets, uint32_t n_wheres, const uint64_t *groups, bool *any) {
    if (!offsets) return fail(WAX_VS_ERR_NULL, "where_group_offsets is NULL");
    if (offsets[0] != 0) return fail(WAX_VS_ERR_ARGUMENT, "where_group_offsets[0] must be 0");
    for (uint32_t w = 0; w < n_wheres; ++w) {
        if (offsets[w + 1] < offsets[w]) return fail(WAX_VS_ERR_ARGUMENT, "where_group_offsets decrease at where %u", w);
        if (offsets[w + 1] - offsets[w] > kMaxWhereGroups)
            return fail(WAX_VS_ERR_ARGUMENT, "where %u has %llu group ids, at most %u are allowed", w,
                        static_cast<unsigned long long>(offsets[w + 1] - offsets[w]), kMaxWhereGroups);
    }
    if (offsets[n_wheres] && !groups) return fail(WAX_VS_ERR_NULL, "where_groups is NULL");
    *any = offsets[n_wheres] != 0;
    return WAX_VS_OK;
}

int32_t wax_vs_search_batch_where_groups(wax_vs_engine *e, const float *queries, uint32_t n_queries, uint32_t query_len,
                                         int64_t top_k, const uint64_t *frame_ids, const uint64_t *filter_offsets,
                                         const int32_t *filter_modes, uint32_t n_filters, const uint32_t *query_filter,
                                         const wax_vs_where_near *wheres, uint32_t n_wheres, const uint32_t *query_where,
                                         const uint64_t *where_term_offsets, const uint64_t *where_terms,
                                         const uint64_t *where_group_offsets, const uint64_t *where_groups,
                                         uint64_t *out_ids, float *out_scores, uint32_t out_stride, uint32_t *out_n) {
    if (!e || !out_n) return fail(WAX_VS_ERR_NULL, "NULL argument");
    SearchRequest req(queries, n_queries, query_len, top_k);
    int32_t rc;
    bool any = false;
    if ((rc = request_filters(req, frame_ids, filter_offsets, filter_modes, n_filters, query_filter)) ||
        (rc = request_where_list(req, wheres, n_wheres, query_where)) ||
        (rc = check_group_offsets(where_group_offsets, n_wheres, where_groups, &any)))
        return rc;
    if (!any)                          // no where has a group: the entry point without the clause
        return where_term_offsets
                   ? wax_vs_search_batch_where_terms(e, queries, n_queries, query_len, top_k, frame_ids, filter_offsets,
                                                     filter_modes, n_filters, query_filter, wheres, n_wheres, query_where,
                                                     where_term_offsets, where_terms, out_ids, out_scores, out_stride, out_n)
                   : wax_vs_search_batch_where_near(e, queries, n_queries, query_len, top_k, frame_ids, filter_offsets,
                                                    filter_modes, n_filters, query_filter, wheres, n_wheres, query_where,
                                                    out_ids, out_scores, out_stride, out_n);
    if (where_term_offsets) {
        if ((rc = check_term_offsets(where_term_offsets, n_wheres, where_terms, kMaxWhereTerms, "where_term_offsets")))
            return rc;
    }
    if ((rc = near_clauses(wheres, n_wheres, req.wheres))) return rc;
    if (where_term_offsets) request_id_lists(req, n_wheres, where_term_offsets, where_terms, &Clause::terms);
    request_id_lists(req, n_wheres, where_group_offsets, where_groups, &Clause::groups);
    canonical_wheres(req);
    return search_where(e, req, out_ids, out_scores, out_stride, out_n);
}

// ---- root clauses: PhotoRAG's and VideoRAG's test on each hit's root, as a word per group (waxvs_roots.cuh) -----------
// Upsert by group id: a later entry for the same id wins, and an id no row carries yet is kept for the rows that take it.
// The table is keyed by group, so no row mutator touches it.  A multi-device handle keeps the whole table on every shard
// (rebalance then has nothing to move) and reports one engine's count.
int32_t wax_vs_set_root_tags(wax_vs_engine *e, const uint64_t *group_ids, const uint64_t *tags, uint64_t n,
                             uint64_t *out_assigned) {
    if (e && e->multi) {
        const wax_vs_engine *first = e->multi->shards[0];
        return multi_set(e->multi, out_assigned, [&](wax_vs_engine *s, uint64_t *got) {
            return wax_vs_set_root_tags(s, group_ids, tags, n, s == first ? got : nullptr);
        });
    }
    if (!e) return fail(WAX_VS_ERR_NULL, "engine is NULL");
    if (out_assigned) *out_assigned = 0;
    if (n == 0) return WAX_VS_OK;
    if (!group_ids || !tags) return fail(WAX_VS_ERR_NULL, "NULL argument");
    // the call's distinct ids ascending, each with its last entry's word
    std::vector<uint64_t> order(n);
    for (uint64_t i = 0; i < n; ++i) order[i] = i;
    std::stable_sort(order.begin(), order.end(), [&](uint64_t a, uint64_t b) { return group_ids[a] < group_ids[b]; });
    std::vector<uint64_t> ids, words;
    for (uint64_t i = 0; i < n; ++i) {
        const uint64_t g = group_ids[order[i]];
        if (!ids.empty() && ids.back() == g) words.back() = tags[order[i]];
        else ids.push_back(g), words.push_back(tags[order[i]]);
    }
    std::unique_lock<std::shared_mutex> w(e->rw);
    DeviceGuard g(e->device);
    drain_device_path(e);
    auto &rt = e->roots;
    std::vector<uint64_t> m_ids, m_tags;            // the table merged with the call's entries, which win
    m_ids.reserve(rt.ids.size() + ids.size());
    m_tags.reserve(rt.ids.size() + ids.size());
    size_t i = 0, j = 0;
    while (i < rt.ids.size() || j < ids.size()) {
        if (j == ids.size() || (i < rt.ids.size() && rt.ids[i] < ids[j])) {
            m_ids.push_back(rt.ids[i]), m_tags.push_back(rt.tags[i]), ++i;
        } else {
            if (i < rt.ids.size() && rt.ids[i] == ids[j]) ++i;
            m_ids.push_back(ids[j]), m_tags.push_back(words[j]), ++j;
        }
    }
    rt.ids.swap(m_ids);
    rt.tags.swap(m_tags);
    rt.col_valid = false;
    if (out_assigned) *out_assigned = ids.size();
    return WAX_VS_OK;
}

// The root clauses of n_wheres wheres into r.wheres (NULL: none).  *any = some where has one.
static void request_root_clauses(SearchRequest &r, const wax_vs_root_clause *roots, uint32_t n_wheres, bool *any) {
    *any = false;
    if (!roots) return;
    for (uint32_t w = 0; w < n_wheres; ++w) {
        r.wheres[w].root = RootClause{roots[w].all_tags, roots[w].no_tags};
        *any = *any || root_active(r.wheres[w].root);
    }
}

int32_t wax_vs_search_batch_where_roots(wax_vs_engine *e, const float *queries, uint32_t n_queries, uint32_t query_len,
                                        int64_t top_k, const uint64_t *frame_ids, const uint64_t *filter_offsets,
                                        const int32_t *filter_modes, uint32_t n_filters, const uint32_t *query_filter,
                                        const wax_vs_where_near *wheres, uint32_t n_wheres, const uint32_t *query_where,
                                        const uint64_t *where_term_offsets, const uint64_t *where_terms,
                                        const uint64_t *where_group_offsets, const uint64_t *where_groups,
                                        const wax_vs_root_clause *where_roots, uint64_t *out_ids, float *out_scores,
                                        uint32_t out_stride, uint32_t *out_n) {
    if (!e || !out_n) return fail(WAX_VS_ERR_NULL, "NULL argument");
    SearchRequest req(queries, n_queries, query_len, top_k);
    int32_t rc;
    bool any_group = false, any_root = false;
    if ((rc = request_filters(req, frame_ids, filter_offsets, filter_modes, n_filters, query_filter)) ||
        (rc = request_where_list(req, wheres, n_wheres, query_where)) ||
        (rc = check_group_offsets(where_group_offsets, n_wheres, where_groups, &any_group)) ||
        (where_term_offsets &&
         (rc = check_term_offsets(where_term_offsets, n_wheres, where_terms, kMaxWhereTerms, "where_term_offsets"))) ||
        (rc = near_clauses(wheres, n_wheres, req.wheres)))
        return rc;
    request_root_clauses(req, where_roots, n_wheres, &any_root);
    if (!any_root)                     // no where has a root clause: the entry point without the clause
        return wax_vs_search_batch_where_groups(e, queries, n_queries, query_len, top_k, frame_ids, filter_offsets,
                                                filter_modes, n_filters, query_filter, wheres, n_wheres, query_where,
                                                where_term_offsets, where_terms, where_group_offsets, where_groups, out_ids,
                                                out_scores, out_stride, out_n);
    if (where_term_offsets) request_id_lists(req, n_wheres, where_term_offsets, where_terms, &Clause::terms);
    request_id_lists(req, n_wheres, where_group_offsets, where_groups, &Clause::groups);
    canonical_wheres(req);
    return search_where(e, req, out_ids, out_scores, out_stride, out_n);
}

// ---- sharded where search -----------------------------------------------------------------------------------------
// The scratch of a collective where search on c, sized before the call plans anything for the bounds of one query on
// this shard: one unit of at most n_rows listed rows, at most kWhereGatherRows gathered, kMaxWhereTerms required ids.
// A buffer that grew during the call would free its old memory, and cudaFree waits for the whole device, where a peer's
// exchange may already be waiting for this rank (ranks that share a GPU).  Mutators release the row-sized ones under the
// write lock (invalidate_row_caches), so this only ever allocates.
static int32_t reserve_shard_scratch(wax_vs_engine *e, SearchCtx *c) {
    const size_t rows = std::max<size_t>(e->n_rows, 1), words = (rows + 31) / 32;
    int32_t rc;
    if ((rc = c->d_queries.ensure(e->dims, "query buffer")) || (rc = c->h_queries.ensure(e->dims, "query staging")) ||
        (rc = c->d_out.ensure(kShardKCap, "result buffer")) || (rc = c->d_shard_local.ensure(kShardKCap, "shard candidates")) ||
        (rc = c->d_filter_rows.ensure(rows, "filter rows")) || (rc = c->d_mask.ensure(words, "row filters")) ||
        (rc = c->d_filter_spec.ensure(4, "filter spec")) || (rc = c->d_query_filter.ensure(1, "query filters")) ||
        (rc = c->d_gather_span.ensure(1, "gather spans")) || (rc = c->d_gather_keys.ensure(kWhereGatherRows, "gather keys")) ||
        (rc = c->d_where_items.ensure(1, "where predicates")) || (rc = c->d_where_counts.ensure(1, "where counts")) ||
        (rc = c->d_term_ids.ensure(kMaxWhereTerms, "required terms")) ||
        (rc = c->d_term_spans.ensure(kMaxWhereTerms, "term spans")) || (rc = c->d_term_units.ensure(1, "term units")) ||
        (rc = c->d_term_counts.ensure(1, "term counts")) || (rc = c->d_term_deny.ensure(rows, "term deny-lists")))
        return rc;
    return WAX_VS_OK;
}

// The host-path collective search of the shard entry points, under the read lock it takes (caller: e and out_n checked,
// the request built).  A request without an id filter (wax_vs_shard_search): the rank's fused scan, the in-kernel
// exchange and merge, the merged list delivered into mapped host memory.  Otherwise the rank plans its shard for the one
// query as the where entry points do and runs the plan with exactly one exchange: a gathered unit is exchanged by the
// stand-alone kernel, a row bitset rides in the fused scan, and a shard where nothing passes exchanges padding.
static int32_t shard_search_host(wax_vs_engine *e, const SearchRequest &req, uint64_t *out_ids, float *out_scores,
                                 uint32_t out_cap, uint32_t *out_n) {
    std::shared_lock<std::shared_mutex> r(e->rw);
    *out_n = 0;
    if (!e->shard.connected) return fail(WAX_VS_ERR_ARGUMENT, "the shard group is not connected (wax_vs_shard_open / _connect)");
    int32_t rc;
    if ((rc = check_query(e, req.queries, req.query_len))) return rc;
    const uint32_t k_eff = clamp_topk(req.top_k);
    if (k_eff > static_cast<uint32_t>(kShardKCap))
        return fail(WAX_VS_ERR_UNSUPPORTED, "sharded search supports top_k <= %d (got %u)", kShardKCap, k_eff);
    if (!out_ids || !out_scores) return fail(WAX_VS_ERR_NULL, "output buffer is NULL");
    DeviceGuard g(e->device);
    if (!g.ok) return g.error();
    auto &sh = e->shard;
    std::lock_guard<std::mutex> sg(sh.mu);      // one host-path collective at a time: it owns sh.ctx and h_final
    SearchCtx *c = sh.ctx;
    c->row_keys = device_row_keys(e);
    const uint64_t *d_ids = nullptr;
    if ((rc = sync_device_ids(e, &d_ids))) return rc;
    uint64_t launches = 0;
    const bool planned = req.query_filter != nullptr;
    WherePlan wp;
    if (planned && e->n_rows &&
        ((rc = reserve_shard_scratch(e, c)) || (rc = plan_request(e, c, req, k_eff, wp))))
        return rc;
    FilteredPlan &plan = wp.plan;
    ShardParams sp = shard_params_next(e);
    sp.host_out = sh.h_final; sp.host_flag = sh.h_flag;      // mapped pinned: the kernel delivers the result itself
    if (!planned) {
        HostDelivery hd{req.queries, nullptr, nullptr, 0};       // the query rides in the kernel parameters when it fits
        rc = enqueue_search(e, c, nullptr, k_eff, sh.row_offset, sh.d_final, d_ids, c->stream, &launches, nullptr, &sp, &hd);
    } else if (plan.order.empty()) {                              // an empty shard, or nothing on it passes: padding
        sp.final_out = sh.d_final;
        if ((rc = c->d_shard_local.ensure(kShardKCap, "shard candidates"))) return rc;
        CUDA_TRY(cudaMemsetAsync(c->d_shard_local, 0, k_eff * sizeof(wax_vs_candidate), c->stream));
        rc = enqueue_exchange(sp, c->d_shard_local, k_eff, c->stream, &launches);
    } else {                    // every rank exchanges k_eff entries, its list padded past its allowed rows
        sp.final_out = sh.d_final;
        plan.k_max = plan.k_of[0] = k_eff;
        FilteredTarget tgt;
        tgt.row_offset = sh.row_offset; tgt.d_ids = d_ids; tgt.shard = &sp;
        rc = run_filtered(e, c, req.queries, wp, tgt);
    }
    if (rc) { cudaStreamSynchronize(c->stream); return rc; }
    if ((rc = shard_wait_host(e, sp.seq))) { cudaStreamSynchronize(c->stream); return rc; }
    if (planned) CUDA_TRY(cudaStreamSynchronize(c->stream));   // the host arrays must outlive their uploads
    uint32_t m = 0;
    for (uint32_t i = 0; i < k_eff; ++i) {
        const wax_vs_candidate &cd = sh.h_final[i];
        if (cd.valid != 1u) continue;
        if (m >= out_cap) return fail(WAX_VS_ERR_BUFFER, "output buffers hold %u entries, need more", out_cap);
        out_ids[m] = cd.frame_id;
        out_scores[m] = score_from_distance(e->similarity, cd.distance);
        ++m;
    }
    *out_n = m;
    return WAX_VS_OK;
}

int32_t wax_vs_shard_search_where(wax_vs_engine *e, const float *query, uint32_t query_len, int64_t top_k,
                                  const uint64_t *frame_ids, uint64_t n_ids, int32_t mode, const wax_vs_where_near *where,
                                  const uint64_t *terms, uint32_t n_terms, uint64_t *out_ids, float *out_scores,
                                  uint32_t out_cap, uint32_t *out_n) {
    WAX_VS_MULTI_REFUSE(e, "wax_vs_shard_search_where");
    if (!e || !out_n || !where) return fail(WAX_VS_ERR_NULL, "NULL argument");
    SearchRequest req(query, 1, query_len, top_k);
    const uint64_t term_offsets[2] = {0, n_terms};
    int32_t rc;
    if ((rc = request_one_filter(req, frame_ids, n_ids, mode, true)) ||
        (rc = request_term_clauses(req, where, 1, term_offsets, terms)))
        return rc;
    request_one_where(req);
    return shard_search_host(e, req, out_ids, out_scores, out_cap, out_n);
}

// The rank-local half of a batched sharded where search (wax_vs_search_batch_where_device, and each shard of a
// multi-device handle): the request's plan on this shard, run on the caller's stream with global rows and frame ids,
// then each planned query's list scattered to its place in d_candidates (every other slot is padding).
static int32_t search_where_device(wax_vs_engine *e, const SearchRequest &req, const float *d_queries, uint64_t row_offset,
                                   wax_vs_candidate *d_candidates, void *cuda_stream) {
    const uint32_t n_queries = req.n_queries;
    if (n_queries == 0) return WAX_VS_OK;
    std::shared_lock<std::shared_mutex> r(e->rw);
    DeviceGuard g(e->device);
    if (!g.ok) return g.error();
    SearchCtx *c = nullptr;
    int32_t rc;
    if ((rc = ctx_for_stream(e, cuda_stream, &c))) return rc;
    const uint32_t k_out = clamp_topk(req.top_k);
    e->async_pending.store(true);
    CUDA_TRY(cudaMemsetAsync(d_candidates, 0, static_cast<size_t>(n_queries) * k_out * sizeof(wax_vs_candidate), c->stream));
    if (e->n_rows == 0) return WAX_VS_OK;
    const uint64_t *d_ids = nullptr;
    if ((rc = sync_device_ids(e, &d_ids))) return rc;
    WherePlan wp;
    if ((rc = plan_request(e, c, req, req.top_k, wp))) return rc;
    const FilteredPlan &plan = wp.plan;
    if (plan.k_max == 0) return WAX_VS_OK;
    FilteredTarget tgt;
    tgt.row_offset = row_offset; tgt.d_ids = d_ids; tgt.device_queries = true;
    if ((rc = run_filtered(e, c, d_queries, wp, tgt))) return rc;
    const uint32_t n_staged = static_cast<uint32_t>(plan.order.size());
    const size_t total = static_cast<size_t>(n_staged) * plan.k_max;
    const int grid = static_cast<int>(std::max<size_t>(1, std::min<size_t>(static_cast<size_t>(e->sm_count) * 8, (total + 255) / 256)));
    scatter_candidates_kernel<<<grid, 256, 0, c->stream>>>(c->d_out, plan.k_max, c->d_order, c->d_order + n_staged, n_staged,
                                                           k_out, d_candidates);
    CUDA_TRY(cudaGetLastError());
    CUDA_TRY(cudaStreamSynchronize(c->stream));     // the host arrays of the plan must outlive their uploads
    return WAX_VS_OK;
}

// The plan of wax_vs_search_batch_where_terms (or of _near, without term lists) on this rank's shard.
int32_t wax_vs_search_batch_where_device(wax_vs_engine *e, const float *d_queries, uint32_t n_queries, int64_t top_k,
                                         const uint64_t *frame_ids, const uint64_t *filter_offsets,
                                         const int32_t *filter_modes, uint32_t n_filters, const uint32_t *query_filter,
                                         const wax_vs_where_near *wheres, uint32_t n_wheres, const uint32_t *query_where,
                                         const uint64_t *where_term_offsets, const uint64_t *where_terms,
                                         uint64_t row_offset, wax_vs_candidate *d_candidates, void *cuda_stream) {
    WAX_VS_MULTI_REFUSE(e, "wax_vs_search_batch_where_device");
    if (!e) return fail(WAX_VS_ERR_NULL, "NULL argument");
    SearchRequest req(nullptr, n_queries, e->dims, top_k);
    int32_t rc;
    if ((rc = request_filters(req, frame_ids, filter_offsets, filter_modes, n_filters, query_filter)) ||
        (rc = request_where_list(req, wheres, n_wheres, query_where)))
        return rc;
    if (!d_queries || !d_candidates) return fail(WAX_VS_ERR_NULL, "NULL argument");
    if ((rc = where_term_offsets ? request_term_clauses(req, wheres, n_wheres, where_term_offsets, where_terms)
                                 : near_clauses(wheres, n_wheres, req.wheres)))
        return rc;
    return search_where_device(e, req, d_queries, row_offset, d_candidates, cuda_stream);
}

// The row-sharded form: every rank passes the SAME ids; a rank resolves the ones its shard holds (the others are
// unknown to it and ignored), its fused scan consults the bitset below the top-k, and the usual in-kernel exchange
// merges the ranks' lists -- the answer is the filtered top-k of the whole corpus, identical on every rank.
int32_t wax_vs_shard_search_filtered(wax_vs_engine *e, const float *query, uint32_t query_len, int64_t top_k,
                                     const uint64_t *frame_ids, uint64_t n_ids, int32_t mode, uint64_t *out_ids,
                                     float *out_scores, uint32_t out_cap, uint32_t *out_n) {
    WAX_VS_MULTI_REFUSE(e, "wax_vs_shard_search_filtered");
    if (!e || !out_n) return fail(WAX_VS_ERR_NULL, "NULL argument");
    SearchRequest req(query, 1, query_len, top_k);
    const int32_t rc = request_one_filter(req, frame_ids, n_ids, mode, true);
    if (rc) return rc;
    request_one_where(req);
    return shard_search_host(e, req, out_ids, out_scores, out_cap, out_n);
}

// ---- grouped search (waxvs_group.cuh) -----------------------------------------------------------------------------
// PhotoRAG and VideoRAG group frames by parentId ?? id on the host after over-fetching frames
// (PhotoRAGOrchestrator.swift:244-308, VideoRAGOrchestrator.swift:252-350,406-440); here the grouping is exact and runs
// on the device over the emitting scan's per-row distance keys.

int32_t wax_vs_set_groups(wax_vs_engine *e, const uint64_t *frame_ids, const uint64_t *group_ids, uint64_t n,
                          uint64_t *out_assigned) {
    if (e && e->multi) return multi_set(e->multi, out_assigned, [&](wax_vs_engine *s, uint64_t *got) { return wax_vs_set_groups(s, frame_ids, group_ids, n, got); });
    if (!e) return fail(WAX_VS_ERR_NULL, "engine is NULL");
    if (out_assigned) *out_assigned = 0;
    if (n == 0) return WAX_VS_OK;
    if (!frame_ids || !group_ids) return fail(WAX_VS_ERR_NULL, "NULL argument");
    std::unique_lock<std::shared_mutex> w(e->rw);
    DeviceGuard g(e->device);
    drain_device_path(e);
    if (!e->groups_set) {              // from implicit (every row its own group) to an explicit array
        e->groups.resize(e->n_rows);
        for (uint64_t r = 0; r < e->n_rows; ++r) e->groups[r] = frame_id_of(e, r);
        e->groups_set = true;
    }
    std::vector<uint32_t> written(static_cast<size_t>((e->n_rows + 31) / 32), 0u);
    uint64_t assigned = 0;
    for (uint64_t i = 0; i < n; ++i) {
        const uint32_t row = row_of(e, frame_ids[i]);
        if (row == 0xFFFFFFFFu) continue;                // unknown frame: ignored
        e->groups[row] = group_ids[i];                   // a later entry for the same frame wins
        const uint32_t wd = row >> 5, b = 1u << (row & 31u);
        if (!(written[wd] & b)) { written[wd] |= b; ++assigned; }
    }
    e->gindex.valid = false;
    e->roots.col_valid = false;
    if (out_assigned) *out_assigned = assigned;
    return WAX_VS_OK;
}

// Frame attributes (waxvs_where.cuh): the timestamp and tag columns the where predicates test.  Upsert by frame id as
// set_groups: unknown ids are ignored, a later entry for the same frame wins, a NULL column is left as it is.
int32_t wax_vs_set_attributes(wax_vs_engine *e, const uint64_t *frame_ids, const int64_t *timestamps, const uint64_t *tags,
                              uint64_t n, uint64_t *out_assigned) {
    if (e && e->multi) return multi_set(e->multi, out_assigned, [&](wax_vs_engine *s, uint64_t *got) { return wax_vs_set_attributes(s, frame_ids, timestamps, tags, n, got); });
    if (!e) return fail(WAX_VS_ERR_NULL, "engine is NULL");
    if (out_assigned) *out_assigned = 0;
    if (n == 0) return WAX_VS_OK;
    if (!frame_ids) return fail(WAX_VS_ERR_NULL, "frame_ids is NULL");
    std::unique_lock<std::shared_mutex> w(e->rw);
    DeviceGuard g(e->device);
    drain_device_path(e);
    if (!e->attrs_set) {               // from implicit (every row 0, 0) to explicit arrays
        e->attrs.assign(e->n_rows, AttrRow{0, 0});
        e->attrs_set = true;
    }
    std::vector<uint32_t> written(static_cast<size_t>((e->n_rows + 31) / 32), 0u);
    uint64_t assigned = 0;
    for (uint64_t i = 0; i < n; ++i) {
        const uint32_t row = row_of(e, frame_ids[i]);
        if (row == 0xFFFFFFFFu) continue;                // unknown frame: ignored
        if (timestamps) e->attrs[row].ts = timestamps[i];
        if (tags) e->attrs[row].tags = tags[i];
        const uint32_t wd = row >> 5, b = 1u << (row & 31u);
        if (!(written[wd] & b)) { written[wd] |= b; ++assigned; }
    }
    e->attrs_dev_valid = false;
    if (out_assigned) *out_assigned = assigned;
    return WAX_VS_OK;
}

// The device group index of the current corpus and grouping, built on c's stream by the first grouped search after a
// mutation or set_groups: (group id, row) pairs radix-sorted by CUB (stable, so each group's rows stay in row order),
// group heads flagged and prefix-summed into dense group indices.  Readers hold the read lock; group_mu serialises the
// build, and the build completes before the index is published.
static int32_t ensure_group_index(wax_vs_engine *e, SearchCtx *c) {
    std::lock_guard<std::mutex> lk(e->group_mu);
    auto &gi = e->gindex;
    if (gi.valid) return WAX_VS_OK;
    const uint32_t n = static_cast<uint32_t>(e->n_rows);
    cudaStream_t s = c->stream;
    int32_t rc;
    const uint64_t *d_ids = nullptr;
    if (!e->groups_set && (rc = sync_device_ids(e, &d_ids))) return rc;
    DevBuf<uint64_t> keys_in, keys_out, d_groups;
    DevBuf<uint32_t> vals, incl;
    DevBuf<uint8_t> temp;
    size_t sort_bytes = 0, scan_bytes = 0;
    CUDA_TRY(cub::DeviceRadixSort::SortPairs(nullptr, sort_bytes, keys_in.p, keys_out.p, vals.p, gi.perm.p, static_cast<int>(n),
                                             0, 64, s));
    CUDA_TRY(cub::DeviceScan::InclusiveSum(nullptr, scan_bytes, vals.p, incl.p, static_cast<int>(n), s));
    if ((rc = keys_in.ensure(n, "group sort keys")) || (rc = keys_out.ensure(n, "sorted group keys")) ||
        (rc = vals.ensure(n, "group sort rows")) || (rc = incl.ensure(n, "group numbering")) ||
        (rc = temp.ensure(std::max<size_t>(std::max(sort_bytes, scan_bytes), 1), "group index scratch")) ||
        (rc = gi.perm.ensure(n, "group index rows")) || (rc = gi.row_group.ensure(n, "group index groups")) ||
        (rc = gi.starts.ensure(static_cast<size_t>(n) + 1, "group index starts")))
        return rc;
    if (e->groups_set) {
        if ((rc = d_groups.ensure(n, "group ids"))) return rc;
        CUDA_TRY(cudaMemcpyAsync(d_groups, e->groups.data(), static_cast<size_t>(n) * sizeof(uint64_t), cudaMemcpyHostToDevice, s));
    }
    const int grid = static_cast<int>(std::max<uint64_t>(1, std::min<uint64_t>(static_cast<uint64_t>(e->sm_count) * 8, (n + 255) / 256)));
    group_sort_input_kernel<<<grid, 256, 0, s>>>(keys_in, vals, n, e->groups_set ? d_groups.p : nullptr, d_ids, e->id_base);
    CUDA_TRY(cudaGetLastError());
    CUDA_TRY(cub::DeviceRadixSort::SortPairs(temp.p, sort_bytes, keys_in.p, keys_out.p, vals.p, gi.perm.p, static_cast<int>(n),
                                             0, 64, s));
    group_heads_kernel<<<grid, 256, 0, s>>>(keys_out, n, vals);        // the row values are no longer needed
    CUDA_TRY(cudaGetLastError());
    CUDA_TRY(cub::DeviceScan::InclusiveSum(temp.p, scan_bytes, vals.p, incl.p, static_cast<int>(n), s));
    group_finish_kernel<<<grid, 256, 0, s>>>(gi.perm, incl, n, gi.row_group, gi.starts);
    CUDA_TRY(cudaGetLastError());
    uint32_t n_groups = 0;
    CUDA_TRY(cudaMemcpyAsync(&n_groups, incl.p + (n - 1), sizeof(uint32_t), cudaMemcpyDeviceToHost, s));
    CUDA_TRY(cudaStreamSynchronize(s));
    CUDA_TRY(cudaMemcpy(gi.starts.p + n_groups, &n, sizeof(uint32_t), cudaMemcpyHostToDevice));
    if ((rc = gi.ids.ensure(n_groups, "group index ids"))) return rc;
    group_ids_kernel<<<grid, 256, 0, s>>>(keys_out, gi.starts, n_groups, gi.ids);
    CUDA_TRY(cudaGetLastError());
    CUDA_TRY(cudaStreamSynchronize(s));              // keys_out is released on return
    gi.n_groups = n_groups;
    gi.valid = true;
    std::lock_guard<std::mutex> pg(e->pool_mu);
    ++e->group_index_builds;
    return WAX_VS_OK;
}

// The root column of the current corpus, grouping and root tags (waxvs_roots.cuh), built on c's stream by the first
// search with a root clause after a mutation, set_groups or set_root_tags: the group index brought up, the sorted table
// uploaded, one root_column_kernel launch.  Readers hold the read lock; root_mu serialises the build, which completes
// before the column is published.
static int32_t ensure_root_column(wax_vs_engine *e, SearchCtx *c) {
    int32_t rc;
    if ((rc = ensure_group_index(e, c))) return rc;
    std::lock_guard<std::mutex> lk(e->root_mu);
    auto &rt = e->roots;
    if (rt.col_valid) return WAX_VS_OK;
    const auto &gi = e->gindex;
    const uint32_t n_roots = static_cast<uint32_t>(rt.ids.size());
    cudaStream_t s = c->stream;
    DevBuf<uint64_t> d_ids, d_tags;
    if ((rc = rt.col.ensure(std::max<uint64_t>(e->n_rows, 1), "root column")) ||
        (rc = d_ids.ensure(std::max<uint32_t>(n_roots, 1), "root tag ids")) ||
        (rc = d_tags.ensure(std::max<uint32_t>(n_roots, 1), "root tags")))
        return rc;
    if (n_roots) {
        CUDA_TRY(cudaMemcpyAsync(d_ids, rt.ids.data(), n_roots * sizeof(uint64_t), cudaMemcpyHostToDevice, s));
        CUDA_TRY(cudaMemcpyAsync(d_tags, rt.tags.data(), n_roots * sizeof(uint64_t), cudaMemcpyHostToDevice, s));
    }
    const uint64_t warps = (static_cast<uint64_t>(gi.n_groups) + 31) / 32;
    const int grid = static_cast<int>(std::max<uint64_t>(1, std::min<uint64_t>(static_cast<uint64_t>(e->sm_count) * 8, (warps + 7) / 8)));
    root_column_kernel<<<grid, 256, 0, s>>>(gi.ids, gi.starts, gi.perm, gi.n_groups, d_ids, d_tags, n_roots, rt.col);
    CUDA_TRY(cudaGetLastError());
    CUDA_TRY(cudaStreamSynchronize(s));              // the table is released on return
    rt.col_valid = true;
    std::lock_guard<std::mutex> pg(e->pool_mu);
    ++e->root_column_builds;
    return WAX_VS_OK;
}

static uint32_t host_orderable(float f) {            // orderable_u32 on the host
    uint32_t u;
    memcpy(&u, &f, sizeof u);
    return u ^ ((u & 0x80000000u) ? 0xFFFFFFFFu : 0x80000000u);
}
static float host_from_orderable(uint32_t k) {       // inverse of orderable_u32
    const uint32_t u = k ^ ((k & 0x80000000u) ? 0x80000000u : 0xFFFFFFFFu);
    float f;
    memcpy(&f, &u, sizeof f);
    return f;
}

// Expansion plan: span i = (first CSR position, rows, result offset) gets its per_group best rows at its result offset.
// Level 0 sorts tiles of kExpandTile CSR positions, each later level merges kExpandTile / per_group of the previous
// level's lists, until one list per span is left (a span of one tile is final at level 0).  Level l > 0 reads the level
// buffer (l - 1) & 1 and writes l & 1; buf_keys = the keys each buffer must hold.
struct ExpandPlan {
    std::vector<std::vector<ExpandItem>> levels;   // level 0: begin = CSR position
    std::vector<uint32_t> tile_span;               // level-0 item -> its span
    uint64_t buf_keys[2] = {0, 0};
};
static void plan_expansion(const std::vector<uint3> &spans, uint32_t per_group, ExpandPlan &plan) {
    struct Pending { uint32_t dst, lists, off; };
    plan.levels.assign(1, {});
    plan.tile_span.clear();
    plan.buf_keys[0] = plan.buf_keys[1] = 0;
    std::vector<Pending> pending;
    uint32_t off = 0;
    for (uint32_t i = 0; i < static_cast<uint32_t>(spans.size()); ++i) {
        const uint3 sp_i = spans[i];
        const uint32_t tiles = (sp_i.y + kExpandTile - 1) / kExpandTile;
        if (tiles == 1) {
            plan.levels[0].push_back({sp_i.x, sp_i.y, sp_i.z, 1u});
            plan.tile_span.push_back(i);
            continue;
        }
        for (uint32_t t = 0; t < tiles; ++t) {
            plan.levels[0].push_back({sp_i.x + t * kExpandTile, std::min(kExpandTile, sp_i.y - t * kExpandTile), off + t * per_group, 0u});
            plan.tile_span.push_back(i);
        }
        pending.push_back({sp_i.z, tiles, off});
        off += tiles * per_group;
    }
    plan.buf_keys[0] = off;
    const uint32_t fan = kExpandTile / per_group;
    while (!pending.empty()) {
        const size_t lv = plan.levels.size();
        plan.levels.emplace_back();
        std::vector<Pending> next;
        off = 0;
        for (const Pending &pd : pending) {
            const uint32_t m = (pd.lists + fan - 1) / fan;
            if (m == 1) { plan.levels[lv].push_back({pd.off, pd.lists * per_group, pd.dst, 1u}); continue; }
            for (uint32_t t = 0; t < m; ++t)
                plan.levels[lv].push_back({pd.off + t * fan * per_group, std::min(fan, pd.lists - t * fan) * per_group,
                                           off + t * per_group, 0u});
            next.push_back({pd.dst, m, off});
            off += m * per_group;
        }
        plan.buf_keys[lv & 1] = std::max<uint64_t>(plan.buf_keys[lv & 1], off);
        pending.swap(next);
    }
}
// Levels >= 1 of `plan` on stream s, after the caller's level 0 (the caller sizes the level buffers c->d_expand[0..1]
// from plan.buf_keys first): d_items = their items, in level order; each span's last list goes to `result`.  No level
// >= 1 is empty: plan_expansion adds one only while spans are pending, and each pending span contributes an item.
static int32_t enqueue_expand_merges(wax_vs_engine *e, SearchCtx *c, const ExpandPlan &plan, const ExpandItem *d_items,
                                     uint32_t per_group, uint64_t *result, cudaStream_t s, uint64_t *launches) {
    for (size_t lv = 1; lv < plan.levels.size(); ++lv) {
        const uint32_t items = static_cast<uint32_t>(plan.levels[lv].size());
        group_expand_kernel<<<items, 1024, 0, s>>>(d_items, 0u, e->gindex.perm, nullptr, c->d_expand[(lv - 1) & 1], per_group,
                                                   c->d_expand[lv & 1], result);
        CUDA_TRY(cudaGetLastError());
        ++*launches;
        d_items += items;
    }
    return WAX_VS_OK;
}

// Grouped delivery: row -> frame id and group id, distance -> score, as entry m of the outputs.
static void deliver_group_row(const wax_vs_engine *e, uint32_t row, float d, uint32_t m, uint64_t *out_ids, float *out_scores,
                              uint64_t *out_groups) {
    const uint64_t id = frame_id_of(e, row);
    out_ids[m] = id;
    out_scores[m] = score_from_distance(e->similarity, d);
    out_groups[m] = e->groups_set ? e->groups[row] : id;
}
// n_slots groups of per_group keys (dist_key << 32 | row), group-major, each group's list ending at its first
// WAXVS_KEY_NONE -> entries; returns how many.
static uint32_t deliver_group_keys(const wax_vs_engine *e, const uint64_t *keys, uint32_t n_slots, uint32_t per_group,
                                   uint64_t *out_ids, float *out_scores, uint64_t *out_groups) {
    uint32_t m = 0;
    for (uint32_t i = 0; i < n_slots; ++i)
        for (uint32_t j = 0; j < per_group; ++j) {
            const uint64_t key = keys[static_cast<size_t>(i) * per_group + j];
            if (key == WAXVS_KEY_NONE) break;
            deliver_group_row(e, static_cast<uint32_t>(key), host_from_orderable(static_cast<uint32_t>(key >> 32)), m++, out_ids,
                              out_scores, out_groups);
        }
    return m;
}

// One grouped search under the caller's read lock and scratch context (re-taking the shared lock inside a batch could
// wait behind a queued writer): the host query, the filter's resolved rows (nullptr: unfiltered; the filter allows some
// row) with `where` ANDed into its bitset (nullptr: none) and the rows of a planned group unit set in it (nullptr: none;
// then `rows` is empty, in mode 0), the answer at out_* and *out_n -- or, with out_keys, as n_top x per_group keys
// (dist_key << 32 | row, group-major, padded with WAXVS_KEY_NONE) there instead.  The arguments are checked by the caller.
static int32_t grouped_one(wax_vs_engine *e, SearchCtx *c, const float *query, uint32_t n_top, uint32_t per_group,
                           const std::vector<uint32_t> *rows, int32_t mode, const Clause *where, uint64_t *out_ids,
                           float *out_scores, uint64_t *out_groups, uint32_t *out_n, uint64_t *out_keys = nullptr,
                           const GroupUnitR *unit = nullptr) {
    const uint32_t n = static_cast<uint32_t>(e->n_rows);
    const bool filtered = rows != nullptr;
    cudaStream_t s = c->stream;
    int32_t rc;
    if ((rc = ensure_group_index(e, c))) return rc;
    const auto &gi = e->gindex;
    uint64_t launches = 0;

    // (1) the emitting scan under the row filter: c->d_dist_keys
    if ((rc = stage_queries(e, c, query, 1, s))) return rc;
    if ((rc = c->d_out.ensure(n_top, "result buffer"))) return rc;
    if ((rc = c->h_out.ensure(n_top, "result staging"))) return rc;
    if (filtered) {
        std::vector<GroupUnitR> unit_bits;
        if (unit) {
            unit_bits.push_back(*unit);
            unit_bits.back().slot = 0;
        }
        if ((rc = stage_filter_rows(e, c, *rows, rows->size(), mode, s, &launches)) ||
            (where && (rc = apply_where_bits(e, c, {where_item(*where)}, s, &launches))) ||
            (rc = launch_group_filter(e, c, unit_bits, nullptr, c->d_mask, s, &launches))) {
            cudaStreamSynchronize(s);
            return rc;
        }
    }
    if ((rc = enqueue_search(e, c, c->d_queries, 1, 0, c->d_out, nullptr, s, &launches, filtered ? c->d_mask.p : nullptr,
                             nullptr, nullptr, true))) {
        cudaStreamSynchronize(s);
        return rc;
    }
    // (2) each group's best row, written at that row of an otherwise empty key array
    if ((rc = c->d_group_best.ensure(std::max<uint32_t>(gi.n_groups, 1), "group minima"))) return rc;
    if ((rc = c->d_group_keys.ensure(n, "group keys"))) return rc;
    CUDA_TRY(cudaMemsetAsync(c->d_group_best, 0xFF, static_cast<size_t>(gi.n_groups) * sizeof(unsigned long long), s));
    const uint64_t reduce_warps = (static_cast<uint64_t>(n) + 32 * kReduceRun - 1) / (32 * kReduceRun);
    const int rgrid = static_cast<int>(std::max<uint64_t>(1, std::min<uint64_t>(static_cast<uint64_t>(e->sm_count) * 16, (reduce_warps + 7) / 8)));
    group_reduce_kernel<<<rgrid, 256, 0, s>>>(gi.perm, gi.row_group, c->d_dist_keys, n, c->d_group_best);
    const int kgrid = static_cast<int>(std::max<uint64_t>(1, std::min<uint64_t>(static_cast<uint64_t>(e->sm_count) * 8, (n + 255) / 256)));
    group_keys_kernel<<<kgrid, 256, 0, s>>>(gi.row_group, c->d_group_best, n, c->d_group_keys);
    CUDA_TRY(cudaGetLastError());
    launches += 2;
    // (3) the top groups' best rows, in the total order
    ScanParams sp{};
    sp.k = n_top; sp.out = c->d_out;
    if ((rc = enqueue_select(e, c, c->d_group_keys, n, n_top, sp, s, &launches))) { cudaStreamSynchronize(s); return rc; }
    CUDA_TRY(cudaMemcpyAsync(c->h_out, c->d_out, n_top * sizeof(wax_vs_candidate), cudaMemcpyDeviceToHost, s));
    uint32_t n_sel = 0;
    if (per_group > 1) {
        // (4) expansion: each selected group's per_group best rows (plan_expansion)
        if ((rc = c->d_group_spans.ensure(n_top, "group spans")) || (rc = c->h_group_spans.ensure(n_top, "group span staging")))
            return rc;
        group_spans_kernel<<<(n_top + 255) / 256, 256, 0, s>>>(c->d_out, n_top, gi.row_group, gi.starts, c->d_group_spans);
        CUDA_TRY(cudaGetLastError());
        ++launches;
        CUDA_TRY(cudaMemcpyAsync(c->h_group_spans, c->d_group_spans, n_top * sizeof(uint2), cudaMemcpyDeviceToHost, s));
        CUDA_TRY(cudaStreamSynchronize(s));
        while (n_sel < n_top && c->h_group_spans[n_sel].y > 0) ++n_sel;   // valid candidates come first
        std::vector<uint3> spans(n_sel);
        for (uint32_t i = 0; i < n_sel; ++i) spans[i] = make_uint3(c->h_group_spans[i].x, c->h_group_spans[i].y, i * per_group);
        ExpandPlan plan;
        plan_expansion(spans, per_group, plan);
        std::vector<ExpandItem> all;
        for (const auto &lvl : plan.levels) all.insert(all.end(), lvl.begin(), lvl.end());
        const size_t n_res = static_cast<size_t>(std::max<uint32_t>(n_sel, 1)) * per_group;
        if ((rc = c->d_expand_items.ensure(std::max<size_t>(all.size(), 1), "expansion items")) ||
            (rc = c->d_expand[0].ensure(std::max<uint64_t>(plan.buf_keys[0], 1), "expansion lists")) ||
            (rc = c->d_expand[1].ensure(std::max<uint64_t>(plan.buf_keys[1], 1), "expansion lists")) ||
            (rc = c->d_expand[2].ensure(n_res, "expansion result")) || (rc = c->h_expand.ensure(n_res, "expansion staging")))
            return rc;
        if (!all.empty())
            CUDA_TRY(cudaMemcpyAsync(c->d_expand_items, all.data(), all.size() * sizeof(ExpandItem), cudaMemcpyHostToDevice, s));
        const uint32_t tiles = static_cast<uint32_t>(plan.levels[0].size());
        if (tiles) {
            group_expand_kernel<<<tiles, 1024, 0, s>>>(c->d_expand_items, 1u, gi.perm, c->d_dist_keys, nullptr, per_group,
                                                       c->d_expand[0], c->d_expand[2]);
            CUDA_TRY(cudaGetLastError());
            ++launches;
        }
        if ((rc = enqueue_expand_merges(e, c, plan, c->d_expand_items + tiles, per_group, c->d_expand[2], s, &launches)))
            return rc;
        if (n_sel)
            CUDA_TRY(cudaMemcpyAsync(c->h_expand, c->d_expand[2], static_cast<size_t>(n_sel) * per_group * sizeof(uint64_t),
                                     cudaMemcpyDeviceToHost, s));
        CUDA_TRY(cudaStreamSynchronize(s));          // also keeps the item list alive until its copy is done
        if (out_keys) {
            std::fill(out_keys, out_keys + static_cast<size_t>(n_top) * per_group, WAXVS_KEY_NONE);
            std::copy(c->h_expand.p, c->h_expand.p + static_cast<size_t>(n_sel) * per_group, out_keys);
            return WAX_VS_OK;
        }
        *out_n = deliver_group_keys(e, c->h_expand, n_sel, per_group, out_ids, out_scores, out_groups);
        return WAX_VS_OK;
    }
    CUDA_TRY(cudaStreamSynchronize(s));              // also keeps `rows` alive until its copy is done
    if (out_keys) {
        for (uint32_t i = 0; i < n_top; ++i)
            out_keys[i] = c->h_out[i].valid ? (static_cast<uint64_t>(host_orderable(c->h_out[i].distance)) << 32) | c->h_out[i].row
                                            : WAXVS_KEY_NONE;
        return WAX_VS_OK;
    }
    // (5) delivery: row -> frame id and group id, distance -> score
    uint32_t m = 0;
    for (uint32_t i = 0; i < n_top; ++i)
        if (c->h_out[i].valid)
            deliver_group_row(e, static_cast<uint32_t>(c->h_out[i].row), c->h_out[i].distance, m++, out_ids, out_scores, out_groups);
    *out_n = m;
    return WAX_VS_OK;
}

// ---- batched grouped search (waxvs_group_batch.cuh) -----------------------------------------------------------------
constexpr uint64_t kExpandBatchKeys = 1ull << 24;   // level-buffer keys one round of batched expansions may hold

// The expansions the cover kernel listed, in a reproducible order, into the batch's result keys c->d_bg_keys: level 0
// scores the CSR tiles for the item's query (group_score_tile_kernel) under bitset query_slot[query] of c->d_mask
// (WAX_VS_NO_FILTER: unfiltered), the later levels merge as the single query does.  Rounds of spans keep the level
// buffers within kExpandBatchKeys; the buffers are sized once for the largest round.
static int32_t enqueue_batch_expansion(wax_vs_engine *e, SearchCtx *c, const CoverExpand *list, uint32_t n_list,
                                       uint32_t n_top, uint32_t per_group, const std::vector<uint32_t> &query_slot,
                                       uint64_t *launches) {
    struct Round { ExpandPlan plan; std::vector<uint32_t> span_query; };
    std::vector<Round> rounds;
    std::vector<uint3> spans;
    std::vector<uint32_t> span_query;
    uint64_t round_keys = 0;
    auto close_round = [&]() {
        rounds.emplace_back();
        plan_expansion(spans, per_group, rounds.back().plan);
        rounds.back().span_query.swap(span_query);
        spans.clear();
        round_keys = 0;
    };
    for (uint32_t i = 0; i < n_list; ++i) {
        const CoverExpand &x = list[i];
        const uint64_t keys = static_cast<uint64_t>((x.count + kExpandTile - 1) / kExpandTile) * per_group;
        if (!spans.empty() && round_keys + keys > kExpandBatchKeys) close_round();
        spans.push_back(make_uint3(x.begin, x.count, (x.query * n_top + x.slot) * per_group));
        span_query.push_back(x.query);
        round_keys += keys;
    }
    if (!spans.empty()) close_round();
    std::vector<ScoreItem> tiles;
    std::vector<ExpandItem> merges;
    uint64_t buf[2] = {1, 1};
    for (const Round &rd : rounds) {
        for (size_t t = 0; t < rd.plan.levels[0].size(); ++t) {
            const ExpandItem &it = rd.plan.levels[0][t];
            const uint32_t q = rd.span_query[rd.plan.tile_span[t]];
            tiles.push_back({q, it.begin, it.count, it.dst_off, it.final_out, query_slot[q]});
        }
        for (size_t lv = 1; lv < rd.plan.levels.size(); ++lv)
            merges.insert(merges.end(), rd.plan.levels[lv].begin(), rd.plan.levels[lv].end());
        buf[0] = std::max(buf[0], rd.plan.buf_keys[0]);
        buf[1] = std::max(buf[1], rd.plan.buf_keys[1]);
    }
    cudaStream_t s = c->stream;
    int32_t rc;
    if ((rc = c->d_score_items.ensure(std::max<size_t>(tiles.size(), 1), "expansion tiles")) ||
        (rc = c->d_expand_items.ensure(std::max<size_t>(merges.size(), 1), "expansion items")) ||
        (rc = c->d_expand[0].ensure(buf[0], "expansion lists")) || (rc = c->d_expand[1].ensure(buf[1], "expansion lists")))
        return rc;
    CUDA_TRY(cudaMemcpyAsync(c->d_score_items, tiles.data(), tiles.size() * sizeof(ScoreItem), cudaMemcpyHostToDevice, s));
    if (!merges.empty())
        CUDA_TRY(cudaMemcpyAsync(c->d_expand_items, merges.data(), merges.size() * sizeof(ExpandItem), cudaMemcpyHostToDevice, s));
    const auto score = e->similarity == WAX_VS_COSINE ? group_score_tile_kernel<kCosine>
                       : e->similarity == WAX_VS_DOT  ? group_score_tile_kernel<kDot>
                                                      : group_score_tile_kernel<kL2>;
    const uint32_t words = static_cast<uint32_t>((e->n_rows + 31) / 32);
    size_t first_tile = 0, first_merge = 0;
    for (const Round &rd : rounds) {
        const uint32_t n0 = static_cast<uint32_t>(rd.plan.levels[0].size());
        score<<<n0, 256, 0, s>>>(c->d_score_items + first_tile, e->d_corpus, c->d_queries, e->dims, e->gindex.perm,
                                  c->d_mask.p, words, per_group, c->d_expand[0], c->d_bg_keys);
        CUDA_TRY(cudaGetLastError());
        ++*launches;
        first_tile += n0;
        if ((rc = enqueue_expand_merges(e, c, rd.plan, c->d_expand_items + first_merge, per_group, c->d_bg_keys, s, launches)))
            return rc;
        for (size_t lv = 1; lv < rd.plan.levels.size(); ++lv) first_merge += rd.plan.levels[lv].size();
    }
    CUDA_TRY(cudaStreamSynchronize(s));              // also keeps the item lists alive until their copies are done
    return WAX_VS_OK;
}

// The expansions `list` (query = an index of `unit`, which names the query's pair or WAX_VS_NO_FILTER, unfiltered) into
// c->d_bg_keys [query][n_top][per_group], queries staged in c->d_queries in the same indexing and the pairs' rows in
// c->d_filter_rows.  The list, appended in any order, is sorted by (unit, query, group rank) for a reproducible launch
// plan and run in passes of at most `fit` distinct units' bitsets (build_pass_bits); each pass ends in a synchronise, so
// the next one may rebuild the bitsets.
static int32_t expand_in_passes(wax_vs_engine *e, SearchCtx *c, CoverExpand *list, uint32_t n_exp,
                                const std::vector<uint32_t> &unit, const WherePlan &wp, uint32_t n_top,
                                uint32_t per_group, uint64_t *launches, uint64_t *passes) {
    std::sort(list, list + n_exp, [&](const CoverExpand &a, const CoverExpand &b) {
        if (unit[a.query] != unit[b.query]) return unit[a.query] < unit[b.query];
        return a.query != b.query ? a.query < b.query : a.slot < b.slot;
    });
    const uint64_t words = (e->n_rows + 31) / 32;
    const uint64_t fit = std::max<uint64_t>(1, e->tune.filter_bitset_bytes / (words * sizeof(uint32_t)));
    std::vector<uint32_t> query_slot(unit.size(), WAX_VS_NO_FILTER);
    int32_t rc;
    for (uint32_t i0 = 0; i0 < n_exp;) {
        std::vector<uint32_t> which;         // the pass's units, in bitset order
        uint32_t i1 = i0;
        for (; i1 < n_exp; ++i1) {
            const uint32_t u = unit[list[i1].query];
            if (u != WAX_VS_NO_FILTER && (which.empty() || which.back() != u)) {
                if (which.size() == fit) break;
                which.push_back(u);
            }
            query_slot[list[i1].query] = u == WAX_VS_NO_FILTER ? WAX_VS_NO_FILTER : static_cast<uint32_t>(which.size() - 1);
        }
        if (!which.empty()) {
            if ((rc = build_pass_bits(e, c, wp, which, launches))) return rc;
            ++*passes;
        }
        if ((rc = enqueue_batch_expansion(e, c, list + i0, i1 - i0, n_top, per_group, query_slot, launches))) {
            cudaStreamSynchronize(c->stream);
            return rc;
        }
        i0 = i1;
    }
    return WAX_VS_OK;
}

// The request's grouped arguments: per_group in [1, WAX_VS_MAX_PER_GROUP], at most WAX_VS_MAX_RESULTS rows per query.
static int32_t check_grouped_args(const SearchRequest &r) {
    if (r.per_group == 0 || r.per_group > WAX_VS_MAX_PER_GROUP)
        return fail(WAX_VS_ERR_ARGUMENT, "per_group must be in [1, %d] (got %u)", WAX_VS_MAX_PER_GROUP, r.per_group);
    const uint32_t n_top = clamp_topk(r.top_k);
    if (static_cast<uint64_t>(n_top) * r.per_group > WAX_VS_MAX_RESULTS)
        return fail(WAX_VS_ERR_ARGUMENT, "clamp(top_groups) x per_group = %llu exceeds %d",
                    static_cast<unsigned long long>(n_top) * r.per_group, WAX_VS_MAX_RESULTS);
    return WAX_VS_OK;
}

// Every grouped entry point on one engine after its argument checks, `queries` being the request's on the host: query i
// searches the rows passing wheres[query_where[i]] AND id filter query_filter[i], either of which may be WAX_VS_NO_FILTER.
// The (where, id filter) pairs are the units of the where search (plan_where_pairs), planned by the batched filtered
// search at k_c; a query no row passes answers nothing.  Without `batched`, or when the coverage level does not take the
// batch, every query runs grouped_one.  The batch pipeline:
//  - coverage: each staged query's exact top-k_c rows (run_filtered), then group_cover_kernel, when every staged query
//    is in the gather class, or every one in the tensor class and the batch goes to the tensor-core levels;
//  - expansion: the cover kernel's list sorted by (unit, query, group rank), in passes of at most filter_bitset_bytes
//    of distinct units' bitsets (build_pass_bits, as run_filtered builds them), each item scored under its unit's;
//  - crowded queries: grouped_one under the query's own pair (grouped_one_args).
// With `heads` (the sharded round 1) the answers go to the device instead, as [query][n_top][per_group] records with
// global rows: the covered queries' keys are converted there, the crowded queries' are uploaded into their slots; the
// caller zeroed the records, and the host outputs are not used.
struct ShardHeads {
    uint64_t row_offset;
    wax_vs_group_candidate *d_heads;
};
static int32_t search_grouped_host(wax_vs_engine *e, const SearchRequest &req, const float *queries, uint64_t *out_ids,
                                   float *out_scores, uint64_t *out_groups, uint32_t out_stride, uint32_t *out_n,
                                   const ShardHeads *heads = nullptr) {
    const uint32_t n_queries = req.n_queries, per_group = req.per_group;
    const uint32_t n_top = clamp_topk(req.top_k);
    std::shared_lock<std::shared_mutex> r(e->rw);
    for (uint32_t i = 0; i < n_queries; ++i) out_n[i] = 0;
    if (e->n_rows == 0 || n_queries == 0) return WAX_VS_OK;      // as wax_vs_search (:448)
    int32_t rc;
    if ((rc = check_query(e, queries, req.query_len))) return rc;
    const uint32_t n = static_cast<uint32_t>(e->n_rows);
    const uint32_t need = static_cast<uint32_t>(std::min<uint64_t>(static_cast<uint64_t>(n_top) * per_group, n));
    if (!heads && out_stride < need) return fail(WAX_VS_ERR_BUFFER, "output buffers hold %u entries, need %u", out_stride, need);
    DeviceGuard g(e->device);
    if (!g.ok) return g.error();
    CtxLease lease(e);
    if ((rc = lease.acquire())) return rc;
    SearchCtx *c = lease.c;
    // The coverage level: each query's exact top-k_c rows, when the batch goes to the tensor-core levels or the gather
    // class of the batched filtered search; every other batch runs the single-query pipeline per query.
    const uint32_t k_c = std::min(kCoverMax, std::max(128u, 4u * n_top));
    WherePlan wp;
    if ((rc = plan_request(e, c, req, k_c, wp))) return rc;
    const FilteredPlan &plan = wp.plan;
    const uint32_t nq = static_cast<uint32_t>(plan.order.size());    // the staged queries: some row passes
    const bool cover = req.batched && nq > 0 && n_top <= kCoverMax / 4 &&
                       (plan.n_gather == nq || (plan.n_tensor == nq && batch_tensor_eligible(e, nq, plan.k_max)));
    cudaStream_t s = c->stream;
    std::vector<uint32_t> crowded;                   // queries for the single-query pipeline
    uint64_t covered = 0, expanded = 0, expansion_passes = 0, launches = 0;
    if (!cover) {
        crowded = plan.order;
    } else {
        if ((rc = ensure_group_index(e, c))) return rc;
        if ((rc = run_filtered(e, c, queries, wp))) return rc;
        const uint32_t slots = n_top * per_group;
        const size_t nkeys = static_cast<size_t>(nq) * slots;
        if ((rc = c->d_bg_keys.ensure(nkeys, "grouped batch keys")) || (rc = c->h_bg_keys.ensure(nkeys, "grouped batch staging")) ||
            (rc = c->d_bg_status.ensure(nq + 1u, "grouped batch status")) ||
            (rc = c->h_bg_status.ensure(nq + 1u, "grouped batch status staging")) ||
            (rc = c->d_bg_expand.ensure(static_cast<size_t>(nq) * n_top, "grouped batch expansions")) ||
            (rc = c->h_bg_expand.ensure(static_cast<size_t>(nq) * n_top, "grouped batch expansion staging")))
            return rc;
        CUDA_TRY(cudaMemsetAsync(c->d_bg_status + nq, 0, sizeof(uint32_t), s));
        group_cover_kernel<<<nq, kCoverMax, 0, s>>>(c->d_out, plan.k_max, k_c, e->gindex.row_group, e->gindex.starts, n_top,
                                                    per_group, c->d_bg_keys, c->d_bg_status, c->d_bg_expand, c->d_bg_status + nq);
        CUDA_TRY(cudaGetLastError());
        ++launches;
        CUDA_TRY(cudaMemcpyAsync(c->h_bg_status, c->d_bg_status, (nq + 1u) * sizeof(uint32_t), cudaMemcpyDeviceToHost, s));
        CUDA_TRY(cudaStreamSynchronize(s));
        const uint32_t n_exp = c->h_bg_status[nq];
        if (n_exp) {
            CUDA_TRY(cudaMemcpyAsync(c->h_bg_expand, c->d_bg_expand, n_exp * sizeof(CoverExpand), cudaMemcpyDeviceToHost, s));
            CUDA_TRY(cudaStreamSynchronize(s));
            std::vector<uint32_t> unit(nq);          // staged query -> its pair (WAX_VS_NO_FILTER, unfiltered, sorts last)
            for (uint32_t j = 0; j < nq; ++j) unit[j] = wp.pair_of[plan.order[j]];
            if ((rc = expand_in_passes(e, c, c->h_bg_expand, n_exp, unit, wp, n_top, per_group, &launches, &expansion_passes)))
                return rc;
            expanded = n_exp;
        }
        if (heads) {
            ShardRowInfo ri{heads->row_offset, e->id_base, nullptr, device_row_keys(e), e->gindex.row_group, e->gindex.ids};
            if ((rc = sync_device_ids(e, &ri.ids)) || (rc = c->d_order.ensure(nq, "query order"))) return rc;
            CUDA_TRY(cudaMemcpyAsync(c->d_order, plan.order.data(), nq * sizeof(uint32_t), cudaMemcpyHostToDevice, s));
            const int grid = static_cast<int>(std::max<size_t>(1, std::min<size_t>(static_cast<size_t>(e->sm_count) * 8, (nkeys + 255) / 256)));
            shard_group_heads_kernel<<<grid, 256, 0, s>>>(c->d_bg_keys, nq, slots, c->d_order, c->d_bg_status, ri, heads->d_heads);
            CUDA_TRY(cudaGetLastError());
            ++launches;
        } else {
            CUDA_TRY(cudaMemcpyAsync(c->h_bg_keys, c->d_bg_keys, nkeys * sizeof(uint64_t), cudaMemcpyDeviceToHost, s));
        }
        CUDA_TRY(cudaStreamSynchronize(s));
        for (uint32_t j = 0; j < nq; ++j) {
            const uint32_t qi = plan.order[j];
            if (!c->h_bg_status[j]) { crowded.push_back(qi); continue; }
            if (heads) { ++covered; continue; }
            const size_t o = static_cast<size_t>(qi) * out_stride;
            out_n[qi] = deliver_group_keys(e, c->h_bg_keys + static_cast<size_t>(j) * slots, n_top, per_group, out_ids + o,
                                           out_scores + o, out_groups + o);
            ++covered;
        }
    }
    std::sort(crowded.begin(), crowded.end());
    // crowded queries (and batches the coverage level does not take): the single-query pipeline, same lock and context,
    // under the query's own pair as the one-filter grouped search takes it -- an id filter alone as it is, an allow-list
    // as its rows that pass the where (plan_where_pairs listed them), a group unit as its rows set in an empty bitset by
    // the device, a deny-list (or none) AND any other where as the deny-list in mode 1 with the predicate and its box
    // ANDed into the bitset
    const FilterSet &ids = wp.ids, &fs = wp.fs;
    for (uint32_t qi : crowded) {
        const uint32_t p = wp.pair_of[qi], f = req.query_filter[qi];
        const GroupUnitR *unit = p != WAX_VS_NO_FILTER && !fs.group_of.empty() && fs.group_of[p] != WAX_VS_NO_FILTER
                                    ? &fs.group_units[fs.group_of[p]] : nullptr;
        const uint32_t w = unit ? WAX_VS_NO_FILTER : req.query_where[qi];
        const bool row_where = w != WAX_VS_NO_FILTER && (f == WAX_VS_NO_FILTER || req.filter_modes[f] == 1);
        std::vector<uint32_t> rows;
        int32_t mode = unit ? 0 : 1;
        if (row_where) {
            if (f != WAX_VS_NO_FILTER) rows.assign(ids.rows.begin() + ids.first[f], ids.rows.begin() + ids.first[f] + ids.count[f]);
        } else if (p != WAX_VS_NO_FILTER && !unit) {
            rows.assign(fs.rows.begin() + fs.first[p], fs.rows.begin() + fs.first[p] + fs.count[p]);
            mode = wp.modes[p];
        }
        if (heads) {                                 // the answer's keys -> records, uploaded into the query's slots
            const size_t slots = static_cast<size_t>(n_top) * per_group;
            std::vector<uint64_t> keys(slots);
            if ((rc = grouped_one(e, c, queries + static_cast<size_t>(qi) * e->dims, n_top, per_group,
                                  p == WAX_VS_NO_FILTER ? nullptr : &rows, mode, row_where ? &req.wheres[w] : nullptr, nullptr,
                                  nullptr, nullptr, nullptr, keys.data(), unit)))
                return rc;
            std::vector<wax_vs_group_candidate> recs(slots, wax_vs_group_candidate{});
            for (size_t i = 0; i < slots; ++i) {
                if (keys[i] == WAXVS_KEY_NONE) continue;
                const uint32_t row = static_cast<uint32_t>(keys[i]);
                const uint64_t id = frame_id_of(e, row);
                recs[i] = wax_vs_group_candidate{host_from_orderable(static_cast<uint32_t>(keys[i] >> 32)), 1u,
                                                 heads->row_offset + (e->keys_set ? e->keys[row] : row), id,
                                                 e->groups_set ? e->groups[row] : id};
            }
            CUDA_TRY(cudaMemcpyAsync(heads->d_heads + qi * slots, recs.data(), slots * sizeof(wax_vs_group_candidate),
                                     cudaMemcpyHostToDevice, s));
            CUDA_TRY(cudaStreamSynchronize(s));      // recs must outlive its copy
            continue;
        }
        const size_t o = static_cast<size_t>(qi) * out_stride;
        if ((rc = grouped_one(e, c, queries + static_cast<size_t>(qi) * e->dims, n_top, per_group,
                              p == WAX_VS_NO_FILTER ? nullptr : &rows, mode, row_where ? &req.wheres[w] : nullptr, out_ids + o,
                              out_scores + o, out_groups + o, out_n + qi, nullptr, unit)))
            return rc;
    }
    if (!req.batched) return WAX_VS_OK;
    std::lock_guard<std::mutex> pg(e->pool_mu);
    e->grouped_batch_covered_queries += covered;
    e->grouped_batch_expanded_groups += expanded;
    e->grouped_batch_fallback_queries += crowded.size();
    e->grouped_batch_expansion_passes += expansion_passes;
    return WAX_VS_OK;
}

// The grouped entry points after their argument checks: on one engine, or across the shards of a multi-device handle,
// which first zeroes out_n as one engine does.
static int32_t search_grouped(wax_vs_engine *e, const SearchRequest &req, uint64_t *out_ids, float *out_scores,
                              uint64_t *out_groups, uint32_t out_stride, uint32_t *out_n) {
    if (!e->multi) return search_grouped_host(e, req, req.queries, out_ids, out_scores, out_groups, out_stride, out_n);
    for (uint32_t i = 0; i < req.n_queries; ++i) out_n[i] = 0;
    return multi_search_grouped(e->multi, e->dims, e->similarity, req, out_ids, out_scores, out_groups, out_stride, out_n);
}

// The one-filter grouped entry points, after their where (if any) went into req: the outputs, the grouped arguments,
// one id filter (an empty deny-list is none) and at most one where for every query.
static int32_t search_grouped_one_filter(wax_vs_engine *e, SearchRequest &req, const uint64_t *frame_ids, uint64_t n_ids,
                                         int32_t mode, uint64_t *out_ids, float *out_scores, uint64_t *out_groups,
                                         uint32_t out_stride, uint32_t *out_n) {
    if (!e || !out_n || !out_ids || !out_scores || !out_groups) return fail(WAX_VS_ERR_NULL, "NULL argument");
    int32_t rc;
    if ((rc = check_grouped_args(req)) || (rc = request_one_filter(req, frame_ids, n_ids, mode, true))) return rc;
    request_one_where(req);
    return search_grouped(e, req, out_ids, out_scores, out_groups, out_stride, out_n);
}

int32_t wax_vs_search_grouped(wax_vs_engine *e, const float *query, uint32_t query_len, int64_t top_groups,
                              uint32_t per_group, const uint64_t *frame_ids, uint64_t n_ids, int32_t mode,
                              uint64_t *out_ids, float *out_scores, uint64_t *out_groups, uint32_t out_cap,
                              uint32_t *out_n) {
    SearchRequest req(query, 1, query_len, top_groups, per_group, false);
    return search_grouped_one_filter(e, req, frame_ids, n_ids, mode, out_ids, out_scores, out_groups, out_cap, out_n);
}

// A batch of one stays a batch.
int32_t wax_vs_search_batch_grouped(wax_vs_engine *e, const float *queries, uint32_t n_queries, uint32_t query_len,
                                    int64_t top_groups, uint32_t per_group, const uint64_t *frame_ids, uint64_t n_ids,
                                    int32_t mode, uint64_t *out_ids, float *out_scores, uint64_t *out_groups,
                                    uint32_t out_stride, uint32_t *out_n) {
    SearchRequest req(queries, n_queries, query_len, top_groups, per_group, true);
    return search_grouped_one_filter(e, req, frame_ids, n_ids, mode, out_ids, out_scores, out_groups, out_stride, out_n);
}

int32_t wax_vs_search_batch_grouped_where(wax_vs_engine *e, const float *queries, uint32_t n_queries, uint32_t query_len,
                                          int64_t top_groups, uint32_t per_group, const uint64_t *frame_ids, uint64_t n_ids,
                                          int32_t mode, const wax_vs_where *where, uint64_t *out_ids, float *out_scores,
                                          uint64_t *out_groups, uint32_t out_stride, uint32_t *out_n) {
    if (!where) return fail(WAX_VS_ERR_NULL, "where is NULL");
    SearchRequest req(queries, n_queries, query_len, top_groups, per_group, n_queries > 1);
    request_plain_clauses(req, where, 1);
    return search_grouped_one_filter(e, req, frame_ids, n_ids, mode, out_ids, out_scores, out_groups, out_stride, out_n);
}

int32_t wax_vs_search_batch_grouped_where_near(wax_vs_engine *e, const float *queries, uint32_t n_queries,
                                               uint32_t query_len, int64_t top_groups, uint32_t per_group,
                                               const uint64_t *frame_ids, uint64_t n_ids, int32_t mode,
                                               const wax_vs_where_near *where, uint64_t *out_ids, float *out_scores,
                                               uint64_t *out_groups, uint32_t out_stride, uint32_t *out_n) {
    if (!where) return fail(WAX_VS_ERR_NULL, "where is NULL");
    SearchRequest req(queries, n_queries, query_len, top_groups, per_group, n_queries > 1);
    const int32_t rc = near_clauses(where, 1, req.wheres);
    return rc ? rc
              : search_grouped_one_filter(e, req, frame_ids, n_ids, mode, out_ids, out_scores, out_groups, out_stride, out_n);
}

int32_t wax_vs_search_batch_grouped_multi_where(wax_vs_engine *e, const float *queries, uint32_t n_queries,
                                                uint32_t query_len, int64_t top_groups, uint32_t per_group,
                                                const uint64_t *frame_ids, const uint64_t *filter_offsets,
                                                const int32_t *filter_modes, uint32_t n_filters,
                                                const uint32_t *query_filter, const wax_vs_where_near *wheres,
                                                uint32_t n_wheres, const uint32_t *query_where, uint64_t *out_ids,
                                                float *out_scores, uint64_t *out_groups, uint32_t out_stride,
                                                uint32_t *out_n) {
    if (!e || !out_n || !out_ids || !out_scores || !out_groups) return fail(WAX_VS_ERR_NULL, "NULL argument");
    SearchRequest req(queries, n_queries, query_len, top_groups, per_group, n_queries > 1);
    int32_t rc;
    if ((rc = check_grouped_args(req)) ||
        (rc = request_filters(req, frame_ids, filter_offsets, filter_modes, n_filters, query_filter)) ||
        (rc = request_where_list(req, wheres, n_wheres, query_where)) || (rc = near_clauses(wheres, n_wheres, req.wheres)))
        return rc;
    return search_grouped(e, req, out_ids, out_scores, out_groups, out_stride, out_n);
}

int32_t wax_vs_search_batch_grouped_multi_where_groups(wax_vs_engine *e, const float *queries, uint32_t n_queries,
                                                       uint32_t query_len, int64_t top_groups, uint32_t per_group,
                                                       const uint64_t *frame_ids, const uint64_t *filter_offsets,
                                                       const int32_t *filter_modes, uint32_t n_filters,
                                                       const uint32_t *query_filter, const wax_vs_where_near *wheres,
                                                       uint32_t n_wheres, const uint32_t *query_where,
                                                       const uint64_t *where_group_offsets, const uint64_t *where_groups,
                                                       uint64_t *out_ids, float *out_scores, uint64_t *out_groups,
                                                       uint32_t out_stride, uint32_t *out_n) {
    if (!e || !out_n || !out_ids || !out_scores || !out_groups) return fail(WAX_VS_ERR_NULL, "NULL argument");
    SearchRequest req(queries, n_queries, query_len, top_groups, per_group, n_queries > 1);
    int32_t rc;
    bool any = false;
    if ((rc = check_grouped_args(req)) ||
        (rc = request_filters(req, frame_ids, filter_offsets, filter_modes, n_filters, query_filter)) ||
        (rc = request_where_list(req, wheres, n_wheres, query_where)) ||
        (rc = check_group_offsets(where_group_offsets, n_wheres, where_groups, &any)))
        return rc;
    if (!any)                          // no where has a group: the entry point without the clause
        return wax_vs_search_batch_grouped_multi_where(e, queries, n_queries, query_len, top_groups, per_group, frame_ids,
                                                       filter_offsets, filter_modes, n_filters, query_filter, wheres,
                                                       n_wheres, query_where, out_ids, out_scores, out_groups, out_stride,
                                                       out_n);
    if ((rc = near_clauses(wheres, n_wheres, req.wheres))) return rc;
    request_id_lists(req, n_wheres, where_group_offsets, where_groups, &Clause::groups);
    canonical_wheres(req);
    return search_grouped(e, req, out_ids, out_scores, out_groups, out_stride, out_n);
}

int32_t wax_vs_search_batch_grouped_multi_where_roots(wax_vs_engine *e, const float *queries, uint32_t n_queries,
                                                      uint32_t query_len, int64_t top_groups, uint32_t per_group,
                                                      const uint64_t *frame_ids, const uint64_t *filter_offsets,
                                                      const int32_t *filter_modes, uint32_t n_filters,
                                                      const uint32_t *query_filter, const wax_vs_where_near *wheres,
                                                      uint32_t n_wheres, const uint32_t *query_where,
                                                      const uint64_t *where_group_offsets, const uint64_t *where_groups,
                                                      const wax_vs_root_clause *where_roots, uint64_t *out_ids,
                                                      float *out_scores, uint64_t *out_groups, uint32_t out_stride,
                                                      uint32_t *out_n) {
    if (!e || !out_n || !out_ids || !out_scores || !out_groups) return fail(WAX_VS_ERR_NULL, "NULL argument");
    SearchRequest req(queries, n_queries, query_len, top_groups, per_group, n_queries > 1);
    int32_t rc;
    bool any_group = false, any_root = false;
    if ((rc = check_grouped_args(req)) ||
        (rc = request_filters(req, frame_ids, filter_offsets, filter_modes, n_filters, query_filter)) ||
        (rc = request_where_list(req, wheres, n_wheres, query_where)) ||
        (rc = check_group_offsets(where_group_offsets, n_wheres, where_groups, &any_group)) ||
        (rc = near_clauses(wheres, n_wheres, req.wheres)))
        return rc;
    request_root_clauses(req, where_roots, n_wheres, &any_root);
    if (!any_root)                     // no where has a root clause: the entry point without the clause
        return wax_vs_search_batch_grouped_multi_where_groups(e, queries, n_queries, query_len, top_groups, per_group,
                                                              frame_ids, filter_offsets, filter_modes, n_filters,
                                                              query_filter, wheres, n_wheres, query_where,
                                                              where_group_offsets, where_groups, out_ids, out_scores,
                                                              out_groups, out_stride, out_n);
    request_id_lists(req, n_wheres, where_group_offsets, where_groups, &Clause::groups);
    canonical_wheres(req);
    return search_grouped(e, req, out_ids, out_scores, out_groups, out_stride, out_n);
}

// ---- sharded grouped search (waxvs_group_batch.cuh, waxvs_shard.cuh) ------------------------------------------------
// The checks of the sharded grouped entry points: those of wax_vs_search_batch_grouped_multi_where but the host outputs,
// then the cap on the groups, before the engine is locked, so every rank fails alike before any exchange; then the
// device pointers.  Builds the clauses.
static int32_t request_shard_grouped(SearchRequest &req, const uint64_t *frame_ids, const uint64_t *filter_offsets,
                                     const int32_t *filter_modes, uint32_t n_filters, const uint32_t *query_filter,
                                     const wax_vs_where_near *wheres, uint32_t n_wheres, const uint32_t *query_where,
                                     const float *d_queries, const void *d_out) {
    int32_t rc;
    if ((rc = check_grouped_args(req)) ||
        (rc = request_filters(req, frame_ids, filter_offsets, filter_modes, n_filters, query_filter)) ||
        (rc = request_where_list(req, wheres, n_wheres, query_where)))
        return rc;
    if (clamp_topk(req.top_k) > WAX_VS_SHARD_MAX_GROUPS)
        return fail(WAX_VS_ERR_UNSUPPORTED, "sharded grouped search takes clamp(top_groups) <= %d (got %u)",
                    WAX_VS_SHARD_MAX_GROUPS, clamp_topk(req.top_k));
    if (!d_queries || !d_out) return fail(WAX_VS_ERR_NULL, "NULL argument");
    return near_clauses(wheres, n_wheres, req.wheres);
}

// Round 1 (wax_vs_shard_grouped_heads_device, and each shard of a multi-device handle): this shard's
// search_grouped_host, delivered as records on the device (ShardHeads).  The queries come to the host once, as the host
// form takes them.
static int32_t grouped_heads_device(wax_vs_engine *e, const SearchRequest &req, const float *d_queries, uint64_t row_offset,
                                    wax_vs_group_candidate *d_heads, void *cuda_stream) {
    const uint32_t n_queries = req.n_queries;
    if (n_queries == 0) return WAX_VS_OK;
    const size_t slots = static_cast<size_t>(clamp_topk(req.top_k)) * req.per_group;
    std::vector<float> queries(static_cast<size_t>(n_queries) * e->dims);
    {
        DeviceGuard g(e->device);
        if (!g.ok) return g.error();
        const cudaStream_t s = static_cast<cudaStream_t>(cuda_stream);
        CUDA_TRY(cudaMemsetAsync(d_heads, 0, n_queries * slots * sizeof(wax_vs_group_candidate), s));
        CUDA_TRY(cudaMemcpyAsync(queries.data(), d_queries, queries.size() * sizeof(float), cudaMemcpyDeviceToHost, s));
        CUDA_TRY(cudaStreamSynchronize(s));
    }
    std::vector<uint32_t> no_n(n_queries);
    const ShardHeads heads{row_offset, d_heads};
    return search_grouped_host(e, req, queries.data(), nullptr, nullptr, nullptr, 0, no_n.data(), &heads);
}

int32_t wax_vs_shard_grouped_heads_device(wax_vs_engine *e, const float *d_queries, uint32_t n_queries, int64_t top_groups,
                                          uint32_t per_group, const uint64_t *frame_ids, const uint64_t *filter_offsets,
                                          const int32_t *filter_modes, uint32_t n_filters, const uint32_t *query_filter,
                                          const wax_vs_where_near *wheres, uint32_t n_wheres, const uint32_t *query_where,
                                          uint64_t row_offset, wax_vs_group_candidate *d_heads, void *cuda_stream) {
    WAX_VS_MULTI_REFUSE(e, "wax_vs_shard_grouped_heads_device");
    if (!e) return fail(WAX_VS_ERR_NULL, "NULL argument");
    SearchRequest req(nullptr, n_queries, e->dims, top_groups, per_group, n_queries > 1);
    const int32_t rc = request_shard_grouped(req, frame_ids, filter_offsets, filter_modes, n_filters, query_filter, wheres,
                                             n_wheres, query_where, d_queries, d_heads);
    return rc ? rc : grouped_heads_device(e, req, d_queries, row_offset, d_heads, cuda_stream);
}

// Merge 1 (merge_group_heads_kernel): stateless, enqueued on the caller's stream.
int32_t wax_vs_merge_group_heads_device(wax_vs_engine *e, const wax_vs_group_candidate *d_gathered, uint32_t world,
                                        uint32_t n_queries, int64_t top_groups, uint32_t per_group,
                                        wax_vs_group_candidate *d_chosen, void *cuda_stream) {
    WAX_VS_MULTI_REFUSE(e, "wax_vs_merge_group_heads_device");
    if (!e || !d_gathered || !d_chosen) return fail(WAX_VS_ERR_NULL, "NULL argument");
    if (world == 0 || world > WAX_VS_SHARD_MAX_RANKS)
        return fail(WAX_VS_ERR_ARGUMENT, "world must be in [1, %d] (got %u)", WAX_VS_SHARD_MAX_RANKS, world);
    if (per_group == 0 || per_group > WAX_VS_MAX_PER_GROUP)
        return fail(WAX_VS_ERR_ARGUMENT, "per_group must be in [1, %d] (got %u)", WAX_VS_MAX_PER_GROUP, per_group);
    const uint32_t n_top = clamp_topk(top_groups);
    if (n_top > WAX_VS_SHARD_MAX_GROUPS)
        return fail(WAX_VS_ERR_UNSUPPORTED, "sharded grouped search takes clamp(top_groups) <= %d (got %u)",
                    WAX_VS_SHARD_MAX_GROUPS, n_top);
    if (n_queries == 0) return WAX_VS_OK;
    DeviceGuard g(e->device);
    if (!g.ok) return g.error();
    uint32_t pow2 = 32;
    while (pow2 < world * n_top) pow2 <<= 1;
    const size_t smem = static_cast<size_t>(pow2) * (sizeof(uint64_t) + 3 * sizeof(uint32_t));
    using Gathered = GatheredLists<wax_vs_group_candidate>;
    CUDA_TRY(grant_smem(e, merge_group_heads_kernel<Gathered>, smem));
    merge_group_heads_kernel<<<n_queries, 1024, smem, static_cast<cudaStream_t>(cuda_stream)>>>(
        Gathered{d_gathered, static_cast<size_t>(n_queries) * n_top * per_group}, world, n_queries, n_top, per_group, pow2,
        d_chosen);
    CUDA_TRY(cudaGetLastError());
    return WAX_VS_OK;
}

// Round 2 on the caller's stream (wax_vs_shard_grouped_expand_device, and each shard of a multi-device handle): the
// lookup kernel copies the groups this rank listed and lists the ones it must score; those run as the batched grouped
// search's expansions (expand_in_passes) under each query's (where, id filter) pair, and their keys become records.
static int32_t grouped_expand_device(wax_vs_engine *e, const SearchRequest &req, const float *d_queries,
                                     const wax_vs_group_candidate *d_chosen, const wax_vs_group_candidate *d_own_heads,
                                     uint64_t row_offset, wax_vs_candidate *d_rows, void *cuda_stream) {
    const uint32_t n_queries = req.n_queries, per_group = req.per_group;
    if (n_queries == 0) return WAX_VS_OK;
    std::shared_lock<std::shared_mutex> r(e->rw);
    DeviceGuard g(e->device);
    if (!g.ok) return g.error();
    SearchCtx *c = nullptr;
    int32_t rc;
    if ((rc = ctx_for_stream(e, cuda_stream, &c))) return rc;
    const cudaStream_t s = c->stream;
    const uint32_t n_top = clamp_topk(req.top_k);
    const size_t n_slots = static_cast<size_t>(n_queries) * n_top;
    e->async_pending.store(true);
    CUDA_TRY(cudaMemsetAsync(d_rows, 0, n_slots * per_group * sizeof(wax_vs_candidate), s));
    if (e->n_rows == 0) return WAX_VS_OK;
    if ((rc = ensure_group_index(e, c))) return rc;
    const auto &gi = e->gindex;
    if ((rc = c->d_bg_expand.ensure(n_slots, "grouped batch expansions")) ||
        (rc = c->h_bg_expand.ensure(n_slots, "grouped batch expansion staging")) ||
        (rc = c->d_bg_status.ensure(1, "grouped batch status")) || (rc = c->h_bg_status.ensure(1, "grouped batch status staging")))
        return rc;
    CUDA_TRY(cudaMemsetAsync(c->d_bg_status, 0, sizeof(uint32_t), s));
    const uint64_t warps_per_cta = 256 / 32;
    shard_group_lookup_kernel<<<static_cast<uint32_t>((n_slots + warps_per_cta - 1) / warps_per_cta), 256, 0, s>>>(
        d_chosen, d_own_heads, n_queries, n_top, per_group, gi.ids, gi.n_groups, gi.starts, d_rows, c->d_bg_expand,
        c->d_bg_status);
    CUDA_TRY(cudaGetLastError());
    CUDA_TRY(cudaMemcpyAsync(c->h_bg_status, c->d_bg_status, sizeof(uint32_t), cudaMemcpyDeviceToHost, s));
    CUDA_TRY(cudaStreamSynchronize(s));
    const uint32_t n_exp = c->h_bg_status[0];
    if (n_exp == 0) return WAX_VS_OK;
    uint64_t launches = 1, passes = 0;
    CUDA_TRY(cudaMemcpyAsync(c->h_bg_expand, c->d_bg_expand, n_exp * sizeof(CoverExpand), cudaMemcpyDeviceToHost, s));
    // the call's (where, id filter) pairs, their rows staged as run_filtered stages them, the queries in caller order
    WherePlan wp;
    if ((rc = plan_request(e, c, req, req.top_k, wp, false)) || (rc = stage_pair_rows(e, c, wp.fs, &launches))) return rc;
    const size_t qfloats = static_cast<size_t>(n_queries) * e->dims;
    if ((rc = c->d_queries.ensure(qfloats, "query buffer")) ||
        (rc = c->d_bg_keys.ensure(n_slots * per_group, "grouped batch keys")))
        return rc;
    CUDA_TRY(cudaMemcpyAsync(c->d_queries, d_queries, qfloats * sizeof(float), cudaMemcpyDeviceToDevice, s));
    CUDA_TRY(cudaStreamSynchronize(s));              // the expansion list is on the host
    if ((rc = expand_in_passes(e, c, c->h_bg_expand, n_exp, wp.pair_of, wp, n_top, per_group, &launches, &passes)))
        return rc;
    ShardRowInfo ri{row_offset, e->id_base, nullptr, device_row_keys(e), gi.row_group, gi.ids};
    if ((rc = sync_device_ids(e, &ri.ids))) return rc;
    shard_group_expanded_kernel<<<n_exp, 128, 0, s>>>(c->d_bg_expand, c->d_bg_keys, n_top, per_group, ri, d_rows);
    CUDA_TRY(cudaGetLastError());
    CUDA_TRY(cudaStreamSynchronize(s));              // the host arrays of the plan must outlive their uploads
    std::lock_guard<std::mutex> pg(e->pool_mu);
    e->shard_grouped_expanded_groups += n_exp;
    return WAX_VS_OK;
}

int32_t wax_vs_shard_grouped_expand_device(wax_vs_engine *e, const float *d_queries, uint32_t n_queries,
                                           int64_t top_groups, uint32_t per_group, const uint64_t *frame_ids,
                                           const uint64_t *filter_offsets, const int32_t *filter_modes, uint32_t n_filters,
                                           const uint32_t *query_filter, const wax_vs_where_near *wheres,
                                           uint32_t n_wheres, const uint32_t *query_where,
                                           const wax_vs_group_candidate *d_chosen,
                                           const wax_vs_group_candidate *d_own_heads, uint64_t row_offset,
                                           wax_vs_candidate *d_rows, void *cuda_stream) {
    WAX_VS_MULTI_REFUSE(e, "wax_vs_shard_grouped_expand_device");
    if (!e) return fail(WAX_VS_ERR_NULL, "NULL argument");
    SearchRequest req(nullptr, n_queries, e->dims, top_groups, per_group, n_queries > 1);
    const int32_t rc = request_shard_grouped(req, frame_ids, filter_offsets, filter_modes, n_filters, query_filter, wheres,
                                             n_wheres, query_where, d_queries, d_rows);
    if (rc) return rc;
    if (!d_chosen || !d_own_heads) return fail(WAX_VS_ERR_NULL, "NULL argument");
    return grouped_expand_device(e, req, d_queries, d_chosen, d_own_heads, row_offset, d_rows, cuda_stream);
}

// ---- persistence ---------------------------------------------------------------------------------------------
static uint64_t mv2v_length(const wax_vs_engine *e) {
    return 36ull + e->n_rows * e->dims * 4ull + 8ull + e->n_rows * 8ull;
}

int32_t wax_vs_serialized_length(wax_vs_engine *e, uint64_t *out) {
    if (e && e->multi && out) { std::shared_lock<std::shared_mutex> r(e->multi->rw); *out = multi_mv2v_length(e->multi->total(), e->dims); return WAX_VS_OK; }
    if (!e || !out) return fail(WAX_VS_ERR_NULL, "NULL argument");
    std::shared_lock<std::shared_mutex> r(e->rw);
    *out = mv2v_length(e);
    return WAX_VS_OK;
}

int32_t wax_vs_serialize(wax_vs_engine *e, uint8_t *dst, uint64_t cap, uint64_t *out_len) {
    if (e && e->multi) return multi_serialize(e->multi, e->dims, e->similarity, dst, cap, out_len);
    if (!e || !dst) return fail(WAX_VS_ERR_NULL, "NULL argument");
    std::shared_lock<std::shared_mutex> r(e->rw);
    const uint64_t need = mv2v_length(e);
    if (out_len) *out_len = need;
    if (cap < need) return fail(WAX_VS_ERR_BUFFER, "serialize needs %llu bytes, buffer has %llu",
                                static_cast<unsigned long long>(need), static_cast<unsigned long long>(cap));
    DeviceGuard g(e->device);
    uint8_t *p = dst;
    const uint8_t magic[4] = {0x4D, 0x56, 0x32, 0x56};  // "MV2V" (:686)
    memcpy(p, magic, 4); p += 4;
    const uint16_t version = 1; memcpy(p, &version, 2); p += 2;  // :687-688
    *p++ = 2;                                                     // encoding (:689)
    *p++ = e->similarity;                                         // :690
    memcpy(p, &e->dims, 4); p += 4;                               // :691-692
    memcpy(p, &e->n_rows, 8); p += 8;                             // :693-694
    const uint64_t vbytes = e->n_rows * e->dims * 4ull;
    memcpy(p, &vbytes, 8); p += 8;                                // :697-699
    memset(p, 0, 8); p += 8;                                      // reserved (:700)
    if (vbytes) {                                                 // :703-705, through the pinned double-buffered D2H pipeline
        std::lock_guard<std::mutex> ig(e->ingest_mu);             // serialize holds only the READ lock: one exporter at a time
        int32_t rc = download_bytes(e, p, e->d_corpus, vbytes);
        if (rc) return rc;
    }
    p += vbytes;
    const uint64_t ibytes = e->n_rows * 8ull;
    memcpy(p, &ibytes, 8); p += 8;                                // :707-709
    if (e->ids_identity) {
        for (uint64_t i = 0; i < e->n_rows; ++i) { const uint64_t id = e->id_base + i; memcpy(p + i * 8, &id, 8); }
    } else if (ibytes) {
        memcpy(p, e->ids.data(), ibytes);                         // :710
    }
    return WAX_VS_OK;
}

// deserialize for wax_vs_deserialize (all rows, no keys) and wax_vs_deserialize_rows (rows [first, first + n), keyed).
static int32_t deserialize_rows(wax_vs_engine *e, const uint8_t *src, uint64_t len, bool all, uint64_t first, uint64_t n) {
    if (!e || !src) return fail(WAX_VS_ERR_NULL, "NULL argument");
    std::unique_lock<std::shared_mutex> w(e->rw);
    // Reason strings follow MetalVectorEngine.deserialize (:716-815) / VectorSerializer.decodeVecSegment (:84-157).
    if (len < 36) return fail(WAX_VS_ERR_FORMAT, "Metal segment too small: %llu bytes", static_cast<unsigned long long>(len));
    const uint8_t magic[4] = {0x4D, 0x56, 0x32, 0x56};
    if (memcmp(src, magic, 4) != 0) return fail(WAX_VS_ERR_FORMAT, "Metal segment magic mismatch");
    uint16_t version; memcpy(&version, src + 4, 2);
    if (version != 1) return fail(WAX_VS_ERR_FORMAT, "Unsupported Metal segment version %u", version);
    if (src[6] != 2) return fail(WAX_VS_ERR_FORMAT, "Unsupported Metal segment encoding %u", src[6]);
    if (src[7] > 2 || src[7] != e->similarity)
        return fail(WAX_VS_ERR_FORMAT, "Metric mismatch: expected %u, got %u", e->similarity, src[7]);
    uint32_t dims; memcpy(&dims, src + 8, 4);
    if (dims != e->dims) return fail(WAX_VS_ERR_FORMAT, "Dimension mismatch: expected %u, got %u", e->dims, dims);
    uint64_t count, vbytes; memcpy(&count, src + 12, 8); memcpy(&vbytes, src + 20, 8);
    for (int i = 0; i < 8; ++i)
        if (src[28 + i] != 0) return fail(WAX_VS_ERR_FORMAT, "Metal segment reserved bytes must be zero");
    if (count > 0xFFFFFFFFull) return fail(WAX_VS_ERR_CAPACITY, "capacity exceeded: limit %llu, requested %llu", 0xFFFFFFFFull, static_cast<unsigned long long>(count));
    if (vbytes != count * static_cast<uint64_t>(dims) * 4ull) return fail(WAX_VS_ERR_FORMAT, "Vector data length mismatch");
    if (len < 36 + vbytes + 8) return fail(WAX_VS_ERR_FORMAT, "Metal segment missing frameId length");
    uint64_t ibytes; memcpy(&ibytes, src + 36 + vbytes, 8);
    if (ibytes != count * 8ull) return fail(WAX_VS_ERR_FORMAT, "FrameId data length mismatch");
    if (len != 36 + vbytes + 8 + ibytes)
        return fail(WAX_VS_ERR_FORMAT, "vec segment length mismatch: expected %llu, got %llu",
                    static_cast<unsigned long long>(36 + vbytes + 8 + ibytes), static_cast<unsigned long long>(len));
    if (all) first = 0, n = count;
    else if (first > count || n > count - first)
        return fail(WAX_VS_ERR_ARGUMENT, "rows [%llu, %llu + %llu) are outside the segment's %llu rows",
                    static_cast<unsigned long long>(first), static_cast<unsigned long long>(first),
                    static_cast<unsigned long long>(n), static_cast<unsigned long long>(count));
    const size_t row_bytes = static_cast<size_t>(dims) * 4u;
    DeviceGuard g(e->device);
    drain_device_path(e);
    int32_t rc = set_capacity(e, std::max<uint64_t>(n, 64));  // reservedCapacity = max(...) (:791-792)
    if (rc) return rc;
    if (n && (rc = upload_bytes(e, e->d_corpus, src + 36 + first * row_bytes, n * row_bytes)))  // :794-799, pinned H2D
        return rc;
    e->n_rows = n;
    e->ids.resize(n);
    if (n) memcpy(e->ids.data(), src + 36 + vbytes + 8 + first * 8, n * 8);  // :809-811
    e->ids_identity = false;
    e->map_valid = false;
    e->ids_sorted = true;
    for (uint64_t i = 1; i < n && e->ids_sorted; ++i) e->ids_sorted = e->ids[i] > e->ids[i - 1];
    e->d_ids_dirty = true;
    e->keys_set = !all;                     // a slice's rows keep their positions in the segment as keys
    e->keys.resize(e->keys_set ? n : 0);
    for (uint64_t i = 0; i < e->keys.size(); ++i) e->keys[i] = first + i;
    e->keys.shrink_to_fit();
    if ((rc = upload_row_keys(e, 0))) return rc;
    e->groups_set = false;                  // MV2V has no groups: the caller re-applies them (wax_vs_set_groups)
    e->groups.clear(); e->groups.shrink_to_fit();
    e->attrs_set = false;                   // nor attributes: the caller re-applies them (wax_vs_set_attributes)
    e->attrs.clear(); e->attrs.shrink_to_fit();
    e->locs_set = false;
    e->locs.clear(); e->locs.shrink_to_fit();
    clear_terms(e);
    e->roots.ids.clear(); e->roots.ids.shrink_to_fit();   // nor root tags: the caller re-applies them (wax_vs_set_root_tags)
    e->roots.tags.clear(); e->roots.tags.shrink_to_fit();
    invalidate_row_caches(e, 0);
    return WAX_VS_OK;
}

int32_t wax_vs_deserialize(wax_vs_engine *e, const uint8_t *src, uint64_t len) {
    if (e && e->multi) return multi_deserialize(e->multi, e->dims, e->similarity, src, len);
    return deserialize_rows(e, src, len, true, 0, 0);
}

int32_t wax_vs_deserialize_rows(wax_vs_engine *e, const uint8_t *src, uint64_t len, uint64_t first, uint64_t n) {
    WAX_VS_MULTI_REFUSE(e, "wax_vs_deserialize_rows");
    return deserialize_rows(e, src, len, false, first, n);
}

int32_t wax_vs_export_rows(wax_vs_engine *e, uint64_t first, uint64_t n, uint64_t *out_ids, float *out_vectors,
                           uint64_t *out_keys) {
    WAX_VS_MULTI_REFUSE(e, "wax_vs_export_rows");
    if (!e) return fail(WAX_VS_ERR_NULL, "engine is NULL");
    std::shared_lock<std::shared_mutex> r(e->rw);
    if (first > e->n_rows || n > e->n_rows - first) return fail(WAX_VS_ERR_ARGUMENT, "row range out of bounds");
    for (uint64_t i = 0; i < n; ++i) {
        if (out_ids) out_ids[i] = frame_id_of(e, first + i);
        if (out_keys) out_keys[i] = e->keys_set ? e->keys[first + i] : first + i;
    }
    if (out_vectors && n) {
        DeviceGuard g(e->device);
        if (!g.ok) return g.error();
        std::lock_guard<std::mutex> ig(e->ingest_mu);             // one exporter at a time (as serialize)
        return download_bytes(e, out_vectors, e->d_corpus + first * e->dims, n * e->dims * sizeof(float));
    }
    return WAX_VS_OK;
}

int32_t wax_vs_export_rows_device(wax_vs_engine *e, uint64_t first, uint64_t n, float *d_out, void *cuda_stream) {
    WAX_VS_MULTI_REFUSE(e, "wax_vs_export_rows_device");
    if (!e) return fail(WAX_VS_ERR_NULL, "engine is NULL");
    std::shared_lock<std::shared_mutex> r(e->rw);
    if (first > e->n_rows || n > e->n_rows - first) return fail(WAX_VS_ERR_ARGUMENT, "row range out of bounds");
    if (n == 0) return WAX_VS_OK;
    if (!d_out) return fail(WAX_VS_ERR_NULL, "d_out is NULL");
    DeviceGuard g(e->device);
    if (!g.ok) return g.error();
    e->async_pending.store(true);              // a mutator drains the copy before it moves a row
    CUDA_TRY(cudaMemcpyAsync(d_out, e->d_corpus + first * e->dims, n * e->dims * sizeof(float), cudaMemcpyDeviceToDevice,
                             static_cast<cudaStream_t>(cuda_stream)));
    return WAX_VS_OK;
}

int32_t wax_vs_export_columns(wax_vs_engine *e, uint64_t first, uint64_t n, wax_vs_row_columns *out_columns,
                              uint64_t *out_term_offsets, uint64_t *out_terms, uint64_t terms_cap, uint64_t *out_terms_len,
                              uint32_t *out_set) {
    WAX_VS_MULTI_REFUSE(e, "wax_vs_export_columns");
    if (!e) return fail(WAX_VS_ERR_NULL, "engine is NULL");
    std::shared_lock<std::shared_mutex> r(e->rw);
    if (first > e->n_rows || n > e->n_rows - first) return fail(WAX_VS_ERR_ARGUMENT, "row range out of bounds");
    uint64_t len = 0;
    if (e->terms_set)
        for (uint64_t i = first; i < first + n; ++i) len += e->term_refs[i].n;
    if (out_terms && terms_cap < len)
        return fail(WAX_VS_ERR_BUFFER, "terms_cap %llu < %llu term ids in the rows", static_cast<unsigned long long>(terms_cap),
                    static_cast<unsigned long long>(len));
    if (out_terms_len) *out_terms_len = len;
    if (out_set)
        *out_set = (e->groups_set ? WAX_VS_COLUMN_GROUPS : 0u) | (e->attrs_set ? WAX_VS_COLUMN_ATTRIBUTES : 0u) |
                   (e->locs_set ? WAX_VS_COLUMN_LOCATIONS : 0u) | (e->terms_set ? WAX_VS_COLUMN_TERMS : 0u);
    uint64_t pos = 0;
    for (uint64_t j = 0; j < n; ++j) {
        const uint64_t row = first + j;
        if (out_columns) {
            const AttrRow a = e->attrs_set ? e->attrs[row] : AttrRow{0, 0};
            const LocRow l = e->locs_set ? e->locs[row] : LocRow{kNoLocation, 0};
            out_columns[j] = wax_vs_row_columns{e->groups_set ? e->groups[row] : frame_id_of(e, row), a.ts, a.tags, l.lat, l.lon};
        }
        const wax_vs_engine::TermRef t = e->terms_set ? e->term_refs[row] : wax_vs_engine::TermRef{0, 0};
        if (out_term_offsets) out_term_offsets[j] = pos;
        if (out_terms && t.n) memcpy(out_terms + pos, e->term_pool.data() + t.off, t.n * sizeof(uint64_t));
        pos += t.n;
    }
    if (out_term_offsets) out_term_offsets[n] = pos;
    return WAX_VS_OK;
}

// ---- instrumentation ------------------------------------------------------------------------------------------
int32_t wax_vs_debug_pool_stats(wax_vs_engine *e, uint64_t *allocations, uint64_t *reuses) {
    WAX_VS_MULTI_REFUSE(e, "wax_vs_debug_pool_stats");
    if (!e) return fail(WAX_VS_ERR_NULL, "engine is NULL");
    std::lock_guard<std::mutex> g(e->pool_mu);
    if (allocations) *allocations = e->pool_allocs;
    if (reuses) *reuses = e->pool_reuses;
    return WAX_VS_OK;
}

int32_t wax_vs_debug_fill_synthetic(wax_vs_engine *e, uint64_t seed, uint64_t first_row, uint64_t rows,
                                    uint64_t id_base, int32_t normalize) {
    WAX_VS_MULTI_REFUSE(e, "wax_vs_debug_fill_synthetic");
    if (!e) return fail(WAX_VS_ERR_NULL, "engine is NULL");
    if (rows > 0xFFFFFFFFull) return fail(WAX_VS_ERR_CAPACITY, "capacity exceeded: limit %llu, requested %llu", 0xFFFFFFFFull, static_cast<unsigned long long>(rows));
    std::unique_lock<std::shared_mutex> w(e->rw);
    DeviceGuard g(e->device);
    drain_device_path(e);
    e->n_rows = 0;
    int32_t rc = set_capacity(e, std::max<uint64_t>(rows, 64));
    if (rc) return rc;
    if (rows) {
        const unsigned blocks = static_cast<unsigned>((rows + 255) / 256);
        synth_fill_kernel<<<blocks, 256>>>(e->d_corpus, rows, e->dims, seed, first_row, normalize);
        CUDA_TRY(cudaGetLastError());
        CUDA_TRY(cudaDeviceSynchronize());
    }
    e->n_rows = rows;
    e->ids.clear(); e->ids.shrink_to_fit();
    e->ids_identity = true; e->id_base = id_base;
    e->map = IdMap(); e->map_valid = true; e->ids_sorted = true;
    e->d_ids_dirty = true;
    e->keys_set = false;
    e->keys.clear(); e->keys.shrink_to_fit();
    e->groups_set = false;
    e->groups.clear(); e->groups.shrink_to_fit();
    e->attrs_set = false;
    e->attrs.clear(); e->attrs.shrink_to_fit();
    e->locs_set = false;
    e->locs.clear(); e->locs.shrink_to_fit();
    clear_terms(e);
    invalidate_row_caches(e, 0);
    return WAX_VS_OK;
}

int32_t wax_vs_debug_read_rows(wax_vs_engine *e, uint64_t first, uint64_t n, float *dst) {
    WAX_VS_MULTI_REFUSE(e, "wax_vs_debug_read_rows");
    if (!e || !dst) return fail(WAX_VS_ERR_NULL, "NULL argument");
    std::shared_lock<std::shared_mutex> r(e->rw);
    if (first + n > e->n_rows) return fail(WAX_VS_ERR_ARGUMENT, "row range out of bounds");
    DeviceGuard g(e->device);
    if (n) CUDA_TRY(cudaMemcpy(dst, e->d_corpus + first * e->dims, n * e->dims * sizeof(float), cudaMemcpyDeviceToHost));
    return WAX_VS_OK;
}

int32_t wax_vs_debug_time_search(wax_vs_engine *e, uint32_t n_queries, int64_t top_k, uint64_t seed,
                                 uint32_t warmup, uint32_t iters, float *out_ms_total, uint64_t *out_launches) {
    WAX_VS_MULTI_REFUSE(e, "wax_vs_debug_time_search");
    if (!e || !out_ms_total) return fail(WAX_VS_ERR_NULL, "NULL argument");
    if (n_queries == 0) n_queries = 1;
    std::shared_lock<std::shared_mutex> r(e->rw);
    DeviceGuard g(e->device);
    CtxLease lease(e);
    int32_t rc = lease.acquire();
    if (rc) return rc;
    SearchCtx *c = lease.c;
    const uint32_t k_eff = clamp_topk(top_k);
    const size_t qfloats = static_cast<size_t>(n_queries) * e->dims;
    if ((rc = c->d_queries.ensure(qfloats, "query buffer"))) return rc;
    if ((rc = c->d_out.ensure(static_cast<size_t>(n_queries) * k_eff, "result buffer"))) return rc;
    // n_queries distinct unit queries (generator stream `seed`); step i searches query i mod n_queries.
    synth_fill_kernel<<<(n_queries + 255) / 256, 256, 0, c->stream>>>(c->d_queries, n_queries, e->dims, seed, 0, 1);
    CUDA_TRY(cudaGetLastError());
    uint64_t launches = 0;
    // time_overlap: consecutive (independent) queries alternate over two streams so that one scan's tail overlaps
    // the next one's prologue -- what the sharded engine does with search_many_async.
    CtxLease lease2(e);
    if (e->tune.time_overlap) {
        if ((rc = lease2.acquire())) return rc;
        if ((rc = lease2.c->d_out.ensure(static_cast<size_t>(n_queries) * k_eff, "result buffer"))) return rc;
    }
    SearchCtx *c2 = lease2.c;
    // the shadow the route takes is cached per corpus version: bring it up to date outside the timed region
    if (shadow_route_applies(e)) {
        bool use = false;
        RouteForm form = kRouteBf16;
        TmaConfig cfg{};
        if ((rc = select_route_form(e, c->stream, false, &use, &form, &cfg))) return rc;
    }
    for (uint32_t it = 0; it < warmup + iters; ++it) {
        if (it == warmup) {
            launches = 0;
            if (c2) { CUDA_TRY(cudaEventRecord(c2->ev0, c2->stream)); CUDA_TRY(cudaStreamWaitEvent(c->stream, c2->ev0, 0)); }
            CUDA_TRY(cudaEventRecord(c->ev0, c->stream));
            if (c2) CUDA_TRY(cudaStreamWaitEvent(c2->stream, c->ev0, 0));
        }
        const uint32_t qi = it % n_queries;
        SearchCtx *cc = (c2 && (it & 1u)) ? c2 : c;
        if (c2 && it == 0) { CUDA_TRY(cudaEventRecord(c->ev1, c->stream)); CUDA_TRY(cudaStreamWaitEvent(c2->stream, c->ev1, 0)); }  // queries ready
        rc = enqueue_search(e, cc, c->d_queries + static_cast<size_t>(qi) * e->dims, k_eff, 0,
                            cc->d_out + static_cast<size_t>(qi) * k_eff, nullptr, cc->stream, &launches, nullptr, nullptr,
                            nullptr, false, true);
        if (rc) { cudaStreamSynchronize(c->stream); if (c2) cudaStreamSynchronize(c2->stream); return rc; }
    }
    if (c2) { CUDA_TRY(cudaEventRecord(c2->ev1, c2->stream)); CUDA_TRY(cudaStreamWaitEvent(c->stream, c2->ev1, 0)); }
    CUDA_TRY(cudaEventRecord(c->ev1, c->stream));
    CUDA_TRY(cudaStreamSynchronize(c->stream));
    CUDA_TRY(cudaEventElapsedTime(out_ms_total, c->ev0, c->ev1));
    if (out_launches) *out_launches = launches;
    return WAX_VS_OK;
}

int32_t wax_vs_debug_stream_read(wax_vs_engine *e, uint32_t iters, float *out_best_ms, uint64_t *out_bytes) {
    WAX_VS_MULTI_REFUSE(e, "wax_vs_debug_stream_read");
    if (!e || !out_best_ms || !out_bytes) return fail(WAX_VS_ERR_NULL, "NULL argument");
    std::shared_lock<std::shared_mutex> r(e->rw);
    DeviceGuard g(e->device);
    CtxLease lease(e);
    int32_t rc = lease.acquire();
    if (rc) return rc;
    SearchCtx *c = lease.c;
    const uint64_t bytes = e->n_rows * e->dims * sizeof(float) / 16 * 16;
    *out_bytes = bytes;
    *out_best_ms = 0.0f;
    if (bytes == 0) return WAX_VS_OK;
    float best = 1e30f;
    for (uint32_t it = 0; it < iters + 2; ++it) {
        CUDA_TRY(cudaEventRecord(c->ev0, c->stream));
        stream_read_kernel<<<e->sm_count * 4, 512, 0, c->stream>>>(reinterpret_cast<const uint4 *>(e->d_corpus),
                                                                     bytes / 16, c->d_ticket + 2);
        CUDA_TRY(cudaGetLastError());
        CUDA_TRY(cudaEventRecord(c->ev1, c->stream));
        CUDA_TRY(cudaStreamSynchronize(c->stream));
        float ms = 0;
        CUDA_TRY(cudaEventElapsedTime(&ms, c->ev0, c->ev1));
        if (it >= 2 && ms < best) best = ms;
    }
    CUDA_TRY(cudaMemsetAsync(c->d_ticket, 0, 4 * sizeof(uint32_t), c->stream));
    CUDA_TRY(cudaStreamSynchronize(c->stream));
    *out_best_ms = best;
    return WAX_VS_OK;
}

// Host <-> device transfer rates of this machine, in GB/s, for `bytes` of pageable host memory:
//   [0] one-thread memcpy pageable -> pinned     [1] the staging copy with the engine's worker threads
//   [2] DMA pinned -> HBM                         [3] DMA HBM -> pinned
//   [4] upload pipeline pageable -> HBM           [5] download pipeline HBM -> pageable       [6] worker threads
int32_t wax_vs_debug_transfer_probe(wax_vs_engine *e, uint64_t bytes, float *out7) {
    WAX_VS_MULTI_REFUSE(e, "wax_vs_debug_transfer_probe");
    if (!e || !out7) return fail(WAX_VS_ERR_NULL, "NULL argument");
    std::unique_lock<std::shared_mutex> w(e->rw);
    DeviceGuard g(e->device);
    bytes = std::max<uint64_t>(bytes, 1u << 20);
    int32_t rc = ingest_staging(e, bytes);
    if (rc) return rc;
    auto &ig = e->ing;
    if ((rc = ig.d_stage.ensure(static_cast<size_t>((bytes + 3) / 4), "probe buffer"))) return rc;
    std::vector<uint8_t> host(bytes, 1);
    auto secs = [](auto t0) { return std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count(); };
    uint8_t *probe_pin = nullptr;
    {
        std::lock_guard<std::mutex> pool(g_staging_mu);
        if ((rc = shared_staging())) return rc;
        probe_pin = g_staging[0];
    }
    const size_t chunk = std::min<size_t>(kStagingBytes, bytes);
    auto best = [&](auto fn) { double b = 1e30; for (int i = 0; i < 3; ++i) { auto t0 = std::chrono::steady_clock::now(); fn(); b = std::min(b, secs(t0)); } return b; };
    out7[0] = static_cast<float>(chunk / 1e9 / best([&] { memcpy(probe_pin, host.data(), chunk); }));
    out7[1] = static_cast<float>(chunk / 1e9 / best([&] { parallel_memcpy(probe_pin, host.data(), chunk, ig.threads); }));
    out7[2] = static_cast<float>(chunk / 1e9 / best([&] { cudaMemcpyAsync(ig.d_stage, probe_pin, chunk, cudaMemcpyHostToDevice, ig.stream); cudaStreamSynchronize(ig.stream); }));
    out7[3] = static_cast<float>(chunk / 1e9 / best([&] { cudaMemcpyAsync(probe_pin, ig.d_stage, chunk, cudaMemcpyDeviceToHost, ig.stream); cudaStreamSynchronize(ig.stream); }));
    out7[4] = static_cast<float>(bytes / 1e9 / best([&] { upload_bytes(e, ig.d_stage, host.data(), bytes); }));
    out7[5] = static_cast<float>(bytes / 1e9 / best([&] { download_bytes(e, host.data(), ig.d_stage, bytes); }));
    out7[6] = static_cast<float>(ig.threads);
    CUDA_TRY(cudaGetLastError());
    return WAX_VS_OK;
}

// Where a single fused search spends its time (TMA-staged kernels with the selection tail): averages over `iters`
// searches, microseconds: [0] kernel start -> last warp leaves the scan loop, [1] -> last CTA has selected its k,
// [2] -> the last CTA starts the grid stage, [3] -> result written (kernel end), [4] event-timed duration of the
// launch on the stream (launch overhead = [4] - [3]).
int32_t wax_vs_debug_phase_trace(wax_vs_engine *e, int64_t top_k, uint32_t iters, float *out5) {
    WAX_VS_MULTI_REFUSE(e, "wax_vs_debug_phase_trace");
    if (!e || !out5) return fail(WAX_VS_ERR_NULL, "NULL argument");
    std::unique_lock<std::shared_mutex> w(e->rw);
    DeviceGuard g(e->device);
    CtxLease lease(e, true);     // also detaches the trace buffer
    int32_t rc = lease.acquire();
    if (rc) return rc;
    SearchCtx *c = lease.c;
    const uint32_t k_eff = clamp_topk(top_k);
    if ((rc = c->d_queries.ensure(static_cast<size_t>(e->dims), "query buffer"))) return rc;
    if ((rc = c->d_out.ensure(static_cast<size_t>(k_eff), "result buffer"))) return rc;
    synth_fill_kernel<<<1, 256, 0, c->stream>>>(c->d_queries, 1, e->dims, 99, 0, 1);
    unsigned long long *d_trace = nullptr;
    CUDA_TRY(cudaMalloc(&d_trace, 8 * sizeof(unsigned long long)));
    double acc[5] = {0, 0, 0, 0, 0};
    uint64_t launches = 0;
    for (uint32_t it = 0; it < iters + 3; ++it) {
        const unsigned long long init[8] = {~0ull, 0, 0, 0, 0, 0, 0, 0};
        cudaMemcpyAsync(d_trace, init, sizeof init, cudaMemcpyHostToDevice, c->stream);
        cudaStreamSynchronize(c->stream);
        e->debug_trace = d_trace;
        cudaEventRecord(c->ev0, c->stream);
        rc = enqueue_search(e, c, c->d_queries, k_eff, 0, c->d_out, nullptr, c->stream, &launches);
        cudaEventRecord(c->ev1, c->stream);
        e->debug_trace = nullptr;
        if (rc) { cudaStreamSynchronize(c->stream); cudaFree(d_trace); return rc; }
        unsigned long long t[8];
        cudaMemcpyAsync(t, d_trace, sizeof t, cudaMemcpyDeviceToHost, c->stream);
        cudaStreamSynchronize(c->stream);
        float ms = 0;
        cudaEventElapsedTime(&ms, c->ev0, c->ev1);
        if (it < 3) continue;
        for (int i = 0; i < 4; ++i) acc[i] += (t[i + 1] > t[0] && t[0] != ~0ull) ? (t[i + 1] - t[0]) * 1e-3 : 0.0;
        acc[4] += ms * 1e3;
    }
    cudaFree(d_trace);
    for (int i = 0; i < 5; ++i) out5[i] = static_cast<float>(acc[i] / std::max(iters, 1u));
    CUDA_TRY(cudaGetLastError());
    return WAX_VS_OK;
}

int32_t wax_vs_debug_batch_stats(wax_vs_engine *e, uint64_t *tensor_queries, uint64_t *fallback_queries) {
    WAX_VS_MULTI_REFUSE(e, "wax_vs_debug_batch_stats");
    if (!e) return fail(WAX_VS_ERR_NULL, "engine is NULL");
    std::lock_guard<std::mutex> g(e->pool_mu);
    if (tensor_queries) *tensor_queries = e->batch_tensor_queries;
    if (fallback_queries) *fallback_queries = e->batch_fallback_queries;
    return WAX_VS_OK;
}

int32_t wax_vs_debug_last_scan(wax_vs_engine *e, uint32_t out[10]) {
    WAX_VS_MULTI_REFUSE(e, "wax_vs_debug_last_scan");
    if (!e || !out) return fail(WAX_VS_ERR_NULL, "NULL argument");
    std::lock_guard<std::mutex> g(e->pool_mu);
    memcpy(out, e->last_scan, sizeof e->last_scan);
    return WAX_VS_OK;
}

int32_t wax_vs_debug_counter(wax_vs_engine *e, const char *name, uint64_t *out) {
    if (e && e->multi && name && out) return multi_counter(e->multi, name, out);
    if (!e || !name || !out) return fail(WAX_VS_ERR_NULL, "NULL argument");
    std::lock_guard<std::mutex> g(e->pool_mu);
    const wax_vs_engine::Shadow &bf = e->shadows[kRouteBf16], &i8 = e->shadows[kRouteInt8], &u4 = e->shadows[kRouteU4];
    if (!strcmp(name, "batch_tensor_queries")) *out = e->batch_tensor_queries;
    else if (!strcmp(name, "batch_fallback_queries")) *out = e->batch_fallback_queries;
    else if (!strcmp(name, "batch_bf16_queries")) *out = e->batch_bf16_queries;
    else if (!strcmp(name, "batch_retry_queries")) *out = e->batch_retry_queries;               // TF32 filter level
    else if (!strcmp(name, "batch_filter_bf16_queries")) *out = e->batch_filter_bf16_queries;   // bf16-shadow filter level
    else if (!strcmp(name, "shadow_bytes")) *out = bf.valid ? bf.rows * e->dims * sizeof(__nv_bfloat16) : 0;   // live rows
    else if (!strcmp(name, "shadow_capacity_bytes")) *out = bf.codes.cap * sizeof(uint32_t);                   // HBM held
    else if (!strcmp(name, "shadow_unavailable")) *out = bf.unavailable ? 1 : 0;   // bf16 shadow did not fit: TF32 level runs
    else if (!strcmp(name, "batch_tf32_queries")) *out = e->batch_tf32_queries;
    else if (!strcmp(name, "filter_bitset_passes")) *out = e->filter_bitset_passes;   // per-query filters: tensor sub-batches
    else if (!strcmp(name, "group_index_builds")) *out = e->group_index_builds;       // grouped search: device index builds
    else if (!strcmp(name, "where_group_units")) *out = e->where_group_units;         // where_groups search: units planned ...
    else if (!strcmp(name, "where_group_rows_walked")) *out = e->where_group_rows_walked;   // ... and the positions they walk
    else if (!strcmp(name, "root_column_builds")) *out = e->root_column_builds;       // where_roots search: root column builds
    else if (!strcmp(name, "attribute_uploads")) *out = e->attribute_uploads;         // where search: attribute mirror builds
    else if (!strcmp(name, "location_uploads")) *out = e->location_uploads;           // where_near search: location mirror builds
    else if (!strcmp(name, "term_index_builds")) *out = e->term_index_builds;         // where_terms search: term index builds
    else if (!strcmp(name, "term_index_bytes"))                                       // ... and the HBM the index holds
        *out = e->tindex.keys.cap * sizeof(uint64_t) + e->tindex.start.cap * sizeof(uint64_t) + e->tindex.postings.cap * sizeof(uint32_t);
    else if (!strcmp(name, "grouped_batch_covered_queries")) *out = e->grouped_batch_covered_queries;     // answered by the coverage level
    else if (!strcmp(name, "grouped_batch_expanded_groups")) *out = e->grouped_batch_expanded_groups;     // (query, group) expansions
    else if (!strcmp(name, "grouped_batch_fallback_queries")) *out = e->grouped_batch_fallback_queries;   // single-query pipeline
    else if (!strcmp(name, "grouped_batch_expansion_passes")) *out = e->grouped_batch_expansion_passes;   // bitset passes of the expansion
    else if (!strcmp(name, "shard_grouped_expanded_groups")) *out = e->shard_grouped_expanded_groups;     // sharded round 2: groups scored
    else if (!strcmp(name, "ingest_h2d_bytes")) *out = e->ingest_h2d_bytes;
    else if (!strcmp(name, "ingest_d2h_bytes")) *out = e->ingest_d2h_bytes;
    else if (!strcmp(name, "norms_rows")) *out = e->norms_rows;       // rows whose cached 1/|v| is valid
    else if (!strcmp(name, "shadow_rows")) *out = bf.rows;     // rows whose bf16 shadow is valid
    else if (!strcmp(name, "int8_shadow_bytes")) *out = i8.valid ? i8.rows * (e->dims + sizeof(float)) : 0;   // codes + scales
    else if (!strcmp(name, "int8_shadow_rows")) *out = i8.rows;  // rows whose int8 shadow is valid
    else if (!strcmp(name, "u4_shadow_bytes")) *out = u4.valid ? u4.rows * (e->dims / 2 + sizeof(float)) : 0;
    else if (!strcmp(name, "u4_shadow_rows")) *out = u4.rows;
    else if (!strcmp(name, "single_u4_queries")) *out = e->single_route_queries[kRouteU4];
    else if (!strcmp(name, "single_int8_queries")) *out = e->single_route_queries[kRouteInt8];   // single queries nominated from it
    else if (!strcmp(name, "batch_heap_bump")) *out = e->heap_bump;          // sizes above the model's nominee-heap choice (adaptive)
    else if (!strcmp(name, "batch_last_heap")) *out = e->last_heap;          // nominee heap entries of the last bf16 level-1 launch
    else if (!strcmp(name, "single_shadow_queries") || !strcmp(name, "single_shadow_fallbacks")) {
        // single queries the shadow route answered / the fp32 scan answered after a failed proof, as the guarded scans
        // counted them (contexts a concurrent call holds are not in the pool: read this when the engine is idle)
        const int slot = !strcmp(name, "single_shadow_queries") ? 0 : 1;
        uint64_t n = 0;
        auto add = [&](const SearchCtx *c) { if (c->h_proof_count) n += *static_cast<volatile uint32_t *>(c->h_proof_count + slot); };
        for (const SearchCtx *c : e->pool) add(c);
        for (const auto &kv : e->stream_ctx) add(kv.second);
        *out = n;
    }
    else if (!strcmp(name, "pool_allocs")) *out = e->pool_allocs;
    else if (!strcmp(name, "pool_reuses")) *out = e->pool_reuses;
    else return fail(WAX_VS_ERR_ARGUMENT, "unknown counter '%s'", name);
    return WAX_VS_OK;
}

int32_t wax_vs_debug_time_search_batch(wax_vs_engine *e, uint32_t n_queries, int64_t top_k, uint64_t seed,
                                       uint32_t warmup, uint32_t iters, float *out_ms_total,
                                       uint64_t *out_launches, uint32_t *out_unproven) {
    WAX_VS_MULTI_REFUSE(e, "wax_vs_debug_time_search_batch");
    if (!e || !out_ms_total) return fail(WAX_VS_ERR_NULL, "NULL argument");
    if (n_queries == 0) n_queries = 1;
    std::shared_lock<std::shared_mutex> r(e->rw);
    DeviceGuard g(e->device);
    const uint32_t k_eff = static_cast<uint32_t>(std::min<uint64_t>(clamp_topk(top_k), std::max<uint64_t>(e->n_rows, 1)));
    if (!batch_tensor_eligible(e, n_queries, k_eff))
        return fail(WAX_VS_ERR_UNSUPPORTED, "batch of %u queries, k=%u, dims=%u is not eligible for the tensor path", n_queries, k_eff, e->dims);
    CtxLease lease(e);
    int32_t rc = lease.acquire();
    if (rc) return rc;
    SearchCtx *c = lease.c;
    const size_t qfloats = static_cast<size_t>(n_queries) * e->dims;
    if ((rc = c->d_queries.ensure(qfloats, "query buffer"))) return rc;
    if ((rc = c->d_out.ensure(static_cast<size_t>(n_queries) * k_eff, "result buffer"))) return rc;
    if ((rc = c->d_ok.ensure(static_cast<size_t>(n_queries), "proof flags"))) return rc;
    if ((rc = c->h_ok.ensure(static_cast<size_t>(n_queries), "proof flag staging"))) return rc;
    synth_fill_kernel<<<(n_queries + 255) / 256, 256, 0, c->stream>>>(c->d_queries, n_queries, e->dims, seed, 0, 1);
    CUDA_TRY(cudaGetLastError());
    if ((rc = ensure_norms(e, c->stream))) return rc;   // cached per corpus version: outside the timed region
    if (batch_bf16_wanted(e) && (rc = ensure_shadow(e, c->stream))) return rc;   // likewise
    uint64_t launches = 0;
    for (uint32_t it = 0; it < warmup + iters; ++it) {
        if (it == warmup) { launches = 0; CUDA_TRY(cudaEventRecord(c->ev0, c->stream)); }
        uint32_t used_heap = 0;
        rc = enqueue_batch_tensor(e, c, c->d_queries, n_queries, k_eff, 0, c->d_out, c->d_ok, nullptr, c->stream, &launches,
                                  true, nullptr, nullptr, RowFilter{}, &used_heap);
        if (rc) { cudaStreamSynchronize(c->stream); return rc; }
        if (used_heap) { std::lock_guard<std::mutex> pg(e->pool_mu); e->last_heap = used_heap; }
    }
    CUDA_TRY(cudaEventRecord(c->ev1, c->stream));
    CUDA_TRY(cudaMemcpyAsync(c->h_ok, c->d_ok, n_queries * sizeof(uint32_t), cudaMemcpyDeviceToHost, c->stream));
    CUDA_TRY(cudaStreamSynchronize(c->stream));
    CUDA_TRY(cudaEventElapsedTime(out_ms_total, c->ev0, c->ev1));
    if (out_launches) *out_launches = launches;
    if (out_unproven) {
        uint32_t bad = 0;
        for (uint32_t i = 0; i < n_queries; ++i) bad += c->h_ok[i] ? 0u : 1u;
        *out_unproven = bad;
    }
    return WAX_VS_OK;
}

int32_t wax_vs_debug_batch_nominations(wax_vs_engine *e, const float *queries, uint32_t n_queries, int64_t top_k,
                                       const uint32_t *allow_bits, float *out_scores, uint32_t *out_ok,
                                       uint64_t *out_heaps, uint64_t heaps_cap, uint32_t *out_shape) {
    WAX_VS_MULTI_REFUSE(e, "wax_vs_debug_batch_nominations");
    if (!e || !queries || !out_scores || !out_ok || !out_shape) return fail(WAX_VS_ERR_NULL, "NULL argument");
    std::shared_lock<std::shared_mutex> r(e->rw);
    DeviceGuard g(e->device);
    if (!g.ok) return g.error();
    const uint32_t k_eff = static_cast<uint32_t>(std::min<uint64_t>(clamp_topk(top_k), std::max<uint64_t>(e->n_rows, 1)));
    if (n_queries == 0 || e->n_rows == 0 || k_eff > 128u || e->dims % kBatchKBlock != 0 || e->dims > 8192 ||
        (e->similarity != WAX_VS_COSINE && e->similarity != WAX_VS_DOT && !(e->similarity == WAX_VS_L2 && e->tune.batch_l2)))
        return fail(WAX_VS_ERR_UNSUPPORTED, "batch of %u queries, k=%u, dims=%u has no tensor-core nomination pass",
                    n_queries, k_eff, e->dims);
    CtxLease lease(e);
    int32_t rc = lease.acquire();
    if (rc) return rc;
    SearchCtx *c = lease.c;
    const size_t qfloats = static_cast<size_t>(n_queries) * e->dims;
    const size_t n_scores = static_cast<size_t>(n_queries) * e->n_rows;
    if ((rc = c->d_queries.ensure(qfloats, "query buffer"))) return rc;
    if ((rc = c->d_out.ensure(static_cast<size_t>(n_queries) * k_eff, "result buffer"))) return rc;
    if ((rc = c->d_ok.ensure(static_cast<size_t>(n_queries), "proof flags"))) return rc;
    DevBuf<float> scores;
    if ((rc = scores.ensure(n_scores, "nomination scores"))) return rc;
    CUDA_TRY(cudaMemsetAsync(scores, 0xFF, n_scores * sizeof(float), c->stream));   // NaN payload: "never written"
    CUDA_TRY(cudaMemcpyAsync(c->d_queries, queries, qfloats * sizeof(float), cudaMemcpyHostToDevice, c->stream));
    const uint32_t *d_mask = nullptr;
    if (allow_bits) {
        const size_t words = static_cast<size_t>((e->n_rows + 31) / 32);
        if ((rc = c->d_mask.ensure(words, "row filter"))) return rc;
        CUDA_TRY(cudaMemcpyAsync(c->d_mask, allow_bits, words * sizeof(uint32_t), cudaMemcpyHostToDevice, c->stream));
        d_mask = c->d_mask;
    }
    NominationDump dump{};
    dump.d_scores = scores;
    uint64_t launches = 0;
    rc = enqueue_batch_tensor(e, c, c->d_queries, n_queries, k_eff, 0, c->d_out, c->d_ok, nullptr, c->stream, &launches,
                              true, nullptr, nullptr, RowFilter{d_mask}, nullptr, &dump);
    if (rc) { cudaStreamSynchronize(c->stream); return rc; }
    CUDA_TRY(cudaStreamSynchronize(c->stream));
    std::copy(dump.shape, dump.shape + 7, out_shape);
    CUDA_TRY(cudaMemcpy(out_scores, scores, n_scores * sizeof(float), cudaMemcpyDeviceToHost));
    CUDA_TRY(cudaMemcpy(out_ok, c->d_ok, n_queries * sizeof(uint32_t), cudaMemcpyDeviceToHost));
    const uint64_t n_heap = static_cast<uint64_t>(dump.shape[5]) * dump.shape[6] * dump.shape[4] * kBatchM;
    if (!out_heaps || heaps_cap < n_heap)
        return fail(WAX_VS_ERR_BUFFER, "the heaps need %llu entries (%llu given)", static_cast<unsigned long long>(n_heap),
                    static_cast<unsigned long long>(heaps_cap));
    CUDA_TRY(cudaMemcpy(out_heaps, c->d_heaps, n_heap * sizeof(uint64_t), cudaMemcpyDeviceToHost));
    return WAX_VS_OK;
}

// wax_vs_debug_shadow_nominations, wax_vs_debug_int8_nominations and wax_vs_debug_u4_nominations (keys_cap, out_bound: the
// 4-bit form only -- its nominees are grid x kU4CtaNominees keys, and {rho_max, rho_q, tau_excl} go to out_bound)
static int32_t debug_route_nominations(wax_vs_engine *e, const float *query, int64_t top_k, const uint32_t *allow_bits,
                                       uint64_t *out_keys, uint32_t *out_ok, wax_vs_candidate *out_result,
                                       uint32_t *out_shape, RouteForm form, uint64_t keys_cap = 0, float *out_bound = nullptr) {
    const RouteFormSpec &fs = kRouteSpec[form];
    if (!e || !query || !out_keys || !out_ok || !out_result || !out_shape || (fs.grid_rescore && !out_bound))
        return fail(WAX_VS_ERR_NULL, "NULL argument");
    std::shared_lock<std::shared_mutex> r(e->rw);
    const uint32_t k_eff = static_cast<uint32_t>(std::min<uint64_t>(clamp_topk(top_k), std::max<uint64_t>(e->n_rows, 1)));
    TmaConfig cfg{};
    // (the coded forms also where the bf16 shadow did not fit, as in the route)
    if (e->n_rows == 0 || k_eff > 32u || (e->similarity != WAX_VS_COSINE && e->similarity != WAX_VS_DOT) ||
        e->tune.batch_bf16 == 0 || e->dims % kBatchKBlockBf16 != 0 ||
        (form == kRouteBf16 && e->shadows[kRouteBf16].unavailable) || !pick_route_config(e, form, &cfg))
        return fail(WAX_VS_ERR_UNSUPPORTED, "no %s-shadow route for k=%u, dims=%u in this shape", fs.name, k_eff, e->dims);
    DeviceGuard g(e->device);
    if (!g.ok) return g.error();
    CtxLease lease(e);
    int32_t rc = lease.acquire();
    if (rc) return rc;
    SearchCtx *c = lease.c;
    if ((rc = ensure_route_shadow(e, form, c->stream, true))) return rc;
    if (!e->shadows[form].valid) return fail(WAX_VS_ERR_UNSUPPORTED, "the %s shadow does not fit in device memory", fs.name);
    if ((rc = c->d_out.ensure(k_eff, "result buffer"))) return rc;
    const uint32_t *d_mask = nullptr;
    if (allow_bits) {
        const size_t words = static_cast<size_t>((e->n_rows + 31) / 32);
        if ((rc = c->d_mask.ensure(words, "row filter"))) return rc;
        CUDA_TRY(cudaMemcpyAsync(c->d_mask, allow_bits, words * sizeof(uint32_t), cudaMemcpyHostToDevice, c->stream));
        d_mask = c->d_mask;
    }
    ScanParams p = scan_params(e, c, nullptr, k_eff, 0, c->d_out, nullptr, d_mask);
    if ((rc = place_host_query(e, c, p, query, true, c->stream))) return rc;
    uint64_t launches = 0;
    if ((rc = enqueue_shadow_nominations(e, c, p, cfg, c->stream, &launches, out_shape, form))) {
        cudaStreamSynchronize(c->stream);
        return rc;
    }
    CUDA_TRY(cudaStreamSynchronize(c->stream));
    if (fs.grid_rescore) {
        const uint64_t n_keys = static_cast<uint64_t>(out_shape[4]) * kU4CtaNominees;
        if (keys_cap < n_keys)
            return fail(WAX_VS_ERR_BUFFER, "the nominees need %llu entries (%llu given)", static_cast<unsigned long long>(n_keys),
                        static_cast<unsigned long long>(keys_cap));
        CUDA_TRY(cudaMemcpy(out_keys, c->d_heaps, n_keys * sizeof(uint64_t), cudaMemcpyDeviceToHost));
        uint32_t aux[3];
        CUDA_TRY(cudaMemcpy(aux, c->d_u4_aux, sizeof aux, cudaMemcpyDeviceToHost));
        out_bound[0] = e->shadows[form].rho_max;
        memcpy(out_bound + 1, &aux[1], sizeof(float));
        // the cut word as a score: -inf when no row was left out
        if (aux[2] == 0xFFFFFFFFu) out_bound[2] = -INFINITY;
        else { const uint32_t u = aux[2] ^ ((aux[2] & 0x80000000u) ? 0x80000000u : 0xFFFFFFFFu); float f; memcpy(&f, &u, 4); out_bound[2] = -f; }
    } else {
        CUDA_TRY(cudaMemcpy2D(out_keys, sizeof(uint64_t), c->d_heaps, kNomineeStride * sizeof(uint64_t), sizeof(uint64_t),
                              kShadowNominees, cudaMemcpyDeviceToHost));
    }
    CUDA_TRY(cudaMemcpy(out_ok, c->d_ok, sizeof(uint32_t), cudaMemcpyDeviceToHost));
    CUDA_TRY(cudaMemcpy(out_result, c->d_out, k_eff * sizeof(wax_vs_candidate), cudaMemcpyDeviceToHost));
    for (uint32_t i = 0; i < k_eff; ++i)
        if (out_result[i].valid) out_result[i].frame_id = frame_id_of(e, out_result[i].row);
    return WAX_VS_OK;
}

int32_t wax_vs_debug_shadow_nominations(wax_vs_engine *e, const float *query, int64_t top_k, const uint32_t *allow_bits,
                                        uint64_t *out_keys, uint32_t *out_ok, wax_vs_candidate *out_result,
                                        uint32_t *out_shape) {
    WAX_VS_MULTI_REFUSE(e, "wax_vs_debug_shadow_nominations");
    return debug_route_nominations(e, query, top_k, allow_bits, out_keys, out_ok, out_result, out_shape, kRouteBf16);
}

int32_t wax_vs_debug_int8_nominations(wax_vs_engine *e, const float *query, int64_t top_k, const uint32_t *allow_bits,
                                      uint64_t *out_keys, uint32_t *out_ok, wax_vs_candidate *out_result,
                                      uint32_t *out_shape) {
    WAX_VS_MULTI_REFUSE(e, "wax_vs_debug_int8_nominations");
    return debug_route_nominations(e, query, top_k, allow_bits, out_keys, out_ok, out_result, out_shape, kRouteInt8);
}

int32_t wax_vs_debug_u4_nominations(wax_vs_engine *e, const float *query, int64_t top_k, const uint32_t *allow_bits,
                                    uint64_t *out_keys, uint64_t keys_cap, uint32_t *out_ok, wax_vs_candidate *out_result,
                                    uint32_t *out_shape, float *out_bound) {
    WAX_VS_MULTI_REFUSE(e, "wax_vs_debug_u4_nominations");
    return debug_route_nominations(e, query, top_k, allow_bits, out_keys, out_ok, out_result, out_shape, kRouteU4,
                                   keys_cap, out_bound);
}

// wax_vs_debug_read_shadow, wax_vs_debug_read_int8_shadow and wax_vs_debug_read_u4_shadow: rows [first, first + n) of the
// form-f shadow, brought up to date first -- the stored codes, and for the coded forms each row's scale and rho_max.  The
// bf16 shadow is read out whenever the engine keeps one, a coded one where the route could take its form.
static int32_t debug_read_route_shadow(wax_vs_engine *e, RouteForm f, uint64_t first, uint64_t n, void *dst_codes,
                                       float *dst_scales, float *out_rho_max) {
    const RouteFormSpec &fs = kRouteSpec[f];
    std::shared_lock<std::shared_mutex> r(e->rw);
    if (first > e->n_rows || n > e->n_rows - first) return fail(WAX_VS_ERR_ARGUMENT, "row range out of bounds");
    TmaConfig cfg{};
    if (f == kRouteBf16 ? !batch_bf16_wanted(e)
                        : (e->similarity != WAX_VS_COSINE && e->similarity != WAX_VS_DOT) || !pick_route_config(e, f, &cfg))
        return fail(WAX_VS_ERR_UNSUPPORTED, "no %s shadow for dims=%u with this metric and these options", fs.name, e->dims);
    DeviceGuard g(e->device);
    if (!g.ok) return g.error();
    CtxLease lease(e);
    int32_t rc = lease.acquire();
    if (rc) return rc;
    if ((rc = ensure_route_shadow(e, f, lease.c->stream, true))) return rc;
    const wax_vs_engine::Shadow &sh = e->shadows[f];
    if (!sh.valid) return fail(WAX_VS_ERR_UNSUPPORTED, "the %s shadow does not fit in device memory", fs.name);
    const size_t words = shadow_words(e, f);
    if (n) {
        CUDA_TRY(cudaMemcpy(dst_codes, sh.codes + first * words, n * words * sizeof(uint32_t), cudaMemcpyDeviceToHost));
        if (fs.scaled) CUDA_TRY(cudaMemcpy(dst_scales, sh.scale + first, n * sizeof(float), cudaMemcpyDeviceToHost));
    }
    if (fs.scaled) *out_rho_max = sh.rho_max;
    return WAX_VS_OK;
}

int32_t wax_vs_debug_read_u4_shadow(wax_vs_engine *e, uint64_t first, uint64_t n, uint8_t *dst_codes, float *dst_half_steps,
                                    float *out_rho_max) {
    WAX_VS_MULTI_REFUSE(e, "wax_vs_debug_read_u4_shadow");
    if (!e || !dst_codes || !dst_half_steps || !out_rho_max) return fail(WAX_VS_ERR_NULL, "NULL argument");
    return debug_read_route_shadow(e, kRouteU4, first, n, dst_codes, dst_half_steps, out_rho_max);
}

int32_t wax_vs_debug_read_int8_shadow(wax_vs_engine *e, uint64_t first, uint64_t n, uint8_t *dst_codes, float *dst_scales,
                                      float *out_rho_max) {
    WAX_VS_MULTI_REFUSE(e, "wax_vs_debug_read_int8_shadow");
    if (!e || !dst_codes || !dst_scales || !out_rho_max) return fail(WAX_VS_ERR_NULL, "NULL argument");
    return debug_read_route_shadow(e, kRouteInt8, first, n, dst_codes, dst_scales, out_rho_max);
}

int32_t wax_vs_debug_read_shadow(wax_vs_engine *e, uint64_t first, uint64_t n, uint16_t *dst) {
    WAX_VS_MULTI_REFUSE(e, "wax_vs_debug_read_shadow");
    if (!e || !dst) return fail(WAX_VS_ERR_NULL, "NULL argument");
    return debug_read_route_shadow(e, kRouteBf16, first, n, dst, nullptr, nullptr);
}

int32_t wax_vs_debug_set_option(wax_vs_engine *e, const char *key, int64_t value) {
    if (e && e->multi && key) return multi_set_option(e->multi, key, value);
    if (!e || !key) return fail(WAX_VS_ERR_NULL, "NULL argument");
    std::unique_lock<std::shared_mutex> w(e->rw);
    const int v = static_cast<int>(value);
    if (!strcmp(key, "variant")) e->tune.variant = v;
    else if (!strcmp(key, "rows_per_step")) e->tune.rows_per_step = v;
    else if (!strcmp(key, "stages")) e->tune.stages = v;
    else if (!strcmp(key, "warps")) e->tune.warps = v;
    else if (!strcmp(key, "grid")) e->tune.grid = v;
    else if (!strcmp(key, "l2_hint")) e->tune.l2_hint = v;
    else if (!strcmp(key, "chunk_steps")) e->tune.chunk_steps = v;
    else if (!strcmp(key, "fused_k_max")) e->tune.fused_k_max = std::max(0, std::min(128, v));
    else if (!strcmp(key, "batch_tensor")) e->tune.batch_tensor = v;
    else if (!strcmp(key, "batch_min")) e->tune.batch_min = v;
    else if (!strcmp(key, "batch_noinsert")) e->tune.batch_noinsert = v;
    else if (!strcmp(key, "batch_heap")) e->tune.batch_heap = v;
    else if (!strcmp(key, "batch_large_k")) e->tune.batch_large_k = v;
    else if (!strcmp(key, "tma_max_dims")) e->tune.tma_max_dims = static_cast<uint32_t>(std::max(v, 0));
    else if (!strcmp(key, "batch_pair")) e->tune.batch_pair = v;
    else if (!strcmp(key, "batch_ares")) e->tune.batch_ares = v;
    else if (!strcmp(key, "batch_bf16")) { e->tune.batch_bf16 = v; e->shadows[kRouteBf16].unavailable = false; e->bf16_skip_batches = 0; }
    else if (!strcmp(key, "batch_rescore")) e->tune.batch_rescore = v;
    else if (!strcmp(key, "batch_retry")) e->tune.batch_retry = v;
    else if (!strcmp(key, "filter_cap")) e->tune.filter_cap = v;
    else if (!strcmp(key, "filter_bf16")) e->tune.filter_bf16 = v;
    else if (!strcmp(key, "batch_l2")) e->tune.batch_l2 = v;
    else if (!strcmp(key, "filter_bitset_bytes")) e->tune.filter_bitset_bytes = static_cast<uint64_t>(std::max<int64_t>(value, 0));
    else if (!strcmp(key, "rebalance_slab_bytes")) e->tune.rebalance_slab_bytes = static_cast<uint64_t>(std::max<int64_t>(value, 1));
    else if (!strcmp(key, "single_shadow")) e->tune.single_shadow = v;
    else if (!strcmp(key, "shadow_scan")) {     // also closes the skip window, including failures not yet seen
        std::lock_guard<std::mutex> pg(e->pool_mu);
        e->tune.shadow_scan = v;
        e->shadow_scan_skip = 0;
        auto seen = [](SearchCtx *c) { if (c->h_proof_count) c->seen_failed = *static_cast<volatile uint32_t *>(c->h_proof_count + 1); };
        for (SearchCtx *c : e->pool) seen(c);
        for (auto &kv : e->stream_ctx) seen(kv.second);
    }
    else if (!strcmp(key, "shadow_rows_per_step")) e->tune.route[kRouteBf16].rows_per_step = v;
    else if (!strcmp(key, "shadow_warps")) e->tune.route[kRouteBf16].warps = v;
    else if (!strcmp(key, "shadow_stages")) e->tune.route[kRouteBf16].stages = v;
    else if (!strcmp(key, "shadow_scan_min_bytes")) e->tune.route[kRouteBf16].min_bytes = static_cast<uint64_t>(std::max<int64_t>(value, 0));
    else if (!strcmp(key, "int8_scan_min_bytes")) {     // also lets an int8 shadow that did not fit be tried again
        e->tune.route[kRouteInt8].min_bytes = static_cast<uint64_t>(std::max<int64_t>(value, 0));
        e->shadows[kRouteInt8].unavailable = false;
        e->shadows[kRouteInt8].coarse = false;
    }
    else if (!strcmp(key, "u4_scan_min_bytes")) {       // also retries a 4-bit shadow that did not fit, and ends a demotion
        e->tune.route[kRouteU4].min_bytes = static_cast<uint64_t>(std::max<int64_t>(value, 0));
        e->shadows[kRouteU4].unavailable = false;
        e->shadows[kRouteU4].coarse = false;
        e->u4_demoted = 0; e->u4_demote_window = 16; e->u4_probing = false;
    }
    else if (!strcmp(key, "u4_rows_per_step")) e->tune.route[kRouteU4].rows_per_step = v;
    else if (!strcmp(key, "u4_warps")) e->tune.route[kRouteU4].warps = v;
    else if (!strcmp(key, "u4_stages")) e->tune.route[kRouteU4].stages = v;
    else if (!strcmp(key, "int8_rows_per_step")) e->tune.route[kRouteInt8].rows_per_step = v;
    else if (!strcmp(key, "int8_warps")) e->tune.route[kRouteInt8].warps = v;
    else if (!strcmp(key, "int8_stages")) e->tune.route[kRouteInt8].stages = v;
    else if (!strcmp(key, "shard_fused")) e->tune.shard_fused = v;
    else if (!strcmp(key, "tail_select")) e->tune.tail_select = v;
    else if (!strcmp(key, "inline_query")) e->tune.inline_query = v;
    else if (!strcmp(key, "host_delivery")) e->tune.host_delivery = v;
    else if (!strcmp(key, "shard_timeout_ms")) e->shard.timeout_ns = static_cast<unsigned long long>(std::max<int64_t>(value, 1)) * 1000000ull;
    else if (!strcmp(key, "time_overlap")) e->tune.time_overlap = v;
    else if (!strcmp(key, "ldg_ctas_per_sm")) e->tune.ldg_ctas_per_sm = std::max(1, v);
    else return fail(WAX_VS_ERR_ARGUMENT, "unknown option '%s'", key);
    return WAX_VS_OK;
}

}  // extern "C"
