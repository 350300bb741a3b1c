// waxvs_where.cuh -- frame attributes on the device: the time-range, tag and location predicates of the where searches
// (wax_vs_search_batch_where and its _near, _terms and grouped forms).
//
// Wax post-filters every vector hit on the frame's metadata (UnifiedSearch.passesFrameFilter,
// Sources/Wax/UnifiedSearch/UnifiedSearch.swift:1241-1258): a timeRange (TimeRange.contains, SearchRequest.swift:90-105:
// after inclusive, before exclusive) and the status / supersededBy / kind flags.  Here each row carries two columns, a
// timestamp and a 64-bit tag mask (16 bytes per row, AttrRow), and a predicate (WherePred) is evaluated on the device in
// one streaming pass; what it produces feeds the row-filter machinery of the filtered search unchanged:
//   where_count_kernel:   how many rows pass each predicate of a call (sizes the plan: k_i and the query classes);
//   where_bits_kernel:    ANDs a predicate into a row bitset the filter builders made (filter_bits_*_kernel), a warp per
//                         32-row word, one ballot per predicate;
//   where_compact_kernel: lists the rows passing a narrow predicate into the concatenated filter rows (the gather class).
// All three read each row's 16 bytes once per launch and test every predicate of the launch against it in registers;
// the predicates of a launch (at most kWhereChunk) sit in shared memory.
//
// Each kernel has two forms, chosen by the host per launch.  The located form (kLocated = true) adds PhotoRAG's location
// box: each row also carries its location bins (LocRow, 8 bytes, one 8-byte load per row beside the AttrRow's LDG.128),
// and each predicate a box of bins (WhereNearItem) tested in registers next to the time and tag clauses.  The plain form
// takes WhereItems, reads no location and ignores `locs`.
//
// Either form also has a rooted variant (kRooted = true) for PhotoRAG's and VideoRAG's root test: each row also carries
// its group's root-tag word (one 8-byte load per row from the root column, waxvs_roots.cuh), and each item the where's
// root clause (Rooted<Item>), tested in registers beside the others.  The unrooted forms load nothing and ignore `roots`.
// The term and group-clause kernels (waxvs_terms.cuh, waxvs_where_groups.cuh) take the same variant of their units.
#pragma once
#include <cstdint>
#include <type_traits>

namespace waxvs {

// Row attributes as the device mirror holds them (16 bytes, one LDG.128 per row).
struct alignas(16) AttrRow {
    int64_t ts;
    uint64_t tags;
};

// wax_vs_where, field for field.
struct WherePred {
    int64_t after, before;
    uint64_t all_tags, no_tags;
};

// One predicate of a launch and what it applies to: the bitset index (where_bits_kernel) or the first slot of its rows in
// the concatenated list (where_compact_kernel); unused by where_count_kernel.
struct WhereItem {
    WherePred pred;
    uint64_t slot;
};

// A row's location as PhotoRAG bins it (locationBin(from:), PhotoRAGOrchestrator.swift:868-875): floor(lat * 100) and
// floor(lon * 100), saturated to int32.  A row without a location has lat == kNoLocation, below every box.
struct alignas(8) LocRow {
    int32_t lat, lon;
};
constexpr int32_t kNoLocation = INT32_MIN;

// A box of bins (buildLocationAllowlist, PhotoRAGOrchestrator.swift:788-854): lat bin in [lat_lo, lat_hi] and lon bin in
// [lon_lo0, lon_hi0] or [lon_lo1, lon_hi1] (the second range is empty unless the box wraps the antimeridian).  "No
// location clause" is the box of every int32 pair, rows without a location included.
struct LocBox {
    int32_t lat_lo, lat_hi, lon_lo0, lon_hi0, lon_lo1, lon_hi1;
};
constexpr LocBox kNoLocBox{INT32_MIN, INT32_MAX, INT32_MIN, INT32_MAX, 1, 0};

// A WhereItem with its predicate's box (64 bytes): the item of the located form.
struct WhereNearItem {
    WherePred pred;
    uint64_t slot;
    LocBox box;
};
// A root clause (wax_vs_root_clause): the row's group's root-tag word holds every bit of all_tags and none of no_tags.
// {0, 0} is no clause.
struct RootClause {
    uint64_t all_tags, no_tags;
};

// An item or unit of the rooted forms: the unrooted one with its where's root clause after it.
template <class Base> struct Rooted : Base {
    RootClause root;
};
template <class Base, bool kRooted> using RootedIf = std::conditional_t<kRooted, Rooted<Base>, Base>;
template <bool kLocated, bool kRooted = false>
using WhereItemOf = RootedIf<std::conditional_t<kLocated, WhereNearItem, WhereItem>, kRooted>;

constexpr uint32_t kWhereChunk = 256;     // predicates per launch (shared memory: 10 KiB of items -- 16 KiB in the
                                          // located form, 4 KiB more rooted -- and 8 KiB of counts)
constexpr uint32_t kWhereThreads = 256;

// TimeRange.contains with INT64_MAX as "no upper bound" (a timestamp of INT64_MAX then passes), and the two tag tests.
__host__ __device__ __forceinline__ bool where_passes(const WherePred &w, int64_t ts, uint64_t tags) {
    return ts >= w.after && (ts < w.before || w.before == INT64_MAX) && (tags & w.all_tags) == w.all_tags &&
           (tags & w.no_tags) == 0u;
}

__host__ __device__ __forceinline__ bool loc_passes(const LocBox &b, int32_t lat, int32_t lon) {
    return lat >= b.lat_lo && lat <= b.lat_hi && ((lon >= b.lon_lo0 && lon <= b.lon_hi0) || (lon >= b.lon_lo1 && lon <= b.lon_hi1));
}

__device__ __forceinline__ AttrRow load_attr(const AttrRow *attrs, uint32_t row) {
    const longlong2 v = __ldg(reinterpret_cast<const longlong2 *>(attrs) + row);
    return AttrRow{v.x, static_cast<uint64_t>(v.y)};
}

// Row `row`'s location, or one in no box past the end; the plain where form (kLocated = false) loads nothing.
template <bool kLocated = true>
__device__ __forceinline__ LocRow load_loc(const LocRow *locs, uint32_t row, bool live) {
    if (!kLocated || !live) return LocRow{kNoLocation, 0};
    const int2 v = __ldg(reinterpret_cast<const int2 *>(locs) + row);
    return LocRow{v.x, v.y};
}

__host__ __device__ __forceinline__ bool root_passes(const RootClause &c, uint64_t root) {
    return (root & c.all_tags) == c.all_tags && (root & c.no_tags) == 0u;
}

// Row `row`'s root-tag word, or 0 past the end; the unrooted forms load nothing.
template <bool kRooted>
__device__ __forceinline__ uint64_t load_root(const uint64_t *roots, uint32_t row, bool live) {
    if (!kRooted || !live) return 0u;
    return static_cast<uint64_t>(__ldg(reinterpret_cast<const unsigned long long *>(roots) + row));
}

__device__ __forceinline__ bool item_passes(const WhereItem &it, const AttrRow &a, const LocRow &, uint64_t) {
    return where_passes(it.pred, a.ts, a.tags);
}
__device__ __forceinline__ bool item_passes(const WhereNearItem &it, const AttrRow &a, const LocRow &l, uint64_t) {
    return where_passes(it.pred, a.ts, a.tags) && loc_passes(it.box, l.lat, l.lon);
}
template <class Item>
__device__ __forceinline__ bool item_passes(const Rooted<Item> &it, const AttrRow &a, const LocRow &l, uint64_t root) {
    return item_passes(static_cast<const Item &>(it), a, l, root) && root_passes(it.root, root);
}

// A rooted term or group-clause unit's root clause on row `row` (waxvs_terms.cuh, waxvs_where_groups.cuh).
template <class Unit>
__device__ __forceinline__ bool unit_root_passes(const Rooted<Unit> &u, const uint64_t *roots, uint32_t row) {
    return root_passes(u.root, load_root<true>(roots, row, true));
}

template <class Item>
__device__ __forceinline__ void stage_items(Item *s_items, const Item *items, uint32_t n_items) {
    uint64_t *dst = reinterpret_cast<uint64_t *>(s_items);
    const uint64_t *src = reinterpret_cast<const uint64_t *>(items);
    for (uint32_t i = threadIdx.x; i < n_items * (sizeof(Item) / 8); i += blockDim.x) dst[i] = src[i];
}

// counts[i] += rows of [0, n) passing items[i], i < n_items <= kWhereChunk.  Each warp adds its ballots' popcounts to its
// own shared counters (no atomics), the CTA sums them and issues one global atomic per (CTA, predicate).
template <bool kLocated, bool kRooted>
__global__ void __launch_bounds__(kWhereThreads) where_count_kernel(const AttrRow *__restrict__ attrs,
                                                                    const LocRow *__restrict__ locs, uint32_t n,
                                                                    const WhereItemOf<kLocated, kRooted> *__restrict__ items,
                                                                    uint32_t n_items, uint32_t *__restrict__ counts,
                                                                    const uint64_t *__restrict__ roots) {
    __shared__ WhereItemOf<kLocated, kRooted> s_items[kWhereChunk];
    __shared__ uint32_t s_count[kWhereThreads / 32][kWhereChunk];
    const uint32_t lane = threadIdx.x & 31u, warp = threadIdx.x >> 5;
    stage_items(s_items, items, n_items);
    for (uint32_t i = threadIdx.x; i < (kWhereThreads / 32) * kWhereChunk; i += blockDim.x) (&s_count[0][0])[i] = 0u;
    __syncthreads();
    const uint32_t stride = gridDim.x * blockDim.x;
    for (uint32_t base = blockIdx.x * blockDim.x; base < n; base += stride) {     // warp-uniform bounds
        const uint32_t row = base + threadIdx.x;
        const bool live = row < n;
        const AttrRow a = live ? load_attr(attrs, row) : AttrRow{0, 0};
        const LocRow l = load_loc<kLocated>(locs, row, live);
        const uint64_t root = load_root<kRooted>(roots, row, live);
        for (uint32_t i = 0; i < n_items; ++i) {
            const uint32_t b = __ballot_sync(0xFFFFFFFFu, live && item_passes(s_items[i], a, l, root));
            if (lane == 0) s_count[warp][i] += __popc(b);
        }
    }
    __syncthreads();
    for (uint32_t i = threadIdx.x; i < n_items; i += blockDim.x) {
        uint32_t sum = 0;
#pragma unroll
        for (uint32_t w = 0; w < kWhereThreads / 32; ++w) sum += s_count[w][i];
        if (sum) atomicAdd(counts + i, sum);
    }
}

// bits[items[i].slot * words + word] &= the predicate's ballot over the word's 32 rows (rows >= n fail).  A warp owns a
// word, so the read-modify-write needs no atomic; a bitset is named by at most one item of a launch.
template <bool kLocated, bool kRooted>
__global__ void __launch_bounds__(kWhereThreads) where_bits_kernel(const AttrRow *__restrict__ attrs,
                                                                   const LocRow *__restrict__ locs, uint32_t n,
                                                                   uint32_t words, uint32_t *__restrict__ bits,
                                                                   const WhereItemOf<kLocated, kRooted> *__restrict__ items,
                                                                   uint32_t n_items, const uint64_t *__restrict__ roots) {
    __shared__ WhereItemOf<kLocated, kRooted> s_items[kWhereChunk];
    const uint32_t lane = threadIdx.x & 31u;
    stage_items(s_items, items, n_items);
    __syncthreads();
    const uint32_t warps = (gridDim.x * blockDim.x) >> 5;
    for (uint32_t word = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; word < words; word += warps) {
        const uint32_t row = (word << 5) + lane;
        const bool live = row < n;
        const AttrRow a = live ? load_attr(attrs, row) : AttrRow{0, 0};
        const LocRow l = load_loc<kLocated>(locs, row, live);
        const uint64_t root = load_root<kRooted>(roots, row, live);
        for (uint32_t i = 0; i < n_items; ++i) {
            const uint32_t b = __ballot_sync(0xFFFFFFFFu, live && item_passes(s_items[i], a, l, root));
            if (lane == 0 && b != 0xFFFFFFFFu) bits[s_items[i].slot * words + word] &= b;
        }
    }
}

// The rows passing items[i], written to rows_out[items[i].slot + j] for j < the predicate's count (cursor[i], zeroed by
// the caller, ends at that count).  The order within a list is arbitrary: the gather class sorts by (distance, row).
template <bool kLocated, bool kRooted>
__global__ void __launch_bounds__(kWhereThreads) where_compact_kernel(const AttrRow *__restrict__ attrs,
                                                                      const LocRow *__restrict__ locs, uint32_t n,
                                                                      const WhereItemOf<kLocated, kRooted> *__restrict__ items,
                                                                      uint32_t n_items, uint32_t *__restrict__ cursor,
                                                                      uint32_t *__restrict__ rows_out,
                                                                      const uint64_t *__restrict__ roots) {
    __shared__ WhereItemOf<kLocated, kRooted> s_items[kWhereChunk];
    const uint32_t lane = threadIdx.x & 31u;
    stage_items(s_items, items, n_items);
    __syncthreads();
    const uint32_t warps = (gridDim.x * blockDim.x) >> 5;
    const uint32_t below = (1u << lane) - 1u;
    for (uint32_t word = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; word < (n + 31u) / 32u; word += warps) {
        const uint32_t row = (word << 5) + lane;
        const bool live = row < n;
        const AttrRow a = live ? load_attr(attrs, row) : AttrRow{0, 0};
        const LocRow l = load_loc<kLocated>(locs, row, live);
        const uint64_t root = load_root<kRooted>(roots, row, live);
        for (uint32_t i = 0; i < n_items; ++i) {
            const bool pass = live && item_passes(s_items[i], a, l, root);
            const uint32_t b = __ballot_sync(0xFFFFFFFFu, pass);
            if (!b) continue;
            uint32_t at = 0;
            if (lane == 0) at = atomicAdd(cursor + i, static_cast<uint32_t>(__popc(b)));
            at = __shfl_sync(0xFFFFFFFFu, at, 0);
            if (pass) rows_out[s_items[i].slot + at + __popc(b & below)] = row;
        }
    }
}

}  // namespace waxvs
