// waxvs_terms.cuh -- term clauses of a where (wax_vs_search_batch_where_terms): Wax's metadataFilter (requiredEntries,
// requiredTags, requiredLabels; UnifiedSearch.matches(metadataFilter:meta:), UnifiedSearch.swift:1215-1239) as sets of
// 64-bit term ids, evaluated on the device from an inverted index.
//
// The index is a cache of the host term lists, built by CUB (radix sort of (term, row) pairs, stable, so each posting
// list is in ascending row order; group_heads_kernel flags the heads, a prefix sum numbers them):
//   term_keys[T]    the distinct term ids, ascending;
//   term_start[T+1] where each term's postings start (64-bit);
//   postings[P]     rows.
// A unit (a distinct (where contents, id filter) pair with required terms) never looks at the other rows of the corpus:
//   term_spans_kernel:  the posting span of each distinct required id of a call (binary search in term_keys);
//   term_filter_kernel: for each unit, the postings of its rarest term are the candidates; a lane takes one, checks the
//                       other terms by binary search in their posting spans, the time and tag clauses (AttrRow), the box
//                       (LocRow, only with one) and the unit's deny-list (binary search in its sorted rows, only with
//                       one).  One kernel, three uses: count the rows that pass, list them into the unit's slot (a
//                       narrow unit, one atomic per warp ballot), or set their bits in the unit's bitset (a wide unit).
//                       O(rarest posting) per unit.
#pragma once
#include <cstdint>

#include "waxvs_where.cuh"

namespace waxvs {

constexpr uint32_t kMaxWhereTerms = 32;        // required ids per where (wax_vs_search_batch_where_terms)
constexpr uint32_t kTermThreads = 256;

// A term's postings: postings[start, start + count); count 0 when no row holds it.
struct TermSpan {
    uint64_t start;
    uint32_t count, pad;
};

// One unit of term_filter_kernel (600 bytes, staged in shared memory): spans[0] is the rarest required term (its postings
// are the candidates), spans[1 .. n_spans) the others.
struct TermUnit {
    WherePred pred;
    LocBox box;
    uint32_t has_box, n_spans;
    uint64_t slot;              // listing: first entry of the unit's rows in rows_out; bits: the unit's bitset index
    TermSpan deny;              // the unit's deny-list: ascending rows deny_rows[deny.start, + deny.count)
    TermSpan spans[kMaxWhereTerms];
};

// Index build: heads[i] = 1 where sorted[i] starts a term (group_heads_kernel), incl = their inclusive prefix sum.
// term_start[T] = P is written by the host.
__global__ void term_index_finish_kernel(const uint64_t *__restrict__ sorted, const uint32_t *__restrict__ incl, uint32_t n,
                                         uint64_t *__restrict__ term_keys, uint64_t *__restrict__ term_start) {
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x)
        if (i == 0 || incl[i - 1] != incl[i]) {
            const uint32_t t = incl[i] - 1u;
            term_keys[t] = sorted[i];
            term_start[t] = i;
        }
}

// spans[i] = the postings of ids[i], or a span of count 0 when no row holds it.
__global__ void term_spans_kernel(const uint64_t *__restrict__ term_keys, const uint64_t *__restrict__ term_start,
                                  uint32_t n_terms, const uint64_t *__restrict__ ids, uint32_t n_ids,
                                  TermSpan *__restrict__ spans) {
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n_ids; i += gridDim.x * blockDim.x) {
        const uint64_t id = ids[i];
        uint32_t lo = 0, hi = n_terms;                 // first key >= id
        while (lo < hi) {
            const uint32_t mid = (lo + hi) >> 1;
            if (term_keys[mid] < id) lo = mid + 1u; else hi = mid;
        }
        TermSpan s{0, 0, 0};
        if (lo < n_terms && term_keys[lo] == id)
            s = TermSpan{term_start[lo], static_cast<uint32_t>(term_start[lo + 1] - term_start[lo]), 0};
        spans[i] = s;
    }
}

// Whether the ascending list p[0, n) holds row.
__device__ __forceinline__ bool posting_has(const uint32_t *__restrict__ p, uint32_t n, uint32_t row) {
    uint32_t lo = 0, hi = n;
    while (lo < hi) {
        const uint32_t mid = (lo + hi) >> 1;
        if (__ldg(p + mid) < row) lo = mid + 1u; else hi = mid;
    }
    return lo < n && __ldg(p + lo) == row;
}

// Unit blockIdx.y's rows passing every clause: counted into counts[y] (zeroed by the caller), and with rows_out listed at
// rows_out[units[y].slot + j], j < counts[y] (the order within a list is arbitrary: the gather class sorts by (distance,
// row), the bitset builder sets bits), or with bits set in bits[units[y].slot * words ..] (counts may then be nullptr).
// The rooted form (Rooted<TermUnit>) also tests the unit's root clause on the row's word in `roots`.
template <bool kRooted>
__global__ void __launch_bounds__(kTermThreads) term_filter_kernel(const uint32_t *__restrict__ postings,
                                                                   const AttrRow *__restrict__ attrs,
                                                                   const LocRow *__restrict__ locs,
                                                                   const uint32_t *__restrict__ deny_rows,
                                                                   const RootedIf<TermUnit, kRooted> *__restrict__ units,
                                                                   uint32_t *__restrict__ counts,
                                                                   uint32_t *__restrict__ rows_out,
                                                                   uint32_t *__restrict__ bits, uint32_t words,
                                                                   const uint64_t *__restrict__ roots) {
    using Unit = RootedIf<TermUnit, kRooted>;
    __shared__ Unit s;
    {
        uint64_t *dst = reinterpret_cast<uint64_t *>(&s);
        const uint64_t *src = reinterpret_cast<const uint64_t *>(units + blockIdx.y);
        for (uint32_t i = threadIdx.x; i < sizeof(Unit) / 8; i += blockDim.x) dst[i] = src[i];
    }
    __syncthreads();
    const uint32_t lane = threadIdx.x & 31u, below = (1u << lane) - 1u;
    const uint32_t *cand = postings + s.spans[0].start;
    const uint32_t n_cand = s.spans[0].count;
    for (uint32_t base = blockIdx.x * blockDim.x; base < n_cand; base += gridDim.x * blockDim.x) {   // warp-uniform
        const uint32_t i = base + threadIdx.x;
        bool pass = i < n_cand;
        uint32_t row = 0;
        if (pass) {
            row = __ldg(cand + i);
            for (uint32_t t = 1; t < s.n_spans && pass; ++t)
                pass = posting_has(postings + s.spans[t].start, s.spans[t].count, row);
            if (pass) {
                const AttrRow a = load_attr(attrs, row);
                pass = where_passes(s.pred, a.ts, a.tags);
            }
            if constexpr (kRooted)
                if (pass) pass = unit_root_passes(s, roots, row);
            if (pass && s.has_box) {
                const LocRow l = load_loc(locs, row, true);
                pass = loc_passes(s.box, l.lat, l.lon);
            }
            if (pass && s.deny.count) pass = !posting_has(deny_rows + s.deny.start, s.deny.count, row);
        }
        if (bits) {
            if (pass) atomicOr(bits + s.slot * words + (row >> 5), 1u << (row & 31u));
            continue;
        }
        const uint32_t b = __ballot_sync(0xFFFFFFFFu, pass);
        if (!b) continue;
        uint32_t at = 0;
        if (lane == 0) at = atomicAdd(counts + blockIdx.y, static_cast<uint32_t>(__popc(b)));
        at = __shfl_sync(0xFFFFFFFFu, at, 0);
        if (pass && rows_out) rows_out[s.slot + at + __popc(b & below)] = row;
    }
}

}  // namespace waxvs
