// waxvs_where_groups.cuh -- group clauses of a where (wax_vs_search_batch_where_groups,
// wax_vs_search_batch_grouped_multi_where_groups): "the row's group is one of these ids", VideoRAG's videoIDs filter
// (VideoRAGOrchestrator.swift:239-247 unions segmentIdsByVideoID over the chosen videos on every request), evaluated on
// the device from the group index of grouped search (waxvs_group.cuh).
//
// That index is an inverted index from group to rows: ids[G] the distinct group ids ascending, starts[G+1] / perm[N] each
// group's rows as a CSR span, row_group[N] each row's dense group.  A unit (a distinct (where contents, id filter) pair
// with a group clause) never looks at the other rows of the corpus:
//   where_group_spans_kernel: each distinct group id of a call -> its dense group and CSR span (binary search in ids);
//   where_group_filter_kernel: for each unit, the candidates are either the positions of its group spans (a position
//                       finds its span by binary search in the spans' prefix, perm gives the row; the term clause, if
//                       any, is checked by binary search in the posting spans) or, when the where's rarest posting list
//                       is shorter than its group union, that list's rows (the group is then checked by binary search of
//                       row_group[row] in the unit's ascending dense groups).  Then the time and tag clauses (AttrRow),
//                       the box (LocRow, only with one) and the unit's deny-list (only with one).  One kernel, three
//                       uses, as term_filter_kernel: count, list into the unit's slot, or set bits in the unit's bitset.
//                       O(rows of the unit's groups), or O(rarest posting), per unit.
#pragma once
#include <cstdint>

#include "waxvs_terms.cuh"

namespace waxvs {

constexpr uint32_t kMaxWhereGroups = 65536;    // group ids per where (wax_vs_search_batch_where_groups)

// One group of a unit: rows perm[start, start + count), dense group `dense`, and `before` = the unit's candidate
// positions in the groups before it (the exclusive prefix of the counts).
struct GroupSpan {
    uint32_t start, count, dense, before;
};

// One unit of where_group_filter_kernel (staged in shared memory).  Its groups are gspans[gspan0, + n_gspans) with a
// row each, in ascending dense order (groups no row carries are dropped); spans[0, n_spans) are its term clause's
// posting spans, spans[0] the rarest.  walk_terms: the candidates are spans[0]'s postings, otherwise the groups' rows
// (n_cand positions either way).
struct GroupUnit {
    WherePred pred;
    LocBox box;
    uint32_t has_box, n_spans;
    uint64_t slot;              // listing: first entry of the unit's rows in rows_out; bits: the unit's bitset index
    TermSpan deny;              // the unit's deny-list: ascending rows deny_rows[deny.start, + deny.count)
    uint64_t gspan0;
    uint32_t n_gspans, walk_terms;
    uint32_t n_cand, pad;
    TermSpan spans[kMaxWhereTerms];
};

// out[i] = (start, count, dense, 0) of group ids[i] in the index, count 0 when no row carries it.
__global__ void where_group_spans_kernel(const uint64_t *__restrict__ group_ids, const uint32_t *__restrict__ starts,
                                         uint32_t n_groups, const uint64_t *__restrict__ ids, uint32_t n_ids,
                                         GroupSpan *__restrict__ out) {
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n_ids; i += gridDim.x * blockDim.x) {
        const uint64_t id = ids[i];
        uint32_t lo = 0, hi = n_groups;                // first id >= the requested one
        while (lo < hi) {
            const uint32_t mid = (lo + hi) >> 1;
            if (group_ids[mid] < id) lo = mid + 1u; else hi = mid;
        }
        GroupSpan s{0, 0, 0, 0};
        if (lo < n_groups && group_ids[lo] == id) s = GroupSpan{starts[lo], starts[lo + 1] - starts[lo], lo, 0};
        out[i] = s;
    }
}

// Unit blockIdx.y's rows passing every clause: counted into counts[y] (zeroed by the caller), and with rows_out listed at
// rows_out[units[y].slot + j], j < counts[y] (in no particular order), or with bits set in bits[units[y].slot * words ..]
// (counts may then be nullptr).  The rooted form (Rooted<GroupUnit>) also tests the unit's root clause on the row's word
// in `roots`.
template <bool kRooted>
__global__ void __launch_bounds__(kTermThreads) where_group_filter_kernel(const uint32_t *__restrict__ perm,
                                                                          const uint32_t *__restrict__ row_group,
                                                                          const uint32_t *__restrict__ postings,
                                                                          const GroupSpan *__restrict__ gspans,
                                                                          const AttrRow *__restrict__ attrs,
                                                                          const LocRow *__restrict__ locs,
                                                                          const uint32_t *__restrict__ deny_rows,
                                                                          const RootedIf<GroupUnit, kRooted> *__restrict__ units,
                                                                          uint32_t *__restrict__ counts,
                                                                          uint32_t *__restrict__ rows_out,
                                                                          uint32_t *__restrict__ bits, uint32_t words,
                                                                          const uint64_t *__restrict__ roots) {
    using Unit = RootedIf<GroupUnit, kRooted>;
    __shared__ Unit s;
    {
        uint64_t *dst = reinterpret_cast<uint64_t *>(&s);
        const uint64_t *src = reinterpret_cast<const uint64_t *>(units + blockIdx.y);
        for (uint32_t i = threadIdx.x; i < sizeof(Unit) / 8; i += blockDim.x) dst[i] = src[i];
    }
    __syncthreads();
    const uint32_t lane = threadIdx.x & 31u, below = (1u << lane) - 1u;
    const GroupSpan *gs = gspans + s.gspan0;
    const uint32_t n_g = s.n_gspans, n_cand = s.n_cand;
    for (uint32_t base = blockIdx.x * blockDim.x; base < n_cand; base += gridDim.x * blockDim.x) {   // warp-uniform
        const uint32_t i = base + threadIdx.x;
        bool pass = i < n_cand;
        uint32_t row = 0;
        if (pass) {
            if (s.walk_terms) {
                row = __ldg(postings + s.spans[0].start + i);
                for (uint32_t t = 1; t < s.n_spans && pass; ++t)
                    pass = posting_has(postings + s.spans[t].start, s.spans[t].count, row);
                if (pass) {                            // the row's dense group among the unit's (ascending)
                    const uint32_t g = __ldg(row_group + row);
                    uint32_t lo = 0, hi = n_g;
                    while (lo < hi) {
                        const uint32_t mid = (lo + hi) >> 1;
                        if (__ldg(&gs[mid].dense) < g) lo = mid + 1u; else hi = mid;
                    }
                    pass = lo < n_g && __ldg(&gs[lo].dense) == g;
                }
            } else {
                uint32_t lo = 0, hi = n_g - 1u;        // the last span with before <= i
                while (lo < hi) {
                    const uint32_t mid = (lo + hi + 1u) >> 1;
                    if (__ldg(&gs[mid].before) <= i) lo = mid; else hi = mid - 1u;
                }
                row = __ldg(perm + __ldg(&gs[lo].start) + (i - __ldg(&gs[lo].before)));
                for (uint32_t t = 0; t < s.n_spans && pass; ++t)
                    pass = posting_has(postings + s.spans[t].start, s.spans[t].count, row);
            }
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
