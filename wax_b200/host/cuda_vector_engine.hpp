// cuda_vector_engine.hpp -- header-only C++17 mirror of Wax's `VectorSearchEngine` over the C-ABI
// (for C++ hosts; the Swift actor in swift/ and the Python mirror in wax_b200/engine.py bind the same entry
// points).  Member names follow the protocol (Sources/WaxVectorSearch/VectorSearchEngine.swift:10-18) and
// MetalVectorEngine's public surface (MetalVectorEngine.swift:144-146,153,330-446,682-815).
#pragma once
#include <cstdint>
#include <stdexcept>
#include <string>
#include <utility>
#include <vector>

#include "../../include/wax_vs_cuda.h"

namespace wax {

enum class VectorMetric : uint8_t { cosine = WAX_VS_COSINE, dot = WAX_VS_DOT, l2 = WAX_VS_L2 };

// WaxError cases thrown on this path.
struct WaxError : std::runtime_error { using std::runtime_error::runtime_error; };
struct EncodingError : WaxError { using WaxError::WaxError; };
struct CapacityExceeded : WaxError { using WaxError::WaxError; };
struct InvalidToc : WaxError { using WaxError::WaxError; };

class CUDAVectorEngine {
public:
    using Hit = std::pair<uint64_t, float>;  // (frameId, score)

    static bool isAvailable() {
        int32_t n = 0;
        return wax_vs_device_count(&n) == WAX_VS_OK && n > 0;
    }
    CUDAVectorEngine(VectorMetric metric, uint32_t dimensions) : metric_(metric), dimensions_(dimensions) {
        check(wax_vs_create(dimensions, static_cast<uint8_t>(metric), nullptr, 0, &h_));
    }
    // Two or more device ordinals: a multi-device handle, the corpus sharded by rows, shard r on devices[r] (an ordinal
    // may repeat: shards then share that device, a test and debug configuration).  One ordinal: that device.
    CUDAVectorEngine(VectorMetric metric, uint32_t dimensions, const std::vector<int32_t> &devices)
        : metric_(metric), dimensions_(dimensions) {
        check(wax_vs_create(dimensions, static_cast<uint8_t>(metric), devices.empty() ? nullptr : devices.data(),
                            static_cast<int32_t>(devices.size()), &h_));
    }
    ~CUDAVectorEngine() { wax_vs_destroy(h_); }
    CUDAVectorEngine(const CUDAVectorEngine &) = delete;
    CUDAVectorEngine &operator=(const CUDAVectorEngine &) = delete;

    uint32_t dimensions() const { return dimensions_; }
    uint64_t count() const { uint64_t n = 0; check(wax_vs_count(h_, &n)); return n; }

    std::vector<Hit> search(const std::vector<float> &vector, int64_t topK) const {
        const int64_t lim = topK < 1 ? 1 : (topK > WAX_VS_MAX_RESULTS ? WAX_VS_MAX_RESULTS : topK);
        std::vector<uint64_t> ids(static_cast<size_t>(lim));
        std::vector<float> scores(static_cast<size_t>(lim));
        uint32_t n = 0;
        check(wax_vs_search(h_, vector.data(), static_cast<uint32_t>(vector.size()), topK, ids.data(), scores.data(),
                            static_cast<uint32_t>(lim), &n));
        std::vector<Hit> out(n);
        for (uint32_t i = 0; i < n; ++i) out[i] = {ids[i], scores[i]};
        return out;
    }
    void add(uint64_t frameId, const std::vector<float> &vector) {
        check(wax_vs_add(h_, frameId, vector.data(), static_cast<uint32_t>(vector.size())));
    }
    void addBatch(const std::vector<uint64_t> &frameIds, const std::vector<std::vector<float>> &vectors) {
        if (frameIds.empty()) return;
        if (frameIds.size() != vectors.size()) throw EncodingError("addBatch: frameIds.count != vectors.count");
        std::vector<float> flat;
        flat.reserve(vectors.size() * dimensions_);
        for (const auto &v : vectors) {
            if (v.size() != dimensions_)
                throw EncodingError("vector dimension mismatch: expected " + std::to_string(dimensions_) + ", got " +
                                    std::to_string(v.size()));
            flat.insert(flat.end(), v.begin(), v.end());
        }
        check(wax_vs_add_batch(h_, frameIds.data(), flat.data(), frameIds.size(), dimensions_));
    }
    // addBatchStreaming (MetalVectorEngine.swift:404-421): chunks of `chunkSize` through addBatch.
    void addBatchStreaming(const std::vector<uint64_t> &frameIds, const std::vector<std::vector<float>> &vectors,
                           size_t chunkSize = 256) {
        if (frameIds.empty()) return;
        if (frameIds.size() != vectors.size()) throw EncodingError("addBatchStreaming: frameIds.count != vectors.count");
        if (chunkSize == 0) chunkSize = 256;
        for (size_t lo = 0; lo < frameIds.size(); lo += chunkSize) {
            const size_t hi = lo + chunkSize < frameIds.size() ? lo + chunkSize : frameIds.size();
            addBatch(std::vector<uint64_t>(frameIds.begin() + lo, frameIds.begin() + hi),
                     std::vector<std::vector<float>>(vectors.begin() + lo, vectors.begin() + hi));
        }
    }
    void reserve(uint64_t rows) { check(wax_vs_reserve(h_, rows)); }   // reserveIfNeeded (:857-871)
    void remove(uint64_t frameId) { check(wax_vs_remove(h_, frameId)); }
    // Many frames in one pass (one compaction in HBM, one hash rebuild); returns how many rows were deleted.
    uint64_t removeBatch(const std::vector<uint64_t> &frameIds) {
        uint64_t gone = 0;
        check(wax_vs_remove_batch(h_, frameIds.data(), frameIds.size(), &gone));
        return gone;
    }
    // A multi-device handle: even out the shards' rows in place, every answer unchanged; returns how many rows moved
    // (0 on one engine).
    uint64_t rebalance() {
        uint64_t moved = 0;
        check(wax_vs_rebalance(h_, &moved));
        return moved;
    }

    // A batch of independent queries (no reference counterpart: VectorSearchEngine.swift:13 takes one vector).  Eligible
    // batches take the tensor-core levels; the results are identical to one search() per query.
    std::vector<std::vector<Hit>> searchBatch(const std::vector<std::vector<float>> &vectors, int64_t topK) const {
        std::vector<std::vector<Hit>> out(vectors.size());
        if (vectors.empty()) return out;
        std::vector<float> flat;
        flat.reserve(vectors.size() * dimensions_);
        for (const auto &v : vectors) {
            if (v.size() != dimensions_)
                throw EncodingError("vector dimension mismatch: expected " + std::to_string(dimensions_) + ", got " +
                                    std::to_string(v.size()));
            flat.insert(flat.end(), v.begin(), v.end());
        }
        const int64_t lim = topK < 1 ? 1 : (topK > WAX_VS_MAX_RESULTS ? WAX_VS_MAX_RESULTS : topK);
        // stride = min(clamp(topK), count); a concurrent add may grow the count between count() and the search, the
        // library then answers WAX_VS_ERR_BUFFER and the buffers are re-sized (clamp(topK) always suffices)
        const uint64_t rows = count();
        uint32_t stride = static_cast<uint32_t>(rows < static_cast<uint64_t>(lim) ? (rows ? rows : 1) : lim);
        std::vector<uint64_t> ids;
        std::vector<float> scores;
        std::vector<uint32_t> ns(vectors.size());
        int32_t rc = WAX_VS_OK;
        for (int attempt = 0; attempt < 2; ++attempt) {
            ids.assign(vectors.size() * stride, 0);
            scores.assign(vectors.size() * stride, 0.0f);
            rc = wax_vs_search_batch(h_, flat.data(), static_cast<uint32_t>(vectors.size()), dimensions_, topK, ids.data(),
                                     scores.data(), stride, ns.data());
            if (rc != WAX_VS_ERR_BUFFER) break;
            stride = static_cast<uint32_t>(lim);
        }
        check(rc);
        for (size_t q = 0; q < vectors.size(); ++q) {
            out[q].resize(ns[q]);
            for (uint32_t i = 0; i < ns[q]; ++i) out[q][i] = {ids[q * stride + i], scores[q * stride + i]};
        }
        return out;
    }

    // The frame filter of UnifiedSearch (UnifiedSearch.swift:58,1195-1200,1241-1258) pushed below the top-k:
    // allow == true: only the listed frameIds may be returned; false: they are excluded (deleted / superseded frames).
    std::vector<Hit> searchFiltered(const std::vector<float> &vector, int64_t topK, const std::vector<uint64_t> &frameIds,
                                    bool allow) const {
        const int64_t lim = topK < 1 ? 1 : (topK > WAX_VS_MAX_RESULTS ? WAX_VS_MAX_RESULTS : topK);
        std::vector<uint64_t> ids(static_cast<size_t>(lim));
        std::vector<float> scores(static_cast<size_t>(lim));
        uint32_t n = 0;
        check(wax_vs_search_filtered(h_, vector.data(), static_cast<uint32_t>(vector.size()), topK, frameIds.data(),
                                     frameIds.size(), allow ? 0 : 1, ids.data(), scores.data(), static_cast<uint32_t>(lim), &n));
        std::vector<Hit> out(n);
        for (uint32_t i = 0; i < n; ++i) out[i] = {ids[i], scores[i]};
        return out;
    }

    // searchFiltered for a batch of queries under ONE filter, one pass over the corpus (wax_vs_search_batch_filtered).
    std::vector<std::vector<Hit>> searchBatchFiltered(const std::vector<std::vector<float>> &vectors, int64_t topK,
                                                      const std::vector<uint64_t> &frameIds, bool allow) const {
        std::vector<std::vector<Hit>> out(vectors.size());
        if (vectors.empty()) return out;
        std::vector<float> flat;
        flat.reserve(vectors.size() * dimensions_);
        for (const auto &v : vectors) {
            if (v.size() != dimensions_)
                throw EncodingError("vector dimension mismatch: expected " + std::to_string(dimensions_) + ", got " +
                                    std::to_string(v.size()));
            flat.insert(flat.end(), v.begin(), v.end());
        }
        const uint32_t lim = static_cast<uint32_t>(topK < 1 ? 1 : (topK > WAX_VS_MAX_RESULTS ? WAX_VS_MAX_RESULTS : topK));
        std::vector<uint64_t> ids(vectors.size() * lim);
        std::vector<float> scores(vectors.size() * lim);
        std::vector<uint32_t> ns(vectors.size());
        check(wax_vs_search_batch_filtered(h_, flat.data(), static_cast<uint32_t>(vectors.size()), dimensions_, topK,
                                           frameIds.data(), frameIds.size(), allow ? 0 : 1, ids.data(), scores.data(), lim,
                                           ns.data()));
        for (size_t q = 0; q < vectors.size(); ++q) {
            out[q].resize(ns[q]);
            for (uint32_t i = 0; i < ns[q]; ++i) out[q][i] = {ids[q * lim + i], scores[q * lim + i]};
        }
        return out;
    }

    // One frame filter per query (each request of a batch carries its own SearchRequest.frameFilter):
    // query q searches under filters[queryFilter[q]] (first = frameIds, second = allow), or unfiltered for
    // WAX_VS_NO_FILTER (wax_vs_search_batch_multi_filtered).
    std::vector<std::vector<Hit>> searchBatchMultiFiltered(const std::vector<std::vector<float>> &vectors, int64_t topK,
                                                           const std::vector<std::pair<std::vector<uint64_t>, bool>> &filters,
                                                           const std::vector<uint32_t> &queryFilter) const {
        std::vector<std::vector<Hit>> out(vectors.size());
        if (queryFilter.size() != vectors.size())
            throw EncodingError("queryFilter has " + std::to_string(queryFilter.size()) + " entries for " +
                                std::to_string(vectors.size()) + " queries");
        if (vectors.empty()) return out;
        std::vector<float> flat;
        flat.reserve(vectors.size() * dimensions_);
        for (const auto &v : vectors) {
            if (v.size() != dimensions_)
                throw EncodingError("vector dimension mismatch: expected " + std::to_string(dimensions_) + ", got " +
                                    std::to_string(v.size()));
            flat.insert(flat.end(), v.begin(), v.end());
        }
        std::vector<uint64_t> frameIds, offsets(1, 0);
        std::vector<int32_t> modes;
        for (const auto &f : filters) {
            frameIds.insert(frameIds.end(), f.first.begin(), f.first.end());
            offsets.push_back(frameIds.size());
            modes.push_back(f.second ? 0 : 1);
        }
        const uint32_t lim = static_cast<uint32_t>(topK < 1 ? 1 : (topK > WAX_VS_MAX_RESULTS ? WAX_VS_MAX_RESULTS : topK));
        std::vector<uint64_t> ids(vectors.size() * lim);
        std::vector<float> scores(vectors.size() * lim);
        std::vector<uint32_t> ns(vectors.size());
        check(wax_vs_search_batch_multi_filtered(h_, flat.data(), static_cast<uint32_t>(vectors.size()), dimensions_, topK,
                                                 frameIds.data(), offsets.data(), modes.data(),
                                                 static_cast<uint32_t>(filters.size()), queryFilter.data(), ids.data(),
                                                 scores.data(), lim, ns.data()));
        for (size_t q = 0; q < vectors.size(); ++q) {
            out[q].resize(ns[q]);
            for (uint32_t i = 0; i < ns[q]; ++i) out[q][i] = {ids[q * lim + i], scores[q * lim + i]};
        }
        return out;
    }

    // Assign frames to groups (wax_vs_set_groups): frameIds[i] -> groupIds[i] (e.g. a derived frame to its parentId);
    // a frame never assigned is its own group.  Groups are not serialized: re-apply them after deserialize().
    uint64_t setGroups(const std::vector<uint64_t> &frameIds, const std::vector<uint64_t> &groupIds) {
        if (frameIds.size() != groupIds.size()) throw EncodingError("setGroups: frameIds.count != groupIds.count");
        uint64_t assigned = 0;
        if (frameIds.empty()) return 0;
        check(wax_vs_set_groups(h_, frameIds.data(), groupIds.data(), frameIds.size(), &assigned));
        return assigned;
    }

    // The best perGroup frames of each of the topGroups best groups, exact (wax_vs_search_grouped), group-major:
    // (groupId, hits best first), groups best first.  frameIds / allow filter as searchFiltered; an empty deny-list is
    // no filter.
    using Group = std::pair<uint64_t, std::vector<Hit>>;
    std::vector<Group> searchGrouped(const std::vector<float> &vector, int64_t topGroups, uint32_t perGroup = 1,
                                     const std::vector<uint64_t> &frameIds = {}, bool allow = false) const {
        const int64_t lim = topGroups < 1 ? 1 : (topGroups > WAX_VS_MAX_RESULTS ? WAX_VS_MAX_RESULTS : topGroups);
        const int64_t want = lim * (perGroup ? perGroup : 1);
        const size_t cap = static_cast<size_t>(want > WAX_VS_MAX_RESULTS ? WAX_VS_MAX_RESULTS : want);
        std::vector<uint64_t> ids(cap), groups(cap);
        std::vector<float> scores(cap);
        uint32_t n = 0;
        check(wax_vs_search_grouped(h_, vector.data(), static_cast<uint32_t>(vector.size()), topGroups, perGroup,
                                    frameIds.data(), frameIds.size(), allow ? 0 : 1, ids.data(), scores.data(), groups.data(),
                                    static_cast<uint32_t>(cap), &n));
        std::vector<Group> out;
        for (uint32_t i = 0; i < n; ++i) {
            if (out.empty() || out.back().first != groups[i]) out.push_back({groups[i], {}});
            out.back().second.push_back({ids[i], scores[i]});
        }
        return out;
    }

    // searchGrouped for a batch of queries under ONE filter (wax_vs_search_batch_grouped): one answer per query, each
    // identical to searchGrouped for that query alone.
    std::vector<std::vector<Group>> searchBatchGrouped(const std::vector<std::vector<float>> &vectors, int64_t topGroups,
                                                       uint32_t perGroup = 1, const std::vector<uint64_t> &frameIds = {},
                                                       bool allow = false) const {
        std::vector<std::vector<Group>> out(vectors.size());
        if (vectors.empty()) return out;
        const int64_t lim = topGroups < 1 ? 1 : (topGroups > WAX_VS_MAX_RESULTS ? WAX_VS_MAX_RESULTS : topGroups);
        const int64_t want = lim * (perGroup ? perGroup : 1);
        const size_t cap = static_cast<size_t>(want > WAX_VS_MAX_RESULTS ? WAX_VS_MAX_RESULTS : want);
        std::vector<float> flat;
        flat.reserve(vectors.size() * dimensions_);
        for (const auto &v : vectors) {
            if (v.size() != dimensions_) throw EncodingError("searchBatchGrouped: vector dimension mismatch");
            flat.insert(flat.end(), v.begin(), v.end());
        }
        std::vector<uint64_t> ids(vectors.size() * cap), groups(vectors.size() * cap);
        std::vector<float> scores(vectors.size() * cap);
        std::vector<uint32_t> ns(vectors.size());
        check(wax_vs_search_batch_grouped(h_, flat.data(), static_cast<uint32_t>(vectors.size()), dimensions_, topGroups,
                                          perGroup, frameIds.data(), frameIds.size(), allow ? 0 : 1, ids.data(),
                                          scores.data(), groups.data(), static_cast<uint32_t>(cap), ns.data()));
        for (size_t q = 0; q < vectors.size(); ++q)
            for (uint32_t i = 0; i < ns[q]; ++i) {
                const size_t j = q * cap + i;
                if (out[q].empty() || out[q].back().first != groups[j]) out[q].push_back({groups[j], {}});
                out[q].back().second.push_back({ids[j], scores[j]});
            }
        return out;
    }

    // Frame attributes (wax_vs_set_attributes): timestamps / tags per frame, upsert; a null column is left unchanged.
    // Not serialized: re-apply them after deserialize().
    uint64_t setAttributes(const std::vector<uint64_t> &frameIds, const std::vector<int64_t> *timestamps,
                           const std::vector<uint64_t> *tags) {
        if ((timestamps && timestamps->size() != frameIds.size()) || (tags && tags->size() != frameIds.size()))
            throw EncodingError("setAttributes: column length != frameIds.count");
        uint64_t assigned = 0;
        if (frameIds.empty()) return 0;
        check(wax_vs_set_attributes(h_, frameIds.data(), timestamps ? timestamps->data() : nullptr,
                                    tags ? tags->data() : nullptr, frameIds.size(), &assigned));
        return assigned;
    }

    // A batch whose query i searches the frames passing wheres[queryWhere[i]] (WAX_VS_NO_FILTER: none)
    // (wax_vs_search_batch_where; no id filters here -- the C call takes them too).
    std::vector<std::vector<Hit>> searchBatchWhere(const std::vector<std::vector<float>> &vectors, int64_t topK,
                                                   const std::vector<wax_vs_where> &wheres,
                                                   const std::vector<uint32_t> &queryWhere) const {
        std::vector<std::vector<Hit>> out(vectors.size());
        if (vectors.empty()) return out;
        if (queryWhere.size() != vectors.size()) throw EncodingError("searchBatchWhere: queryWhere.count != vectors.count");
        const uint32_t lim = static_cast<uint32_t>(topK < 1 ? 1 : (topK > WAX_VS_MAX_RESULTS ? WAX_VS_MAX_RESULTS : topK));
        std::vector<float> flat;
        flat.reserve(vectors.size() * dimensions_);
        for (const auto &v : vectors) {
            if (v.size() != dimensions_) throw EncodingError("searchBatchWhere: vector dimension mismatch");
            flat.insert(flat.end(), v.begin(), v.end());
        }
        const uint64_t offsets[1] = {0};
        const std::vector<uint32_t> queryFilter(vectors.size(), WAX_VS_NO_FILTER);
        std::vector<uint64_t> ids(vectors.size() * lim);
        std::vector<float> scores(vectors.size() * lim);
        std::vector<uint32_t> ns(vectors.size());
        check(wax_vs_search_batch_where(h_, flat.data(), static_cast<uint32_t>(vectors.size()), dimensions_, topK, nullptr,
                                        offsets, nullptr, 0, queryFilter.data(), wheres.data(),
                                        static_cast<uint32_t>(wheres.size()), queryWhere.data(), ids.data(), scores.data(),
                                        lim, ns.data()));
        for (size_t q = 0; q < vectors.size(); ++q)
            for (uint32_t i = 0; i < ns[q]; ++i) out[q].push_back({ids[q * lim + i], scores[q * lim + i]});
        return out;
    }

    // searchBatchGrouped over the frames passing `where` and the optional filter (wax_vs_search_batch_grouped_where).
    std::vector<std::vector<Group>> searchBatchGroupedWhere(const std::vector<std::vector<float>> &vectors,
                                                            int64_t topGroups, uint32_t perGroup, const wax_vs_where &where,
                                                            const std::vector<uint64_t> &frameIds = {},
                                                            bool allow = false) const {
        std::vector<std::vector<Group>> out(vectors.size());
        if (vectors.empty()) return out;
        const int64_t lim = topGroups < 1 ? 1 : (topGroups > WAX_VS_MAX_RESULTS ? WAX_VS_MAX_RESULTS : topGroups);
        const int64_t want = lim * (perGroup ? perGroup : 1);
        const size_t cap = static_cast<size_t>(want > WAX_VS_MAX_RESULTS ? WAX_VS_MAX_RESULTS : want);
        std::vector<float> flat;
        flat.reserve(vectors.size() * dimensions_);
        for (const auto &v : vectors) {
            if (v.size() != dimensions_) throw EncodingError("searchBatchGroupedWhere: vector dimension mismatch");
            flat.insert(flat.end(), v.begin(), v.end());
        }
        std::vector<uint64_t> ids(vectors.size() * cap), groups(vectors.size() * cap);
        std::vector<float> scores(vectors.size() * cap);
        std::vector<uint32_t> ns(vectors.size());
        check(wax_vs_search_batch_grouped_where(h_, flat.data(), static_cast<uint32_t>(vectors.size()), dimensions_,
                                                topGroups, perGroup, frameIds.data(), frameIds.size(), allow ? 0 : 1,
                                                &where, ids.data(), scores.data(), groups.data(),
                                                static_cast<uint32_t>(cap), ns.data()));
        for (size_t q = 0; q < vectors.size(); ++q)
            for (uint32_t i = 0; i < ns[q]; ++i) {
                const size_t j = q * cap + i;
                if (out[q].empty() || out[q].back().first != groups[j]) out[q].push_back({groups[j], {}});
                out[q].back().second.push_back({ids[j], scores[j]});
            }
        return out;
    }

    // searchBatchGroupedWhere with a where and an id filter of each query's own (wax_vs_search_batch_grouped_multi_where):
    // query i searches the frames passing wheres[queryWhere[i]] AND filters[queryFilter[i]] (WAX_VS_NO_FILTER: none; a
    // filter is (frame ids, allow)).
    std::vector<std::vector<Group>> searchBatchGroupedMultiWhere(
        const std::vector<std::vector<float>> &vectors, int64_t topGroups, uint32_t perGroup,
        const std::vector<wax_vs_where_near> &wheres, const std::vector<uint32_t> &queryWhere,
        const std::vector<std::pair<std::vector<uint64_t>, bool>> &filters = {},
        const std::vector<uint32_t> &queryFilter = {}) const {
        std::vector<std::vector<Group>> out(vectors.size());
        if (vectors.empty()) return out;
        if (queryWhere.size() != vectors.size() || (!queryFilter.empty() && queryFilter.size() != vectors.size()))
            throw EncodingError("searchBatchGroupedMultiWhere: queryWhere / queryFilter.count != vectors.count");
        const int64_t lim = topGroups < 1 ? 1 : (topGroups > WAX_VS_MAX_RESULTS ? WAX_VS_MAX_RESULTS : topGroups);
        const int64_t want = lim * (perGroup ? perGroup : 1);
        const size_t cap = static_cast<size_t>(want > WAX_VS_MAX_RESULTS ? WAX_VS_MAX_RESULTS : want);
        std::vector<float> flat;
        flat.reserve(vectors.size() * dimensions_);
        for (const auto &v : vectors) {
            if (v.size() != dimensions_) throw EncodingError("searchBatchGroupedMultiWhere: vector dimension mismatch");
            flat.insert(flat.end(), v.begin(), v.end());
        }
        std::vector<uint64_t> frameIds, offsets(1, 0);
        std::vector<int32_t> modes;
        for (const auto &f : filters) {
            frameIds.insert(frameIds.end(), f.first.begin(), f.first.end());
            offsets.push_back(frameIds.size());
            modes.push_back(f.second ? 0 : 1);
        }
        const std::vector<uint32_t> noFilter(vectors.size(), WAX_VS_NO_FILTER);
        const std::vector<uint32_t> &qf = queryFilter.empty() ? noFilter : queryFilter;
        std::vector<uint64_t> ids(vectors.size() * cap), groups(vectors.size() * cap);
        std::vector<float> scores(vectors.size() * cap);
        std::vector<uint32_t> ns(vectors.size());
        check(wax_vs_search_batch_grouped_multi_where(
            h_, flat.data(), static_cast<uint32_t>(vectors.size()), dimensions_, topGroups, perGroup, frameIds.data(),
            offsets.data(), modes.data(), static_cast<uint32_t>(filters.size()), qf.data(), wheres.data(),
            static_cast<uint32_t>(wheres.size()), queryWhere.data(), ids.data(), scores.data(), groups.data(),
            static_cast<uint32_t>(cap), ns.data()));
        for (size_t q = 0; q < vectors.size(); ++q)
            for (uint32_t i = 0; i < ns[q]; ++i) {
                const size_t j = q * cap + i;
                if (out[q].empty() || out[q].back().first != groups[j]) out[q].push_back({groups[j], {}});
                out[q].back().second.push_back({ids[j], scores[j]});
            }
        return out;
    }

    // searchBatchGroupedMultiWhere with the group ids each where admits (wax_vs_search_batch_grouped_multi_where_groups):
    // VideoRAG's request, the best segments of the best videos among the chosen ones, for many queries at once.
    std::vector<std::vector<Group>> searchBatchGroupedMultiWhereGroups(
        const std::vector<std::vector<float>> &vectors, int64_t topGroups, uint32_t perGroup,
        const std::vector<wax_vs_where_near> &wheres, const std::vector<std::vector<uint64_t>> &whereGroups,
        const std::vector<uint32_t> &queryWhere, const std::vector<std::pair<std::vector<uint64_t>, bool>> &filters = {},
        const std::vector<uint32_t> &queryFilter = {}) const {
        std::vector<std::vector<Group>> out(vectors.size());
        if (vectors.empty()) return out;
        if (queryWhere.size() != vectors.size() || (!queryFilter.empty() && queryFilter.size() != vectors.size()))
            throw EncodingError("searchBatchGroupedMultiWhereGroups: queryWhere / queryFilter.count != vectors.count");
        if (whereGroups.size() != wheres.size())
            throw EncodingError("searchBatchGroupedMultiWhereGroups: whereGroups.count != wheres.count");
        const int64_t lim = topGroups < 1 ? 1 : (topGroups > WAX_VS_MAX_RESULTS ? WAX_VS_MAX_RESULTS : topGroups);
        const int64_t want = lim * (perGroup ? perGroup : 1);
        const size_t cap = static_cast<size_t>(want > WAX_VS_MAX_RESULTS ? WAX_VS_MAX_RESULTS : want);
        std::vector<float> flat;
        flat.reserve(vectors.size() * dimensions_);
        for (const auto &v : vectors) {
            if (v.size() != dimensions_) throw EncodingError("searchBatchGroupedMultiWhereGroups: vector dimension mismatch");
            flat.insert(flat.end(), v.begin(), v.end());
        }
        std::vector<uint64_t> frameIds, offsets(1, 0), groupOffsets(1, 0), groupIds;
        std::vector<int32_t> modes;
        for (const auto &f : filters) {
            frameIds.insert(frameIds.end(), f.first.begin(), f.first.end());
            offsets.push_back(frameIds.size());
            modes.push_back(f.second ? 0 : 1);
        }
        for (const auto &g : whereGroups) {
            groupIds.insert(groupIds.end(), g.begin(), g.end());
            groupOffsets.push_back(groupIds.size());
        }
        const std::vector<uint32_t> noFilter(vectors.size(), WAX_VS_NO_FILTER);
        const std::vector<uint32_t> &qf = queryFilter.empty() ? noFilter : queryFilter;
        std::vector<uint64_t> ids(vectors.size() * cap), groups(vectors.size() * cap);
        std::vector<float> scores(vectors.size() * cap);
        std::vector<uint32_t> ns(vectors.size());
        check(wax_vs_search_batch_grouped_multi_where_groups(
            h_, flat.data(), static_cast<uint32_t>(vectors.size()), dimensions_, topGroups, perGroup, frameIds.data(),
            offsets.data(), modes.data(), static_cast<uint32_t>(filters.size()), qf.data(), wheres.data(),
            static_cast<uint32_t>(wheres.size()), queryWhere.data(), groupOffsets.data(), groupIds.data(), ids.data(),
            scores.data(), groups.data(), static_cast<uint32_t>(cap), ns.data()));
        for (size_t q = 0; q < vectors.size(); ++q)
            for (uint32_t i = 0; i < ns[q]; ++i) {
                const size_t j = q * cap + i;
                if (out[q].empty() || out[q].back().first != groups[j]) out[q].push_back({groups[j], {}});
                out[q].back().second.push_back({ids[j], scores[j]});
            }
        return out;
    }

    // searchBatchGroupedMultiWhereGroups with a root clause in each where (wax_vs_search_batch_grouped_multi_where_roots):
    // PhotoRAG's and VideoRAG's request, the best frames of the best photos or videos whose root is live, with no
    // over-fetch.  whereRoots[w] = {all_tags, no_tags} on the root-tag word of the frame's group ({0, 0}: none).
    std::vector<std::vector<Group>> searchBatchGroupedMultiWhereRoots(
        const std::vector<std::vector<float>> &vectors, int64_t topGroups, uint32_t perGroup,
        const std::vector<wax_vs_where_near> &wheres, const std::vector<std::vector<uint64_t>> &whereGroups,
        const std::vector<wax_vs_root_clause> &whereRoots, const std::vector<uint32_t> &queryWhere,
        const std::vector<std::pair<std::vector<uint64_t>, bool>> &filters = {},
        const std::vector<uint32_t> &queryFilter = {}) const {
        std::vector<std::vector<Group>> out(vectors.size());
        if (vectors.empty()) return out;
        if (queryWhere.size() != vectors.size() || (!queryFilter.empty() && queryFilter.size() != vectors.size()))
            throw EncodingError("searchBatchGroupedMultiWhereRoots: queryWhere / queryFilter.count != vectors.count");
        if (whereGroups.size() != wheres.size() || whereRoots.size() != wheres.size())
            throw EncodingError("searchBatchGroupedMultiWhereRoots: whereGroups / whereRoots.count != wheres.count");
        const int64_t lim = topGroups < 1 ? 1 : (topGroups > WAX_VS_MAX_RESULTS ? WAX_VS_MAX_RESULTS : topGroups);
        const int64_t want = lim * (perGroup ? perGroup : 1);
        const size_t cap = static_cast<size_t>(want > WAX_VS_MAX_RESULTS ? WAX_VS_MAX_RESULTS : want);
        std::vector<float> flat;
        flat.reserve(vectors.size() * dimensions_);
        for (const auto &v : vectors) {
            if (v.size() != dimensions_) throw EncodingError("searchBatchGroupedMultiWhereRoots: vector dimension mismatch");
            flat.insert(flat.end(), v.begin(), v.end());
        }
        std::vector<uint64_t> frameIds, offsets(1, 0), groupOffsets(1, 0), groupIds;
        std::vector<int32_t> modes;
        for (const auto &f : filters) {
            frameIds.insert(frameIds.end(), f.first.begin(), f.first.end());
            offsets.push_back(frameIds.size());
            modes.push_back(f.second ? 0 : 1);
        }
        for (const auto &g : whereGroups) {
            groupIds.insert(groupIds.end(), g.begin(), g.end());
            groupOffsets.push_back(groupIds.size());
        }
        const std::vector<uint32_t> noFilter(vectors.size(), WAX_VS_NO_FILTER);
        const std::vector<uint32_t> &qf = queryFilter.empty() ? noFilter : queryFilter;
        std::vector<uint64_t> ids(vectors.size() * cap), groups(vectors.size() * cap);
        std::vector<float> scores(vectors.size() * cap);
        std::vector<uint32_t> ns(vectors.size());
        check(wax_vs_search_batch_grouped_multi_where_roots(
            h_, flat.data(), static_cast<uint32_t>(vectors.size()), dimensions_, topGroups, perGroup, frameIds.data(),
            offsets.data(), modes.data(), static_cast<uint32_t>(filters.size()), qf.data(), wheres.data(),
            static_cast<uint32_t>(wheres.size()), queryWhere.data(), groupOffsets.data(), groupIds.data(),
            whereRoots.data(), ids.data(), scores.data(), groups.data(), static_cast<uint32_t>(cap), ns.data()));
        for (size_t q = 0; q < vectors.size(); ++q)
            for (uint32_t i = 0; i < ns[q]; ++i) {
                const size_t j = q * cap + i;
                if (out[q].empty() || out[q].back().first != groups[j]) out[q].push_back({groups[j], {}});
                out[q].back().second.push_back({ids[j], scores[j]});
            }
        return out;
    }

    // Frame locations in degrees (wax_vs_set_locations): upsert; a NaN pair clears a frame's location.  Not serialized:
    // re-apply them after deserialize().
    uint64_t setLocations(const std::vector<uint64_t> &frameIds, const std::vector<double> &latitudes,
                          const std::vector<double> &longitudes) {
        if (latitudes.size() != frameIds.size() || longitudes.size() != frameIds.size())
            throw EncodingError("setLocations: column length != frameIds.count");
        uint64_t assigned = 0;
        if (frameIds.empty()) return 0;
        check(wax_vs_set_locations(h_, frameIds.data(), latitudes.data(), longitudes.data(), frameIds.size(), &assigned));
        return assigned;
    }

    // searchBatchWhere with PhotoRAG's location box in each predicate (wax_vs_search_batch_where_near).
    std::vector<std::vector<Hit>> searchBatchWhereNear(const std::vector<std::vector<float>> &vectors, int64_t topK,
                                                       const std::vector<wax_vs_where_near> &wheres,
                                                       const std::vector<uint32_t> &queryWhere) const {
        std::vector<std::vector<Hit>> out(vectors.size());
        if (vectors.empty()) return out;
        if (queryWhere.size() != vectors.size()) throw EncodingError("searchBatchWhereNear: queryWhere.count != vectors.count");
        const uint32_t lim = static_cast<uint32_t>(topK < 1 ? 1 : (topK > WAX_VS_MAX_RESULTS ? WAX_VS_MAX_RESULTS : topK));
        std::vector<float> flat;
        flat.reserve(vectors.size() * dimensions_);
        for (const auto &v : vectors) {
            if (v.size() != dimensions_) throw EncodingError("searchBatchWhereNear: vector dimension mismatch");
            flat.insert(flat.end(), v.begin(), v.end());
        }
        const uint64_t offsets[1] = {0};
        const std::vector<uint32_t> queryFilter(vectors.size(), WAX_VS_NO_FILTER);
        std::vector<uint64_t> ids(vectors.size() * lim);
        std::vector<float> scores(vectors.size() * lim);
        std::vector<uint32_t> ns(vectors.size());
        check(wax_vs_search_batch_where_near(h_, flat.data(), static_cast<uint32_t>(vectors.size()), dimensions_, topK,
                                             nullptr, offsets, nullptr, 0, queryFilter.data(), wheres.data(),
                                             static_cast<uint32_t>(wheres.size()), queryWhere.data(), ids.data(),
                                             scores.data(), lim, ns.data()));
        for (size_t q = 0; q < vectors.size(); ++q)
            for (uint32_t i = 0; i < ns[q]; ++i) out[q].push_back({ids[q * lim + i], scores[q * lim + i]});
        return out;
    }

    // Frame term sets (wax_vs_set_terms): replace each named frame's set; an empty list clears it.  Not serialized:
    // re-apply them after deserialize().
    uint64_t setTerms(const std::vector<uint64_t> &frameIds, const std::vector<std::vector<uint64_t>> &termLists) {
        if (termLists.size() != frameIds.size()) throw EncodingError("setTerms: termLists.count != frameIds.count");
        std::vector<uint64_t> offsets(1, 0), flat;
        for (const auto &t : termLists) {
            flat.insert(flat.end(), t.begin(), t.end());
            offsets.push_back(flat.size());
        }
        uint64_t assigned = 0;
        check(wax_vs_set_terms(h_, frameIds.data(), offsets.data(), flat.data(), frameIds.size(), &assigned));
        return assigned;
    }

    // searchBatchWhereNear with the term ids each where requires (wax_vs_search_batch_where_terms).
    std::vector<std::vector<Hit>> searchBatchWhereTerms(const std::vector<std::vector<float>> &vectors, int64_t topK,
                                                        const std::vector<wax_vs_where_near> &wheres,
                                                        const std::vector<std::vector<uint64_t>> &whereTerms,
                                                        const std::vector<uint32_t> &queryWhere) const {
        std::vector<std::vector<Hit>> out(vectors.size());
        if (vectors.empty()) return out;
        if (queryWhere.size() != vectors.size()) throw EncodingError("searchBatchWhereTerms: queryWhere.count != vectors.count");
        if (whereTerms.size() != wheres.size()) throw EncodingError("searchBatchWhereTerms: whereTerms.count != wheres.count");
        const uint32_t lim = static_cast<uint32_t>(topK < 1 ? 1 : (topK > WAX_VS_MAX_RESULTS ? WAX_VS_MAX_RESULTS : topK));
        std::vector<float> flat;
        flat.reserve(vectors.size() * dimensions_);
        for (const auto &v : vectors) {
            if (v.size() != dimensions_) throw EncodingError("searchBatchWhereTerms: vector dimension mismatch");
            flat.insert(flat.end(), v.begin(), v.end());
        }
        std::vector<uint64_t> termOffsets(1, 0), terms;
        for (const auto &t : whereTerms) {
            terms.insert(terms.end(), t.begin(), t.end());
            termOffsets.push_back(terms.size());
        }
        const uint64_t offsets[1] = {0};
        const std::vector<uint32_t> queryFilter(vectors.size(), WAX_VS_NO_FILTER);
        std::vector<uint64_t> ids(vectors.size() * lim);
        std::vector<float> scores(vectors.size() * lim);
        std::vector<uint32_t> ns(vectors.size());
        check(wax_vs_search_batch_where_terms(h_, flat.data(), static_cast<uint32_t>(vectors.size()), dimensions_, topK,
                                              nullptr, offsets, nullptr, 0, queryFilter.data(), wheres.data(),
                                              static_cast<uint32_t>(wheres.size()), queryWhere.data(), termOffsets.data(),
                                              terms.data(), ids.data(), scores.data(), lim, ns.data()));
        for (size_t q = 0; q < vectors.size(); ++q)
            for (uint32_t i = 0; i < ns[q]; ++i) out[q].push_back({ids[q * lim + i], scores[q * lim + i]});
        return out;
    }

    // searchBatchWhereTerms with the group ids each where admits, one of which must be the frame's group
    // (wax_vs_search_batch_where_groups): VideoRAG's videoIDs as the roots of the chosen videos.
    std::vector<std::vector<Hit>> searchBatchWhereGroups(const std::vector<std::vector<float>> &vectors, int64_t topK,
                                                         const std::vector<wax_vs_where_near> &wheres,
                                                         const std::vector<std::vector<uint64_t>> &whereTerms,
                                                         const std::vector<std::vector<uint64_t>> &whereGroups,
                                                         const std::vector<uint32_t> &queryWhere) const {
        std::vector<std::vector<Hit>> out(vectors.size());
        if (vectors.empty()) return out;
        if (queryWhere.size() != vectors.size()) throw EncodingError("searchBatchWhereGroups: queryWhere.count != vectors.count");
        if (whereTerms.size() != wheres.size() || whereGroups.size() != wheres.size())
            throw EncodingError("searchBatchWhereGroups: whereTerms / whereGroups.count != wheres.count");
        const uint32_t lim = static_cast<uint32_t>(topK < 1 ? 1 : (topK > WAX_VS_MAX_RESULTS ? WAX_VS_MAX_RESULTS : topK));
        std::vector<float> flat;
        flat.reserve(vectors.size() * dimensions_);
        for (const auto &v : vectors) {
            if (v.size() != dimensions_) throw EncodingError("searchBatchWhereGroups: vector dimension mismatch");
            flat.insert(flat.end(), v.begin(), v.end());
        }
        std::vector<uint64_t> termOffsets(1, 0), terms, groupOffsets(1, 0), groups;
        for (const auto &t : whereTerms) {
            terms.insert(terms.end(), t.begin(), t.end());
            termOffsets.push_back(terms.size());
        }
        for (const auto &g : whereGroups) {
            groups.insert(groups.end(), g.begin(), g.end());
            groupOffsets.push_back(groups.size());
        }
        const uint64_t offsets[1] = {0};
        const std::vector<uint32_t> queryFilter(vectors.size(), WAX_VS_NO_FILTER);
        std::vector<uint64_t> ids(vectors.size() * lim);
        std::vector<float> scores(vectors.size() * lim);
        std::vector<uint32_t> ns(vectors.size());
        check(wax_vs_search_batch_where_groups(h_, flat.data(), static_cast<uint32_t>(vectors.size()), dimensions_, topK,
                                               nullptr, offsets, nullptr, 0, queryFilter.data(), wheres.data(),
                                               static_cast<uint32_t>(wheres.size()), queryWhere.data(), termOffsets.data(),
                                               terms.data(), groupOffsets.data(), groups.data(), ids.data(), scores.data(),
                                               lim, ns.data()));
        for (size_t q = 0; q < vectors.size(); ++q)
            for (uint32_t i = 0; i < ns[q]; ++i) out[q].push_back({ids[q * lim + i], scores[q * lim + i]});
        return out;
    }

    // Groups' root-tag words (wax_vs_set_root_tags): upsert by group id, e.g. IS_ROOT, DELETED and SUPERSEDED bits from
    // each root's FrameMeta; a group never given one has the word 0.  Keyed by group, so row mutations leave them alone;
    // not serialized: re-apply them after deserialize().
    uint64_t setRootTags(const std::vector<uint64_t> &groupIds, const std::vector<uint64_t> &tags) {
        if (groupIds.size() != tags.size()) throw EncodingError("setRootTags: groupIds.count != tags.count");
        uint64_t assigned = 0;
        if (groupIds.empty()) return 0;
        check(wax_vs_set_root_tags(h_, groupIds.data(), tags.data(), groupIds.size(), &assigned));
        return assigned;
    }

    // searchBatchWhereGroups with a root clause in each where (wax_vs_search_batch_where_roots): whereRoots[w] =
    // {all_tags, no_tags} on the root-tag word of the frame's group ({0, 0}: none).
    std::vector<std::vector<Hit>> searchBatchWhereRoots(const std::vector<std::vector<float>> &vectors, int64_t topK,
                                                        const std::vector<wax_vs_where_near> &wheres,
                                                        const std::vector<std::vector<uint64_t>> &whereTerms,
                                                        const std::vector<std::vector<uint64_t>> &whereGroups,
                                                        const std::vector<wax_vs_root_clause> &whereRoots,
                                                        const std::vector<uint32_t> &queryWhere) const {
        std::vector<std::vector<Hit>> out(vectors.size());
        if (vectors.empty()) return out;
        if (queryWhere.size() != vectors.size()) throw EncodingError("searchBatchWhereRoots: queryWhere.count != vectors.count");
        if (whereTerms.size() != wheres.size() || whereGroups.size() != wheres.size() || whereRoots.size() != wheres.size())
            throw EncodingError("searchBatchWhereRoots: whereTerms / whereGroups / whereRoots.count != wheres.count");
        const uint32_t lim = static_cast<uint32_t>(topK < 1 ? 1 : (topK > WAX_VS_MAX_RESULTS ? WAX_VS_MAX_RESULTS : topK));
        std::vector<float> flat;
        flat.reserve(vectors.size() * dimensions_);
        for (const auto &v : vectors) {
            if (v.size() != dimensions_) throw EncodingError("searchBatchWhereRoots: vector dimension mismatch");
            flat.insert(flat.end(), v.begin(), v.end());
        }
        std::vector<uint64_t> termOffsets(1, 0), terms, groupOffsets(1, 0), groups;
        for (const auto &t : whereTerms) {
            terms.insert(terms.end(), t.begin(), t.end());
            termOffsets.push_back(terms.size());
        }
        for (const auto &g : whereGroups) {
            groups.insert(groups.end(), g.begin(), g.end());
            groupOffsets.push_back(groups.size());
        }
        const uint64_t offsets[1] = {0};
        const std::vector<uint32_t> queryFilter(vectors.size(), WAX_VS_NO_FILTER);
        std::vector<uint64_t> ids(vectors.size() * lim);
        std::vector<float> scores(vectors.size() * lim);
        std::vector<uint32_t> ns(vectors.size());
        check(wax_vs_search_batch_where_roots(h_, flat.data(), static_cast<uint32_t>(vectors.size()), dimensions_, topK,
                                              nullptr, offsets, nullptr, 0, queryFilter.data(), wheres.data(),
                                              static_cast<uint32_t>(wheres.size()), queryWhere.data(), termOffsets.data(),
                                              terms.data(), groupOffsets.data(), groups.data(), whereRoots.data(),
                                              ids.data(), scores.data(), lim, ns.data()));
        for (size_t q = 0; q < vectors.size(); ++q)
            for (uint32_t i = 0; i < ns[q]; ++i) out[q].push_back({ids[q * lim + i], scores[q * lim + i]});
        return out;
    }

    // searchBatchGroupedWhere with a location box (wax_vs_search_batch_grouped_where_near).
    std::vector<std::vector<Group>> searchBatchGroupedWhereNear(const std::vector<std::vector<float>> &vectors,
                                                                int64_t topGroups, uint32_t perGroup,
                                                                const wax_vs_where_near &where,
                                                                const std::vector<uint64_t> &frameIds = {},
                                                                bool allow = false) const {
        std::vector<std::vector<Group>> out(vectors.size());
        if (vectors.empty()) return out;
        const int64_t lim = topGroups < 1 ? 1 : (topGroups > WAX_VS_MAX_RESULTS ? WAX_VS_MAX_RESULTS : topGroups);
        const int64_t want = lim * (perGroup ? perGroup : 1);
        const size_t cap = static_cast<size_t>(want > WAX_VS_MAX_RESULTS ? WAX_VS_MAX_RESULTS : want);
        std::vector<float> flat;
        flat.reserve(vectors.size() * dimensions_);
        for (const auto &v : vectors) {
            if (v.size() != dimensions_) throw EncodingError("searchBatchGroupedWhereNear: vector dimension mismatch");
            flat.insert(flat.end(), v.begin(), v.end());
        }
        std::vector<uint64_t> ids(vectors.size() * cap), groups(vectors.size() * cap);
        std::vector<float> scores(vectors.size() * cap);
        std::vector<uint32_t> ns(vectors.size());
        check(wax_vs_search_batch_grouped_where_near(h_, flat.data(), static_cast<uint32_t>(vectors.size()), dimensions_,
                                                     topGroups, perGroup, frameIds.data(), frameIds.size(), allow ? 0 : 1,
                                                     &where, ids.data(), scores.data(), groups.data(),
                                                     static_cast<uint32_t>(cap), ns.data()));
        for (size_t q = 0; q < vectors.size(); ++q)
            for (uint32_t i = 0; i < ns[q]; ++i) {
                const size_t j = q * cap + i;
                if (out[q].empty() || out[q].back().first != groups[j]) out[q].push_back({groups[j], {}});
                out[q].back().second.push_back({ids[j], scores[j]});
            }
        return out;
    }

    // static load(from:metric:dimensions:) (MetalVectorEngine.swift:318-328): the committed blob (may be empty = none
    // committed yet), then the pending embedding mutations as ONE upsert batch (sequential semantics in the library).
    static CUDAVectorEngine *load(const std::vector<uint8_t> *committedBlob, const std::vector<uint64_t> &pendingIds,
                                  const std::vector<std::vector<float>> &pendingVectors, VectorMetric metric,
                                  uint32_t dimensions) {
        auto *engine = new CUDAVectorEngine(metric, dimensions);
        try {
            if (committedBlob) engine->deserialize(*committedBlob);
            engine->addBatch(pendingIds, pendingVectors);
        } catch (...) {
            delete engine;
            throw;
        }
        return engine;
    }
    std::vector<uint8_t> serialize() const {
        uint64_t len = 0;
        check(wax_vs_serialized_length(h_, &len));
        std::vector<uint8_t> blob(len);
        check(wax_vs_serialize(h_, blob.data(), len, &len));
        return blob;
    }
    void deserialize(const std::vector<uint8_t> &blob) { check(wax_vs_deserialize(h_, blob.data(), blob.size())); }
    wax_vs_engine *handle() const { return h_; }

private:
    static void check(int32_t rc) {
        if (rc == WAX_VS_OK) return;
        const std::string reason = wax_vs_last_error();
        if (rc == WAX_VS_ERR_DIMENSION) throw EncodingError(reason);
        if (rc == WAX_VS_ERR_CAPACITY) throw CapacityExceeded(reason);
        throw InvalidToc(reason);
    }
    VectorMetric metric_;
    uint32_t dimensions_;
    wax_vs_engine *h_ = nullptr;
};

}  // namespace wax
