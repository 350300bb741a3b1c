//
//  CUDAVectorEngine.swift
//
//  UNCOMPILED SOURCE: this image has no Swift toolchain (see DESIGN.md section 1). It is the literal
//  binding a Wax maintainer adds next to MetalVectorEngine.swift; it was desk-checked against
//  include/wax_vs_cuda.h but has never been through swiftc.
//
//  A `VectorSearchEngine` (Sources/WaxVectorSearch/VectorSearchEngine.swift:10-18) backed by
//  libwaxvs_cuda.so. Public surface mirrors `MetalVectorEngine` (MetalVectorEngine.swift:17):
//  isAvailable, init(metric:dimensions:), load(from:metric:dimensions:), search, add, addBatch,
//  addBatchStreaming, remove, serialize, deserialize, stageForCommit.
//
#if canImport(WaxVectorSearchCUDAC)
import Foundation
import WaxCore
import WaxVectorSearchCUDAC   // module map over include/wax_vs_cuda.h, linked against libwaxvs_cuda.so

public actor CUDAVectorEngine {
    private static let maxResults = 10_000

    private let metric: VectorMetric
    public let dimensions: Int
    private nonisolated(unsafe) let handle: OpaquePointer
    private let io: BlockingIOExecutor        // calls block the thread: never run them on the cooperative pool
    private var dirty = false

    public static var isAvailable: Bool {     // MetalVectorEngine.isAvailable (:144-146)
        var n: Int32 = 0
        return wax_vs_device_count(&n) == WAX_VS_OK && n > 0
    }

    /// `devices`: the CUDA ordinals to use; empty = the current device.  Two or more make a multi-device handle: the
    /// corpus sharded by rows, shard r on devices[r], every answer equal to one engine's (an ordinal may repeat: shards
    /// then share that device, a test and debug configuration).
    public init(metric: VectorMetric, dimensions: Int, devices: [Int32] = []) throws {
        guard dimensions > 0 else { throw WaxError.invalidToc(reason: "dimensions must be > 0") }
        guard dimensions <= Constants.maxEmbeddingDimensions else {
            throw WaxError.capacityExceeded(limit: UInt64(Constants.maxEmbeddingDimensions), requested: UInt64(dimensions))
        }
        var h: OpaquePointer?
        let rc = devices.isEmpty
            ? wax_vs_create(UInt32(dimensions), metric.toVecSimilarity().rawValue, nil, 0, &h)
            : devices.withUnsafeBufferPointer {
                wax_vs_create(UInt32(dimensions), metric.toVecSimilarity().rawValue, $0.baseAddress, Int32($0.count), &h)
            }
        guard rc == WAX_VS_OK, let h else { throw Self.error(rc) }   // catchable: callers fall back to USearch (WaxSession.swift:484-497)
        self.handle = h
        self.metric = metric
        self.dimensions = dimensions
        self.io = BlockingIOExecutor(label: "com.wax.cuda", qos: .userInitiated)
    }

    deinit { wax_vs_destroy(handle) }

    /// MetalVectorEngine.load(from:metric:dimensions:) (:318-328)
    public static func load(from wax: Wax, metric: VectorMetric, dimensions: Int) async throws -> CUDAVectorEngine {
        let engine = try CUDAVectorEngine(metric: metric, dimensions: dimensions)
        if let bytes = try await wax.readCommittedVecIndexBytes() { try await engine.deserialize(bytes) }
        let pending = await wax.pendingEmbeddingMutations()
        if !pending.isEmpty {
            try await engine.addBatch(frameIds: pending.map(\.frameId), vectors: pending.map(\.vector))
        }
        return engine
    }

    public func search(vector: [Float], topK: Int) async throws -> [(frameId: UInt64, score: Float)] {
        let handle = self.handle
        let cap = min(max(topK, 1), Self.maxResults)
        return try await io.run {
            var ids = [UInt64](repeating: 0, count: cap)
            var scores = [Float](repeating: 0, count: cap)
            var n: UInt32 = 0
            let rc = vector.withUnsafeBufferPointer { q in
                wax_vs_search(handle, q.baseAddress, UInt32(vector.count), Int64(topK), &ids, &scores, UInt32(cap), &n)
            }
            guard rc == WAX_VS_OK else { throw Self.error(rc) }
            return (0..<Int(n)).map { (ids[$0], scores[$0]) }
        }
    }

    /// Batched form (no counterpart in the reference protocol): one tensor-core pass over the corpus nominates,
    /// an exact fp32 re-score decides; results are identical to calling `search` per query.
    public func searchBatch(vectors: [[Float]], topK: Int) async throws -> [[(frameId: UInt64, score: Float)]] {
        guard !vectors.isEmpty else { return [] }
        let dims = dimensions
        for v in vectors where v.count != dims {
            throw WaxError.encodingError(reason: "vector dimension mismatch: expected \(dims), got \(v.count)")
        }
        let handle = self.handle
        let cap = min(max(topK, 1), Self.maxResults)
        return try await io.run {
            var flat = [Float](); flat.reserveCapacity(vectors.count * dims)
            for v in vectors { flat.append(contentsOf: v) }
            var ids = [UInt64](repeating: 0, count: vectors.count * cap)
            var scores = [Float](repeating: 0, count: vectors.count * cap)
            var counts = [UInt32](repeating: 0, count: vectors.count)
            let rc = wax_vs_search_batch(handle, flat, UInt32(vectors.count), UInt32(dims), Int64(topK),
                                         &ids, &scores, UInt32(cap), &counts)
            guard rc == WAX_VS_OK else { throw Self.error(rc) }
            return (0..<vectors.count).map { q in (0..<Int(counts[q])).map { (ids[q * cap + $0], scores[q * cap + $0]) } }
        }
    }

    /// Frame filter pushed below the top-k (replaces the post-hoc filter + 3 x topK over-fetch of
    /// UnifiedSearch.swift:58,1241-1258): `allow == true` keeps only `frameIds`, `false` excludes them.
    public func search(vector: [Float], topK: Int, frameIds: [UInt64], allow: Bool) async throws -> [(frameId: UInt64, score: Float)] {
        let handle = self.handle
        let cap = min(max(topK, 1), Self.maxResults)
        return try await io.run {
            var ids = [UInt64](repeating: 0, count: cap)
            var scores = [Float](repeating: 0, count: cap)
            var n: UInt32 = 0
            let rc = wax_vs_search_filtered(handle, vector, UInt32(vector.count), Int64(topK), frameIds,
                                            UInt64(frameIds.count), allow ? 0 : 1, &ids, &scores, UInt32(cap), &n)
            guard rc == WAX_VS_OK else { throw Self.error(rc) }
            return (0..<Int(n)).map { (ids[$0], scores[$0]) }
        }
    }

    /// The same filter for a batch of queries in one pass over the corpus (wax_vs_search_batch_filtered).
    public func searchBatch(vectors: [[Float]], topK: Int, frameIds: [UInt64], allow: Bool) async throws -> [[(frameId: UInt64, score: Float)]] {
        guard !vectors.isEmpty else { return [] }
        let dims = dimensions
        for v in vectors where v.count != dims {
            throw WaxError.encodingError(reason: "vector dimension mismatch: expected \(dims), got \(v.count)")
        }
        let handle = self.handle
        let cap = min(max(topK, 1), Self.maxResults)
        return try await io.run {
            var flat = [Float](); flat.reserveCapacity(vectors.count * dims)
            for v in vectors { flat.append(contentsOf: v) }
            var ids = [UInt64](repeating: 0, count: vectors.count * cap)
            var scores = [Float](repeating: 0, count: vectors.count * cap)
            var counts = [UInt32](repeating: 0, count: vectors.count)
            let rc = wax_vs_search_batch_filtered(handle, flat, UInt32(vectors.count), UInt32(dims), Int64(topK), frameIds,
                                                  UInt64(frameIds.count), allow ? 0 : 1, &ids, &scores, UInt32(cap), &counts)
            guard rc == WAX_VS_OK else { throw Self.error(rc) }
            return (0..<vectors.count).map { q in (0..<Int(counts[q])).map { (ids[q * cap + $0], scores[q * cap + $0]) } }
        }
    }

    /// Assign frames to groups (wax_vs_set_groups): `frameIds[i]` -> `groupIds[i]`, e.g. a derived frame to its
    /// `parentId`; unset frames are their own group.  Groups are not part of MV2V: re-apply them after `deserialize`.
    @discardableResult
    public func setGroups(frameIds: [UInt64], groupIds: [UInt64]) async throws -> Int {
        guard frameIds.count == groupIds.count else {
            throw WaxError.encodingError(reason: "setGroups: frameIds.count != groupIds.count")
        }
        guard !frameIds.isEmpty else { return 0 }
        let handle = self.handle
        let assigned: UInt64 = try await io.run {
            var n: UInt64 = 0
            let rc = wax_vs_set_groups(handle, frameIds, groupIds, UInt64(frameIds.count), &n)
            guard rc == WAX_VS_OK else { throw Self.error(rc) }
            return n
        }
        return Int(assigned)
    }

    /// The best `perGroup` frames of each of the `topGroups` best groups, exact (wax_vs_search_grouped): what PhotoRAG
    /// (PhotoRAGOrchestrator.swift:244-308) and VideoRAG (VideoRAGOrchestrator.swift:252-440) now approximate by
    /// over-fetching frames and grouping them by `parentId ?? id`.  `frameIds` / `allow` filter as `search(...allow:)`;
    /// an empty deny-list (`allow == false`) is no filter.
    public func searchGrouped(vector: [Float], topGroups: Int, perGroup: Int = 1, frameIds: [UInt64] = [],
                              allow: Bool = false) async throws -> [(groupId: UInt64, hits: [(frameId: UInt64, score: Float)])] {
        let handle = self.handle
        let cap = max(1, min(min(max(topGroups, 1), Self.maxResults) * max(perGroup, 1), Self.maxResults))
        return try await io.run {
            var ids = [UInt64](repeating: 0, count: cap)
            var scores = [Float](repeating: 0, count: cap)
            var groups = [UInt64](repeating: 0, count: cap)
            var n: UInt32 = 0
            let rc = wax_vs_search_grouped(handle, vector, UInt32(vector.count), Int64(topGroups), UInt32(max(perGroup, 0)),
                                           frameIds, UInt64(frameIds.count), allow ? 0 : 1, &ids, &scores, &groups,
                                           UInt32(cap), &n)
            guard rc == WAX_VS_OK else { throw Self.error(rc) }
            var out: [(groupId: UInt64, hits: [(frameId: UInt64, score: Float)])] = []
            for i in 0..<Int(n) {
                if out.last?.groupId != groups[i] { out.append((groups[i], [])) }
                out[out.count - 1].hits.append((ids[i], scores[i]))
            }
            return out
        }
    }

    /// `searchGrouped` for a batch of queries under ONE filter (wax_vs_search_batch_grouped), for a server batching
    /// PhotoRAG / VideoRAG requests: one answer per query, each identical to `searchGrouped` for that query alone.
    public func searchBatchGrouped(vectors: [[Float]], topGroups: Int, perGroup: Int = 1, frameIds: [UInt64] = [],
                                   allow: Bool = false) async throws
        -> [[(groupId: UInt64, hits: [(frameId: UInt64, score: Float)])]] {
        guard !vectors.isEmpty else { return [] }
        let dims = dimensions
        for v in vectors where v.count != dims {
            throw WaxError.encodingError(reason: "vector dimension mismatch: expected \(dims), got \(v.count)")
        }
        let handle = self.handle
        let cap = max(1, min(min(max(topGroups, 1), Self.maxResults) * max(perGroup, 1), Self.maxResults))
        return try await io.run {
            var flat = [Float](); flat.reserveCapacity(vectors.count * dims)
            for v in vectors { flat.append(contentsOf: v) }
            var ids = [UInt64](repeating: 0, count: vectors.count * cap)
            var scores = [Float](repeating: 0, count: vectors.count * cap)
            var groups = [UInt64](repeating: 0, count: vectors.count * cap)
            var counts = [UInt32](repeating: 0, count: vectors.count)
            let rc = wax_vs_search_batch_grouped(handle, flat, UInt32(vectors.count), UInt32(dims), Int64(topGroups),
                                                 UInt32(max(perGroup, 0)), frameIds, UInt64(frameIds.count), allow ? 0 : 1,
                                                 &ids, &scores, &groups, UInt32(cap), &counts)
            guard rc == WAX_VS_OK else { throw Self.error(rc) }
            return (0..<vectors.count).map { q in
                var out: [(groupId: UInt64, hits: [(frameId: UInt64, score: Float)])] = []
                for i in (q * cap)..<(q * cap + Int(counts[q])) {
                    if out.last?.groupId != groups[i] { out.append((groups[i], [])) }
                    out[out.count - 1].hits.append((ids[i], scores[i]))
                }
                return out
            }
        }
    }

    /// Frame attributes (wax_vs_set_attributes): a timestamp and a tag mask per frame, evaluated by `searchBatchWhere`
    /// below the top-k in place of `UnifiedSearch.passesFrameFilter`'s time and flag clauses (INTEGRATION.md maps
    /// `FrameMeta` onto them).  `nil` leaves that column unchanged; not part of MV2V: re-apply after `deserialize`.
    @discardableResult
    public func setAttributes(frameIds: [UInt64], timestamps: [Int64]?, tags: [UInt64]?) async throws -> Int {
        guard timestamps.map({ $0.count == frameIds.count }) ?? true, tags.map({ $0.count == frameIds.count }) ?? true else {
            throw WaxError.encodingError(reason: "setAttributes: column length != frameIds.count")
        }
        guard !frameIds.isEmpty else { return 0 }
        let handle = self.handle
        let assigned: UInt64 = try await io.run {
            var n: UInt64 = 0
            let rc = wax_vs_set_attributes(handle, frameIds, timestamps, tags, UInt64(frameIds.count), &n)
            guard rc == WAX_VS_OK else { throw Self.error(rc) }
            return n
        }
        return Int(assigned)
    }

    /// A batch whose query i searches the frames passing `wheres[queryWhere[i]]` (nil: every frame), exact
    /// (wax_vs_search_batch_where).
    public func searchBatchWhere(vectors: [[Float]], topK: Int, wheres: [wax_vs_where],
                                 queryWhere: [Int?]) async throws -> [[(frameId: UInt64, score: Float)]] {
        guard !vectors.isEmpty else { return [] }
        let dims = dimensions
        for v in vectors where v.count != dims {
            throw WaxError.encodingError(reason: "vector dimension mismatch: expected \(dims), got \(v.count)")
        }
        let handle = self.handle
        let cap = min(max(topK, 1), Self.maxResults)
        return try await io.run {
            var flat = [Float](); flat.reserveCapacity(vectors.count * dims)
            for v in vectors { flat.append(contentsOf: v) }
            let offsets: [UInt64] = [0]
            let queryFilter = [UInt32](repeating: WAX_VS_NO_FILTER, count: vectors.count)
            let qw = queryWhere.map { $0.map(UInt32.init) ?? WAX_VS_NO_FILTER }
            var ids = [UInt64](repeating: 0, count: vectors.count * cap)
            var scores = [Float](repeating: 0, count: vectors.count * cap)
            var counts = [UInt32](repeating: 0, count: vectors.count)
            let rc = wax_vs_search_batch_where(handle, flat, UInt32(vectors.count), UInt32(dims), Int64(topK), nil, offsets,
                                               nil, 0, queryFilter, wheres, UInt32(wheres.count), qw, &ids, &scores,
                                               UInt32(cap), &counts)
            guard rc == WAX_VS_OK else { throw Self.error(rc) }
            return (0..<vectors.count).map { q in (0..<Int(counts[q])).map { (ids[q * cap + $0], scores[q * cap + $0]) } }
        }
    }

    /// `searchBatchGrouped` over the frames passing `where` and the optional filter (wax_vs_search_batch_grouped_where):
    /// PhotoRAG / VideoRAG's `timeRange` and superseded / deleted skips below the top-k.
    public func searchBatchGroupedWhere(vectors: [[Float]], topGroups: Int, perGroup: Int = 1, where predicate: wax_vs_where,
                                        frameIds: [UInt64] = [], allow: Bool = false) async throws
        -> [[(groupId: UInt64, hits: [(frameId: UInt64, score: Float)])]] {
        guard !vectors.isEmpty else { return [] }
        let dims = dimensions
        for v in vectors where v.count != dims {
            throw WaxError.encodingError(reason: "vector dimension mismatch: expected \(dims), got \(v.count)")
        }
        let handle = self.handle
        let cap = max(1, min(min(max(topGroups, 1), Self.maxResults) * max(perGroup, 1), Self.maxResults))
        return try await io.run {
            var flat = [Float](); flat.reserveCapacity(vectors.count * dims)
            for v in vectors { flat.append(contentsOf: v) }
            var w = predicate
            var ids = [UInt64](repeating: 0, count: vectors.count * cap)
            var scores = [Float](repeating: 0, count: vectors.count * cap)
            var groups = [UInt64](repeating: 0, count: vectors.count * cap)
            var counts = [UInt32](repeating: 0, count: vectors.count)
            let rc = wax_vs_search_batch_grouped_where(handle, flat, UInt32(vectors.count), UInt32(dims), Int64(topGroups),
                                                       UInt32(max(perGroup, 0)), frameIds, UInt64(frameIds.count),
                                                       allow ? 0 : 1, &w, &ids, &scores, &groups, UInt32(cap), &counts)
            guard rc == WAX_VS_OK else { throw Self.error(rc) }
            return (0..<vectors.count).map { q in
                var out: [(groupId: UInt64, hits: [(frameId: UInt64, score: Float)])] = []
                for i in (q * cap)..<(q * cap + Int(counts[q])) {
                    if out.last?.groupId != groups[i] { out.append((groups[i], [])) }
                    out[out.count - 1].hits.append((ids[i], scores[i]))
                }
                return out
            }
        }
    }

    /// Frame locations in degrees (wax_vs_set_locations), for the frames PhotoRAG puts into `locationBins`: the engine
    /// stores their 0.01° bins and `searchBatchWhereNear` tests PhotoRAG's location box below the top-k in place of
    /// `buildLocationAllowlist`.  A NaN pair clears a location; not part of MV2V: re-apply after `deserialize`.
    @discardableResult
    public func setLocations(frameIds: [UInt64], latitudes: [Double], longitudes: [Double]) async throws -> Int {
        guard latitudes.count == frameIds.count, longitudes.count == frameIds.count else {
            throw WaxError.encodingError(reason: "setLocations: column length != frameIds.count")
        }
        guard !frameIds.isEmpty else { return 0 }
        let handle = self.handle
        let assigned: UInt64 = try await io.run {
            var n: UInt64 = 0
            let rc = wax_vs_set_locations(handle, frameIds, latitudes, longitudes, UInt64(frameIds.count), &n)
            guard rc == WAX_VS_OK else { throw Self.error(rc) }
            return n
        }
        return Int(assigned)
    }

    /// `searchBatchWhere` with PhotoRAG's location box in each predicate (wax_vs_search_batch_where_near).
    public func searchBatchWhereNear(vectors: [[Float]], topK: Int, wheres: [wax_vs_where_near],
                                     queryWhere: [Int?]) async throws -> [[(frameId: UInt64, score: Float)]] {
        guard !vectors.isEmpty else { return [] }
        let dims = dimensions
        for v in vectors where v.count != dims {
            throw WaxError.encodingError(reason: "vector dimension mismatch: expected \(dims), got \(v.count)")
        }
        let handle = self.handle
        let cap = min(max(topK, 1), Self.maxResults)
        return try await io.run {
            var flat = [Float](); flat.reserveCapacity(vectors.count * dims)
            for v in vectors { flat.append(contentsOf: v) }
            let offsets: [UInt64] = [0]
            let queryFilter = [UInt32](repeating: WAX_VS_NO_FILTER, count: vectors.count)
            let qw = queryWhere.map { $0.map(UInt32.init) ?? WAX_VS_NO_FILTER }
            var ids = [UInt64](repeating: 0, count: vectors.count * cap)
            var scores = [Float](repeating: 0, count: vectors.count * cap)
            var counts = [UInt32](repeating: 0, count: vectors.count)
            let rc = wax_vs_search_batch_where_near(handle, flat, UInt32(vectors.count), UInt32(dims), Int64(topK), nil,
                                                    offsets, nil, 0, queryFilter, wheres, UInt32(wheres.count), qw, &ids,
                                                    &scores, UInt32(cap), &counts)
            guard rc == WAX_VS_OK else { throw Self.error(rc) }
            return (0..<vectors.count).map { q in (0..<Int(counts[q])).map { (ids[q * cap + $0], scores[q * cap + $0]) } }
        }
    }

    /// `searchBatchGroupedWhere` with a where and an id filter of each request's own
    /// (wax_vs_search_batch_grouped_multi_where): a server batching PhotoRAG / VideoRAG requests from many sessions.
    /// Query i searches the frames passing `wheres[queryWhere[i]]` AND `filters[queryFilter[i]]` (nil: none; a filter is
    /// its frame ids and whether they are an allow-list); each answer equals `searchGrouped` under the allow-list of
    /// exactly those frames.
    public func searchBatchGroupedMultiWhere(vectors: [[Float]], topGroups: Int, perGroup: Int = 1,
                                             wheres: [wax_vs_where_near], queryWhere: [Int?],
                                             filters: [(frameIds: [UInt64], allow: Bool)] = [],
                                             queryFilter: [Int?]? = nil) async throws
        -> [[(groupId: UInt64, hits: [(frameId: UInt64, score: Float)])]] {
        guard !vectors.isEmpty else { return [] }
        let dims = dimensions
        for v in vectors where v.count != dims {
            throw WaxError.encodingError(reason: "vector dimension mismatch: expected \(dims), got \(v.count)")
        }
        let perQueryFilter = queryFilter ?? [Int?](repeating: nil, count: vectors.count)
        guard queryWhere.count == vectors.count, perQueryFilter.count == vectors.count else {
            throw WaxError.encodingError(reason: "searchBatchGroupedMultiWhere: queryWhere / queryFilter.count != vectors.count")
        }
        let handle = self.handle
        let cap = max(1, min(min(max(topGroups, 1), Self.maxResults) * max(perGroup, 1), Self.maxResults))
        return try await io.run {
            var flat = [Float](); flat.reserveCapacity(vectors.count * dims)
            for v in vectors { flat.append(contentsOf: v) }
            var frameIds = [UInt64]()
            var offsets: [UInt64] = [0]
            var modes = [Int32]()
            for f in filters {
                frameIds.append(contentsOf: f.frameIds)
                offsets.append(UInt64(frameIds.count))
                modes.append(f.allow ? 0 : 1)
            }
            let qf = perQueryFilter.map { $0.map(UInt32.init) ?? WAX_VS_NO_FILTER }
            let qw = queryWhere.map { $0.map(UInt32.init) ?? WAX_VS_NO_FILTER }
            var ids = [UInt64](repeating: 0, count: vectors.count * cap)
            var scores = [Float](repeating: 0, count: vectors.count * cap)
            var groups = [UInt64](repeating: 0, count: vectors.count * cap)
            var counts = [UInt32](repeating: 0, count: vectors.count)
            let rc = wax_vs_search_batch_grouped_multi_where(handle, flat, UInt32(vectors.count), UInt32(dims),
                                                             Int64(topGroups), UInt32(max(perGroup, 0)), frameIds, offsets,
                                                             modes, UInt32(filters.count), qf, wheres, UInt32(wheres.count),
                                                             qw, &ids, &scores, &groups, UInt32(cap), &counts)
            guard rc == WAX_VS_OK else { throw Self.error(rc) }
            return (0..<vectors.count).map { q in
                var out: [(groupId: UInt64, hits: [(frameId: UInt64, score: Float)])] = []
                for i in (q * cap)..<(q * cap + Int(counts[q])) {
                    if out.last?.groupId != groups[i] { out.append((groups[i], [])) }
                    out[out.count - 1].hits.append((ids[i], scores[i]))
                }
                return out
            }
        }
    }

    /// `searchBatchGroupedMultiWhere` with the group ids each where admits
    /// (wax_vs_search_batch_grouped_multi_where_groups): VideoRAG's request -- the best segments of the best videos among
    /// `videoIDs`, inside its `timeRange` -- for many requests at once, each answer equal to `searchGrouped` under the
    /// allow-list of exactly the frames that pass.
    public func searchBatchGroupedMultiWhereGroups(vectors: [[Float]], topGroups: Int, perGroup: Int = 1,
                                                   wheres: [wax_vs_where_near], whereGroups: [[UInt64]],
                                                   queryWhere: [Int?], filters: [(frameIds: [UInt64], allow: Bool)] = [],
                                                   queryFilter: [Int?]? = nil) async throws
        -> [[(groupId: UInt64, hits: [(frameId: UInt64, score: Float)])]] {
        guard !vectors.isEmpty else { return [] }
        let dims = dimensions
        for v in vectors where v.count != dims {
            throw WaxError.encodingError(reason: "vector dimension mismatch: expected \(dims), got \(v.count)")
        }
        let perQueryFilter = queryFilter ?? [Int?](repeating: nil, count: vectors.count)
        guard queryWhere.count == vectors.count, perQueryFilter.count == vectors.count else {
            throw WaxError.encodingError(reason: "searchBatchGroupedMultiWhereGroups: queryWhere / queryFilter.count != vectors.count")
        }
        guard whereGroups.count == wheres.count else {
            throw WaxError.encodingError(reason: "searchBatchGroupedMultiWhereGroups: whereGroups.count != wheres.count")
        }
        let handle = self.handle
        let cap = max(1, min(min(max(topGroups, 1), Self.maxResults) * max(perGroup, 1), Self.maxResults))
        return try await io.run {
            var flat = [Float](); flat.reserveCapacity(vectors.count * dims)
            for v in vectors { flat.append(contentsOf: v) }
            var frameIds = [UInt64]()
            var offsets: [UInt64] = [0]
            var modes = [Int32]()
            for f in filters {
                frameIds.append(contentsOf: f.frameIds)
                offsets.append(UInt64(frameIds.count))
                modes.append(f.allow ? 0 : 1)
            }
            var groupOffsets: [UInt64] = [0]
            var groupIds = [UInt64]()
            for g in whereGroups { groupIds.append(contentsOf: g); groupOffsets.append(UInt64(groupIds.count)) }
            let qf = perQueryFilter.map { $0.map(UInt32.init) ?? WAX_VS_NO_FILTER }
            let qw = queryWhere.map { $0.map(UInt32.init) ?? WAX_VS_NO_FILTER }
            var ids = [UInt64](repeating: 0, count: vectors.count * cap)
            var scores = [Float](repeating: 0, count: vectors.count * cap)
            var groups = [UInt64](repeating: 0, count: vectors.count * cap)
            var counts = [UInt32](repeating: 0, count: vectors.count)
            let rc = wax_vs_search_batch_grouped_multi_where_groups(handle, flat, UInt32(vectors.count), UInt32(dims),
                                                                    Int64(topGroups), UInt32(max(perGroup, 0)), frameIds,
                                                                    offsets, modes, UInt32(filters.count), qf, wheres,
                                                                    UInt32(wheres.count), qw, groupOffsets, groupIds, &ids,
                                                                    &scores, &groups, UInt32(cap), &counts)
            guard rc == WAX_VS_OK else { throw Self.error(rc) }
            return (0..<vectors.count).map { q in
                var out: [(groupId: UInt64, hits: [(frameId: UInt64, score: Float)])] = []
                for i in (q * cap)..<(q * cap + Int(counts[q])) {
                    if out.last?.groupId != groups[i] { out.append((groups[i], [])) }
                    out[out.count - 1].hits.append((ids[i], scores[i]))
                }
                return out
            }
        }
    }

    /// `searchBatchGroupedMultiWhereGroups` with a root clause in each where
    /// (wax_vs_search_batch_grouped_multi_where_roots): PhotoRAG's and VideoRAG's request -- the best frames of the best
    /// photos or videos whose root is live (`whereRoots[w]` = IS_ROOT, DELETED | SUPERSEDED on the root-tag word of the
    /// frame's group) -- with no over-fetch and no filtering afterwards.
    public func searchBatchGroupedMultiWhereRoots(vectors: [[Float]], topGroups: Int, perGroup: Int = 1,
                                                  wheres: [wax_vs_where_near], whereGroups: [[UInt64]],
                                                  whereRoots: [wax_vs_root_clause], queryWhere: [Int?],
                                                  filters: [(frameIds: [UInt64], allow: Bool)] = [],
                                                  queryFilter: [Int?]? = nil) async throws
        -> [[(groupId: UInt64, hits: [(frameId: UInt64, score: Float)])]] {
        guard !vectors.isEmpty else { return [] }
        let dims = dimensions
        for v in vectors where v.count != dims {
            throw WaxError.encodingError(reason: "vector dimension mismatch: expected \(dims), got \(v.count)")
        }
        let perQueryFilter = queryFilter ?? [Int?](repeating: nil, count: vectors.count)
        guard queryWhere.count == vectors.count, perQueryFilter.count == vectors.count else {
            throw WaxError.encodingError(reason: "searchBatchGroupedMultiWhereRoots: queryWhere / queryFilter.count != vectors.count")
        }
        guard whereGroups.count == wheres.count, whereRoots.count == wheres.count else {
            throw WaxError.encodingError(reason: "searchBatchGroupedMultiWhereRoots: whereGroups / whereRoots.count != wheres.count")
        }
        let handle = self.handle
        let cap = max(1, min(min(max(topGroups, 1), Self.maxResults) * max(perGroup, 1), Self.maxResults))
        return try await io.run {
            var flat = [Float](); flat.reserveCapacity(vectors.count * dims)
            for v in vectors { flat.append(contentsOf: v) }
            var frameIds = [UInt64]()
            var offsets: [UInt64] = [0]
            var modes = [Int32]()
            for f in filters {
                frameIds.append(contentsOf: f.frameIds)
                offsets.append(UInt64(frameIds.count))
                modes.append(f.allow ? 0 : 1)
            }
            var groupOffsets: [UInt64] = [0]
            var groupIds = [UInt64]()
            for g in whereGroups { groupIds.append(contentsOf: g); groupOffsets.append(UInt64(groupIds.count)) }
            let qf = perQueryFilter.map { $0.map(UInt32.init) ?? WAX_VS_NO_FILTER }
            let qw = queryWhere.map { $0.map(UInt32.init) ?? WAX_VS_NO_FILTER }
            var ids = [UInt64](repeating: 0, count: vectors.count * cap)
            var scores = [Float](repeating: 0, count: vectors.count * cap)
            var groups = [UInt64](repeating: 0, count: vectors.count * cap)
            var counts = [UInt32](repeating: 0, count: vectors.count)
            let rc = wax_vs_search_batch_grouped_multi_where_roots(handle, flat, UInt32(vectors.count), UInt32(dims),
                                                                   Int64(topGroups), UInt32(max(perGroup, 0)), frameIds,
                                                                   offsets, modes, UInt32(filters.count), qf, wheres,
                                                                   UInt32(wheres.count), qw, groupOffsets, groupIds,
                                                                   whereRoots, &ids, &scores, &groups, UInt32(cap), &counts)
            guard rc == WAX_VS_OK else { throw Self.error(rc) }
            return (0..<vectors.count).map { q in
                var out: [(groupId: UInt64, hits: [(frameId: UInt64, score: Float)])] = []
                for i in (q * cap)..<(q * cap + Int(counts[q])) {
                    if out.last?.groupId != groups[i] { out.append((groups[i], [])) }
                    out[out.count - 1].hits.append((ids[i], scores[i]))
                }
                return out
            }
        }
    }

    /// Frame term sets (wax_vs_set_terms): each named frame's whole set is replaced, an empty list clears it.  The caller
    /// interns `("entry", key, value)`, `("tag", key, value)` and `("label", s)` exactly, so that `searchBatchWhereTerms`
    /// is `matches(metadataFilter:meta:)` below the top-k.  Not part of MV2V: re-apply after `deserialize`.
    @discardableResult
    public func setTerms(frameIds: [UInt64], termLists: [[UInt64]]) async throws -> Int {
        guard termLists.count == frameIds.count else {
            throw WaxError.encodingError(reason: "setTerms: termLists.count != frameIds.count")
        }
        guard !frameIds.isEmpty else { return 0 }
        let handle = self.handle
        let assigned: UInt64 = try await io.run {
            var offsets: [UInt64] = [0]
            var flat = [UInt64]()
            for t in termLists { flat.append(contentsOf: t); offsets.append(UInt64(flat.count)) }
            var n: UInt64 = 0
            let rc = wax_vs_set_terms(handle, frameIds, offsets, flat, UInt64(frameIds.count), &n)
            guard rc == WAX_VS_OK else { throw Self.error(rc) }
            return n
        }
        return Int(assigned)
    }

    /// `searchBatchWhereNear` with the term ids each where requires (wax_vs_search_batch_where_terms), at most 32 per
    /// where: a session-scoped `wax_recall` without a frame allow-list.
    public func searchBatchWhereTerms(vectors: [[Float]], topK: Int, wheres: [wax_vs_where_near], whereTerms: [[UInt64]],
                                      queryWhere: [Int?]) async throws -> [[(frameId: UInt64, score: Float)]] {
        guard !vectors.isEmpty else { return [] }
        guard whereTerms.count == wheres.count else {
            throw WaxError.encodingError(reason: "searchBatchWhereTerms: whereTerms.count != wheres.count")
        }
        let dims = dimensions
        for v in vectors where v.count != dims {
            throw WaxError.encodingError(reason: "vector dimension mismatch: expected \(dims), got \(v.count)")
        }
        let handle = self.handle
        let cap = min(max(topK, 1), Self.maxResults)
        return try await io.run {
            var flat = [Float](); flat.reserveCapacity(vectors.count * dims)
            for v in vectors { flat.append(contentsOf: v) }
            var termOffsets: [UInt64] = [0]
            var terms = [UInt64]()
            for t in whereTerms { terms.append(contentsOf: t); termOffsets.append(UInt64(terms.count)) }
            let offsets: [UInt64] = [0]
            let queryFilter = [UInt32](repeating: WAX_VS_NO_FILTER, count: vectors.count)
            let qw = queryWhere.map { $0.map(UInt32.init) ?? WAX_VS_NO_FILTER }
            var ids = [UInt64](repeating: 0, count: vectors.count * cap)
            var scores = [Float](repeating: 0, count: vectors.count * cap)
            var counts = [UInt32](repeating: 0, count: vectors.count)
            let rc = wax_vs_search_batch_where_terms(handle, flat, UInt32(vectors.count), UInt32(dims), Int64(topK), nil,
                                                     offsets, nil, 0, queryFilter, wheres, UInt32(wheres.count), qw,
                                                     termOffsets, terms, &ids, &scores, UInt32(cap), &counts)
            guard rc == WAX_VS_OK else { throw Self.error(rc) }
            return (0..<vectors.count).map { q in (0..<Int(counts[q])).map { (ids[q * cap + $0], scores[q * cap + $0]) } }
        }
    }

    /// `searchBatchWhereTerms` with the group ids each where admits, at most 65 536 per where
    /// (wax_vs_search_batch_where_groups): a frame passes when its group (its `setGroups` id, else its frame id) is one of
    /// them.  VideoRAG's `videoIDs` as the roots of the chosen videos, without a frame allow-list.
    public func searchBatchWhereGroups(vectors: [[Float]], topK: Int, wheres: [wax_vs_where_near], whereTerms: [[UInt64]],
                                       whereGroups: [[UInt64]], queryWhere: [Int?]) async throws
        -> [[(frameId: UInt64, score: Float)]] {
        guard !vectors.isEmpty else { return [] }
        guard whereTerms.count == wheres.count, whereGroups.count == wheres.count else {
            throw WaxError.encodingError(reason: "searchBatchWhereGroups: whereTerms / whereGroups.count != wheres.count")
        }
        let dims = dimensions
        for v in vectors where v.count != dims {
            throw WaxError.encodingError(reason: "vector dimension mismatch: expected \(dims), got \(v.count)")
        }
        let handle = self.handle
        let cap = min(max(topK, 1), Self.maxResults)
        return try await io.run {
            var flat = [Float](); flat.reserveCapacity(vectors.count * dims)
            for v in vectors { flat.append(contentsOf: v) }
            var termOffsets: [UInt64] = [0]
            var terms = [UInt64]()
            for t in whereTerms { terms.append(contentsOf: t); termOffsets.append(UInt64(terms.count)) }
            var groupOffsets: [UInt64] = [0]
            var groupIds = [UInt64]()
            for g in whereGroups { groupIds.append(contentsOf: g); groupOffsets.append(UInt64(groupIds.count)) }
            let offsets: [UInt64] = [0]
            let queryFilter = [UInt32](repeating: WAX_VS_NO_FILTER, count: vectors.count)
            let qw = queryWhere.map { $0.map(UInt32.init) ?? WAX_VS_NO_FILTER }
            var ids = [UInt64](repeating: 0, count: vectors.count * cap)
            var scores = [Float](repeating: 0, count: vectors.count * cap)
            var counts = [UInt32](repeating: 0, count: vectors.count)
            let rc = wax_vs_search_batch_where_groups(handle, flat, UInt32(vectors.count), UInt32(dims), Int64(topK), nil,
                                                      offsets, nil, 0, queryFilter, wheres, UInt32(wheres.count), qw,
                                                      termOffsets, terms, groupOffsets, groupIds, &ids, &scores,
                                                      UInt32(cap), &counts)
            guard rc == WAX_VS_OK else { throw Self.error(rc) }
            return (0..<vectors.count).map { q in (0..<Int(counts[q])).map { (ids[q * cap + $0], scores[q * cap + $0]) } }
        }
    }

    /// Groups' root-tag words (wax_vs_set_root_tags): upsert by group id, the bits (IS_ROOT, DELETED, SUPERSEDED) set
    /// from each root's `FrameMeta`; a group never given one has the word 0.  Keyed by group, so adds, removes and
    /// `setGroups` leave them alone.  Not part of MV2V: re-apply after `deserialize`.
    @discardableResult
    public func setRootTags(groupIds: [UInt64], tags: [UInt64]) async throws -> Int {
        guard groupIds.count == tags.count else {
            throw WaxError.encodingError(reason: "setRootTags: groupIds.count != tags.count")
        }
        guard !groupIds.isEmpty else { return 0 }
        let handle = self.handle
        let assigned: UInt64 = try await io.run {
            var n: UInt64 = 0
            let rc = wax_vs_set_root_tags(handle, groupIds, tags, UInt64(groupIds.count), &n)
            guard rc == WAX_VS_OK else { throw Self.error(rc) }
            return n
        }
        return Int(assigned)
    }

    /// `searchBatchWhereGroups` with a root clause in each where (wax_vs_search_batch_where_roots): a frame passes when
    /// its group's root-tag word holds every bit of `all_tags` and none of `no_tags` -- PhotoRAG's and VideoRAG's test
    /// on each hit's root, below the top-k.
    public func searchBatchWhereRoots(vectors: [[Float]], topK: Int, wheres: [wax_vs_where_near], whereTerms: [[UInt64]],
                                      whereGroups: [[UInt64]], whereRoots: [wax_vs_root_clause], queryWhere: [Int?]) async throws
        -> [[(frameId: UInt64, score: Float)]] {
        guard !vectors.isEmpty else { return [] }
        guard whereTerms.count == wheres.count, whereGroups.count == wheres.count, whereRoots.count == wheres.count else {
            throw WaxError.encodingError(reason: "searchBatchWhereRoots: whereTerms / whereGroups / whereRoots.count != wheres.count")
        }
        let dims = dimensions
        for v in vectors where v.count != dims {
            throw WaxError.encodingError(reason: "vector dimension mismatch: expected \(dims), got \(v.count)")
        }
        let handle = self.handle
        let cap = min(max(topK, 1), Self.maxResults)
        return try await io.run {
            var flat = [Float](); flat.reserveCapacity(vectors.count * dims)
            for v in vectors { flat.append(contentsOf: v) }
            var termOffsets: [UInt64] = [0]
            var terms = [UInt64]()
            for t in whereTerms { terms.append(contentsOf: t); termOffsets.append(UInt64(terms.count)) }
            var groupOffsets: [UInt64] = [0]
            var groupIds = [UInt64]()
            for g in whereGroups { groupIds.append(contentsOf: g); groupOffsets.append(UInt64(groupIds.count)) }
            let offsets: [UInt64] = [0]
            let queryFilter = [UInt32](repeating: WAX_VS_NO_FILTER, count: vectors.count)
            let qw = queryWhere.map { $0.map(UInt32.init) ?? WAX_VS_NO_FILTER }
            var ids = [UInt64](repeating: 0, count: vectors.count * cap)
            var scores = [Float](repeating: 0, count: vectors.count * cap)
            var counts = [UInt32](repeating: 0, count: vectors.count)
            let rc = wax_vs_search_batch_where_roots(handle, flat, UInt32(vectors.count), UInt32(dims), Int64(topK), nil,
                                                     offsets, nil, 0, queryFilter, wheres, UInt32(wheres.count), qw,
                                                     termOffsets, terms, groupOffsets, groupIds, whereRoots, &ids, &scores,
                                                     UInt32(cap), &counts)
            guard rc == WAX_VS_OK else { throw Self.error(rc) }
            return (0..<vectors.count).map { q in (0..<Int(counts[q])).map { (ids[q * cap + $0], scores[q * cap + $0]) } }
        }
    }

    /// `searchBatchGroupedWhere` with a location box (wax_vs_search_batch_grouped_where_near): PhotoRAG's location query
    /// and `timeRange` below the top-k, without a frame allow-list.
    public func searchBatchGroupedWhereNear(vectors: [[Float]], topGroups: Int, perGroup: Int = 1,
                                            where predicate: wax_vs_where_near, frameIds: [UInt64] = [],
                                            allow: Bool = false) async throws
        -> [[(groupId: UInt64, hits: [(frameId: UInt64, score: Float)])]] {
        guard !vectors.isEmpty else { return [] }
        let dims = dimensions
        for v in vectors where v.count != dims {
            throw WaxError.encodingError(reason: "vector dimension mismatch: expected \(dims), got \(v.count)")
        }
        let handle = self.handle
        let cap = max(1, min(min(max(topGroups, 1), Self.maxResults) * max(perGroup, 1), Self.maxResults))
        return try await io.run {
            var flat = [Float](); flat.reserveCapacity(vectors.count * dims)
            for v in vectors { flat.append(contentsOf: v) }
            var w = predicate
            var ids = [UInt64](repeating: 0, count: vectors.count * cap)
            var scores = [Float](repeating: 0, count: vectors.count * cap)
            var groups = [UInt64](repeating: 0, count: vectors.count * cap)
            var counts = [UInt32](repeating: 0, count: vectors.count)
            let rc = wax_vs_search_batch_grouped_where_near(handle, flat, UInt32(vectors.count), UInt32(dims),
                                                            Int64(topGroups), UInt32(max(perGroup, 0)), frameIds,
                                                            UInt64(frameIds.count), allow ? 0 : 1, &w, &ids, &scores,
                                                            &groups, UInt32(cap), &counts)
            guard rc == WAX_VS_OK else { throw Self.error(rc) }
            return (0..<vectors.count).map { q in
                var out: [(groupId: UInt64, hits: [(frameId: UInt64, score: Float)])] = []
                for i in (q * cap)..<(q * cap + Int(counts[q])) {
                    if out.last?.groupId != groups[i] { out.append((groups[i], [])) }
                    out[out.count - 1].hits.append((ids[i], scores[i]))
                }
                return out
            }
        }
    }

    public func add(frameId: UInt64, vector: [Float]) async throws {
        try await addBatch(frameIds: [frameId], vectors: [vector])
    }

    public func addBatch(frameIds: [UInt64], vectors: [[Float]]) async throws {
        guard !frameIds.isEmpty else { return }
        guard frameIds.count == vectors.count else {
            throw WaxError.encodingError(reason: "addBatch: frameIds.count != vectors.count")
        }
        let dims = dimensions
        for v in vectors where v.count != dims {
            throw WaxError.encodingError(reason: "vector dimension mismatch: expected \(dims), got \(v.count)")
        }
        let handle = self.handle
        try await io.run {
            var flat = [Float](); flat.reserveCapacity(vectors.count * dims)
            for v in vectors { flat.append(contentsOf: v) }       // [[Float]] -> row-major n x dims
            let rc = wax_vs_add_batch(handle, frameIds, flat, UInt64(frameIds.count), UInt32(dims))
            guard rc == WAX_VS_OK else { throw Self.error(rc) }
        }
        dirty = true
    }

    public func addBatchStreaming(frameIds: [UInt64], vectors: [[Float]], chunkSize: Int = 256) async throws {
        guard frameIds.count > chunkSize else { return try await addBatch(frameIds: frameIds, vectors: vectors) }
        for start in stride(from: 0, to: frameIds.count, by: chunkSize) {
            let end = min(start + chunkSize, frameIds.count)
            try await addBatch(frameIds: Array(frameIds[start..<end]), vectors: Array(vectors[start..<end]))
        }
    }

    public func remove(frameId: UInt64) async throws {
        let handle = self.handle
        try await io.run {
            let rc = wax_vs_remove(handle, frameId)
            guard rc == WAX_VS_OK else { throw Self.error(rc) }
        }
        dirty = true
    }

    /// Many frames in one pass: one order-preserving compaction in HBM and one id-map rebuild instead of one
    /// tail `memmove` per id (`MetalVectorEngine.swift:431-441`).  Unknown ids are ignored.
    @discardableResult
    public func removeBatch(frameIds: [UInt64]) async throws -> Int {
        guard !frameIds.isEmpty else { return 0 }
        let handle = self.handle
        let removed: UInt64 = try await io.run {
            var gone: UInt64 = 0
            let rc = frameIds.withUnsafeBufferPointer { wax_vs_remove_batch(handle, $0.baseAddress, UInt64($0.count), &gone) }
            guard rc == WAX_VS_OK else { throw Self.error(rc) }
            return gone
        }
        if removed > 0 { dirty = true }
        return Int(removed)
    }

    /// A multi-device handle: even out the shards' rows in place, each row moving with its group, attributes, location
    /// and terms.  Every answer stays the same, so the serialized bytes do too.  Returns the rows moved (0 on one engine).
    @discardableResult
    public func rebalance() async throws -> Int {
        let handle = self.handle
        let moved: UInt64 = try await io.run {
            var moved: UInt64 = 0
            let rc = wax_vs_rebalance(handle, &moved)
            guard rc == WAX_VS_OK else { throw Self.error(rc) }
            return moved
        }
        return Int(moved)
    }

    public func serialize() async throws -> Data {
        let handle = self.handle
        return try await io.run {
            var len: UInt64 = 0
            guard wax_vs_serialized_length(handle, &len) == WAX_VS_OK else { throw Self.error(WAX_VS_ERR_CUDA) }
            var data = Data(count: Int(len))
            let rc = data.withUnsafeMutableBytes { wax_vs_serialize(handle, $0.bindMemory(to: UInt8.self).baseAddress, len, &len) }
            guard rc == WAX_VS_OK else { throw Self.error(rc) }
            return data
        }
    }

    public func deserialize(_ data: Data) async throws {
        let handle = self.handle
        try await io.run {
            let rc = data.withUnsafeBytes { wax_vs_deserialize(handle, $0.bindMemory(to: UInt8.self).baseAddress, UInt64(data.count)) }
            guard rc == WAX_VS_OK else { throw Self.error(rc) }
        }
        dirty = false
    }

    public func stageForCommit(into wax: Wax) async throws {      // MetalVectorEngine.swift:818-828
        if !dirty { return }
        let blob = try await serialize()
        var count: UInt64 = 0
        _ = wax_vs_count(handle, &count)
        try await wax.stageVecIndexForNextCommit(bytes: blob, vectorCount: count, dimension: UInt32(dimensions),
                                                 similarity: metric.toVecSimilarity())
        dirty = false
    }

    /// rc -> the WaxError case the Metal engine throws for the same condition.
    private static func error(_ rc: Int32) -> WaxError {
        let reason = String(cString: wax_vs_last_error())
        switch rc {
        case WAX_VS_ERR_DIMENSION: return .encodingError(reason: reason)
        case WAX_VS_ERR_CAPACITY: return .capacityExceeded(limit: UInt64(UInt32.max), requested: 0)
        default: return .invalidToc(reason: reason)
        }
    }
}

extension CUDAVectorEngine: VectorSearchEngine {}
#endif
