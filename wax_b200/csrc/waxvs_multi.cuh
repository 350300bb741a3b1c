// waxvs_multi.cuh -- the multi-device handle (DESIGN.md section 4.16): wax_vs_create with n_devices >= 2 returns one
// handle over n shards, shard r an ordinary keyed engine on devices[r], behind the same C-ABI.  Every answer it serves
// equals that of one engine with the same call history: ids, order including exact ties, score bits, counts, MV2V bytes,
// error codes and reasons.
//
//   * rows: a row's key is its insertion sequence number in the whole corpus, so key order is the single engine's row
//     order (DESIGN.md section 4.15).  New ids are placed by the rule of sharded.plan_add_batch (ported below unchanged),
//     so this handle and the multi-process ShardedVectorEngine place rows alike;
//   * searches: every non-empty shard answers into a list of its own device memory (wax_vs_search_device for one query,
//     wax_vs_search_batch_device for a batch), then device 0 waits on an event of each shard's stream and ONE merge
//     launch reads the lists in place through peer memory (merge_gathered_kernel<PeerLists>), followed by one D2H copy
//     and one synchronise;
//   * rebalance: sharded.plan_rebalance (ported below unchanged) moves each donor's tail to the receivers, which merge
//     the rows by key with their side columns (absorb_rows), so every answer stays the same;
//   * threads: one persistent worker per shard lets the shards proceed concurrently through the entries that may
//     synchronise (the batched levels, the mutators).  Each concurrent caller leases its own per-shard streams and
//     buffers (MultiCtx), as CtxLease does for one engine.
//
// Included by waxvs_engine.cu after its helpers.  Each served public entry dispatches here in its first line, but the
// filtered, where and grouped ones, which first check their arguments and build their request (SearchRequest) exactly as
// one engine does, then reach here through search_where / search_grouped.  Every other entry refuses a multi-device
// handle (multi_refuse).
#pragma once
#include <condition_variable>
#include <deque>
#include <functional>
#include <memory>

// One persistent thread per shard, running the jobs posted to it in order.
struct MultiWorker {
    std::thread th;
    std::mutex mu;
    std::condition_variable cv;
    std::deque<std::function<void()>> jobs;
    bool stop = false;
    void loop() {
        for (;;) {
            std::function<void()> job;
            {
                std::unique_lock<std::mutex> g(mu);
                cv.wait(g, [&] { return stop || !jobs.empty(); });
                if (jobs.empty()) return;
                job = std::move(jobs.front());
                jobs.pop_front();
            }
            job();
        }
    }
    void post(std::function<void()> job) {
        { std::lock_guard<std::mutex> g(mu); jobs.push_back(std::move(job)); }
        cv.notify_one();
    }
};

// A caller's per-shard scratch: a stream, the queries and the candidate list on the shard's device, and an event that
// device 0's merge waits on; on device 0 also the merged lists and their pinned host copy.
struct MultiCtx {
    struct Part {
        int device = 0;
        cudaStream_t stream = nullptr;
        cudaEvent_t done = nullptr;
        DevBuf<float> d_queries;
        DevBuf<wax_vs_candidate> d_cands;
        DevBuf<wax_vs_group_candidate> d_heads;    // grouped search, round 1
    };
    std::deque<Part> part;                         // a deque: its Parts own buffers and never move
    DevBuf<wax_vs_candidate> d_merged;             // on device 0
    PinnedBuf<wax_vs_candidate> h_merged;
    DevBuf<wax_vs_group_candidate> d_chosen;       // grouped search: merge 1's top groups, on device 0 ...
    PinnedBuf<wax_vs_group_candidate> h_chosen;
    cudaEvent_t chosen = nullptr;                  // ... and the event round 2 waits on
    ~MultiCtx() {
        for (Part &p : part) {
            DeviceGuard g(p.device);
            p.d_queries.release();
            p.d_cands.release();
            p.d_heads.release();
            if (p.done) cudaEventDestroy(p.done);
            if (p.stream) cudaStreamDestroy(p.stream);
        }
        if (!part.empty()) {
            DeviceGuard g(part[0].device);
            d_merged.release();
            h_merged.release();
            d_chosen.release();
            h_chosen.release();
            if (chosen) cudaEventDestroy(chosen);
        }
    }
};

struct MultiEngine {
    std::vector<int> devices;
    std::vector<wax_vs_engine *> shards;
    std::vector<uint64_t> rows;                    // rows per shard
    uint64_t next_key = 0;                         // the first unused row key
    std::shared_mutex rw;                          // readers: searches / serialize; writer: mutators
    std::vector<std::unique_ptr<MultiWorker>> workers;
    std::mutex pool_mu;
    std::vector<MultiCtx *> pool;
    int n() const { return static_cast<int>(shards.size()); }
    uint64_t total() const { uint64_t t = 0; for (uint64_t r : rows) t += r; return t; }
};

static int32_t multi_refuse(const char *entry) {
    return fail(WAX_VS_ERR_UNSUPPORTED, "%s is not served by a multi-device handle", entry);
}
#define WAX_VS_MULTI_REFUSE(e, entry) \
    if ((e) && (e)->multi) return multi_refuse(entry)

// fn(r) on every listed shard's worker, concurrently; waits for all.  The first failure in shard order is returned, its
// reason copied from the worker's thread into the caller's wax_vs_last_error().
static int32_t multi_run(MultiEngine *m, const std::vector<int> &which, const std::function<int32_t(int)> &fn) {
    const size_t n = which.size();
    std::vector<int32_t> rc(n, WAX_VS_OK);
    std::vector<std::string> why(n);
    std::mutex mu;
    std::condition_variable cv;
    size_t left = n;
    for (size_t i = 0; i < n; ++i)
        m->workers[which[i]]->post([&, i] {
            const int32_t c = fn(which[i]);
            if (c != WAX_VS_OK) why[i] = wax_vs_last_error();
            std::lock_guard<std::mutex> g(mu);
            rc[i] = c;
            if (--left == 0) cv.notify_one();
        });
    std::unique_lock<std::mutex> g(mu);
    cv.wait(g, [&] { return left == 0; });
    for (size_t i = 0; i < n; ++i)
        if (rc[i] != WAX_VS_OK) return fail(rc[i], "%s", why[i].c_str());
    return WAX_VS_OK;
}
static int32_t multi_run_all(MultiEngine *m, const std::function<int32_t(int)> &fn) {
    std::vector<int> all(m->n());
    for (int r = 0; r < m->n(); ++r) all[r] = r;
    return multi_run(m, all, fn);
}

static int32_t multi_ctx_acquire(MultiEngine *m, MultiCtx **out) {
    {
        std::lock_guard<std::mutex> g(m->pool_mu);
        if (!m->pool.empty()) {
            *out = m->pool.back();
            m->pool.pop_back();
            return WAX_VS_OK;
        }
    }
    std::unique_ptr<MultiCtx> c(new (std::nothrow) MultiCtx());
    if (!c) return fail(WAX_VS_ERR_CUDA, "out of host memory");
    c->part.resize(m->n());
    for (int r = 0; r < m->n(); ++r) {
        MultiCtx::Part &p = c->part[r];
        p.device = m->devices[r];
        DeviceGuard g(p.device);
        if (!g.ok) return g.error();
        CUDA_TRY(cudaStreamCreateWithFlags(&p.stream, cudaStreamNonBlocking));
        CUDA_TRY(cudaEventCreateWithFlags(&p.done, cudaEventDisableTiming));
        if (r == 0) CUDA_TRY(cudaEventCreateWithFlags(&c->chosen, cudaEventDisableTiming));
    }
    *out = c.release();
    return WAX_VS_OK;
}
struct MultiLease {
    MultiEngine *m;
    MultiCtx *c = nullptr;
    explicit MultiLease(MultiEngine *eng) : m(eng) {}
    MultiLease(const MultiLease &) = delete;
    MultiLease &operator=(const MultiLease &) = delete;
    ~MultiLease() {
        if (!c) return;
        std::lock_guard<std::mutex> g(m->pool_mu);
        m->pool.push_back(c);
    }
    int32_t acquire() { return multi_ctx_acquire(m, &c); }
};

// ---- lifetime -------------------------------------------------------------------------------------------------------
static void multi_destroy(MultiEngine *m) {
    for (auto &w : m->workers) {
        { std::lock_guard<std::mutex> g(w->mu); w->stop = true; }
        w->cv.notify_one();
        w->th.join();
    }
    for (MultiCtx *c : m->pool) delete c;
    for (wax_vs_engine *s : m->shards) wax_vs_destroy(s);
    delete m;
}

// The checks that need no device run in wax_vs_create before this.  Distinct devices must reach each other's memory:
// the merge on devices[0] reads every shard's list in place.
static int32_t multi_create(uint32_t dims, uint8_t similarity, const int32_t *devices, int32_t n, wax_vs_engine **out) {
    int count = 0;
    if (cudaGetDeviceCount(&count) != cudaSuccess || count <= 0) {
        cudaGetLastError();
        return fail(WAX_VS_ERR_CUDA, "CUDA device not available");
    }
    for (int32_t r = 0; r < n; ++r)
        if (devices[r] >= count) return fail(WAX_VS_ERR_ARGUMENT, "device ordinal %d out of range (0..%d)", devices[r], count - 1);
    for (int32_t r = 1; r < n; ++r) {
        if (devices[r] == devices[0]) continue;
        int a = 0, b = 0;
        if (cudaDeviceCanAccessPeer(&a, devices[0], devices[r]) != cudaSuccess ||
            cudaDeviceCanAccessPeer(&b, devices[r], devices[0]) != cudaSuccess || !a || !b) {
            cudaGetLastError();
            return fail(WAX_VS_ERR_UNSUPPORTED, "devices %d and %d cannot access each other's memory", devices[0], devices[r]);
        }
        for (int way = 0; way < 2; ++way) {        // device 0 reads the shards' lists; round 2 of grouped reads d_chosen
            const int from = way ? devices[r] : devices[0], to = way ? devices[0] : devices[r];
            DeviceGuard g(from);
            if (!g.ok) return g.error();
            const cudaError_t err = cudaDeviceEnablePeerAccess(to, 0);
            if (err != cudaSuccess && err != cudaErrorPeerAccessAlreadyEnabled)
                return fail(WAX_VS_ERR_CUDA, "cudaDeviceEnablePeerAccess(%d -> %d) failed: %s", from, to, cudaGetErrorString(err));
            cudaGetLastError();
        }
    }
    wax_vs_engine *h = new (std::nothrow) wax_vs_engine();
    MultiEngine *m = new (std::nothrow) MultiEngine();
    if (!h || !m) { delete h; delete m; return fail(WAX_VS_ERR_CUDA, "out of host memory"); }
    h->device = devices[0]; h->dims = dims; h->similarity = similarity; h->multi = m;
    m->devices.assign(devices, devices + n);
    m->rows.assign(n, 0);
    for (int32_t r = 0; r < n; ++r) {
        wax_vs_engine *s = nullptr;
        const int32_t rc = wax_vs_create(dims, similarity, devices + r, 1, &s);
        if (rc) { multi_destroy(m); h->multi = nullptr; delete h; return rc; }
        m->shards.push_back(s);
        m->workers.emplace_back(new MultiWorker());
        MultiWorker *w = m->workers.back().get();
        w->th = std::thread([w] { w->loop(); });
    }
    *out = h;
    return WAX_VS_OK;
}

// ---- corpus ---------------------------------------------------------------------------------------------------------
// How many of m_new new rows each shard takes: the shards with the fewest rows first, to one level, ties to lower shards
// (sharded.fill_emptiest).
static std::vector<uint64_t> multi_fill_emptiest(const std::vector<uint64_t> &counts, uint64_t m_new) {
    std::vector<uint64_t> alloc(counts.size(), 0);
    if (m_new == 0) return alloc;
    uint64_t lo = *std::min_element(counts.begin(), counts.end()), hi = *std::max_element(counts.begin(), counts.end()) + m_new;
    auto need = [&](uint64_t level) { uint64_t s = 0; for (uint64_t c : counts) s += level > c ? level - c : 0; return s; };
    while (lo < hi) {                                  // the largest level L with sum(max(0, L - count)) <= m_new
        const uint64_t mid = (lo + hi + 1) / 2;
        if (need(mid) <= m_new) lo = mid; else hi = mid - 1;
    }
    uint64_t rest = m_new;
    for (size_t r = 0; r < counts.size(); ++r) { alloc[r] = lo > counts[r] ? lo - counts[r] : 0; rest -= alloc[r]; }
    for (size_t r = 0; r < counts.size() && rest; ++r)   // fewer than the shards at the level: one more each
        if (counts[r] + alloc[r] == lo) { ++alloc[r]; --rest; }
    return alloc;
}

static int32_t multi_add_batch(MultiEngine *m, const uint64_t *frame_ids, const float *rows, uint64_t n, uint32_t dims,
                               uint32_t vector_len) {
    if (n == 0) return WAX_VS_OK;
    if (!frame_ids || !rows) return fail(WAX_VS_ERR_NULL, "NULL argument");
    if (vector_len != dims) return fail(WAX_VS_ERR_DIMENSION, "vector dimension mismatch: expected %u, got %u", dims, vector_len);
    std::unique_lock<std::shared_mutex> w(m->rw);
    const int R = m->n();
    // sharded.plan_add_batch: held ids are upserted by their owner; the distinct new ids, in order of first appearance,
    // take the next keys and are split in contiguous chunks over the shards; every occurrence follows its first one.
    std::vector<std::vector<uint8_t>> held(R);
    int32_t rc = multi_run_all(m, [&](int r) -> int32_t {
        held[r].assign(n, 0);
        return m->rows[r] ? wax_vs_contains(m->shards[r], frame_ids, n, held[r].data()) : WAX_VS_OK;
    });
    if (rc) return rc;
    std::vector<int> dest(n, -1);
    std::vector<uint64_t> seq_of(n, 0);
    std::unordered_map<uint64_t, uint64_t> seq;        // new id -> its sequence number among the batch's new ids
    for (uint64_t i = 0; i < n; ++i) {
        for (int r = 0; r < R && dest[i] < 0; ++r)
            if (held[r][i]) dest[i] = r;
        if (dest[i] < 0) seq_of[i] = seq.emplace(frame_ids[i], seq.size()).first->second;
    }
    const std::vector<uint64_t> alloc = multi_fill_emptiest(m->rows, seq.size());
    std::vector<uint64_t> end(R), first_key(R);
    uint64_t acc = 0;
    for (int r = 0; r < R; ++r) { first_key[r] = m->next_key + acc; acc += alloc[r]; end[r] = acc; }
    std::vector<std::vector<uint64_t>> items(R);
    for (uint64_t i = 0; i < n; ++i) {
        if (dest[i] < 0) dest[i] = static_cast<int>(std::upper_bound(end.begin(), end.end(), seq_of[i]) - end.begin());
        items[dest[i]].push_back(i);
    }
    std::vector<int> busy;
    for (int r = 0; r < R; ++r) if (!items[r].empty()) busy.push_back(r);
    std::vector<uint64_t> appended(R, 0);
    rc = multi_run(m, busy, [&](int r) -> int32_t {
        if (items[r].size() == n)                      // the whole batch: no copy
            return wax_vs_add_batch_keyed(m->shards[r], frame_ids, rows, n, dims, first_key[r], &appended[r]);
        std::vector<uint64_t> ids(items[r].size());
        std::vector<float> vec(items[r].size() * dims);
        for (size_t j = 0; j < items[r].size(); ++j) {
            ids[j] = frame_ids[items[r][j]];
            memcpy(vec.data() + j * dims, rows + items[r][j] * dims, dims * sizeof(float));
        }
        return wax_vs_add_batch_keyed(m->shards[r], ids.data(), vec.data(), ids.size(), dims, first_key[r], &appended[r]);
    });
    for (int r = 0; r < R; ++r) m->rows[r] += appended[r];
    m->next_key += seq.size();             // even after a failure: a shard that appended holds these keys
    return rc;
}

static int32_t multi_remove_batch(MultiEngine *m, const uint64_t *frame_ids, uint64_t n, uint64_t *out_removed) {
    if (out_removed) *out_removed = 0;
    if (n == 0) return WAX_VS_OK;
    if (!frame_ids) return fail(WAX_VS_ERR_NULL, "frame_ids is NULL");
    std::unique_lock<std::shared_mutex> w(m->rw);
    std::vector<int> busy;
    for (int r = 0; r < m->n(); ++r) if (m->rows[r]) busy.push_back(r);
    std::vector<uint64_t> gone(m->n(), 0);
    const int32_t rc = multi_run(m, busy, [&](int r) -> int32_t { return wax_vs_remove_batch(m->shards[r], frame_ids, n, &gone[r]); });
    uint64_t sum = 0;
    for (int r = 0; r < m->n(); ++r) { m->rows[r] -= gone[r]; sum += gone[r]; }
    if (out_removed) *out_removed = sum;
    return rc;
}

// ---- rebalance ------------------------------------------------------------------------------------------------------
struct MultiMove {
    int donor, receiver;
    uint64_t rows;
};
// sharded.plan_rebalance, ported unchanged: targets of T / R rows, the T % R extra rows to the shards that hold the most
// (ties to lower shards); donors and receivers in shard order, each donor's tail dealt out in key order.
static std::vector<MultiMove> multi_plan_rebalance(const std::vector<uint64_t> &counts) {
    const size_t R = counts.size();
    uint64_t total = 0;
    for (uint64_t c : counts) total += c;
    std::vector<uint64_t> target(R, total / R);
    std::vector<size_t> order(R);
    for (size_t r = 0; r < R; ++r) order[r] = r;
    std::stable_sort(order.begin(), order.end(), [&](size_t a, size_t b) { return counts[a] > counts[b]; });
    for (uint64_t i = 0; i < total % R; ++i) ++target[order[i]];
    std::vector<uint64_t> take(R);
    for (size_t r = 0; r < R; ++r) take[r] = target[r] > counts[r] ? target[r] - counts[r] : 0;
    std::vector<MultiMove> moves;
    size_t r = 0;
    for (size_t d = 0; d < R; ++d) {
        for (uint64_t left = counts[d] > target[d] ? counts[d] - target[d] : 0; left;) {
            while (take[r] == 0) ++r;
            const uint64_t n = std::min(left, take[r]);
            moves.push_back(MultiMove{static_cast<int>(d), static_cast<int>(r), n});
            left -= n;
            take[r] -= n;
        }
    }
    return moves;
}

// Each receiver merges its incoming runs in move order on its own worker (absorb_rows), the receivers concurrently: a
// shard is a donor or a receiver, never both, so the donors are only read meanwhile.  Then each donor drops the rows of
// its completed moves, all from its tail, by wax_vs_remove_batch: a truncation, its rows [0, new_n) and their caches stay
// valid.  A failed move changes nothing on its receiver, and its rows stay on the donor.
static int32_t multi_rebalance(MultiEngine *m, uint64_t *out_moved) {
    std::unique_lock<std::shared_mutex> w(m->rw);
    const std::vector<MultiMove> moves = multi_plan_rebalance(m->rows);
    if (moves.empty()) return WAX_VS_OK;
    const int R = m->n();
    std::vector<uint64_t> tail(m->rows), first(moves.size());   // tail[d]: where donor d's next run starts
    for (const MultiMove &mv : moves) tail[mv.donor] -= mv.rows;
    std::vector<std::vector<size_t>> into(R);
    for (size_t i = 0; i < moves.size(); ++i) {
        first[i] = tail[moves[i].donor];
        tail[moves[i].donor] += moves[i].rows;
        into[moves[i].receiver].push_back(i);
    }
    std::vector<int> receivers, donors;
    for (int r = 0; r < R; ++r) if (!into[r].empty()) receivers.push_back(r);
    std::vector<uint8_t> done(moves.size(), 0);
    const int32_t rc = multi_run(m, receivers, [&](int r) -> int32_t {
        for (size_t i : into[r]) {
            if (const int32_t mrc = absorb_rows(m->shards[r], m->shards[moves[i].donor], first[i], moves[i].rows)) return mrc;
            done[i] = 1;
        }
        return WAX_VS_OK;
    });
    const std::string why = rc ? wax_vs_last_error() : "";
    std::vector<std::vector<uint64_t>> drop(R);
    uint64_t moved = 0;
    for (size_t i = 0; i < moves.size(); ++i) {
        if (!done[i]) continue;
        for (uint64_t row = first[i]; row < first[i] + moves[i].rows; ++row)
            drop[moves[i].donor].push_back(frame_id_of(m->shards[moves[i].donor], row));
        m->rows[moves[i].receiver] += moves[i].rows;
        moved += moves[i].rows;
    }
    for (int d = 0; d < R; ++d) if (!drop[d].empty()) donors.push_back(d);
    std::vector<uint64_t> gone(R, 0);
    const int32_t drc = multi_run(m, donors, [&](int d) -> int32_t {
        return wax_vs_remove_batch(m->shards[d], drop[d].data(), drop[d].size(), &gone[d]);
    });
    for (int d = 0; d < R; ++d) m->rows[d] -= gone[d];
    if (out_moved) *out_moved = moved;
    if (rc) return fail(rc, "%s", why.c_str());
    return drc;
}

static int32_t multi_reserve(MultiEngine *m, uint64_t rows) {
    if (rows > 0xFFFFFFFFull)
        return fail(WAX_VS_ERR_CAPACITY, "capacity exceeded: limit %llu, requested %llu", 0xFFFFFFFFull,
                    static_cast<unsigned long long>(rows));
    std::unique_lock<std::shared_mutex> w(m->rw);
    const uint64_t each = (rows + m->n() - 1) / m->n();
    return multi_run_all(m, [&](int r) -> int32_t { return wax_vs_reserve(m->shards[r], each); });
}

static uint64_t multi_mv2v_length(uint64_t rows, uint32_t dims) { return 36ull + rows * dims * 4ull + 8ull + rows * 8ull; }

// MV2V bytes of the whole corpus: each shard's rows go straight to their key-rank positions in the caller's buffer
// (sharded.plan_serialize's rule), one export per run of consecutive positions.  A shard whose runs average fewer than
// kExportRun rows (a corpus built by single adds alternates shards row by row) exports instead in chunks of kExportChunk
// rows through a staging buffer, so the export calls are bounded by rows / kExportChunk, not by rows.
constexpr uint64_t kExportRun = 64, kExportChunk = 1u << 16;
static int32_t multi_serialize(MultiEngine *m, uint32_t dims, uint8_t similarity, uint8_t *dst, uint64_t cap, uint64_t *out_len) {
    if (!dst) return fail(WAX_VS_ERR_NULL, "NULL argument");
    std::shared_lock<std::shared_mutex> r_lock(m->rw);
    const uint64_t total = m->total(), need = multi_mv2v_length(total, dims);
    if (out_len) *out_len = need;
    if (cap < need) return fail(WAX_VS_ERR_BUFFER, "serialize needs %llu bytes, buffer has %llu",
                                static_cast<unsigned long long>(need), static_cast<unsigned long long>(cap));
    const int R = m->n();
    std::vector<std::vector<uint64_t>> keys(R);
    int32_t rc = multi_run_all(m, [&](int r) -> int32_t {
        keys[r].resize(m->rows[r]);
        return m->rows[r] ? wax_vs_export_rows(m->shards[r], 0, m->rows[r], nullptr, nullptr, keys[r].data()) : WAX_VS_OK;
    });
    if (rc) return rc;
    // position of every row = the rank of its key among all keys (each shard's keys increase: an R-way merge)
    std::vector<std::vector<uint64_t>> pos(R);
    std::vector<size_t> at(R, 0);
    for (int r = 0; r < R; ++r) pos[r].resize(keys[r].size());
    for (uint64_t p = 0; p < total; ++p) {
        int best = -1;
        for (int r = 0; r < R; ++r)
            if (at[r] < keys[r].size() && (best < 0 || keys[r][at[r]] < keys[best][at[best]])) best = r;
        pos[best][at[best]++] = p;
    }
    uint8_t *p = dst;
    const uint8_t magic[4] = {0x4D, 0x56, 0x32, 0x56};
    memcpy(p, magic, 4); p += 4;
    const uint16_t version = 1; memcpy(p, &version, 2); p += 2;
    *p++ = 2;
    *p++ = similarity;
    memcpy(p, &dims, 4); p += 4;
    memcpy(p, &total, 8); p += 8;
    const uint64_t vbytes = total * dims * 4ull, ibytes = total * 8ull;
    memcpy(p, &vbytes, 8); p += 8;
    memset(p, 0, 8); p += 8;
    float *vecs = reinterpret_cast<float *>(p);
    uint8_t *ids_out = p + vbytes + 8;
    memcpy(p + vbytes, &ibytes, 8);
    return multi_run_all(m, [&](int r) -> int32_t {
        std::vector<uint64_t> ids;
        const uint64_t rows = pos[r].size();
        uint64_t runs = 0;
        for (uint64_t i = 0; i < rows; ++i) runs += i == 0 || pos[r][i] != pos[r][i - 1] + 1;
        if (runs * kExportRun > rows) {            // short runs (rows added one by one): chunks through a bounded staging
            const uint64_t chunk = std::min<uint64_t>(rows, kExportChunk);
            std::vector<float> stage(chunk * dims);
            ids.resize(chunk);
            for (uint64_t i = 0; i < rows; i += chunk) {
                const uint64_t len = std::min(chunk, rows - i);
                const int32_t erc = wax_vs_export_rows(m->shards[r], i, len, ids.data(), stage.data(), nullptr);
                if (erc) return erc;
                for (uint64_t j = 0; j < len; ++j) {
                    memcpy(vecs + pos[r][i + j] * dims, stage.data() + j * dims, dims * sizeof(float));
                    memcpy(ids_out + pos[r][i + j] * 8, &ids[j], 8);
                }
            }
            return WAX_VS_OK;
        }
        for (uint64_t i = 0; i < pos[r].size();) {
            uint64_t j = i + 1;
            while (j < pos[r].size() && pos[r][j] == pos[r][j - 1] + 1) ++j;
            ids.resize(j - i);
            const int32_t erc = wax_vs_export_rows(m->shards[r], i, j - i, ids.data(), vecs + pos[r][i] * dims, nullptr);
            if (erc) return erc;
            memcpy(ids_out + pos[r][i] * 8, ids.data(), ids.size() * 8);
            i = j;
        }
        return WAX_VS_OK;
    });
}

// Shard r loads the blob's rows shard_range(count, n, r).  Shard 0 checks the blob first, exactly as
// wax_vs_deserialize would, so a malformed blob changes nothing; a failure after that leaves every shard empty.
static int32_t multi_deserialize(MultiEngine *m, uint32_t dims, uint8_t similarity, const uint8_t *src, uint64_t len) {
    if (!src) return fail(WAX_VS_ERR_NULL, "NULL argument");
    std::unique_lock<std::shared_mutex> w(m->rw);
    const int R = m->n();
    uint64_t count = 0;
    if (len >= 36) memcpy(&count, src + 12, 8);
    auto lo = [&](int r) -> uint64_t { return count * r / R; };
    int32_t rc = wax_vs_deserialize_rows(m->shards[0], src, len, lo(0), lo(1) - lo(0));
    if (rc == WAX_VS_OK) {
        std::vector<int> rest;
        for (int r = 1; r < R; ++r) rest.push_back(r);
        rc = multi_run(m, rest, [&](int r) -> int32_t {
            return wax_vs_deserialize_rows(m->shards[r], src, len, lo(r), (count * (r + 1) / R) - lo(r));
        });
        if (rc == WAX_VS_OK) {
            for (int r = 0; r < R; ++r) m->rows[r] = count * (r + 1) / R - lo(r);
            m->next_key = count;
            return WAX_VS_OK;
        }
    } else if (rc != WAX_VS_ERR_CUDA) {
        return rc;                                     // the blob's checks: nothing changed
    }
    const std::string why = wax_vs_last_error();
    uint8_t empty[44] = {0x4D, 0x56, 0x32, 0x56, 1, 0, 2, similarity};
    memcpy(empty + 8, &dims, 4);
    for (int r = 0; r < R; ++r) wax_vs_deserialize_rows(m->shards[r], empty, sizeof empty, 0, 0);
    m->rows.assign(R, 0);
    m->next_key = 0;
    return fail(rc, "%s", why.c_str());
}

// ---- search ---------------------------------------------------------------------------------------------------------
static std::vector<int> multi_live(const MultiEngine *m) {      // an empty shard takes no launch and is left out of merges
    std::vector<int> live;
    for (int r = 0; r < m->n(); ++r) if (m->rows[r]) live.push_back(r);
    return live;
}
static int32_t multi_check_query(uint32_t dims, const float *queries, uint32_t query_len) {   // check_query's rules
    if (!queries) return fail(WAX_VS_ERR_NULL, "query is NULL");
    if (query_len != dims) return fail(WAX_VS_ERR_DIMENSION, "vector dimension mismatch: expected %u, got %u", dims, query_len);
    return WAX_VS_OK;
}

// Each live shard: its own H2D copy of the queries (no scan reads peer memory), then run(r, d_queries, stream), then an
// event device 0 waits on.  On the workers, or from the caller's thread when run only enqueues.
using MultiShardRun = std::function<int32_t(int, const float *, cudaStream_t)>;
static int32_t multi_fan_out(MultiEngine *m, MultiCtx *c, const std::vector<int> &live, const float *queries, uint32_t n_queries,
                             uint32_t dims, bool on_workers, const MultiShardRun &run) {
    auto one = [&](int r) -> int32_t {
        MultiCtx::Part &p = c->part[r];
        DeviceGuard g(p.device);
        if (!g.ok) return g.error();
        int32_t rc;
        if ((rc = p.d_queries.ensure(static_cast<size_t>(n_queries) * dims, "queries"))) return rc;
        CUDA_TRY(cudaMemcpyAsync(p.d_queries, queries, static_cast<size_t>(n_queries) * dims * sizeof(float),
                                 cudaMemcpyHostToDevice, p.stream));
        if ((rc = run(r, p.d_queries, p.stream))) return rc;
        CUDA_TRY(cudaEventRecord(p.done, p.stream));
        return WAX_VS_OK;
    };
    if (on_workers) return multi_run(m, live, one);
    for (int r : live) if (const int32_t rc = one(r)) return rc;
    return WAX_VS_OK;
}
// Device 0's stream waits on every live shard's event (shard 0's list is in its order already).
static int32_t multi_wait_shards(MultiCtx *c, const std::vector<int> &live) {
    for (int r : live)
        if (r != 0) CUDA_TRY(cudaStreamWaitEvent(c->part[0].stream, c->part[r].done, 0));
    return WAX_VS_OK;
}
// The live shards' [n][k] lists (Part::d_cands) -> [n][k_out] on device 0 by ONE merge launch reading them in place.
static int32_t multi_merge_lists(MultiCtx *c, const std::vector<int> &live, uint32_t n, uint32_t k, uint32_t k_out) {
    int32_t rc;
    if ((rc = c->d_merged.ensure(static_cast<size_t>(n) * k_out, "merged candidates"))) return rc;
    PeerLists<wax_vs_candidate> lists{};
    for (size_t i = 0; i < live.size(); ++i) lists.list[i] = c->part[live[i]].d_cands;
    if ((rc = multi_wait_shards(c, live))) return rc;
    merge_gathered_kernel<<<n, 128, 0, c->part[0].stream>>>(lists, static_cast<uint32_t>(live.size()), n, k, k_out, c->d_merged);
    CUDA_TRY(cudaGetLastError());
    return WAX_VS_OK;
}
static int32_t multi_download_merged(MultiCtx *c, size_t n) {
    int32_t rc;
    if ((rc = c->h_merged.ensure(n, "result staging"))) return rc;
    CUDA_TRY(cudaMemcpyAsync(c->h_merged, c->d_merged, n * sizeof(wax_vs_candidate), cudaMemcpyDeviceToHost, c->part[0].stream));
    CUDA_TRY(cudaStreamSynchronize(c->part[0].stream));
    return WAX_VS_OK;
}
// The merged [n][k] lists -> the caller's ids and scores (the valid entries, best first), out_n per query.
static void multi_deliver(const MultiCtx *c, uint8_t similarity, uint32_t n, uint32_t k, uint64_t *out_ids, float *out_scores,
                          uint32_t out_stride, uint32_t *out_n) {
    for (uint32_t q = 0; q < n; ++q) {
        uint32_t got = 0;
        for (uint32_t i = 0; i < k; ++i) {
            const wax_vs_candidate &cd = c->h_merged[static_cast<size_t>(q) * k + i];
            if (!cd.valid) continue;
            out_ids[static_cast<size_t>(q) * out_stride + got] = cd.frame_id;
            out_scores[static_cast<size_t>(q) * out_stride + got] = score_from_distance(similarity, cd.distance);
            ++got;
        }
        out_n[q] = got;
    }
}

// search_host's contract: the empty handle answers before the query is validated, then the query, the outputs and
// the buffer size, in that order and with the same reasons.
static int32_t multi_search(MultiEngine *m, uint32_t dims, uint8_t similarity, const float *queries, uint32_t n_queries,
                            uint32_t query_len, int64_t top_k, uint64_t *out_ids, float *out_scores, uint32_t out_stride,
                            uint32_t *out_n) {
    if (!out_n) return fail(WAX_VS_ERR_NULL, "NULL argument");
    std::shared_lock<std::shared_mutex> r_lock(m->rw);
    const uint64_t total = m->total();
    if (total == 0) {
        for (uint32_t i = 0; i < n_queries; ++i) out_n[i] = 0;
        return WAX_VS_OK;
    }
    if (n_queries == 0) return WAX_VS_OK;
    int32_t rc;
    if ((rc = multi_check_query(dims, queries, query_len))) return rc;
    const uint32_t k = clamp_topk(top_k);
    const uint32_t k_eff = static_cast<uint32_t>(std::min<uint64_t>(k, total));
    if (!out_ids || !out_scores) return fail(WAX_VS_ERR_NULL, "output buffer is NULL");
    if (out_stride < k_eff) return fail(WAX_VS_ERR_BUFFER, "output buffers hold %u entries, need %u", out_stride, k_eff);

    MultiLease lease(m);
    if ((rc = lease.acquire())) return rc;
    MultiCtx *c = lease.c;
    const std::vector<int> live = multi_live(m);
    // wax_vs_search_device only enqueues: one query is issued from this thread
    rc = multi_fan_out(m, c, live, queries, n_queries, dims, n_queries > 1, [&](int r, const float *dq, cudaStream_t s) -> int32_t {
        MultiCtx::Part &p = c->part[r];
        int32_t prc;
        if ((prc = p.d_cands.ensure(static_cast<size_t>(n_queries) * k, "shard candidates"))) return prc;
        return n_queries == 1 ? wax_vs_search_device(m->shards[r], dq, 1, k, 0, p.d_cands, s)
                              : wax_vs_search_batch_device(m->shards[r], dq, n_queries, k, 0, p.d_cands, s);
    });
    if (rc) return rc;
    DeviceGuard g(c->part[0].device);
    if (!g.ok) return g.error();
    if ((rc = multi_merge_lists(c, live, n_queries, k, k_eff)) || (rc = multi_download_merged(c, static_cast<size_t>(n_queries) * k_eff)))
        return rc;
    multi_deliver(c, similarity, n_queries, k_eff, out_ids, out_scores, out_stride, out_n);
    return WAX_VS_OK;
}

// The filtered and where entry points, after their argument checks (search_where zeroed out_n): every live shard plans
// its rows for the request (search_where_device) and the lists merge as above.  One engine's buffer check needs
// max_i min(clamp(k), rows query i allows); the merged lists hold min(clamp(k), allowed rows with a finite distance)
// valid entries per query, the same number whenever the allowed rows are finite.
static int32_t multi_search_where(MultiEngine *m, uint32_t dims, uint8_t similarity, const SearchRequest &req,
                                  uint64_t *out_ids, float *out_scores, uint32_t out_stride, uint32_t *out_n) {
    const uint32_t n_queries = req.n_queries;
    std::shared_lock<std::shared_mutex> r_lock(m->rw);
    if (m->total() == 0 || n_queries == 0) return WAX_VS_OK;
    int32_t rc;
    if ((rc = multi_check_query(dims, req.queries, req.query_len))) return rc;
    const uint32_t k = clamp_topk(req.top_k);
    MultiLease lease(m);
    if ((rc = lease.acquire())) return rc;
    MultiCtx *c = lease.c;
    const std::vector<int> live = multi_live(m);
    rc = multi_fan_out(m, c, live, req.queries, n_queries, dims, true, [&](int r, const float *dq, cudaStream_t s) -> int32_t {
        MultiCtx::Part &p = c->part[r];
        int32_t prc;
        if ((prc = p.d_cands.ensure(static_cast<size_t>(n_queries) * k, "shard candidates"))) return prc;
        return search_where_device(m->shards[r], req, dq, 0, p.d_cands, s);
    });
    if (rc) return rc;
    DeviceGuard g(c->part[0].device);
    if (!g.ok) return g.error();
    if ((rc = multi_merge_lists(c, live, n_queries, k, k)) || (rc = multi_download_merged(c, static_cast<size_t>(n_queries) * k)))
        return rc;
    uint32_t k_max = 0;
    for (uint32_t q = 0; q < n_queries; ++q) {
        uint32_t v = 0;
        for (uint32_t i = 0; i < k; ++i) v += c->h_merged[static_cast<size_t>(q) * k + i].valid != 0;
        k_max = std::max(k_max, v);
    }
    if (k_max == 0) return WAX_VS_OK;
    if (!out_ids || !out_scores) return fail(WAX_VS_ERR_NULL, "output buffer is NULL");
    if (out_stride < k_max) return fail(WAX_VS_ERR_BUFFER, "output buffers hold %u entries, need %u", out_stride, k_max);
    multi_deliver(c, similarity, n_queries, k, out_ids, out_scores, out_stride, out_n);
    return WAX_VS_OK;
}

// Grouped search, the protocol of the sharded grouped form (DESIGN.md section 4.14) with the shards' buffers read in place
// on device 0: round 1 (grouped_heads_device) on every live shard, merge 1 (merge_group_heads_kernel over PeerLists) on
// device 0; with per_group > 1 round 2 (grouped_expand_device, reading d_chosen on device 0) and the per-(query, group)
// merge of the rows.  After the argument checks (search_grouped zeroed out_n).
static int32_t multi_search_grouped(MultiEngine *m, uint32_t dims, uint8_t similarity, const SearchRequest &req,
                                    uint64_t *out_ids, float *out_scores, uint64_t *out_groups, uint32_t out_stride,
                                    uint32_t *out_n) {
    const uint32_t n_queries = req.n_queries, G = clamp_topk(req.top_k), P = req.per_group;
    if (G > WAX_VS_SHARD_MAX_GROUPS)
        return fail(WAX_VS_ERR_UNSUPPORTED, "sharded grouped search takes clamp(top_groups) <= %d (got %u)",
                    WAX_VS_SHARD_MAX_GROUPS, G);
    std::shared_lock<std::shared_mutex> r_lock(m->rw);
    const uint64_t total = m->total();
    if (total == 0 || n_queries == 0) return WAX_VS_OK;
    int32_t rc;
    if ((rc = multi_check_query(dims, req.queries, req.query_len))) return rc;
    const uint32_t need = static_cast<uint32_t>(std::min<uint64_t>(static_cast<uint64_t>(G) * P, total));
    if (out_stride < need) return fail(WAX_VS_ERR_BUFFER, "output buffers hold %u entries, need %u", out_stride, need);
    MultiLease lease(m);
    if ((rc = lease.acquire())) return rc;
    MultiCtx *c = lease.c;
    const std::vector<int> live = multi_live(m);
    const size_t slots = static_cast<size_t>(n_queries) * G * P;
    rc = multi_fan_out(m, c, live, req.queries, n_queries, dims, true, [&](int r, const float *dq, cudaStream_t s) -> int32_t {
        MultiCtx::Part &p = c->part[r];
        int32_t prc;
        if ((prc = p.d_heads.ensure(slots, "group heads"))) return prc;
        return grouped_heads_device(m->shards[r], req, dq, 0, p.d_heads, s);
    });
    if (rc) return rc;
    MultiCtx::Part &p0 = c->part[0];
    {
        DeviceGuard g(p0.device);
        if (!g.ok) return g.error();
        if ((rc = c->d_chosen.ensure(static_cast<size_t>(n_queries) * G, "chosen groups")) ||
            (rc = c->h_chosen.ensure(static_cast<size_t>(n_queries) * G, "chosen groups staging")))
            return rc;
        PeerLists<wax_vs_group_candidate> heads{};
        for (size_t i = 0; i < live.size(); ++i) heads.list[i] = c->part[live[i]].d_heads;
        const uint32_t world = static_cast<uint32_t>(live.size());
        uint32_t pow2 = 32;
        while (pow2 < world * G) pow2 <<= 1;
        const size_t smem = static_cast<size_t>(pow2) * (sizeof(uint64_t) + 3 * sizeof(uint32_t));
        CUDA_TRY(grant_smem(m->shards[0], merge_group_heads_kernel<PeerLists<wax_vs_group_candidate>>, smem));
        if ((rc = multi_wait_shards(c, live))) return rc;
        merge_group_heads_kernel<<<n_queries, 1024, smem, p0.stream>>>(heads, world, n_queries, G, P, pow2, c->d_chosen);
        CUDA_TRY(cudaGetLastError());
        CUDA_TRY(cudaEventRecord(c->chosen, p0.stream));
    }
    if (P > 1) {
        rc = multi_run(m, live, [&](int r) -> int32_t {
            MultiCtx::Part &p = c->part[r];
            DeviceGuard g(p.device);
            if (!g.ok) return g.error();
            int32_t prc;
            if ((prc = p.d_cands.ensure(slots, "group rows"))) return prc;
            CUDA_TRY(cudaStreamWaitEvent(p.stream, c->chosen, 0));
            if ((prc = grouped_expand_device(m->shards[r], req, p.d_queries, c->d_chosen, p.d_heads, 0, p.d_cands, p.stream)))
                return prc;
            CUDA_TRY(cudaEventRecord(p.done, p.stream));
            return WAX_VS_OK;
        });
        if (rc) return rc;
    }
    DeviceGuard g(p0.device);
    if (!g.ok) return g.error();
    if (P > 1 && ((rc = multi_merge_lists(c, live, n_queries * G, P, P)) || (rc = multi_download_merged(c, slots))))
        return rc;
    CUDA_TRY(cudaMemcpyAsync(c->h_chosen, c->d_chosen, static_cast<size_t>(n_queries) * G * sizeof(wax_vs_group_candidate),
                             cudaMemcpyDeviceToHost, p0.stream));
    CUDA_TRY(cudaStreamSynchronize(p0.stream));
    for (uint32_t q = 0; q < n_queries; ++q) {
        uint32_t got = 0;
        for (uint32_t j = 0; j < G; ++j) {
            const wax_vs_group_candidate &grp = c->h_chosen[static_cast<size_t>(q) * G + j];
            if (!grp.valid) continue;
            for (uint32_t i = 0; i < P; ++i) {
                float distance;
                uint64_t frame;
                if (P == 1) {
                    distance = grp.distance, frame = grp.frame_id;
                } else {
                    const wax_vs_candidate &cd = c->h_merged[(static_cast<size_t>(q) * G + j) * P + i];
                    if (!cd.valid) continue;
                    distance = cd.distance, frame = cd.frame_id;
                }
                const size_t at = static_cast<size_t>(q) * out_stride + got++;
                out_ids[at] = frame;
                out_scores[at] = score_from_distance(similarity, distance);
                out_groups[at] = grp.group_id;
            }
        }
        out_n[q] = got;
    }
    return WAX_VS_OK;
}

// set_attributes / set_locations / set_terms / set_groups: the full lists go to every shard (a shard ignores the frames
// it does not hold), *out_assigned is the shards' sum.  Every shard runs the same argument checks before it writes.
static int32_t multi_set(MultiEngine *m, uint64_t *out_assigned, const std::function<int32_t(wax_vs_engine *, uint64_t *)> &set) {
    if (out_assigned) *out_assigned = 0;
    std::unique_lock<std::shared_mutex> w(m->rw);
    std::vector<uint64_t> got(m->n(), 0);
    const int32_t rc = multi_run_all(m, [&](int r) -> int32_t { return set(m->shards[r], &got[r]); });
    if (rc) return rc;
    if (out_assigned) for (uint64_t v : got) *out_assigned += v;
    return WAX_VS_OK;
}

// ---- instrumentation ------------------------------------------------------------------------------------------------
static int32_t multi_set_option(MultiEngine *m, const char *key, int64_t value) {
    std::unique_lock<std::shared_mutex> w(m->rw);
    for (wax_vs_engine *s : m->shards) {
        const int32_t rc = wax_vs_debug_set_option(s, key, value);
        if (rc) return rc;
    }
    return WAX_VS_OK;
}

// "shard_rows.<r>": shard r's rows; any other name: the shards' counters summed.
static int32_t multi_counter(MultiEngine *m, const char *name, uint64_t *out) {
    unsigned r = 0;
    int used = 0;
    if (sscanf(name, "shard_rows.%u%n", &r, &used) == 1 && name[used] == '\0' && r < static_cast<unsigned>(m->n())) {
        std::shared_lock<std::shared_mutex> r_lock(m->rw);
        *out = m->rows[r];
        return WAX_VS_OK;
    }
    uint64_t sum = 0;
    for (wax_vs_engine *s : m->shards) {
        uint64_t v = 0;
        const int32_t rc = wax_vs_debug_counter(s, name, &v);
        if (rc) return rc;
        sum += v;
    }
    *out = sum;
    return WAX_VS_OK;
}
