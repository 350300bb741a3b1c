"""GPU, BASELINE.json full sizes (10 M x 384): size-independent properties + a full streaming oracle scan.

The oracle regenerates the synthetic corpus row by row (bit-identical generator), so no 15 GB host buffer is
needed; on the GPU box's host cores the 10 M-row scan takes a few seconds."""
import ctypes as C

import numpy as np
import pytest

from wax_b200 import CUDAVectorEngine, VectorMetric, sharded

pytestmark = pytest.mark.gpu

N_FULL, DIMS, SEED = 10_000_000, 384, 2      # BASELINE configs[1]: "10M x 384 fp32 corpus, 1 query, top-10 cosine"


@pytest.fixture(scope="module")
def full_engine():
    eng = CUDAVectorEngine(VectorMetric.cosine, DIMS)
    eng.fill_synthetic(SEED, N_FULL)
    yield eng
    eng.close()


def test_full_size_top10_bit_exact_against_streaming_oracle(oracle, full_engine):
    q = oracle.synth_row(1002, 0, DIMS, True)
    got = full_engine.search(q, 10)
    rows, d, s = oracle.search_synth(oracle.COSINE, SEED, 0, N_FULL, DIMS, True, q, 10,
                                     mode=oracle.ACC_F32_TREE, threads=oracle.host_threads())
    assert [g[0] for g in got] == rows.tolist()
    assert np.array_equal(np.float32([g[1] for g in got]).view(np.uint32), s.view(np.uint32))
    # fp64 truth for the returned rows: scores within 1e-4, order identical
    exact = [1.0 - oracle.distance(oracle.COSINE, oracle.ACC_F64, q, oracle.synth_row(SEED, r, DIMS, True)) for r in rows]
    assert np.max(np.abs(np.float64([g[1] for g in got]) - np.float64(exact))) <= 1e-4
    assert all(a > b for a, b in zip(exact, exact[1:]))


N_SAMPLED = 16          # queries of the full-size batch that are checked against the streaming oracle


@pytest.fixture(scope="module")
def c3_queries(oracle):
    """BASELINE configs[2]: 1024 queries against the 10 M x 384 corpus."""
    return oracle.synth_rows(1010, 0, 1024, DIMS, normalize=True)


@pytest.fixture(scope="module")
def c3_oracle_top100(oracle, c3_queries):
    """ONE streaming oracle pass over the 10 M synthetic rows for the sampled queries (each row generated once for
    all of them), kernel accumulation order, top-100: the top-72 / top-10 answers are its prefixes (total order)."""
    sample = list(range(0, 1024, 1024 // N_SAMPLED))[:N_SAMPLED]
    rows, d, s, n = oracle.search_synth_multi(oracle.COSINE, SEED, 0, N_FULL, DIMS, True, c3_queries[sample], 100,
                                              mode=oracle.ACC_F32_TREE, threads=oracle.host_threads())
    assert n.tolist() == [100] * N_SAMPLED
    return sample, rows, s


def _check_against_f64(oracle, metric, seed, n_rows, dims, normalize, queries, k, got_ids, got_scores):
    """north_star's bar against the fp64 truth: scores within 1e-4, ids identical outside fp64 near-ties (< 2e-6).
    One extra reference row (k + 1) exposes a near-tie at the k-th boundary."""
    from helpers import assert_tie_aware_order
    rows, d, s, n = oracle.search_synth_multi(metric, seed, 0, n_rows, dims, normalize, queries, k + 1,
                                              mode=oracle.ACC_F64, threads=oracle.host_threads())
    for i in range(len(queries)):
        ref64 = [1.0 - float(x) if metric == oracle.COSINE else -float(x) for x in d[i].astype(np.float64)]
        assert np.max(np.abs(np.float64(got_scores[i]) - np.float64(ref64[:k]))) <= 1e-4
        boundary_tie = abs(ref64[k] - ref64[k - 1]) <= 2e-6
        if not boundary_tie:
            assert sorted(int(x) for x in got_ids[i]) == sorted(rows[i][:k].tolist())
        assert_tie_aware_order(got_ids[i], rows[i][:k].tolist(), ref64[:k], 2e-6)


def test_full_size_k72_and_k100_against_the_full_oracle_top100(oracle, full_engine, c3_queries, c3_oracle_top100):
    """k = 100 (emit + radix-select path when fused_k_max < 100; fused lists otherwise), the production k = 72 and
    k = 10 against the oracle's COMPLETE top-100 of the 10 M rows: every id and every score bit, so a missed
    neighbour anywhere in the list fails."""
    sample, rows, s = c3_oracle_top100
    for j in (0, 7):
        q = c3_queries[sample[j]]
        for k in (100, 72, 10):
            got = full_engine.search(q, k)
            assert [g[0] for g in got] == rows[j][:k].tolist(), (j, k)
            assert np.array_equal(np.float32([g[1] for g in got]).view(np.uint32), s[j][:k].view(np.uint32)), (j, k)
    full_engine.set_option("fused_k_max", 32)                  # force the emit + radix-select path for k = 72 / 100
    try:
        q = c3_queries[sample[3]]
        for k in (100, 72):
            got = full_engine.search(q, k)
            assert [g[0] for g in got] == rows[3][:k].tolist(), ("select", k)
            assert np.array_equal(np.float32([g[1] for g in got]).view(np.uint32), s[3][:k].view(np.uint32))
    finally:
        full_engine.set_option("fused_k_max", 128)


def test_config2_full_size_batch_1024_top10_cosine(oracle, full_engine, c3_queries, c3_oracle_top100):
    """BASELINE configs[2] at its stated size: 10 M x 384, batch 1024, top-10 cosine through wax_vs_search_batch (the
    wgmma nomination levels).  (1) the WHOLE batch equals the single-query fused scan on the GPU; (2) the sampled
    queries equal the streaming oracle -- ids and score bits in the kernels' accumulation order; (3) within 1e-4 and
    tie-aware order against the fp64 oracle."""
    t0, f0 = full_engine.batch_stats()
    b0 = full_engine.counter("batch_bf16_queries")
    ids, scores, ns = full_engine.search_batch_arrays(c3_queries, 10)
    t1, f1 = full_engine.batch_stats()
    assert ns.tolist() == [10] * 1024
    assert (t1 - t0) + (f1 - f0) == 1024, "the batch did not take the tensor path"
    assert full_engine.counter("batch_bf16_queries") - b0 == 1024, "bf16 shadow nominations did not run"
    assert f1 - f0 <= 10, f"{f1 - f0} of 1024 queries fell back to the exact scan on unstructured data"
    full_engine.set_option("batch_tensor", 0)
    try:
        for i in range(1024):                                   # (1) 1024 fused single-query scans, ~2 ms each
            one = full_engine.search(c3_queries[i], 10)
            assert [g[0] for g in one] == ids[i].tolist(), i
            assert np.array_equal(np.float32([g[1] for g in one]).view(np.uint32), scores[i].view(np.uint32)), i
    finally:
        full_engine.set_option("batch_tensor", 1)
    sample, rows, s = c3_oracle_top100                          # (2)
    for j, qi in enumerate(sample):
        assert ids[qi].tolist() == rows[j][:10].tolist(), qi
        assert np.array_equal(scores[qi].view(np.uint32), s[j][:10].view(np.uint32)), qi
    four = sample[:4]                                           # (3) full fp64 scan for four of them
    _check_against_f64(oracle, oracle.COSINE, SEED, N_FULL, DIMS, True, c3_queries[four], 10,
                       [ids[i] for i in four], [scores[i] for i in four])


def test_full_size_filtered_batch_and_large_k_batch_against_the_oracle_top100(oracle, full_engine, c3_queries, c3_oracle_top100):
    """At 10 M x 384, against the oracle's COMPLETE top-100 of the sampled queries: (1) one deny-list for the whole
    1024-query batch (the five best rows of every sampled query): the filtered batch must return, for each sampled query,
    exactly the oracle list with the denied rows struck out -- ids and score bits; (2) a batch with k = 200 (tensor levels:
    nominee threshold + filter level) must carry the oracle's top-100 as its first hundred rows."""
    sample, rows, s = c3_oracle_top100
    deny = np.unique(np.concatenate([rows[j][:5] for j in range(len(sample))])).astype(np.uint64)   # implicit ids = rows
    denied = set(deny.tolist())
    t0, f0 = full_engine.batch_stats()
    got = full_engine.search_batch_filtered(c3_queries, 10, deny=deny)
    t1, f1 = full_engine.batch_stats()
    assert (t1 - t0) + (f1 - f0) == 1024 and f1 - f0 <= 10
    for j, qi in enumerate(sample):
        keep = [i for i in range(100) if int(rows[j][i]) not in denied][:10]
        assert [g[0] for g in got[qi]] == [int(rows[j][i]) for i in keep], qi
        assert np.array_equal(np.float32([g[1] for g in got[qi]]).view(np.uint32), s[j][keep].view(np.uint32)), qi
    qs = c3_queries[sample]
    t0, f0 = full_engine.batch_stats()
    ids, scores, ns = full_engine.search_batch_arrays(qs, 200)
    t1, f1 = full_engine.batch_stats()
    assert (t1 - t0) + (f1 - f0) == len(sample) and f1 - f0 <= 1, "the k = 200 batch did not take the tensor levels"
    assert ns.tolist() == [200] * len(sample)
    for j in range(len(sample)):
        assert ids[j][:100].tolist() == rows[j].tolist(), j
        assert np.array_equal(scores[j][:100].view(np.uint32), s[j].view(np.uint32)), j
        assert np.all(scores[j][:-1] >= scores[j][1:])


def test_config4_full_size_10m_x_768_batch_256_top100_dot(oracle):
    """BASELINE configs[4] at its stated size: 10 M x 768 fp32 rows that are NOT normalised, batch 256, top-100 under
    the dot metric (USearch ip: d = 1 - q.v, score = q.v - 1, VectorMetric.swift:21-43).  Same three checks."""
    n, dims, seed, b, k = 10_000_000, 768, 5, 256, 100
    eng = CUDAVectorEngine(VectorMetric.dot, dims)
    try:
        eng.fill_synthetic(seed, n, normalize=False)
        qs = oracle.synth_rows(1011, 0, b, dims, normalize=True)
        t0, f0 = eng.batch_stats()
        ids, scores, ns = eng.search_batch_arrays(qs, k)
        t1, f1 = eng.batch_stats()
        assert ns.tolist() == [k] * b
        assert (t1 - t0) + (f1 - f0) == b, "the batch did not take the tensor path"
        assert eng.counter("batch_bf16_queries") == b
        assert f1 - f0 <= 4, f"{f1 - f0} of {b} queries fell back to the exact scan"
        eng.set_option("batch_tensor", 0)
        for i in range(b):                                      # whole batch == fused single-query scan (k = 100)
            one = eng.search(qs[i], k)
            assert [g[0] for g in one] == ids[i].tolist(), i
            assert np.array_equal(np.float32([g[1] for g in one]).view(np.uint32), scores[i].view(np.uint32)), i
        eng.set_option("batch_tensor", 1)
        sample = list(range(0, b, b // 8))[:8]
        rows, d, s, cnt = oracle.search_synth_multi(oracle.DOT, seed, 0, n, dims, False, qs[sample], k,
                                                    mode=oracle.ACC_F32_TREE, threads=oracle.host_threads())
        assert cnt.tolist() == [k] * 8
        for j, qi in enumerate(sample):
            assert ids[qi].tolist() == rows[j].tolist(), qi
            assert np.array_equal(scores[qi].view(np.uint32), s[j].view(np.uint32)), qi
            assert np.array_equal(scores[qi], -d[j])            # score = -(1 - q.v)
        two = sample[:2]
        _check_against_f64(oracle, oracle.DOT, seed, n, dims, False, qs[two], k, [ids[i] for i in two],
                           [scores[i] for i in two])
    finally:
        eng.close()


def test_full_size_planted_neighbours_are_found(oracle, full_engine):
    """Rows built to be the query's nearest neighbours must come back first, in the planted order, wherever
    they sit in the 15 GB stream (first row, a middle row, the last row)."""
    q = oracle.synth_row(1003, 0, DIMS, True)
    rng = np.random.default_rng(0)
    planted = {}
    for rank, row in enumerate((N_FULL - 1, 0, 4_999_999, 7_777_777)):
        noise = rng.standard_normal(DIMS).astype(np.float32)
        planted[row] = (q + np.float32(0.02 * (rank + 1)) * noise / np.linalg.norm(noise)).astype(np.float32)
    before = full_engine.search(q, 10)
    full_engine.add_batch(list(planted), np.stack(list(planted.values())))     # upsert in place (ids == rows)
    assert full_engine.count == N_FULL
    got = full_engine.search(q, 10)
    assert [g[0] for g in got[:4]] == list(planted)
    assert [g for g in got[4:]] == [b for b in before if b[0] not in planted][:6]
    for (fid, score), vec in zip(got[:4], planted.values()):
        assert abs(score - (1.0 - oracle.distance(oracle.COSINE, oracle.ACC_F64, q, vec))) <= 1e-4
    full_engine.fill_synthetic(SEED, N_FULL)                                    # restore for other tests


def test_shard_invariance_through_the_device_entry_point(oracle):
    """Three engines holding contiguous shards + wax_vs_search_device + the host merge give exactly the
    single-engine answer (what the NCCL all-gather path computes, here inside one process)."""
    import torch
    from wax_b200 import _lib as L
    total, k = 300_007, 10
    q = oracle.synth_row(1004, 0, DIMS, True)
    single = CUDAVectorEngine(VectorMetric.cosine, DIMS)
    single.fill_synthetic(9, total)
    expect = single.search(q, k)
    d_q = torch.from_numpy(q).cuda()
    parts = []
    for r in range(3):
        lo, hi = sharded.shard_range(total, 3, r)
        eng = CUDAVectorEngine(VectorMetric.cosine, DIMS)
        eng.fill_synthetic(9, hi - lo, first_row=lo, id_base=lo)
        buf = torch.zeros(k * 24, dtype=torch.uint8, device="cuda")
        rc = L.lib().wax_vs_search_device(eng.handle, C.c_void_p(d_q.data_ptr()), 1, k, lo, C.c_void_p(buf.data_ptr()),
                                          C.c_void_p(torch.cuda.current_stream().cuda_stream))
        assert rc == 0, L.last_error()
        torch.cuda.synchronize()
        parts.append(buf.cpu().numpy().view(sharded.CAND_DTYPE).copy())
    best = sharded.merge_candidates(np.concatenate(parts), k)
    scores = sharded.score_from_distance(0, best["distance"])
    assert [(int(i), float(s)) for i, s in zip(best["frame_id"], scores)] == expect
    assert best["row"].tolist() == [e[0] for e in expect]          # id_base == shard offset -> id == global row


def test_single_rank_sharded_engine(oracle):
    """ShardedVectorEngine with world_size 1 (no process group): same answer as the plain engine."""
    import torch
    eng = sharded.ShardedVectorEngine(VectorMetric.cosine, DIMS, total_rows=100_000)
    eng.fill_synthetic(11)
    q = oracle.synth_row(1005, 0, DIMS, True)
    got = eng.search(q, 10)
    rows, _, s = oracle.search_synth(oracle.COSINE, 11, 0, 100_000, DIMS, True, q, 10, mode=oracle.ACC_F32_TREE, threads=8)
    assert [g[0] for g in got] == rows.tolist() and np.array_equal(np.float32([g[1] for g in got]), s)


def test_single_rank_micro_batched_exchange(oracle):
    """search_many_async: several queries, one exchange -- same answers as one query at a time."""
    import torch
    eng = sharded.ShardedVectorEngine(VectorMetric.cosine, DIMS, total_rows=60_000)
    eng.fill_synthetic(12)
    qs = oracle.synth_rows(1006, 0, 5, DIMS)
    d_qs = torch.from_numpy(qs).cuda()
    many = eng.finish_many(eng.search_many_async(d_qs, 10, slot=0))
    assert many == [eng.search(q, 10) for q in qs]
    h1 = eng.search_many_async(d_qs[:2], 10, slot=0)
    h2 = eng.search_many_async(d_qs[2:], 10, slot=1)             # two micro-batches in flight
    assert eng.finish_many(h1) + eng.finish_many(h2) == many


def test_single_rank_sharded_search_batch(oracle):
    """ShardedVectorEngine.search_batch (wax_vs_search_batch_device + vectorised merge): identical to one query at a
    time, through the tensor-core levels (the counters say so), with a shard offset in the global rows."""
    import torch
    eng = sharded.ShardedVectorEngine(VectorMetric.cosine, DIMS, total_rows=90_000)
    eng.fill_synthetic(13)
    qs = oracle.synth_rows(1007, 0, 140, DIMS)
    one_by_one = [eng.search(q, 10) for q in qs]
    assert eng.search_batch(qs, 10) == one_by_one
    assert eng.engine.counter("batch_bf16_queries") == 140
    assert eng.search_batch(torch.from_numpy(qs).cuda(), 10) == one_by_one      # device-resident queries
    # global rows: a second engine holding the same rows as rows [50_000, 140_000) of a larger corpus
    eng.row_lo, eng.row_hi = 50_000, 140_000
    ids, scores, ns = eng.search_batch_arrays(qs[:8], 10)
    assert ns.tolist() == [10] * 8 and [int(i) for i in ids[0]] == [g[0] for g in one_by_one[0]]   # frame ids unchanged
    assert np.array_equal(scores[0], np.float32([g[1] for g in one_by_one[0]]))
    # pipelined form: two batches in flight on the worker thread, same answers
    eng.row_lo, eng.row_hi = 0, 90_000
    h1 = eng.search_batch_submit(qs[:70], 10)
    h2 = eng.search_batch_submit(torch.from_numpy(qs[70:]).cuda(), 10)
    i1, s1, n1 = eng.finish_batch(h1)
    i2, s2, n2 = eng.finish_batch(h2)
    got = [[(int(i), float(s)) for i, s in zip(ii, ss)] for ii, ss in zip(np.concatenate([i1, i2]), np.concatenate([s1, s2]))]
    assert got == one_by_one and n1.tolist() == [10] * 70 and n2.tolist() == [10] * 70
    # k larger than the shard: padded by the scan path
    tiny = sharded.ShardedVectorEngine(VectorMetric.cosine, DIMS, total_rows=6)
    tiny.fill_synthetic(14)
    got = tiny.search_batch(qs[:5], 10)
    assert [len(g) for g in got] == [6] * 5 and got == [tiny.search(q, 10) for q in qs[:5]]
