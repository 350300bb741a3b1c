"""GPU: the single-query bf16-shadow route (DESIGN 4.1) must answer exactly as the fp32 scan does.

A single cosine / dot query with k <= 32 on a large corpus is nominated by the SHADOW form of the streaming scan (the
bf16 copy of the corpus, half the bytes), re-scored exactly and proven by the batched path's finish kernel, and the fp32
scan that follows is guarded by that proof: it returns at entry when the proof held and answers the query when it
failed.  Every answer here is compared with the fp32 scan forced by the `shadow_scan = 0` option, ids and score bits;
samples are compared with the CPU oracle (ACC_F32_TREE).  The counters say which route answered: single_shadow_queries
(the proof held) and single_shadow_fallbacks (the fp32 scan answered after a failed proof).
"""
import ctypes as C

import numpy as np
import pytest

from helpers import hidden_winner, unit_rows
from test_gpu_degenerate_queries import cosine_corpus, degenerate_queries, positive_rows
from wax_b200 import CUDAVectorEngine, VectorMetric

pytestmark = pytest.mark.gpu

COS, DOT = VectorMetric.cosine, VectorMetric.dot
SKIP = 16           # eligible queries that take the fp32 scan directly after a failed proof


def bits(hits):
    return [(i, int(np.float32(s).view(np.uint32))) for i, s in hits]


def counts(eng):
    return eng.counter("single_shadow_queries"), eng.counter("single_shadow_fallbacks")


def fp32(eng, call):
    """call() on the fp32 scan alone (the route switched off); switching it back on also clears the skip window."""
    eng.set_option("shadow_scan", 0)
    try:
        return call()
    finally:
        eng.set_option("shadow_scan", 1)


def routed(eng, call, proven=1, failed=0):
    """call() on the default path; asserts how many queries the route answered and how many its proof refused."""
    q0, f0 = counts(eng)
    out = call()
    q1, f1 = counts(eng)
    assert (q1 - q0, f1 - f0) == (proven, failed), f"route answered {q1 - q0}, refused {f1 - f0}"
    return out


def engine_synth(metric, n, dims, seed):
    eng = CUDAVectorEngine(metric, dims)
    eng.fill_synthetic(seed, n, normalize=metric is COS)
    eng.set_option("shadow_scan_min_bytes", 0)
    return eng


def engine_rows(metric, corpus, min_bytes=0):
    eng = CUDAVectorEngine(metric, corpus.shape[1])
    eng.add_batch(list(range(corpus.shape[0])), corpus)
    eng.set_option("shadow_scan_min_bytes", min_bytes)
    return eng


def check_oracle(oracle, metric, eng, n, q, k, got):
    corpus = eng.read_rows(0, n)
    r, _, s = oracle.search(metric.value, corpus, q, k, mode=oracle.ACC_F32_TREE, threads=8)
    assert bits(got) == list(zip(r.tolist(), s.view(np.uint32).tolist()))


@pytest.mark.parametrize("n", [1, 127, 128, 129, 50_001])
@pytest.mark.parametrize("dims", [128, 384, 768, 1536])
@pytest.mark.parametrize("metric", [COS, DOT])
def test_route_equals_fp32_scan(oracle, metric, dims, n):
    eng = engine_synth(metric, n, dims, seed=300 + dims + n % 7)
    qs = oracle.synth_rows(301 + dims, 0, 3, dims, normalize=True)
    for k in (1, 10, 32):
        want = fp32(eng, lambda: [eng.search(q, k) for q in qs])
        got = routed(eng, lambda: [eng.search(q, k) for q in qs], proven=len(qs))
        assert [bits(g) for g in got] == [bits(w) for w in want], f"k={k}"
        assert len(got[0]) == min(k, n)
    check_oracle(oracle, metric, eng, n, qs[0], 10, eng.search(qs[0], 10))
    eng.close()


@pytest.mark.parametrize("metric", [COS, DOT])
def test_route_at_one_million_rows(oracle, metric):
    eng = engine_synth(metric, 1_000_000, 384, seed=310)
    qs = oracle.synth_rows(311, 0, 4, 384, normalize=True)
    for k in (1, 10, 32):
        want = fp32(eng, lambda: [eng.search(q, k) for q in qs])
        got = routed(eng, lambda: [eng.search(q, k) for q in qs], proven=len(qs))
        assert [bits(g) for g in got] == [bits(w) for w in want], f"k={k}"
    ms, launches = eng.time_search(10, 8, warmup=2, n_queries=4, seed=312)
    assert ms > 0 and launches == 3 * 8           # shadow scan, finish, guarded scan
    eng.close()


@pytest.mark.parametrize("metric", [COS, DOT])
def test_filtered_single_queries(oracle, metric):
    n, dims = 200_000, 384
    eng = engine_synth(metric, n, dims, seed=320)
    rng = np.random.default_rng(321)
    deny = np.sort(rng.choice(n, 30_000, replace=False)).tolist()
    allow = np.sort(rng.choice(n, 40_000, replace=False)).tolist()      # above the gather size: the row bitset
    qs = oracle.synth_rows(322, 0, 3, dims, normalize=True)
    for kind, fids in (("deny", deny), ("allow", allow)):
        for k in (1, 10, 32):
            want = fp32(eng, lambda: [eng.search_filtered(q, k, **{kind: fids}) for q in qs])
            got = routed(eng, lambda: [eng.search_filtered(q, k, **{kind: fids}) for q in qs], proven=len(qs))
            assert [bits(g) for g in got] == [bits(w) for w in want], (kind, k)
    top = eng.search_filtered(qs[0], 10, deny=[g[0] for g in eng.search(qs[0], 5)])
    assert bits(top[:5]) == bits(eng.search(qs[0], 10)[5:])
    eng.close()


def test_delivery_modes_and_search_device(oracle):
    import torch
    from wax_b200 import _lib as L, sharded
    n, dims, k = 300_000, 384, 10
    eng = engine_synth(COS, n, dims, seed=330)
    qs = oracle.synth_rows(331, 0, 3, dims, normalize=True)
    want = fp32(eng, lambda: [eng.search(q, k) for q in qs])
    for delivery in (1, 0):
        for inline in (1, 0):
            eng.set_option("host_delivery", delivery); eng.set_option("inline_query", inline)
            got = routed(eng, lambda: [eng.search(q, k) for q in qs], proven=len(qs))
            assert [bits(g) for g in got] == [bits(w) for w in want], (delivery, inline)
    stream = torch.cuda.Stream()
    d_q = torch.from_numpy(qs).cuda()
    buf = torch.zeros(len(qs) * k * 24, dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()
    q0, f0 = counts(eng)
    rc = L.lib().wax_vs_search_device(eng.handle, C.c_void_p(d_q.data_ptr()), len(qs), k, 0, C.c_void_p(buf.data_ptr()),
                                      C.c_void_p(stream.cuda_stream))
    assert rc == 0, L.last_error()
    stream.synchronize()
    assert counts(eng) == (q0 + len(qs), f0)
    cands = buf.cpu().numpy().view(sharded.CAND_DTYPE).reshape(len(qs), k)
    for c, w in zip(cands, want):
        assert [int(x["frame_id"]) for x in c] == [i for i, _ in w]
        assert [float(np.float32(1.0) - x["distance"]) for x in c] == [s for _, s in w]
    eng.close()


def assert_refused_then_skip_window(eng, q, k, ordinary, want_q, want_ordinary):
    """q is refused (answered by the fp32 scan, counted), the next SKIP eligible queries take the fp32 scan directly,
    then the route is probed again."""
    assert len(ordinary) == SKIP + 1
    got = routed(eng, lambda: eng.search(q, k), proven=0, failed=1)
    assert bits(got) == bits(want_q)
    got = routed(eng, lambda: [eng.search(o, k) for o in ordinary[:SKIP]], proven=0, failed=0)
    assert [bits(g) for g in got] == [bits(w) for w in want_ordinary[:SKIP]]
    q0, f0 = counts(eng)
    assert bits(eng.search(ordinary[SKIP], k)) == bits(want_ordinary[SKIP])
    q1, f1 = counts(eng)
    assert (q1 - q0) + (f1 - f0) == 1, "the route was not probed again after the skip window"


def test_ties_are_refused(oracle):
    """All-ones rows (every row ties) and period-256 duplicates (each row ~200 times): the k' nominees all tie with the
    k-th result, nothing can be excluded, the fp32 scan answers."""
    dims, n, k = 384, 50_000, 10
    rng = np.random.default_rng(340)
    base = unit_rows(rng, 256, dims)
    for corpus in (np.ones((n, dims), np.float32), base[np.arange(n) % 256]):
        eng = engine_rows(COS, corpus)
        q = base[3] + np.float32(0.01) * unit_rows(rng, 1, dims)[0]
        ordinary = unit_rows(rng, SKIP + 1, dims)
        want_q = fp32(eng, lambda: eng.search(q, k))
        want_o = fp32(eng, lambda: [eng.search(o, k) for o in ordinary])
        assert_refused_then_skip_window(eng, q, k, ordinary, want_q, want_o)
        if corpus[0, 0] == 1.0:
            assert [i for i, _ in want_q] == list(range(k))
        eng.close()


def test_hidden_winner_is_refused(oracle):
    """The best row's score' rounds below 140 decoys (more than the 128 nominees): it is never nominated, and the bound
    is too wide to exclude it -- the fp32 scan returns it."""
    dims, n = 256, 20_000
    rng = np.random.default_rng(350)
    q, corpus = hidden_winner(rng, dims, n, True, n_decoys=140)
    eng = engine_rows(DOT, corpus)
    ordinary = unit_rows(rng, SKIP + 1, dims)
    want_q = fp32(eng, lambda: eng.search(q[0], 1))
    want_o = fp32(eng, lambda: [eng.search(o, 1) for o in ordinary])
    assert want_q[0][0] == 0
    assert_refused_then_skip_window(eng, q[0], 1, ordinary, want_q, want_o)
    eng.close()


def test_huge_dot_rows_are_refused(oracle):
    """A dot row of |v| ~ 1e20 far below every result widens the bound (it scales with the largest row norm) past every
    gap: the proof refuses and the fp32 scan answers."""
    dims, n, k = 384, 30_000, 10
    rng = np.random.default_rng(360)
    corpus = positive_rows(rng, n, dims)
    corpus[777] = -corpus[777] * np.float32(1e20)
    eng = engine_rows(DOT, corpus)
    q = positive_rows(rng, 1, dims)[0]
    ordinary = positive_rows(rng, SKIP + 1, dims)
    want_q = fp32(eng, lambda: eng.search(q, k))
    want_o = fp32(eng, lambda: [eng.search(o, k) for o in ordinary])
    assert_refused_then_skip_window(eng, q, k, ordinary, want_q, want_o)
    eng.close()


@pytest.mark.parametrize("metric", [COS, DOT])
def test_degenerate_queries_and_rows(oracle, metric):
    """The degenerate queries (zero, subnormal and overflowing |q|^2, NaN and +-Inf components) and, for cosine, rows
    whose sum v^2 is zero, subnormal or overflows: the fp32 scan's answers, whichever route gives them."""
    dims, n, k = 384, 40_000, 10
    rng = np.random.default_rng(370 + metric.value)
    ordinary = positive_rows(rng, 4, dims)
    if metric is COS:
        corpus = cosine_corpus(rng, n, dims, ordinary)
    else:
        corpus = positive_rows(rng, n, dims) * np.float32(10.0) ** rng.uniform(-1, 1, (n, 1)).astype(np.float32)
    names, deg = degenerate_queries(rng, dims)
    qs = np.concatenate([ordinary, deg])
    labels = ["ordinary"] * len(ordinary) + names
    eng = engine_rows(metric, corpus)
    want = fp32(eng, lambda: [eng.search(q, k) for q in qs])
    for name, q, w in zip(labels, qs, want):
        eng.set_option("shadow_scan", 1)           # clears the skip window a refused query opens
        q0, f0 = counts(eng)
        assert bits(eng.search(q, k)) == bits(w), name
        q1, f1 = counts(eng)
        assert (q1 - q0) + (f1 - f0) == 1, f"{name} did not take the route"
        if name in ("zero", "nan_component", "pos_inf_component", "a2_overflow"):
            assert f1 - f0 == 1, f"{name}: a proof was claimed for a query whose fp32 |q|^2 cannot bound the error"
    got = [eng.search(q, k) for q in ordinary]
    check_oracle(oracle, metric, eng, n, ordinary[0], k, got[0])
    eng.close()


def test_shadow_follows_appends_removes_and_overwrites(oracle):
    dims, n, k = 384, 60_000, 10
    eng = engine_synth(COS, n, dims, seed=380)
    qs = oracle.synth_rows(381, 0, 3, dims, normalize=True)

    def same(rows, proven=3):
        want = fp32(eng, lambda: [eng.search(q, k) for q in qs])
        got = routed(eng, lambda: [eng.search(q, k) for q in qs], proven=proven)
        assert [bits(g) for g in got] == [bits(w) for w in want]
        assert eng.counter("shadow_rows") == rows
        return got

    same(n)
    extra = np.stack([qs[0], qs[1] * np.float32(2.0)] + list(unit_rows(np.random.default_rng(382), 98, dims)))
    eng.add_batch(list(range(10**6, 10**6 + 100)), extra)
    assert eng.counter("shadow_rows") == n                  # the valid prefix stays: the append extends it
    got = same(n + 100)
    assert got[0][0][0] == 10**6 and got[1][0][0] == 10**6 + 1
    eng.remove(10**6)
    same(n + 99)
    eng.add(5, qs[2])                                        # overwrite in place
    got = same(n + 99)
    assert got[2][0][0] == 5
    eng.close()


def test_ineligible_searches_take_the_fp32_scan(oracle):
    """No route for: batch_bf16 = 0, k > 32, corpora below the size threshold, l2."""
    dims, n = 384, 100_000
    eng = engine_synth(COS, n, dims, seed=390)
    qs = oracle.synth_rows(391, 0, 2, dims, normalize=True)
    want = fp32(eng, lambda: [eng.search(q, 10) for q in qs])
    eng.set_option("batch_bf16", 0)
    assert routed(eng, lambda: [eng.search(q, 10) for q in qs], proven=0) == want
    eng.set_option("batch_bf16", 1)
    want72 = fp32(eng, lambda: eng.search(qs[0], 72))
    assert routed(eng, lambda: eng.search(qs[0], 72), proven=0) == want72
    eng.set_option("shadow_scan_min_bytes", n * dims * 4 + 1)
    assert routed(eng, lambda: [eng.search(q, 10) for q in qs], proven=0) == want
    eng.set_option("shadow_scan_min_bytes", n * dims * 4)
    assert routed(eng, lambda: [eng.search(q, 10) for q in qs], proven=2) == want
    eng.close()
    l2 = engine_synth(VectorMetric.l2, 20_000, dims, seed=392)
    want = fp32(l2, lambda: l2.search(qs[0], 10))
    assert routed(l2, lambda: l2.search(qs[0], 10), proven=0) == want
    l2.close()
