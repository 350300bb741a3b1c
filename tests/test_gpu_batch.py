"""GPU: the batched path (wgmma TF32 / bf16 nomination + exact fp32 re-score + completeness proof) must return
EXACTLY what the single-query path returns -- same ids, same score bits -- and must actually be the tensor path
(the instrumentation counts queries answered with a completed proof vs. re-run exactly)."""
import numpy as np
import pytest

from wax_b200 import CUDAVectorEngine, VectorMetric

pytestmark = pytest.mark.gpu


# Cosine over rows whose norms spread over 1e-3 .. 1e3: the TF32 epilogue's per-row 1/|v| and the pre-normalised bf16
# shadow rows then differ from row to row (synthetic cosine corpora are unit rows, where a misplaced scale is invisible).
MIXED = "cosine_mixed_norms"


def _metric(metric):
    return VectorMetric.cosine if metric == MIXED else metric


def _engine(oracle, metric, n, dims, seed, normalize=True):
    if metric == MIXED:
        corpus = oracle.synth_rows(seed, 0, n, dims, normalize=True)
        corpus *= np.float32(10.0) ** np.random.default_rng(seed).uniform(-3, 3, (n, 1)).astype(np.float32)
        eng = CUDAVectorEngine(VectorMetric.cosine, dims)
        eng.add_batch(list(range(n)), corpus)
        return eng
    eng = CUDAVectorEngine(metric, dims)
    eng.fill_synthetic(seed, n, normalize=normalize)
    return eng


def _single(eng, qs, k):
    eng.set_option("batch_tensor", 0)
    out = [eng.search(q, k) for q in qs]
    eng.set_option("batch_tensor", 1)
    return out


@pytest.mark.parametrize("dims,n,b,k", [(384, 100_003, 5, 10), (384, 100_003, 129, 10), (384, 50_000, 300, 72),
                                        (768, 30_001, 64, 100), (128, 70_000, 17, 32), (32, 9_999, 8, 1),
                                        (384, 255, 6, 10), (384, 257, 6, 10), (384, 1, 4, 10), (1024, 20_000, 33, 10)])
@pytest.mark.parametrize("metric", [VectorMetric.cosine, VectorMetric.dot, MIXED])
@pytest.mark.parametrize("bf16", [1, 0])
def test_batch_equals_single_query_path(oracle, metric, dims, n, b, k, bf16):
    eng = _engine(oracle, metric, n, dims, seed=900 + dims, normalize=(metric is VectorMetric.cosine))
    eng.set_option("batch_bf16", bf16)      # 1 (the default): bf16 shadow nominations where dims % 64 == 0; 0: TF32
    qs = oracle.synth_rows(901 + b, 0, b, dims, normalize=True)
    t0, f0 = eng.batch_stats()
    got = eng.search_batch(qs, k)
    t1, f1 = eng.batch_stats()
    assert (t1 - t0) + (f1 - f0) == b, "the batch did not go through the tensor path"
    exp = _single(eng, qs, k)
    assert got == exp
    # random data: the proof completes for (nearly) every query -- otherwise the tensor path is not doing its job
    if n >= 1000:
        assert f1 - f0 <= max(1, b // 50), f"{f1 - f0} of {b} queries fell back to the exact path"
    # and the single-query path is itself bit-exact against the oracle (spot check one query)
    corpus = eng.read_rows(0, n)
    r, d, s = oracle.search(_metric(metric).value, corpus, qs[0], k, mode=oracle.ACC_F32_TREE, threads=4)
    assert [g[0] for g in got[0]] == r.tolist()
    assert np.array_equal(np.float32([g[1] for g in got[0]]).view(np.uint32), s.view(np.uint32))


def test_batch_with_near_duplicates_stays_exact(oracle):
    """Adversarial for TF32: thousands of rows within 1e-5 of the query's best match.  The proof cannot complete
    (TF32 cannot separate them), so those queries are re-run exactly -- results still identical."""
    dims, n = 384, 20_000
    rng = np.random.default_rng(3)
    base = oracle.synth_row(77, 0, dims, True)
    corpus = oracle.synth_rows(78, 0, n, dims)
    corpus[:3000] = base + rng.standard_normal((3000, dims)).astype(np.float32) * np.float32(1e-6)
    eng = CUDAVectorEngine(VectorMetric.cosine, dims)
    eng.add_batch(list(range(n)), corpus)
    qs = np.stack([base, oracle.synth_row(79, 0, dims, True), base * np.float32(2.5), corpus[5000]])
    got = eng.search_batch(qs, 10)
    assert got == _single(eng, qs, 10)
    r, _, s = oracle.search(oracle.COSINE, corpus, qs[0], 10, mode=oracle.ACC_F32_TREE, threads=4)
    assert [g[0] for g in got[0]] == r.tolist()
    # the adversarial queries could not be proven at level 1: they were answered by a filter pass or by the exact scan
    assert eng.batch_stats()[1] + eng.counter("batch_filter_bf16_queries") + eng.counter("batch_retry_queries") >= 1


def test_batch_edge_rows_and_mutation_invalidates_norm_cache(oracle):
    dims = 384
    corpus = oracle.synth_rows(80, 0, 4000, dims)
    corpus[7] = 0.0
    corpus[8, 5] = np.nan
    corpus[9, 6] = np.inf
    eng = CUDAVectorEngine(VectorMetric.cosine, dims)
    eng.add_batch(list(range(4000)), corpus)
    qs = oracle.synth_rows(81, 0, 6, dims)
    assert eng.search_batch(qs, 10) == _single(eng, qs, 10)
    # mutate: scale a row by 1000 (norm changes a lot) and append rows; cached norms must be rebuilt
    eng.add(11, corpus[11] * np.float32(1000.0))
    eng.add_batch([5000, 5001], np.stack([qs[0], qs[1] * np.float32(3.0)]))
    eng.remove(3)
    got = eng.search_batch(qs, 10)
    assert got == _single(eng, qs, 10)
    assert got[0][0][0] == 5000 and got[1][0][0] == 5001
    assert 8 not in [i for i, _ in eng.search_batch(qs, 4000)[0]]


def test_batch_edge_rows_and_mutation_invalidates_norm_cache_dot(oracle):
    """The same edge rows and mutations for dot, whose proof bound scales with the corpus' max |v| (cached with the
    norms): overwriting a row with a larger norm must raise that bound, so the level-1 proofs it allowed are refused."""
    dims = 384
    corpus = oracle.synth_rows(80, 0, 4000, dims)
    corpus[7] = 0.0
    corpus[8, 5] = np.nan
    corpus[9, 6] = np.inf
    eng = CUDAVectorEngine(VectorMetric.dot, dims)
    eng.add_batch(list(range(4000)), corpus)
    qs = oracle.synth_rows(81, 0, 6, dims)
    assert eng.search_batch(qs, 10) == _single(eng, qs, 10)
    ok_before = eng.batch_nominations(qs, 10)["ok"]
    assert ok_before.sum() >= 3, ok_before          # unit rows: max|v| = 1 proves most queries at level 1
    eng.add(11, corpus[11] * np.float32(1000.0))
    ok_after = eng.batch_nominations(qs, 10)["ok"]
    assert ok_after.sum() == 0, ok_after            # max|v| = 1000 now: eps ~ 8 |q|, nothing is provable
    eng.add_batch([5000, 5001], np.stack([qs[0], qs[1] * np.float32(3.0)]))
    eng.remove(3)
    got = eng.search_batch(qs, 10)
    assert got == _single(eng, qs, 10)
    assert 8 not in [i for i, _ in eng.search_batch(qs, 4000)[0]]


def test_ineligible_batches_use_the_loop(oracle):
    eng = _engine(oracle, VectorMetric.l2, 5000, 384, seed=5)
    qs = oracle.synth_rows(82, 0, 9, 384)
    t0, f0 = eng.batch_stats()
    assert eng.search_batch(qs, 10) == [eng.search(q, 10) for q in qs]     # l2: not on the tensor path
    eng2 = _engine(oracle, VectorMetric.cosine, 5000, 100, seed=6)         # dims % 32 != 0
    qs2 = oracle.synth_rows(83, 0, 9, 100)
    assert eng2.search_batch(qs2, 10) == [eng2.search(q, 10) for q in qs2]
    assert eng.batch_stats() == (t0, f0) and eng2.batch_stats() == (0, 0)


@pytest.mark.parametrize("dims,n,b,k", [(384, 100_003, 256, 10), (384, 100_003, 300, 10), (768, 30_001, 200, 100),
                                        (384, 50_000, 1024, 72), (128, 257, 129, 10)])
@pytest.mark.parametrize("metric", [VectorMetric.cosine, VectorMetric.dot, MIXED])
def test_cta_pair_mode_equals_single_query_path(oracle, metric, dims, n, b, k):
    """CTA-pair shape (two CTAs of a cluster, one row slice; each loads half of every corpus tile and multicasts it
    into both): same nominees -> same proof -> identical results."""
    eng = _engine(oracle, metric, n, dims, seed=950 + dims, normalize=(metric is VectorMetric.cosine))
    eng.set_option("batch_bf16", 0)
    eng.set_option("batch_pair", 1)
    qs = oracle.synth_rows(951 + b, 0, b, dims, normalize=True)
    t0, f0 = eng.batch_stats()
    got = eng.search_batch(qs, k)
    t1, f1 = eng.batch_stats()
    assert (t1 - t0) + (f1 - f0) == b
    assert got == _single(eng, qs, k)
    if n >= 1000:
        assert f1 - f0 <= max(1, b // 50), f"{f1 - f0} of {b} queries fell back to the exact path"


@pytest.mark.parametrize("dims,n,b,k", [(384, 100_003, 256, 10), (384, 100_003, 300, 10), (768, 30_001, 200, 100),
                                        (384, 50_000, 1024, 72), (128, 257, 129, 10), (64, 9_999, 8, 1),
                                        (512, 40_000, 140, 32), (384, 1, 4, 10), (1024, 20_000, 33, 10)])
@pytest.mark.parametrize("metric", [VectorMetric.cosine, VectorMetric.dot, MIXED])
@pytest.mark.parametrize("pair,ares", [(0, 1), (0, 0), (1, 1), (1, 0)])
def test_bf16_shadow_nominations_equal_single_query_path(oracle, metric, dims, n, b, k, pair, ares):
    """bf16 nominations (bf16 wgmmas over a bf16 shadow of the corpus, queries resident in shared memory or
    streamed, single CTA or a multicasting CTA pair): the nominees differ from the TF32 ones, the RESULTS may not -- the exact
    fp32 re-score and the completeness proof (with the coarser 2^-7 bound) make them identical to the single-query
    path, ids and score bits."""
    eng = _engine(oracle, metric, n, dims, seed=990 + dims, normalize=(metric is VectorMetric.cosine))
    eng.set_option("batch_bf16", 1)
    eng.set_option("batch_pair", pair)
    eng.set_option("batch_ares", ares)
    qs = oracle.synth_rows(991 + b, 0, b, dims, normalize=True)
    t0, f0 = eng.batch_stats()
    got = eng.search_batch(qs, k)
    t1, f1 = eng.batch_stats()
    assert (t1 - t0) + (f1 - f0) == b
    assert eng.counter("batch_bf16_queries") == b, "the batch was not nominated from the bf16 shadow"
    assert eng.counter("shadow_bytes") == n * dims * 2
    assert got == _single(eng, qs, k)
    if n >= 1000:
        assert f1 - f0 <= max(1, b // 50), f"{f1 - f0} of {b} queries fell back to the exact path"


@pytest.mark.parametrize("dims,n,b,k", [(768, 60_001, 256, 100), (384, 100_003, 130, 128), (64, 9_999, 8, 1)])
@pytest.mark.parametrize("metric", [VectorMetric.cosine, VectorMetric.dot])
def test_bf16_mid_heap_shape_equals_single_query_path(oracle, metric, dims, n, b, k):
    """24-entry heaps, streamed queries (bf16): a shape the cost model picks when k exceeds the slice count (configs[4]:
    top-100 over 66 slices).  Forced here; same answers as the single-query path, ids and score bits."""
    eng = _engine(oracle, metric, n, dims, seed=770 + dims, normalize=(metric is VectorMetric.cosine))
    eng.set_option("batch_bf16", 1)
    eng.set_option("batch_ares", 0)
    eng.set_option("batch_heap", 24)
    qs = oracle.synth_rows(771 + b, 0, b, dims, normalize=True)
    t0, f0 = eng.batch_stats()
    got = eng.search_batch(qs, k)
    t1, f1 = eng.batch_stats()
    assert (t1 - t0) + (f1 - f0) == b
    assert eng.counter("batch_bf16_queries") == b
    assert got == _single(eng, qs, k)
    if n >= 1000:
        assert f1 - f0 <= max(1, b // 50), f"{f1 - f0} of {b} queries fell back to the exact path"


def _planted(oracle, dims, n, n_planted, top, step, seed, stride):
    """Random unit corpus; row i*stride (i < n_planted) has cosine top - i*step to a unit query q.  The planted rows
    are spread out so that no row slice's 16-entry nominee heap fills up with them."""
    rng = np.random.default_rng(seed)
    q = oracle.synth_row(seed, 0, dims, True).astype(np.float64)
    q /= np.linalg.norm(q)
    corpus = oracle.synth_rows(seed + 1, 0, n, dims)
    for i in range(n_planted):
        r = rng.standard_normal(dims)
        r -= r.dot(q) * q
        r /= np.linalg.norm(r)
        c = top - i * step
        corpus[i * stride] = (c * q + np.sqrt(1.0 - c * c) * r).astype(np.float32)
    return q.astype(np.float32), corpus


def test_bf16_unproven_queries_retry_on_tf32_before_the_exact_scan(oracle):
    """600 planted neighbours 2e-5 apart: the 10th result clears the 257th nominee by 0.005 -- inside the bf16
    bound (0.008), outside the TF32 one (0.0025).  The bf16 pass must flag those queries, the TF32 retry must prove
    them, nothing reaches the exact scan, and the results are identical to the single-query path."""
    dims, n = 384, 60_000
    q, corpus = _planted(oracle, dims, n, 600, 0.95, 2e-5, seed=4100, stride=100)
    eng = CUDAVectorEngine(VectorMetric.cosine, dims)
    eng.add_batch(list(range(n)), corpus)
    eng.set_option("batch_bf16", 1)
    eng.set_option("filter_bf16", 0)      # this test is about the TF32 filter level; the bf16-shadow one is tested below
    qs = np.stack([q, q * np.float32(2.0), q * np.float32(0.5), q * np.float32(3.0), q * np.float32(1.5),
                   oracle.synth_row(4200, 0, dims, True)])
    t0, f0 = eng.batch_stats()
    got = eng.search_batch(qs, 10)
    t1, f1 = eng.batch_stats()
    assert got == _single(eng, qs, 10)
    assert [i for i, _ in got[0]] == [100 * i for i in range(10)]
    assert eng.counter("batch_retry_queries") >= 5
    assert f1 - f0 == 0, "the TF32 retry level should have proven every query"
    # adaptive level choice: most of that batch failed the bf16 bound, so the next batches start at TF32
    n_bf16 = eng.counter("batch_bf16_queries")
    assert eng.search_batch(qs, 10) == got
    assert eng.counter("batch_bf16_queries") == n_bf16
    assert eng.batch_stats()[1] - f0 == 0
    # retry disabled (setting batch_bf16 re-arms the bf16 level): the same queries go straight to the exact scan
    eng.set_option("batch_bf16", 1)
    eng.set_option("batch_retry", 0)
    got2 = eng.search_batch(qs, 10)
    assert got2 == got
    assert eng.counter("batch_bf16_queries") == n_bf16 + len(qs)
    assert eng.batch_stats()[1] - f0 >= 5


def test_unproven_queries_take_a_filter_pass_over_the_bf16_shadow_first(oracle):
    """Same planted neighbours.  By default the queries the bf16 nominations cannot prove get ONE filter pass over the
    bf16 shadow (half the bytes of an exact scan, so it is used even for a single unproven query): every row within
    the bf16 bound of the exact k-th score is listed and re-scored exactly -- complete by construction.  No TF32 pass,
    no exact scan, identical results; with a tiny candidate cap the lists overflow and the later levels answer."""
    dims, n = 384, 60_000
    q, corpus = _planted(oracle, dims, n, 600, 0.95, 2e-5, seed=4100, stride=100)
    eng = CUDAVectorEngine(VectorMetric.cosine, dims)
    eng.add_batch(list(range(n)), corpus)
    qs = np.stack([q, q * np.float32(2.0), q * np.float32(0.5), q * np.float32(3.0), q * np.float32(1.5),
                   oracle.synth_row(4200, 0, dims, True)])
    expect = _single(eng, qs, 10)
    t0, f0 = eng.batch_stats()
    assert eng.search_batch(qs, 10) == expect
    assert eng.counter("batch_filter_bf16_queries") >= 5 and eng.counter("batch_retry_queries") == 0
    assert eng.batch_stats()[1] - f0 == 0
    # ONE unprovable query in an otherwise easy batch: still the shadow filter pass, not a 2x more expensive exact scan
    eng.set_option("batch_bf16", 1)                       # re-arm the bf16 level (the adaptive choice suspended it)
    easy = oracle.synth_rows(4300, 0, 12, dims)
    mixed = np.concatenate([easy[:5], q[None, :], easy[5:]])
    b0 = eng.counter("batch_filter_bf16_queries")
    got = eng.search_batch(mixed, 10)
    assert got == _single(eng, mixed, 10) and got[5] == expect[0]
    assert eng.counter("batch_filter_bf16_queries") - b0 == 1 and eng.batch_stats()[1] - f0 == 0
    # overflow of the bf16 list -> TF32 filter (sub-batch large enough) -> exact scan: same answers
    eng.set_option("batch_bf16", 1)
    eng.set_option("filter_cap", 64)
    assert eng.search_batch(qs, 10) == expect
    assert eng.batch_stats()[1] - f0 >= 5


def test_bf16_shadow_follows_mutations(oracle):
    dims = 384
    corpus = oracle.synth_rows(85, 0, 6000, dims)
    corpus[7] = 0.0
    corpus[8, 5] = np.nan
    corpus[9, 6] = np.inf
    eng = CUDAVectorEngine(VectorMetric.cosine, dims)
    eng.add_batch(list(range(6000)), corpus)
    eng.set_option("batch_bf16", 1)
    qs = oracle.synth_rows(86, 0, 8, dims)
    assert eng.search_batch(qs, 10) == _single(eng, qs, 10)
    eng.add(11, corpus[11] * np.float32(1000.0))
    eng.add_batch([7000, 7001], np.stack([qs[0], qs[1] * np.float32(3.0)]))
    eng.remove(3)
    got = eng.search_batch(qs, 10)
    assert got == _single(eng, qs, 10)
    assert got[0][0][0] == 7000 and got[1][0][0] == 7001
    assert eng.counter("shadow_bytes") == 6001 * dims * 2


def test_single_shadow_mode_routes_single_queries_through_the_shadow(oracle):
    """Opt-in `single_shadow`: one query is ranked against the bf16 shadow on the tensor path, re-scored exactly and
    proven -- same ids and score bits as the fused fp32 scan; an unprovable query (near-duplicates) falls back to the
    scan and switches the mode off for the next queries (adaptive level choice)."""
    dims, n = 384, 80_000
    eng = _engine(oracle, VectorMetric.cosine, n, dims, seed=1200)
    qs = oracle.synth_rows(1201, 0, 5, dims)
    expect = [eng.search(q, 10) for q in qs]
    assert eng.counter("batch_bf16_queries") == 0
    eng.set_option("single_shadow", 1)
    assert [eng.search(q, 10) for q in qs] == expect
    assert eng.counter("batch_bf16_queries") == 5 and eng.batch_stats() == (5, 0)
    assert eng.search_batch(qs[:2], 10) == expect[:2]            # below batch_min: the shadow path as well
    assert eng.counter("batch_bf16_queries") == 7
    # k > 128 is not eligible: the scan answers
    got200 = eng.search(qs[0], 200)
    assert eng.counter("batch_bf16_queries") == 7
    eng.set_option("single_shadow", 0)
    assert got200 == eng.search(qs[0], 200)
    eng.set_option("single_shadow", 1)
    # near-duplicates of the query: unprovable at bf16 level 1 -> one filter pass over the shadow (400 candidates, still
    # half the bytes of the exact scan) answers it, identical result; the bf16 level is suspended for the next queries
    base = oracle.synth_row(1202, 0, dims, True)
    rng = np.random.default_rng(9)
    dup = base + rng.standard_normal((400, dims)).astype(np.float32) * np.float32(1e-6)
    eng.add_batch(list(range(400)), dup)
    eng.set_option("single_shadow", 0)
    want = eng.search(base, 10)
    eng.set_option("single_shadow", 1)
    n0 = eng.counter("batch_bf16_queries")
    assert eng.search(base, 10) == want
    assert eng.counter("batch_bf16_queries") == n0 + 1
    assert eng.batch_stats()[1] == 0 and eng.counter("batch_filter_bf16_queries") == 1
    assert eng.search(qs[1], 10) == expect[1]
    assert eng.counter("batch_bf16_queries") == n0 + 1          # suspended: answered by the fp32 scan


def _clustered(n, dims, n_centres, sigma, seed, normalize=True):
    rng = np.random.default_rng(seed)
    centres = rng.standard_normal((n_centres, dims)).astype(np.float32)
    centres /= np.linalg.norm(centres, axis=1, keepdims=True)
    corpus = centres[rng.integers(0, n_centres, n)] + np.float32(sigma / np.sqrt(dims)) * rng.standard_normal((n, dims)).astype(np.float32)
    if normalize:
        corpus /= np.linalg.norm(corpus, axis=1, keepdims=True)
    else:
        corpus *= rng.uniform(0.5, 2.0, size=(n, 1)).astype(np.float32)
    qs = corpus[rng.integers(0, n, 96)] + np.float32(0.2 / np.sqrt(dims)) * rng.standard_normal((96, dims)).astype(np.float32)
    return corpus.astype(np.float32), qs.astype(np.float32)


@pytest.mark.parametrize("metric", [VectorMetric.cosine, VectorMetric.dot])
@pytest.mark.parametrize("bf16", [1, 0])
def test_filter_level_answers_tight_clusters_without_exact_scans(oracle, metric, bf16):
    """Tightly clustered rows (2 000 per cluster, pairwise cosine > 0.98): the k-th result is closer to the 257th
    nominee than any tensor-core bound, so level 1 cannot prove anything.  The filter level (one TF32 pass that
    collects EVERY row above `exact k-th score of the nominees - eps`, exact re-score of all of them) must answer those
    queries -- identical ids and score bits, no exact scan."""
    dims, n = 384, 60_000
    corpus, qs = _clustered(n, dims, 30, 0.1, seed=77)          # unit rows for both metrics (dot then ranks like cosine)
    eng = CUDAVectorEngine(metric, dims)
    eng.add_batch(list(range(n)), corpus)
    eng.set_option("batch_bf16", bf16)
    t0, f0 = eng.batch_stats()
    got = eng.search_batch(qs, 10)
    t1, f1 = eng.batch_stats()
    assert got == _single(eng, qs, 10)
    r, d, s = oracle.search(metric.value, corpus, qs[3], 10, mode=oracle.ACC_F32_TREE, threads=4)
    assert [g[0] for g in got[3]] == r.tolist()
    assert np.array_equal(np.float32([g[1] for g in got[3]]).view(np.uint32), s.view(np.uint32))
    assert eng.counter("batch_retry_queries") + eng.counter("batch_filter_bf16_queries") >= 48, "no filter level was exercised"
    assert f1 - f0 == 0, f"{f1 - f0} queries needed an exact scan"
    # a list that overflows is reported, not truncated: those queries take the exact scan, same answers
    eng.set_option("batch_bf16", bf16)
    eng.set_option("filter_cap", 64)
    got2 = eng.search_batch(qs, 10)
    assert got2 == got
    assert eng.batch_stats()[1] - f1 >= 48


def test_batch_larger_than_one_launch_of_query_groups(oracle):
    """More query groups than SMs (132 x 128 = 16 896 queries on an H100): the batch is processed in several launches that
    share the scratch (heaps, thresholds, converted queries) -- every slice of the batch must still be right."""
    dims, n, b = 64, 5_000, 19_100
    eng = _engine(oracle, VectorMetric.cosine, n, dims, seed=1300)
    qs = oracle.synth_rows(1301, 0, b, dims, normalize=True)
    ids, scores, ns = eng.search_batch_arrays(qs, 5)
    assert eng.counter("batch_bf16_queries") == b and ns.tolist() == [5] * b
    eng.set_option("batch_tensor", 0)
    for qi in (0, 127, 128, 16_895, 16_896, 16_897, 18_943, 18_944, 18_945, 19_099):
        want = eng.search(qs[qi], 5)
        assert [int(i) for i in ids[qi]] == [w[0] for w in want], qi
        assert np.array_equal(scores[qi], np.float32([w[1] for w in want])), qi


@pytest.mark.parametrize("metric", [VectorMetric.cosine, VectorMetric.dot])
@pytest.mark.parametrize("dims,n,b,k", [(384, 150_000, 40, 200), (384, 150_000, 130, 500), (768, 70_000, 9, 1000),
                                        (128, 70_000, 300, 1024), (384, 100_003, 1100, 160)])
def test_large_k_batches_take_the_tensor_levels(oracle, metric, dims, n, b, k):
    """128 < k <= 1024 (the production candidate limit reaches 1 000, UnifiedSearch.swift:1195-1200): level 1 keeps 64
    nominees per slice and re-scores 1 024 of them exactly -- rarely a proof, but their k-th exact score is a valid
    threshold for the filter level, which lists EVERY row above it.  Same ids and score bits as the single-query emit +
    radix-select path, without looping it."""
    eng = _engine(oracle, metric, n, dims, seed=880 + dims, normalize=(metric is VectorMetric.cosine))
    qs = oracle.synth_rows(881 + b, 0, b, dims, normalize=True)
    t0, f0 = eng.batch_stats()
    got = eng.search_batch(qs, k)
    t1, f1 = eng.batch_stats()
    assert (t1 - t0) + (f1 - f0) == b, "the batch did not take the tensor-core levels"
    assert f1 - f0 <= max(1, b // 20), f"{f1 - f0} of {b} queries fell back to the exact scan"
    sample = sorted(set(range(0, b, max(1, b // 12))) | {b - 1})
    eng.set_option("batch_tensor", 0)
    for qi in sample:
        assert got[qi] == eng.search(qs[qi], k), (qi,)
    eng.set_option("batch_tensor", 1)
    assert all(len(hits) == min(k, n) for hits in got)
    eng.set_option("batch_large_k", 0)                          # opt-out: the loop answers, same results
    t2, f2 = eng.batch_stats()
    assert eng.search_batch(qs[:5], k) == got[:5]
    assert eng.batch_stats() == (t2, f2)


def test_nominee_heap_size_follows_k_and_adapts_to_unproven_queries(oracle):
    """The bf16 level-1 shape: the nominee heap per (slice, query) is sized from k and the slice count (expected cost of a
    batch = shape time + P(an unproven query) x one more pass), and the data overrules the model -- a batch that leaves
    queries unproven bumps the next batches one size up.  Results never depend on the choice."""
    dims, n = 384, 120_000
    eng = _engine(oracle, VectorMetric.cosine, n, dims, seed=1500)
    qs = oracle.synth_rows(1501, 0, 1024, dims, normalize=True)
    want = {k: _single(eng, qs[:3], k) for k in (10, 72)}
    heaps = {}
    for k in (10, 72, 128):
        got = eng.search_batch(qs, k)
        heaps[k] = eng.counter("batch_last_heap")
        if k in want:
            assert got[:3] == want[k]
    assert heaps[10] == 16 and heaps[72] in (24, 32) and heaps[128] == 64, heaps      # 8 groups x 18 slices
    # planted near-duplicates inside one slice: 16-entry heaps cannot prove k = 10 there -> the filter level answers
    # (same results) and the engine bumps the heap size for the following batches
    base = oracle.synth_row(1502, 0, dims, True)
    rng = np.random.default_rng(3)
    dup = base + rng.standard_normal((40, dims)).astype(np.float32) * np.float32(2e-3)
    eng.add_batch(list(range(100, 140)), dup)                        # rows 100..139 overwritten: one row slice
    probe = np.vstack([base[None, :], qs[:129]])
    eng.set_option("batch_tensor", 0)
    ref = [eng.search(q, 10) for q in probe[:2]]
    eng.set_option("batch_tensor", 1)
    assert eng.counter("batch_heap_bump") == 0
    got = eng.search_batch(probe, 10)
    assert got[:2] == ref
    assert eng.counter("batch_heap_bump") == 1, "an unproven query must bump the nominee heap size"
    eng.search_batch(probe, 10)
    assert eng.counter("batch_last_heap") > 16
