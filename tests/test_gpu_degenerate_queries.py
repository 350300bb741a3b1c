"""Degenerate QUERIES on the batched path: every route must answer them exactly as the single-query path does.

The completeness proof of batch_finish_kernel scales its error bound by the query's fp32 norm sqrt(fl(sum q^2)).  That
bound only holds while fl(sum q^2) is a normal float: a query whose squares underflow (|q_i| ~ 1e-23) has qn = 0 and
an error bound of ~0, although its score' values still differ from the exact scores; one whose sum overflows, or that
holds NaN / Inf, has no finite bound at all.  Such queries must not be proven: they go to the exact scan, which defines
their answer (USearch's rules, DESIGN section 3: cosine with |q|^2 = 0 gives distance 1 to every non-zero row).

Each degenerate query rides in a batch of ordinary ones, so these tests also show that one bad query does not change
its neighbours' answers.  The reference is the single-query path (batch_tensor = 0, or search / search_filtered /
search_grouped per query), itself bit-exact against the CPU oracle in ACC_F32_TREE; a sample is checked against the
oracle directly.  The bar: ids and score bits identical.  The one CPU test pins the oracle's own answers for these
queries.
"""
import numpy as np
import pytest

from helpers import hidden_winner, unit_rows
from wax_b200 import CUDAVectorEngine, VectorMetric

COS, DOT, L2 = VectorMetric.cosine, VectorMetric.dot, VectorMetric.l2
BF16_MAX_MIDPOINT = (2.0 - 2.0 ** -8) * 2.0 ** 127     # finite fp32 values above this round to +-inf in bf16


def degenerate_queries(rng, dims):
    """(names, [m, dims] fp32): one query per class, all but the non-finite ones with finite components."""
    sign = np.where(rng.random(dims) < 0.5, -1.0, 1.0)
    base = unit_rows(rng, 1, dims)[0]

    def with_component(x):
        q = base.copy()
        q[int(rng.integers(dims))] = x
        return q

    classes = [
        ("zero", np.zeros(dims)),
        ("negative_zero", -np.zeros(dims)),
        ("a2_underflow_negative", np.full(dims, -1e-23)),  # sum q^2 rounds to 0; every score' < 0 on a positive corpus
        ("a2_underflow_mixed", 1e-23 * sign),
        ("a2_subnormal_3e-22", 3e-22 * sign),               # sum q^2 ~ 3e-41
        ("a2_subnormal_1e-21", 1e-21 * sign),               # sum q^2 ~ 4e-40
        ("subnormal_components", 1e-40 * sign),
        ("a2_overflow", 1e20 * sign),
        ("near_flt_max", 3.4e38 * sign),                    # finite in fp32, +-inf in bf16
        ("nan_component", with_component(np.nan)),
        ("pos_inf_component", with_component(np.inf)),
        ("neg_inf_component", with_component(-np.inf)),
    ]
    qs = np.stack([q for _, q in classes]).astype(np.float32)
    assert np.all(np.abs(qs[8]) > BF16_MAX_MIDPOINT) and np.isfinite(qs[8]).all()
    return [name for name, _ in classes], qs


def positive_rows(rng, n, dims):
    return np.abs(unit_rows(rng, n, dims))


def cosine_corpus(rng, n, dims, queries):
    """Positive unit rows plus, for the first four ordinary queries, copies scaled so that sum v^2 underflows to 0
    (inv_norm = 0, a zero shadow row), is subnormal, or overflows (|v| ~ 1e20) -- spread over different row slices."""
    corpus = positive_rows(rng, n, dims)
    for i in range(4):
        for j, scale in enumerate((1e-24, 1e-20, 1e20)):
            corpus[(3 * i + j + 1) * (n // 13)] = queries[i] * np.float32(scale)
    with np.errstate(over="ignore", under="ignore"):
        sq = np.sum(corpus.astype(np.float32) ** 2, axis=1, dtype=np.float32)
    assert (sq == 0).sum() == 4 and np.isinf(sq).sum() == 4 and ((sq > 0) & (sq < np.finfo(np.float32).tiny)).sum() == 4
    return corpus


def make_corpus(metric, rng, n, dims, queries):
    if metric is COS:
        return cosine_corpus(rng, n, dims, queries)
    if metric is DOT:   # positive rows with norms over 0.1 .. 10: the negated underflowing query scores < 0 everywhere
        return positive_rows(rng, n, dims) * np.float32(10.0) ** rng.uniform(-1, 1, (n, 1)).astype(np.float32)
    return unit_rows(rng, n, dims)


def engine(metric, corpus, opts=()):
    eng = CUDAVectorEngine(metric, corpus.shape[1])
    eng.add_batch(list(range(corpus.shape[0])), corpus)
    for key, value in dict(opts).items():
        eng.set_option(key, value)
    return eng


def bits(hits):
    return [(i, int(np.float32(s).view(np.uint32))) for i, s in hits]


def flat(res):
    return [(g, f, int(np.float32(s).view(np.uint32))) for g, hits in res for f, s in hits]


def single(eng, qs, k):
    eng.set_option("batch_tensor", 0)
    out = [eng.search(q, k) for q in qs]
    eng.set_option("batch_tensor", 1)
    return out


def on_level(eng, bf16, call):
    """call() on the nomination level under test.  A batch whose queries are mostly refused suspends the bf16 level for
    the next 16 batches (adaptive level choice); setting batch_bf16 lifts that, so every call here runs on the level it
    names.  Returns (result, queries nominated from the bf16 shadow, queries nominated in TF32) of that call."""
    eng.set_option("batch_bf16", bf16)
    b0, t0 = eng.counter("batch_bf16_queries"), eng.counter("batch_tf32_queries")
    out = call()
    return out, eng.counter("batch_bf16_queries") - b0, eng.counter("batch_tf32_queries") - t0


def assert_level(bf16, nb, nt, n, where):
    assert (nb, nt) == ((n, 0) if bf16 else (0, n)), f"{where}: {nb} bf16 / {nt} TF32 queries, expected {n} on bf16={bf16}"


def interleave(ordinary, degenerate):
    """Ordinary queries with the degenerate ones in the middle; returns (batch, indices of the degenerate ones)."""
    h = ordinary.shape[0] // 2
    qs = np.concatenate([ordinary[:h], degenerate, ordinary[h:]])
    return qs, np.arange(h, h + degenerate.shape[0])


def assert_same(got, want, names, where):
    for i, (g, w) in enumerate(zip(got, want)):
        assert bits(g) == bits(w), f"{where}: query {i} ({names.get(i, 'ordinary')}) differs from the single-query path"


def check_oracle(oracle, metric, corpus, qs, got, idx, k, names):
    for i in idx:
        r, _, s = oracle.search(metric.value, corpus, qs[i], k, mode=oracle.ACC_F32_TREE, threads=8)
        assert bits(got[i]) == list(zip(r.tolist(), s.view(np.uint32).tolist())), f"{names[i]} differs from the oracle"


# (id, metric, dims, rows, ordinary queries, options, ks): the kernel forms and levels of the batched path
CASES = [
    ("cos_bf16_resident", COS, 384, 20_000, 8, dict(batch_bf16=1, batch_ares=1), (1, 10, 72, 128)),
    ("cos_bf16_streamed", COS, 384, 20_000, 8, dict(batch_bf16=1, batch_ares=0), (10,)),
    ("cos_tf32", COS, 384, 20_000, 8, dict(batch_bf16=0), (1, 10, 128)),
    ("cos_tf32_pair", COS, 384, 40_000, 130, dict(batch_bf16=0, batch_pair=1), (10,)),
    ("cos_bf16_768", COS, 768, 20_000, 8, dict(batch_bf16=1), (10,)),
    ("cos_large_k", COS, 384, 60_000, 8, dict(batch_bf16=1), (300,)),
    ("dot_bf16", DOT, 384, 20_000, 8, dict(batch_bf16=1), (10, 72)),
    ("dot_tf32", DOT, 384, 20_000, 8, dict(batch_bf16=0), (1, 128)),
    ("dot_large_k", DOT, 384, 40_000, 8, dict(), (300,)),
    ("l2_bf16", L2, 384, 20_000, 8, dict(batch_l2=1, batch_bf16=1), (10, 128)),
    ("l2_tf32", L2, 384, 20_000, 8, dict(batch_l2=1, batch_bf16=0), (10,)),
]


@pytest.mark.gpu
@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_batch_answers_degenerate_queries_like_the_single_query_path(oracle, case):
    name, metric, dims, n, b, opts, ks = case
    rng = np.random.default_rng(sum(name.encode()))
    ordinary = positive_rows(rng, b, dims) if metric is not L2 else unit_rows(rng, b, dims)
    corpus = make_corpus(metric, rng, n, dims, ordinary)
    names, deg = degenerate_queries(rng, dims)
    qs, idx = interleave(ordinary, deg)
    label = dict(zip(idx.tolist(), names))
    eng = engine(metric, corpus, opts)
    bf16 = opts.get("batch_bf16", 1)
    resident = []
    for k in ks:
        if k <= 128:            # the kernel form this batch runs in
            d = on_level(eng, bf16, lambda: eng.batch_nominations(qs, k))[0]
            assert d["bf16"] == bf16 and d["pair"] == opts.get("batch_pair", 0), (k, d["bf16"], d["pair"])
            resident.append(d["ares"])
        t0, f0 = eng.batch_stats()
        got, nb, nt = on_level(eng, bf16, lambda: eng.search_batch(qs, k))
        t1, f1 = eng.batch_stats()
        assert (t1 - t0) + (f1 - f0) == len(qs), "the batch did not take the tensor-core levels"
        assert_level(bf16, nb, nt, len(qs), f"{name} k={k}")
        assert_same(got, single(eng, qs, k), label, f"{name} k={k}")
        if k == ks[0]:
            check_oracle(oracle, metric, corpus, qs, got, idx, k, label)
    if "batch_ares" in opts:   # resident queries need a two-stage ring beside them: not every heap size leaves room
        assert any(resident) == bool(opts["batch_ares"]), resident
    eng.close()


@pytest.mark.gpu
@pytest.mark.parametrize("metric", [COS, DOT])
@pytest.mark.parametrize("bf16", [1, 0])
def test_one_hot_queries_on_a_quantised_corpus(oracle, metric, bf16):
    """Rows of +-1 only: a one-hot query scores every row +-1 exactly, so thousands of rows across all slices tie at the
    k-th place, and the answer is decided by the row index alone."""
    rng = np.random.default_rng(61 + bf16)
    dims, n = 384, 30_000
    corpus = np.where(rng.random((n, dims)) < 0.5, -1.0, 1.0).astype(np.float32)
    hot = np.zeros((4, dims), np.float32)
    hot[0, 5], hot[1, 200], hot[2, 383], hot[3, 0] = 1.0, -3.0, 0.5, 2.0 ** -60
    qs, idx = interleave(unit_rows(rng, 8, dims), hot)
    label = {int(i): f"one_hot_{j}" for j, i in enumerate(idx)}
    eng = engine(metric, corpus, dict(batch_bf16=bf16))
    for k in (10, 128):
        got, nb, nt = on_level(eng, bf16, lambda: eng.search_batch(qs, k))
        assert_level(bf16, nb, nt, len(qs), f"k={k}")
        assert_same(got, single(eng, qs, k), label, f"k={k}")
        check_oracle(oracle, metric, corpus, qs, got, idx, k, label)
        assert [i for i, _ in got[idx[0]]] == np.flatnonzero(corpus[:, 5] > 0)[:k].tolist()
    eng.close()


@pytest.mark.gpu
@pytest.mark.parametrize("metric", [COS, DOT])
@pytest.mark.parametrize("bf16", [1, 0])
def test_filtered_batches_with_degenerate_queries(metric, bf16):
    """search_batch_filtered (a large allow-list and a deny-list: the tensor class) and search_batch_multi_filtered
    (gather, tensor and unfiltered queries in one batch) against the per-query filtered search."""
    rng = np.random.default_rng(71 + metric.value)
    dims, n = 384, 40_000
    ordinary = positive_rows(rng, 8, dims)
    corpus = make_corpus(metric, rng, n, dims, ordinary)
    names, deg = degenerate_queries(rng, dims)
    qs, idx = interleave(ordinary, deg)
    label = dict(zip(idx.tolist(), names))
    eng = engine(metric, corpus)
    allow = np.sort(rng.choice(n, 24_000, replace=False)).astype(np.uint64)
    deny = np.sort(rng.choice(n, 12_000, replace=False)).astype(np.uint64)
    small = np.sort(rng.choice(n, 500, replace=False)).astype(np.uint64)
    for k in (10, 72):
        for kind, fids in (("allow", allow), ("deny", deny)):
            got, nb, nt = on_level(eng, bf16, lambda: eng.search_batch_filtered(qs, k, **{kind: fids}))
            assert_level(bf16, nb, nt, len(qs), f"{kind} k={k}")
            assert_same(got, [eng.search_filtered(q, k, **{kind: fids.tolist()}) for q in qs], label, f"{kind} k={k}")
        filters = [("allow", small), ("allow", allow), ("deny", deny)]
        for shift in range(4):      # every degenerate query under every filter class
            query_filter = [None if (i + shift) % 4 == 3 else (i + shift) % 4 for i in range(len(qs))]
            got, nb, nt = on_level(eng, bf16, lambda: eng.search_batch_multi_filtered(qs, k, filters, query_filter))
            n_tensor = sum(f != 0 for f in query_filter)                 # filter 0 (500 rows) is the gather class
            assert_level(bf16, nb, nt, n_tensor, f"multi-filtered k={k} shift={shift}")
            want = [eng.search(q, k) if f is None else eng.search_filtered(q, k, **{filters[f][0]: filters[f][1]})
                    for q, f in zip(qs, query_filter)]
            assert_same(got, want, label, f"multi-filtered k={k} shift={shift}")
    eng.close()


@pytest.mark.gpu
@pytest.mark.parametrize("metric", [COS, DOT])
@pytest.mark.parametrize("bf16", [1, 0])
def test_grouped_batches_with_degenerate_queries(metric, bf16):
    """search_batch_grouped: its coverage list is the batched top-k_c, so a wrong proof shows up as wrong groups."""
    rng = np.random.default_rng(81 + metric.value)
    dims, n = 384, 40_000
    ordinary = positive_rows(rng, 8, dims)
    corpus = make_corpus(metric, rng, n, dims, ordinary)
    names, deg = degenerate_queries(rng, dims)
    qs, idx = interleave(ordinary, deg)
    label = dict(zip(idx.tolist(), names))
    eng = engine(metric, corpus)
    ids = np.arange(n, dtype=np.uint64)
    eng.set_groups(ids, ids // 8 * 8)
    covered = eng.counter("grouped_batch_covered_queries")
    for top, per in ((10, 1), (10, 3)):
        got, nb, nt = on_level(eng, bf16, lambda: eng.search_batch_grouped(qs, top, per_group=per))
        assert (nb > 0, nt > 0) == (bool(bf16), not bf16), f"top={top} per={per}: {nb} bf16 / {nt} TF32 queries"
        for i, q in enumerate(qs):
            assert flat(got[i]) == flat(eng.search_grouped(q, top, per_group=per)), (label.get(i, "ordinary"), top, per)
    assert eng.counter("grouped_batch_covered_queries") > covered, "the grouped batch did not take the coverage level"
    eng.close()


@pytest.mark.gpu
def test_single_shadow_route_answers_degenerate_queries_like_the_scan():
    """single_shadow = 1: one query at a time through the bf16-shadow nominations and the same finish kernel."""
    rng = np.random.default_rng(91)
    dims, n = 384, 20_000
    ordinary = positive_rows(rng, 4, dims)
    corpus = cosine_corpus(rng, n, dims, ordinary)
    names, deg = degenerate_queries(rng, dims)
    eng = engine(COS, corpus)
    want = [eng.search(q, 10) for q in deg]
    eng.set_option("single_shadow", 1)
    for name, q, w in zip(names, deg, want):
        eng.set_option("batch_bf16", 1)         # re-arm the bf16 level: an unproven query suspends it for the next ones
        n0 = eng.counter("batch_bf16_queries")
        assert bits(eng.search(q, 10)) == bits(w), name
        assert eng.counter("batch_bf16_queries") == n0 + 1, f"{name} did not take the shadow route"
    eng.close()


@pytest.mark.gpu
@pytest.mark.parametrize("bf16", [1, 0])
def test_dot_hidden_winner_at_a_tiny_query_scale(bf16):
    """Rows of |v| ~ 2^60 and a query of components ~ 2^-76: fl(sum q^2) = 0, so a bound scaled by |q| max|v| is 0,
    while the nomination error (~2^-8 |q||v| for bf16) still hides the best row below 24 decoys.  The proof must refuse."""
    rng = np.random.default_rng(101 + bf16)
    dims, n = 256, 6_000
    q, corpus = hidden_winner(rng, dims, n, bf16, n_decoys=24, scale_log2=60)
    q = q * np.float32(2.0 ** -76)
    with np.errstate(under="ignore"):
        assert np.sum(q * q, dtype=np.float32) == 0.0
    assert np.argmax(corpus.astype(np.float64) @ q[0].astype(np.float64)) == 0
    qs = np.concatenate([q, unit_rows(rng, 5, dims)])
    eng = engine(DOT, corpus, dict(batch_bf16=bf16, batch_heap=16, batch_ares=0))
    d = eng.batch_nominations(qs, 1)
    sc = d["scores"][0]
    assert np.sum(sc[1:25] > sc[0]) == 24, "the construction did not hide the winner"
    assert d["ok"][0] == 0, "level 1 claimed a proof for a query whose fp32 |q|^2 is 0"
    got = eng.search_batch(qs, 1)
    want = single(eng, qs, 1)
    assert want[0][0][0] == 0
    assert bits(got[0]) == bits(want[0]) and [bits(g) for g in got] == [bits(w) for w in want]
    eng.close()


@pytest.mark.gpu
@pytest.mark.parametrize("bf16", [1, 0])
def test_cosine_query_whose_norm_underflows_is_not_proven(bf16):
    """q = -1e-23 everywhere against positive rows: every score' is negative and ordered by row, but USearch gives every
    non-zero row distance 1 when fl(|q|^2) = 0, so the answer is rows 0..k-1 -- which the nominations do not hold."""
    rng = np.random.default_rng(111 + bf16)
    dims, n, k = 384, 20_000, 10
    corpus = positive_rows(rng, n, dims)
    q = np.full((1, dims), -1e-23, np.float32)
    qs = np.concatenate([q, positive_rows(rng, 5, dims)])
    eng = engine(COS, corpus, dict(batch_bf16=bf16))
    d = eng.batch_nominations(qs, k)
    assert np.all(d["scores"][0] < 0)
    assert d["ok"][0] == 0, "level 1 claimed a proof for a query whose fp32 |q|^2 is 0"
    got = eng.search_batch(qs, k)
    assert got[0] == [(i, 0.0) for i in range(k)]
    assert [bits(g) for g in got] == [bits(w) for w in single(eng, qs, k)]
    eng.close()


@pytest.mark.gpu
def test_healthy_neighbours_stay_on_the_tensor_path():
    """130 ordinary queries and every degenerate class in one batch: only the degenerate queries (plus the usual
    handful) may leave the tensor-core levels."""
    rng = np.random.default_rng(121)
    dims, n = 384, 60_000
    corpus = unit_rows(rng, n, dims)
    names, deg = degenerate_queries(rng, dims)
    qs, idx = interleave(unit_rows(rng, 130, dims), deg)
    eng = engine(COS, corpus)
    bump0 = eng.counter("batch_heap_bump")
    t0, f0 = eng.batch_stats()
    got = eng.search_batch(qs, 10)
    t1, f1 = eng.batch_stats()
    bump1 = eng.counter("batch_heap_bump")
    print(f"\n[degenerate queries] exact re-runs {f1 - f0} of {len(qs)} ({len(deg)} degenerate); "
          f"batch_heap_bump {bump0} -> {bump1}")
    assert (t1 - t0) + (f1 - f0) == len(qs)
    assert f1 - f0 <= len(deg) + 3, f"{f1 - f0} queries fell back to the exact scan"
    assert_same(got, single(eng, qs, 10), dict(zip(idx.tolist(), names)), "mixed batch")
    eng.close()


def test_oracle_answers_for_degenerate_queries(oracle):
    """The ground truth the tests above rely on: in each accumulation mode the oracle applies USearch's rules to that
    mode's own |q|^2.  Cosine: |q|^2 = 0 gives distance 0 to rows with |v|^2 = 0 and 1 to every other row; |q|^2 = inf
    gives distance 1 wherever q.v is finite; a NaN or Inf component leaves only the rows with |v|^2 = 0 (distance 1).
    Dot and l2 return nothing for a NaN or Inf query."""
    rng = np.random.default_rng(131)
    dims, n, k = 384, 2_000, 12
    corpus = positive_rows(rng, n, dims)
    corpus[5] = 0.0                                          # |v|^2 = 0 in every mode
    corpus[9] = corpus[9] * np.float32(1e-24)                # fl32(|v|^2) = 0, but not in fp64
    names, deg = degenerate_queries(rng, dims)
    q = dict(zip(names, deg))
    f32, f64 = oracle.ACC_F32_TREE, oracle.ACC_F64

    def run(metric, query, mode):
        r, d, _ = oracle.search(metric, corpus, query, k, mode=mode)
        return r.tolist(), d.tolist()

    zero_rule = {f32: [5, 9] + [i for i in range(k) if i not in (5, 9)][:k - 2],
                 f64: [5] + [i for i in range(k + 1) if i != 5][:k - 1]}
    for name in ("zero", "negative_zero", "a2_underflow_negative", "a2_underflow_mixed", "subnormal_components"):
        r, d = run(oracle.COSINE, q[name], f32)
        assert r == zero_rule[f32] and d == [0.0, 0.0] + [1.0] * (k - 2), name
    for name in ("zero", "negative_zero"):
        r, d = run(oracle.COSINE, q[name], f64)
        assert r == zero_rule[f64] and d == [0.0] + [1.0] * (k - 1), name
    # in fp64 the tiny queries keep a non-zero norm: they rank like the same query scaled up by a power of two (exact)
    for name, e in (("a2_underflow_mixed", 80), ("subnormal_components", 140), ("a2_overflow", -66)):
        scaled = np.ldexp(q[name], e).astype(np.float32)
        assert np.all(np.abs(scaled) > 1e-3) and np.all(np.abs(scaled) < 1e3)
        assert run(oracle.COSINE, q[name], f64) == run(oracle.COSINE, scaled, f64), name
    # a subnormal fp32 |q|^2 is not zero: the cosine order, not the zero rule
    for name in ("a2_subnormal_3e-22", "a2_subnormal_1e-21"):
        r, d = run(oracle.COSINE, q[name], f32)
        assert r[0] == run(oracle.COSINE, q[name], f64)[0][0] and r[0] not in (5, 9) and d[0] < 1.0, name
    r, d = run(oracle.COSINE, q["a2_overflow"], f32)
    assert r == list(range(k)) and d == [1.0] * k
    r, d = run(oracle.COSINE, q["near_flt_max"], f32)
    assert len(r) == k and d == [1.0] * k
    for name in ("nan_component", "pos_inf_component", "neg_inf_component"):
        assert run(oracle.COSINE, q[name], f32) == ([5, 9], [1.0, 1.0]), name
        assert run(oracle.COSINE, q[name], f64) == ([5], [1.0]), name
        for metric in (oracle.DOT, oracle.L2):
            for mode in (f32, f64):
                assert run(metric, q[name], mode) == ([], []), (name, metric, mode)
