"""GPU: the batched tensor-core path at long rows, 1 056 to 8 192 dims, and just past its limit (8 224).

batch_tensor_eligible admits every dims % 32 == 0 up to 8 192, and the proofs of batch_finish_kernel / l2_proof budget
dims * 2^-23 * |q||v| for the fp32 accumulation of the wgmma pass.  At 8 192 dims that slack is 2^-10 relative, 40 % of
the TF32 operand bound and more than the bf16 one leaves spare, so it has to hold on its own.  Here:

(a) the accumulation error alone: rows and queries whose components are exact in bf16 (hence TF32), so every product is
    exact and score' - fp64(q.v) is what the accumulator lost, against dims * 2^-23 * sum |q_i v_i| for every (query,
    row) of every streamed form (resident queries need dims / 64 k-blocks of 16 KB: they cannot fit at these lengths);
(b) the whole nomination bound the proofs use (cosine, dot, l2) and the heap invariants, at 2 048, 4 096 and 8 192;
(c) batched answers equal to the single-query path, ids and score bits, with the route pinned by the counters: bf16
    only where dims % 64 == 0, and no tensor-core level at all at 8 224.
"""
import zlib

import numpy as np
import pytest

from helpers import hidden_winner, unit_rows
from test_gpu_batch_l2 import _measure as _measure_l2
from test_gpu_nomination import _check_heaps, _data, _measure
from wax_b200 import CUDAVectorEngine, InvalidToc, VectorMetric, Where

pytestmark = pytest.mark.gpu

COS, DOT, L2 = VectorMetric.cosine, VectorMetric.dot, VectorMetric.l2
DIMS = [1056, 1536, 2048, 3072, 4096, 4128, 6144, 8160, 8192, 8224]
TENSOR_DIMS = [d for d in DIMS if d <= 8192]          # all are multiples of 32
ROUTE = ("batch_tensor_queries", "batch_fallback_queries", "batch_bf16_queries", "batch_tf32_queries")


def _bf16_dims(dims):
    """The bf16 nominations need whole 64-element k-blocks: 1 056, 4 128 and 8 160 are TF32 only."""
    return dims % 64 == 0


def _engine(metric, corpus, ids=None, **opts):
    eng = CUDAVectorEngine(metric, corpus.shape[1])
    eng.add_batch(np.arange(corpus.shape[0], dtype=np.uint64) if ids is None else ids, corpus)
    if metric is L2:
        eng.set_option("batch_l2", 1)
    for key, value in opts.items():
        eng.set_option(key, value)
    return eng


def _route(eng):
    return np.array([eng.counter(name) for name in ROUTE], np.int64)


def _single(eng, qs, k):
    eng.set_option("batch_tensor", 0)
    out = [eng.search(q, k) for q in qs]
    eng.set_option("batch_tensor", 1)
    return out


# ---- (a) the accumulation error, isolated ---------------------------------------------------------------------------

def _exact_components(rng, shape, spread):
    """Positive m 2^e, m an integer in [128, 255] (8 significant bits: exact in bf16 and TF32), e in [-spread, spread]."""
    return rng.integers(128, 256, shape) * np.exp2(rng.integers(-spread, spread + 1, shape) - 8.0)


def _exact_data(rng, n, b, dims):
    """Rows: all-positive with exponents spread over 2^+-3 (truncated alignments add up), all-positive with one exponent
    (the sum grows steadily), random signs, and mirrored rows v[h:] = -v[:h] with the last sign flipped.  Queries: all
    positive, and mirrored q[h:] = q[:h], which meet the mirrored rows with a large sum |q_i v_i| and a small q.v."""
    h, r = dims // 2, n // 4
    rows = np.concatenate([_exact_components(rng, (r, dims), 3), _exact_components(rng, (r, dims), 0),
                           _exact_components(rng, (r, dims), 3) * rng.choice([-1.0, 1.0], (r, dims)),
                           np.zeros((n - 3 * r, dims))])
    mirror = _exact_components(rng, (n - 3 * r, h), 3)
    rows[3 * r:] = np.concatenate([mirror, -mirror], axis=1)
    rows[3 * r:, -1] *= -1.0
    qs = _exact_components(rng, (b, dims), 3)
    qs[b // 2:, h:] = qs[b // 2:, :h]
    return rows.astype(np.float32), qs.astype(np.float32)


ACC_FORMS = [(bf16, heap, pair) for bf16 in (1, 0) for heap in (16, 64) for pair in (0, 1)]


@pytest.mark.parametrize("dims", DIMS)
def test_accumulation_error_stays_within_the_slack(dims):
    """score' of products that are all exact: |score' - q.v| <= dims 2^-23 sum |q_i v_i| at every (query, row), for
    bf16 / TF32, 16- / 64-entry heaps, single CTA / CTA pair.  The resident-query form is asked for and must not be
    taken (its query k-blocks alone outgrow shared memory); TF32-only lengths must not take bf16."""
    rng = np.random.default_rng(dims)
    n, b = 2_125, 130                        # a partial last tile; two query groups, so the CTA pair runs
    corpus, qs = _exact_data(rng, n, b, dims)
    eng = _engine(DOT, corpus, batch_ares=1)
    if dims > 8192:
        with pytest.raises(InvalidToc, match="no tensor-core nomination pass"):
            eng.batch_nominations(qs, 10)
        eng.close()
        return
    c64, q64 = corpus.astype(np.float64), qs.astype(np.float64)
    ref = q64 @ c64.T
    slack = dims * 2.0 ** -23 * (np.abs(q64) @ np.abs(c64).T)
    line = []
    for bf16, heap, pair in ACC_FORMS:
        for key, value in (("batch_bf16", bf16), ("batch_heap", heap), ("batch_pair", pair)):
            eng.set_option(key, value)
        d = eng.batch_nominations(qs, 10)
        assert d["bf16"] == int(bf16 == 1 and _bf16_dims(dims)), "bf16 nominations at a length without whole bf16 k-blocks"
        assert d["ares"] == 0 and d["kprime"] == heap and d["pair"] == pair
        assert dims // (64 if d["bf16"] else 32) > d["stages"], "the k-block loop must wrap the TMA ring"
        err = np.abs(d["scores"].astype(np.float64) - ref)
        ratio = err / slack
        worst = np.unravel_index(np.argmax(ratio), ratio.shape)
        assert np.all(err <= slack), (f"bf16={d['bf16']} heap={heap} pair={pair}: accumulation error / slack "
                                      f"{ratio[worst]:.3f} at (query, row) {worst}")
        _check_heaps(d, n, b)
        form = "bf16" if d["bf16"] else ("tf32" if bf16 == 0 else "tf32(bf16 asked)")
        line.append(f"{form}_h{heap}{'_pair' if pair else ''} {ratio.max():.4f}")
    print(f"\n[accumulation] dims {dims}: largest error / (dims 2^-23 sum|q_i v_i|): " + ", ".join(line))
    eng.close()


# ---- (b) the whole nomination bound, at length ------------------------------------------------------------------------

BOUND_COMBOS = [("unit", COS, 3_077, 129), ("mixed", COS, 5_000, 300), ("dot", DOT, 5_000, 129),
                ("worst", None, 3_077, 300)]


@pytest.mark.parametrize("bf16", [1, 0])
@pytest.mark.parametrize("dims", [2048, 4096, 8192])
def test_nomination_scores_stay_within_the_proof_bound_at_length(dims, bf16):
    """Cosine / dot score' within eps_rel |q||v| + dims 2^-23 |q||v| (the finish kernel's bound) and l2 score' within
    E(|v|) of l2_proof, at every (query, row); the heaps hold what the scores nominate."""
    rng = np.random.default_rng(zlib.crc32(f"long{dims}_{bf16}".encode()))
    ratios, l2_ratios = {}, {}
    for kind, metric, n, b in BOUND_COMBOS:
        # the cosine bf16 shadow is normalised on the device: the worst-case corpus runs as dot there
        metric = metric or (DOT if bf16 else COS)
        corpus, qs = _data(kind, rng, n, b, dims)
        eng = _engine(metric, corpus, batch_bf16=bf16)
        d, ratios[kind] = _measure(eng, metric, corpus, qs)
        assert d["bf16"] == bf16
        eng.close()
        eng = _engine(L2, corpus, batch_bf16=bf16)
        d, l2_ratios[kind] = _measure_l2(eng, corpus, qs)
        assert d["bf16"] == bf16
        eng.close()
    form = "bf16" if bf16 else "tf32"
    print(f"\n[nomination bound] dims {dims} {form}: largest error / (eps_rel |q||v|) "
          + ", ".join(f"{k} {v:.4f}" for k, v in ratios.items())
          + "; l2 error / E(|v|) " + ", ".join(f"{k} {v:.4f}" for k, v in l2_ratios.items()))
    if bf16:   # TF32 errors stay below 0.30 of the bf16 bound: these came from the bf16 shadow
        assert ratios["worst"] > 0.5, f"largest bf16 error ratio {ratios['worst']:.3f}"


# ---- (c) end to end ----------------------------------------------------------------------------------------------------

def _corpus(oracle, metric, n, dims, seed):
    """Synthetic rows (unit for cosine and l2, raw [-1, 1] components for dot) with three zero rows and a NaN row."""
    corpus = oracle.synth_rows(seed, 0, n, dims, normalize=metric is not DOT)
    corpus[[11, n // 2, n - 1]] = 0.0
    corpus[12, dims // 3] = np.nan
    return corpus


@pytest.mark.parametrize("metric", [COS, DOT, L2], ids=lambda m: m.name)
@pytest.mark.parametrize("dims", DIMS)
def test_batch_equals_single_query_path_at_length(oracle, dims, metric):
    """k in {1, 10, 100, 200} (200 takes the large-k shape) and batches of 5, 129 and 300: every answer equals the
    single-query path.  Up to 8 192 every query goes through the tensor-core levels, bf16 only at whole bf16 k-blocks;
    at 8 224 the batch loops the single-query path and no tensor-core counter moves."""
    n = 20_000                               # >= 64 k for k = 200
    corpus = _corpus(oracle, metric, n, dims, seed=dims + 10 * metric.value)
    eng = _engine(metric, corpus)
    qs = oracle.synth_rows(dims + 10 * metric.value + 1, 0, 300, dims, normalize=True)
    qs[7] = corpus[777]                      # a query with an exact match in the corpus
    tensor = dims <= 8192
    start = _route(eng)
    for k in (1, 10, 100, 200):
        want = _single(eng, qs, k)
        for b in (5, 129, 300):
            before = _route(eng)
            got = eng.search_batch(qs[:b], k)
            delta = _route(eng) - before
            assert got == want[:b], (dims, metric.name, k, b)
            if tensor:
                assert delta[0] + delta[1] == b and delta[2] + delta[3] == b, f"k={k} b={b}: not the tensor levels {delta}"
            else:
                assert not delta.any(), f"k={k} b={b}: the tensor-core levels ran at {dims} dims {delta}"
        if k == 10:
            r, _, s = oracle.search(metric.value, corpus, qs[0], k, mode=oracle.ACC_F32_TREE, threads=8)
            assert [g[0] for g in want[0]] == r.tolist()
            assert np.array_equal(np.float32([g[1] for g in want[0]]).view(np.uint32), s.view(np.uint32))
    total = _route(eng) - start
    if tensor:
        assert total[0] > 0, f"no query was answered by the tensor-core levels {total}"
        if _bf16_dims(dims):
            assert total[2] > 0, "no batch nominated from the bf16 shadow"
        else:
            assert total[2] == 0 and total[3] == total[0] + total[1], "bf16 nominations at a TF32-only length"
    eng.close()


@pytest.mark.parametrize("dims", TENSOR_DIMS)
def test_proof_refuses_a_hidden_winner_at_length(dims):
    """The hidden-winner corpus at these lengths: the true best row's score' rounds below the 24 decoys of its slice, so
    level 1 must not prove the query (dot, and l2 with the query scaled by 2^6), and the batch still answers exactly."""
    n = 6_000
    for bf16 in ((1, 0) if _bf16_dims(dims) else (0,)):
        rng = np.random.default_rng(dims + bf16)
        q, corpus = hidden_winner(rng, dims, n, bf16, n_decoys=24)
        for metric in (DOT, L2):
            qs = np.concatenate([q * np.float32(64.0 if metric is L2 else 1.0), unit_rows(rng, 5, dims)])
            eng = _engine(metric, corpus, batch_bf16=bf16, batch_heap=16, batch_ares=0)
            d, _ = _measure_l2(eng, corpus, qs, k=1) if metric is L2 else _measure(eng, metric, corpus, qs, k=1)
            assert d["bf16"] == bf16
            sc = d["scores"][0]
            assert np.sum(sc[1:25] > sc[0]) == 24, f"{metric.name} bf16={bf16}: the construction did not hide the winner"
            assert not _check_heaps(d, n, qs.shape[0])[0, 0], "the hidden winner was nominated after all"
            assert d["ok"][0] == 0, "level 1 claimed a proof for a query whose best row it never nominated"
            for k in (1, 10):
                got = eng.search_batch(qs, k)
                assert got == _single(eng, qs, k) and got[0][0][0] == 0, (metric.name, bf16, k)
            eng.close()


@pytest.mark.parametrize("dims", [4096, 8192])
def test_grouped_filtered_and_where_batches_at_length(oracle, dims):
    """One batch each of search_batch_grouped, search_batch_multi_filtered and search_batch_where over the tensor-core
    levels, every answer equal to the per-query search."""
    n, b = 20_000, 129
    rng = np.random.default_rng(dims + 7)
    corpus = oracle.synth_rows(dims + 8, 0, n, dims, normalize=True)
    ids = np.arange(n, dtype=np.uint64) * 3 + 17
    eng = _engine(COS, corpus, ids=ids)
    qs = oracle.synth_rows(dims + 9, 0, b, dims, normalize=True)

    eng.set_groups(ids, ids[(np.arange(n) // 8) * 8])
    covered = eng.counter("grouped_batch_covered_queries")
    got = eng.search_batch_grouped(qs, 12, per_group=3)
    assert eng.counter("grouped_batch_covered_queries") > covered, "the grouped batch did not take the coverage level"
    for i in range(0, b, 8):
        assert got[i] == eng.search_grouped(qs[i], 12, per_group=3), i

    # deny-lists and a large allow-list: the tensor class (allow-lists up to 16 384 rows are gathered instead)
    filters = [("deny", ids[rng.choice(n, 2_000, replace=False)]), ("allow", ids[rng.choice(n, 17_000, replace=False)]),
               ("deny", ids[:5_000])]
    query_filter = [None if i % 4 == 3 else i % 4 for i in range(b)]
    before = _route(eng)
    got = eng.search_batch_multi_filtered(qs, 10, filters, query_filter)
    delta = _route(eng) - before
    assert delta[0] + delta[1] == b and delta[0] > 0, f"the filtered batch did not take the tensor-core levels {delta}"
    eng.set_option("batch_tensor", 0)
    for i in range(b):
        f = query_filter[i]
        want = eng.search(qs[i], 10) if f is None else eng.search_filtered(qs[i], 10, **{filters[f][0]: filters[f][1]})
        assert got[i] == want, i
    eng.set_option("batch_tensor", 1)

    ts = np.arange(n, dtype=np.int64) * 10
    tags = (rng.random(n) < 0.05).astype(np.uint64)
    assert eng.set_attributes(ids, ts, tags) == n
    wheres = [Where(after=int(ts[1_000]), no_tags=1), Where(before=int(ts[n - 500]))]
    query_where = [i % 2 for i in range(b)]
    before = _route(eng)
    got = eng.search_batch_where(qs, 10, wheres, query_where)
    delta = _route(eng) - before
    assert delta[0] + delta[1] == b and delta[0] > 0, f"the where batch did not take the tensor-core levels {delta}"
    for i in range(b):
        w = wheres[query_where[i]]
        passing = (ts >= w.after) & (ts < w.before) & ((tags & np.uint64(w.no_tags)) == 0)
        assert got[i] == eng.search_filtered(qs[i], 10, allow=ids[passing]), i
    eng.close()
