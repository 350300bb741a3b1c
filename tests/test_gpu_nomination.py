"""GPU: the batched path's nomination stage, measured stage by stage (wax_vs_debug_batch_nominations).

The batched path is exact because batch_finish_kernel PROVES that no row it did not re-score can beat the k-th result.
The proof rests on two facts about the wgmma nomination pass, checked here directly instead of through end results:

(a) every nomination score' is within eps_rel * |q||v| (cosine: eps_rel * |q|) of the exact score, plus the fp32
    accumulation slack dims * 2^-23 -- measured against fp64 for every (query, row) of every kernel form, on shapes whose
    k-block count does not divide the TMA ring depth, and on a worst-case rounding corpus;
(b) the dumped heaps hold exactly what the scores nominate: every row absent from the heaps scores at most tau_excl, the
    largest root among the heaps that filled;
(c) when a winner's score' rounds below a slice full of decoys, the proof refuses and the answer is still exact -- also
    for dot rows whose |v|^2 overflows fp32.
"""
import re
import zlib
from pathlib import Path

import numpy as np
import pytest

from helpers import hidden_winner as _hidden_winner, unit_rows as _unit
from wax_b200 import CUDAVectorEngine, VectorMetric

pytestmark = pytest.mark.gpu


def _kernel_eps(name):
    """The constant the finish kernel proves with (waxvs_batch.cuh), so the measurement checks what the kernel uses."""
    src = (Path(__file__).resolve().parents[1] / "wax_b200" / "csrc" / "waxvs_batch.cuh").read_text()
    m = re.search(rf"constexpr float {name} = ([0-9.]+)f \* 0x1p-([0-9]+)f;", src)
    return float(m.group(1)) * 2.0 ** -int(m.group(2))


TF32_EPS = _kernel_eps("kTf32Eps")     # 1.25 * 2^-9
BF16_EPS = _kernel_eps("kBf16Eps")     # 1.03 * 2^-7
KEY_NONE = np.uint64(0xFFFFFFFFFFFFFFFF)
COS, DOT = VectorMetric.cosine, VectorMetric.dot

# (name, options, two dims): each form's dims give a k-block count that is not a multiple of its ring depth
# (TF32: dims / 32 k-blocks, bf16: dims / 64; rings 4 / 3 / 3 / 2 streamed, 2..6 with resident queries).
FORMS = [
    ("tf32_h16", dict(batch_bf16=0, batch_heap=16, batch_pair=0), (160, 416)),
    ("tf32_h16_pair", dict(batch_bf16=0, batch_heap=16, batch_pair=1), (160, 416)),
    ("tf32_h64", dict(batch_bf16=0, batch_heap=64, batch_pair=0), (160, 416)),
    ("bf16_h16", dict(batch_bf16=1, batch_ares=0, batch_heap=16, batch_pair=0), (320, 576)),
    ("bf16_h16_pair", dict(batch_bf16=1, batch_ares=0, batch_heap=16, batch_pair=1), (320, 576)),
    ("bf16_h24", dict(batch_bf16=1, batch_ares=0, batch_heap=24, batch_pair=0), (320, 448)),
    ("bf16_h32", dict(batch_bf16=1, batch_ares=0, batch_heap=32, batch_pair=0), (320, 448)),
    ("bf16_h64", dict(batch_bf16=1, batch_ares=0, batch_heap=64, batch_pair=0), (320, 576)),
    ("bf16_h64_pair", dict(batch_bf16=1, batch_ares=0, batch_heap=64, batch_pair=1), (320, 576)),
    ("bf16_ares_h16", dict(batch_bf16=1, batch_ares=1, batch_heap=16, batch_pair=0), (320, 192)),
    ("bf16_ares_h24", dict(batch_bf16=1, batch_ares=1, batch_heap=24, batch_pair=0), (256, 192)),
    ("bf16_ares_h24_pair", dict(batch_bf16=1, batch_ares=1, batch_heap=24, batch_pair=1), (256, 192)),
    ("bf16_ares_h64", dict(batch_bf16=1, batch_ares=1, batch_heap=64, batch_pair=0), (192, 128)),
]


def _engine(metric, corpus, opts):
    eng = CUDAVectorEngine(metric, corpus.shape[1])
    eng.add_batch(list(range(corpus.shape[0])), corpus)
    for key, value in opts.items():
        eng.set_option(key, value)
    return eng


def _worst(rng, n, dims):
    """Positive components just below 1 + j 2^-7 + 2^-8 (small j), times a random power of two per row: that value is a
    bf16 rounding midpoint and a TF32 value, so bf16 rounds every component DOWN by ~2^-8 relative and TF32 truncation
    by ~2^-10.  All product errors then have the same sign and the error of q.v approaches 2^-7 |q||v| (bf16) or 2^-9
    |q||v| (TF32 truncation)."""
    j = rng.integers(0, 4, (n, dims))
    m = (1.0 + j * 2.0 ** -7 + 2.0 ** -8) * (1.0 - 2.0 ** -18)
    return (m * np.exp2(rng.integers(-3, 4, (n, 1)))).astype(np.float32)


def _data(kind, rng, n, b, dims):
    if kind == "unit":
        return _unit(rng, n, dims), _unit(rng, b, dims)
    if kind == "mixed":      # cosine over rows with norms spread over 1e-3 .. 1e3
        return (_unit(rng, n, dims) * np.float32(10.0) ** rng.uniform(-3, 3, (n, 1)).astype(np.float32)), _unit(rng, b, dims)
    if kind == "dot":        # un-normalised rows and queries
        scale = lambda k: np.float32(10.0) ** rng.uniform(-1, 1, (k, 1)).astype(np.float32)
        return (rng.standard_normal((n, dims)).astype(np.float32) * scale(n),
                rng.standard_normal((b, dims)).astype(np.float32) * scale(b))
    assert kind == "worst"
    return _worst(rng, n, dims), _worst(rng, b, dims)


def _decode(keys):
    """nominee_key -> (score', row): key = (orderable(-score') << 32) | row."""
    k32 = (keys >> np.uint64(32)).astype(np.uint32)
    u = k32 ^ np.where(k32 & np.uint32(0x80000000), np.uint32(0x80000000), np.uint32(0xFFFFFFFF))
    return -u.view(np.float32), (keys & np.uint64(0xFFFFFFFF)).astype(np.int64)


def _check_heaps(d, n, nq, allowed=None):
    """The invariants batch_finish_kernel relies on.  Returns the [nq, n] mask of nominated rows."""
    scores, heaps = d["scores"], d["heaps"]
    slices, groups, kprime = d["slices"], d["groups"], d["kprime"]
    tiles = (n + 127) // 128
    nominated = np.zeros((nq, n), bool)
    tau_excl = np.full(nq, -np.inf)
    for s in range(slices):
        lo, hi = tiles * s // slices * 128, min(tiles * (s + 1) // slices * 128, n)
        for g in range(groups):
            qs = np.arange(g * 128, g * 128 + 128)
            live = qs < nq
            keys = heaps[s * groups + g].T[live]            # [queries, kprime]
            qs = qs[live]
            if not qs.size:
                continue
            real = keys != KEY_NONE
            sc, rows = _decode(keys)
            assert np.all((rows[real] >= lo) & (rows[real] < hi)), f"a heap of slice {s} holds a row outside [{lo}, {hi})"
            qq = np.broadcast_to(qs[:, None], keys.shape)
            assert np.array_equal(sc[real].view(np.uint32), scores[qq[real], rows[real]].view(np.uint32)), \
                "a heap entry's score differs from the score' the epilogue compared"
            for i in range(qs.size):
                r = rows[i][real[i]]
                assert np.unique(r).size == r.size, "duplicate row in a heap"
                nominated[qs[i], r] = True
            full = real[:, 0]                              # node 0 is a real key only once the heap has filled
            tau_excl[qs[full]] = np.maximum(tau_excl[qs[full]], sc[full, 0])
    if allowed is not None:
        assert not nominated[:, ~allowed].any(), "a row outside the allow-list reached a heap"
    missed = ~nominated & (scores > tau_excl[:, None].astype(np.float32))
    if allowed is not None:
        missed &= allowed[None, :]
    assert not missed.any(), f"{missed.sum()} rows above tau_excl are missing from the heaps (first: {np.argwhere(missed)[:3]})"
    return nominated


def _measure(eng, metric, corpus, qs, k=10, allowed=None):
    """Run the read-out; check coverage and the per-row bound.  Returns (dump, largest error / eps_rel bound)."""
    n, dims = corpus.shape
    d = eng.batch_nominations(qs, k, allow_rows=None if allowed is None else np.flatnonzero(allowed))
    scores = d["scores"]
    assert not np.any(scores.view(np.uint32) == 0xFFFFFFFF), "some (query, row) score' was never written"
    c64, q64 = corpus.astype(np.float64), qs.astype(np.float64)
    vn, qn = np.linalg.norm(c64, axis=1), np.linalg.norm(q64, axis=1)
    ref = q64 @ c64.T
    if metric is COS:
        ref = ref / np.where(vn > 0, vn, 1.0)[None, :]
        scale = np.broadcast_to(qn[:, None], ref.shape)
    else:
        scale = qn[:, None] * vn[None, :]
    eps_rel = BF16_EPS if d["bf16"] else TF32_EPS
    err = np.abs(scores.astype(np.float64) - ref)
    bound = eps_rel * scale + dims * 2.0 ** -23 * scale
    bad = ~(err <= bound)
    assert not bad.any(), (f"score' outside the proof's bound for {bad.sum()} entries; worst error / bound "
                           f"{np.max(err / bound):.3f} at {np.unravel_index(np.argmax(err / bound), err.shape)}")
    _check_heaps(d, n, qs.shape[0], allowed)
    return d, float(np.max(err / (eps_rel * scale)))


COMBOS = [  # (data, metric, which dims, rows, batch)
    ("unit", COS, 0, 1, 4), ("mixed", COS, 1, 127, 129), ("dot", DOT, 0, 128, 127), ("worst", DOT, 1, 129, 300),
    ("worst", None, 0, 3077, 300), ("mixed", COS, 1, 20_077, 300), ("dot", DOT, 0, 20_077, 129),
]


@pytest.mark.parametrize("name,opts,dims", FORMS, ids=[f[0] for f in FORMS])
def test_nomination_scores_stay_within_the_proof_bound(name, opts, dims):
    """(a) + (b) for every form: score' against fp64 at every (query, row), heaps against the scores."""
    rng = np.random.default_rng(zlib.crc32(name.encode()))
    bf16 = opts["batch_bf16"] == 1
    ratios, wrapped = {}, False
    for kind, metric, di, n, b in COMBOS:
        # the cosine bf16 shadow is normalised on the device, so its rounding cannot be steered from the host: the
        # worst-case corpus runs as dot there (the same bf16 operand rounding)
        metric = metric or (DOT if bf16 else COS)
        corpus, qs = _data(kind, rng, n, b, dims[di])
        eng = _engine(metric, corpus, opts)
        d, ratio = _measure(eng, metric, corpus, qs)
        eng.close()
        assert d["bf16"] == int(bf16) and d["kprime"] == opts["batch_heap"]
        assert d["ares"] == opts.get("batch_ares", 0) and d["pair"] == int(opts["batch_pair"] == 1 and d["groups"] >= 2)
        kb = dims[di] // (64 if bf16 else 32)
        wrapped |= kb > d["stages"] and kb % d["stages"] != 0
        ratios[(kind, metric.name, dims[di], n, b)] = ratio
    worst = max(ratios.values())
    print(f"\n[nomination bound] {name}: largest error / (eps_rel |q||v|) = {worst:.4f} "
          f"(worst-case corpus {max(v for k, v in ratios.items() if k[0] == 'worst'):.4f})")
    assert wrapped, "no shape of this form wraps the TMA ring in the middle of a tile"
    if bf16:   # TF32 errors stay below 1.25 * 2^-9 / (1.03 * 2^-7) = 0.30 of the bf16 bound: these came from bf16
        assert worst > 0.5, f"largest bf16 error ratio {worst:.3f}: the scores did not come from the bf16 shadow"


@pytest.mark.parametrize("bf16", [1, 0])
def test_chunk_with_many_winners_after_warm_up(bf16):
    """A 32-row chunk late in a slice with 20 rows above a warm heap's threshold at once: the staging takes the lowest
    8 set bits at a time (the warm-up path), and the heaps must still hold what the scores nominate."""
    rng = np.random.default_rng(17 + bf16)
    dims, n, b = 384, 20_077, 300
    corpus, qs = _unit(rng, n, dims), _unit(rng, b, dims)
    tiles, slices = (n + 127) // 128, 33             # 300 queries in CTA pairs: 2 units x 33 slices fill 132 SMs
    opts = dict(batch_bf16=bf16, batch_ares=0, batch_heap=16, batch_pair=1)
    chunk0 = ((tiles * 1 // slices) - 1) * 128 + 64   # third chunk of the last tile of slice 0
    near = qs[0] + 0.02 * rng.standard_normal((20, dims)).astype(np.float32)
    corpus[chunk0 + np.arange(0, 32)[:20]] = near / np.linalg.norm(near, axis=1, keepdims=True)
    eng = _engine(COS, corpus, opts)
    d, _ = _measure(eng, COS, corpus, qs)
    assert d["slices"] == slices and d["pair"] == 1
    planted = chunk0 + np.arange(20)
    best = planted[np.argsort(-d["scores"][0, planted], kind="stable")[:16]]
    in_heap = set(_decode(d["heaps"][0 * d["groups"] + 0][:, 0])[1].tolist())
    assert set(best.tolist()) <= in_heap, "the 16 best planted rows of the chunk must be the slice's nominees"
    eng.close()


@pytest.mark.parametrize("bf16", [1, 0])
def test_filtered_batch_never_nominates_a_disallowed_row(bf16):
    """search_batch_filtered shape: an allow-list below the nomination.  The best rows of every query are disallowed;
    none may reach a heap, and every allowed row above tau_excl must."""
    rng = np.random.default_rng(23 + bf16)
    dims, n, b = 384, 9_001, 129
    corpus, qs = _unit(rng, n, dims), _unit(rng, b, dims)
    allowed = np.ones(n, bool)
    allowed[::3] = False
    corpus[np.arange(0, 3 * b, 3)] = qs                  # every query's exact match sits on a disallowed row
    eng = _engine(COS, corpus, dict(batch_bf16=bf16, batch_heap=16))
    d, _ = _measure(eng, COS, corpus, qs, allowed=allowed)
    assert d["bf16"] == bf16
    ids = np.flatnonzero(allowed).astype(np.uint64)
    got = eng.search_batch_filtered(qs, 10, allow=ids)
    eng.set_option("batch_tensor", 0)
    assert got == [eng.search_filtered(q, 10, allow=ids.tolist()) for q in qs[:8]] + got[8:]
    eng.close()


@pytest.mark.parametrize("bf16", [1, 0])
def test_proof_refuses_a_hidden_winner(bf16):
    """(c) The true best row's score' rounds below more than k' decoys of its slice: the best row is not nominated,
    so level 1 must NOT prove the query, and the batch must still return exactly the single-query result."""
    rng = np.random.default_rng(31 + bf16)
    dims, n = 256, 6_000
    q, corpus = _hidden_winner(rng, dims, n, bf16, n_decoys=24)
    qs = np.concatenate([q, _unit(rng, 5, dims)])
    eng = _engine(DOT, corpus, dict(batch_bf16=bf16, batch_heap=16, batch_ares=0))
    d, _ = _measure(eng, DOT, corpus, qs, k=1)
    sc = d["scores"][0]
    exact = corpus.astype(np.float64) @ q[0].astype(np.float64)
    assert np.argmax(exact) == 0 and np.sum(sc[1:25] > sc[0]) == 24, "the construction did not hide the winner"
    assert not _check_heaps(d, n, qs.shape[0])[0, 0], "the hidden winner was nominated after all"
    assert d["ok"][0] == 0, "level 1 claimed a proof for a query whose best row it never nominated"
    got = eng.search_batch(qs, 1)
    eng.set_option("batch_tensor", 0)
    assert got == [eng.search(x, 1) for x in qs] and got[0][0][0] == 0
    eng.close()


@pytest.mark.parametrize("bf16", [1, 0])
def test_dot_rows_whose_norm_overflows_fp32_keep_the_batch_exact(bf16):
    """Finite rows with |v| ~ 1e20 (|v|^2 overflows fp32) have finite exact dot scores, so the dot proof's max|v| must
    cover them.  The hidden-winner construction at that scale, in a unit corpus: if the bound left those rows out, eps
    would stay ~1e-1 and level 1 would "prove" a top-k that misses the best row."""
    rng = np.random.default_rng(41 + bf16)
    dims, n = 384, 20_000
    q, corpus = _hidden_winner(rng, dims, n, bf16, n_decoys=24, scale_log2=62)
    with np.errstate(over="ignore"):
        assert np.isinf(np.sum(corpus[:25] ** 2, axis=1, dtype=np.float32)).all() and np.isfinite(corpus).all()
    qs = np.concatenate([q, _unit(rng, 7, dims)])
    eng = _engine(DOT, corpus, dict(batch_bf16=bf16, batch_heap=16, batch_ares=0))
    got = eng.search_batch(qs, 10)
    eng.set_option("batch_tensor", 0)
    want = [eng.search(x, 10) for x in qs]
    assert want[0][0][0] == 0
    assert [[i for i, _ in hits] for hits in got] == [[i for i, _ in hits] for hits in want]
    assert got == want
    eng.close()
