"""GPU: the single-query bf16-shadow route's nominations, checked stage by stage (wax_vs_debug_shadow_nominations).

When the finish kernel proves a single query (DESIGN 4.1), the fp32 scan returns at entry and nothing checks the answer
afterwards.  The proof is sound only if the SHADOW form of the scan gets two things right, checked here directly in
every (C, R) shape `launch_shadow_scan` compiles, for cosine and dot, both tails, and dynamic and static scheduling:

(a) bound: every nominee's score' is q.v~ (v~ the bf16 shadow row) up to the fp32 accumulation, hence within
    kBf16Eps |q||v| (cosine: |q|) of the exact score -- and on a worst-case corpus the error is the bf16 rounding of the
    row alone, not of the query too;
(b) completeness: every row left out scores at most entry 0 (the 128th nominee) -- with rows planted at row 0, the last
    row, every lane position of a step, the first and last row of a dynamic claim and the ragged last step; with n <= 128
    rows and with an allow-list of <= 128 rows of a 1 M-row corpus, every candidate row is nominated.

Also: the shadow's bits (RNE, the clamp near FLT_MAX, subnormals, -0, the cosine 1/|v| pre-scale), the nominee layout
the finish reads, row-order tie breaking, the proof at the boundary of the 128 nominees, the finish's answer against the
fp32 scan and the CPU oracle, the route end to end in every shape option, and rows whose score' overflows.
"""
import re
import zlib
from pathlib import Path

import numpy as np
import pytest

from helpers import hidden_winner, unit_rows
from test_gpu_nomination import BF16_EPS, KEY_NONE, _decode, _worst
from test_gpu_shadow_scan import bits, counts, fp32, routed
from wax_b200 import CUDAVectorEngine, VectorMetric
from wax_b200.engine import InvalidToc

pytestmark = pytest.mark.gpu

ROOT = Path(__file__).resolve().parents[1]
COS, DOT = VectorMetric.cosine, VectorMetric.dot
K_PRIME = 128
SM_BUDGET = 232448 - 4096          # pick_tma_config: the opt-in shared memory minus the kernels' static shared memory


def _shadow_forms():
    """Every (C, R) launch_shadow_scan compiles (waxvs_engine.cu), so a form added later is tested too."""
    src = (ROOT / "wax_b200" / "csrc" / "waxvs_engine.cu").read_text()
    body = re.search(r"static cudaError_t launch_shadow_scan\(.*?\n}\n", src, re.S).group(0)
    return [(int(c), int(r)) for c, r in re.findall(r"WAXVS_CASE\((\d+), (\d+)\);", body)]


FORMS = _shadow_forms()
# (name, options): the tails and the schedules; grid = 7 makes the automatic claim 8 steps long on these corpora
SCHEDULES = [("auto", dict(chunk_steps=-1, grid=0)), ("auto_grid7", dict(chunk_steps=-1, grid=7)),
             ("static", dict(chunk_steps=0, grid=0))]
TAILS = [1, 0]


def _engine(metric, dims, R, corpus=None, synth=None):
    eng = CUDAVectorEngine(metric, dims)
    if synth is not None:
        eng.fill_synthetic(synth[0], synth[1], normalize=True)
    else:
        eng.add_batch(list(range(corpus.shape[0])), corpus)
    eng.set_option("shadow_scan_min_bytes", 0)
    eng.set_option("shadow_rows_per_step", R)
    return eng


def _set(eng, **opts):
    for key, value in opts.items():
        eng.set_option(key, value)


def _widen(h):
    """bf16 bit patterns -> fp32, exactly."""
    return (h.astype(np.uint32) << np.uint32(16)).view(np.float32)


def _bf16_rne(x):
    """fp32 -> bf16 bits, round to nearest even; a finite value that rounds to +-inf is clamped to the largest finite
    bf16 (shadow_bf16_kernel)."""
    u = np.ascontiguousarray(x, np.float32).view(np.uint32).astype(np.uint64)
    h = ((u + np.uint64(0x7FFF) + ((u >> np.uint64(16)) & np.uint64(1))) >> np.uint64(16)).astype(np.uint32) & np.uint32(0xFFFF)
    clamp = ((h & np.uint32(0x7FFF)) == np.uint32(0x7F80)) & np.isfinite(x)
    return np.where(clamp, (h & np.uint32(0x8000)) | np.uint32(0x7F7F), h).astype(np.uint16)


def _dot64(m, q, block=8192):
    """(m @ q, |m| @ |q|, row norms of m) in fp64, a block of rows at a time."""
    q64 = q.astype(np.float64)
    s, a, nrm = np.empty(m.shape[0]), np.empty(m.shape[0]), np.empty(m.shape[0])
    for i in range(0, m.shape[0], block):
        b = m[i:i + block].astype(np.float64)
        s[i:i + block] = b @ q64
        a[i:i + block] = np.abs(b) @ np.abs(q64)
        nrm[i:i + block] = np.sqrt(np.einsum("ij,ij->i", b, b))
    return s, a, nrm


class Ref:
    """fp64 references of one query against an engine's corpus (fp32 rows) and its bf16 shadow."""

    def __init__(self, eng, metric, q, corpus):
        n, dims = corpus.shape
        self.n = n
        self.approx, mag, _ = _dot64(_widen(eng.read_shadow(0, n)), q)   # q.v~: what score' computes, up to accumulation
        self.slack = dims * 2.0 ** -23 * mag                             # ... and that accumulation's fp32 error
        exact, _, vn = _dot64(corpus, q)
        qn = float(np.linalg.norm(q.astype(np.float64)))
        if metric is COS:
            self.exact = exact / np.where(vn > 0, vn, 1.0)
            self.scale = np.full(n, qn)
        else:
            self.exact, self.scale = exact, qn * vn


def _check_layout(keys, allowed):
    """The nominee layout batch_finish_kernel reads.  Returns (scores', rows) of the real entries by entry index, and
    the number of candidate rows (allowed, in range) there are."""
    n_cand = int(allowed.sum())
    real = keys != KEY_NONE
    want_real = min(n_cand, K_PRIME)
    assert real.sum() == want_real, f"{real.sum()} real nominees, expected {want_real}"
    if n_cand < K_PRIME:      # slots n_cand..127 are padding: entries n_cand+1..127 and entry 0
        assert not real[0] and real[1:n_cand + 1].all() and not real[n_cand + 1:].any(), "padding out of place"
    else:
        assert real.all()
        assert keys[0] == keys.max(), "entry 0 is not the worst nominee"
    assert np.all(keys[1:-1] <= keys[2:]), "entries 1.. are not ascending"
    sc, rows = _decode(keys)
    sc, rows = sc[real], rows[real]
    assert np.all((rows >= 0) & (rows < allowed.size)), "a nominee row is out of range"
    assert np.unique(rows).size == rows.size, "a row was nominated twice"
    assert allowed[rows].all(), "a row the filter excludes was nominated"
    assert not np.isnan(sc).any(), "a NaN score' was nominated"
    return sc, rows, n_cand


def _check(d, ref, allowed=None):
    """(a) and (b) for one read-out.  Returns the largest |score' - exact| / (kBf16Eps |q||v|) over the nominees."""
    allowed = np.ones(ref.n, bool) if allowed is None else allowed
    sc, rows, n_cand = _check_layout(d["keys"], allowed)
    nominated = np.zeros(ref.n, bool)
    nominated[rows] = True
    entry0 = float(sc[0])
    sc, rows = sc[np.isfinite(sc)], rows[np.isfinite(sc)]   # a non-finite score' is nominated as +inf: it bounds nothing
    sc64 = sc.astype(np.float64)
    err = np.abs(sc64 - ref.approx[rows])
    assert np.all(err <= ref.slack[rows]), \
        f"score' differs from fp64 q.v~ by more than the accumulation slack (worst {np.max(err / ref.slack[rows]):.2f}x)"
    err = np.abs(sc64 - ref.exact[rows])
    bound = BF16_EPS * ref.scale[rows] + ref.slack[rows]
    assert np.all(err <= bound), f"score' outside the proof's bound (worst {np.max(err / bound):.3f}x)"
    if n_cand <= K_PRIME:
        assert np.array_equal(nominated, allowed), "fewer candidates than nominees, yet a candidate was left out"
    else:
        missed = ~nominated & allowed & (ref.approx > entry0 + 2 * ref.slack)
        assert not missed.any(), f"{missed.sum()} rows above entry 0 were left out (first: {np.flatnonzero(missed)[:5]})"
    with np.errstate(invalid="ignore", divide="ignore"):
        return float(np.nanmax(np.abs(sc64 - ref.exact[rows]) / (BF16_EPS * ref.scale[rows])))


def _risky_rows(n, R, chunks):
    """Row 0, the last row, every lane position of one step, the first and last row of the second and of the last
    claim for each claim length, the ragged last step."""
    steps = -(-n // R)
    rows = {0, n - 1}
    rows |= {steps // 2 * R + j for j in range(R)}
    for c in chunks:
        if c > 1:
            last = (steps - 1) // c * c
            rows |= {c * R, 2 * c * R - 1, last * R, min(last * R + c * R, n) - 1}
    rows |= set(range((steps - 1) * R, n))
    return np.array(sorted(r for r in rows if 0 <= r < n))


def _planted(rng, q, count, metric):
    """Rows whose cosine with q is 0.5 .. 0.9 (distinct): far above every random unit row, so all must be nominated."""
    qh = q.astype(np.float64) / np.linalg.norm(q)
    x = rng.standard_normal((count, q.size))
    x -= (x @ qh)[:, None] * qh[None, :]
    x /= np.linalg.norm(x, axis=1, keepdims=True)
    c = rng.permutation(np.linspace(0.5, 0.9, count))
    rows = c[:, None] * qh[None, :] + np.sqrt(1 - c * c)[:, None] * x
    if metric is DOT:
        rows *= rng.uniform(0.9, 1.2, (count, 1))
    return rows.astype(np.float32)


def _readout(eng, q, k, allow=None, **opts):
    _set(eng, **opts)
    return eng.shadow_nominations(q, k, allow_rows=allow)


@pytest.mark.parametrize("metric", [COS, DOT], ids=["cos", "dot"])
@pytest.mark.parametrize("C,R", FORMS, ids=[f"C{c}_R{r}" for c, r in FORMS])
def test_shadow_nominations_in_every_form(oracle, C, R, metric):
    """(a) + (b) on a corpus with planted rows at the structurally risky places, both tails, three schedules and a
    filter; the finish against the fp32 scan and the oracle; the shadow's bits."""
    dims, n, k_cycle = 128 * C, 40_009, (1, 10, 32)
    rng = np.random.default_rng(zlib.crc32(f"{C},{R},{metric.name}".encode()))
    q = unit_rows(rng, 1, dims)[0]
    eng = _engine(metric, dims, R, synth=(500 + C * 17 + R, n))
    chunks = set()
    for _, sched in SCHEDULES:       # the shape depends on the options and n only: learn the claim lengths first
        chunks.add(_readout(eng, q, 10, **sched)["chunk_steps"])
    risky = _risky_rows(n, R, chunks)
    assert n % R != 0 and risky.size <= 64
    # the risky rows plus random ones, 64 in all: every result of k <= 32 is planted, entry 0 is a random row far below
    extra = rng.permutation(np.setdiff1d(rng.choice(n, 200, replace=False), risky))[:64 - risky.size]
    planted = np.sort(np.concatenate([risky, extra]))
    eng.add_batch(planted.tolist(), _planted(rng, q, planted.size, metric))     # overwrite in place
    corpus = eng.read_rows(0, n)
    ref = Ref(eng, metric, q, corpus)
    if metric is DOT:
        assert np.array_equal(eng.read_shadow(0, n), _bf16_rne(corpus)), "the dot shadow is not RNE-bf16 of the rows"
    else:
        _check_cosine_shadow(eng.read_shadow(0, n), corpus)
    want = {k: fp32(eng, lambda: eng.search(q, k)) for k in k_cycle}
    steps, worst, i = -(-n // R), 0.0, 0
    for tail in TAILS:
        for name, sched in SCHEDULES:
            k = k_cycle[i % 3]
            i += 1
            d = _readout(eng, q, k, tail_select=tail, **sched)
            assert (d["C"], d["R"], d["tail_select"]) == (C, R, tail), f"{name}: launched {d}"
            assert (d["chunk_steps"] == 0) == (sched["chunk_steps"] == 0), f"{name}: launched {d}"
            if name == "auto_grid7":
                assert d["grid"] == 7 and d["chunk_steps"] > 1 and steps % d["chunk_steps"] != 0, \
                    f"no ragged last claim: {steps} steps in claims of {d['chunk_steps']}"
            worst = max(worst, _check(d, ref))
            assert set(planted.tolist()) <= set(_decode(d["keys"])[1].tolist())
            assert d["ok"] == 1, f"{name}, tail {tail}: the planted winners should be proven"
            assert bits(d["result"]) == bits(want[k]), f"{name}, tail {tail}, k={k}: the finish differs from the fp32 scan"
    _set(eng, tail_select=1, chunk_steps=-1, grid=0)
    r, _, s = oracle.search(metric.value, corpus, q, 10, mode=oracle.ACC_F32_TREE, threads=8)
    d = eng.shadow_nominations(q, 10)
    assert bits(d["result"]) == list(zip(r.tolist(), s.view(np.uint32).tolist())), "the finish differs from the oracle"
    allowed = np.ones(n, bool)
    allowed[planted[::2]] = False
    allowed[rng.integers(0, n, 5000)] = False
    ids = np.flatnonzero(allowed)
    d = eng.shadow_nominations(q, 10, allow_rows=ids)
    _check(d, ref, allowed)
    assert d["ok"] == 1 and bits(d["result"]) == bits(fp32(eng, lambda: eng.search_filtered(q, 10, allow=ids.tolist())))
    print(f"\n[shadow bound] C={C} R={R} {metric.name} warps={d['warps']} stages={d['stages']} grid={d['grid']}: "
          f"largest |score' - score| / (kBf16Eps |q||v|) = {worst:.4f}")
    eng.close()


def _check_cosine_shadow(shadow, corpus, block=8192):
    """Every element within one bf16 rounding, plus a few fp32 ulps, of v / |v| in fp64."""
    for i in range(0, corpus.shape[0], block):
        c64 = corpus[i:i + block].astype(np.float64)
        t = c64 / np.sqrt(np.einsum("ij,ij->i", c64, c64))[:, None]
        err = np.abs(_widen(shadow[i:i + block]).astype(np.float64) - t)
        bound = (2.0 ** -8 + 8 * 2.0 ** -24) * np.abs(t) + 2.0 ** -133
        assert np.all(err <= bound), f"cosine shadow off by {np.max(err / bound):.3f}x one bf16 rounding (rows {i}..)"


@pytest.mark.parametrize("C,R", FORMS, ids=[f"C{c}_R{r}" for c, r in FORMS])
def test_worst_case_dot_bound_ratio(C, R):
    """Components just below a bf16 rounding midpoint, positive query and rows: the bf16 row loses ~2^-8 of every
    product in the same direction, so the error approaches 2^-8 / (1.03 2^-7) ~ 0.49 of the proof's bound.  Above 0.3
    says the scores came from bf16 rows; below 0.6 says the query was not rounded too (that would double it)."""
    dims, n = 128 * C, 3_077
    rng = np.random.default_rng(zlib.crc32(f"worst{C},{R}".encode()))
    corpus, q = _worst(rng, n, dims), _worst(rng, 1, dims)[0]
    eng = _engine(DOT, dims, R, corpus)
    ref = Ref(eng, DOT, q, corpus)
    ratios = []
    for tail in TAILS:
        d = _readout(eng, q, 10, tail_select=tail)
        assert (d["C"], d["R"]) == (C, R)
        ratios.append(_check(d, ref))
    ratio = max(ratios)
    print(f"\n[shadow bound] C={C} R={R} worst-case dot corpus: largest |score' - score| / (kBf16Eps |q||v|) = {ratio:.4f}")
    assert ratio > 0.3, f"ratio {ratio:.3f}: the scores did not come from the bf16 shadow"
    assert ratio < 0.6, f"ratio {ratio:.3f}: more than the row's rounding (was the query rounded as well?)"
    eng.close()


@pytest.mark.parametrize("metric", [COS, DOT], ids=["cos", "dot"])
@pytest.mark.parametrize("C,R", FORMS, ids=[f"C{c}_R{r}" for c, r in FORMS])
def test_every_row_is_nominated_when_there_are_few(C, R, metric):
    """n <= 128 rows, and an allow-list of <= 128 rows of a 1 M-row corpus at the risky places: the nominees are
    exactly the candidate rows, in both tails and every schedule."""
    dims = 128 * C
    rng = np.random.default_rng(zlib.crc32(f"few{C},{R},{metric.name}".encode()))
    q = unit_rows(rng, 1, dims)[0]
    sizes = sorted({1, R - 1, R, R + 1, 127, 128} - {0})
    rows = unit_rows(rng, 128, dims)
    eng, have = None, 0
    for n in sizes:
        if eng is None:
            eng = _engine(metric, dims, R, rows[:n])
        else:
            eng.add_batch(list(range(have, n)), rows[have:n])
        have = n
        ref = Ref(eng, metric, q, rows[:n])
        for tail in TAILS:
            for _, sched in SCHEDULES:
                d = _readout(eng, q, 10, tail_select=tail, **sched)
                assert (d["C"], d["R"]) == (C, R)
                _check(d, ref)
    eng.close()

    n = 1_000_000
    eng = _engine(metric, dims, R, synth=(700 + C + R, n))
    chunks = {_readout(eng, q, 10, **sched)["chunk_steps"] for _, sched in SCHEDULES}
    risky = _risky_rows(n, R, chunks)
    for tail, size in ((1, 128), (0, 113)):
        extra = rng.permutation(np.setdiff1d(rng.choice(n, 400, replace=False), risky))[:size - risky.size]
        allow = np.sort(np.concatenate([risky, extra]))
        allowed = np.zeros(n, bool)
        allowed[allow] = True
        assert allow.size == size
        for _, sched in SCHEDULES:
            d = _readout(eng, q, 10, allow=allow, tail_select=tail, **sched)
            _, got, _ = _check_layout(d["keys"], allowed)
            assert np.array_equal(np.sort(got), allow), "the nominees are not exactly the allowed rows"
    eng.close()


@pytest.mark.parametrize("C,R", FORMS, ids=[f"C{c}_R{r}" for c, r in FORMS])
def test_ties_break_by_row(C, R):
    """300 identical best rows spread over the corpus: the nominees are the first 128 of them by row, in both tails."""
    dims, n = 128 * C, 9_001
    rng = np.random.default_rng(zlib.crc32(f"ties{C},{R}".encode()))
    corpus = unit_rows(rng, n, dims)
    q = unit_rows(rng, 1, dims)[0]
    tied = np.sort(rng.choice(n, 300, replace=False))
    corpus[tied] = q
    eng = _engine(COS, dims, R, corpus)
    for tail in TAILS:
        for _, sched in SCHEDULES:
            d = _readout(eng, q, 10, tail_select=tail, **sched)
            _, rows, _ = _check_layout(d["keys"], np.ones(n, bool))
            assert rows.tolist() == [tied[K_PRIME - 1]] + tied[:K_PRIME - 1].tolist(), \
                "the tied nominees are not the first 128 tied rows, in the finish's layout"
    eng.close()


@pytest.mark.parametrize("decoys", [126, 127, 128, 129])
def test_proof_at_the_nominee_boundary(decoys):
    """helpers.hidden_winner: the best row's score' rounds below `decoys` rows.  With <= 127 decoys the winner is a
    nominee (at 127 it is entry 0, the worst) and the finish returns it; with >= 128 it is left out and the proof must
    refuse.  At 127 the winner's own score' is the exclusion threshold and its margin to the exact score (~0.9) is
    below the bound (~2.1), so the proof refuses there too; at 126 the threshold is a random row far below.  The
    search equals the fp32 scan whatever the proof says."""
    dims, n = 256, 20_000
    rng = np.random.default_rng(900 + decoys)
    q, corpus = hidden_winner(rng, dims, n, True, n_decoys=decoys)
    q = q[0]
    eng = _engine(DOT, dims, 8, corpus)
    ref = Ref(eng, DOT, q, corpus)
    want = fp32(eng, lambda: eng.search(q, 1))
    assert want[0][0] == 0
    for tail in TAILS:
        d = _readout(eng, q, 1, tail_select=tail)
        _check(d, ref)
        rows = _decode(d["keys"])[1]
        if decoys <= 127:
            assert 0 in rows.tolist() and d["result"][0][0] == 0, "the winner is a nominee and the finish's best row"
            if decoys == 127:
                assert rows[0] == 0, "the winner is the worst nominee"
            assert d["ok"] == (1 if decoys <= 126 else 0)
        else:
            assert 0 not in rows.tolist() and d["ok"] == 0, "a proof for a query whose best row was never nominated"
        if d["ok"]:
            assert bits(d["result"]) == bits(want)
    eng.set_option("tail_select", 1)
    proven = 1 if decoys <= 126 else 0
    assert bits(routed(eng, lambda: eng.search(q, 1), proven=proven, failed=1 - proven)) == bits(want)
    eng.close()


@pytest.mark.parametrize("metric", [COS, DOT], ids=["cos", "dot"])
@pytest.mark.parametrize("C,R", FORMS, ids=[f"C{c}_R{r}" for c, r in FORMS])
def test_route_end_to_end_in_every_shape(C, R, metric):
    """The route answers (single_shadow_queries advances) and equals the fp32 scan with the shadow shape options set:
    warps 1 / 5 / auto, stages 2 / 4, grid 7 and the merge tail."""
    dims, n, k = 128 * C, 30_001, 10
    rng = np.random.default_rng(zlib.crc32(f"e2e{C},{R},{metric.name}".encode()))
    eng = _engine(metric, dims, R, synth=(800 + C + R, n))
    qs = unit_rows(rng, 2, dims)
    want = fp32(eng, lambda: [eng.search(x, k) for x in qs])
    assert [bits(g) for g in routed(eng, lambda: [eng.search(x, k) for x in qs], proven=2)] == [bits(w) for w in want]
    for warps in (1, 5, 0):
        for stages in (2, 4):
            for grid, tail in ((0, 1), (7, 0)):
                _set(eng, shadow_warps=warps, shadow_stages=stages, grid=grid, tail_select=tail)
                # pick_tma_config: an explicit warp count whose ring does not fit is refused (auto shrinks to fit)
                if not warps or warps * stages * (R * dims * 2 + 12) + warps * 1024 + 16 <= SM_BUDGET:
                    d = eng.shadow_nominations(qs[0], k)
                    assert (d["C"], d["R"], d["stages"], d["tail_select"]) == (C, R, stages, tail), d
                    assert (not warps or d["warps"] == warps) and (not grid or d["grid"] == grid), d
                    got = routed(eng, lambda: [eng.search(x, k) for x in qs], proven=2)
                else:                    # no route: the fp32 scan answers
                    with pytest.raises(InvalidToc, match="rc=-8"):
                        eng.shadow_nominations(qs[0], k)
                    got = routed(eng, lambda: [eng.search(x, k) for x in qs], proven=0)
                assert [bits(g) for g in got] == [bits(w) for w in want], (warps, stages, grid, tail)
    eng.close()


def test_overflowing_shadow_products_are_rescored():
    """Regression: a dot row whose bf16 copy rounds up across fp32 overflow.  v_0 = -v_1 = (2 - 2^-9) 2^126 round up to
    2^127 and q_i = 2: the exact products are finite and cancel, the shadow's overflow to +inf and -inf, so score' is
    NaN while the exact score (252) is the best.  Such a row used to be left out of the nominees without counting as
    excluded, so with <= 128 candidate rows the proof held and the route returned a top-k without the best row.  A
    non-finite score' is now nominated as +inf and re-scored exactly."""
    dims, k = 128, 10
    rng = np.random.default_rng(1200)
    a = np.float32(2.0 ** 126 * (2 - 2.0 ** -9))
    corpus = unit_rows(rng, 3000, dims)
    corpus[77] = 1.0
    corpus[77, :2] = (a, -a)
    q = np.full(dims, 2.0, np.float32)
    # 100 rows (nothing is excluded: the proof holds), then 3000 (the row's |v| widens the bound past every gap: refused)
    for n, proven in ((100, 1), (3000, 0)):
        eng = _engine(DOT, dims, 8, corpus[:n])
        assert _widen(eng.read_shadow(77, 1))[0, 0] == np.float32(2.0 ** 127)
        ref = Ref(eng, DOT, q, corpus[:n])
        want = fp32(eng, lambda: eng.search(q, k))
        assert want[0][0] == 77
        for tail in TAILS:
            d = _readout(eng, q, k, tail_select=tail)
            sc, rows = _decode(d["keys"])
            assert 77 in rows.tolist(), "the row with a non-finite score' was not nominated"
            assert sc[rows.tolist().index(77)] == np.inf
            _check(d, ref)
            assert d["ok"] == proven and d["result"][0][0] == 77
            if proven:
                assert bits(d["result"]) == bits(want)
        eng.set_option("tail_select", 1)
        assert bits(routed(eng, lambda: eng.search(q, k), proven=proven, failed=1 - proven)) == bits(want)
        eng.close()


def test_shadow_bits_at_the_edges():
    """Dot shadow = RNE-bf16 of the rows, bit for bit: components within 2^-8 of +-FLT_MAX are clamped to the largest
    finite bf16 (never +-inf), subnormals round like any other value, -0 stays -0.  Cosine: v / |v| within one bf16
    rounding, over norms 1e-3 .. 1e3."""
    dims, n = 128, 517
    rng = np.random.default_rng(1000)
    fmax = np.finfo(np.float32).max
    tie = np.float32(2.0 ** 127 * (2 - 2.0 ** -8))         # halfway between the largest finite bf16 and 2^128
    edge = np.array([fmax, -fmax, tie, -tie, np.nextafter(tie, np.float32(0)), -np.nextafter(tie, np.float32(0)),
                     np.nextafter(fmax, np.float32(0)), 1e-40, -1e-40, 1e-45, -1e-45, 2.0 ** -133 * 1.5, 1.17e-38,
                     -0.0, 0.0, 1.0 + 2.0 ** -8, 1.0 + 3 * 2.0 ** -8, -(1.0 + 2.0 ** -8)], np.float32)
    corpus = rng.standard_normal((n, dims)).astype(np.float32)
    corpus[:200] = rng.choice(edge, (200, dims))
    corpus[200:300] *= np.float32(2.0) ** rng.integers(-140, 120, (100, dims)).astype(np.float32)
    want = _bf16_rne(corpus)
    assert (want == np.uint16(0x7F7F)).any() and (want == np.uint16(0x8000)).any()
    eng = _engine(DOT, dims, 8, corpus)
    got = eng.read_shadow(0, n)
    bad = got != want
    assert not bad.any(), f"{bad.sum()} shadow elements differ, first {np.argwhere(bad)[:3].tolist()}"
    assert np.array_equal(eng.read_shadow(300, 17), want[300:317])
    with pytest.raises(InvalidToc, match="rc=-6"):
        eng.read_shadow(n - 3, 4)
    eng.close()
    corpus = unit_rows(rng, n, dims) * np.float32(10.0) ** rng.uniform(-3, 3, (n, 1)).astype(np.float32)
    eng = _engine(COS, dims, 8, corpus)
    _check_cosine_shadow(eng.read_shadow(0, n), corpus)
    eng.close()


def test_ineligible_read_outs_are_refused():
    """l2, k > 32, dims that are no unrolled shape and an engine without a shadow: WAX_VS_ERR_UNSUPPORTED."""
    rng = np.random.default_rng(1100)
    for metric, dims, k, opts in ((VectorMetric.l2, 128, 10, {}), (COS, 128, 33, {}), (COS, 192, 10, {}),
                                  (DOT, 128, 10, dict(batch_bf16=0))):
        eng = CUDAVectorEngine(metric, dims)
        eng.add_batch(list(range(300)), unit_rows(rng, 300, dims))
        _set(eng, **opts)
        with pytest.raises(InvalidToc, match="rc=-8"):
            eng.shadow_nominations(unit_rows(rng, 1, dims)[0], k)
        if opts:
            with pytest.raises(InvalidToc, match="rc=-8"):
                eng.read_shadow(0, 1)
        eng.close()
