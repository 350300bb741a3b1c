"""GPU: the int8 form of the single-query shadow route (DESIGN 4.1).

For fp32 corpora of at least `int8_scan_min_bytes` whose measured int8 bound is no coarser than the bf16 one, a single
cosine / dot query with k <= 32 is nominated by the INT8 form of the streaming scan (one byte per element plus one scale
per row: half the bytes of the bf16 shadow), then re-scored exactly and proven by the finish with eps_rel = rho_max / M,
and the guarded fp32 scan answers only when the proof fails.  Checked here, with `int8_scan_min_bytes` lowered so that
small corpora take the int8 form:
  * the stored codes, scales and rho_max against a numpy model (-0, subnormal, zero, huge dot and non-finite rows);
  * in every (C, R) shape `launch_int8_scan` compiles, both metrics, both tails, static and dynamic claims: every
    nominee's score' against fp64 s (q.c) and against the bound, and completeness (every row left out scores at most the
    128th nominee), with winners planted at every lane position, claim edges and the ragged last step;
  * <= 128 candidates all nominated, also under an allow-list; ties; a hidden winner built for int8 rounding behind
    126..129 decoys; products that overflow;
  * the route end to end against the forced fp32 scan, ids and score bits, also under allow / deny lists, a where bitset,
    both delivery modes and search_device; the skip window after a refused int8 proof; which shadow the selection takes
    (a corpus too coarse for the int8 form gives its shadow back); appends, removes and overwrites;
  * device memory: the int8 shadow never takes the room the bf16 shadow would have had, and a bf16 shadow that does
    not fit no longer turns the int8 form off.
"""
import re
from pathlib import Path

import numpy as np
import pytest

from helpers import unit_rows
from test_gpu_nomination import KEY_NONE, _decode
from test_gpu_shadow_scan import SKIP, assert_refused_then_skip_window, bits, counts, fp32
from wax_b200 import CUDAVectorEngine, VectorMetric

pytestmark = pytest.mark.gpu

ROOT = Path(__file__).resolve().parents[1]
COS, DOT = VectorMetric.cosine, VectorMetric.dot
K_PRIME = 128


def _int8_forms():
    """Every (C, R) launch_int8_scan compiles (waxvs_engine.cu), so a form added later is tested too."""
    src = (ROOT / "wax_b200" / "csrc" / "waxvs_engine.cu").read_text()
    body = re.search(r"static cudaError_t launch_int8_scan\(.*?\n}\n", src, re.S).group(0)
    return [(int(c), int(r)) for c, r in re.findall(r"WAXVS_CASE\((\d+), (\d+)\);", body)]


FORMS = _int8_forms()
SCHEDULES = [("auto", dict(chunk_steps=-1, grid=0)), ("auto_grid7", dict(chunk_steps=-1, grid=7)),
             ("static", dict(chunk_steps=0, grid=0))]


def _set(eng, **opts):
    for key, value in opts.items():
        eng.set_option(key, value)


def _engine(metric, corpus, **opts):
    eng = CUDAVectorEngine(metric, corpus.shape[1])
    eng.add_batch(list(range(corpus.shape[0])), corpus)
    _set(eng, shadow_scan_min_bytes=0, int8_scan_min_bytes=0, **opts)
    return eng


def _vhat(metric, corpus):
    """The rows the shadow codes: cosine rows times the cached fp32 1/|v| (0 for a zero sum of squares), dot rows as is."""
    if metric is DOT:
        return corpus.astype(np.float32)
    s2 = np.einsum("ij,ij->i", corpus.astype(np.float64), corpus.astype(np.float64))
    live = np.einsum("ij,ij->i", corpus, corpus, dtype=np.float32) > 0         # fp32 sum of squares, as on the device
    inv = np.where(live, np.float32(1.0) / np.sqrt(np.where(live, s2, 1.0)).astype(np.float32), np.float32(0.0))
    inv = inv.astype(np.float32)
    return (corpus * inv[:, None]).astype(np.float32)


def _model(vhat):
    """(codes + 128 as uint8, scales, rho per row in fp64) as shadow_int8_kernel stores them; non-finite rows rho = inf."""
    with np.errstate(all="ignore"):
        m = np.abs(vhat).max(axis=1)
        s = (m / np.float32(127.0)).astype(np.float32)
        bad = ~np.isfinite(vhat).all(axis=1) | ~np.isfinite(s)
        c = np.where((s[:, None] > 0) & ~bad[:, None], np.rint(vhat / s[:, None]), 0.0)
        c = np.clip(np.nan_to_num(c), -127, 127)
        r = vhat.astype(np.float64) - s.astype(np.float64)[:, None] * c
        rho = np.sqrt(np.einsum("ij,ij->i", r, r))
    rho[bad] = np.inf
    return (c + 128).astype(np.uint8), s, rho


def _special_rows(rng, n, dims, metric):
    v = rng.uniform(-1.0, 1.0, (n, dims)).astype(np.float32)
    v[3] = 0.0                                                         # zero row
    v[4] = -0.0                                                        # -0 row
    v[5] = np.float32(2.0 ** -149) * rng.integers(-5, 6, dims)         # subnormal components
    v[6, ::2] = -0.0
    v[7] *= np.float32(2.0 ** -130)                                    # tiny normal / subnormal mix
    if metric is DOT:
        v[8] *= np.float32(1e36)                                       # huge dot row
    return v


@pytest.mark.parametrize("metric", [COS, DOT])
@pytest.mark.parametrize("dims", [128, 384, 1536])
def test_stored_codes_scales_and_bound(metric, dims):
    rng = np.random.default_rng(dims + (metric is DOT))
    corpus = _special_rows(rng, 700, dims, metric)
    eng = _engine(metric, corpus)
    codes, scales, rho_max = eng.read_int8_shadow(0, corpus.shape[0])
    vhat = _vhat(metric, corpus)
    want_codes, want_s, _ = _model(vhat)
    if metric is DOT:           # the rows are coded as they are: bit for bit
        assert np.array_equal(scales.view(np.uint32), want_s.view(np.uint32)), "scales"
        assert np.array_equal(codes, want_codes), "codes"
    else:                       # the device's 1/|v| may differ from this model's by an ulp: a code may move by one
        assert np.allclose(scales, want_s, rtol=2.0 ** -21, atol=0), "scales"
        diff = np.abs(codes.astype(np.int32) - want_codes.astype(np.int32))
        assert diff.max() <= 1 and (diff > 0).mean() < 1e-3, "codes"
    # rho_max bounds every row's residual, measured in fp64 from the stored codes and scales
    r = vhat.astype(np.float64) - scales.astype(np.float64)[:, None] * (codes.astype(np.float64) - 128.0)
    rho = np.sqrt(np.einsum("ij,ij->i", r, r))
    tol = 2.0 ** -20 if metric is COS else 2.0 ** -40
    assert rho_max >= rho.max() * (1 - tol) and rho_max <= rho.max() * (1 + 2.0 ** -20) + 1e-45, (rho_max, rho.max())
    zero = [3, 4]
    assert (codes[zero] == 128).all() and (scales[zero] == 0).all(), "zero and -0 rows"
    assert eng.counter("int8_shadow_rows") == corpus.shape[0]
    assert eng.counter("int8_shadow_bytes") == corpus.shape[0] * (dims + 4)
    # a non-finite row makes the bound +inf: the route then keeps the bf16 shadow
    bad = corpus[:40].copy()
    bad[9, 1] = np.inf
    eng.add_batch(list(range(10_000, 10_040)), bad)
    assert eng.read_int8_shadow(0, 1)[2] == np.inf
    eng.close()


def _check_nominations(d, vhat, codes, scales, rho_max, q, allowed):
    """Layout, score' against fp64 s (q.c), the bound against the rows the shadow coded, and completeness.  Returns the
    nominated rows."""
    keys = d["keys"]
    n = vhat.shape[0]
    n_cand = int(allowed.sum())
    real = keys != KEY_NONE
    assert real.sum() == min(n_cand, K_PRIME)
    if n_cand >= K_PRIME:
        assert keys[0] == keys.max(), "entry 0 is not the worst nominee"
    assert np.all(keys[1:-1] <= keys[2:]), "entries 1.. are not ascending"
    sc, rows = _decode(keys)
    sc, rows = sc[real].astype(np.float64), rows[real]
    assert allowed[rows].all() and np.unique(rows).size == rows.size
    c = codes.astype(np.float64) - 128.0
    q64 = q.astype(np.float64)
    approx = scales.astype(np.float64) * (c @ q64)                     # s (q.c) in fp64
    mag = scales.astype(np.float64) * (np.abs(c) @ np.abs(q64))
    slack = vhat.shape[1] * 2.0 ** -23 * mag + 2.0 ** -23 * np.abs(approx) + 1e-37
    fin = np.isfinite(sc)
    assert np.all(np.abs(sc[fin] - approx[rows[fin]]) <= slack[rows[fin]]), "score' is not s (q.c)"
    exact = vhat.astype(np.float64) @ q64
    qn = float(np.linalg.norm(q64))
    # (+ 2^-20 |q|: this model's cosine rows may differ from the device's by an ulp of 1/|v|)
    assert np.all(np.abs(approx - exact) <= qn * rho_max * (1 + 1e-6) + qn * 2.0 ** -20 + 1e-30), "the bound does not hold"
    nominated = np.zeros(n, bool)
    nominated[rows] = True
    if n_cand > K_PRIME:
        entry0 = float(sc[0]) if real[0] else np.inf
        left = allowed & ~nominated
        assert np.all(approx[left] <= entry0 + slack[left] + slack.max()), "a row left out beats the 128th nominee"
    else:
        assert nominated[allowed].all(), "a candidate row was not nominated"
    return rows


@pytest.mark.parametrize("tail", [1, 0])
@pytest.mark.parametrize("sched", [s[0] for s in SCHEDULES])
@pytest.mark.parametrize("metric", [COS, DOT])
@pytest.mark.parametrize("form", FORMS, ids=[f"C{c}_R{r}" for c, r in FORMS])
def test_nominations_in_every_form(form, metric, sched, tail):
    C, R = form
    dims = 128 * C
    rng = np.random.default_rng(C * 100 + R + (metric is DOT))
    n = 20_000 + 3 * R + 1                                             # a ragged last step
    corpus = rng.uniform(-1.0, 1.0, (n, dims)).astype(np.float32)
    q = rng.uniform(-1.0, 1.0, dims).astype(np.float32)
    # planted winners: every lane position of one step, both ends, the ragged last step, claim edges (8-step claims)
    planted = sorted({0, n - 1, n - 2} | {100 * R + j for j in range(R)} | {8 * R * 7 - 1, 8 * R * 7, 8 * R * 13})
    for i, row in enumerate(planted):
        corpus[row] = q * np.float32(1.0 + 0.01 * i)
    eng = _engine(metric, corpus, int8_rows_per_step=R, tail_select=tail, **dict(SCHEDULES)[sched])
    d = eng.int8_nominations(q, 10)
    assert (d["C"], d["R"]) == (C, R), d
    codes, scales, rho_max = eng.read_int8_shadow(0, n)
    vhat = _vhat(metric, corpus)
    rows = _check_nominations(d, vhat, codes, scales, rho_max, q, np.ones(n, bool))
    assert set(planted) <= set(rows.tolist()), "a planted winner was not nominated"
    want = fp32(eng, lambda: eng.search(q, 10))
    assert bits(d["result"]) == bits(want)
    # <= 128 candidates under an allow-list: every one is nominated
    allow = rng.choice(n, 100, replace=False)
    allowed = np.zeros(n, bool)
    allowed[allow] = True
    d = eng.int8_nominations(q, 10, allow_rows=allow)
    _check_nominations(d, vhat, codes, scales, rho_max, q, allowed)
    eng.close()


@pytest.mark.parametrize("metric", [COS, DOT])
def test_small_corpora_and_ties(metric):
    rng = np.random.default_rng(7)
    for n in (1, 5, 127, 128, 129):
        corpus = rng.uniform(-1.0, 1.0, (n, 384)).astype(np.float32)
        eng = _engine(metric, corpus)
        q = rng.uniform(-1.0, 1.0, 384).astype(np.float32)
        d = eng.int8_nominations(q, min(10, n))
        codes, scales, rho = eng.read_int8_shadow(0, n)
        _check_nominations(d, _vhat(metric, corpus), codes, scales, rho, q, np.ones(n, bool))
        assert bits(d["result"]) == bits(fp32(eng, lambda: eng.search(q, 10)))
        eng.close()
    corpus = np.tile(rng.uniform(-1.0, 1.0, (1, 384)).astype(np.float32), (300, 1))   # 300 identical rows: ties
    eng = _engine(metric, corpus)
    d = eng.int8_nominations(corpus[0], 10)
    _, rows = _decode(d["keys"])
    assert sorted(rows[1:].tolist()) == list(range(127)) and rows[0] == 127, "ties must break on the row index"
    assert [i for i, _ in d["result"]] == list(range(10))
    eng.close()


def _int8_hidden_winner(rng, dims, n, n_decoys):
    """Dot corpus: row 0 is the true best for q = ones, but every component but the first sits just below a code rounding
    midpoint (s = 1), so its score' is (dims - 1) (1/2 - 2^-10) below its score; decoys hold exact codes with exact scores
    spread over (0.15, 0.9) of that gap below the best.  The other rows are small and unrelated."""
    base = rng.integers(0, 4, dims).astype(np.float64)
    base[0] = 127.0
    best = base + 0.5 - 2.0 ** -10
    best[0] = 127.0
    q = np.ones(dims)
    s_best = best.sum()
    gap = s_best - base.sum()
    decoys = np.empty((n_decoys, dims))
    for i, t in enumerate(np.linspace(0.9, 0.15, n_decoys)):
        row = base.copy()
        for c in rng.permutation(np.arange(1, dims)):
            if row.sum() >= s_best - t * gap:
                break
            row[c] += 1.0
        assert s_best - t * gap <= row.sum() < s_best
        decoys[i] = row
    corpus = rng.uniform(-1.0, 1.0, (n, dims))
    corpus[0] = best
    corpus[1:1 + n_decoys] = decoys
    return q.astype(np.float32), corpus.astype(np.float32)


@pytest.mark.parametrize("n_decoys", [126, 127, 128, 129])
def test_hidden_winner_behind_int8_rounding(n_decoys):
    rng = np.random.default_rng(n_decoys)
    q, corpus = _int8_hidden_winner(rng, 384, 5_000, n_decoys)
    eng = _engine(DOT, corpus)
    d = eng.int8_nominations(q, 1)
    _, rows = _decode(d["keys"])
    want = fp32(eng, lambda: eng.search(q, 1))
    assert want[0][0] == 0
    if 0 not in rows.tolist():
        assert d["ok"] == 0, "the proof held with the true winner left out"
    else:
        assert bits(d["result"]) == bits(want)
    assert (0 in rows.tolist()) == (n_decoys < K_PRIME), "the construction puts the winner 1 + n_decoys-th by score'"
    eng.close()


def test_overflowing_products_are_nominated_first():
    rng = np.random.default_rng(3)
    corpus = rng.uniform(-1.0, 1.0, (3_000, 128)).astype(np.float32)
    corpus[17] = np.float32(3e38)
    eng = _engine(DOT, corpus)
    q = np.full(128, 2.0, np.float32)
    d = eng.int8_nominations(q, 5)
    sc, rows = _decode(d["keys"])
    assert rows[1] == 17 and np.isinf(sc[1]), "an overflowing score' must be nominated first"
    assert d["ok"] == 0
    eng.close()


@pytest.mark.parametrize("metric", [COS, DOT])
@pytest.mark.parametrize("dims", [128, 384, 768, 1536])
def test_route_equals_fp32_scan(oracle, metric, dims):
    n = 30_000 + dims % 7
    eng = CUDAVectorEngine(metric, dims)
    eng.fill_synthetic(400 + dims, n, normalize=metric is COS)
    _set(eng, shadow_scan_min_bytes=0, int8_scan_min_bytes=0)
    qs = oracle.synth_rows(401 + dims, 0, 3, dims, normalize=True)
    deny = list(range(0, n, 5))
    for k in (1, 10, 32):
        want = fp32(eng, lambda: [eng.search(q, k) for q in qs])
        i0, (p0, f0) = eng.counter("single_int8_queries"), counts(eng)
        got = [eng.search(q, k) for q in qs]
        assert eng.counter("single_int8_queries") - i0 == len(qs), "the int8 form did not nominate"
        assert counts(eng) == (p0 + len(qs), f0), "the int8 proof did not hold"
        assert [bits(g) for g in got] == [bits(w) for w in want], f"k={k}"
        want = fp32(eng, lambda: eng.search_filtered(qs[0], k, deny=deny))
        assert bits(eng.search_filtered(qs[0], k, deny=deny)) == bits(want)
    eng.close()


def test_selection_takes_the_shadow_that_proves():
    rng = np.random.default_rng(11)
    unit = rng.uniform(-1.0, 1.0, (20_000, 384)).astype(np.float32)
    outlier = unit.copy()
    outlier[:, 5] *= np.float32(40.0)
    q = rng.uniform(-1.0, 1.0, 384).astype(np.float32)
    for corpus, min_bytes, want_int8 in ((unit, 0, True), (outlier, 0, False), (unit, 1 << 40, False)):
        eng = _engine(COS, corpus)
        eng.set_option("int8_scan_min_bytes", min_bytes)
        i0, (p0, _) = eng.counter("single_int8_queries"), counts(eng)
        got = eng.search(q, 10)
        assert (eng.counter("single_int8_queries") - i0 == 1) == want_int8
        assert counts(eng)[0] == p0 + 1, "the route did not answer"
        assert bits(got) == bits(fp32(eng, lambda: eng.search(q, 10)))
        eng.close()


def test_appends_removes_and_overwrites():
    rng = np.random.default_rng(12)
    corpus = rng.uniform(-1.0, 1.0, (8_000, 256)).astype(np.float32)
    eng = _engine(COS, corpus)
    q = rng.uniform(-1.0, 1.0, 256).astype(np.float32)

    def same():
        i0 = eng.counter("single_int8_queries")
        got = eng.search(q, 10)
        assert eng.counter("single_int8_queries") == i0 + 1
        assert bits(got) == bits(fp32(eng, lambda: eng.search(q, 10)))
        assert eng.counter("int8_shadow_rows") == eng.count

    same()
    rho0 = eng.read_int8_shadow(0, 1)[2]
    more = rng.uniform(-1.0, 1.0, (3_000, 256)).astype(np.float32)
    more[7] = q * np.float32(5.0)
    eng.add_batch(list(range(8_000, 11_000)), more)                   # append: extends, can only raise rho_max
    same()
    assert eng.read_int8_shadow(0, 1)[2] >= rho0
    assert eng.search(q, 1)[0][0] == 8_007
    eng.remove_batch(list(range(100, 200)) + [8_007])                  # remove: prefix kept
    same()
    eng.add_batch([5], q[None, :] * np.float32(2.0))                   # overwrite: rebuilt from scratch
    same()
    assert eng.search(q, 1)[0][0] == 5
    # what the mutations left equals a shadow built from scratch over the same rows
    codes, scales, rho = eng.read_int8_shadow(0, eng.count)
    fresh = _engine(COS, eng.read_rows(0, eng.count))
    codes1, scales1, rho1 = fresh.read_int8_shadow(0, eng.count)
    assert np.array_equal(codes, codes1) and np.array_equal(scales, scales1) and rho >= rho1
    fresh.close()
    eng.close()


def _int8_routed(eng, call, n):
    """call() through the int8 form: n route queries, each nominated from the int8 shadow and proven."""
    (p0, f0), i0 = counts(eng), eng.counter("single_int8_queries")
    out = call()
    assert eng.counter("single_int8_queries") - i0 == n, "the int8 form did not nominate"
    assert counts(eng) == (p0 + n, f0), "the int8 proof did not hold"
    return out


def test_filtered_where_and_device_delivery(oracle):
    import ctypes as C
    import torch
    from test_gpu_where import _attributes
    from wax_b200 import Where, _lib as L, sharded
    n, dims, k = 200_000, 384, 10
    eng = CUDAVectorEngine(COS, dims)
    eng.fill_synthetic(500, n, id_base=3)
    _set(eng, shadow_scan_min_bytes=0, int8_scan_min_bytes=0)
    rng = np.random.default_rng(501)
    qs = oracle.synth_rows(502, 0, 3, dims, normalize=True)
    ids = np.arange(n) + 3
    deny = np.sort(rng.choice(ids, 30_000, replace=False)).tolist()
    allow = np.sort(rng.choice(ids, 40_000, replace=False)).tolist()      # above the gather size: the row bitset
    for kind, fids in (("deny", deny), ("allow", allow)):
        for kk in (1, 10, 32):
            want = fp32(eng, lambda: [eng.search_filtered(q, kk, **{kind: fids}) for q in qs])
            got = _int8_routed(eng, lambda: [eng.search_filtered(q, kk, **{kind: fids}) for q in qs], len(qs))
            assert [bits(g) for g in got] == [bits(w) for w in want], (kind, kk)
    ts, tags = _attributes(np.random.default_rng(503), n)
    eng.set_attributes(ids.astype(np.uint64), ts, tags)
    for w in (Where(after=int(ts[n // 10]), before=int(ts[n // 10 + n // 5])), Where(no_tags=3)):
        want = fp32(eng, lambda: eng.search_where(qs[0], k, w))
        assert bits(_int8_routed(eng, lambda: eng.search_where(qs[0], k, w), 1)) == bits(want)
    want = fp32(eng, lambda: [eng.search(q, k) for q in qs])
    for delivery in (1, 0):
        for inline in (1, 0):
            _set(eng, host_delivery=delivery, inline_query=inline)
            got = _int8_routed(eng, lambda: [eng.search(q, k) for q in qs], len(qs))
            assert [bits(g) for g in got] == [bits(w) for w in want], (delivery, inline)
    stream = torch.cuda.Stream()
    d_q = torch.from_numpy(qs).cuda()
    buf = torch.zeros(len(qs) * k * 24, dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()
    (p0, f0), i0 = counts(eng), eng.counter("single_int8_queries")
    rc = L.lib().wax_vs_search_device(eng.handle, C.c_void_p(d_q.data_ptr()), len(qs), k, 0, C.c_void_p(buf.data_ptr()),
                                      C.c_void_p(stream.cuda_stream))
    assert rc == 0, L.last_error()
    stream.synchronize()
    assert counts(eng) == (p0 + len(qs), f0) and eng.counter("single_int8_queries") == i0 + len(qs)
    cands = buf.cpu().numpy().view(sharded.CAND_DTYPE).reshape(len(qs), k)
    for c, w in zip(cands, want):
        assert [int(x["frame_id"]) for x in c] == [i for i, _ in w]
        assert [float(np.float32(1.0) - x["distance"]) for x in c] == [s for _, s in w]
    eng.close()


def test_refused_int8_proof_opens_the_skip_window():
    """All-ones rows code exactly (rho_max = 0, the int8 form is taken) but every row ties: the proof is refused, the fp32
    scan answers, the next SKIP eligible queries skip the route, then the int8 form is probed again."""
    dims, n, k = 384, 50_000, 10
    rng = np.random.default_rng(510)
    eng = _engine(COS, np.ones((n, dims), np.float32))
    q = unit_rows(rng, 1, dims)[0]
    ordinary = unit_rows(rng, SKIP + 1, dims)
    want_q = fp32(eng, lambda: eng.search(q, k))
    want_o = fp32(eng, lambda: [eng.search(o, k) for o in ordinary])
    i0 = eng.counter("single_int8_queries")
    assert_refused_then_skip_window(eng, q, k, ordinary, want_q, want_o)
    assert eng.counter("single_int8_queries") == i0 + 2, "the refused query and the probe after the window take int8"
    eng.close()


def test_a_coarse_corpus_gives_its_int8_shadow_back():
    rng = np.random.default_rng(520)
    corpus = rng.uniform(-1.0, 1.0, (20_000, 384)).astype(np.float32)
    corpus[:, 5] *= np.float32(40.0)                                   # an outlier dimension
    eng = _engine(COS, corpus)
    q = rng.uniform(-1.0, 1.0, 384).astype(np.float32)
    for extra in range(3):                                             # appends do not build it again
        assert bits(eng.search(q, 10)) == bits(fp32(eng, lambda: eng.search(q, 10)))
        assert eng.counter("single_int8_queries") == 0 and eng.counter("int8_shadow_bytes") == 0
        more = rng.uniform(-1.0, 1.0, (1_000, 384)).astype(np.float32)
        eng.add_batch(list(range(100_000 + 1_000 * extra, 101_000 + 1_000 * extra)), more)
    # overwriting rows measures the bound anew: with every outlier row rewritten the int8 form is taken again
    eng.add_batch(list(range(20_000)), rng.uniform(-1.0, 1.0, (20_000, 384)).astype(np.float32))
    assert bits(eng.search(q, 10)) == bits(fp32(eng, lambda: eng.search(q, 10)))
    assert eng.counter("single_int8_queries") == 1 and eng.counter("int8_shadow_bytes") > 0
    eng.close()


def _ballast(leave):
    """A torch allocation that leaves `leave` bytes of device memory free (None when that much is not free)."""
    import torch
    free, _ = torch.cuda.mem_get_info()
    if free < leave + (64 << 20):
        return None
    return torch.empty(free - leave, dtype=torch.uint8, device="cuda")


@pytest.mark.parametrize("room", ["both", "bf16_only", "int8_only"])
def test_single_then_batched_on_a_grown_corpus_keeps_the_routes_the_memory_allows(oracle, room):
    """A 1 M x 384 corpus grown by appends (capacity above the live rows), then device memory filled so that, beyond the
    engines' headroom (max(2 GiB, 10 % of the device)), there is room for both shadows, for the bf16 shadow alone, or
    for the int8 shadow alone.  A single query, then a batch, then a single query again: the bf16 shadow must keep every
    byte it would have had without the int8 one (so the batch nominates in bf16 whenever it fits), and a bf16 shadow that
    does not fit must not turn the int8 form off."""
    import torch
    n, dims = 1_000_000, 384
    rng = np.random.default_rng(530)
    eng = CUDAVectorEngine(COS, dims)
    for first in range(0, n, 125_000):
        eng.add_batch(list(range(first, first + 125_000)), rng.uniform(-1.0, 1.0, (125_000, dims)).astype(np.float32))
    qs = oracle.synth_rows(531, 0, 16, dims, normalize=True)
    want = fp32(eng, lambda: [eng.search(q, 10) for q in qs[:2]])   # search scratch before the free memory is measured
    assert eng.counter("int8_shadow_bytes") == 0 and eng.counter("shadow_bytes") == 0
    torch.cuda.synchronize()
    total = torch.cuda.mem_get_info()[1]
    headroom = max(2 << 30, total // 10)
    bf16, int8 = n * dims * 2, n * (dims + 4)
    leave = headroom + {"both": bf16 + int8 + (400 << 20), "bf16_only": bf16 + int8 // 2,
                        "int8_only": int8 + (bf16 - int8) // 2}[room]
    ballast = _ballast(leave)
    if ballast is None:
        pytest.skip("not enough free device memory for this layout")
    try:
        (p0, _), i0 = counts(eng), eng.counter("single_int8_queries")
        assert bits(eng.search(qs[0], 10)) == bits(want[0])
        b0 = eng.counter("batch_bf16_queries")
        eng.search_batch(qs, 10)
        assert bits(eng.search(qs[1], 10)) == bits(want[1])
        (p1, _), i1 = counts(eng), eng.counter("single_int8_queries")
        bf16_batch = eng.counter("batch_bf16_queries") - b0
        if room == "both":
            assert i1 - i0 == 2 and p1 - p0 == 2 and bf16_batch == 16 and eng.counter("shadow_unavailable") == 0
        elif room == "bf16_only":                          # the int8 shadow gives way: the parent's layout
            assert i1 - i0 == 0 and p1 - p0 == 2 and bf16_batch == 16 and eng.counter("shadow_unavailable") == 0
            assert eng.counter("int8_shadow_bytes") == 0
        else:                                              # no bf16 shadow: the batch in TF32, single queries on int8
            assert i1 - i0 == 2 and p1 - p0 == 2 and bf16_batch == 0 and eng.counter("shadow_unavailable") == 1
    finally:
        del ballast
        torch.cuda.empty_cache()
        eng.close()
