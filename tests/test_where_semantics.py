"""CPU: the frame-attribute predicates of wax_vs_search_batch_where / wax_vs_search_batch_grouped_where -- their meaning,
pinned against a numpy restatement of Wax's post-filter, and the argument checks that run before any CUDA call."""
import ctypes as C

import numpy as np
import pytest

from wax_b200 import Where
from wax_b200 import _lib as L

I64_MIN, I64_MAX = np.iinfo(np.int64).min, np.iinfo(np.int64).max
DELETED, SUPERSEDED, SURROGATE = 1 << 0, 1 << 1, 1 << 2          # caller-fixed bits, as INTEGRATION.md assigns them


def passes_frame_filter(ts, tags, after, before, include_deleted, include_superseded, include_surrogates):
    """The time and flag clauses of UnifiedSearch.passesFrameFilter (Sources/Wax/UnifiedSearch/UnifiedSearch.swift:
    1241-1258) over arrays: timeRange.contains (SearchRequest.swift:100-103: `timestamp < after` and
    `timestamp >= before` fail, a nil bound does not test), then status == .deleted, supersededBy != nil and
    kind == "surrogate" each excluded unless included -- here as tag bits."""
    ok = np.ones(ts.shape, bool)
    if after is not None:
        ok &= ~(ts < after)
    if before is not None:
        ok &= ~(ts >= before)
    if not include_deleted:
        ok &= (tags & DELETED) == 0
    if not include_superseded:
        ok &= (tags & SUPERSEDED) == 0
    if not include_surrogates:
        ok &= (tags & SURROGATE) == 0
    return ok


def where_for(after, before, include_deleted, include_superseded, include_surrogates):
    """The mapping INTEGRATION.md documents: a nil bound is INT64_MIN / INT64_MAX, includeX == false puts X's bit in
    no_tags."""
    no = (0 if include_deleted else DELETED) | (0 if include_superseded else SUPERSEDED) | \
         (0 if include_surrogates else SURROGATE)
    return Where(after=I64_MIN if after is None else after, before=I64_MAX if before is None else before, no_tags=no)


def evaluate(where, ts, tags):
    return np.array([where.passes(int(t), int(g)) for t, g in zip(ts, tags)], bool)


def test_where_restates_the_time_and_flag_clauses_of_passes_frame_filter():
    rng = np.random.default_rng(7)
    edges = np.array([I64_MIN, I64_MIN + 1, -1, 0, 1, 99, 100, 101, I64_MAX - 1, I64_MAX], np.int64)
    ts = np.concatenate([edges, rng.integers(-1000, 1000, 300, dtype=np.int64)])
    tags = rng.integers(0, 16, ts.size).astype(np.uint64)
    bounds = [None, I64_MIN, -1, 0, 100, 101, I64_MAX - 1]
    for after in bounds:
        for before in bounds + [None]:
            for flags in [(True, True, True), (False, True, True), (False, False, False), (True, False, True)]:
                want = passes_frame_filter(ts, tags.astype(np.int64), after, before, *flags)
                if before == I64_MAX:          # a non-nil Int64.max bound excludes Int64.max itself; the C bound cannot
                    continue
                got = evaluate(where_for(after, before, *flags), ts, tags)
                assert (got == want).all(), (after, before, flags)


def test_where_edges():
    ts = np.array([I64_MIN, -5, 0, 5, I64_MAX], np.int64)
    tags = np.zeros(ts.size, np.uint64)
    assert evaluate(Where(), ts, tags).all()                                   # the defaults bound nothing
    assert evaluate(Where(before=I64_MAX), ts, tags)[-1]                        # INT64_MAX passes "no upper bound"
    assert evaluate(Where(after=I64_MIN), ts, tags)[0]
    assert not evaluate(Where(after=5, before=5), ts, tags).any()               # after == before admits nothing
    assert not evaluate(Where(after=6, before=5), ts, tags).any()
    assert list(evaluate(Where(after=-5, before=5), ts, tags)) == [False, True, True, False, False]
    t = np.array([0b011, 0b001, 0b110, 0], np.uint64)
    z = np.zeros(4, np.int64)
    assert list(evaluate(Where(all_tags=0b001), z, t)) == [True, True, False, False]
    assert list(evaluate(Where(no_tags=0b100), z, t)) == [True, True, False, True]
    assert not evaluate(Where(all_tags=0b001, no_tags=0b001), z, t).any()      # overlapping masks admit nothing
    assert list(evaluate(Where(all_tags=1 << 63), z, np.array([1 << 63, 0, 0, 0], np.uint64))) == [True, False, False, False]


def test_where_struct_layout():
    assert C.sizeof(L.Where) == 32
    assert [L.Where.after.offset, L.Where.before.offset, L.Where.all_tags.offset, L.Where.no_tags.offset] == [0, 8, 16, 24]


# ---- argument checks: they return before the engine is locked or any CUDA call is made, so a placeholder handle (a
# zeroed block the library never reads on these paths) stands in for an engine on a CPU-only box
_placeholder = (C.c_uint8 * (1 << 16))()
ENG = C.cast(_placeholder, C.c_void_p)


def _where_call(eng=ENG, n_queries=2, frame_ids=None, offsets=(0,), modes=(), query_filter=None, wheres=(Where(),),
                query_where=(0, 0), out_n=True):
    q = np.zeros(n_queries * 4, np.float32)
    off = np.asarray(offsets, np.uint64)
    md = np.asarray(modes, np.int32)
    qf = None if query_filter is None else np.asarray(query_filter, np.uint32)
    qw = None if query_where is None else np.asarray(query_where, np.uint32)
    warr = None if wheres is None else (L.Where * max(len(wheres), 1))(*[w.to_c() for w in wheres])
    fids = None if frame_ids is None else np.asarray(frame_ids, np.uint64)
    ns = np.zeros(max(n_queries, 1), np.uint32)
    ids = np.zeros(64, np.uint64)
    sc = np.zeros(64, np.float32)
    p = lambda a, t: None if a is None else a.ctypes.data_as(C.POINTER(t))
    return L.lib().wax_vs_search_batch_where(
        eng, p(q, C.c_float), n_queries, 4, 10, p(fids, C.c_uint64), p(off, C.c_uint64), p(md, C.c_int32) if md.size else None,
        len(modes), p(qf, C.c_uint32), None if warr is None else C.cast(warr, C.c_void_p), 0 if wheres is None else len(wheres),
        p(qw, C.c_uint32), p(ids, C.c_uint64), p(sc, C.c_float), 32, p(ns, C.c_uint32) if out_n else None)


def test_search_batch_where_argument_checks():
    nf = [L.NO_FILTER, L.NO_FILTER]
    assert _where_call(eng=None, query_filter=nf) == L.ERR_NULL
    assert _where_call(query_filter=nf, out_n=False) == L.ERR_NULL
    assert _where_call(query_filter=None) == L.ERR_NULL                                  # query_filter NULL, n > 0
    assert _where_call(query_filter=nf, query_where=None) == L.ERR_NULL                  # query_where NULL, n > 0
    assert _where_call(query_filter=nf, query_where=(0, 1)) == L.ERR_ARGUMENT            # where 1 of 1
    assert "names where 1 of 1" in L.last_error()
    assert _where_call(query_filter=nf, wheres=(), query_where=(0, L.NO_FILTER)) == L.ERR_ARGUMENT
    assert _where_call(query_filter=[0, L.NO_FILTER]) == L.ERR_ARGUMENT                  # filter 0 of 0
    assert _where_call(offsets=(0, 1), modes=(2,), frame_ids=[5], query_filter=[0, 0]) == L.ERR_ARGUMENT   # bad mode
    assert _where_call(offsets=(1, 1), modes=(0,), frame_ids=[5], query_filter=[0, 0]) == L.ERR_ARGUMENT   # offsets[0]
    assert _where_call(offsets=(0, 2, 1), modes=(0, 0), frame_ids=[5, 6], query_filter=[0, 1]) == L.ERR_ARGUMENT
    assert _where_call(offsets=(0, 2), modes=(0,), frame_ids=None, query_filter=[0, 0]) == L.ERR_NULL     # ids NULL


def _grouped_call(eng=ENG, where=True, per_group=2, top_groups=5, mode=1, n_ids=0):
    q = np.zeros(8, np.float32)
    w = Where().to_c()
    ids = np.zeros(64, np.uint64)
    sc = np.zeros(64, np.float32)
    gr = np.zeros(64, np.uint64)
    ns = np.zeros(2, np.uint32)
    p = lambda a, t: a.ctypes.data_as(C.POINTER(t))
    return L.lib().wax_vs_search_batch_grouped_where(
        eng, p(q, C.c_float), 2, 4, top_groups, per_group, None, n_ids, mode,
        C.cast(C.pointer(w), C.c_void_p) if where else None, p(ids, C.c_uint64), p(sc, C.c_float), p(gr, C.c_uint64), 32,
        p(ns, C.c_uint32))


def test_search_batch_grouped_where_argument_checks():
    assert _grouped_call(where=False) == L.ERR_NULL
    assert "where is NULL" in L.last_error()
    assert _grouped_call(eng=None) == L.ERR_NULL
    assert _grouped_call(per_group=0) == L.ERR_ARGUMENT
    assert _grouped_call(per_group=L.MAX_PER_GROUP + 1) == L.ERR_ARGUMENT
    assert _grouped_call(top_groups=10_000, per_group=2) == L.ERR_ARGUMENT
    assert _grouped_call(mode=3) == L.ERR_ARGUMENT
    assert _grouped_call(n_ids=3) == L.ERR_NULL                                          # frame_ids NULL, n_ids > 0


def test_set_attributes_argument_checks():
    lib = L.lib()
    out = C.c_uint64(7)
    assert lib.wax_vs_set_attributes(None, None, None, None, 0, C.byref(out)) == L.ERR_NULL
    assert lib.wax_vs_set_attributes(ENG, None, None, None, 0, C.byref(out)) == L.OK and out.value == 0   # n == 0
    assert lib.wax_vs_set_attributes(ENG, None, None, None, 3, None) == L.ERR_NULL                       # ids NULL
