"""Term clauses on the host (no GPU): TermDictionary and Where.passes against a transcription of Wax's
UnifiedSearch.matches(metadataFilter:meta:), and the argument checks of wax_vs_set_terms and
wax_vs_search_batch_where_terms, which return before any device use."""
from __future__ import annotations

import ctypes as C
import itertools
import random

import numpy as np

from wax_b200 import TermDictionary, Where
from wax_b200 import _lib as L


# ---- UnifiedSearch.swift:1215-1239, transcribed -----------------------------------------------------------------------
def swift_matches(required_entries, required_tags, required_labels, metadata, tags, labels) -> bool:
    """metadata: dict or None (a nil meta.metadata); tags: [(key, value)]; labels: [str]."""
    if required_entries:
        if metadata is None:
            return False
        for key, value in required_entries.items():
            if metadata.get(key) != value:
                return False
    if required_tags:
        for rk, rv in required_tags:
            if not any(k == rk and v == rv for k, v in tags):
                return False
    if required_labels:
        for label in required_labels:
            if label not in labels:
                return False
    return True


def engine_matches(d: TermDictionary, frame, flt) -> bool:
    metadata, tags, labels = frame
    terms = d.frame_terms(metadata, tags, labels)
    return Where(terms=d.filter_terms(*flt)).passes(0, 0, None, terms)


KEYS, VALUES = ["session_id", "kind", "k2"], ["a", "b", "c"]
FRAMES = [
    (None, [], []),                                                   # nil metadata, nothing else
    ({}, [], []),                                                     # empty metadata
    ({"session_id": "a"}, [], []),
    ({"session_id": "b", "kind": "a"}, [("kind", "a")], ["a"]),
    (None, [("session_id", "a")], ["session_id"]),                    # the same strings as a tag and a label
    ({"session_id": "a", "kind": "b", "k2": "c"}, [("k2", "c"), ("k2", "a")], ["b", "c"]),
    ({"kind": "a"}, [("session_id", "a"), ("session_id", "a")], ["a", "a"]),   # duplicate tags and labels
]
FILTERS = [
    ({}, [], []),                                                     # empty requirement lists
    ({"session_id": "a"}, [], []),
    ({"session_id": "b"}, [], []),                                    # one key, another candidate value
    ({"session_id": "a", "kind": "b"}, [], []),
    ({}, [("kind", "a")], []),
    ({}, [("session_id", "a")], []),
    ({}, [("kind", "a"), ("kind", "a")], []),                         # duplicate requirements
    ({}, [], ["a"]),
    ({}, [], ["a", "a", "b"]),
    ({}, [], ["session_id"]),
    ({"session_id": "a"}, [("k2", "c")], ["b"]),                      # all three kinds
    ({"session_id": "zz"}, [], []),                                   # a value no frame was given
    ({}, [("nope", "x")], ["nope"]),
]


def test_listed_cases_match_swift():
    d = TermDictionary()
    for frame in FRAMES:                     # frames are interned before the filters are looked up, as in a store
        d.frame_terms(*frame)
    for frame, flt in itertools.product(FRAMES, FILTERS):
        assert engine_matches(d, frame, flt) == swift_matches(*flt, *frame), (frame, flt)


def test_random_metadata_matches_swift():
    rng = random.Random(11)
    d = TermDictionary()

    def rand_frame():
        metadata = None if rng.random() < 0.2 else {k: rng.choice(VALUES) for k in rng.sample(KEYS, rng.randint(0, 3))}
        tags = [(rng.choice(KEYS), rng.choice(VALUES)) for _ in range(rng.randint(0, 3))]
        labels = [rng.choice(VALUES + KEYS) for _ in range(rng.randint(0, 3))]
        return metadata, tags, labels

    def rand_filter():
        entries = {k: rng.choice(VALUES) for k in rng.sample(KEYS, rng.choice([0, 0, 1, 1, 2]))}
        tags = [(rng.choice(KEYS), rng.choice(VALUES)) for _ in range(rng.choice([0, 0, 1, 2]))]
        labels = [rng.choice(VALUES + KEYS) for _ in range(rng.choice([0, 0, 1, 2]))]
        return entries, tags, labels

    frames = [rand_frame() for _ in range(300)]
    for f in frames:
        d.frame_terms(*f)
    hits = 0
    for _ in range(400):
        flt = rand_filter()
        for frame in frames[:60]:
            want = swift_matches(*flt, *frame)
            hits += want
            assert engine_matches(d, frame, flt) == want, (frame, flt)
    assert hits > 100                      # both answers occur


def test_dictionary_interns_exactly():
    d = TermDictionary()
    a = d.intern("entry", "session_id", "a")
    assert d.intern("entry", "session_id", "a") == a
    ids = {a, d.intern("tag", "session_id", "a"), d.intern("label", "session_id"), d.intern("entry", "session_i", "da"),
           d.intern("entry", "session_id", "b")}
    assert len(ids) == 5 and len(d) == 5                 # kinds, keys and values never collide
    assert d.lookup("entry", "nope", "x") == TermDictionary.UNKNOWN
    assert TermDictionary.UNKNOWN not in ids
    assert d.filter_terms({"session_id": "a"}, [("session_id", "a")], ["x"]) == tuple(sorted({a, 1, TermDictionary.UNKNOWN}))
    assert d.filter_terms() == ()
    try:
        d.intern("entry", "only-a-key")
    except ValueError:
        pass
    else:
        raise AssertionError("an entry needs a key and a value")


def test_where_terms_on_the_host():
    w = Where(terms=(3, 5, 5))
    assert w.passes(0, 0, None, [5, 3, 9]) and not w.passes(0, 0, None, [5]) and not w.passes(0, 0, None, None)
    assert Where().passes(0, 0, None, None)              # an empty list is no clause
    assert not Where(after=1, terms=(3,)).passes(0, 0, None, [3])


# ---- argument checks: they return before the engine is locked or any CUDA call is made, so a placeholder handle (a
# zeroed block the library never reads on these paths) stands in for an engine on a CPU-only box
_placeholder = (C.c_uint8 * (1 << 16))()
ENG = C.cast(_placeholder, C.c_void_p)
u64 = lambda *v: (C.c_uint64 * max(len(v), 1))(*v)


def test_set_terms_argument_checks():
    lib = L.lib()
    out = C.c_uint64(7)
    assert lib.wax_vs_set_terms(None, u64(1), u64(0, 1), u64(5), 1, C.byref(out)) == L.ERR_NULL
    assert lib.wax_vs_set_terms(ENG, u64(1), None, u64(5), 1, C.byref(out)) == L.ERR_NULL and out.value == 0
    assert lib.wax_vs_set_terms(ENG, None, u64(0, 1), u64(5), 1, None) == L.ERR_NULL          # ids NULL
    assert lib.wax_vs_set_terms(ENG, u64(1), u64(0, 1), None, 1, None) == L.ERR_NULL          # terms NULL
    assert lib.wax_vs_set_terms(ENG, u64(1), u64(1, 1), u64(5), 1, None) == L.ERR_ARGUMENT    # offsets[0] != 0
    assert "must be 0" in L.last_error()
    assert lib.wax_vs_set_terms(ENG, u64(1, 2), u64(0, 2, 1), u64(5, 6), 2, None) == L.ERR_ARGUMENT   # decreasing
    assert "decrease" in L.last_error()
    assert lib.wax_vs_set_terms(ENG, None, u64(0), None, 0, C.byref(out)) == L.OK and out.value == 0   # n == 0


def _terms_call(eng=ENG, offsets=(0, 1), terms=(5,), n_wheres=1, query_where=(0, 0), out_n=True):
    q = np.zeros(2 * 4, np.float32)
    foff = np.zeros(1, np.uint64)
    qf = np.full(2, L.NO_FILTER, np.uint32)
    qw = None if query_where is None else np.asarray(query_where, np.uint32)
    warr = (L.WhereNear * max(n_wheres, 1))(*[Where().to_c_near() for _ in range(n_wheres)])
    toff = None if offsets is None else np.asarray(offsets, np.uint64)
    tl = None if terms is None else np.asarray(terms, np.uint64)
    ns = np.zeros(2, np.uint32)
    ids = np.zeros(64, np.uint64)
    sc = np.zeros(64, np.float32)
    p = lambda a, t: None if a is None else a.ctypes.data_as(C.POINTER(t))
    return L.lib().wax_vs_search_batch_where_terms(
        eng, p(q, C.c_float), 2, 4, 10, None, p(foff, C.c_uint64), None, 0, p(qf, C.c_uint32), C.cast(warr, C.c_void_p),
        n_wheres, p(qw, C.c_uint32), p(toff, C.c_uint64), p(tl, C.c_uint64), p(ids, C.c_uint64), p(sc, C.c_float), 32,
        p(ns, C.c_uint32) if out_n else None)


def test_search_batch_where_terms_argument_checks():
    assert _terms_call(eng=None) == L.ERR_NULL
    assert _terms_call(out_n=False) == L.ERR_NULL
    assert _terms_call(query_where=None) == L.ERR_NULL
    assert _terms_call(query_where=(0, 1)) == L.ERR_ARGUMENT                       # where 1 of 1
    assert _terms_call(offsets=None) == L.ERR_NULL
    assert _terms_call(terms=None) == L.ERR_NULL                                   # a where has a term
    assert _terms_call(offsets=(1, 1)) == L.ERR_ARGUMENT
    assert _terms_call(offsets=(0, 2, 1), n_wheres=2, terms=(5, 6)) == L.ERR_ARGUMENT
    assert "decrease" in L.last_error()
    assert _terms_call(offsets=(0, 33), terms=tuple(range(33))) == L.ERR_ARGUMENT  # more than 32 in one where
    assert "at most 32" in L.last_error()
