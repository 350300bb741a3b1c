"""CPU: the host model of a where's root clause (Where.passes with the frame's group's root-tag word), the binding's
packing and choice of entry, the argument errors that fire without a device, the sharded engine's refusal, and a model
showing that the clause is PhotoRAG's root test after ranking."""
import ctypes as C

import numpy as np
import pytest

from wax_b200 import Where
from wax_b200 import _lib
from wax_b200.engine import _WhereArgs, root_clauses

IS_ROOT, DELETED, SUPERSEDED = 1, 2, 4
PHOTO = Where(root_all_tags=IS_ROOT, root_no_tags=DELETED | SUPERSEDED)


def test_passes_tests_the_root_tag_word():
    assert PHOTO.passes(0, 0, root_tags=IS_ROOT)
    assert PHOTO.passes(0, 0, root_tags=IS_ROOT | 8)                        # other bits are the caller's
    assert not PHOTO.passes(0, 0, root_tags=IS_ROOT | DELETED)
    assert not PHOTO.passes(0, 0, root_tags=IS_ROOT | SUPERSEDED)
    assert not PHOTO.passes(0, 0, root_tags=0)                               # a root without meta never got IS_ROOT
    assert Where().passes(0, 0)                                              # (0, 0): no clause, no word needed
    assert Where(root_no_tags=DELETED).passes(0, 0, root_tags=0)             # a group never given a word has 0
    assert not Where(root_all_tags=3, root_no_tags=1).passes(0, 0, root_tags=3)   # overlapping bits admit nothing
    with pytest.raises(ValueError):
        PHOTO.passes(0, 0)                                                   # the clause needs the group's word
    assert not Where().has_root_clause and Where(root_no_tags=1).has_root_clause


def test_root_clause_is_anded_with_every_other_clause():
    w = Where(after=10, before=20, no_tags=1, terms=(5,), groups=(3,), near=(48.85, 2.35, 5000.0),
              root_all_tags=IS_ROOT, root_no_tags=DELETED)
    loc = (4885, 235)
    assert w.passes(15, 0, loc, terms=[5], group=3, root_tags=IS_ROOT)
    assert not w.passes(15, 0, loc, terms=[5], group=3, root_tags=IS_ROOT | DELETED)   # root
    assert not w.passes(15, 1, loc, terms=[5], group=3, root_tags=IS_ROOT)             # tag
    assert not w.passes(25, 0, loc, terms=[5], group=3, root_tags=IS_ROOT)             # time
    assert not w.passes(15, 0, loc, terms=[], group=3, root_tags=IS_ROOT)              # terms
    assert not w.passes(15, 0, loc, terms=[5], group=4, root_tags=IS_ROOT)             # group
    assert not w.passes(15, 0, None, terms=[5], group=3, root_tags=IS_ROOT)            # location


def test_root_clauses_pack_every_where_in_order():
    arr = root_clauses([PHOTO, Where(), Where(root_no_tags=(1 << 64) - 1)])
    assert C.sizeof(_lib.RootClause) == 16
    assert [(r.all_tags, r.no_tags) for r in arr] == [(IS_ROOT, DELETED | SUPERSEDED), (0, 0), (0, (1 << 64) - 1)]
    assert len(root_clauses([])) == 1                                        # never a zero-length array


def test_where_args_select_the_roots_entry_only_when_a_root_clause_is_asked():
    a = _WhereArgs([Where(), Where(groups=(1,))], [0, 1], None, None, 2)
    assert not a.with_roots and a.with_groups
    b = _WhereArgs([Where(), PHOTO], [0, 1], None, None, 2)
    assert b.with_roots and not b.with_groups and not b.with_terms
    assert b.near and b.warr is b.warr_near                                  # the roots entries read wax_vs_where_near
    (roots,) = b.root_args()
    got = C.cast(roots, C.POINTER(_lib.RootClause))
    assert [(got[i].all_tags, got[i].no_tags) for i in range(2)] == [(0, 0), (IS_ROOT, DELETED | SUPERSEDED)]
    assert b.group_args()[1] is None and b.goff.tolist() == [0, 0, 0]       # no group ids: NULL, which the ABI allows


def test_entries_refuse_a_null_engine_without_a_device():
    L = _lib.lib()
    out_n = (C.c_uint32 * 1)()
    assert L.wax_vs_search_batch_where_roots(None, None, 0, 0, 1, None, None, None, 0, None, None, 0, None, None, None,
                                             None, None, None, None, None, 0, out_n) == _lib.ERR_NULL
    assert L.wax_vs_search_batch_grouped_multi_where_roots(None, None, 0, 0, 1, 1, None, None, None, 0, None, None, 0,
                                                           None, None, None, None, None, None, None, 0,
                                                           out_n) == _lib.ERR_NULL
    g = (C.c_uint64 * 1)(5)
    assert L.wax_vs_set_root_tags(None, g, g, 1, None) == _lib.ERR_NULL
    assert "engine is NULL" in _lib.last_error()


def test_the_sharded_engine_refuses_a_root_clause():
    from wax_b200.sharded import ShardedVectorEngine
    eng = ShardedVectorEngine.__new__(ShardedVectorEngine)                   # the refusal comes before any collective
    eng.dimensions = 4
    eng._torch = eng._dist = None
    q = np.zeros((1, 4), np.float32)
    with pytest.raises(ValueError, match="no root clause"):
        eng.search_batch_where(q, 10, [PHOTO], [0])
    with pytest.raises(ValueError, match="no root clause"):
        eng.search_batch_grouped(q, 10, 1, wheres=[PHOTO], query_where=[0])


def _photo_rag_loop(ranked, parent_of, meta, limit):
    """PhotoRAGOrchestrator's grouping over a ranked frame list (:264-308): each hit's root is parentId ?? id, a root
    with no meta, not a root, deleted or superseded is dropped, and the best hit per root is kept until `limit` roots."""
    out, seen = [], set()
    for fid, _ in ranked:
        root = parent_of.get(fid, fid)
        m = meta.get(root)
        if m is None or m["kind"] != "root" or m["deleted"] or m["superseded_by"] is not None:
            continue
        if root in seen:
            continue
        seen.add(root)
        out.append(root)
        if len(out) == limit:
            break
    return out


def test_the_clause_is_photo_rags_root_test_over_an_exhaustive_ranking():
    rng = np.random.default_rng(1)
    n_roots, per = 300, 6
    frames, parent_of, meta = [], {}, {}
    for r in range(n_roots):
        root = 10_000 + r * 100
        kinds = rng.random()
        if kinds < 0.05:                                                     # a root with no meta at all
            pass
        else:
            meta[root] = {"kind": "root" if rng.random() > 0.05 else "derived", "deleted": rng.random() < 0.05,
                          "superseded_by": (root + 1) if rng.random() < 0.1 else None}
        frames.append(root)
        for j in range(1, per):
            frames.append(root + j)
            parent_of[root + j] = root
    scores = rng.standard_normal(len(frames))
    ranked = sorted(zip(frames, scores), key=lambda t: -t[1])              # exhaustive: every frame, best first
    words = {}
    for root, m in meta.items():                                             # the bindings' FrameMeta -> word
        words[root] = ((IS_ROOT if m["kind"] == "root" else 0) | (DELETED if m["deleted"] else 0) |
                       (SUPERSEDED if m["superseded_by"] is not None else 0))
    for limit in (1, 12, 50, n_roots):
        want = _photo_rag_loop(ranked, parent_of, meta, limit)
        got, seen = [], set()                                                # grouped search under the root clause
        for fid, _ in ranked:
            root = parent_of.get(fid, fid)
            if not PHOTO.passes(0, 0, group=root, root_tags=words.get(root, 0)) or root in seen:
                continue
            seen.add(root)
            got.append(root)
            if len(got) == limit:
                break
        assert got == want, limit
