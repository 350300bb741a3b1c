"""CPU: the host model of a where's group clause (Where.passes with a frame's group), the binding's packing of the group
lists, and the argument errors of the group entry points that fire without a device."""
import ctypes as C

import numpy as np
import pytest

from wax_b200 import Where
from wax_b200 import _lib
from wax_b200.engine import _WhereArgs, group_offsets


def test_passes_requires_one_of_the_groups():
    w = Where(groups=(7, 9, 9))
    assert w.passes(0, 0, group=7) and w.passes(0, 0, group=9)
    assert not w.passes(0, 0, group=8)
    assert Where().passes(0, 0, group=8)                                   # no clause: any group
    assert Where(groups=()).passes(0, 0)                                   # an empty list is no clause
    with pytest.raises(ValueError):
        w.passes(0, 0)                                                     # the clause needs the frame's group


def test_group_clause_is_anded_with_the_other_clauses():
    w = Where(after=10, before=20, no_tags=1, terms=(5,), groups=(3,))
    assert w.passes(15, 0, terms=[5], group=3)
    assert not w.passes(15, 1, terms=[5], group=3)                         # tag
    assert not w.passes(25, 0, terms=[5], group=3)                         # time
    assert not w.passes(15, 0, terms=[], group=3)                          # terms
    assert not w.passes(15, 0, terms=[5], group=4)                         # group
    assert not Where(groups=((1 << 64) - 1,)).passes(0, 0, group=0)           # an id no row carries matches nothing


def test_group_offsets_pack_every_where_in_order():
    wheres = [Where(groups=(4, 2, 4)), Where(), Where(groups=((1 << 64) - 1,)), Where(after=3)]
    off, ids = group_offsets(wheres)
    assert off.dtype == np.uint64 and ids.dtype == np.uint64
    assert off.tolist() == [0, 3, 3, 4, 4]
    assert ids.tolist() == [4, 2, 4, (1 << 64) - 1]                        # duplicates kept: the engine drops them
    off, ids = group_offsets([])
    assert off.tolist() == [0] and ids.size == 0


def test_where_args_select_the_group_entry_only_when_a_group_is_asked():
    a = _WhereArgs([Where(), Where(terms=(1,))], [0, 1], None, None, 2)
    assert not a.with_groups and a.with_terms
    b = _WhereArgs([Where(), Where(groups=(1,))], [0, 1], None, None, 2)
    assert b.with_groups and not b.with_terms
    assert b.near and b.warr is b.warr_near                                 # the group entries read wax_vs_where_near
    off, ids = b.group_args()
    assert C.cast(off, C.c_void_p).value is not None and C.cast(ids, C.c_void_p).value is not None
    assert b.goff.tolist() == [0, 0, 1]
    empty = _WhereArgs([Where(groups=())], [0], None, None, 1)
    assert empty.group_args()[1] is None                                    # no ids: NULL, which the ABI allows


def test_entries_refuse_a_null_engine_without_a_device():
    L = _lib.lib()
    out_n = (C.c_uint32 * 1)()
    assert L.wax_vs_search_batch_where_groups(None, None, 0, 0, 1, None, None, None, 0, None, None, 0, None, None, None,
                                              None, None, None, None, 0, out_n) == _lib.ERR_NULL
    assert L.wax_vs_search_batch_grouped_multi_where_groups(None, None, 0, 0, 1, 1, None, None, None, 0, None, None, 0,
                                                            None, None, None, None, None, None, 0, out_n) == _lib.ERR_NULL
