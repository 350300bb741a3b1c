"""GPU: the rank-level rebalance entries (wax_vs_export_rows_device, wax_vs_export_columns, wax_vs_absorb_rows) and
ShardedVectorEngine.rebalance() against one engine with the same history.

(a) Keyed engines as ranks in one process, moved by sharded.plan_rebalance through the new entries exactly as
    ShardedVectorEngine.rebalance moves them: after every step every search form equals the single engine's, bit for bit.
(b) Every argument error of the new entries, with its code and reason, and nothing changed by a refused call.
(c) ShardedVectorEngine at world 2 under gloo, both processes on one GPU: MV2V bytes and each rank's rows and columns.
(d) 4 M x 384 rows at R = 2 on the single-query route, rebalanced in 256 MiB slabs."""
import ctypes as C
import os
import socket
import sys
from pathlib import Path

import numpy as np
import pytest

from helpers import unit_rows
from test_gpu_sharded_corpus import DIMS, KeyedRanks, _hits_bits, _merge, check_answers
from test_gpu_sharded_grouped import _bits, _run
from wax_b200 import CUDAVectorEngine, VectorMetric, WaxError, Where, sharded
from wax_b200 import _lib as L
from wax_b200.engine import _WhereArgs

pytestmark = pytest.mark.gpu
ROOT = Path(__file__).resolve().parents[1]


def move_rows(engines, chunk_rows=None):
    """plan_rebalance over `engines` through the rank-level entries: each donor's tail, in key order, to the receivers,
    in chunks; then each donor drops what it gave.  Returns the moves."""
    counts = [e.count for e in engines]
    targets, moves = sharded.plan_rebalance(counts)
    tail = list(counts)
    for d, _, n in moves:
        tail[d] -= n
    drop = {}
    for d, r, n in moves:
        step = chunk_rows or n
        for lo in range(0, n, step):
            m = min(step, n - lo)
            ids, _, keys = engines[d].export_rows(tail[d] + lo, m, vectors=False)
            engines[r].absorb_rows(ids, keys, engines[d].export_vectors(tail[d] + lo, m),
                                   engines[d].export_columns(tail[d] + lo, m))
            drop.setdefault(d, []).append(ids)
        tail[d] += n
    for d, parts in drop.items():
        engines[d].remove_batch(np.concatenate(parts))
    assert [e.count for e in engines] == targets.tolist()
    return moves


class Ranks(KeyedRanks):
    def rebalance(self):
        moves = move_rows(self.engines)
        assert not sharded.plan_rebalance([e.count for e in self.engines])[1]
        return moves

    def metadata(self, rng, frac=0.6):
        """Groups, attributes, locations and terms of a random part of the live frames, on every engine (a rank ignores
        the frames it does not hold: one that holds none keeps no column)."""
        ids = self.single.export_rows(0, self.single.count, vectors=False)[0]
        if ids.size == 0:
            return
        pick = rng.choice(ids, max(1, int(ids.size * frac)), replace=False)
        groups = pick % 11
        ts, tags = rng.integers(0, 100, pick.size), rng.integers(0, 8, pick.size).astype(np.uint64)
        lat, lon = rng.uniform(40.0, 40.2, pick.size), rng.uniform(-74.2, -74.0, pick.size)
        lat[::4], lon[::4] = np.nan, np.nan                         # no location
        terms = [[int(t) for t in rng.choice(12, rng.integers(0, 4), replace=False)] for _ in pick]
        for e in [self.single] + self.engines:
            e.set_groups(pick, groups)
            e.set_attributes(pick, ts, tags)
            e.set_locations(pick, lat, lon)
            e.set_terms(pick, terms)


WHERES = [Where(after=20, before=70), Where(all_tags=2), Where(near=(40.1, -74.1, 9000.0)), Where(terms=(3,)),
          Where(no_tags=1, terms=(1, 5))]


def check_everything(ks, qs, rng):
    """check_answers (device search, fused exchange, where, grouped) plus k = 1 and the allow, deny and per-query filters
    under time, tag, box and term clauses, and grouped search with per_group 1 and 3 under filters and wheres."""
    import torch
    check_answers(ks, qs)
    b = len(qs)
    ids = ks.single.export_rows(0, ks.single.count, vectors=False)[0]
    some = [int(x) for x in rng.choice(ids, min(ids.size, 60), replace=False)] if ids.size else []
    filters = [("allow", some), ("deny", some[:20]), ("allow", some[::3] + [10**9])]
    qf = [None if i % 4 == 3 else i % 3 for i in range(b)]
    qw = [None if i % 5 == 4 else i % len(WHERES) for i in range(b)]
    a = _WhereArgs(WHERES, qw, filters, qf, b)
    d_qs = torch.from_numpy(np.ascontiguousarray(qs, np.float32)).cuda()
    for k in (1, 10, 72, 200):
        gathered = torch.zeros(ks.world * b * k * 24, dtype=torch.uint8, device="cuda")
        for r, e in enumerate(ks.engines):
            rc = L.lib().wax_vs_search_batch_where_device(e.handle, C.c_void_p(d_qs.data_ptr()), b, k, *a.filter_args(),
                                                          *a.where_args(near=True), *a.term_args(), 0,
                                                          C.c_void_p(gathered.data_ptr() + r * b * k * 24), None)
            assert rc == 0, L.last_error()
        torch.cuda.synchronize()
        got = _merge(ks, gathered, b, k)
        want = ks.single.search_batch_where(qs, k, WHERES, qw, filters, qf)
        for i in range(b):
            assert _hits_bits(got[i]) == _hits_bits(want[i]), ("filtered where", k, i)
        if k == 1:
            for i in range(b):
                assert _hits_bits(_merge_one(ks, qs[i], 1)) == _hits_bits(ks.single.search(qs[i], 1))
    if ids.size:
        plain = [w for w in WHERES if not w.terms]
        qwg = [None if i % 4 == 0 else i % len(plain) for i in range(b)]
        for p in (1, 3):
            got = _run(ks, qs, 6, p, plain, qwg, filters, qf, check_rounds=False)
            want = ks.single.search_batch_grouped_multi_where(qs, 6, p, plain, qwg, filters, qf)
            assert [_bits(x) for x in got] == [_bits(x) for x in want], ("grouped", p)


def _merge_one(ks, q, k):
    import torch
    d_q = torch.from_numpy(np.ascontiguousarray(q, np.float32).reshape(1, -1)).cuda()
    gathered = torch.zeros(ks.world * k * 24, dtype=torch.uint8, device="cuda")
    for r, e in enumerate(ks.engines):
        rc = L.lib().wax_vs_search_device(e.handle, C.c_void_p(d_q.data_ptr()), 1, k, 0,
                                          C.c_void_p(gathered.data_ptr() + r * k * 24), None)
        assert rc == 0, L.last_error()
    torch.cuda.synchronize()
    return _merge(ks, gathered, 1, k)[0]


@pytest.mark.parametrize("metric", [VectorMetric.cosine, VectorMetric.dot, VectorMetric.l2])
@pytest.mark.parametrize("world", [2, 3, 4])
def test_ranks_moved_through_the_entries_answer_as_one_engine(world, metric):
    rng = np.random.default_rng(40 * world + metric.value)
    pool = unit_rows(rng, 30, DIMS) * (np.float32(1.5) if metric is VectorMetric.dot else np.float32(1))
    qs = np.concatenate([pool[:3], unit_rows(rng, 3, DIMS)])          # pool rows: exact ties with interleaving keys
    ks = Ranks(metric, world)
    try:
        for e in ks.engines:
            e.set_option("rebalance_slab_bytes", DIMS * 4 * 13)       # slabs of 13 rows
        ids = rng.permutation(np.arange(1, 1200)).astype(np.uint64)
        ks.add_batch(ids, pool[rng.integers(0, len(pool), ids.size)])
        up = np.concatenate([ids[:30], [5000, 5001, 5000]]).astype(np.uint64)
        ks.add_batch(up, pool[rng.integers(0, len(pool), up.size)])
        check_everything(ks, qs, rng)

        # every row of rank 0 goes; columns are set while rank 0 is empty (on the donors' side only)
        ks.remove_batch(ks.engines[0].export_rows(0, ks.engines[0].count, vectors=False)[0])
        ks.metadata(rng)
        assert ks.rebalance()
        check_everything(ks, qs, rng)
        assert bytes(ks.serialize()) == bytes(ks.single.serialize())

        # new rows without columns land on the emptiest ranks; a key range goes; rebalance
        more = np.arange(20_000, 20_300, dtype=np.uint64)
        ks.add_batch(more, pool[rng.integers(0, len(pool), more.size)])
        order = ks.single.export_rows(0, ks.single.count, vectors=False)[0]
        ks.remove_batch(order[order.size // 5: order.size * 3 // 5])
        ks.rebalance()
        check_everything(ks, qs, rng)

        # everything but the last rank goes, columns set again, then rebalance; upserts of moved frames
        keep = ks.engines[-1]
        for e in ks.engines[:-1]:
            ks.remove_batch(e.export_rows(0, e.count, vectors=False)[0])
        ks.metadata(rng, 0.3)
        ks.rebalance()
        moved = ks.engines[0].export_rows(0, min(ks.engines[0].count, 20), vectors=False)[0]
        ks.add_batch(moved, pool[rng.integers(0, len(pool), moved.size)])
        ks.remove_batch(moved[:5])
        assert keep.count and bytes(ks.serialize()) == bytes(ks.single.serialize())
        check_everything(ks, qs, rng)
    finally:
        ks.close()


def test_entries_check_their_arguments():
    import torch
    rng = np.random.default_rng(3)
    rows = unit_rows(rng, 8, DIMS)
    eng = CUDAVectorEngine(VectorMetric.cosine, DIMS)
    plain = CUDAVectorEngine(VectorMetric.cosine, DIMS)
    multi = CUDAVectorEngine(VectorMetric.cosine, DIMS, devices=[0, 0])
    lib = L.lib()
    u64 = C.POINTER(C.c_uint64)

    def raw(ids, keys, vecs, h=None):
        ids, keys = np.asarray(ids, np.uint64), np.asarray(keys, np.uint64)
        return lib.wax_vs_absorb_rows(h or eng.handle, ids.ctypes.data_as(u64), keys.ctypes.data_as(u64),
                                      C.c_void_p(vecs.data_ptr()), ids.size, 0, None, None, None)

    def refused(rc, code, reason):
        assert rc == code, (rc, L.last_error())
        assert reason in L.last_error(), L.last_error()

    try:
        assert eng.add_batch_keyed([1, 2, 3], rows[:3], 10) == 3
        before = bytes(eng.serialize())
        d = torch.from_numpy(rows[3:6]).cuda()
        refused(raw([4, 5, 6], [20, 20, 21], d), L.ERR_ARGUMENT, "keys must strictly increase")
        refused(raw([4, 5, 6], [21, 20, 22], d), L.ERR_ARGUMENT, "keys must strictly increase")
        refused(raw([4, 5, 6], [5, 11, 30], d), L.ERR_ARGUMENT, "key 11 is already held")
        refused(raw([4, 2, 6], [5, 6, 30], d), L.ERR_ARGUMENT, "frame 2 is already held")
        refused(raw([4, 7, 4], [5, 6, 30], d), L.ERR_ARGUMENT, "frame 4 appears twice")
        host = torch.from_numpy(rows[3:6].copy())
        refused(raw([4, 5, 6], [5, 6, 30], host), L.ERR_ARGUMENT, "not memory on the engine's device")
        ids3, keys3 = np.array([4, 5, 6], np.uint64), np.array([5, 6, 30], np.uint64)
        refused(lib.wax_vs_absorb_rows(eng.handle, None, keys3.ctypes.data_as(u64), C.c_void_p(d.data_ptr()), 3, 0,
                                       None, None, None), L.ERR_NULL, "NULL argument")
        refused(lib.wax_vs_absorb_rows(eng.handle, ids3.ctypes.data_as(u64), keys3.ctypes.data_as(u64), None, 3, 0,
                                       None, None, None), L.ERR_NULL, "NULL argument")
        refused(lib.wax_vs_absorb_rows(eng.handle, ids3.ctypes.data_as(u64), keys3.ctypes.data_as(u64),
                                       C.c_void_p(d.data_ptr()), 3, L.COLUMN_GROUPS, None, None, None),
                L.ERR_NULL, "columns is NULL")
        refused(lib.wax_vs_absorb_rows(eng.handle, ids3.ctypes.data_as(u64), keys3.ctypes.data_as(u64),
                                       C.c_void_p(d.data_ptr()), 3, L.COLUMN_TERMS, None, None, None),
                L.ERR_NULL, "term_offsets is NULL")
        refused(lib.wax_vs_absorb_rows(eng.handle, ids3.ctypes.data_as(u64), keys3.ctypes.data_as(u64),
                                       C.c_void_p(d.data_ptr()), 3, 16, None, None, None),
                L.ERR_ARGUMENT, "unknown column bits")
        refused(lib.wax_vs_absorb_rows(None, None, None, None, 3, 0, None, None, None), L.ERR_NULL, "engine is NULL")
        assert bytes(eng.serialize()) == before and eng.row_keys().tolist() == [10, 11, 12]

        plain.add_batch([7], rows[:1])                                 # rows without keys
        refused(raw([4], [5], d[:1], plain.handle), L.ERR_ARGUMENT, "holds rows without keys")
        assert plain.count == 1

        out = torch.zeros((3, DIMS), dtype=torch.float32, device="cuda")
        refused(lib.wax_vs_export_rows_device(eng.handle, 2, 2, C.c_void_p(out.data_ptr()), None), L.ERR_ARGUMENT,
                "row range out of bounds")
        refused(lib.wax_vs_export_rows_device(eng.handle, 0, 2, None, None), L.ERR_NULL, "d_out is NULL")
        refused(lib.wax_vs_export_columns(eng.handle, 1, 3, None, None, None, 0, None, None), L.ERR_ARGUMENT,
                "row range out of bounds")
        eng.set_terms([1, 2], [[4, 9], [1, 2, 3]])
        length = C.c_uint64(0)
        small = np.zeros(2, np.uint64)
        refused(lib.wax_vs_export_columns(eng.handle, 0, 3, None, None, small.ctypes.data_as(u64), 2, C.byref(length),
                                          None), L.ERR_BUFFER, "terms_cap 2 < 5")

        # the good call: rows 4..6 merge between the held keys, with their columns
        cols = eng.export_columns(0, 3)
        assert cols.set == L.COLUMN_TERMS and cols.term_offsets.tolist() == [0, 2, 5, 5]
        assert cols.terms.tolist() == [4, 9, 1, 2, 3] and cols.records["group"].tolist() == [1, 2, 3]
        assert (cols.records["lat_bin"] == L.NO_LOCATION).all()
        eng.absorb_rows(ids3, keys3, d, None)
        assert eng.row_keys().tolist() == [5, 6, 10, 11, 12, 30]
        assert eng.export_rows(0, 6, vectors=False)[0].tolist() == [4, 5, 1, 2, 3, 6]
        assert torch.equal(eng.export_vectors(0, 6).cpu(), torch.from_numpy(rows[[3, 4, 0, 1, 2, 5]]))

        for entry, call in (("wax_vs_absorb_rows", lambda: raw([4], [5], d[:1], multi.handle)),
                            ("wax_vs_export_rows_device",
                             lambda: lib.wax_vs_export_rows_device(multi.handle, 0, 0, C.c_void_p(out.data_ptr()), None)),
                            ("wax_vs_export_columns",
                             lambda: lib.wax_vs_export_columns(multi.handle, 0, 0, None, None, None, 0, None, None))):
            refused(call(), L.ERR_UNSUPPORTED, f"{entry} is not served by a multi-device handle")
    finally:
        for e in (eng, plain, multi):
            e.close()


# -- (c) ShardedVectorEngine.rebalance at world 2 under gloo, both ranks on one GPU
def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def _sharded_worker(rank, world, port, out_dir):
    import torch
    import torch.distributed as dist
    sys.path.insert(0, str(ROOT))
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    torch.cuda.set_device(0)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        rng = np.random.default_rng(77)
        dims = 64
        eng = sharded.ShardedVectorEngine(VectorMetric.cosine, dims, device=0)
        one = CUDAVectorEngine(VectorMetric.cosine, dims, device=0)
        eng.engine.set_option("rebalance_slab_bytes", dims * 4 * 13)
        pool = unit_rows(rng, 20, dims)
        ids = rng.permutation(np.arange(3000)).astype(np.uint64)
        vecs = pool[rng.integers(0, 20, ids.size)]
        for lo in range(0, ids.size, 500):
            eng.add_batch(ids[lo:lo + 500], vecs[lo:lo + 500])
            one.add_batch(ids[lo:lo + 500], vecs[lo:lo + 500])
        pick = ids[::2]
        for e in (eng, one):
            e.set_groups(pick, pick % 7)
            e.set_attributes(pick, (pick % 50).astype(np.int64), pick % 4)
        mine = eng.engine.export_rows(0, eng.engine.count, vectors=False)[0] if rank == 0 else np.zeros(0, np.uint64)
        gone = [None]
        gone[0] = mine[: mine.size * 9 // 10].tolist() if rank == 0 else None
        dist.broadcast_object_list(gone, src=0)
        eng.remove_batch(gone[0])
        one.remove_batch(gone[0])
        assert eng.count() == one.count
        blob = eng.serialize()
        if rank == 0:
            assert bytes(blob) == bytes(one.serialize())
        counts = eng._counts.copy()
        targets, moves = sharded.plan_rebalance(counts)
        keys_before = eng.engine.row_keys()
        moved = eng.rebalance(chunk_rows=100)
        assert moved == sum(n for _, _, n in moves) > 0
        assert eng._counts.tolist() == targets.tolist() and eng.engine.count == targets[rank]
        blob = eng.serialize()
        if rank == 0:
            assert bytes(blob) == bytes(one.serialize())
        # each rank's rows against the plan: rank 0 received the donor's lowest tail keys, merged by key
        every = [None] * world
        dist.all_gather_object(every, keys_before.tolist())
        d, r, n = moves[0]
        expect = sorted(every[rank][: targets[rank]] if rank == d else every[rank] + every[d][targets[d]:targets[d] + n])
        got_ids, _, got_keys = eng.engine.export_rows(0, eng.engine.count, vectors=False)
        assert got_keys.tolist() == expect
        cols = eng.engine.export_columns(0, eng.engine.count)
        one_ids = one.export_rows(0, one.count, vectors=False)[0]
        one_cols = one.export_columns(0, one.count)
        where = {int(f): j for j, f in enumerate(one_ids)}
        at = [where[int(f)] for f in got_ids]
        assert np.array_equal(cols.records, one_cols.records[at])
        assert cols.set == one_cols.set == L.COLUMN_GROUPS | L.COLUMN_ATTRIBUTES
        assert eng.rebalance() == 0
        np.save(Path(out_dir) / f"ok{rank}.npy", np.array([moved]))
        eng.close()
        one.close()
    finally:
        dist.destroy_process_group()


def test_sharded_engine_rebalance_under_gloo(tmp_path):
    import torch.multiprocessing as mp
    mp.spawn(_sharded_worker, args=(2, _free_port(), str(tmp_path)), nprocs=2, join=True)
    assert int(np.load(tmp_path / "ok0.npy")[0]) == int(np.load(tmp_path / "ok1.npy")[0]) > 0


# -- (d) one large case on the single-query route
class _Big:
    def __init__(self, metric, world, dims):
        self.metric, self.world, self.dims, self.next_key = metric, world, dims, 0
        self.single = CUDAVectorEngine(metric, dims)
        self.engines = [CUDAVectorEngine(metric, dims) for _ in range(world)]

    def add_batch(self, ids, rows):
        self.single.add_batch(ids, rows)
        dest, first_key, appended, self.next_key = sharded.plan_add_batch(
            ids, np.full(ids.size, -1), [e.count for e in self.engines], self.next_key)
        for r, e in enumerate(self.engines):
            mine = np.flatnonzero(dest == r)
            if mine.size:
                assert e.add_batch_keyed(ids[mine], rows[mine], int(first_key[r])) == appended[r]


def test_large_rebalance_on_the_single_query_route():
    """4 M x 384 cosine at R = 2, rank 0 cut to 0.5 M rows: the move of 0.75 M rows goes in 256 MiB chunks through the
    entries, each merged in the default 256 MiB slabs; single queries and a batch equal one engine's before and after."""
    rng = np.random.default_rng(21)
    dims, n, chunk = 384, 4_000_000, 1_000_000
    big = _Big(VectorMetric.cosine, 2, dims)
    try:
        for lo in range(0, n, chunk):
            big.add_batch(np.arange(lo, lo + chunk, dtype=np.uint64), rng.standard_normal((chunk, dims), dtype=np.float32))
        r0 = big.engines[0].export_rows(0, big.engines[0].count, vectors=False)[0]
        gone = r0[: r0.size - 500_000]
        big.single.remove_batch(gone)
        big.engines[0].remove_batch(gone)
        assert [e.count for e in big.engines] == [500_000, 2_000_000]
        qs = rng.standard_normal((6, dims)).astype(np.float32)

        def same():
            for q in qs:
                assert _hits_bits(_merge_one(big, q, 10)) == _hits_bits(big.single.search(q, 10))

        def route_queries():
            return sum(e.counter(c) for e in big.engines
                       for c in ("single_shadow_queries", "single_int8_queries", "single_u4_queries"))

        seen = route_queries()
        same()
        assert route_queries() > seen
        moves = move_rows(big.engines, chunk_rows=(256 << 20) // (4 * dims))
        assert moves == [(1, 0, 750_000)]
        seen = route_queries()
        same()
        assert route_queries() > seen
    finally:
        for e in [big.single] + big.engines:
            e.close()
