"""CPU: ShardedVectorEngine.rebalance() on gloo ranks (world 2 and 3), each rank's engine a list-based stand-in with the
keyed engine's semantics, side columns included.  After every step of seeded add / set / skew / rebalance scripts the
rows per rank, the rows moved, the MV2V bytes and every row's group, attributes, location and terms equal what one
engine with the same history holds; an injected failure in one receiver loses and duplicates nothing."""
import os
import socket
import sys
from pathlib import Path

import numpy as np
import pytest

from helpers import EngineModel

ROOT = Path(__file__).resolve().parents[1]
DIMS = 4
DEFAULT_LOC = (-(1 << 31), 0)


def _bin(lat, lon):
    if np.isnan(lat) or np.isnan(lon):
        return DEFAULT_LOC
    return int(np.floor(lat * 100)), int(np.floor(lon * 100))


class ColumnStore:
    """One rank's store on lists with the keyed engine's semantics (wax_vs_add_batch_keyed, wax_vs_remove_batch,
    wax_vs_export_rows, wax_vs_set_*), plus the three rank-level rebalance entries (wax_vs_export_rows_device,
    wax_vs_export_columns, wax_vs_absorb_rows).  A column is "set" once its setter has been called, as on the engine."""

    def __init__(self, dims=DIMS, fail_absorb_at=None):
        self.dims, self.ids, self.vecs, self.keys = dims, [], [], []
        self.groups, self.attrs, self.locs, self.terms = {}, {}, {}, {}     # by frame id, only once set
        self.set_bits = 0
        self.fail_absorb_at, self.absorbs = fail_absorb_at, 0

    @property
    def count(self):
        return len(self.ids)

    def contains(self, ids):
        held = set(self.ids)
        return np.array([int(i) in held for i in np.asarray(ids, np.uint64).reshape(-1)], bool)

    def add_batch_keyed(self, ids, vecs, first_key):
        assert not self.keys or first_key > self.keys[-1]
        appended = 0
        for i, v in zip(np.asarray(ids, np.uint64).tolist(), np.asarray(vecs, np.float32)):
            if i in self.ids:
                self.vecs[self.ids.index(i)] = v.copy()
            else:
                self.ids.append(i), self.vecs.append(v.copy()), self.keys.append(first_key + appended)
                appended += 1
        return appended

    def remove_batch(self, ids):
        gone = set(np.asarray(ids, np.uint64).tolist()) & set(self.ids)
        keep = [j for j, i in enumerate(self.ids) if i not in gone]
        self.ids, self.vecs, self.keys = [self.ids[j] for j in keep], [self.vecs[j] for j in keep], [self.keys[j] for j in keep]
        for col in (self.groups, self.attrs, self.locs, self.terms):
            for i in gone:
                col.pop(i, None)
        return len(gone)

    def export_rows(self, first, n, vectors=True):
        vecs = np.array(self.vecs[first:first + n], np.float32).reshape(n, self.dims) if vectors else None
        return (np.array(self.ids[first:first + n], np.uint64), vecs, np.array(self.keys[first:first + n], np.uint64))

    def _setter(self, bit, col, ids, values):
        self.set_bits |= bit
        held, named = set(self.ids), set()
        for i, v in zip(np.asarray(ids, np.uint64).tolist(), values):
            if i in held:
                col[i] = v
                named.add(i)
        return len(named)

    def set_groups(self, ids, groups):
        return self._setter(1, self.groups, ids, [int(g) for g in groups])

    def set_attributes(self, ids, timestamps=None, tags=None):
        ids = np.asarray(ids, np.uint64).tolist()
        old = [self.attrs.get(i, (0, 0)) for i in ids]
        vals = [(int(timestamps[j]) if timestamps is not None else old[j][0], int(tags[j]) if tags is not None else old[j][1])
                for j in range(len(ids))]
        return self._setter(2, self.attrs, ids, vals)

    def set_locations(self, ids, lats, lons):
        return self._setter(4, self.locs, ids, [_bin(a, b) for a, b in zip(lats, lons)])

    def set_terms(self, ids, lists):
        return self._setter(8, self.terms, ids, [tuple(sorted(set(int(x) for x in t))) for t in lists])

    def columns_of(self, i):
        return (self.groups.get(i, i), self.attrs.get(i, (0, 0)), self.locs.get(i, DEFAULT_LOC), self.terms.get(i, ()))

    # -- the rank-level rebalance entries
    def export_vectors(self, first, n):
        import torch
        return torch.from_numpy(np.array(self.vecs[first:first + n], np.float32).reshape(n, self.dims))

    def export_columns(self, first, n):
        from wax_b200.engine import ROW_COLUMNS_DTYPE, RowColumns
        recs = np.zeros(n, ROW_COLUMNS_DTYPE)
        lists = []
        for j, i in enumerate(self.ids[first:first + n]):
            g, (ts, tags), (lat, lon), terms = self.columns_of(i)
            recs[j] = (g, ts, tags, lat, lon)
            lists.append(terms)
        offsets = np.zeros(n + 1, np.uint64)
        offsets[1:] = np.cumsum([len(t) for t in lists])
        return RowColumns(self.set_bits, recs, offsets, np.array([x for t in lists for x in t], np.uint64))

    def absorb_rows(self, ids, keys, vectors, columns):
        self.absorbs += 1
        if self.absorbs == self.fail_absorb_at:
            from wax_b200.engine import InvalidToc
            raise InvalidToc("injected absorb failure")
        ids, keys = np.asarray(ids, np.uint64).tolist(), np.asarray(keys, np.uint64).tolist()
        assert all(b > a for a, b in zip(keys, keys[1:])) and not set(keys) & set(self.keys) and not set(ids) & set(self.ids)
        vecs = vectors.numpy()
        rows = sorted(list(zip(self.keys, self.ids, self.vecs)) + [(k, i, vecs[j].copy()) for j, (k, i) in
                                                                   enumerate(zip(keys, ids))], key=lambda t: t[0])
        self.keys, self.ids, self.vecs = [r[0] for r in rows], [r[1] for r in rows], [r[2] for r in rows]
        bits = int(columns.set)
        for j, i in enumerate(ids):
            rec, terms = columns.records[j], columns.terms[columns.term_offsets[j]:columns.term_offsets[j + 1]]
            if bits & 1:
                self.groups[i] = int(rec["group"])
            if bits & 2:
                self.attrs[i] = (int(rec["timestamp"]), int(rec["tags"]))
            if bits & 4:
                self.locs[i] = (int(rec["lat_bin"]), int(rec["lon_bin"]))
            if bits & 8:
                self.terms[i] = tuple(int(x) for x in terms)
        self.set_bits |= bits


class ColumnModel(EngineModel):
    """One engine's rows and side columns (defaults for rows never given one)."""

    def __init__(self):
        super().__init__(None, 0, DIMS)
        self.cols = {}

    def add_batch(self, ids, vecs):
        super().add_batch(ids, vecs)
        for i in ids:
            self.cols.setdefault(int(i), [int(i), (0, 0), DEFAULT_LOC, ()])

    def remove(self, i):
        super().remove(i)
        self.cols.pop(int(i), None)

    def blob(self):
        from wax_b200 import sharded
        ids = np.array(self.ids, np.uint64)
        return (sharded.mv2v_header(0, DIMS, len(self.ids)) + self.corpus().tobytes() + np.uint64(ids.size * 8).tobytes() +
                ids.tobytes())


def script(rng, world):
    """(op, args): adds with upserts and in-batch duplicates, the four setters, skews, rebalances."""
    ops, nxt, live = [], 0, []

    def add(n_new, n_up):
        nonlocal nxt
        ids = list(range(nxt, nxt + n_new)) + ([int(x) for x in rng.choice(live, n_up)] if live and n_up else [])
        nxt += n_new
        ids += [int(x) for x in rng.choice(ids, 3)]                # in-batch duplicates
        ops.append(("add", ids, rng.integers(-3, 4, (len(ids), DIMS)).astype(np.float32)))
        live.extend(i for i in range(nxt - n_new, nxt))

    def setters():
        pick = [int(x) for x in rng.choice(live, max(1, len(live) // 2), replace=False)] + [10 ** 9]
        ops.append(("groups", pick, [int(g) for g in rng.integers(0, 7, len(pick))]))
        ops.append(("attrs", pick, (rng.integers(0, 1000, len(pick)).tolist(), rng.integers(0, 16, len(pick)).tolist())))
        lat = rng.uniform(-80, 80, len(pick))
        lat[::5] = np.nan
        ops.append(("locs", pick, (lat.tolist(), rng.uniform(-170, 170, len(pick)).tolist())))
        ops.append(("terms", pick, [[int(x) for x in rng.integers(0, 30, rng.integers(0, 5))] for _ in pick]))

    add(60, 0)
    add(40, 10)
    setters()
    ops.append(("rebalance", None, None))
    ops.append(("skew_rank", int(rng.integers(0, world)), None))      # all of one rank's rows
    ops.append(("rebalance", None, None))
    add(30, 5)
    lo = int(rng.integers(0, nxt // 2))
    ops.append(("remove", list(range(lo, lo + nxt // 3)), None))      # a key range
    ops.append(("rebalance", None, None))
    setters()
    ops.append(("skew_all_but", int(rng.integers(0, world)), None))   # all but one rank's rows
    ops.append(("rebalance", None, None))
    add(25, 5)
    ops.append(("rebalance", None, None))
    return ops


def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def _check_columns(eng, store, model, world):
    """Every rank's rows carry the columns one engine would give them (gathered on every rank)."""
    import torch.distributed as dist
    mine = {i: store.columns_of(i) for i in store.ids}
    every = [None] * world
    dist.all_gather_object(every, mine)
    union = {}
    for part in every:
        assert not set(part) & set(union), "a row is held twice"
        union.update(part)
    assert sorted(union) == sorted(model.cols)
    for i, c in union.items():
        g, a, loc, terms = model.cols[i]
        assert c == (g, a, loc, terms), (i, c, model.cols[i])


def _worker(rank, world, port, seed, chunk_rows, fail, out_dir):
    import torch.distributed as dist
    sys.path.insert(0, str(ROOT))
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        import wax_b200
        from wax_b200 import sharded
        store = ColumnStore(fail_absorb_at=fail[1] if fail and fail[0] == rank else None)
        eng = sharded.ShardedVectorEngine(wax_b200.VectorMetric.cosine, DIMS, local_store=store)
        model = ColumnModel()
        rng = np.random.default_rng(seed)
        raised = []
        for step, (op, ids, arg) in enumerate(script(rng, world)):
            if op == "add":
                model.add_batch(ids, arg)
                eng.add_batch(ids, arg)
            elif op in ("groups", "attrs", "locs", "terms"):
                fn = {"groups": eng.set_groups, "attrs": eng.set_attributes, "locs": eng.set_locations,
                      "terms": eng.set_terms}[op]
                fn(ids, *(arg if isinstance(arg, tuple) else (arg,)))
                for j, i in enumerate(ids):
                    if i not in model.cols:
                        continue
                    c = model.cols[i]
                    if op == "groups":
                        c[0] = arg[j]
                    elif op == "attrs":
                        c[1] = (arg[0][j], arg[1][j])
                    elif op == "locs":
                        c[2] = _bin(arg[0][j], arg[1][j])
                    else:
                        c[3] = tuple(sorted(set(arg[j])))
            elif op in ("remove", "skew_rank", "skew_all_but"):
                if op == "remove":
                    gone = ids
                else:
                    every = [None] * world
                    dist.all_gather_object(every, list(store.ids))
                    gone = [i for r, part in enumerate(every) for i in part if (r == ids) == (op == "skew_rank")]
                before = len(model.ids)
                for i in gone:
                    model.remove(i)
                assert eng.remove_batch(gone) == before - len(model.ids)
            else:
                counts = eng._counts.copy()
                targets, moves = sharded.plan_rebalance(counts)
                fid = [None]
                if moves:                                  # the first row the first move takes, named by its donor
                    d, r, _ = moves[0]
                    if rank == d:
                        fid[0] = store.ids[int(counts[d]) - sum(m[2] for m in moves if m[0] == d)]
                    dist.broadcast_object_list(fid, src=d)
                try:
                    moved = eng.rebalance(chunk_rows=chunk_rows)
                except wax_b200.WaxError as exc:
                    raised.append(str(exc))
                    moved = None
                got = [None] * world
                dist.all_gather_object(got, (moved, store.count))
                assert eng._counts.tolist() == [g[1] for g in got]
                if moved is not None:
                    assert [g[0] for g in got] == [sum(m[2] for m in moves)] * world, got
                    assert [g[1] for g in got] == targets.tolist(), (got, targets)
                    assert eng.rebalance(chunk_rows=chunk_rows) == 0
                if moves and moved is not None:            # an upsert and a remove of a moved frame reach its new owner
                    assert (fid[0] in store.ids) == (rank == moves[0][1])
                    vec = np.full((1, DIMS), 9.0, np.float32)
                    model.add_batch(fid, vec)
                    eng.add_batch(fid, vec)
                    blob = eng.serialize()
                    if rank == 0:
                        assert bytes(blob) == model.blob()
                    model.remove(fid[0])
                    assert eng.remove_batch(fid) == 1
                    assert fid[0] not in store.ids
            assert eng.count() == len(model.ids)
            assert all(b > a for a, b in zip(store.keys, store.keys[1:]))
            blob = eng.serialize(chunk_rows=5)
            if rank == 0:
                assert bytes(blob) == model.blob(), step
            _check_columns(eng, store, model, world)
        np.save(Path(out_dir) / f"r{rank}.npy", np.array([len(raised)]))
        if raised:
            (Path(out_dir) / f"why{rank}.txt").write_text(raised[0])
    finally:
        dist.destroy_process_group()


@pytest.mark.parametrize("world,seed,chunk_rows", [(2, 0, None), (2, 1, 7), (3, 2, None), (3, 3, 5)])
def test_rebalance_keeps_every_answer_of_one_engine(tmp_path, world, seed, chunk_rows):
    import torch.multiprocessing as mp
    mp.spawn(_worker, args=(world, _free_port(), seed, chunk_rows, None, str(tmp_path)), nprocs=world, join=True)
    assert all(int(np.load(tmp_path / f"r{r}.npy")[0]) == 0 for r in range(world))


@pytest.mark.parametrize("world,fail", [(2, (1, 2)), (3, (2, 1))])
def test_a_failed_absorb_loses_and_duplicates_nothing(tmp_path, world, fail):
    """One receiver fails in its absorb (chunks of 3 rows, so it fails mid-move): every rank raises the same error with
    that rank's reason, the rows it merged before stay with it, the rest stay on the donors; the columns and the MV2V
    bytes still equal one engine's after every step."""
    import torch.multiprocessing as mp
    mp.spawn(_worker, args=(world, _free_port(), 11, 3, fail, str(tmp_path)), nprocs=world, join=True)
    counts = [int(np.load(tmp_path / f"r{r}.npy")[0]) for r in range(world)]
    assert counts == [1] * world
    whys = {(tmp_path / f"why{r}.txt").read_text() for r in range(world)}
    assert len(whys) == 1 and f"rank {fail[0]}" in whys.pop()
