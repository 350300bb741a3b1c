"""CPU: the corpus planning of the row-sharded engine (wax_b200/sharded.py: plan_add_batch, plan_serialize, the MV2V
slices of deserialize) against the single engine's mutation semantics on plain lists, and the collective choreography of
ShardedVectorEngine's corpus methods on two gloo ranks with a CPU stand-in for each rank's engine."""
import os
import socket
import sys
from pathlib import Path

import numpy as np
import pytest

from helpers import EngineModel

ROOT = Path(__file__).resolve().parents[1]
DIMS = 4


class ListStore:
    """One rank's store on lists, with the keyed engine's semantics (wax_vs_add_batch_keyed, wax_vs_remove_batch,
    wax_vs_deserialize_rows, wax_vs_export_rows): upsert in place, append with the next key, order-preserving remove."""

    def __init__(self, dims=DIMS):
        self.dims, self.ids, self.vecs, self.keys = dims, [], [], []

    @property
    def count(self):
        return len(self.ids)

    def contains(self, ids):
        held = set(self.ids)
        return np.array([int(i) in held for i in np.asarray(ids, np.uint64).reshape(-1)], bool)

    def add_batch_keyed(self, ids, vecs, first_key):
        assert not self.keys or first_key > self.keys[-1], "first key not above the last key"
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
        return len(gone)

    def deserialize_rows(self, blob, first, n):
        count, dims = int(np.frombuffer(blob, np.uint64, 1, 12)[0]), int(np.frombuffer(blob, np.uint32, 1, 8)[0])
        assert bytes(blob[:4]) == b"MV2V" and dims == self.dims and first + n <= count
        vecs = np.frombuffer(blob, np.float32, count * dims, 36).reshape(count, dims)
        ids = np.frombuffer(blob, np.uint64, count, 44 + count * dims * 4)
        self.ids = ids[first:first + n].tolist()
        self.vecs = [v.copy() for v in vecs[first:first + n]]
        self.keys = list(range(first, first + n))

    def export_rows(self, first, n, vectors=True):
        vecs = np.array(self.vecs[first:first + n], np.float32).reshape(n, self.dims) if vectors else None
        return (np.array(self.ids[first:first + n], np.uint64), vecs, np.array(self.keys[first:first + n], np.uint64))


def model_blob(model, similarity=0):
    from wax_b200 import sharded
    corpus = model.corpus()
    ids = np.array(model.ids, np.uint64)
    return (sharded.mv2v_header(similarity, model.dims, len(model.ids)) + corpus.tobytes() +
            np.uint64(ids.size * 8).tobytes() + ids.tobytes())


class PlannedRanks:
    """`world` ListStores driven by the planning functions, as ShardedVectorEngine drives its ranks."""

    def __init__(self, world):
        self.ranks, self.next_key = [ListStore() for _ in range(world)], 0

    def add_batch(self, ids, vecs):
        from wax_b200 import sharded
        ids = np.asarray(ids, np.uint64)
        owner = np.full(ids.size, -1, np.int64)
        for r, st in enumerate(self.ranks):
            owner[st.contains(ids)] = r
        counts = [st.count for st in self.ranks]
        dest, first_key, appended, self.next_key = sharded.plan_add_batch(ids, owner, counts, self.next_key)
        for r, st in enumerate(self.ranks):
            mine = np.flatnonzero(dest == r)
            got = st.add_batch_keyed(ids[mine], vecs[mine], int(first_key[r])) if mine.size else 0
            assert got == appended[r]
        return counts, appended

    def remove_batch(self, ids):
        return sum(st.remove_batch(ids) for st in self.ranks)

    def reload(self, blob):
        from wax_b200 import sharded
        count = sharded.mv2v_count(blob)
        for r, st in enumerate(self.ranks):
            lo, hi = sharded.shard_range(count, len(self.ranks), r)
            st.deserialize_rows(blob, lo, hi - lo)
        self.next_key = count

    def check(self, model):
        """Keys increase on every rank; rows in key order are the model's rows in position order; plan_serialize agrees."""
        from wax_b200 import sharded
        for st in self.ranks:
            assert all(b > a for a, b in zip(st.keys, st.keys[1:])), st.keys
            assert all(k < self.next_key for k in st.keys)
        rows = sorted((k, i, v) for st in self.ranks for k, i, v in zip(st.keys, st.ids, st.vecs))
        assert [i for _, i, _ in rows] == model.ids
        assert all(np.array_equal(v, w) for (_, _, v), w in zip(rows, model.rows))
        pos = sharded.plan_serialize([np.array(st.keys, np.uint64) for st in self.ranks])
        order = [None] * len(model.ids)
        for st, p in zip(self.ranks, pos):
            for i, j in zip(st.ids, p):
                order[j] = i
        assert order == model.ids


def random_script(rng, steps):
    """(op, args): add_batch with upserts and in-batch duplicates, remove_batch with unknown and repeated ids, reload."""
    next_id, live, script = 0, [], []
    for _ in range(steps):
        op = rng.choice(["add", "add", "add", "remove", "reload"])
        if op == "add":
            n_new, n_up = int(rng.integers(0, 40)), int(rng.integers(0, 10)) if live else 0
            ids = list(range(next_id, next_id + n_new)) + [int(x) for x in rng.choice(live, n_up)] if live else \
                list(range(next_id, next_id + n_new))
            next_id += n_new
            ids += [int(x) for x in rng.choice(ids, int(rng.integers(0, 4)))] if ids else []     # in-batch duplicates
            ids = [int(x) for x in rng.permutation(ids)] if rng.random() < 0.5 else ids
            if rng.random() < 0.2:
                ids = [i + 1_000_000 for i in ids[:5]] + ids        # ids out of order
            script.append(("add", ids, rng.standard_normal((len(ids), DIMS)).astype(np.float32)))
            live = sorted(set(live) | set(ids))
        elif op == "remove" and live:
            gone = [int(x) for x in rng.choice(live, int(rng.integers(1, max(2, len(live) // 3))))] + [10**9]
            script.append(("remove", gone, None))
            live = sorted(set(live) - set(gone))
        else:
            script.append(("reload", None, None))
    return script


@pytest.mark.parametrize("seed", range(6))
@pytest.mark.parametrize("world", [1, 2, 3, 4])
def test_planned_ranks_follow_the_single_engine(world, seed):
    rng = np.random.default_rng(1000 * world + seed)
    model, ranks = EngineModel(None, 0, DIMS), PlannedRanks(world)
    for op, ids, vecs in random_script(rng, 14):
        if op == "add":
            model.add_batch(ids, vecs)
            ranks.add_batch(ids, vecs)
        elif op == "remove":
            before = len(model.ids)
            for i in ids:
                model.remove(i)
            assert ranks.remove_batch(ids) == before - len(model.ids)
        else:
            ranks.reload(model_blob(model))
        ranks.check(model)


def test_new_ids_fill_the_emptiest_ranks_in_contiguous_chunks():
    from wax_b200 import sharded
    assert sharded.fill_emptiest([5, 0, 3], 4).tolist() == [0, 4, 0]
    assert sharded.fill_emptiest([2, 2, 2], 4).tolist() == [2, 1, 1]
    assert sharded.fill_emptiest([9, 0], 3).tolist() == [0, 3]
    ids = np.array([7, 1, 2, 1, 3, 4, 5], np.uint64)         # 7 is held by rank 0; 1 repeats
    dest, first_key, appended, nxt = sharded.plan_add_batch(ids, [0, -1, -1, -1, -1, -1, -1], [4, 1, 2], 10)
    # five distinct new ids (1, 2, 3, 4, 5) -> keys 10..14; the levels: rank 1 takes 3, rank 2 takes 2
    assert appended.tolist() == [0, 3, 2] and nxt == 15
    assert dest.tolist() == [0, 1, 1, 1, 1, 2, 2]
    assert first_key.tolist()[1:] == [10, 13]


def test_serialize_positions_follow_keys():
    from wax_b200 import sharded
    pos = sharded.plan_serialize([np.array([0, 4, 5], np.uint64), np.array([], np.uint64), np.array([1, 2, 9], np.uint64)])
    assert [p.tolist() for p in pos] == [[0, 3, 4], [], [1, 2, 5]]


# -- two gloo ranks: the collectives of ShardedVectorEngine's corpus methods, with ListStore as each rank's engine
def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def _worker(rank, world, port, script, out_dir):
    import torch.distributed as dist
    sys.path.insert(0, str(ROOT))
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        import wax_b200
        from wax_b200 import sharded
        store = ListStore()
        eng = sharded.ShardedVectorEngine(wax_b200.VectorMetric.cosine, DIMS, local_store=store)
        model = EngineModel(None, 0, DIMS)
        for step, (op, ids, vecs) in enumerate(script):
            if op == "add":
                model.add_batch(ids, vecs)
                eng.add_batch(ids, vecs)
            elif op == "remove":
                before = len(model.ids)
                for i in ids:
                    model.remove(i)
                assert eng.remove_batch(ids) == before - len(model.ids)
            else:
                eng.deserialize(model_blob(model))
            assert eng.count() == len(model.ids)
            assert all(b > a for a, b in zip(store.keys, store.keys[1:]))
            blob = eng.serialize(chunk_rows=7)
            if rank == 0:
                assert bytes(blob) == model_blob(model), step
            else:
                assert blob is None
        np.save(Path(out_dir) / f"n{rank}.npy", np.array([store.count]))
    finally:
        dist.destroy_process_group()


def test_two_rank_corpus_methods_equal_one_engine(tmp_path):
    import torch.multiprocessing as mp
    rng = np.random.default_rng(5)
    script = random_script(rng, 12)
    mp.spawn(_worker, args=(2, _free_port(), script, str(tmp_path)), nprocs=2, join=True)
    counts = [int(np.load(tmp_path / f"n{r}.npy")[0]) for r in range(2)]
    assert sum(counts) > 0
