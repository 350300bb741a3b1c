"""GPU: the corpus methods of the row-sharded engine (DESIGN.md section 4.15).  The ranks are keyed engines on one device,
driven by the planning functions of wax_b200/sharded.py exactly as ShardedVectorEngine drives them; one engine takes the
same history.  After every step of seeded scripts (add_batch with upserts and in-batch duplicates, remove_batch, reload
from the MV2V bytes) every sharded answer must equal the single engine's, bit for bit: frame ids, order and score bits,
for the device search with the device merge, the fused exchange, the sharded where search and the sharded grouped
search.  The rows repeat a few vectors, so exact ties abound and their keys interleave across the ranks."""
import ctypes as C
import threading

import numpy as np
import pytest

from helpers import unit_rows
from test_gpu_sharded_grouped import _bits, _run
from wax_b200 import CUDAVectorEngine, VectorMetric, WaxError, Where, sharded
from wax_b200 import _lib as L
from wax_b200.engine import _WhereArgs

pytestmark = pytest.mark.gpu

DIMS = 128
POISON = 0xAB


def _hits_bits(hits):
    return [(f, np.float32(s).view(np.uint32).item()) for f, s in hits]


class KeyedRanks:
    """`world` keyed engines connected as a shard group (row offset 0), and one engine with the same history."""

    def __init__(self, metric, world):
        self.metric, self.world, self.next_key = metric, world, 0
        self.single = CUDAVectorEngine(metric, DIMS)
        self.engines = [CUDAVectorEngine(metric, DIMS) for _ in range(world)]
        self.ranges = [(0, 0)] * world                       # row offsets for the device entry points: keys are global
        for e in [self.single] + self.engines:
            e.set_option("shard_timeout_ms", 8000)
            if metric is VectorMetric.l2:
                e.set_option("batch_l2", 1)
        blobs = [e.shard_open(r, world, 0) for r, e in enumerate(self.engines)]
        for e in self.engines:
            e.shard_connect(blobs)

    def add_batch(self, ids, vecs):
        ids = np.asarray(ids, np.uint64)
        self.single.add_batch(ids, vecs)
        owner = np.full(ids.size, -1, np.int64)
        for r, e in enumerate(self.engines):
            owner[e.contains(ids)] = r
        dest, first_key, appended, self.next_key = sharded.plan_add_batch(
            ids, owner, [e.count for e in self.engines], self.next_key)
        for r, e in enumerate(self.engines):
            mine = np.flatnonzero(dest == r)
            if mine.size:
                assert e.add_batch_keyed(ids[mine], vecs[mine], int(first_key[r])) == appended[r]

    def remove_batch(self, ids):
        want = self.single.remove_batch(ids)
        assert sum(e.remove_batch(ids) for e in self.engines) == want

    def serialize(self):
        """The MV2V bytes of the ranks, rows placed by key (ShardedVectorEngine.serialize without the transport)."""
        keys = [e.row_keys() for e in self.engines]
        for k in keys:
            assert np.all(np.diff(k.astype(np.int64)) > 0)
        pos = sharded.plan_serialize(keys)
        total = sum(len(k) for k in keys)
        ids, vecs = np.zeros(total, np.uint64), np.zeros((total, DIMS), np.float32)
        for e, p in zip(self.engines, pos):
            ids[p], vecs[p], _ = e.export_rows(0, e.count)
        return (sharded.mv2v_header(self.metric.to_vec_similarity(), DIMS, total) + vecs.tobytes() +
                np.uint64(total * 8).tobytes() + ids.tobytes())

    def reload(self, blob):
        self.single.deserialize(blob)
        count = sharded.mv2v_count(blob)
        for r, e in enumerate(self.engines):
            lo, hi = sharded.shard_range(count, self.world, r)
            e.deserialize_rows(blob, lo, hi - lo)
        self.next_key = count

    def label(self):
        """Attributes and groups of every live frame, derived from its id, on every engine (ranks ignore the others)."""
        ids = self.single.export_rows(0, self.single.count, vectors=False)[0]
        if ids.size == 0:
            return
        for e in [self.single] + self.engines:
            e.set_attributes(ids, (ids % 97).astype(np.int64), ids % 4)
            e.set_groups(ids, ids % 13)

    def collective(self, fn):
        out, errors = [None] * self.world, []

        def work(r):
            try:
                out[r] = fn(r, self.engines[r])
            except Exception as exc:  # noqa: BLE001
                errors.append((r, exc))
        threads = [threading.Thread(target=work, args=(r,)) for r in range(self.world)]
        [t.start() for t in threads]; [t.join() for t in threads]
        assert not errors, errors[:1]
        return out

    def close(self):
        for e in self.engines:
            e.shard_close()
        for e in [self.single] + self.engines:
            e.close()


def _merge(ks, gathered, b, k):
    import torch
    out = torch.full((b * k * 24,), POISON, dtype=torch.uint8, device="cuda")
    assert L.lib().wax_vs_merge_candidates_device(ks.single.handle, C.c_void_p(gathered.data_ptr()), ks.world, b, k, k,
                                                  C.c_void_p(out.data_ptr()), None) == 0, L.last_error()
    torch.cuda.synchronize()
    best = out.cpu().numpy().view(sharded.CAND_DTYPE).reshape(b, k)
    sim = ks.metric.to_vec_similarity()
    return [[(int(x["frame_id"]), float(s)) for x, s in zip(row, sharded.score_from_distance(sim, row["distance"]))
             if x["valid"]] for row in best]


def check_answers(ks, qs):
    """Every sharded form against the single engine, bit for bit."""
    import torch
    b, n = len(qs), ks.single.count
    d_qs = torch.from_numpy(np.ascontiguousarray(qs, np.float32)).cuda()
    for k in (10, 72, 200):                                             # device search + device merge
        gathered = torch.full((ks.world * b * k * 24,), POISON, dtype=torch.uint8, device="cuda")
        for r, e in enumerate(ks.engines):
            rc = L.lib().wax_vs_search_device(e.handle, C.c_void_p(d_qs.data_ptr()), b, k, 0,
                                              C.c_void_p(gathered.data_ptr() + r * b * k * 24), None)
            assert rc == 0, L.last_error()
        torch.cuda.synchronize()
        merged = _merge(ks, gathered, b, k)
        for i in range(b):
            assert _hits_bits(merged[i]) == _hits_bits(ks.single.search(qs[i], k)), ("device", k, i)
    if n:
        for k in (10, 72):                                              # the fused exchange
            for i in range(min(b, 3)):
                res = ks.collective(lambda r, e: e.shard_search(qs[i], k))
                assert all(x == res[0] for x in res)
                assert _hits_bits(res[0]) == _hits_bits(ks.single.search(qs[i], k)), ("fused", k, i)
    wheres = [Where(after=10, before=60), Where(no_tags=1), Where(all_tags=2, after=30)]
    qw = [i % 3 for i in range(b)]
    a = _WhereArgs(wheres, qw, None, None, b)
    for k in (10, 200):                                                 # sharded where search
        gathered = torch.full((ks.world * b * k * 24,), POISON, dtype=torch.uint8, device="cuda")
        for r, e in enumerate(ks.engines):
            rc = L.lib().wax_vs_search_batch_where_device(e.handle, C.c_void_p(d_qs.data_ptr()), b, k, *a.filter_args(),
                                                          *a.where_args(near=True), *a.term_args(), 0,
                                                          C.c_void_p(gathered.data_ptr() + r * b * k * 24), None)
            assert rc == 0, L.last_error()
        torch.cuda.synchronize()
        merged = _merge(ks, gathered, b, k)
        want = ks.single.search_batch_where(qs, k, wheres, qw)
        for i in range(b):
            assert _hits_bits(merged[i]) == _hits_bits(want[i]), ("where", k, i)
    if n:
        for g, p in ((5, 3), (12, 1)):                                  # sharded grouped search
            got = _run(ks, qs, g, p, wheres, qw, None, [None] * b, check_rounds=False)
            want = ks.single.search_batch_grouped_multi_where(qs, g, p, wheres, qw, None, [None] * b)
            assert [_bits(x) for x in got] == [_bits(x) for x in want], ("grouped", g, p)


def _script(rng, pool, steps):
    """add_batch with upserts, in-batch duplicates and out-of-order ids, remove_batch with unknown and repeated ids, and
    reload from the engines' own bytes; every vector is one of `pool`'s rows."""
    next_id, live, out = 0, [], []
    for step in range(steps):
        op = "add" if step < 2 else rng.choice(["add", "add", "remove", "reload"])
        if op == "add":
            ids = list(range(next_id, next_id + int(rng.integers(200, 900))))
            next_id += len(ids)
            if live:
                ids += [int(x) for x in rng.choice(live, 50)]
            ids += [int(x) for x in rng.choice(ids, 5)]
            if rng.random() < 0.5:
                ids = [int(x) for x in rng.permutation(ids)]
            out.append(("add", ids, pool[rng.integers(0, len(pool), len(ids))]))
            live = sorted(set(live) | set(ids))
        elif op == "remove":
            gone = [int(x) for x in rng.choice(live, len(live) // 4)] + [10**9]
            out.append(("remove", gone, None))
            live = sorted(set(live) - set(gone))
        else:
            out.append(("reload", None, None))
    return out


@pytest.mark.parametrize("world,metric", [(1, VectorMetric.cosine), (2, VectorMetric.cosine), (3, VectorMetric.l2),
                                          (4, VectorMetric.dot), (4, VectorMetric.cosine)])
def test_keyed_ranks_answer_as_one_engine_after_every_step(world, metric):
    rng = np.random.default_rng(300 + world)
    pool = unit_rows(rng, 40, DIMS) * (np.float32(1.5) if metric is VectorMetric.dot else np.float32(1))
    qs = np.concatenate([pool[:3], unit_rows(rng, 3, DIMS)])          # pool rows: exact ties at the top
    ks = KeyedRanks(metric, world)
    interleaved = False
    try:
        for op, ids, vecs in _script(rng, pool, 6):
            if op == "add":
                ks.add_batch(ids, vecs)
            elif op == "remove":
                ks.remove_batch(ids)
            else:
                ks.reload(ks.serialize())
            assert bytes(ks.serialize()) == bytes(ks.single.serialize())
            spans = sorted((int(k[0]), int(k[-1])) for k in (e.row_keys() for e in ks.engines) if k.size)
            interleaved |= any(a[1] > b[0] for a, b in zip(spans, spans[1:]))     # a rank's keys run past the next's
            ks.label()
            check_answers(ks, qs)
        assert interleaved or world == 1
    finally:
        ks.close()


def test_interleaved_tied_rows_merge_by_row():
    """The device merges order a tie by global row wherever the rows live: ranks whose rows interleave (keyed shards)
    and lists whose distances are all equal.  The merge of contiguous shards cannot tell these apart."""
    import torch
    rng = np.random.default_rng(91)
    eng = CUDAVectorEngine(VectorMetric.cosine, 8)
    try:
        for world, b, k in [(2, 7, 10), (4, 5, 72), (3, 4, 128)]:
            rows = rng.permutation(world * b * k).astype(np.uint64).reshape(world, b, k)
            cands = np.zeros((world, b, k), sharded.CAND_DTYPE)
            cands["distance"] = np.round(rng.random((world, b, k)), 1).astype(np.float32)
            cands["row"], cands["frame_id"], cands["valid"] = rows, rows * np.uint64(3) + np.uint64(1), 1
            for r in range(world):
                for q in range(b):
                    cands[r, q] = cands[r, q][np.lexsort((cands[r, q]["row"], cands[r, q]["distance"]))]
            dev = torch.from_numpy(cands.view(np.uint8).reshape(-1).copy()).cuda()
            out = torch.zeros(b * k * 24, dtype=torch.uint8, device="cuda")
            assert L.lib().wax_vs_merge_candidates_device(eng.handle, C.c_void_p(dev.data_ptr()), world, b, k, k,
                                                          C.c_void_p(out.data_ptr()), None) == 0, L.last_error()
            torch.cuda.synchronize()
            want, _ = sharded.merge_candidates_batch(cands, k)
            assert np.array_equal(out.cpu().numpy().view(sharded.CAND_DTYPE).reshape(b, k), want), (world, b, k)
    finally:
        eng.close()


def test_duplicate_vectors_with_interleaved_keys_across_ranks():
    """Two ranks hold copies of one vector, their keys alternating: every form must list the copies in key order."""
    rng = np.random.default_rng(17)
    v = unit_rows(rng, 1, DIMS)[0]
    other = unit_rows(rng, 300, DIMS)
    ks = KeyedRanks(VectorMetric.cosine, 2)
    try:
        ids = np.arange(400, dtype=np.uint64)
        vecs = np.concatenate([np.repeat(v[None], 100, 0), other])[rng.permutation(400)]
        for lo in range(0, 400, 50):                       # eight batches: each fills the emptier rank in turn
            ks.add_batch(ids[lo:lo + 50], vecs[lo:lo + 50])
        ks.remove_batch(ids[::7])
        ks.label()
        assert all(e.count for e in ks.engines)
        check_answers(ks, np.stack([v, other[0]]))
        assert bytes(ks.serialize()) == bytes(ks.single.serialize())
    finally:
        ks.close()


def test_keyed_entries_check_their_arguments():
    rng = np.random.default_rng(5)
    rows = unit_rows(rng, 6, DIMS)
    eng = CUDAVectorEngine(VectorMetric.cosine, DIMS)
    one = CUDAVectorEngine(VectorMetric.cosine, DIMS)
    try:
        assert eng.add_batch_keyed([1, 2, 3], rows[:3], 10) == 3
        assert eng.row_keys().tolist() == [10, 11, 12]
        with pytest.raises(WaxError, match="not above the last row key"):
            eng.add_batch_keyed([4], rows[3:4], 12)
        assert eng.count == 3
        assert eng.add_batch_keyed([2, 4, 4, 5], rows[:4], 20) == 2     # an upsert keeps its key
        eng.add_batch([6], rows[5:6])                                    # plain add_batch: the next key
        assert eng.row_keys().tolist() == [10, 11, 12, 20, 21, 22]
        eng.remove_batch([1, 4])
        assert eng.row_keys().tolist() == [11, 12, 21, 22]
        assert eng.contains([2, 4, 6, 99]).tolist() == [True, False, True, False]
        ids, vecs, keys = eng.export_rows(1, 2)
        assert ids.tolist() == [3, 5] and keys.tolist() == [12, 21] and np.array_equal(vecs, rows[[2, 3]])
        blob = bytes(eng.serialize())
        one.deserialize_rows(blob, 1, 2)
        assert one.row_keys().tolist() == [1, 2] and one.export_rows(0, 2)[0].tolist() == [3, 5]
        with pytest.raises(WaxError, match="outside the segment"):
            one.deserialize_rows(blob, 3, 2)
        bad, reasons = b"MV2X" + blob[4:], []
        for load in (lambda: one.deserialize(bad), lambda: one.deserialize_rows(bad, 0, 1)):
            with pytest.raises(WaxError) as err:
                load()
            reasons.append(str(err.value))
        assert reasons[0] == reasons[1] and "magic" in reasons[0]
        one.deserialize(blob)                                            # the whole blob: no keys
        assert one.row_keys().tolist() == [0, 1, 2, 3]
        with pytest.raises(WaxError, match="out of bounds"):
            one.export_rows(3, 2)
    finally:
        eng.close()
        one.close()


def test_sharded_engine_corpus_methods_on_one_rank():
    """ShardedVectorEngine without a process group (world 1), built empty: add, add_batch, remove, remove_batch, count,
    serialize and deserialize end to end, every answer and the bytes equal to one engine's."""
    rng = np.random.default_rng(23)
    pool = unit_rows(rng, 30, DIMS)
    sh = sharded.ShardedVectorEngine(VectorMetric.cosine, DIMS)
    single = CUDAVectorEngine(VectorMetric.cosine, DIMS)
    try:
        assert sh.count() == 0 and sh.search(pool[0], 10) == []
        ids = np.arange(2000, dtype=np.uint64)
        vecs = pool[rng.integers(0, 30, 2000)]
        for eng in (sh, single):
            eng.add_batch(ids[:1500], vecs[:1500])
            eng.add(7, pool[1])
            eng.add_batch(ids[1000:], vecs[1000:][::-1].copy())
            eng.remove(12)
        assert sh.remove_batch(ids[::5]) == single.remove_batch(ids[::5])
        assert sh.count() == single.count
        blob = sh.serialize()
        assert bytes(blob) == bytes(single.serialize())
        qs = np.concatenate([pool[:2], unit_rows(rng, 2, DIMS)])

        def same():
            for q in qs:
                for k in (10, 72, 200):
                    assert _hits_bits(sh.search(q, k)) == _hits_bits(single.search(q, k))
            assert sh.search_batch(qs, 10) == single.search_batch(qs, 10)
            where = Where(after=5, before=80)
            for eng in (sh, single):
                fids = single.export_rows(0, single.count, vectors=False)[0]
                eng.set_attributes(fids, (fids % 97).astype(np.int64), fids % 4)
                eng.set_groups(fids, fids % 11)
            assert sh.search_where(qs[0], 10, where) == single.search_where(qs[0], 10, where)
            assert sh.search_grouped(qs[1], 4, 3, where=where) == \
                single.search_batch_grouped_multi_where(qs[1:2], 4, 3, [where], [0])[0]
        same()
        sh.deserialize(blob)
        single.deserialize(blob)
        assert sh.count() == single.count and bytes(sh.serialize()) == bytes(blob)
        same()
    finally:
        sh.close()
        single.close()
