"""GPU: wax_vs_rebalance on the multi-device handle (DESIGN.md section 4.16) against one engine with the same call history.
The placement model of test_gpu_multi_device.Pair is extended with sharded.plan_rebalance: each donor's tail, in key
order (one engine's row order), goes to the receivers.  After every step of a seeded script the MV2V bytes, the rows per
shard and every served search, bit for bit, equal the single engine's, and the groups, attributes, locations and terms
set before a rebalance still apply after it without being set again."""
import numpy as np
import pytest

from test_gpu_multi_device import DIMS, Pair, _devices, _hits, _vectors
from wax_b200 import CUDAVectorEngine, VectorMetric, sharded

pytestmark = pytest.mark.gpu


class RebalancePair(Pair):
    def key_order(self):
        """Every held frame in key order: one engine's row order."""
        n = self.one.count
        return [int(i) for i in self.one.export_rows(0, n, vectors=False)[0]] if n else []

    def rebalance(self):
        targets, moves = sharded.plan_rebalance(self.counts)
        order = self.key_order()
        held = {r: [f for f in order if self.owner[f] == r] for r in range(self.r)}
        dealt = {}
        for d, x, n in moves:
            at = int(targets[d]) + dealt.get(d, 0)
            for f in held[d][at:at + n]:
                self.owner[f] = x
            dealt[d] = dealt.get(d, 0) + n
        self.counts = np.asarray(targets, np.int64)
        assert self.multi.rebalance() == sum(n for _, _, n in moves)
        assert self.one.rebalance() == 0
        return moves

    def moved_frames(self, before):
        return sorted(f for f, o in self.owner.items() if before.get(f, o) != o)


@pytest.mark.parametrize("metric", [VectorMetric.cosine, VectorMetric.dot, VectorMetric.l2])
@pytest.mark.parametrize("r", [2, 3, 4])
def test_rebalance_script_equals_one_engine(metric, r):
    rng = np.random.default_rng(2000 * r + metric.value)
    pool = rng.standard_normal((40, DIMS)).astype(np.float32)       # exact ties whose keys interleave across shards
    p = RebalancePair(metric, r)
    try:
        if metric == VectorMetric.l2:
            p.set_option("batch_l2", 1)
        p.set_option("rebalance_slab_bytes", DIMS * 4 * 13)        # a move of dozens of rows crosses several slabs
        assert p.rebalance() == []                                 # the empty handle
        p.check(rng, ks=(10,), batches=(3,))
        ids = rng.permutation(np.arange(10, 900)).astype(np.uint64)
        p.add_batch(ids, _vectors(rng, ids.size, pool))
        up = np.concatenate([ids[:40], [9000, 9001, 9000]]).astype(np.uint64)
        p.add_batch(up, _vectors(rng, up.size, pool))
        p.set_metadata(rng)
        p.check(rng)

        # 1. every frame on shard 0 goes
        p.remove_batch(np.array([f for f, o in p.owner.items() if o == 0], np.uint64))
        p.check(rng, ks=(10,), batches=(3,))
        before = dict(p.owner)
        moves = p.rebalance()
        assert moves and all(x == 0 or d != 0 for d, x, _ in moves)
        p.check(rng)                                               # metadata is not set again
        assert p.rebalance() == []                                 # balanced now
        p.check(rng, ks=(10,), batches=(3,))

        # upserts and removes of moved frames: found where they now live
        moved = p.moved_frames(before)
        assert moved
        p.add_batch(np.array(moved[:25] + [50_000, 50_001], np.uint64), _vectors(rng, 27, pool))
        p.add(moved[30], pool[3])
        p.remove(moved[31])
        p.remove_batch(np.array(moved[40:60], np.uint64))
        p.check(rng)

        # 2. a key range goes
        order = p.key_order()
        p.remove_batch(np.array(order[len(order) // 5: len(order) * 3 // 5], np.uint64))
        p.rebalance()
        p.check(rng)

        # 3. everything but one shard goes
        keep = r - 1
        p.remove_batch(np.array([f for f, o in p.owner.items() if o != keep], np.uint64))
        p.rebalance()
        p.check(rng)
        more = np.arange(70_000, 70_200, dtype=np.uint64)           # then new rows fill the emptiest shards
        p.add_batch(more, _vectors(rng, more.size, pool))
        p.rebalance()
        p.check(rng)

        # 4. a reload (MV2V carries no metadata), skewed, rebalanced
        p.deserialize(p.one.serialize())
        p.set_metadata(rng)
        p.remove_batch(np.array(p.key_order()[: p.one.count // 2], np.uint64))
        p.rebalance()
        p.check(rng)

        # 5. the empty handle
        p.remove_batch(np.array(p.key_order(), np.uint64))
        assert p.rebalance() == []
        p.check(rng, ks=(10,), batches=(3,))
    finally:
        p.close()


def test_metadata_set_on_one_side_only():
    """Groups, attributes, locations and terms set while the receiving shard held no rows (so it has none of them) arrive
    with the moved rows, and the receiver's own rows answer with the defaults they had."""
    rng = np.random.default_rng(9)
    pool = rng.standard_normal((12, DIMS)).astype(np.float32)
    p = RebalancePair(VectorMetric.cosine, 3)
    try:
        p.set_option("rebalance_slab_bytes", DIMS * 4 * 5)
        p.add_batch(np.arange(1, 301, dtype=np.uint64), _vectors(rng, 300, pool))
        p.remove_batch(np.array([f for f, o in p.owner.items() if o != 2], np.uint64))   # shards 0 and 1 empty
        p.set_metadata(rng)                                          # only shard 2 holds rows to set
        p.rebalance()
        p.check(rng)
        p.add_batch(np.arange(400, 460, dtype=np.uint64), _vectors(rng, 60, pool))       # new rows: no metadata
        p.remove_batch(np.array([f for f, o in p.owner.items() if o == 2][:50], np.uint64))
        p.rebalance()
        p.check(rng)
    finally:
        p.close()


def test_rebalance_refills_a_shard_on_the_single_query_route():
    """4 M x 384 cosine at R = 2 against one engine.  Removing most of shard 0's rows leaves it at 0.5 M rows, still on
    the single-query shadow route (768 MB), shard 1 at 2 M; single queries run on both, then the rebalance refills shard 0
    with 0.75 M rows of shard 1's tail (default 256 MiB slabs, several of them) and the route rebuilds its shadows.  Every
    answer equals one engine's, before and after."""
    rng = np.random.default_rng(12)
    n, dims, chunk = 4_000_000, 384, 1_000_000
    multi = CUDAVectorEngine(VectorMetric.cosine, dims, devices=_devices(2))
    one = CUDAVectorEngine(VectorMetric.cosine, dims)
    try:
        for lo in range(0, n, chunk):                            # each chunk splits in halves: shard 0 takes the first
            rows = rng.standard_normal((chunk, dims), dtype=np.float32)
            ids = np.arange(lo, lo + chunk, dtype=np.uint64)
            multi.add_batch(ids, rows)
            one.add_batch(ids, rows)
        del rows
        gone = np.concatenate([np.arange(lo, lo + chunk // 2, dtype=np.uint64) for lo in range(0, 3 * chunk, chunk)])
        assert multi.remove_batch(gone) == one.remove_batch(gone) == gone.size
        assert [multi.counter(f"shard_rows.{r}") for r in range(2)] == [500_000, 2_000_000]
        qs = rng.standard_normal((24, dims)).astype(np.float32)

        def route_queries():
            return sum(multi.counter(c) for c in ("single_shadow_queries", "single_int8_queries", "single_u4_queries"))

        def same(batch):
            for q in qs[:8]:
                assert _hits(multi.search(q, 10)) == _hits(one.search(q, 10))
            if batch:
                a, b = multi.search_batch_arrays(qs, 10), one.search_batch_arrays(qs, 10)
                assert np.array_equal(a[0], b[0]) and np.array_equal(a[1].view(np.uint32), b[1].view(np.uint32))
                assert np.array_equal(a[2], b[2])

        seen = route_queries()
        same(batch=True)
        assert route_queries() > seen
        assert multi.rebalance() == 750_000
        assert [multi.counter(f"shard_rows.{r}") for r in range(2)] == [1_250_000, 1_250_000]
        seen = route_queries()
        same(batch=True)
        assert route_queries() > seen
        assert multi.rebalance() == 0
        upsert = np.arange(3_900_000, 3_900_100, dtype=np.uint64)   # moved rows, upserted where they now live
        rows = rng.standard_normal((upsert.size, dims)).astype(np.float32)
        multi.add_batch(upsert, rows)
        one.add_batch(upsert, rows)
        assert multi.count == one.count == 2_500_000
        assert [multi.counter(f"shard_rows.{r}") for r in range(2)] == [1_250_000, 1_250_000]
        same(batch=False)
    finally:
        multi.close()
        one.close()
