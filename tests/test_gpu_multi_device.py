"""GPU: the multi-device handle (wax_vs_create with a device list, DESIGN.md section 4.16) against one engine with the
same call history.  Devices are [i % device_count for i in range(R)], so on one GPU the shards share it and on a
multi-GPU box the merge reads real peer memory.  After every step of a seeded script the MV2V bytes, the rows per shard
(sharded.plan_add_batch's model) and every served search, bit for bit, equal the single engine's."""
import ctypes as C
import threading

import numpy as np
import pytest
import torch

from wax_b200 import CUDAVectorEngine, VectorMetric, Where, sharded
from wax_b200 import _lib as L

pytestmark = pytest.mark.gpu

DIMS = 64


def _devices(r):
    return [i % torch.cuda.device_count() for i in range(r)]


def _raw_search(h, qs, top_k, cap, query_len=None):
    """wax_vs_search_batch through ctypes: (rc, reason, ids, score bits, counts)."""
    qs = np.ascontiguousarray(qs, np.float32).reshape(-1, DIMS) if qs is not None else None
    b = 1 if qs is None else qs.shape[0]
    ids = np.zeros((b, max(cap, 1)), np.uint64)
    scores = np.zeros((b, max(cap, 1)), np.float32)
    ns = np.zeros(b, np.uint32)
    qp = qs.ctypes.data_as(C.POINTER(C.c_float)) if qs is not None else None
    rc = L.lib().wax_vs_search_batch(h, qp, b, DIMS if query_len is None else query_len, int(top_k),
                                     ids.ctypes.data_as(C.POINTER(C.c_uint64)),
                                     scores.ctypes.data_as(C.POINTER(C.c_float)), cap,
                                     ns.ctypes.data_as(C.POINTER(C.c_uint32)))
    reason = L.last_error() if rc else ""
    return rc, reason, [ids[i, :ns[i]].tolist() for i in range(b)], [scores[i, :ns[i]].view(np.uint32).tolist()
                                                                      for i in range(b)]


def _hits(hits):
    return [(f, np.float32(s).view(np.uint32).item()) for f, s in hits]


class Pair:
    """A multi-device handle of R shards, one engine, and the placement model of sharded.plan_add_batch."""

    def __init__(self, metric, r):
        self.r = r
        self.multi = CUDAVectorEngine(metric, DIMS, devices=_devices(r))
        self.one = CUDAVectorEngine(metric, DIMS)
        self.counts = np.zeros(r, np.int64)
        self.owner = {}
        self.next_key = 0

    def close(self):
        self.multi.close()
        self.one.close()

    def set_option(self, key, value):
        self.multi.set_option(key, value)
        self.one.set_option(key, value)

    def add_batch(self, ids, vecs):
        ids = np.asarray(ids, np.uint64)
        owner = np.array([self.owner.get(int(i), -1) for i in ids], np.int64)
        dest, _, appended, self.next_key = sharded.plan_add_batch(ids, owner, self.counts, self.next_key)
        for i, d in zip(ids.tolist(), dest.tolist()):
            self.owner.setdefault(i, d)
        self.counts = self.counts + appended
        self.multi.add_batch(ids, vecs)
        self.one.add_batch(ids, vecs)

    def add(self, frame_id, vec):
        owner = np.array([self.owner.get(int(frame_id), -1)], np.int64)
        dest, _, appended, self.next_key = sharded.plan_add_batch([frame_id], owner, self.counts, self.next_key)
        self.owner.setdefault(int(frame_id), int(dest[0]))
        self.counts = self.counts + appended
        self.multi.add(frame_id, vec)
        self.one.add(frame_id, vec)

    def remove(self, frame_id):
        self.multi.remove(frame_id)
        self.one.remove(frame_id)
        if int(frame_id) in self.owner:
            self.counts[self.owner.pop(int(frame_id))] -= 1

    def remove_batch(self, ids):
        gone = self.one.remove_batch(ids)
        assert self.multi.remove_batch(ids) == gone
        for i in set(int(x) for x in ids):
            if i in self.owner:
                self.counts[self.owner.pop(i)] -= 1

    def deserialize(self, blob):
        n = sharded.mv2v_count(blob)
        self.multi.deserialize(blob)
        self.one.deserialize(blob)
        ids = np.frombuffer(bytes(blob), np.uint64, n, 44 + n * DIMS * 4) if n else []
        self.counts = sharded.shard_counts(n, self.r)
        self.owner = {int(i): int(np.searchsorted(np.cumsum(self.counts), p, side="right")) for p, i in enumerate(ids)}
        self.next_key = n

    def set_metadata(self, rng):
        """Attributes, locations, terms and groups for every held frame (the full lists go to every shard)."""
        ids = np.array(sorted(self.owner), np.uint64)
        n = ids.size
        ts = rng.integers(0, 1000, n)
        tags = rng.integers(0, 4, n).astype(np.uint64)
        lat, lon = rng.uniform(40.0, 40.5, n), rng.uniform(-74.0, -73.5, n)
        terms = [list(rng.choice(8, rng.integers(0, 3), replace=False)) for _ in range(n)]
        groups = (ids // 7).astype(np.uint64)
        for name, args in [("set_attributes", (ids, ts, tags)), ("set_locations", (ids, lat, lon)),
                           ("set_terms", (ids, terms)), ("set_groups", (ids, groups))]:
            assert getattr(self.multi, name)(*args) == getattr(self.one, name)(*args), name
        self.metadata = True

    def check_filtered(self, rng, qs, k):
        ids = np.array(sorted(self.owner), np.uint64)
        allow = rng.choice(ids, min(ids.size, 30), replace=False) if ids.size else ids
        deny = rng.choice(ids, ids.size // 2, replace=False) if ids.size else ids
        for kw in ({"allow": allow}, {"deny": deny}, {"allow": []}):
            assert self.multi.search_batch_filtered(qs, k, **kw) == self.one.search_batch_filtered(qs, k, **kw), kw
            assert self.multi.search_filtered(qs[0], k, **kw) == self.one.search_filtered(qs[0], k, **kw), kw
        filters = [("allow", allow), ("deny", deny)]
        qf = [i % 3 if i % 3 < 2 else None for i in range(len(qs))]
        assert (self.multi.search_batch_multi_filtered(qs, k, filters, qf) ==
                self.one.search_batch_multi_filtered(qs, k, filters, qf))
        if not getattr(self, "metadata", False):
            return
        wheres = [Where(after=200, before=700), Where(all_tags=1), Where(near=(40.2, -73.8, 20_000.0)),
                  Where(terms=(1,)), Where(terms=(2, 5), after=100)]
        qw = [i % (len(wheres) + 1) if i % (len(wheres) + 1) < len(wheres) else None for i in range(len(qs))]
        for w in (wheres[:2], wheres[:3], wheres):                 # plain, near and terms entry points
            qwi = [x if x is not None and x < len(w) else None for x in qw]
            assert (self.multi.search_batch_where(qs, k, w, qwi, filters, qf) ==
                    self.one.search_batch_where(qs, k, w, qwi, filters, qf)), len(w)
        for per_group in (1, 3):
            g = min(k, 12)
            assert (self.multi.search_batch_grouped(qs, g, per_group, deny=deny) ==
                    self.one.search_batch_grouped(qs, g, per_group, deny=deny))
            assert (self.multi.search_grouped(qs[0], g, per_group, allow=allow) ==
                    self.one.search_grouped(qs[0], g, per_group, allow=allow))
            for w in (wheres[0], wheres[2]):                       # the plain and the near one-where forms
                assert (self.multi.search_batch_grouped_where(qs, g, per_group, w) ==
                        self.one.search_batch_grouped_where(qs, g, per_group, w))
            gw = wheres[:3]
            qwi = [x if x is not None and x < 3 else None for x in qw]
            assert (self.multi.search_batch_grouped_multi_where(qs, g, per_group, gw, qwi, filters, qf) ==
                    self.one.search_batch_grouped_multi_where(qs, g, per_group, gw, qwi, filters, qf))

    def check(self, rng, ks=(1, 10, 72, 200, 20_000), batches=(1, 3, 64)):
        assert self.multi.count == self.one.count
        assert bytes(self.multi.serialize()) == bytes(self.one.serialize())
        assert [self.multi.counter(f"shard_rows.{r}") for r in range(self.r)] == self.counts.tolist()
        for b in batches:
            qs = rng.standard_normal((b, DIMS)).astype(np.float32)
            for k in ks:
                cap = min(sharded.clamp_topk(k), max(self.one.count, 1))
                got = _raw_search(self.multi.handle, qs, k, cap)
                want = _raw_search(self.one.handle, qs, k, cap)
                assert got == want, (b, k)
            for k in (1, 10, 72):
                self.check_filtered(rng, qs, k)
        q = rng.standard_normal(DIMS).astype(np.float32)
        assert _hits(self.multi.search(q, 10)) == _hits(self.one.search(q, 10))


def _vectors(rng, n, pool):
    """Rows drawn from a small pool, so exact ties abound and their keys interleave across the shards."""
    return pool[rng.integers(0, len(pool), n)]


@pytest.mark.parametrize("metric", [VectorMetric.cosine, VectorMetric.dot, VectorMetric.l2])
@pytest.mark.parametrize("r", [2, 3, 4])
def test_script_equals_one_engine(metric, r):
    rng = np.random.default_rng(1000 * r + metric.value)
    pool = rng.standard_normal((40, DIMS)).astype(np.float32)
    p = Pair(metric, r)
    try:
        if metric == VectorMetric.l2:
            p.set_option("batch_l2", 1)
        p.check(rng)                                                       # empty handle
        p.add_batch([5, 3], _vectors(rng, 2, pool))                          # fewer rows than shards at R = 3, 4
        p.check(rng)
        ids = rng.permutation(np.arange(10, 700)).astype(np.uint64)          # out-of-order ids
        p.add_batch(ids, _vectors(rng, ids.size, pool))
        p.check(rng)
        up = np.concatenate([ids[:50], [9000, 9001, 9000], ids[100:120], [3]]).astype(np.uint64)   # upserts, duplicates
        p.add_batch(up, _vectors(rng, up.size, pool))
        p.set_metadata(rng)
        p.check(rng)
        p.add(77_777, pool[0])
        p.add(int(ids[3]), pool[1])                                        # an upsert through add
        p.remove(int(ids[7]))
        p.check(rng)
        blob = p.one.serialize()
        p.deserialize(blob)                                                # the single engine's blob
        p.set_metadata(rng)                                                # MV2V carries no metadata
        p.check(rng)
        p.remove_batch(np.concatenate([ids[200:260], [123_456_789, 5]]).astype(np.uint64))   # unknown ids too
        p.check(rng)
        more = np.arange(20_000, 20_300, dtype=np.uint64)
        p.add_batch(more, _vectors(rng, more.size, pool))
        p.check(rng)
    finally:
        p.close()


def test_batch_of_1024_on_the_tensor_core_levels():
    rng = np.random.default_rng(7)
    p = Pair(VectorMetric.cosine, 3)
    try:
        n = 60_000
        ids = np.arange(1, n + 1, dtype=np.uint64)
        p.add_batch(ids, rng.standard_normal((n, DIMS)).astype(np.float32))
        p.remove_batch(ids[::7])
        p.check(rng, ks=(10, 72, 200), batches=(1024,))
        assert p.multi.counter("batch_tensor_queries") > 0
    finally:
        p.close()


def test_errors_equal_one_engines():
    rng = np.random.default_rng(3)
    p = Pair(VectorMetric.cosine, 2)
    try:
        h1, h2 = p.multi.handle, p.one.handle
        # the empty handle answers before it validates the query
        assert _raw_search(h1, None, 10, 10, query_len=3) == _raw_search(h2, None, 10, 10, query_len=3)
        p.add_batch(np.arange(1, 40, dtype=np.uint64), rng.standard_normal((39, DIMS)).astype(np.float32))
        qs = rng.standard_normal((2, DIMS)).astype(np.float32)
        for args in [(None, 10, 10), (qs, 10, 10, DIMS + 1), (qs, 10, 9), (qs, 20_000, 38)]:
            got, want = _raw_search(h1, *args), _raw_search(h2, *args)
            assert got == want and got[0] != 0, args
        bad = rng.standard_normal((1, DIMS + 1)).astype(np.float32)
        codes = []
        for h in (h1, h2):
            rc = L.lib().wax_vs_add_batch(h, (C.c_uint64 * 1)(5), bad.ctypes.data_as(C.POINTER(C.c_float)), 1, DIMS + 1)
            codes.append((rc, L.last_error()))
            rc = L.lib().wax_vs_deserialize(h, (C.c_uint8 * 40)(*b"MV2X" + bytes(36)), 40)
            codes.append((rc, L.last_error()))
            n = C.c_uint64(0)
            rc = L.lib().wax_vs_serialize(h, (C.c_uint8 * 8)(), 8, C.byref(n))
            codes.append((rc, L.last_error(), n.value))
            rc = L.lib().wax_vs_debug_counter(h, b"no_such_counter", C.byref(n))
            codes.append((rc, L.last_error()))
            rc = L.lib().wax_vs_debug_set_option(h, b"no_such_option", 1)
            codes.append((rc, L.last_error()))
            codes.append((L.lib().wax_vs_reserve(h, 1 << 33), L.last_error()))
        half = len(codes) // 2
        assert codes[:half] == codes[half:] and all(c[0] != 0 for c in codes)
        p.check(rng)                                                       # nothing changed
    finally:
        p.close()


REFUSED = ["wax_vs_add_batch_keyed", "wax_vs_contains", "wax_vs_search_device", "wax_vs_search_batch_device",
           "wax_vs_shard_open", "wax_vs_shard_close", "wax_vs_merge_candidates_device", "wax_vs_search_batch_where_device",
           "wax_vs_shard_search_where", "wax_vs_shard_grouped_expand_device", "wax_vs_shard_grouped_heads_device", "wax_vs_merge_group_heads_device", "wax_vs_deserialize_rows",
           "wax_vs_export_rows", "wax_vs_debug_fill_synthetic", "wax_vs_debug_time_search", "wax_vs_debug_read_rows",
           "wax_vs_debug_last_scan"]


def test_unserved_entries_are_refused_by_name():
    e = CUDAVectorEngine(VectorMetric.cosine, DIMS, devices=_devices(2))
    try:
        for name in REFUSED:
            argtypes = L.SIGNATURES[name][1]
            args = [e.handle] + [None if t in (C.c_void_p, C.c_char_p) or issubclass(t, C._Pointer) else 0
                                 for t in argtypes[1:]]
            rc = getattr(L.lib(), name)(*args)
            assert rc == L.ERR_UNSUPPORTED, name
            assert L.last_error() == f"{name} is not served by a multi-device handle"
        assert e.count == 0
    finally:
        e.close()


def test_concurrent_searches_equal_their_serial_answers():
    rng = np.random.default_rng(11)
    p = Pair(VectorMetric.cosine, 4)
    try:
        p.add_batch(np.arange(1, 5001, dtype=np.uint64), rng.standard_normal((5000, DIMS)).astype(np.float32))
        work = [(rng.standard_normal((b, DIMS)).astype(np.float32), k) for b, k in [(1, 10), (16, 72), (5, 200), (1, 5)] * 4]
        serial = [_raw_search(p.one.handle, q, k, k) for q, k in work]
        got = [None] * len(work)

        def run(t):
            for i in range(t, len(work), 8):
                got[i] = _raw_search(p.multi.handle, *work[i][:1], work[i][1], work[i][1])

        threads = [threading.Thread(target=run, args=(t,)) for t in range(8)]
        for th in threads:
            th.start()
        for th in threads:
            th.join()
        assert got == serial
    finally:
        p.close()


def test_10m_corpus_on_different_shadow_routes_matches():
    """10 M x 384 cosine (15.4 GB), a handle of 2 shards against one engine on one H100, single queries and a batch of
    1 024.  The handle's shards are told to take the 4-bit route only above 8 GB, so one engine nominates from its 4-bit
    shadow and each 7.7 GB shard from a shadow of more bits: the route counters show that the two sides really differ.  The
    corpus is added in chunks of 1 M rows, so the host never holds all of it."""
    rng = np.random.default_rng(5)
    n, dims, chunk = 10_000_000, 384, 1_000_000
    multi = CUDAVectorEngine(VectorMetric.cosine, dims, devices=_devices(2))
    one = CUDAVectorEngine(VectorMetric.cosine, dims)
    try:
        multi.set_option("u4_scan_min_bytes", 8 << 30)
        for lo in range(0, n, chunk):
            rows = rng.standard_normal((chunk, dims), dtype=np.float32)
            ids = np.arange(lo, lo + chunk, dtype=np.uint64)
            multi.add_batch(ids, rows)
            one.add_batch(ids, rows)
        del rows
        for _ in range(8):
            q = rng.standard_normal(dims).astype(np.float32)
            assert _hits(multi.search(q, 10)) == _hits(one.search(q, 10))
        # one engine nominated from its 4-bit shadow (a failed 4-bit proof may demote a few later queries), the shards never
        assert one.counter("single_u4_queries") > 0 and multi.counter("single_u4_queries") == 0
        qs = rng.standard_normal((1024, dims)).astype(np.float32)
        a, b = multi.search_batch_arrays(qs, 10), one.search_batch_arrays(qs, 10)
        assert np.array_equal(a[0], b[0]) and np.array_equal(a[1].view(np.uint32), b[1].view(np.uint32))
        assert np.array_equal(a[2], b[2])
    finally:
        multi.close()
        one.close()
