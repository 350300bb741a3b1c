"""Row-sharded vector search across GPUs: one process (rank) per GPU, one CUDA engine per rank.

Design (SURVEY.md section 8e; BASELINE.json north_star): rows spread over the ranks (contiguous ranges for
fill_synthetic, or keyed by insertion order for a corpus the collective corpus methods keep, DESIGN.md section 4.15), the
query replicated, the identical fused kernel on every shard, ONE exchange of the per-shard top-k candidates
(k x 24 B per rank) and a merge under the same total order (distance ascending, GLOBAL row ascending), so
results do not depend on the shard count.  Nothing else is exchanged.

Two transports for that exchange:
  * "p2p-fused" (default whenever the ranks can map each other's memory): the exchange is part of the scan launch --
    the kernel's last CTA writes its candidates into every rank's mailbox over NVLink/NVSwitch peer memory, waits for
    the others' flags and merges on the device, delivering the result into mapped host memory (wax_vs_shard_search,
    wax_b200/csrc/waxvs_shard.cuh).  torch.distributed is used ONCE, at construction, to pass the 128-byte mailbox
    handles around.  No collective launch, no D2H copy, no host merge per query.
  * "allgather": torch.distributed all_gather_into_tensor (NCCL) + host merge -- k > 128, the micro-batched /
    batched forms, and the CPU (gloo) tests of the host logic.

The reference has no distributed code at all (SURVEY.md section 2: "none exist"); this is the only
parallelism the build adds.
"""
from __future__ import annotations

import ctypes as C
from typing import Callable, List, Optional, Sequence, Tuple

import numpy as np

CAND_DTYPE = np.dtype([("distance", "<f4"), ("valid", "<u4"), ("row", "<u8"), ("frame_id", "<u8")])
assert CAND_DTYPE.itemsize == 24
# wax_vs_group_candidate: a row of a rank's grouped answer, with its group id (sharded grouped search)
GROUP_CAND_DTYPE = np.dtype([("distance", "<f4"), ("valid", "<u4"), ("row", "<u8"), ("frame_id", "<u8"),
                             ("group_id", "<u8")])
assert GROUP_CAND_DTYPE.itemsize == 32


def shard_range(total_rows: int, world_size: int, rank: int) -> Tuple[int, int]:
    """Contiguous shard [lo, hi): rows r*N/R .. (r+1)*N/R (global row = lo + local row)."""
    lo = (total_rows * rank) // world_size
    hi = (total_rows * (rank + 1)) // world_size
    return lo, hi


# -- corpus planning (DESIGN.md section 4.15): pure functions, so that the tests can drive ranks without a process group.
# A row's key is its insertion sequence number in the whole corpus; ordering rows by key is the single engine's row order.
def fill_emptiest(counts: Sequence[int], m: int) -> np.ndarray:
    """How many of m new rows each rank takes: the ranks with the fewest rows first, to one level (ties to lower ranks)."""
    counts = np.asarray(counts, np.int64)
    alloc = np.zeros(counts.size, np.int64)
    if m <= 0:
        return alloc
    lo, hi = int(counts.min()), int(counts.max()) + m           # the largest level L with sum(max(0, L - count)) <= m
    while lo < hi:
        mid = (lo + hi + 1) // 2
        if int(np.maximum(mid - counts, 0).sum()) <= m:
            lo = mid
        else:
            hi = mid - 1
    alloc = np.maximum(lo - counts, 0)
    rest = m - int(alloc.sum())                                 # fewer than the ranks at the level: one more each
    at_level = np.flatnonzero(counts + alloc == lo)[:rest]
    alloc[at_level] += 1
    return alloc


def plan_rebalance(counts: Sequence[int]):
    """How a rebalance evens out the ranks' rows.  Every rank gets T // R of the T rows; the T % R extra rows go to the
    ranks that hold the most now (ties to lower ranks), which moves the fewest rows and leaves a balanced corpus alone.
    A donor gives up its surplus from its tail (its highest keys), so it only truncates; donors and receivers are taken in
    rank order, and a donor's tail is dealt out in key order, its lowest-key part to the first receiver with a deficit.
    Returns (targets [world], moves [(donor, receiver, rows), ...])."""
    counts = np.asarray(counts, np.int64).reshape(-1)
    world, total = counts.size, int(counts.sum())
    targets = np.full(world, total // world if world else 0, np.int64)
    targets[np.argsort(-counts, kind="stable")[:total % world if world else 0]] += 1
    give = np.maximum(counts - targets, 0)
    take = np.maximum(targets - counts, 0)
    moves = []
    receivers = iter(np.flatnonzero(take).tolist())
    r = next(receivers, None)
    for d in np.flatnonzero(give).tolist():
        left = int(give[d])
        while left:
            n = min(left, int(take[r]))
            moves.append((d, r, n))
            left -= n
            take[r] -= n
            if take[r] == 0:
                r = next(receivers, None)
    return targets, moves


def plan_add_batch(frame_ids, owner, counts: Sequence[int], next_key: int):
    """Where each item of a sharded add_batch goes.  `owner` [n]: the rank holding each id before the batch (-1: none);
    `counts`: rows per rank; `next_key`: the first unused key.  Held ids are upserted by their owner.  The distinct new
    ids, in order of first appearance, take the keys next_key, next_key + 1, ... and are split in contiguous chunks over
    the ranks (fill_emptiest, chunks in rank order); every occurrence of an id goes where its first one goes.
    Returns (dest [n] rank of each item, first_key [world] of each rank's chunk, appended [world], the next unused key)."""
    ids = np.asarray(frame_ids, np.uint64).reshape(-1)
    owner = np.asarray(owner, np.int64).reshape(-1)
    dest = owner.copy()
    new = np.flatnonzero(owner < 0)
    uniq, first, inverse = np.unique(ids[new], return_index=True, return_inverse=True)
    order = np.argsort(first, kind="stable")                    # distinct new ids in batch order
    seq = np.empty(uniq.size, np.int64)
    seq[order] = np.arange(uniq.size)                           # sequence number of each distinct new id
    alloc = fill_emptiest(counts, uniq.size)
    start = np.concatenate([[0], np.cumsum(alloc)[:-1]])
    dest[new] = np.searchsorted(np.cumsum(alloc), seq[inverse.reshape(-1)], side="right")
    return dest, int(next_key) + start, alloc, int(next_key) + uniq.size


def plan_serialize(keys: Sequence[np.ndarray]) -> List[np.ndarray]:
    """The MV2V position of every rank's rows: rows ordered by key, which is the single engine's order.  keys[r] = rank r's
    keys in row order (strictly increasing)."""
    flat = np.concatenate([np.asarray(k, np.uint64).reshape(-1) for k in keys] + [np.zeros(0, np.uint64)])
    pos = np.empty(flat.size, np.int64)
    pos[np.argsort(flat, kind="stable")] = np.arange(flat.size)
    bounds = np.cumsum([0] + [len(k) for k in keys])
    return [pos[bounds[r]:bounds[r + 1]] for r in range(len(keys))]


def mv2v_header(similarity: int, dims: int, count: int) -> bytes:
    """The 36-byte MV2V v1 encoding-2 header (MetalVectorEngine.swift:686-700)."""
    return (b"MV2V" + np.uint16(1).tobytes() + bytes([2, similarity]) + np.uint32(dims).tobytes() +
            np.uint64(count).tobytes() + np.uint64(count * dims * 4).tobytes() + bytes(8))


def mv2v_count(blob) -> int:
    """The row count an MV2V header states (0 when the blob is too short to hold one: the load then reports why)."""
    return int(np.frombuffer(blob, np.uint64, 1, 12)[0]) if len(blob) >= 36 else 0


def shard_counts(total_rows: int, world_size: int) -> np.ndarray:
    """[world] rows of each shard_range."""
    return np.diff([shard_range(total_rows, world_size, r)[0] for r in range(world_size)] + [total_rows]).astype(np.int64)


def clamp_topk(top_k: int) -> int:
    """clampTopK (MetalVectorEngine.swift:842-846)."""
    return 1 if top_k < 1 else min(int(top_k), 10_000)


def merge_candidates(gathered: np.ndarray, top_k: int) -> np.ndarray:
    """Host-side R-way merge: `gathered` is any array of CAND_DTYPE records (all ranks' lists);
    returns the best `top_k` valid ones ordered by (distance, global row)."""
    flat = gathered.reshape(-1)
    flat = flat[flat["valid"] != 0]
    if flat.size == 0:
        return flat
    order = np.lexsort((flat["row"], flat["distance"]))  # primary: distance, secondary: row
    return flat[order[:top_k]]


def merge_candidates_batch(gathered: np.ndarray, top_k: int) -> Tuple[np.ndarray, np.ndarray]:
    """Vectorised R-way merge for a batch: `gathered` is [world, batch, k] CAND_DTYPE; returns ([batch, top_k]
    records ordered by (distance, global row) with the invalid ones last, [batch] count of valid results).
    Same total order as merge_candidates (two stable sorts: by row, then by distance)."""
    world, batch, k = gathered.shape
    flat = np.ascontiguousarray(gathered.transpose(1, 0, 2)).reshape(batch, world * k)
    dist = np.where(flat["valid"] != 0, flat["distance"], np.float32(np.inf))
    by_row = np.argsort(flat["row"], axis=1, kind="stable")
    by_dist = np.argsort(np.take_along_axis(dist, by_row, 1), axis=1, kind="stable")
    order = np.take_along_axis(by_row, by_dist, 1)[:, :top_k]
    best = np.take_along_axis(flat, order, 1)
    return best, (best["valid"] != 0).sum(axis=1).astype(np.uint32)


def score_from_distance(similarity: int, d: np.ndarray) -> np.ndarray:
    """VectorMetric.score(fromDistance:) (VectorMetric.swift:32-43), vectorised, fp32."""
    d = d.astype(np.float32)
    s = (np.float32(1) - d) if similarity == 0 else -d
    return np.where(np.isfinite(d), s, np.float32(0)).astype(np.float32)


class ShardedVectorEngine:
    """`VectorSearchEngine.search` over a corpus row-sharded across the ranks of a torch.distributed group.

    local_search: optional injection point used by the CPU (gloo) tests of the host-side logic -- a callable
    (query ndarray, k) -> ndarray[CAND_DTYPE] of length k.  In production it is None and the local step is
    wax_vs_search_device on the rank's GPU.

    Two ways to hold a corpus: `total_rows` > 0 with fill_synthetic (contiguous row ranges), or an empty engine filled by
    the collective corpus methods (add_batch, remove_batch, deserialize, ...; DESIGN.md section 4.15), which place rows
    on any rank and key them by insertion order.  local_store: optional stand-in for the rank's engine in those methods
    (the CPU tests); it needs count, contains, add_batch_keyed, remove_batch, deserialize_rows and export_rows, and for
    rebalance export_vectors, export_columns and absorb_rows.
    """

    def __init__(self, metric, dimensions: int, total_rows: int = 0, group=None,
                 local_search: Optional[Callable[[np.ndarray, int], np.ndarray]] = None, device=None, local_store=None):
        import torch
        import torch.distributed as dist
        self._torch, self._dist = torch, dist
        self.group = group
        self.rank = dist.get_rank(group) if dist.is_initialized() else 0
        self.world_size = dist.get_world_size(group) if dist.is_initialized() else 1
        self.metric = metric
        self.dimensions = int(dimensions)
        self.total_rows = int(total_rows)
        self.row_lo, self.row_hi = shard_range(self.total_rows, self.world_size, self.rank)
        # corpus bookkeeping, the same on every rank: rows per rank and the next unused row key
        self._counts = shard_counts(self.total_rows, self.world_size)
        self._next_key = self.total_rows
        self._contiguous = self.world_size > 1 and self.total_rows > 0     # fill_synthetic's ranges: no corpus methods
        self._local_search = local_search
        self.engine = None
        self._bufs = {}
        self._comm_stream = None
        if local_search is None and local_store is None:
            from .engine import CUDAVectorEngine
            self.device = torch.device("cuda", torch.cuda.current_device()) if device is None else torch.device(device)
            self.engine = CUDAVectorEngine(metric, dimensions, device=self.device.index)
            self._comm_stream = torch.cuda.Stream(device=self.device)   # all-gather + D2H overlap the next scan
            # two scan streams: consecutive queries alternate, so one scan's tail overlaps the next one's prologue
            self._scan_streams = [torch.cuda.Stream(device=self.device) for _ in range(2)]
            # Overlapping two scans pays when a shard is small (kernel tails/prologues overlap) and costs a little
            # when it is large (twice the bytes in flight per SM).  The 12 GB threshold was chosen on B200 and has not
            # been re-measured on H100.
            self._overlap_scans = (self.row_hi - self.row_lo) * self.dimensions * 4 < 12e9
            self.transport = "allgather"
            self.transport_note = ""
            self._connect_peers()
        else:
            self.device = torch.device("cpu")
            self.transport = "allgather"
            self.engine = local_store

    def _connect_peers(self) -> None:
        """Create this rank's mailbox, exchange the handles (one all-gather of 128 bytes per rank, the only use of
        torch.distributed on this path) and map the peers' mailboxes.  All ranks agree on the outcome: if any rank
        cannot map a peer (no P2P / IPC path) every rank stays on the all-gather transport."""
        torch, dist = self._torch, self._dist
        from . import _lib as L
        from .engine import WaxError
        blob, ok = bytes(L.SHARD_HANDLE_BYTES), self.world_size <= L.SHARD_MAX_RANKS
        if ok:
            try:
                blob = self.engine.shard_open(self.rank, self.world_size, self.row_lo)
            except WaxError as exc:
                ok, self.transport_note = False, str(exc)
        if self.world_size > 1:
            dev = self.device if dist.get_backend(self.group) == "nccl" else torch.device("cpu")
            mine = torch.frombuffer(bytearray(blob), dtype=torch.uint8).to(dev)
            every = torch.empty(self.world_size * L.SHARD_HANDLE_BYTES, dtype=torch.uint8, device=dev)
            dist.all_gather_into_tensor(every, mine, group=self.group)
            flat = every.cpu().numpy().tobytes()
            if ok:
                try:
                    self.engine.shard_connect([flat[i * L.SHARD_HANDLE_BYTES:(i + 1) * L.SHARD_HANDLE_BYTES]
                                               for i in range(self.world_size)])
                except WaxError as exc:
                    ok, self.transport_note = False, str(exc)
            flag = torch.tensor([1 if ok else 0], dtype=torch.int32, device=dev)
            dist.all_reduce(flag, op=dist.ReduceOp.MIN, group=self.group)
            if ok and flag.item() != 1:
                ok, self.transport_note = False, "another rank could not map its peers"
        if ok:
            self.transport = "p2p-fused"
        else:
            self.engine.shard_close()

    def close(self) -> None:
        """Collective: unmap the peers' mailboxes, agree that everyone has (barrier), then release the engine."""
        if self.engine is None or getattr(self, "_closed", False):
            return
        self._closed = True
        if self.transport == "p2p-fused":
            self.engine.shard_close()
            self.transport = "allgather"
        if self.world_size > 1 and self._dist.is_initialized():
            self._dist.barrier(group=self.group)
        self.engine.close()

    # -- corpus
    def fill_synthetic(self, seed: int, normalize: bool = True) -> None:
        """Each rank generates its own shard on device; frameId = global row."""
        self.engine.fill_synthetic(seed, self.row_hi - self.row_lo, first_row=self.row_lo, id_base=self.row_lo,
                                   normalize=normalize)

    # -- corpus: collective, every rank passes the same arguments (DESIGN.md section 4.15)
    def _check_corpus_methods(self) -> None:
        if self._contiguous:
            from .engine import InvalidToc
            raise InvalidToc("the corpus methods need an engine built without total_rows (this one holds contiguous "
                             "ranges for fill_synthetic)")

    def _sum_on_ranks(self, values: np.ndarray) -> np.ndarray:
        """Element-wise sum of an int64 vector over the ranks (one all-reduce)."""
        if self.world_size == 1:
            return values
        torch, dist = self._torch, self._dist
        dev = self.device if dist.get_backend(self.group) == "nccl" else torch.device("cpu")
        t = torch.from_numpy(np.ascontiguousarray(values, np.int64)).to(dev)
        dist.all_reduce(t, op=dist.ReduceOp.SUM, group=self.group)
        return t.cpu().numpy()

    def _gather_to_root(self, values: np.ndarray) -> Optional[np.ndarray]:
        """[world, ...] on rank 0 (None elsewhere): every rank's equally shaped int64 array."""
        if self.world_size == 1:
            return values[None]
        torch, dist = self._torch, self._dist
        dev = self.device if dist.get_backend(self.group) == "nccl" else torch.device("cpu")
        t = torch.from_numpy(np.ascontiguousarray(values, np.int64)).to(dev)
        parts = [torch.empty_like(t) for _ in range(self.world_size)] if self.rank == 0 else None
        dist.gather(t, parts, dst=0, group=self.group)
        return np.stack([p.cpu().numpy() for p in parts]) if self.rank == 0 else None

    def _set_counts(self, counts: np.ndarray) -> None:
        self._counts = np.asarray(counts, np.int64)
        self.total_rows = int(self._counts.sum())

    def count(self) -> int:
        """vectorCount of the whole sharded corpus (the same on every rank)."""
        return self.total_rows

    def add_batch(self, frame_ids: Sequence[int], vectors) -> None:
        """addBatch over the sharded corpus (collective): the same answer, row order and MV2V bytes as one engine given
        the same history.  One all-reduce finds each id's owner; owned ids are upserted in place, the new ones go to the
        ranks with the fewest rows (plan_add_batch)."""
        self._check_corpus_methods()
        ids = np.ascontiguousarray(frame_ids, dtype=np.uint64).reshape(-1)
        if ids.size == 0:
            return
        from .engine import EncodingError, _as_rows
        if ids.size != len(vectors):
            raise EncodingError("addBatch: frameIds.count != vectors.count")
        rows = _as_rows(vectors, self.dimensions)
        held = np.zeros(ids.size + self.world_size, np.int64)
        held[:ids.size] = np.where(self.engine.contains(ids), self.rank + 1, 0)
        held[ids.size + self.rank] = self.engine.count
        held = self._sum_on_ranks(held)
        dest, first_key, appended, next_key = plan_add_batch(ids, held[:ids.size] - 1, held[ids.size:], self._next_key)
        mine = np.flatnonzero(dest == self.rank)
        if mine.size:
            if mine.size == ids.size:                      # the whole batch (always at world 1): no copy
                mine = slice(None)
            got = self.engine.add_batch_keyed(ids[mine], rows[mine], int(first_key[self.rank]))
            assert got == appended[self.rank], (got, appended[self.rank])
        self._set_counts(held[ids.size:] + appended)
        self._next_key = next_key

    def add(self, frame_id: int, vector: Sequence[float]) -> None:
        """add(frameId:vector:) over the sharded corpus (collective)."""
        self.add_batch([frame_id], np.asarray(vector, np.float32).reshape(1, -1))

    def remove_batch(self, frame_ids: Sequence[int]) -> int:
        """remove(frameId:) for many frames over the sharded corpus (collective): every rank removes the ids it holds,
        the survivors keep their keys.  Returns how many rows went, over all ranks."""
        self._check_corpus_methods()
        ids = np.ascontiguousarray(frame_ids, dtype=np.uint64).reshape(-1)
        gone = np.zeros(self.world_size, np.int64)
        gone[self.rank] = self.engine.remove_batch(ids) if ids.size else 0
        gone = self._sum_on_ranks(gone)
        self._set_counts(self._counts - gone)
        return int(gone.sum())

    def remove(self, frame_id: int) -> None:
        """remove(frameId:) over the sharded corpus (collective)."""
        self.remove_batch([frame_id])

    def deserialize(self, data) -> None:
        """Load an MV2V blob (collective, the same bytes on every rank): rank r loads the rows shard_range gives it, keyed
        by their positions in the blob.  A blob deserialize() would refuse is refused on every rank alike."""
        self._check_corpus_methods()
        count = mv2v_count(data)
        lo, hi = shard_range(count, self.world_size, self.rank)
        self.engine.deserialize_rows(data, lo, hi - lo)
        self._set_counts(shard_counts(count, self.world_size))
        self._next_key = count

    def serialize(self, chunk_rows: int = 1 << 16):
        """MV2V bytes of the whole corpus on rank 0 (None on the others): what CUDAVectorEngine.serialize gives for the
        same history.  Collective: the ranks gather their keys on rank 0, then send their rows in chunks of at most
        `chunk_rows`, which rank 0 places by key (plan_serialize)."""
        self._check_corpus_methods()
        count, dims, root = self.engine.count, self.dimensions, self.rank == 0
        counts = self._sum_on_ranks(np.eye(self.world_size, dtype=np.int64)[self.rank] * count)
        width, total = int(counts.max()), int(counts.sum())
        keys = np.zeros(width, np.uint64)
        keys[:count] = self.engine.export_rows(0, count, vectors=False)[2]
        all_keys = self._gather_to_root(keys.view(np.int64))
        if root:
            pos = plan_serialize([all_keys[r, :counts[r]].view(np.uint64) for r in range(self.world_size)])
            out = bytearray(36 + total * dims * 4 + 8 + total * 8)
            out[:36] = mv2v_header(self.metric.to_vec_similarity(), dims, total)
            vbytes = total * dims * 4
            vecs = np.frombuffer(out, np.float32, total * dims, 36).reshape(total, dims)
            out[36 + vbytes:44 + vbytes] = np.uint64(total * 8).tobytes()
            ids_out = np.frombuffer(out, np.uint64, total, 44 + vbytes)

        def place(dst, ids, vec):
            """Rows at MV2V positions `dst` (increasing: a rank's keys increase); a consecutive run is one slice copy."""
            if dst.size and dst[-1] - dst[0] == dst.size - 1:
                dst = slice(int(dst[0]), int(dst[-1]) + 1)
            ids_out[dst], vecs[dst] = ids, vec

        rec = (8 + 4 * dims + 7) // 8 * 8                          # one row on the wire: its id, then its vector
        for first in range(0, width, max(1, int(chunk_rows))):
            m = min(int(chunk_rows), width - first)
            have = max(0, min(m, count - first))
            ids, vec, _ = self.engine.export_rows(first, have) if have else (None, None, None)
            if root and have:                                       # rank 0's own rows skip the wire
                place(pos[0][first:first + have], ids, vec)
            if self.world_size == 1:
                continue
            wire = np.zeros((m, rec), np.uint8)
            if have and not root:
                wire[:have, :8] = ids.view(np.uint8).reshape(have, 8)
                wire[:have, 8:8 + 4 * dims] = vec.view(np.uint8).reshape(have, 4 * dims)
            got = self._gather_to_root(wire.view(np.int64).reshape(-1))
            if root:
                got = got.view(np.uint8).reshape(self.world_size, m, rec)
                for r in range(1, self.world_size):
                    n_r = max(0, min(m, int(counts[r]) - first))
                    place(pos[r][first:first + n_r], np.ascontiguousarray(got[r, :n_r, :8]).view(np.uint64).reshape(-1),
                          np.ascontiguousarray(got[r, :n_r, 8:8 + 4 * dims]).view(np.float32))
        return out if root else None

    def rebalance(self, chunk_rows: Optional[int] = None) -> int:
        """Even out the ranks' rows in place (collective, no arguments needed): every rank ends with the row count
        plan_rebalance gives it, each moved row taking its key, group, attributes, location and terms with it, so every
        answer, serialize() included, stays that of one engine with the same history.  Returns the rows moved, the same
        on every rank.

        One all-reduce of the ranks' row counts confirms the bookkeeping; a balanced corpus stops there.  Then, move by
        move in plan order, the donor sends the next part of its tail (in key order) to the receiver point to point, in
        chunks of at most `chunk_rows` rows (default: 256 MiB of vectors): a header, one fixed-width record per row (id,
        key, group, attributes, location, term count), the vectors (a device tensor under NCCL, host memory under gloo)
        and the term ids.  The receiver merges each chunk by key (absorb_rows), which rewrites its rows above the chunk's
        first key; its extra device memory is one chunk plus the merge's slab buffers.  One all-reduce of the rows each
        move delivered follows; each donor drops those rows.  A receiver that fails keeps what it merged before and
        absorbs nothing more, the rest stays on the donors, and every rank raises the same error with the failing
        rank's reason."""
        self._check_corpus_methods()
        torch, dist = self._torch, self._dist
        from .engine import InvalidToc, ROW_COLUMNS_DTYPE, RowColumns
        counts = self._sum_on_ranks(np.eye(self.world_size, dtype=np.int64)[self.rank] * self.engine.count)
        if not np.array_equal(counts, self._counts):
            raise InvalidToc(f"rebalance: the ranks hold {counts.tolist()} rows, the bookkeeping says {self._counts.tolist()}")
        _, moves = plan_rebalance(counts)
        if not moves:
            return 0
        dims = self.dimensions
        chunk = max(1, int(chunk_rows) if chunk_rows else (256 << 20) // (4 * dims))
        wire = self.device if dist.get_backend(self.group) == "nccl" else torch.device("cpu")
        rec = np.dtype([("id", "<u8"), ("key", "<u8"), ("cols", ROW_COLUMNS_DTYPE), ("n_terms", "<u8")])
        tail = counts.copy()                                       # tail[d]: where donor d's next run starts
        for d, _, rows in moves:
            tail[d] -= rows
        first = []
        for d, _, rows in moves:
            first.append(int(tail[d]))
            tail[d] += rows
        done = np.zeros(len(moves) + self.world_size, np.int64)    # rows each move delivered, then a failure flag per rank
        failure = None
        for i, (d, r, rows) in enumerate(moves):
            if self.rank not in (d, r):
                continue
            for lo in range(0, rows, chunk):
                m = min(chunk, rows - lo)
                if self.rank == d:
                    row = first[i] + lo
                    ids, _, keys = self.engine.export_rows(row, m, vectors=False)
                    cols = self.engine.export_columns(row, m)
                    records = np.zeros(m, rec)
                    records["id"], records["key"], records["cols"] = ids, keys, cols.records
                    records["n_terms"] = np.diff(cols.term_offsets)
                    head = np.array([cols.set, cols.terms.size], np.int64)
                    dist.send(torch.from_numpy(head).to(wire), r, group=self.group)
                    dist.send(torch.from_numpy(records.view(np.uint8).reshape(-1)).to(wire), r, group=self.group)
                    dist.send(self.engine.export_vectors(row, m).to(wire), r, group=self.group)
                    if cols.terms.size:
                        dist.send(torch.from_numpy(cols.terms.view(np.int64)).to(wire), r, group=self.group)
                    continue
                head = torch.empty(2, dtype=torch.int64, device=wire)
                dist.recv(head, d, group=self.group)
                bits, n_terms = (int(x) for x in head.cpu())
                raw = torch.empty(m * rec.itemsize, dtype=torch.uint8, device=wire)
                dist.recv(raw, d, group=self.group)
                vecs = torch.empty((m, dims), dtype=torch.float32, device=wire)
                dist.recv(vecs, d, group=self.group)
                terms = torch.empty(n_terms, dtype=torch.int64, device=wire)
                if n_terms:
                    dist.recv(terms, d, group=self.group)
                if failure is not None:                            # drained, not merged: the rows stay on the donor
                    continue
                records = raw.cpu().numpy().view(rec)
                offsets = np.zeros(m + 1, np.uint64)
                offsets[1:] = np.cumsum(records["n_terms"])
                try:
                    self.engine.absorb_rows(records["id"], records["key"], vecs.to(self.device),
                                            RowColumns(bits, records["cols"], offsets, terms.cpu().numpy().view(np.uint64)))
                    done[i] += m
                except Exception as exc:                           # noqa: BLE001 -- every rank re-raises it below
                    failure = exc
        if failure is not None:
            done[len(moves) + self.rank] = 1
        done = self._sum_on_ranks(done)
        drop = []
        for i, (d, r, rows) in enumerate(moves):
            n_done = int(done[i])
            if self.rank == d and n_done:
                drop.append(self.engine.export_rows(first[i], n_done, vectors=False)[0])
            counts[d] -= n_done
            counts[r] += n_done
        if drop:
            self.engine.remove_batch(np.concatenate(drop))
        self._set_counts(counts)
        failed = np.flatnonzero(done[len(moves):])
        if failed.size:
            src = int(failed[0])
            why = [(type(failure).__name__, str(failure)) if self.rank == src else None]
            dist.broadcast_object_list(why, src=src if self.group is None else dist.get_global_rank(self.group, src),
                                       group=self.group)
            from . import engine as E
            cls = getattr(E, why[0][0], None)
            cls = cls if isinstance(cls, type) and issubclass(cls, E.WaxError) else RuntimeError
            raise cls(f"rebalance: rank {src} could not absorb its rows: {why[0][1]}")
        return int(done[:len(moves)].sum())

    # -- search
    def _buffers(self, k: int, slot: int = 0):
        torch = self._torch
        key = (k, slot)
        if key not in self._bufs:
            local = torch.zeros(k * 24, dtype=torch.uint8, device=self.device)
            gathered = torch.zeros(self.world_size * k * 24, dtype=torch.uint8, device=self.device)
            host = torch.zeros(self.world_size * k * 24, dtype=torch.uint8,
                               pin_memory=(self.device.type == "cuda"))
            self._bufs[key] = (local, gathered, host)
        return self._bufs[key]

    def search_async(self, d_query, top_k: int, slot: int = 0):
        """Enqueue local scan + all-gather + D2H on the current stream; returns a handle for finish().
        Queries are independent, so several may be in flight: give each a distinct `slot` (its result buffers)
        and finish() them in order -- the host merge of query i then overlaps the scan of query i+1."""
        torch, dist = self._torch, self._dist
        k = clamp_topk(top_k)
        local, gathered, host = self._buffers(k, slot)
        if self._local_search is not None:
            cands = np.ascontiguousarray(self._local_search(np.asarray(d_query, np.float32), k), dtype=CAND_DTYPE)
            local.copy_(torch.from_numpy(cands.view(np.uint8).reshape(-1).copy()))
        else:
            from . import _lib as L
            stream = torch.cuda.current_stream(self.device)
            rc = L.lib().wax_vs_search_device(self.engine.handle, C.c_void_p(d_query.data_ptr()), 1, k,
                                              self.row_lo, C.c_void_p(local.data_ptr()),
                                              C.c_void_p(stream.cuda_stream))
            if rc != 0:
                raise RuntimeError(f"wax_vs_search_device rc={rc}: {L.last_error()}")
        if self._comm_stream is not None:
            # exchange + D2H on the communication stream: the compute stream is free to start the next query
            scanned = torch.cuda.Event()
            scanned.record()
            with torch.cuda.stream(self._comm_stream):
                self._comm_stream.wait_event(scanned)
                if self.world_size > 1:
                    dist.all_gather_into_tensor(gathered, local, group=self.group)
                else:
                    gathered.copy_(local)
                host.copy_(gathered, non_blocking=True)
                ev = torch.cuda.Event()
                ev.record()
            return (host, ev, k)
        if self.world_size > 1:
            dist.all_gather_into_tensor(gathered, local, group=self.group)
        else:
            gathered.copy_(local)
        host.copy_(gathered)
        return (host, None, k)

    def search_many_async(self, d_queries, top_k: int, slot: int = 0):
        """G independent queries (`d_queries`: [G, dims] device tensor) with ONE exchange: G fused scans alternating
        over two streams, one all-gather of G*k candidates per rank, one D2H.  Returns a handle for finish_many()."""
        torch, dist = self._torch, self._dist
        from . import _lib as L
        g = int(d_queries.shape[0])
        k = clamp_topk(top_k)
        key = (k, g, slot)
        if key not in self._bufs:
            local = torch.zeros(g * k * 24, dtype=torch.uint8, device=self.device)
            gathered = torch.zeros(self.world_size * g * k * 24, dtype=torch.uint8, device=self.device)
            host = torch.zeros(self.world_size * g * k * 24, dtype=torch.uint8, pin_memory=True)
            self._bufs[key] = (local, gathered, host)
        local, gathered, host = self._bufs[key]
        ready = torch.cuda.Event()
        ready.record()                                   # queries were produced on the current stream
        scanned = []
        n_streams = min(2 if self._overlap_scans else 1, g)
        for st in self._scan_streams[:n_streams]:
            st.wait_event(ready)
        q_base, q_stride = d_queries.data_ptr(), d_queries.stride(0) * 4
        for i in range(g):
            st = self._scan_streams[i % n_streams]
            rc = L.lib().wax_vs_search_device(self.engine.handle, C.c_void_p(q_base + i * q_stride), 1, k,
                                              self.row_lo, C.c_void_p(local.data_ptr() + i * k * 24),
                                              C.c_void_p(st.cuda_stream))
            if rc != 0:
                raise RuntimeError(f"wax_vs_search_device rc={rc}: {L.last_error()}")
        for st in self._scan_streams[:n_streams]:
            ev = torch.cuda.Event()
            ev.record(st)
            scanned.append(ev)
        with torch.cuda.stream(self._comm_stream):
            for ev in scanned:
                self._comm_stream.wait_event(ev)
            if self.world_size > 1:
                dist.all_gather_into_tensor(gathered, local, group=self.group)
            else:
                gathered.copy_(local)
            host.copy_(gathered, non_blocking=True)
            done = torch.cuda.Event()
            done.record()
        return (host, done, k, g)

    def finish_many(self, handle) -> List[List[Tuple[int, float]]]:
        host, done, k, g = handle
        done.synchronize()
        cands = host.numpy().view(CAND_DTYPE).reshape(self.world_size, g, k)
        k_eff = min(k, self.total_rows) if self.total_rows else k
        sim = self.metric.to_vec_similarity()
        out = []
        for i in range(g):
            best = merge_candidates(cands[:, i, :], k_eff)
            scores = score_from_distance(sim, best["distance"])
            out.append([(int(best["frame_id"][j]), float(scores[j])) for j in range(best.size)])
        return out

    def _merge_on_device(self, gathered, b: int, k: int, k_eff: int, stream):
        """[world][b][k] gathered candidates (device bytes) -> [b][k_eff] merged candidates on the device, by the library's
        merge kernel (same (distance, GLOBAL row) rule as the fused exchange); enqueued on `stream`."""
        from . import _lib as L
        merged = self._torch.empty(b * k_eff * 24, dtype=self._torch.uint8, device=self.device)
        rc = L.lib().wax_vs_merge_candidates_device(self.engine.handle, C.c_void_p(gathered.data_ptr()), self.world_size, b, k,
                                                    k_eff, C.c_void_p(merged.data_ptr()), C.c_void_p(stream.cuda_stream))
        if rc != 0:
            raise RuntimeError(f"wax_vs_merge_candidates_device rc={rc}: {L.last_error()}")
        return merged

    def _unpack_merged(self, host_bytes: np.ndarray, b: int, k_eff: int):
        best = host_bytes.view(CAND_DTYPE).reshape(b, k_eff)
        scores = score_from_distance(self.metric.to_vec_similarity(), best["distance"])
        return best["frame_id"].astype(np.uint64), scores, (best["valid"] != 0).sum(axis=1).astype(np.uint32)

    def search_batch_arrays(self, queries, top_k: int):
        """A batch of independent queries against the sharded corpus: every rank runs the batched tensor-core levels
        (wax_vs_search_batch_device: bf16-shadow nominations -> TF32 retry -> exact scan, results identical to
        single-query scans; cosine and dot, l2 with the engine option batch_l2 = 1) on its shard, ONE all-gather carries batch x k candidates per rank, ONE merge kernel
        (wax_vs_merge_candidates_device) ranks them on the device.  `queries`: [batch, dims] host array or device tensor (identical on every rank).  Returns
        (ids [batch, k_eff] uint64, scores [batch, k_eff] float32, n_valid [batch] uint32)."""
        torch, dist = self._torch, self._dist
        k = clamp_topk(top_k)
        k_eff = min(k, self.total_rows) if self.total_rows else k
        if self._local_search is not None:
            qs = np.ascontiguousarray(queries, dtype=np.float32).reshape(-1, self.dimensions)
            b = qs.shape[0]
            local_np = np.zeros((b, k), CAND_DTYPE)
            for i in range(b):
                local_np[i] = np.ascontiguousarray(self._local_search(qs[i], k), dtype=CAND_DTYPE)
            local = torch.from_numpy(local_np.view(np.uint8).reshape(-1).copy())
        else:
            from . import _lib as L
            if isinstance(queries, torch.Tensor):
                d_qs = queries.to(self.device, dtype=torch.float32).contiguous().reshape(-1, self.dimensions)
            else:
                d_qs = torch.from_numpy(np.ascontiguousarray(queries, dtype=np.float32).reshape(-1, self.dimensions)).to(self.device)
            b = int(d_qs.shape[0])
            local = torch.empty(b * k * 24, dtype=torch.uint8, device=self.device)
            stream = torch.cuda.current_stream(self.device)
            rc = L.lib().wax_vs_search_batch_device(self.engine.handle, C.c_void_p(d_qs.data_ptr()), b, k, self.row_lo,
                                                    C.c_void_p(local.data_ptr()), C.c_void_p(stream.cuda_stream))
            if rc != 0:
                raise RuntimeError(f"wax_vs_search_batch_device rc={rc}: {L.last_error()}")
        if b == 0 or self.total_rows == 0:
            return np.zeros((b, 0), np.uint64), np.zeros((b, 0), np.float32), np.zeros(b, np.uint32)
        if self.world_size > 1:
            gathered = torch.empty(self.world_size * b * k * 24, dtype=torch.uint8, device=local.device)
            dist.all_gather_into_tensor(gathered, local, group=self.group)
        else:
            gathered = local
        if self._local_search is None:      # GPU: merge on the device, one D2H of the final batch x k_eff records
            merged = self._merge_on_device(gathered, b, k, k_eff, torch.cuda.current_stream(self.device))
            return self._unpack_merged(merged.cpu().numpy(), b, k_eff)
        cands = gathered.cpu().numpy().view(CAND_DTYPE).reshape(self.world_size, b, k)
        best, n_valid = merge_candidates_batch(cands, k_eff)
        scores = score_from_distance(self.metric.to_vec_similarity(), best["distance"])
        return best["frame_id"].astype(np.uint64), scores, n_valid

    # -- pipelined batches: the host merge of batch i overlaps the tensor-core pass of batch i+1 ----------------------
    def search_batch_submit(self, queries, top_k: int):
        """Start a batch on the engine's worker thread (ONE worker: batches, and therefore the all-gathers, are issued
        in submission order on every rank) and return a future for finish_batch().  The worker does the shard's
        tensor-core levels (a blocking C call that releases the GIL), the all-gather and the D2H copy; the caller is
        free to merge the previous batch meanwhile.  Queries must stay alive until finish_batch()."""
        torch, dist = self._torch, self._dist
        if getattr(self, "_worker", None) is None:
            from concurrent.futures import ThreadPoolExecutor
            self._worker = ThreadPoolExecutor(max_workers=1, thread_name_prefix="waxvs-shard")
            self._batch_stream = torch.cuda.Stream(device=self.device) if self._local_search is None else None
        k = clamp_topk(top_k)
        if self._local_search is not None:
            # CPU (gloo) form used by the tests of the host logic: the injected local search stands in for the GPU
            # step; the worker thread, the submission-ordered all-gathers and the merge are the production ones.
            qs = np.ascontiguousarray(queries, dtype=np.float32).reshape(-1, self.dimensions).copy()
            b = qs.shape[0]

            def work_cpu():
                local_np = np.zeros((b, k), CAND_DTYPE)
                for i in range(b):
                    local_np[i] = np.ascontiguousarray(self._local_search(qs[i], k), dtype=CAND_DTYPE)
                local = torch.from_numpy(local_np.view(np.uint8).reshape(-1).copy())
                if self.world_size > 1:
                    gathered = torch.empty(self.world_size * b * k * 24, dtype=torch.uint8)
                    dist.all_gather_into_tensor(gathered, local, group=self.group)
                else:
                    gathered = local
                return gathered, None, None, None

            return (self._worker.submit(work_cpu), b, k)
        if isinstance(queries, torch.Tensor):
            d_qs = queries.to(self.device, dtype=torch.float32).contiguous().reshape(-1, self.dimensions)
        else:
            d_qs = torch.from_numpy(np.ascontiguousarray(queries, dtype=np.float32).reshape(-1, self.dimensions)).to(self.device)
        ready = torch.cuda.Event()
        ready.record()                                   # the queries were produced on the caller's stream
        b = int(d_qs.shape[0])

        def work():
            from . import _lib as L
            torch.cuda.set_device(self.device)
            with torch.cuda.stream(self._batch_stream):
                self._batch_stream.wait_event(ready)
                local = torch.empty(b * k * 24, dtype=torch.uint8, device=self.device)
                rc = L.lib().wax_vs_search_batch_device(self.engine.handle, C.c_void_p(d_qs.data_ptr()), b, k, self.row_lo,
                                                        C.c_void_p(local.data_ptr()), C.c_void_p(self._batch_stream.cuda_stream))
                if rc != 0:
                    raise RuntimeError(f"wax_vs_search_batch_device rc={rc}: {L.last_error()}")
                if self.world_size > 1:
                    gathered = torch.empty(self.world_size * b * k * 24, dtype=torch.uint8, device=self.device)
                    dist.all_gather_into_tensor(gathered, local, group=self.group)
                else:
                    gathered = local
                k_eff = min(k, self.total_rows) if self.total_rows else k
                merged = self._merge_on_device(gathered, b, k, k_eff, self._batch_stream) if b and self.total_rows else gathered
                host = torch.empty(merged.numel(), dtype=torch.uint8, pin_memory=True)
                host.copy_(merged, non_blocking=True)
                done = torch.cuda.Event()
                done.record()
            return host, done, (gathered, merged), d_qs  # keep the device buffers alive until the copy has finished

        return (self._worker.submit(work), b, k)

    def finish_batch(self, handle):
        """Wait for a submitted batch and merge it: (ids [batch, k_eff], scores, n_valid) as search_batch_arrays."""
        fut, b, k = handle
        host, done, _gathered, _d_qs = fut.result()
        if done is not None:
            done.synchronize()
        k_eff = min(k, self.total_rows) if self.total_rows else k
        if b == 0 or self.total_rows == 0:
            return np.zeros((b, 0), np.uint64), np.zeros((b, 0), np.float32), np.zeros(b, np.uint32)
        if self._local_search is None:      # GPU: the worker already merged on the device
            return self._unpack_merged(host.numpy(), b, k_eff)
        cands = host.numpy().view(CAND_DTYPE).reshape(self.world_size, b, k)
        best, n_valid = merge_candidates_batch(cands, k_eff)
        scores = score_from_distance(self.metric.to_vec_similarity(), best["distance"])
        return best["frame_id"].astype(np.uint64), scores, n_valid

    def search_batch(self, queries, top_k: int) -> List[List[Tuple[int, float]]]:
        ids, scores, ns = self.search_batch_arrays(queries, top_k)
        return [[(int(ids[i, j]), float(scores[i, j])) for j in range(int(ns[i]))] for i in range(ids.shape[0])]

    def finish(self, handle) -> List[Tuple[int, float]]:
        host, ev, k = handle
        if ev is not None:
            ev.synchronize()
        cands = host.numpy().view(CAND_DTYPE)
        k_eff = min(k, self.total_rows) if self.total_rows else k
        best = merge_candidates(cands, k_eff)
        scores = score_from_distance(self.metric.to_vec_similarity(), best["distance"])
        return [(int(best["frame_id"][i]), float(scores[i])) for i in range(best.size)]

    def search(self, vector: Sequence[float], top_k: int) -> List[Tuple[int, float]]:
        torch = self._torch
        q = np.ascontiguousarray(vector, dtype=np.float32).reshape(-1)
        if q.size != self.dimensions:
            from .engine import EncodingError
            raise EncodingError(f"vector dimension mismatch: expected {self.dimensions}, got {q.size}")
        if self.total_rows == 0:
            return []
        if self._local_search is not None:
            return self.finish(self.search_async(q, top_k))
        if self.transport == "p2p-fused" and clamp_topk(top_k) <= 128:
            return self._search_fused(q, top_k)
        d_q = torch.from_numpy(q).to(self.device, non_blocking=False)
        return self.finish(self.search_async(d_q, top_k))

    def search_filtered(self, vector: Sequence[float], top_k: int, allow=None, deny=None) -> List[Tuple[int, float]]:
        """Filtered search over the whole sharded corpus (collective: same query and ids on every rank).  Needs the
        fused peer-memory transport: the filter rides in each rank's scan, the exchange is unchanged."""
        q = np.ascontiguousarray(vector, dtype=np.float32).reshape(-1)
        if q.size != self.dimensions:
            from .engine import EncodingError
            raise EncodingError(f"vector dimension mismatch: expected {self.dimensions}, got {q.size}")
        if self.total_rows == 0:
            return []
        if self.transport != "p2p-fused" or clamp_topk(top_k) > 128:
            from .engine import InvalidToc
            raise InvalidToc("sharded filtered search needs the p2p-fused transport and top_k <= 128")
        return self.engine.shard_search_filtered(q, top_k, allow=allow, deny=deny)

    # -- frame attributes and where search: the clauses ride below every rank's top-k, as in search_filtered
    def set_attributes(self, frame_ids, timestamps=None, tags=None) -> int:
        """CUDAVectorEngine.set_attributes on this rank's engine.  The full lists may be passed (ids this shard does not
        hold are ignored) or only its own frames.  Returns this rank's assigned count."""
        return self.engine.set_attributes(frame_ids, timestamps, tags)

    def set_locations(self, frame_ids, latitudes, longitudes) -> int:
        """CUDAVectorEngine.set_locations on this rank's engine (full lists or this rank's frames)."""
        return self.engine.set_locations(frame_ids, latitudes, longitudes)

    def set_terms(self, frame_ids, term_lists) -> int:
        """CUDAVectorEngine.set_terms on this rank's engine (full lists or this rank's frames)."""
        return self.engine.set_terms(frame_ids, term_lists)

    def search_where(self, vector: Sequence[float], top_k: int, where, allow=None, deny=None) -> List[Tuple[int, float]]:
        """The best `top_k` frames of the whole sharded corpus passing `where` and the optional id filter (collective:
        same arguments on every rank); equal to CUDAVectorEngine.search_where on one engine holding the corpus.  The fused
        transport with top_k <= 128 takes one exchange inside the scan (wax_vs_shard_search_where); otherwise the
        batched device form runs for one query."""
        q = np.ascontiguousarray(vector, dtype=np.float32).reshape(-1)
        if q.size != self.dimensions:
            from .engine import EncodingError
            raise EncodingError(f"vector dimension mismatch: expected {self.dimensions}, got {q.size}")
        if allow is not None and deny is not None:
            raise ValueError("pass at most one of allow= / deny=")
        if self.transport == "p2p-fused" and clamp_topk(top_k) <= 128:
            return self.engine.shard_search_where(q, top_k, where, allow=allow, deny=deny)
        filters = [("allow", allow)] if allow is not None else ([("deny", deny)] if deny is not None else [])
        return self.search_batch_where(q.reshape(1, -1), top_k, [where], [0], filters, [0 if filters else None])[0]

    def search_batch_where(self, vectors, top_k: int, wheres, query_where, filters=None,
                           query_filter=None) -> List[List[Tuple[int, float]]]:
        """CUDAVectorEngine.search_batch_where over the whole sharded corpus (collective): every rank plans its shard with
        wax_vs_search_batch_where_device, ONE all-gather carries batch x k candidates per rank, ONE merge kernel ranks them
        (wax_vs_merge_candidates_device) and ONE copy brings the answers to the host.  Any transport, k up to 10 000."""
        from . import _lib as L
        from .engine import _WhereArgs
        torch, dist = self._torch, self._dist
        qs = np.ascontiguousarray(vectors, dtype=np.float32).reshape(-1, self.dimensions)
        b = qs.shape[0]
        if any(w.groups for w in wheres):
            raise ValueError("the sharded engine takes no group clause")
        if any(w.has_root_clause for w in wheres):
            raise ValueError("the sharded engine takes no root clause")
        a = _WhereArgs(wheres, query_where, filters, query_filter, b)
        if b == 0:
            return []
        k = clamp_topk(top_k)
        d_qs = torch.from_numpy(qs).to(self.device)
        local = torch.empty(b * k * 24, dtype=torch.uint8, device=self.device)
        stream = torch.cuda.current_stream(self.device)
        rc = L.lib().wax_vs_search_batch_where_device(self.engine.handle, C.c_void_p(d_qs.data_ptr()), b, k,
                                                      *a.filter_args(), *a.where_args(near=True), *a.term_args(),
                                                      self.row_lo, C.c_void_p(local.data_ptr()),
                                                      C.c_void_p(stream.cuda_stream))
        if rc != 0:
            raise RuntimeError(f"wax_vs_search_batch_where_device rc={rc}: {L.last_error()}")
        if self.world_size > 1:
            gathered = torch.empty(self.world_size * b * k * 24, dtype=torch.uint8, device=self.device)
            dist.all_gather_into_tensor(gathered, local, group=self.group)
        else:
            gathered = local
        merged = self._merge_on_device(gathered, b, k, k, stream)
        ids, scores, ns = self._unpack_merged(merged.cpu().numpy(), b, k)
        return [[(int(ids[i, j]), float(scores[i, j])) for j in range(int(ns[i]))] for i in range(b)]

    # -- grouped search: the best frames of the top groups, exact, in two exchanges (DESIGN.md section 4.14)
    def set_groups(self, frame_ids, group_ids) -> int:
        """CUDAVectorEngine.set_groups on this rank's engine (full lists or this rank's frames).  Returns this rank's
        assigned count."""
        return self.engine.set_groups(frame_ids, group_ids)

    def _all_gather(self, local):
        """[world][local] bytes on the device: the ranks' buffers in rank order."""
        if self.world_size == 1:
            return local
        gathered = self._torch.empty(self.world_size * local.numel(), dtype=self._torch.uint8, device=self.device)
        self._dist.all_gather_into_tensor(gathered, local, group=self.group)
        return gathered

    def search_batch_grouped(self, vectors, top_groups: int, per_group: int = 1, wheres=None, query_where=None,
                             filters=None, query_filter=None) -> List[List[Tuple[int, List[Tuple[int, float]]]]]:
        """CUDAVectorEngine.search_batch_grouped_multi_where over the whole sharded corpus (collective, any transport;
        arguments as there, wheres and filters optional; clamp(top_groups) <= 256).  Round 1: every rank's own grouped
        answer (wax_vs_shard_grouped_heads_device), one all-gather, the global top groups by their best rows
        (wax_vs_merge_group_heads_device).  per_group > 1 adds round 2: every rank's best rows of each chosen group
        (wax_vs_shard_grouped_expand_device), a second all-gather and the per-group merge (wax_vs_merge_candidates_device).
        One copy brings the answer to the host.  Equal, bit for bit, to the single engine's answer."""
        from . import _lib as L
        from .engine import _check, _WhereArgs
        torch = self._torch
        qs = np.ascontiguousarray(vectors, dtype=np.float32).reshape(-1, self.dimensions)
        b = qs.shape[0]
        wheres = list(wheres or [])
        if any(w.terms for w in wheres):
            raise ValueError("grouped search takes no term clause")
        if any(w.groups for w in wheres):
            raise ValueError("the sharded engine takes no group clause")
        if any(w.has_root_clause for w in wheres):
            raise ValueError("the sharded engine takes no root clause")
        a = _WhereArgs(wheres, [None] * b if query_where is None else query_where, filters, query_filter, b)
        if b == 0:
            return []
        g, p = clamp_topk(top_groups), max(int(per_group), 1)
        lib, h = L.lib(), self.engine.handle
        d_qs = torch.from_numpy(qs).to(self.device)
        stream = torch.cuda.current_stream(self.device)
        s = C.c_void_p(stream.cuda_stream)
        fargs, wargs = a.filter_args(), a.where_args(near=True)
        heads = torch.empty(b * g * p * GROUP_CAND_DTYPE.itemsize, dtype=torch.uint8, device=self.device)
        _check(lib.wax_vs_shard_grouped_heads_device(h, C.c_void_p(d_qs.data_ptr()), b, int(top_groups), int(per_group),
                                                     *fargs, *wargs, self.row_lo, C.c_void_p(heads.data_ptr()), s))
        gathered = self._all_gather(heads)
        chosen = torch.empty(b * g * GROUP_CAND_DTYPE.itemsize, dtype=torch.uint8, device=self.device)
        _check(lib.wax_vs_merge_group_heads_device(h, C.c_void_p(gathered.data_ptr()), self.world_size, b, int(top_groups),
                                                   int(per_group), C.c_void_p(chosen.data_ptr()), s))
        sim = self.metric.to_vec_similarity()
        if p == 1:
            best = chosen.cpu().numpy().view(GROUP_CAND_DTYPE).reshape(b, g)
            scores = score_from_distance(sim, best["distance"])
            return [[(int(best["group_id"][i, j]), [(int(best["frame_id"][i, j]), float(scores[i, j]))])
                     for j in range(g) if best["valid"][i, j]] for i in range(b)]
        rows = torch.empty(b * g * p * CAND_DTYPE.itemsize, dtype=torch.uint8, device=self.device)
        _check(lib.wax_vs_shard_grouped_expand_device(h, C.c_void_p(d_qs.data_ptr()), b, int(top_groups), int(per_group),
                                                      *fargs, *wargs, C.c_void_p(chosen.data_ptr()),
                                                      C.c_void_p(heads.data_ptr()), self.row_lo,
                                                      C.c_void_p(rows.data_ptr()), s))
        merged = self._merge_on_device(self._all_gather(rows), b * g, p, p, stream)
        host = torch.cat([chosen, merged]).cpu().numpy()
        groups = host[:chosen.numel()].view(GROUP_CAND_DTYPE).reshape(b, g)
        best = host[chosen.numel():].view(CAND_DTYPE).reshape(b, g, p)
        scores = score_from_distance(sim, best["distance"])
        return [[(int(groups["group_id"][i, j]), [(int(best["frame_id"][i, j, m]), float(scores[i, j, m]))
                                                   for m in range(p) if best["valid"][i, j, m]])
                 for j in range(g) if groups["valid"][i, j]] for i in range(b)]

    def search_grouped(self, vector: Sequence[float], top_groups: int, per_group: int = 1, where=None, allow=None,
                       deny=None) -> List[Tuple[int, List[Tuple[int, float]]]]:
        """search_batch_grouped for one query (collective): CUDAVectorEngine.search_grouped's answer over the whole sharded
        corpus, under an optional where and at most one of allow= / deny=."""
        q = np.ascontiguousarray(vector, dtype=np.float32).reshape(-1)
        if q.size != self.dimensions:
            from .engine import EncodingError
            raise EncodingError(f"vector dimension mismatch: expected {self.dimensions}, got {q.size}")
        if allow is not None and deny is not None:
            raise ValueError("pass at most one of allow= / deny=")
        filters = [("allow", allow)] if allow is not None else ([("deny", deny)] if deny is not None else [])
        return self.search_batch_grouped(q.reshape(1, -1), top_groups, per_group, [] if where is None else [where],
                                         [None if where is None else 0], filters, [0 if filters else None])[0]

    def _search_fused(self, q: np.ndarray, top_k: int) -> List[Tuple[int, float]]:
        """wax_vs_shard_search: host query in, merged host result out; scan + NVLink exchange + merge in one launch."""
        return self.engine.shard_search(q, top_k)

    def time_search(self, top_k: int, iters: int, warmup: int = 3, n_queries: int = 1, seed: int = 7):
        """Device-timed collective searches, strictly one at a time on one stream (the sharded twin of
        CUDAVectorEngine.time_search).  Returns (ms_total, kernel launches)."""
        return self.engine.time_shard_search(top_k, iters, warmup=warmup, n_queries=n_queries, seed=seed)
