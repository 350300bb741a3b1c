"""Host-side mirror of Wax's `VectorSearchEngine` surface over the CUDA C-ABI.

The reference's host language is Swift, which this image cannot compile; `swift/CUDAVectorEngine.swift`
(uncompiled, see INTEGRATION.md) is the literal binding.  This module is the same surface in Python so the
parity tests read like the reference's own tests (Tests/WaxIntegrationTests/VectorSearchEngineTests.swift):

    protocol VectorSearchEngine            Sources/WaxVectorSearch/VectorSearchEngine.swift:10-18
    enum VectorMetric                      Sources/WaxVectorSearch/VectorMetric.swift:5-54
    actor MetalVectorEngine (public API)   Sources/WaxVectorSearch/MetalVectorEngine.swift:144-146,153,330-446,682-828
    WaxVectorSearchSession.search          Sources/Wax/VectorSearchSession.swift:70-76
    VectorMath.normalizeL2/isNormalizedL2  Sources/Wax/Utilities/VectorMath.swift:15-33,123-127
    WaxError cases                         encodingError / capacityExceeded / invalidToc

Everything numeric happens in libwaxvs_cuda.so; nothing here computes a distance.
"""
from __future__ import annotations

import ctypes as C
import dataclasses
import enum
import threading
from typing import Iterable, List, NamedTuple, Optional, Sequence, Tuple

import numpy as np

from . import _lib as L


# ---- WaxError (the cases the vector engines throw) ---------------------------------------------------------
class WaxError(Exception):
    pass


class EncodingError(WaxError):      # WaxError.encodingError(reason:)
    pass


class CapacityExceeded(WaxError):   # WaxError.capacityExceeded(limit:requested:)
    pass


class InvalidToc(WaxError):         # WaxError.invalidToc(reason:)
    pass


def _raise(rc: int) -> None:
    reason = L.last_error()
    if rc == L.ERR_DIMENSION:
        raise EncodingError(reason)
    if rc == L.ERR_CAPACITY:
        raise CapacityExceeded(reason)
    raise InvalidToc(f"{reason} (rc={rc})")


def _check(rc: int) -> None:
    if rc != L.OK:
        _raise(rc)


# ---- VectorMetric (VectorMetric.swift:5-54) -----------------------------------------------------------------
class VectorMetric(enum.Enum):
    cosine = 0
    dot = 1
    l2 = 2

    def to_vec_similarity(self) -> int:          # toVecSimilarity (:45-54); VecSimilarity raw value
        return self.value

    def score(self, from_distance: float) -> float:  # score(fromDistance:) (:32-43)
        d = np.float32(from_distance)
        if not np.isfinite(d):
            return 0.0
        return float(np.float32(1) - d) if self is VectorMetric.cosine else float(-d)


class VectorEnginePreference(enum.Enum):     # VectorSearchEngine.swift:4-8 (metalPreferred -> the GPU engine)
    auto = 0
    gpu_preferred = 1
    cpu_only = 2


# ---- VectorMath (host-side query preparation only) -------------------------------------------------------------
def normalize_l2(vector: Sequence[float]) -> np.ndarray:
    """VectorMath.normalizeL2 (VectorMath.swift:15-33): x * (1/|x|); empty or zero vectors unchanged."""
    v = np.ascontiguousarray(vector, dtype=np.float32)
    if v.size == 0:
        return v
    s = np.float32(0)
    for x in v:                       # vDSP_svesq: plain fp32 sum of squares
        s = np.float32(s + x * x)
    m = np.float32(np.sqrt(s))
    if not m > 0:
        return v
    return (v * np.float32(np.float32(1) / m)).astype(np.float32)


def is_normalized_l2(vector: Sequence[float], tolerance: float = 1e-3) -> bool:
    """VectorMath.isNormalizedL2 (VectorMath.swift:123-127)."""
    v = np.ascontiguousarray(vector, dtype=np.float32)
    if v.size == 0:
        return False
    s = np.float32(0)
    for x in v:
        s = np.float32(s + x * x)
    return bool(abs(np.float32(np.sqrt(s)) - np.float32(1)) <= np.float32(tolerance))


@dataclasses.dataclass(frozen=True)
class Where:
    """A predicate on a frame's attributes (wax_vs_where): timestamp in [after, before) -- TimeRange.contains,
    SearchRequest.swift:90-105 -- with every bit of all_tags set and no bit of no_tags.  The defaults bound nothing
    (before = INT64_MAX lets a timestamp of INT64_MAX pass)."""
    after: int = L.INT64_MIN
    before: int = L.INT64_MAX
    all_tags: int = 0
    no_tags: int = 0
    # PhotoRAG's location clause (wax_vs_where_near): (latitude, longitude, radius_m), the frames in the box of 0.01-degree
    # bins buildLocationAllowlist would union (see location_box).  None: no location clause.
    near: Optional[Tuple[float, float, float]] = None
    # Term clause (wax_vs_search_batch_where_terms): up to 32 term ids the frame's set must all hold (see set_terms and
    # TermDictionary).  Empty: no term clause.
    terms: Tuple[int, ...] = ()
    # Group clause (wax_vs_search_batch_where_groups): up to 65 536 group ids, one of which must be the frame's group (its
    # set_groups id, else its frame id) -- VideoRAG's videoIDs as the roots of the chosen videos.  Empty: no group clause.
    groups: Tuple[int, ...] = ()
    # Root clause (wax_vs_search_batch_where_roots): the root-tag word of the frame's group (see set_root_tags) must hold
    # every bit of root_all_tags and none of root_no_tags -- PhotoRAG's and VideoRAG's test on each hit's root, e.g.
    # root_all_tags = IS_ROOT, root_no_tags = DELETED | SUPERSEDED.  (0, 0): no root clause.
    root_all_tags: int = 0
    root_no_tags: int = 0

    @property
    def has_root_clause(self) -> bool:
        return bool(self.root_all_tags or self.root_no_tags)

    def passes(self, timestamp: int, tags: int, location: Optional[Tuple[int, int]] = None,
               terms: Optional[Iterable[int]] = None, group: Optional[int] = None,
               root_tags: Optional[int] = None) -> bool:
        """The predicate on the host, as the device evaluates it; `location` is the frame's (latBin, lonBin) or None,
        `terms` its term set or None (no terms), `group` its group id (required when the where has a group clause),
        `root_tags` its group's root-tag word (required when the where has a root clause; 0 for a group never given
        one)."""
        if not (self.after <= timestamp and (timestamp < self.before or self.before == L.INT64_MAX)
                and (tags & self.all_tags) == self.all_tags and (tags & self.no_tags) == 0):
            return False
        if self.has_root_clause:
            if root_tags is None:
                raise ValueError("Where.passes: a where with a root clause needs the frame's group's root tags")
            if (int(root_tags) & self.root_all_tags) != self.root_all_tags or int(root_tags) & self.root_no_tags:
                return False
        if self.groups:
            if group is None:
                raise ValueError("Where.passes: a where with a group clause needs the frame's group")
            if int(group) not in set(int(g) for g in self.groups):
                return False
        if self.terms and not set(int(t) for t in self.terms) <= set(int(t) for t in (terms or ())):
            return False
        box = None if self.near is None else location_box(*self.near)
        if box is None:
            return True
        if location is None:
            return False
        lat_lo, lat_hi, lon_lo, lon_hi = box
        lat_bin, lon_bin = location
        lon_in = lon_lo <= lon_bin <= lon_hi if lon_lo <= lon_hi else (lon_lo <= lon_bin <= 18000 or -18000 <= lon_bin <= lon_hi)
        return lat_lo <= lat_bin <= lat_hi and lon_in

    def to_c(self) -> "L.Where":
        return L.Where(int(self.after), int(self.before), int(self.all_tags), int(self.no_tags))

    def to_c_near(self) -> "L.WhereNear":
        lat, lon, radius = self.near if self.near is not None else (0.0, 0.0, 0.0)
        return L.WhereNear(self.to_c(), float(lat), float(lon), float(radius))


class TermDictionary:
    """Wax's metadata as term ids (the frame side of set_terms, the query side of Where(terms=...)), by exact interning:
    ("entry", key, value) for meta.metadata.entries, ("tag", key, value) for meta.tags and ("label", s) for meta.labels
    each get the next id, so two different requirements never share one and the term clause is exactly
    UnifiedSearch.matches(metadataFilter:meta:).  A requirement no frame was ever given maps to UNKNOWN, an id the
    dictionary never assigns, which therefore matches no frame."""
    UNKNOWN = (1 << 64) - 1

    def __init__(self) -> None:
        self._ids: dict = {}
        self._lock = threading.Lock()

    def __len__(self) -> int:
        return len(self._ids)

    def intern(self, kind: str, *parts: str) -> int:
        """The id of ("entry", key, value), ("tag", key, value) or ("label", s), assigned on first sight."""
        if (kind, len(parts)) not in (("entry", 2), ("tag", 2), ("label", 1)):
            raise ValueError(f"TermDictionary: {kind!r} with {len(parts)} parts")
        key = (kind,) + tuple(str(p) for p in parts)
        with self._lock:
            return self._ids.setdefault(key, len(self._ids))

    def lookup(self, kind: str, *parts: str) -> int:
        """The id of an interned requirement, or UNKNOWN."""
        return self._ids.get((kind,) + tuple(str(p) for p in parts), self.UNKNOWN)

    def frame_terms(self, entries: Optional[dict] = None, tags: Iterable[Tuple[str, str]] = (),
                    labels: Iterable[str] = ()) -> List[int]:
        """A frame's term set: its metadata entries (None for a nil meta.metadata), TagPairs and labels."""
        out = [self.intern("entry", k, v) for k, v in (entries or {}).items()]
        out += [self.intern("tag", k, v) for k, v in tags]
        out += [self.intern("label", s) for s in labels]
        return out

    def filter_terms(self, required_entries: Optional[dict] = None, required_tags: Iterable[Tuple[str, str]] = (),
                     required_labels: Iterable[str] = ()) -> Tuple[int, ...]:
        """A MetadataFilter's requirements as the term ids a Where requires (duplicates kept once)."""
        ids = [self.lookup("entry", k, v) for k, v in (required_entries or {}).items()]
        ids += [self.lookup("tag", k, v) for k, v in required_tags]
        ids += [self.lookup("label", s) for s in required_labels]
        return tuple(sorted(set(ids)))


def location_box(latitude: float, longitude: float, radius_m: float) -> Optional[Tuple[int, int, int, int]]:
    """PhotoRAG's box of bins for a location query (wax_vs_location_box): (minLatBin, maxLatBin, minLonBin, maxLonBin),
    the lon bins wrapping as [minLonBin, 18000] and [-18000, maxLonBin] when minLonBin > maxLonBin, or None where
    buildLocationAllowlist returns nil (no location clause).  Raises WaxError where Swift's Int(_:) would trap."""
    box = (C.c_int32 * 4)()
    active = C.c_int32(0)
    _check(L.lib().wax_vs_location_box(float(latitude), float(longitude), float(radius_m), box, C.byref(active)))
    return tuple(int(x) for x in box) if active.value else None


def location_bin(latitude: float, longitude: float) -> Optional[Tuple[int, int]]:
    """A frame's (latBin, lonBin) as set_locations stores it (wax_vs_location_bin): locationBin(from:); None for a NaN
    pair (no location)."""
    out = (C.c_int32 * 2)()
    has = C.c_int32(0)
    _check(L.lib().wax_vs_location_bin(float(latitude), float(longitude), out, C.byref(has)))
    return (int(out[0]), int(out[1])) if has.value else None


class _WhereArgs:
    """The id filters and wheres of a batched where search as the C ABI takes them (the pointers stay valid while this
    object lives): filters[f] = ("allow" | "deny" | 0 | 1, ids), query_filter / query_where = per-query index or None."""

    def __init__(self, wheres, query_where, filters, query_filter, b: int):
        filters = list(filters or [])
        if query_filter is None:
            query_filter = [None] * b
        if len(query_where) != b or len(query_filter) != b:
            raise ValueError(f"query_where / query_filter need {b} entries")
        modes, lists = [], []
        for mode, fids in filters:
            modes.append({"allow": 0, "deny": 1}[mode] if isinstance(mode, str) else int(mode))
            lists.append(np.ascontiguousarray(fids, dtype=np.uint64).reshape(-1))
        self.offsets = np.zeros(len(lists) + 1, np.uint64)
        self.offsets[1:] = np.cumsum([x.size for x in lists], dtype=np.uint64) if lists else []
        self.fids = np.concatenate(lists) if lists else np.zeros(0, np.uint64)
        self.modes = np.asarray(modes, np.int32)
        self.qf = np.asarray([L.NO_FILTER if f is None else int(f) for f in query_filter], np.uint32)
        self.qw = np.asarray([L.NO_FILTER if w is None else int(w) for w in query_where], np.uint32)
        self.n_wheres = len(wheres)
        self.with_terms = any(len(w.terms) for w in wheres)     # wax_vs_search_batch_where_terms only when a term is asked
        self.with_groups = any(len(w.groups) for w in wheres)   # the _where_groups entries only when a group is asked
        self.with_roots = any(w.has_root_clause for w in wheres)   # the _where_roots entries only when a root clause is
        # ... _where_near only when a box is; the terms, groups and roots entries always take wax_vs_where_near
        self.near = self.with_terms or self.with_groups or self.with_roots or any(w.near is not None for w in wheres)
        self.warr_near = (L.WhereNear * max(len(wheres), 1))(*[w.to_c_near() for w in wheres])
        self.warr = self.warr_near if self.near else (L.Where * max(len(wheres), 1))(*[w.to_c() for w in wheres])
        self.toff = np.zeros(len(wheres) + 1, np.uint64)
        self.toff[1:] = np.cumsum([len(w.terms) for w in wheres], dtype=np.uint64) if wheres else []
        self.tflat = np.fromiter((int(t) for w in wheres for t in w.terms), dtype=np.uint64, count=int(self.toff[-1]))
        self.goff, self.gflat = group_offsets(wheres)
        self.roots = root_clauses(wheres)

    def filter_args(self):
        """frame_ids, filter_offsets, filter_modes, n_filters, query_filter."""
        return (self.fids.ctypes.data_as(C.POINTER(C.c_uint64)) if self.fids.size else None,
                self.offsets.ctypes.data_as(C.POINTER(C.c_uint64)), self.modes.ctypes.data_as(C.POINTER(C.c_int32)),
                self.modes.size, self.qf.ctypes.data_as(C.POINTER(C.c_uint32)))

    def where_args(self, near: bool = False):
        """wheres (wax_vs_where_near when the call needs them or `near`, else wax_vs_where), n_wheres, query_where."""
        return (C.cast(self.warr_near if near else self.warr, C.c_void_p), self.n_wheres,
                self.qw.ctypes.data_as(C.POINTER(C.c_uint32)))

    def term_args(self):
        """where_term_offsets, where_terms."""
        return (self.toff.ctypes.data_as(C.POINTER(C.c_uint64)),
                self.tflat.ctypes.data_as(C.POINTER(C.c_uint64)) if self.tflat.size else None)

    def group_args(self):
        """where_group_offsets, where_groups."""
        return (self.goff.ctypes.data_as(C.POINTER(C.c_uint64)),
                self.gflat.ctypes.data_as(C.POINTER(C.c_uint64)) if self.gflat.size else None)

    def root_args(self):
        """where_roots."""
        return (C.cast(self.roots, C.c_void_p),)


def group_offsets(wheres: Sequence["Where"]) -> Tuple[np.ndarray, np.ndarray]:
    """The group clauses of `wheres` as the C ABI takes them: offsets [len(wheres) + 1] from 0, where w's ids being
    ids[offsets[w]:offsets[w + 1]] in the order given (duplicates kept; the engine drops them)."""
    offsets = np.zeros(len(wheres) + 1, np.uint64)
    offsets[1:] = np.cumsum([len(w.groups) for w in wheres], dtype=np.uint64) if wheres else []
    ids = np.fromiter((int(g) for w in wheres for g in w.groups), dtype=np.uint64, count=int(offsets[-1]))
    return offsets, ids


def root_clauses(wheres: Sequence["Where"]) -> "C.Array":
    """The root clauses of `wheres` as the C ABI takes them: one wax_vs_root_clause per where ((0, 0): none)."""
    return (L.RootClause * max(len(wheres), 1))(*[L.RootClause(int(w.root_all_tags), int(w.root_no_tags)) for w in wheres])


# wax_vs_row_columns: one row's group, attributes and location bins, as wax_vs_export_columns / wax_vs_absorb_rows take them
ROW_COLUMNS_DTYPE = np.dtype([("group", "<u8"), ("timestamp", "<i8"), ("tags", "<u8"), ("lat_bin", "<i4"), ("lon_bin", "<i4")])
assert ROW_COLUMNS_DTYPE.itemsize == 32


class RowColumns(NamedTuple):
    """The side columns of a run of rows (CUDAVectorEngine.export_columns): `set` = the L.COLUMN_* bits of the columns the
    engine holds, `records` [n] ROW_COLUMNS_DTYPE, the term lists as `term_offsets` [n + 1] (from 0) into `terms`."""
    set: int
    records: np.ndarray
    term_offsets: np.ndarray
    terms: np.ndarray


def _clamp_topk(top_k: int) -> int:
    """clampTopK (MetalVectorEngine.swift:842-846)."""
    return max(1, min(int(top_k), L.MAX_RESULTS))


def _as_rows(vectors, dims: int) -> np.ndarray:
    rows = [np.asarray(v, dtype=np.float32).reshape(-1) for v in vectors] if not isinstance(vectors, np.ndarray) \
        else None
    if rows is not None:
        for v in rows:
            if v.size != dims:  # MetalVectorEngine.swift:367-370
                raise EncodingError(f"vector dimension mismatch: expected {dims}, got {v.size}")
        return np.ascontiguousarray(np.stack(rows) if rows else np.zeros((0, dims), np.float32))
    arr = np.ascontiguousarray(vectors, dtype=np.float32)
    if arr.ndim != 2 or arr.shape[1] != dims:
        got = arr.shape[1] if arr.ndim == 2 else arr.size
        raise EncodingError(f"vector dimension mismatch: expected {dims}, got {got}")
    return arr


class CUDAVectorEngine:
    """Drop-in for MetalVectorEngine / USearchVectorEngine behind `VectorSearchEngine`.

    Thread-safety mirrors the actor + AsyncReadWriteLock: searches may run concurrently, mutators are
    exclusive (enforced inside the library).
    """

    @staticmethod
    def is_available() -> bool:                      # MetalVectorEngine.isAvailable (:144-146)
        n = C.c_int32(0)
        return L.lib().wax_vs_device_count(C.byref(n)) == L.OK and n.value > 0

    def __init__(self, metric: VectorMetric = VectorMetric.cosine, dimensions: int = 0,
                 device: Optional[int] = None, devices: Optional[Sequence[int]] = None):   # init(metric:dimensions:) (:153)
        """`devices` with two or more ordinals makes a multi-device handle: the corpus sharded by rows, shard r on
        devices[r], every answer equal to one engine's (DESIGN.md section 4.16).  An ordinal may repeat: shards then
        share that device (a test and debug configuration)."""
        if dimensions <= 0:
            raise InvalidToc("dimensions must be > 0")
        if dimensions > L.MAX_DIMENSIONS:
            raise CapacityExceeded(f"capacity exceeded: limit {L.MAX_DIMENSIONS}, requested {dimensions}")
        if device is not None and devices is not None:
            raise ValueError("pass at most one of device= / devices=")
        self.metric = metric
        self.dimensions = int(dimensions)
        self._device = device if device is not None else (devices[0] if devices else None)
        self._dirty = False
        self._h = C.c_void_p()
        if device is not None:
            devices = [device]
        devs = (C.c_int32 * len(devices))(*devices) if devices else None
        _check(L.lib().wax_vs_create(self.dimensions, metric.to_vec_similarity(), devs,
                                     len(devices) if devices else 0, C.byref(self._h)))
        self._closed = False
        self._lock = threading.Lock()

    @classmethod
    def load(cls, wax, metric: VectorMetric, dimensions: int, device: Optional[int] = None) -> "CUDAVectorEngine":
        """`static load(from:metric:dimensions:)` (MetalVectorEngine.swift:318-328): the committed vector-index blob,
        then the pending (uncommitted) embedding mutations replayed in order as upserts.  `wax` needs
        `read_committed_vec_index_bytes() -> bytes | None` and `pending_embedding_mutations() -> [(frameId, vector)]`
        (objects with `.frame_id` / `.vector` are accepted too); the store behind them is out of scope (SURVEY section 8).
        The replay is ONE add_batch: the library resolves the rows sequentially, so a frameId that occurs twice keeps
        its last vector exactly as the reference's per-embedding loop does."""
        engine = cls(metric, dimensions, device)
        try:
            blob = wax.read_committed_vec_index_bytes()
            if blob is not None:
                engine.deserialize(blob)
            pending = list(wax.pending_embedding_mutations())
            if pending:
                ids = [int(getattr(m, "frame_id", m[0] if isinstance(m, (tuple, list)) else None)) for m in pending]
                vecs = [getattr(m, "vector", m[1] if isinstance(m, (tuple, list)) else None) for m in pending]
                engine.add_batch(ids, vecs)
        except Exception:
            engine.close()
            raise
        return engine

    # -- lifetime
    def close(self) -> None:
        if not getattr(self, "_closed", True):
            self._closed = True
            L.lib().wax_vs_destroy(self._h)

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()

    @property
    def handle(self) -> C.c_void_p:
        return self._h

    @property
    def count(self) -> int:
        n = C.c_uint64(0)
        _check(L.lib().wax_vs_count(self._h, C.byref(n)))
        return n.value

    # -- VectorSearchEngine protocol
    def search(self, vector: Sequence[float], top_k: int) -> List[Tuple[int, float]]:
        """search(vector:topK:) -> [(frameId, score)] best first."""
        q = np.ascontiguousarray(vector, dtype=np.float32).reshape(-1)
        # clamp(topK) entries, as the Swift mirror allocates: sizing from a separate count() call would race with a
        # concurrent add (the library would then need more room than `cap` and report ERR_BUFFER on a valid search)
        cap = _clamp_topk(top_k)
        ids = np.empty(cap, np.uint64)
        scores = np.empty(cap, np.float32)
        n = C.c_uint32(0)
        _check(L.lib().wax_vs_search(self._h, q.ctypes.data_as(C.POINTER(C.c_float)), q.size, int(top_k),
                                     ids.ctypes.data_as(C.POINTER(C.c_uint64)),
                                     scores.ctypes.data_as(C.POINTER(C.c_float)), cap, C.byref(n)))
        return [(int(ids[i]), float(scores[i])) for i in range(n.value)]

    def search_filtered(self, vector: Sequence[float], top_k: int, allow: Optional[Sequence[int]] = None,
                        deny: Optional[Sequence[int]] = None) -> List[Tuple[int, float]]:
        """Filter pushed below the top-k (API extension, SURVEY 8f-4): the best `top_k` rows among the frames in
        `allow` (allow-list) or among all frames except those in `deny` (deny-list).  Replaces the reference's
        post-hoc frame filter + 3 x topK over-fetch (UnifiedSearch.swift:58,1241-1258)."""
        if (allow is None) == (deny is None):
            raise ValueError("pass exactly one of allow= / deny=")
        ids = np.ascontiguousarray(allow if allow is not None else deny, dtype=np.uint64).reshape(-1)
        q = np.ascontiguousarray(vector, dtype=np.float32).reshape(-1)
        cap = _clamp_topk(top_k)
        out_ids = np.empty(cap, np.uint64)
        scores = np.empty(cap, np.float32)
        n = C.c_uint32(0)
        idp = ids.ctypes.data_as(C.POINTER(C.c_uint64)) if ids.size else None
        _check(L.lib().wax_vs_search_filtered(self._h, q.ctypes.data_as(C.POINTER(C.c_float)), q.size, int(top_k), idp,
                                              ids.size, 0 if allow is not None else 1,
                                              out_ids.ctypes.data_as(C.POINTER(C.c_uint64)),
                                              scores.ctypes.data_as(C.POINTER(C.c_float)), cap, C.byref(n)))
        return [(int(out_ids[i]), float(scores[i])) for i in range(n.value)]

    def search_batch_filtered(self, vectors, top_k: int, allow: Optional[Sequence[int]] = None,
                              deny: Optional[Sequence[int]] = None) -> List[List[Tuple[int, float]]]:
        """`search_filtered` for a batch of queries under ONE filter, in one pass over the corpus
        (wax_vs_search_batch_filtered); the same answers as calling search_filtered per query."""
        if (allow is None) == (deny is None):
            raise ValueError("pass exactly one of allow= / deny=")
        fids = np.ascontiguousarray(allow if allow is not None else deny, dtype=np.uint64).reshape(-1)
        qs = _as_rows(vectors, self.dimensions) if len(vectors) else np.zeros((0, self.dimensions), np.float32)
        b = qs.shape[0]
        if b == 0:
            return []
        cap = _clamp_topk(top_k)
        ids = np.zeros((b, cap), np.uint64)
        scores = np.zeros((b, cap), np.float32)
        ns = np.zeros(b, np.uint32)
        idp = fids.ctypes.data_as(C.POINTER(C.c_uint64)) if fids.size else None
        _check(L.lib().wax_vs_search_batch_filtered(self._h, qs.ctypes.data_as(C.POINTER(C.c_float)), b, qs.shape[1],
                                                    int(top_k), idp, fids.size, 0 if allow is not None else 1,
                                                    ids.ctypes.data_as(C.POINTER(C.c_uint64)),
                                                    scores.ctypes.data_as(C.POINTER(C.c_float)), cap,
                                                    ns.ctypes.data_as(C.POINTER(C.c_uint32))))
        return [[(int(ids[i, j]), float(scores[i, j])) for j in range(int(ns[i]))] for i in range(b)]

    def search_batch_multi_filtered(self, vectors, top_k: int, filters: Sequence[Tuple[object, Sequence[int]]],
                                    query_filter: Sequence[Optional[int]]) -> List[List[Tuple[int, float]]]:
        """A batch of queries with one filter PER QUERY (wax_vs_search_batch_multi_filtered): query i searches under
        filters[query_filter[i]], or unfiltered when that entry is None.  A filter is ("allow", ids) or ("deny", ids);
        the mode may also be given as 0 / 1.  Query i's answer equals search_filtered under its filter (search when
        unfiltered); the batch shares one pass over the corpus per group of filters that fits the bitset budget."""
        qs = _as_rows(vectors, self.dimensions) if len(vectors) else np.zeros((0, self.dimensions), np.float32)
        b = qs.shape[0]
        if len(query_filter) != b:
            raise ValueError(f"query_filter has {len(query_filter)} entries for {b} queries")
        if b == 0:
            return []
        modes, lists = [], []
        for mode, fids in filters:
            modes.append({"allow": 0, "deny": 1}[mode] if isinstance(mode, str) else int(mode))
            lists.append(np.ascontiguousarray(fids, dtype=np.uint64).reshape(-1))
        offsets = np.zeros(len(lists) + 1, np.uint64)
        offsets[1:] = np.cumsum([x.size for x in lists], dtype=np.uint64) if lists else []
        fids = np.concatenate(lists) if lists else np.zeros(0, np.uint64)
        modes_arr = np.asarray(modes, np.int32)
        qf = np.asarray([L.NO_FILTER if f is None else int(f) for f in query_filter], np.uint32)
        cap = _clamp_topk(top_k)
        ids = np.zeros((b, cap), np.uint64)
        scores = np.zeros((b, cap), np.float32)
        ns = np.zeros(b, np.uint32)
        _check(L.lib().wax_vs_search_batch_multi_filtered(
            self._h, qs.ctypes.data_as(C.POINTER(C.c_float)), b, qs.shape[1], int(top_k),
            fids.ctypes.data_as(C.POINTER(C.c_uint64)) if fids.size else None,
            offsets.ctypes.data_as(C.POINTER(C.c_uint64)), modes_arr.ctypes.data_as(C.POINTER(C.c_int32)), len(lists),
            qf.ctypes.data_as(C.POINTER(C.c_uint32)), ids.ctypes.data_as(C.POINTER(C.c_uint64)),
            scores.ctypes.data_as(C.POINTER(C.c_float)), cap, ns.ctypes.data_as(C.POINTER(C.c_uint32))))
        return [[(int(ids[i, j]), float(scores[i, j])) for j in range(int(ns[i]))] for i in range(b)]

    def set_groups(self, frame_ids: Sequence[int], group_ids: Sequence[int]) -> int:
        """Assign frames to groups (wax_vs_set_groups): frame_ids[i] -> group_ids[i], unknown frames ignored, a later
        entry for the same frame wins.  A frame never assigned is its own group (Wax's parentId ?? id).  Returns how
        many rows had their group written.  Groups are not serialized: re-apply them after deserialize()."""
        fids = np.ascontiguousarray(frame_ids, dtype=np.uint64).reshape(-1)
        gids = np.ascontiguousarray(group_ids, dtype=np.uint64).reshape(-1)
        if fids.size != gids.size:
            raise ValueError(f"set_groups: {fids.size} frame ids for {gids.size} group ids")
        if fids.size == 0:
            return 0
        n = C.c_uint64(0)
        _check(L.lib().wax_vs_set_groups(self._h, fids.ctypes.data_as(C.POINTER(C.c_uint64)),
                                         gids.ctypes.data_as(C.POINTER(C.c_uint64)), fids.size, C.byref(n)))
        return n.value

    def set_root_tags(self, group_ids: Sequence[int], tags: Sequence[int]) -> int:
        """Set groups' root-tag words (wax_vs_set_root_tags): upsert by group id, a later entry for the same id wins, and
        an id no frame carries yet is kept for the frames that take it.  A group never given one has the word 0.  The
        words are keyed by group, so adds, removes and set_groups leave them alone; they are not serialized: re-apply them
        after deserialize().  Returns the number of distinct group ids named."""
        gids = np.ascontiguousarray(group_ids, dtype=np.uint64).reshape(-1)
        words = np.ascontiguousarray(tags, dtype=np.uint64).reshape(-1)
        if gids.size != words.size:
            raise ValueError(f"set_root_tags: {gids.size} group ids for {words.size} tag words")
        if gids.size == 0:
            return 0
        n = C.c_uint64(0)
        _check(L.lib().wax_vs_set_root_tags(self._h, gids.ctypes.data_as(C.POINTER(C.c_uint64)),
                                            words.ctypes.data_as(C.POINTER(C.c_uint64)), gids.size, C.byref(n)))
        return n.value

    def search_grouped(self, vector: Sequence[float], top_groups: int, per_group: int = 1,
                       allow: Optional[Sequence[int]] = None,
                       deny: Optional[Sequence[int]] = None) -> List[Tuple[int, List[Tuple[int, float]]]]:
        """The best `per_group` frames of each of the `top_groups` best groups (wax_vs_search_grouped), exact:
        [(group_id, [(frame_id, score), ...]), ...], groups best first (a group ranks by its best frame), frames best
        first.  Optional frame filter as search_filtered (at most one of allow= / deny=).  Replaces the over-fetch +
        host grouping of PhotoRAG / VideoRAG (PhotoRAGOrchestrator.swift:244-308, VideoRAGOrchestrator.swift:252-440)."""
        if allow is not None and deny is not None:
            raise ValueError("pass at most one of allow= / deny=")
        fids = np.ascontiguousarray(allow if allow is not None else (deny if deny is not None else []),
                                    dtype=np.uint64).reshape(-1)
        mode = 0 if allow is not None else 1
        q = np.ascontiguousarray(vector, dtype=np.float32).reshape(-1)
        cap = max(1, min(_clamp_topk(top_groups) * max(int(per_group), 1), L.MAX_RESULTS))
        ids = np.empty(cap, np.uint64)
        scores = np.empty(cap, np.float32)
        groups = np.empty(cap, np.uint64)
        n = C.c_uint32(0)
        _check(L.lib().wax_vs_search_grouped(self._h, q.ctypes.data_as(C.POINTER(C.c_float)), q.size, int(top_groups),
                                             int(per_group), fids.ctypes.data_as(C.POINTER(C.c_uint64)) if fids.size
                                             else None, fids.size, mode, ids.ctypes.data_as(C.POINTER(C.c_uint64)),
                                             scores.ctypes.data_as(C.POINTER(C.c_float)),
                                             groups.ctypes.data_as(C.POINTER(C.c_uint64)), cap, C.byref(n)))
        out: List[Tuple[int, List[Tuple[int, float]]]] = []
        for i in range(n.value):
            g = int(groups[i])
            if not out or out[-1][0] != g:
                out.append((g, []))
            out[-1][1].append((int(ids[i]), float(scores[i])))
        return out

    def search_batch_grouped(self, vectors, top_groups: int, per_group: int = 1,
                             allow: Optional[Sequence[int]] = None,
                             deny: Optional[Sequence[int]] = None) -> List[List[Tuple[int, List[Tuple[int, float]]]]]:
        """`search_grouped` for a batch of queries under ONE optional filter (wax_vs_search_batch_grouped): one
        [(group_id, [(frame_id, score), ...]), ...] per query, each identical to search_grouped for that query alone.
        The batch shares one tensor-core pass for its queries' top rows; crowded queries run the single-query path."""
        if allow is not None and deny is not None:
            raise ValueError("pass at most one of allow= / deny=")
        fids = np.ascontiguousarray(allow if allow is not None else (deny if deny is not None else []),
                                    dtype=np.uint64).reshape(-1)
        mode = 0 if allow is not None else 1
        qs = _as_rows(vectors, self.dimensions) if len(vectors) else np.zeros((0, self.dimensions), np.float32)
        b = qs.shape[0]
        if b == 0:
            return []
        cap = max(1, min(_clamp_topk(top_groups) * max(int(per_group), 1), L.MAX_RESULTS))
        ids = np.empty((b, cap), np.uint64)
        scores = np.empty((b, cap), np.float32)
        groups = np.empty((b, cap), np.uint64)
        ns = np.zeros(b, np.uint32)
        _check(L.lib().wax_vs_search_batch_grouped(self._h, qs.ctypes.data_as(C.POINTER(C.c_float)), b, qs.shape[1],
                                                   int(top_groups), int(per_group),
                                                   fids.ctypes.data_as(C.POINTER(C.c_uint64)) if fids.size else None,
                                                   fids.size, mode, ids.ctypes.data_as(C.POINTER(C.c_uint64)),
                                                   scores.ctypes.data_as(C.POINTER(C.c_float)),
                                                   groups.ctypes.data_as(C.POINTER(C.c_uint64)), cap,
                                                   ns.ctypes.data_as(C.POINTER(C.c_uint32))))
        result = []
        for i in range(b):
            out: List[Tuple[int, List[Tuple[int, float]]]] = []
            for j in range(int(ns[i])):
                g = int(groups[i, j])
                if not out or out[-1][0] != g:
                    out.append((g, []))
                out[-1][1].append((int(ids[i, j]), float(scores[i, j])))
            result.append(out)
        return result

    # -- frame attributes: time-range and tag predicates below the top-k
    def set_attributes(self, frame_ids: Sequence[int], timestamps: Optional[Sequence[int]] = None,
                       tags: Optional[Sequence[int]] = None) -> int:
        """Set frames' timestamp and tag mask (wax_vs_set_attributes): upsert by frame id, unknown frames ignored, a later
        entry for the same frame wins; a column passed as None is left unchanged.  A frame never given attributes has
        timestamp 0 and tags 0.  Attributes are not serialized: re-apply them after deserialize().  Returns the number of
        distinct known frames named."""
        fids = np.ascontiguousarray(frame_ids, dtype=np.uint64).reshape(-1)
        ts = None if timestamps is None else np.ascontiguousarray(timestamps, dtype=np.int64).reshape(-1)
        tg = None if tags is None else np.ascontiguousarray(tags, dtype=np.uint64).reshape(-1)
        for name, col in (("timestamps", ts), ("tags", tg)):
            if col is not None and col.size != fids.size:
                raise ValueError(f"set_attributes: {fids.size} frame ids for {col.size} {name}")
        if fids.size == 0:
            return 0
        n = C.c_uint64(0)
        _check(L.lib().wax_vs_set_attributes(
            self._h, fids.ctypes.data_as(C.POINTER(C.c_uint64)),
            ts.ctypes.data_as(C.POINTER(C.c_int64)) if ts is not None else None,
            tg.ctypes.data_as(C.POINTER(C.c_uint64)) if tg is not None else None, fids.size, C.byref(n)))
        return n.value

    def set_locations(self, frame_ids: Sequence[int], latitudes: Sequence[float], longitudes: Sequence[float]) -> int:
        """Set frames' locations in degrees (wax_vs_set_locations): upsert by frame id, unknown frames ignored, a later
        entry for the same frame wins, a NaN pair clears a location.  A frame never given one has none and passes no
        location clause.  Locations are not serialized: re-apply them after deserialize().  Returns the number of
        distinct known frames named."""
        fids = np.ascontiguousarray(frame_ids, dtype=np.uint64).reshape(-1)
        lat = np.ascontiguousarray(latitudes, dtype=np.float64).reshape(-1)
        lon = np.ascontiguousarray(longitudes, dtype=np.float64).reshape(-1)
        if lat.size != fids.size or lon.size != fids.size:
            raise ValueError(f"set_locations: {fids.size} frame ids for {lat.size} latitudes and {lon.size} longitudes")
        if fids.size == 0:
            return 0
        n = C.c_uint64(0)
        _check(L.lib().wax_vs_set_locations(
            self._h, fids.ctypes.data_as(C.POINTER(C.c_uint64)), lat.ctypes.data_as(C.POINTER(C.c_double)),
            lon.ctypes.data_as(C.POINTER(C.c_double)), fids.size, C.byref(n)))
        return n.value

    location_box = staticmethod(location_box)

    def set_terms(self, frame_ids: Sequence[int], term_lists: Sequence[Sequence[int]]) -> int:
        """Replace frames' term sets (wax_vs_set_terms): upsert by frame id, unknown frames ignored, a later entry for the
        same frame wins, duplicate ids kept once, an empty list clears the set.  A frame never given terms has none and
        passes no non-empty term clause.  Terms are not serialized: re-apply them after deserialize().  Returns the
        number of distinct known frames named."""
        fids = np.ascontiguousarray(frame_ids, dtype=np.uint64).reshape(-1)
        if len(term_lists) != fids.size:
            raise ValueError(f"set_terms: {fids.size} frame ids for {len(term_lists)} term lists")
        offsets = np.zeros(fids.size + 1, np.uint64)
        offsets[1:] = np.cumsum([len(t) for t in term_lists], dtype=np.uint64) if fids.size else []
        flat = np.fromiter((int(x) for t in term_lists for x in t), dtype=np.uint64, count=int(offsets[-1]))
        n = C.c_uint64(0)
        _check(L.lib().wax_vs_set_terms(
            self._h, fids.ctypes.data_as(C.POINTER(C.c_uint64)) if fids.size else None,
            offsets.ctypes.data_as(C.POINTER(C.c_uint64)), flat.ctypes.data_as(C.POINTER(C.c_uint64)) if flat.size else None,
            fids.size, C.byref(n)))
        return n.value

    def search_where(self, vector: Sequence[float], top_k: int, where: "Where", allow: Optional[Sequence[int]] = None,
                     deny: Optional[Sequence[int]] = None) -> List[Tuple[int, float]]:
        """The best `top_k` frames passing `where` (and the optional id filter allow= / deny=): the batch of one of
        search_batch_where."""
        if allow is not None and deny is not None:
            raise ValueError("pass at most one of allow= / deny=")
        filters = [("allow", allow)] if allow is not None else ([("deny", deny)] if deny is not None else [])
        return self.search_batch_where([vector], top_k, [where], [0], filters, [0 if filters else None])[0]

    def search_batch_where(self, vectors, top_k: int, wheres: Sequence["Where"], query_where: Sequence[Optional[int]],
                           filters: Optional[Sequence[Tuple[object, Sequence[int]]]] = None,
                           query_filter: Optional[Sequence[Optional[int]]] = None) -> List[List[Tuple[int, float]]]:
        """search_batch_multi_filtered plus a predicate per query (wax_vs_search_batch_where): query i searches the frames
        passing wheres[query_where[i]] AND filters[query_filter[i]] (None = no predicate / no id filter).  Its answer
        equals search_batch_multi_filtered with an allow-list of exactly those frames, score bits included."""
        qs = _as_rows(vectors, self.dimensions) if len(vectors) else np.zeros((0, self.dimensions), np.float32)
        b = qs.shape[0]
        a = _WhereArgs(wheres, query_where, filters, query_filter, b)
        if b == 0:
            return []
        cap = _clamp_topk(top_k)
        ids = np.zeros((b, cap), np.uint64)
        scores = np.zeros((b, cap), np.float32)
        ns = np.zeros(b, np.uint32)
        head = (self._h, qs.ctypes.data_as(C.POINTER(C.c_float)), b, qs.shape[1], int(top_k), *a.filter_args(),
                *a.where_args())
        tail = (ids.ctypes.data_as(C.POINTER(C.c_uint64)), scores.ctypes.data_as(C.POINTER(C.c_float)), cap,
                ns.ctypes.data_as(C.POINTER(C.c_uint32)))
        if a.with_roots:
            terms = a.term_args() if a.with_terms else (None, None)
            _check(L.lib().wax_vs_search_batch_where_roots(*head, *terms, *a.group_args(), *a.root_args(), *tail))
        elif a.with_groups:
            terms = a.term_args() if a.with_terms else (None, None)
            _check(L.lib().wax_vs_search_batch_where_groups(*head, *terms, *a.group_args(), *tail))
        elif a.with_terms:
            _check(L.lib().wax_vs_search_batch_where_terms(*head, *a.term_args(), *tail))
        else:
            entry = L.lib().wax_vs_search_batch_where_near if a.near else L.lib().wax_vs_search_batch_where
            _check(entry(*head, *tail))
        return [[(int(ids[i, j]), float(scores[i, j])) for j in range(int(ns[i]))] for i in range(b)]

    def search_batch_grouped_where(self, vectors, top_groups: int, per_group: int, where: "Where",
                                   allow: Optional[Sequence[int]] = None,
                                   deny: Optional[Sequence[int]] = None) -> List[List[Tuple[int, List[Tuple[int, float]]]]]:
        """search_batch_grouped over the frames passing `where` AND the optional id filter
        (wax_vs_search_batch_grouped_where); each answer equals search_grouped under the allow-list of those frames."""
        if allow is not None and deny is not None:
            raise ValueError("pass at most one of allow= / deny=")
        if where.terms:
            raise ValueError("grouped search takes no term clause")
        fids = np.ascontiguousarray(allow if allow is not None else (deny if deny is not None else []),
                                    dtype=np.uint64).reshape(-1)
        mode = 0 if allow is not None else 1
        qs = _as_rows(vectors, self.dimensions) if len(vectors) else np.zeros((0, self.dimensions), np.float32)
        b = qs.shape[0]
        if where.groups or where.has_root_clause:   # one where and one id filter for every query (an empty deny-list is none)
            filters = [] if allow is None and deny is None else [(mode, fids)]
            one = None if not filters or (mode == 1 and fids.size == 0) else 0
            return self.search_batch_grouped_multi_where(qs, top_groups, per_group, [where], [0] * b, filters, [one] * b)
        if b == 0:
            return []
        cap = max(1, min(_clamp_topk(top_groups) * max(int(per_group), 1), L.MAX_RESULTS))
        ids = np.empty((b, cap), np.uint64)
        scores = np.empty((b, cap), np.float32)
        groups = np.empty((b, cap), np.uint64)
        ns = np.zeros(b, np.uint32)
        w = where.to_c() if where.near is None else where.to_c_near()
        entry = L.lib().wax_vs_search_batch_grouped_where if where.near is None else \
            L.lib().wax_vs_search_batch_grouped_where_near
        _check(entry(
            self._h, qs.ctypes.data_as(C.POINTER(C.c_float)), b, qs.shape[1], int(top_groups), int(per_group),
            fids.ctypes.data_as(C.POINTER(C.c_uint64)) if fids.size else None, fids.size, mode,
            C.cast(C.pointer(w), C.c_void_p), ids.ctypes.data_as(C.POINTER(C.c_uint64)),
            scores.ctypes.data_as(C.POINTER(C.c_float)), groups.ctypes.data_as(C.POINTER(C.c_uint64)), cap,
            ns.ctypes.data_as(C.POINTER(C.c_uint32))))
        result = []
        for i in range(b):
            out: List[Tuple[int, List[Tuple[int, float]]]] = []
            for j in range(int(ns[i])):
                g = int(groups[i, j])
                if not out or out[-1][0] != g:
                    out.append((g, []))
                out[-1][1].append((int(ids[i, j]), float(scores[i, j])))
            result.append(out)
        return result

    def search_batch_grouped_multi_where(self, vectors, top_groups: int, per_group: int, wheres: Sequence["Where"],
                                         query_where: Sequence[Optional[int]],
                                         filters: Optional[Sequence[Tuple[object, Sequence[int]]]] = None,
                                         query_filter: Optional[Sequence[Optional[int]]] = None
                                         ) -> List[List[Tuple[int, List[Tuple[int, float]]]]]:
        """search_batch_grouped with a where and an id filter of each query's own
        (wax_vs_search_batch_grouped_multi_where): query i searches the frames passing wheres[query_where[i]] AND
        filters[query_filter[i]] (None = no predicate / no id filter; arguments as search_batch_where).  Its answer, one
        [(group_id, [(frame_id, score), ...]), ...], equals search_grouped under an allow-list of exactly those frames."""
        if any(w.terms for w in wheres):
            raise ValueError("grouped search takes no term clause")
        qs = _as_rows(vectors, self.dimensions) if len(vectors) else np.zeros((0, self.dimensions), np.float32)
        b = qs.shape[0]
        filters = list(filters or [])
        if query_filter is None:
            query_filter = [None] * b
        if len(query_where) != b or len(query_filter) != b:
            raise ValueError(f"query_where / query_filter need {b} entries")
        if b == 0:
            return []
        modes, lists = [], []
        for mode, fids in filters:
            modes.append({"allow": 0, "deny": 1}[mode] if isinstance(mode, str) else int(mode))
            lists.append(np.ascontiguousarray(fids, dtype=np.uint64).reshape(-1))
        offsets = np.zeros(len(lists) + 1, np.uint64)
        offsets[1:] = np.cumsum([x.size for x in lists], dtype=np.uint64) if lists else []
        fids = np.concatenate(lists) if lists else np.zeros(0, np.uint64)
        modes_arr = np.asarray(modes, np.int32)
        qf = np.asarray([L.NO_FILTER if f is None else int(f) for f in query_filter], np.uint32)
        qw = np.asarray([L.NO_FILTER if w is None else int(w) for w in query_where], np.uint32)
        warr = (L.WhereNear * max(len(wheres), 1))(*[w.to_c_near() for w in wheres])
        cap = max(1, min(_clamp_topk(top_groups) * max(int(per_group), 1), L.MAX_RESULTS))
        ids = np.empty((b, cap), np.uint64)
        scores = np.empty((b, cap), np.float32)
        groups = np.empty((b, cap), np.uint64)
        ns = np.zeros(b, np.uint32)
        head = (self._h, qs.ctypes.data_as(C.POINTER(C.c_float)), b, qs.shape[1], int(top_groups), int(per_group),
                fids.ctypes.data_as(C.POINTER(C.c_uint64)) if fids.size else None,
                offsets.ctypes.data_as(C.POINTER(C.c_uint64)), modes_arr.ctypes.data_as(C.POINTER(C.c_int32)), len(lists),
                qf.ctypes.data_as(C.POINTER(C.c_uint32)), C.cast(warr, C.c_void_p), len(wheres),
                qw.ctypes.data_as(C.POINTER(C.c_uint32)))
        tail = (ids.ctypes.data_as(C.POINTER(C.c_uint64)), scores.ctypes.data_as(C.POINTER(C.c_float)),
                groups.ctypes.data_as(C.POINTER(C.c_uint64)), cap, ns.ctypes.data_as(C.POINTER(C.c_uint32)))
        goff, gflat = group_offsets(wheres)
        group_args = (goff.ctypes.data_as(C.POINTER(C.c_uint64)),
                      gflat.ctypes.data_as(C.POINTER(C.c_uint64)) if gflat.size else None)
        if any(w.has_root_clause for w in wheres):   # the _roots entry only when a root clause is asked
            roots = root_clauses(wheres)
            _check(L.lib().wax_vs_search_batch_grouped_multi_where_roots(*head, *group_args, C.cast(roots, C.c_void_p),
                                                                         *tail))
        elif any(w.groups for w in wheres):   # wax_vs_search_batch_grouped_multi_where_groups only when a group is asked
            _check(L.lib().wax_vs_search_batch_grouped_multi_where_groups(*head, *group_args, *tail))
        else:
            _check(L.lib().wax_vs_search_batch_grouped_multi_where(*head, *tail))
        result = []
        for i in range(b):
            out: List[Tuple[int, List[Tuple[int, float]]]] = []
            for j in range(int(ns[i])):
                g = int(groups[i, j])
                if not out or out[-1][0] != g:
                    out.append((g, []))
                out[-1][1].append((int(ids[i, j]), float(scores[i, j])))
            result.append(out)
        return result

    def search_batch(self, vectors, top_k: int) -> List[List[Tuple[int, float]]]:
        """`search` for a batch of queries (wax_vs_search_batch): the same answers as one call per query.  Cosine and dot
        batches share one tensor-core pass over the corpus, l2 batches too once set_option("batch_l2", 1) is set."""
        ids, scores, ns = self.search_batch_arrays(vectors, top_k)
        return [[(int(ids[i, j]), float(scores[i, j])) for j in range(int(ns[i]))] for i in range(ids.shape[0])]

    def search_batch_arrays(self, vectors, top_k: int):
        """Batched search returning arrays: (ids u64 [B, k_eff], scores f32 [B, k_eff], counts u32 [B]); row i holds
        counts[i] results, best first.  The list-of-tuples form above costs more host time than the GPU pass."""
        qs = _as_rows(vectors, self.dimensions) if len(vectors) else np.zeros((0, self.dimensions), np.float32)
        b = qs.shape[0]
        if b == 0:
            return np.zeros((0, 0), np.uint64), np.zeros((0, 0), np.float32), np.zeros(0, np.uint32)
        # b x min(clamp(topK), count) entries; a concurrent add can grow the count between the two calls, in which
        # case the library answers ERR_BUFFER and the buffers are re-sized (clamp(topK) always suffices)
        cap = max(1, min(_clamp_topk(top_k), max(self.count, 1)))
        for attempt in range(3):
            ids = np.zeros((b, cap), np.uint64)
            scores = np.zeros((b, cap), np.float32)
            ns = np.zeros(b, np.uint32)
            rc = L.lib().wax_vs_search_batch(self._h, qs.ctypes.data_as(C.POINTER(C.c_float)), b, qs.shape[1],
                                             int(top_k), ids.ctypes.data_as(C.POINTER(C.c_uint64)),
                                             scores.ctypes.data_as(C.POINTER(C.c_float)), cap,
                                             ns.ctypes.data_as(C.POINTER(C.c_uint32)))
            if rc != L.ERR_BUFFER:
                break
            cap = _clamp_topk(top_k) if attempt else max(1, min(_clamp_topk(top_k), max(self.count, 1)))
        _check(rc)
        return ids, scores, ns

    def add(self, frame_id: int, vector: Sequence[float]) -> None:
        v = np.ascontiguousarray(vector, dtype=np.float32).reshape(-1)
        _check(L.lib().wax_vs_add(self._h, int(frame_id), v.ctypes.data_as(C.POINTER(C.c_float)), v.size))
        self._dirty = True

    def add_batch(self, frame_ids: Sequence[int], vectors) -> None:
        ids = np.ascontiguousarray(frame_ids, dtype=np.uint64).reshape(-1)
        if ids.size == 0:                         # guard !frameIds.isEmpty (:360)
            return
        if ids.size != len(vectors):              # :361-363
            raise EncodingError("addBatch: frameIds.count != vectors.count")
        rows = _as_rows(vectors, self.dimensions)
        _check(L.lib().wax_vs_add_batch(self._h, ids.ctypes.data_as(C.POINTER(C.c_uint64)),
                                        rows.ctypes.data_as(C.POINTER(C.c_float)), ids.size, rows.shape[1]))
        self._dirty = True

    def add_batch_streaming(self, frame_ids: Sequence[int], vectors, chunk_size: int = 256) -> None:
        """addBatchStreaming (:404-421)."""
        if len(frame_ids) == 0:
            return
        if len(frame_ids) != len(vectors):
            raise EncodingError("addBatchStreaming: frameIds.count != vectors.count")
        if len(frame_ids) <= chunk_size:
            return self.add_batch(frame_ids, vectors)
        for start in range(0, len(frame_ids), chunk_size):
            self.add_batch(frame_ids[start:start + chunk_size], vectors[start:start + chunk_size])

    def remove(self, frame_id: int) -> None:
        before = self.count
        _check(L.lib().wax_vs_remove(self._h, int(frame_id)))
        if self.count != before:
            self._dirty = True

    def remove_batch(self, frame_ids: Sequence[int]) -> int:
        """remove(frameId:) for many frames in one pass (one compaction, one hash rebuild); returns how many rows went.
        Same result as calling remove() for each id."""
        ids = np.ascontiguousarray(frame_ids, dtype=np.uint64).reshape(-1)
        if ids.size == 0:
            return 0
        gone = C.c_uint64(0)
        _check(L.lib().wax_vs_remove_batch(self._h, ids.ctypes.data_as(C.POINTER(C.c_uint64)), ids.size, C.byref(gone)))
        if gone.value:
            self._dirty = True
        return gone.value

    def rebalance(self) -> int:
        """Even out the rows of a multi-device handle's shards in place (wax_vs_rebalance); returns how many rows moved.
        Every answer stays the same, groups, attributes, locations and terms included.  0 on one engine."""
        moved = C.c_uint64(0)
        _check(L.lib().wax_vs_rebalance(self._h, C.byref(moved)))
        return moved.value

    def reserve(self, rows: int) -> None:
        _check(L.lib().wax_vs_reserve(self._h, int(rows)))

    # -- row keys: the rank-local store of the row-sharded engine (DESIGN.md section 4.15)
    def add_batch_keyed(self, frame_ids: Sequence[int], vectors, first_key: int) -> int:
        """add_batch whose appended rows take the keys first_key, first_key + 1, ... (wax_vs_add_batch_keyed); returns how
        many rows it appended.  A first_key not above the last row's key raises WaxError."""
        ids = np.ascontiguousarray(frame_ids, dtype=np.uint64).reshape(-1)
        if ids.size == 0:
            return 0
        if ids.size != len(vectors):
            raise EncodingError("addBatch: frameIds.count != vectors.count")
        rows = _as_rows(vectors, self.dimensions)
        appended = C.c_uint64(0)
        _check(L.lib().wax_vs_add_batch_keyed(self._h, ids.ctypes.data_as(C.POINTER(C.c_uint64)),
                                              rows.ctypes.data_as(C.POINTER(C.c_float)), ids.size, rows.shape[1],
                                              int(first_key), C.byref(appended)))
        self._dirty = True
        return appended.value

    def contains(self, frame_ids: Sequence[int]) -> np.ndarray:
        """[n] bool: whether this engine holds each frame id."""
        ids = np.ascontiguousarray(frame_ids, dtype=np.uint64).reshape(-1)
        out = np.zeros(ids.size, np.uint8)
        if ids.size:
            _check(L.lib().wax_vs_contains(self._h, ids.ctypes.data_as(C.POINTER(C.c_uint64)), ids.size,
                                           out.ctypes.data_as(C.POINTER(C.c_uint8))))
        return out.astype(bool)

    def deserialize_rows(self, data: bytes, first: int, n: int) -> None:
        """Replace the contents with rows [first, first + n) of an MV2V blob, keyed first, first + 1, ...
        (wax_vs_deserialize_rows: the blob is checked as deserialize() checks it)."""
        buf = np.frombuffer(data, np.uint8)
        ptr = buf.ctypes.data_as(C.POINTER(C.c_uint8)) if buf.size else C.cast(C.c_char_p(b""), C.POINTER(C.c_uint8))
        _check(L.lib().wax_vs_deserialize_rows(self._h, ptr, buf.size, int(first), int(n)))
        self._dirty = False

    def export_rows(self, first: int, n: int, vectors: bool = True):
        """Rows [first, first + n): (frame ids uint64 [n], vectors float32 [n, dims] or None, keys uint64 [n])."""
        ids, keys = np.empty(n, np.uint64), np.empty(n, np.uint64)
        vecs = np.empty((n, self.dimensions), np.float32) if vectors else None
        _check(L.lib().wax_vs_export_rows(self._h, int(first), int(n), ids.ctypes.data_as(C.POINTER(C.c_uint64)),
                                          vecs.ctypes.data_as(C.POINTER(C.c_float)) if vectors else None,
                                          keys.ctypes.data_as(C.POINTER(C.c_uint64))))
        return ids, vecs, keys

    def export_vectors(self, first: int, n: int):
        """Rows [first, first + n)'s vectors as a new [n, dims] float32 torch tensor on the engine's device, copied device
        to device on that device's current stream (wax_vs_export_rows_device)."""
        import torch
        dev = torch.device("cuda", torch.cuda.current_device() if self._device is None else self._device)
        out = torch.empty((int(n), self.dimensions), dtype=torch.float32, device=dev)
        _check(L.lib().wax_vs_export_rows_device(self._h, int(first), int(n), C.c_void_p(out.data_ptr()),
                                                 C.c_void_p(torch.cuda.current_stream(dev).cuda_stream)))
        return out

    def export_columns(self, first: int, n: int) -> RowColumns:
        """The side columns of rows [first, first + n) (wax_vs_export_columns): a column the engine does not hold comes
        as the defaults its rows answer with (group = own frame id, attributes 0, no location, no terms)."""
        records = np.empty(int(n), ROW_COLUMNS_DTYPE)
        offsets = np.empty(int(n) + 1, np.uint64)
        length, bits = C.c_uint64(0), C.c_uint32(0)
        _check(L.lib().wax_vs_export_columns(self._h, int(first), int(n), None, None, None, 0, C.byref(length), None))
        terms = np.empty(length.value, np.uint64)
        _check(L.lib().wax_vs_export_columns(self._h, int(first), int(n), records.ctypes.data_as(C.c_void_p),
                                             offsets.ctypes.data_as(C.POINTER(C.c_uint64)),
                                             terms.ctypes.data_as(C.POINTER(C.c_uint64)), terms.size, C.byref(length),
                                             C.byref(bits)))
        return RowColumns(bits.value, records, offsets, terms)

    def absorb_rows(self, frame_ids: Sequence[int], keys: Sequence[int], vectors, columns: Optional[RowColumns] = None) -> None:
        """Merge rows into this engine by key (wax_vs_absorb_rows): frame ids, keys (strictly increasing), `vectors` a
        [n, dims] float32 torch tensor on the engine's device, and the side columns export_columns gave (None: the source
        held none).  The current stream of that device is synchronised first, so the vectors are complete."""
        import torch
        ids = np.ascontiguousarray(frame_ids, dtype=np.uint64).reshape(-1)
        ks = np.ascontiguousarray(keys, dtype=np.uint64).reshape(-1)
        if ids.size != ks.size or tuple(vectors.shape) != (ids.size, self.dimensions) or vectors.dtype != torch.float32:
            raise ValueError(f"absorb_rows: {ids.size} ids, {ks.size} keys and vectors of shape {tuple(vectors.shape)} "
                             f"({vectors.dtype})")
        vecs = vectors.contiguous()
        if vecs.is_cuda:
            torch.cuda.current_stream(vecs.device).synchronize()
        bits = 0 if columns is None else int(columns.set)
        recs = None if columns is None else np.ascontiguousarray(columns.records, ROW_COLUMNS_DTYPE)
        offs = None if columns is None else np.ascontiguousarray(columns.term_offsets, np.uint64)
        terms = None if columns is None else np.ascontiguousarray(columns.terms, np.uint64)
        _check(L.lib().wax_vs_absorb_rows(
            self._h, ids.ctypes.data_as(C.POINTER(C.c_uint64)), ks.ctypes.data_as(C.POINTER(C.c_uint64)),
            C.c_void_p(vecs.data_ptr()), ids.size, bits, recs.ctypes.data_as(C.c_void_p) if recs is not None else None,
            offs.ctypes.data_as(C.POINTER(C.c_uint64)) if offs is not None else None,
            terms.ctypes.data_as(C.POINTER(C.c_uint64)) if terms is not None and terms.size else None))
        if ids.size:
            self._dirty = True

    def row_keys(self) -> np.ndarray:
        """Every row's key, in row order (the row itself on an engine without keys)."""
        return self.export_rows(0, self.count, vectors=False)[2]

    # -- row-sharded search (wax_vs_shard_*; no reference counterpart, SURVEY.md section 8e) ------------------------------
    def shard_open(self, rank: int, world: int, row_offset: int) -> bytes:
        """Become rank `rank` of `world`: allocates this engine's mailbox and returns the handle blob the other ranks
        need to reach it."""
        blob = (C.c_uint8 * L.SHARD_HANDLE_BYTES)()
        _check(L.lib().wax_vs_shard_open(self._h, int(rank), int(world), int(row_offset), blob))
        return bytes(blob)

    def shard_connect(self, blobs: Sequence[bytes]) -> None:
        """Map every rank's mailbox (`blobs` in rank order, this rank's own included)."""
        flat = b"".join(blobs)
        buf = (C.c_uint8 * len(flat)).from_buffer_copy(flat)
        _check(L.lib().wax_vs_shard_connect(self._h, buf, len(blobs)))

    def shard_close(self) -> None:
        _check(L.lib().wax_vs_shard_close(self._h))

    def shard_search(self, vector: Sequence[float], top_k: int) -> List[Tuple[int, float]]:
        """COLLECTIVE search over the whole sharded corpus (every rank calls it with the same query): scan + NVLink
        exchange + merge in one kernel launch, merged result delivered into host memory."""
        q = np.ascontiguousarray(vector, dtype=np.float32).reshape(-1)
        cap = _clamp_topk(top_k)
        ids = np.empty(cap, np.uint64)
        scores = np.empty(cap, np.float32)
        n = C.c_uint32(0)
        _check(L.lib().wax_vs_shard_search(self._h, q.ctypes.data_as(C.POINTER(C.c_float)), q.size, int(top_k),
                                           ids.ctypes.data_as(C.POINTER(C.c_uint64)),
                                           scores.ctypes.data_as(C.POINTER(C.c_float)), cap, C.byref(n)))
        return [(int(ids[i]), float(scores[i])) for i in range(n.value)]

    def shard_search_filtered(self, vector: Sequence[float], top_k: int, allow: Optional[Sequence[int]] = None,
                              deny: Optional[Sequence[int]] = None) -> List[Tuple[int, float]]:
        """COLLECTIVE filtered search (every rank passes the same query and the same ids): each rank's fused scan
        applies the filter to the rows of its own shard, the in-kernel exchange merges -- one launch per rank."""
        if (allow is None) == (deny is None):
            raise ValueError("pass exactly one of allow= / deny=")
        fids = np.ascontiguousarray(allow if allow is not None else deny, dtype=np.uint64).reshape(-1)
        q = np.ascontiguousarray(vector, dtype=np.float32).reshape(-1)
        cap = _clamp_topk(top_k)
        ids = np.empty(cap, np.uint64)
        scores = np.empty(cap, np.float32)
        n = C.c_uint32(0)
        idp = fids.ctypes.data_as(C.POINTER(C.c_uint64)) if fids.size else None
        _check(L.lib().wax_vs_shard_search_filtered(self._h, q.ctypes.data_as(C.POINTER(C.c_float)), q.size, int(top_k),
                                                    idp, fids.size, 0 if allow is not None else 1,
                                                    ids.ctypes.data_as(C.POINTER(C.c_uint64)),
                                                    scores.ctypes.data_as(C.POINTER(C.c_float)), cap, C.byref(n)))
        return [(int(ids[i]), float(scores[i])) for i in range(n.value)]

    def shard_search_where(self, vector: Sequence[float], top_k: int, where: "Where", allow: Optional[Sequence[int]] = None,
                           deny: Optional[Sequence[int]] = None) -> List[Tuple[int, float]]:
        """COLLECTIVE where search (wax_vs_shard_search_where; every rank passes the same query, where and ids): the best
        `top_k` frames of the whole sharded corpus that pass `where` (its time, tag, location and term clauses) and the
        optional id filter; identical to search_where on one engine holding the whole corpus.  top_k <= 128."""
        if allow is not None and deny is not None:
            raise ValueError("pass at most one of allow= / deny=")
        fids = np.ascontiguousarray(allow if allow is not None else (deny if deny is not None else []),
                                    dtype=np.uint64).reshape(-1)
        terms = np.ascontiguousarray([int(t) for t in where.terms], dtype=np.uint64)
        w = where.to_c_near()
        q = np.ascontiguousarray(vector, dtype=np.float32).reshape(-1)
        cap = _clamp_topk(top_k)
        ids = np.empty(cap, np.uint64)
        scores = np.empty(cap, np.float32)
        n = C.c_uint32(0)
        _check(L.lib().wax_vs_shard_search_where(
            self._h, q.ctypes.data_as(C.POINTER(C.c_float)), q.size, int(top_k),
            fids.ctypes.data_as(C.POINTER(C.c_uint64)) if fids.size else None, fids.size, 0 if allow is not None else 1,
            C.byref(w), terms.ctypes.data_as(C.POINTER(C.c_uint64)) if terms.size else None, terms.size,
            ids.ctypes.data_as(C.POINTER(C.c_uint64)), scores.ctypes.data_as(C.POINTER(C.c_float)), cap, C.byref(n)))
        return [(int(ids[i]), float(scores[i])) for i in range(n.value)]

    def time_shard_search(self, top_k: int, iters: int, warmup: int = 3, n_queries: int = 1, seed: int = 7):
        """Device-timed collective searches, strictly one at a time on one stream. Returns (ms_total, launches)."""
        ms, launches = C.c_float(0), C.c_uint64(0)
        _check(L.lib().wax_vs_debug_time_shard_search(self._h, n_queries, int(top_k), seed, warmup, iters,
                                                      C.byref(ms), C.byref(launches)))
        return ms.value, launches.value

    # -- persistence (MV2V encoding = 2)
    def serialize(self) -> bytes:
        n = C.c_uint64(0)
        _check(L.lib().wax_vs_serialized_length(self._h, C.byref(n)))
        buf = bytearray(n.value)          # calloc'ed, written once by the library: no zero-fill pass, no trailing copy
        out = C.c_uint64(0)
        ptr = (C.c_uint8 * len(buf)).from_buffer(buf) if buf else (C.c_uint8 * 1)()
        _check(L.lib().wax_vs_serialize(self._h, ptr, len(buf), C.byref(out)))
        del ptr
        if out.value != len(buf):
            del buf[out.value:]
        return buf                          # bytes-like (compares equal to bytes; pass to deserialize() as is)

    def deserialize(self, data: bytes) -> None:
        buf = np.frombuffer(data, np.uint8)     # zero-copy view of bytes / bytearray / memoryview
        ptr = buf.ctypes.data_as(C.POINTER(C.c_uint8)) if buf.size else C.cast(C.c_char_p(b""), C.POINTER(C.c_uint8))
        _check(L.lib().wax_vs_deserialize(self._h, ptr, buf.size))
        self._dirty = False

    def stage_for_commit(self, into) -> None:
        """stageForCommit(into:) (:818-828): `into` needs stage_vec_index_for_next_commit(bytes, vector_count,
        dimension, similarity) -- the Wax store itself is out of scope (SURVEY.md section 8)."""
        if not self._dirty:
            return
        into.stage_vec_index_for_next_commit(bytes=self.serialize(), vector_count=self.count,
                                             dimension=self.dimensions,
                                             similarity=self.metric.to_vec_similarity())
        self._dirty = False

    # -- instrumentation
    def debug_buffer_pool_stats(self) -> Tuple[int, int]:
        a, r = C.c_uint64(0), C.c_uint64(0)
        _check(L.lib().wax_vs_debug_pool_stats(self._h, C.byref(a), C.byref(r)))
        return a.value, r.value

    def fill_synthetic(self, seed: int, rows: int, first_row: int = 0, id_base: int = 0,
                       normalize: bool = True) -> None:
        _check(L.lib().wax_vs_debug_fill_synthetic(self._h, seed, first_row, rows, id_base, int(normalize)))
        self._dirty = True

    def read_rows(self, first: int, n: int) -> np.ndarray:
        out = np.empty((n, self.dimensions), np.float32)
        _check(L.lib().wax_vs_debug_read_rows(self._h, first, n, out.ctypes.data_as(C.POINTER(C.c_float))))
        return out

    def time_search(self, top_k: int, iters: int, warmup: int = 3, n_queries: int = 1, seed: int = 7):
        """Kernel-only timing (CUDA events on the launching stream). Returns (ms_total, launches)."""
        ms, launches = C.c_float(0), C.c_uint64(0)
        _check(L.lib().wax_vs_debug_time_search(self._h, n_queries, int(top_k), seed, warmup, iters,
                                                C.byref(ms), C.byref(launches)))
        return ms.value, launches.value

    def batch_stats(self) -> Tuple[int, int]:
        """(queries answered by the tensor-core path with a completed proof, queries re-run exactly)."""
        a, b = C.c_uint64(0), C.c_uint64(0)
        _check(L.lib().wax_vs_debug_batch_stats(self._h, C.byref(a), C.byref(b)))
        return a.value, b.value

    def counter(self, name: str) -> int:
        """Named instrumentation counter (wax_vs_debug_counter): batch_bf16_queries, batch_retry_queries, shadow_bytes, ..."""
        v = C.c_uint64(0)
        _check(L.lib().wax_vs_debug_counter(self._h, name.encode(), C.byref(v)))
        return v.value

    def last_scan(self) -> dict:
        """The form of the last fp32 scan this engine launched (wax_vs_debug_last_scan): kernel (1 = TMA-staged,
        2 = direct-load), C, R, warps, stages, grid, chunk_steps (0 = static claims), mode (0 = k <= 32 list,
        1 = k <= 128 list, 2 = emit + select), tail (0 = merge or none, 1 = select staged, 2 = select from L2) and
        inline_query (1 = the query rode in the kernel parameters).  Read it while no search runs."""
        out = np.zeros(10, np.uint32)
        _check(L.lib().wax_vs_debug_last_scan(self._h, out.ctypes.data_as(C.POINTER(C.c_uint32))))
        names = ("kernel", "C", "R", "warps", "stages", "grid", "chunk_steps", "mode", "tail", "inline_query")
        return {name: int(v) for name, v in zip(names, out)}

    def time_search_batch(self, n_queries: int, top_k: int, iters: int, warmup: int = 2, seed: int = 7):
        """Device-only timing of the batched path. Returns (ms_total, launches, unproven_in_last_step)."""
        ms, launches, bad = C.c_float(0), C.c_uint64(0), C.c_uint32(0)
        _check(L.lib().wax_vs_debug_time_search_batch(self._h, n_queries, int(top_k), seed, warmup, iters,
                                                      C.byref(ms), C.byref(launches), C.byref(bad)))
        return ms.value, launches.value, bad.value

    def batch_nominations(self, queries, top_k: int, allow_rows=None):
        """Read-out of the batched path's nomination stage (wax_vs_debug_batch_nominations), in the form the options
        select.  Returns a dict: scores [n_queries, count] fp32 (every score' compared against the threshold; never
        written entries keep the 0xFFFFFFFF NaN payload), ok [n_queries], heaps [slices*groups, kprime, 128] uint64 and
        the launch shape (bf16, ares, pair, stages, kprime, slices, groups).  `allow_rows`: optional row filter."""
        q = np.ascontiguousarray(queries, dtype=np.float32).reshape(-1, self.dimensions)
        nq, n = q.shape[0], self.count
        scores = np.empty((nq, n), np.float32)
        ok = np.empty(nq, np.uint32)
        shape = np.zeros(7, np.uint32)
        bits = None
        if allow_rows is not None:
            mask = np.zeros(((n + 31) // 32) * 32, bool)
            mask[np.asarray(allow_rows, np.int64)] = True
            bits = (mask.reshape(-1, 32).astype(np.uint64) << np.arange(32, dtype=np.uint64)).sum(1).astype(np.uint32)
        u32 = lambda a: a.ctypes.data_as(C.POINTER(C.c_uint32))
        heaps = np.empty(0, np.uint64)
        for _ in range(2):     # the first call reports how many heap entries the shape it picked needs
            rc = L.lib().wax_vs_debug_batch_nominations(
                self._h, q.ctypes.data_as(C.POINTER(C.c_float)), nq, int(top_k), None if bits is None else u32(bits),
                scores.ctypes.data_as(C.POINTER(C.c_float)), u32(ok),
                heaps.ctypes.data_as(C.POINTER(C.c_uint64)) if heaps.size else None, heaps.size, u32(shape))
            if rc != L.ERR_BUFFER or heaps.size:
                break
            heaps = np.empty(int(shape[5]) * int(shape[6]) * int(shape[4]) * 128, np.uint64)
        _check(rc)
        names = ("bf16", "ares", "pair", "stages", "kprime", "slices", "groups")
        out = {name: int(v) for name, v in zip(names, shape)}
        out.update(scores=scores, ok=ok, heaps=heaps.reshape(out["slices"] * out["groups"], out["kprime"], 128))
        return out

    def shadow_nominations(self, vector, top_k: int, allow_rows=None):
        """Read-out of the single-query bf16-shadow route's nomination and finish (wax_vs_debug_shadow_nominations), in
        the shape the options select.  Returns a dict: keys [128] uint64 nominee keys (entry 0 = the worst, entries
        1..127 = the best first), ok (the proof flag), result [(frame_id, score)] of the finish (the search's scores,
        padding dropped) and the launch shape (C, R, warps, stages, grid, chunk_steps, tail_select).  `allow_rows`:
        optional row filter."""
        return self._route_nominations(L.lib().wax_vs_debug_shadow_nominations, vector, top_k, allow_rows)

    def int8_nominations(self, vector, top_k: int, allow_rows=None):
        """shadow_nominations for the int8 form of the route (wax_vs_debug_int8_nominations): the INT8 scan nominates
        from the int8 shadow in the shape the int8_* options select and the finish proves with its measured bound."""
        return self._route_nominations(L.lib().wax_vs_debug_int8_nominations, vector, top_k, allow_rows)

    def u4_nominations(self, vector, top_k: int, allow_rows=None):
        """shadow_nominations for the 4-bit form of the route (wax_vs_debug_u4_nominations): the U4 scan nominates from
        the 4-bit shadow in the shape the u4_* options select, every CTA writes its best 256 keys (keys [grid * 256],
        unordered, padding 0xFFFF...), and the grid-wide re-score proves.  Also rho_max, rho_q (the measured row and
        query coding bounds) and tau_excl (the score' no left-out row exceeds; -inf when none was left out)."""
        return self._route_nominations(L.lib().wax_vs_debug_u4_nominations, vector, top_k, allow_rows, u4=True)

    def _route_nominations(self, fn, vector, top_k: int, allow_rows, u4: bool = False):
        q = np.ascontiguousarray(vector, dtype=np.float32).reshape(self.dimensions)
        n = self.count
        k = max(1, min(int(top_k), n))
        keys = np.empty(256 * 1024 if u4 else 128, np.uint64)
        bound = np.zeros(3, np.float32)
        ok = C.c_uint32(0)
        result = (L.Candidate * k)()
        shape = np.zeros(7, np.uint32)
        bits = None
        if allow_rows is not None:
            mask = np.zeros(((n + 31) // 32) * 32, bool)
            mask[np.asarray(allow_rows, np.int64)] = True
            bits = (mask.reshape(-1, 32).astype(np.uint64) << np.arange(32, dtype=np.uint64)).sum(1).astype(np.uint32)
        u32 = lambda a: a.ctypes.data_as(C.POINTER(C.c_uint32))
        if u4:
            _check(fn(
                self._h, q.ctypes.data_as(C.POINTER(C.c_float)), int(top_k), None if bits is None else u32(bits),
                keys.ctypes.data_as(C.POINTER(C.c_uint64)), keys.size, C.byref(ok), result, u32(shape),
                bound.ctypes.data_as(C.POINTER(C.c_float))))
            keys = keys[:int(shape[4]) * 256]
        else:
            _check(fn(
                self._h, q.ctypes.data_as(C.POINTER(C.c_float)), int(top_k), None if bits is None else u32(bits),
                keys.ctypes.data_as(C.POINTER(C.c_uint64)), C.byref(ok), result, u32(shape)))
        one = np.float32(1.0)
        score = (lambda d: float(one - np.float32(d))) if self.metric is VectorMetric.cosine else (lambda d: float(-np.float32(d)))
        names = ("C", "R", "warps", "stages", "grid", "chunk_steps", "tail_select")
        out = {name: int(v) for name, v in zip(names, shape)}
        out.update(keys=keys, ok=ok.value, result=[(int(c.frame_id), score(c.distance)) for c in result if c.valid])
        if u4:
            out.update(rho_max=float(bound[0]), rho_q=float(bound[1]), tau_excl=float(bound[2]))
        return out

    def read_shadow(self, first: int, n: int) -> np.ndarray:
        """The bf16 shadow of rows [first, first + n) as uint16 bit patterns [n, dims] (wax_vs_debug_read_shadow)."""
        out = np.empty((n, self.dimensions), np.uint16)
        _check(L.lib().wax_vs_debug_read_shadow(self._h, first, n, out.ctypes.data_as(C.POINTER(C.c_uint16))))
        return out

    def read_int8_shadow(self, first: int, n: int):
        """The int8 shadow of rows [first, first + n) (wax_vs_debug_read_int8_shadow): (codes [n, dims] uint8 as stored,
        i.e. code + 128; scales [n] float32; rho_max, the measured bound of the whole shadow)."""
        codes = np.empty((n, self.dimensions), np.uint8)
        scales = np.empty(n, np.float32)
        rho = C.c_float(0.0)
        _check(L.lib().wax_vs_debug_read_int8_shadow(self._h, first, n, codes.ctypes.data_as(C.POINTER(C.c_uint8)),
                                                     scales.ctypes.data_as(C.POINTER(C.c_float)), C.byref(rho)))
        return codes, scales, float(rho.value)

    def read_u4_shadow(self, first: int, n: int):
        """The 4-bit shadow of rows [first, first + n) (wax_vs_debug_read_u4_shadow): (codes [n, dims] uint8 in 0..15,
        unpacked to element order; half_steps [n] float32, a row decodes to h * (2 u - 15); rho_max of the whole shadow)."""
        packed = np.empty((n, self.dimensions // 2), np.uint8)
        half = np.empty(n, np.float32)
        rho = C.c_float(0.0)
        _check(L.lib().wax_vs_debug_read_u4_shadow(self._h, first, n, packed.ctypes.data_as(C.POINTER(C.c_uint8)),
                                                   half.ctypes.data_as(C.POINTER(C.c_float)), C.byref(rho)))
        # byte b of 4-byte word w: element 8w + b in the low nibble, 8w + 4 + b in the high one
        w = packed.reshape(n, -1, 4)
        codes = np.concatenate([w & 15, w >> 4], axis=2).reshape(n, self.dimensions)
        return codes, half, float(rho.value)

    def stream_read_gbs(self, iters: int = 5) -> float:
        """Plain coalesced read of the corpus bytes: the box's streaming-read ceiling in GB/s."""
        ms, nbytes = C.c_float(0), C.c_uint64(0)
        _check(L.lib().wax_vs_debug_stream_read(self._h, iters, C.byref(ms), C.byref(nbytes)))
        return nbytes.value / (ms.value * 1e6) if ms.value > 0 else 0.0

    def set_option(self, key: str, value: int) -> None:
        _check(L.lib().wax_vs_debug_set_option(self._h, key.encode(), int(value)))


class VectorSearchSession:
    """The score-preserving entry `WaxVectorSearchSession.search` (VectorSearchSession.swift:70-76):
    cosine queries that are not unit length (tolerance 1e-3) are normalised on the host first."""

    def __init__(self, engine: CUDAVectorEngine):
        self.engine = engine
        self.metric = engine.metric

    def search(self, vector: Sequence[float], top_k: int):
        q = np.ascontiguousarray(vector, dtype=np.float32)
        if self.metric is VectorMetric.cosine and q.size and not is_normalized_l2(q):
            q = normalize_l2(q)
        return self.engine.search(q, top_k)
