"""CPU: the location clause of wax_vs_search_batch_where_near / wax_vs_search_batch_grouped_where_near -- the box
wax_vs_location_box computes and the bins wax_vs_set_locations stores, pinned against a Python transcription of
PhotoRAG's Swift, and the argument checks that run before any CUDA call."""
import ctypes as C
import math

import numpy as np
import pytest

from wax_b200 import Where, location_bin, location_box
from wax_b200 import _lib as L


# ---- the Swift, transcribed (Sources/Wax/PhotoRAG/...) -----------------------------------------------------------------
class Trap(Exception):
    """Where Swift's Int(_:) traps; the library returns WAX_VS_ERR_ARGUMENT instead."""


def swift_min(x, y):          # Swift.min: `y < x ? y : x`
    return y if y < x else x


def swift_max(x, y):          # Swift.max: `y >= x ? y : x`
    return y if y >= x else x


def swift_int_floor(x):       # Int(floor(x)): Int(_: Double) traps on NaN, +-inf and values outside Int64
    if not (-2.0 ** 63 <= x < 2.0 ** 63):
        raise Trap(x)
    return int(math.floor(x))


def photo_coordinate(lat, lon):
    """PhotoCoordinate.init (PhotoRAGTypes.swift:40-43)."""
    return swift_min(90.0, swift_max(-90.0, lat)), swift_min(180.0, swift_max(-180.0, lon))


def build_location_allowlist_box(lat, lon, radius):
    """PhotoLocationQuery.init (PhotoRAGTypes.swift:53-56) and buildLocationAllowlist (PhotoRAGOrchestrator.swift:
    788-854) up to the bin loop: (latBins, lonRanges), or None where Swift returns nil."""
    lat, lon = photo_coordinate(lat, lon)
    radius = swift_max(0.0, radius)
    if not radius > 0:                                                         # :792
        return None
    lat_delta = radius / 111_000.0                                             # :798
    lon_delta = swift_min(180.0, radius / swift_max(1e-6, 111_000.0 * math.cos(lat * math.pi / 180)))   # :801
    min_lat, max_lat = lat - lat_delta, lat + lat_delta
    min_lon, max_lon = lon - lon_delta, lon + lon_delta
    min_lat_bin = swift_max(-9000, swift_int_floor(min_lat * 100.0))    # :809-813
    max_lat_bin = swift_min(9000, swift_int_floor(max_lat * 100.0))
    min_lon_bin = swift_int_floor(min_lon * 100.0)
    max_lon_bin = swift_int_floor(max_lon * 100.0)
    lat_count = max_lat_bin - min_lat_bin + 1                                  # :817-825
    if min_lon_bin <= max_lon_bin:
        lon_count = max_lon_bin - min_lon_bin + 1
    else:
        lon_count = (18000 - min_lon_bin) + (max_lon_bin - (-18000)) + 1
    if not (lat_count > 0 and lon_count > 0):                                  # :827
        return None
    if not lat_count * lon_count < 100_000:                                    # :830
        return None
    if min_lon_bin <= max_lon_bin:                                             # :837-841
        lon_ranges = [(min_lon_bin, max_lon_bin)]
    else:
        lon_ranges = [(min_lon_bin, 18000), (-18000, max_lon_bin)]
    return (min_lat_bin, max_lat_bin), lon_ranges


def swift_location_bin(lat, lon):
    """locationBin(from:) (PhotoRAGOrchestrator.swift:868-875) on parsed doubles."""
    return swift_int_floor(lat * 100.0), swift_int_floor(lon * 100.0)


# ---- the library against the transcription ---------------------------------------------------------------------------
def library_box(lat, lon, radius):
    box = (C.c_int32 * 4)()
    active = C.c_int32(7)
    rc = L.lib().wax_vs_location_box(lat, lon, radius, box, C.byref(active))
    if rc != L.OK:
        return rc
    return (box[0], box[1], box[2], box[3]) if active.value else None


def expected_box(lat, lon, radius):
    try:
        got = build_location_allowlist_box(lat, lon, radius)
    except Trap:
        return L.ERR_ARGUMENT
    if got is None:
        return None
    (lat_lo, lat_hi), ranges = got
    return (lat_lo, lat_hi, ranges[0][0], ranges[-1][1])


def _guard_radius(lat):
    """The radius at which a box centred at (lat, 0.005) first reaches 100 000 bins, by bisection on the transcription."""
    lo, hi = 1.0, 2e7
    for _ in range(200):
        mid = (lo + hi) / 2
        if build_location_allowlist_box(lat, 0.005, mid) is None:
            hi = mid
        else:
            lo = mid
    return lo, hi


CENTRES = [(90.0, 0.0), (-90.0, 0.0), (89.999, 10.0), (0.0, 0.0), (0.0, 180.0), (0.0, -180.0), (0.0, 179.995),
           (0.0, -179.995), (45.0, 179.995), (0.29, 0.29), (-0.29, -0.29), (0.01, 0.07), (37.7749, -122.4194),
           (51.5, -0.12), (-33.86, 151.21), (-0.0, -0.0), (1e-12, -1e-12), (100.0, 200.0), (-1000.0, -1000.0)]
RADII = [-1.0, 0.0, -0.0, float("nan"), 1.0, 1000.0, 100_000.0, 1e7, 1e-9, 1e21, 1e23, float("inf"), -float("inf")]


def test_location_box_restates_build_location_allowlist():
    radii = list(RADII)
    for lat in (0.0, 45.0, 89.0):
        radii.extend(_guard_radius(lat))                         # either side of the 100 000-bin guard
    for lat, lon in CENTRES:
        for r in radii:
            assert library_box(lat, lon, r) == expected_box(lat, lon, r), (lat, lon, r)


def test_location_box_on_non_finite_centres():
    nan, inf = float("nan"), float("inf")
    for lat in (nan, inf, -inf, 0.0):
        for lon in (nan, inf, -inf, 0.0):
            for r in (1000.0, 100_000.0):
                assert library_box(lat, lon, r) == expected_box(lat, lon, r), (lat, lon, r)
    # a NaN latitude becomes -90 (max(-90, NaN) is -90): the box of the south pole
    assert library_box(nan, 0.0, 1000.0) == library_box(-90.0, 0.0, 1000.0)


def test_location_box_on_random_centres():
    rng = np.random.default_rng(11)
    for _ in range(3000):
        lat = float(rng.uniform(-95, 95))
        lon = float(rng.uniform(-185, 185))
        r = float(10 ** rng.uniform(-1, 7.3))
        if rng.random() < 0.3:                                      # on a bin edge
            lat, lon = round(lat, 2), round(lon, 2)
        assert library_box(lat, lon, r) == expected_box(lat, lon, r), (lat, lon, r)


def test_location_box_edges():
    assert library_box(0.0, 0.0, 0.0) is None                        # radius <= 0: no clause
    assert library_box(0.0, 0.0, float("nan")) is None               # max(0, NaN) is 0
    assert library_box(0.0, 0.0, float("inf")) == L.ERR_ARGUMENT     # Int(-inf) traps in Swift
    assert "not representable" in L.last_error()
    assert library_box(0.0, 0.0, 1e7) is None                        # the 100 000-bin guard
    assert library_box(0.29, 0.0, 1e-3)[0] == 28                     # 0.29 * 100 = 28.999999999999996
    assert library_box(0.0, 0.0, 1.0) == (-1, 0, -1, 0)
    assert location_box(0.0, 0.0, 1.0) == (-1, 0, -1, 0)
    assert location_box(0.0, 0.0, 0.0) is None
    box = location_box(90.0, 0.0, 1.0)                               # at the pole lonDelta is 180: every lon bin
    assert box is not None and box[:2] == (8999, 9000) and box[2:] == (-18000, 18000)


def test_antimeridian_branch_is_unreachable_but_restated():
    # minLonBin > maxLonBin needs a negative lonDelta; PhotoLocationQuery clamps the radius to >= 0
    rng = np.random.default_rng(3)
    for _ in range(500):
        got = build_location_allowlist_box(float(rng.uniform(-90, 90)), float(rng.uniform(-180, 180)),
                                           float(10 ** rng.uniform(0, 6.5)))
        assert got is None or len(got[1]) == 1
    w = Where(near=(0.0, 0.0, 1.0))
    assert w.passes(0, 0, (-1, -1)) and w.passes(0, 0, (0, 0)) and not w.passes(0, 0, (1, 0))
    assert not w.passes(0, 0, None)                                  # a frame without a location is in no bin
    assert Where().passes(0, 0, None) and Where(near=(0.0, 0.0, 0.0)).passes(0, 0, None)


# ---- the frame-bin rule ----------------------------------------------------------------------------------------------
def library_bin(lat, lon):
    out = (C.c_int32 * 2)()
    has = C.c_int32(7)
    rc = L.lib().wax_vs_location_bin(lat, lon, out, C.byref(has))
    if rc != L.OK:
        return rc
    return (out[0], out[1]) if has.value else None


def test_frame_bins_restate_location_bin():
    rng = np.random.default_rng(5)
    coords = [(0.29, -0.29), (0.0, -0.0), (-0.001, 0.001), (90.0, 180.0), (-90.0, -180.0), (179.995, -179.995),
              (100.0, 400.0), (-1000.5, 3600.25), (1e-300, -1e-300), (37.77493, -122.41942)]
    coords += [(float(a), float(b)) for a, b in zip(rng.uniform(-200, 200, 2000), rng.uniform(-400, 400, 2000))]
    coords += [(round(float(a), 2), round(float(b), 2)) for a, b in zip(rng.uniform(-90, 90, 2000),
                                                                         rng.uniform(-180, 180, 2000))]
    for lat, lon in coords:
        assert library_bin(lat, lon) == swift_location_bin(lat, lon), (lat, lon)
        assert location_bin(lat, lon) == swift_location_bin(lat, lon)
    assert library_bin(0.29, 0.0) == (28, 0)


def test_frame_bins_of_non_finite_and_huge_coordinates():
    nan, inf = float("nan"), float("inf")
    assert library_bin(nan, nan) is None                             # a NaN pair: no location
    for lat, lon in [(nan, 0.0), (0.0, nan), (inf, 0.0), (0.0, -inf), (inf, inf), (nan, inf)]:
        assert library_bin(lat, lon) == L.ERR_ARGUMENT, (lat, lon)
    imax = np.iinfo(np.int32).max
    assert library_bin(1e300, -1e300) == (imax, -imax)               # saturated: no box reaches past +-36 000
    assert library_bin(3e7, -3e7) == (imax, -imax)


# ---- argument checks: they return before the engine is locked or any CUDA call is made, so a placeholder handle (a
# zeroed block the library never reads on these paths) stands in for an engine on a CPU-only box
_placeholder = (C.c_uint8 * (1 << 16))()
ENG = C.cast(_placeholder, C.c_void_p)


def test_where_near_struct_layout():
    assert C.sizeof(L.WhereNear) == 56
    assert [L.WhereNear.where.offset, L.WhereNear.latitude.offset, L.WhereNear.longitude.offset,
            L.WhereNear.radius_m.offset] == [0, 32, 40, 48]
    w = Where(after=3, before=9, all_tags=1, no_tags=2, near=(1.5, -2.5, 300.0)).to_c_near()
    assert (w.where.after, w.where.before, w.where.all_tags, w.where.no_tags) == (3, 9, 1, 2)
    assert (w.latitude, w.longitude, w.radius_m) == (1.5, -2.5, 300.0)
    assert Where().to_c_near().radius_m == 0.0                        # no near: no location clause


def test_set_locations_argument_checks():
    lib = L.lib()
    out = C.c_uint64(7)
    d = lambda *v: (C.c_double * len(v))(*v)
    u = lambda *v: (C.c_uint64 * len(v))(*v)
    assert lib.wax_vs_set_locations(None, None, None, None, 0, C.byref(out)) == L.ERR_NULL
    assert lib.wax_vs_set_locations(ENG, None, None, None, 0, C.byref(out)) == L.OK and out.value == 0   # n == 0
    assert lib.wax_vs_set_locations(ENG, None, d(0.0), d(0.0), 1, None) == L.ERR_NULL                    # ids NULL
    assert lib.wax_vs_set_locations(ENG, u(1), None, d(0.0), 1, None) == L.ERR_NULL
    assert lib.wax_vs_set_locations(ENG, u(1), d(0.0), None, 1, None) == L.ERR_NULL
    for lat, lon in [(float("nan"), 0.0), (0.0, float("inf")), (-float("inf"), float("nan"))]:
        assert lib.wax_vs_set_locations(ENG, u(1, 2), d(0.0, lat), d(0.0, lon), 2, None) == L.ERR_ARGUMENT
        assert "not finite" in L.last_error()
    assert lib.wax_vs_location_box(0.0, 0.0, 1.0, None, None) == L.ERR_NULL
    assert lib.wax_vs_location_bin(0.0, 0.0, None, None) == L.ERR_NULL


def _near_call(eng=ENG, n_queries=2, query_filter=(L.NO_FILTER, L.NO_FILTER), wheres=(Where(),), query_where=(0, 0),
               out_n=True):
    q = np.zeros(n_queries * 4, np.float32)
    off = np.zeros(1, np.uint64)
    qf = None if query_filter is None else np.asarray(query_filter, np.uint32)
    qw = None if query_where is None else np.asarray(query_where, np.uint32)
    warr = None if wheres is None else (L.WhereNear * max(len(wheres), 1))(*[w.to_c_near() for w in wheres])
    ns = np.zeros(max(n_queries, 1), np.uint32)
    ids = np.zeros(64, np.uint64)
    sc = np.zeros(64, np.float32)
    p = lambda a, t: None if a is None else a.ctypes.data_as(C.POINTER(t))
    return L.lib().wax_vs_search_batch_where_near(
        eng, p(q, C.c_float), n_queries, 4, 10, None, p(off, C.c_uint64), None, 0, p(qf, C.c_uint32),
        None if warr is None else C.cast(warr, C.c_void_p), 0 if wheres is None else len(wheres), p(qw, C.c_uint32),
        p(ids, C.c_uint64), p(sc, C.c_float), 32, p(ns, C.c_uint32) if out_n else None)


def test_search_batch_where_near_argument_checks():
    assert _near_call(eng=None) == L.ERR_NULL
    assert _near_call(out_n=False) == L.ERR_NULL
    assert _near_call(query_filter=None) == L.ERR_NULL
    assert _near_call(query_where=None) == L.ERR_NULL
    assert _near_call(query_where=(0, 1)) == L.ERR_ARGUMENT
    assert "names where 1 of 1" in L.last_error()
    assert _near_call(query_filter=(0, L.NO_FILTER)) == L.ERR_ARGUMENT                   # filter 0 of 0
    # a box Swift could not compute, even in a predicate no query names
    bad = Where(near=(0.0, 0.0, float("inf")))
    assert _near_call(wheres=(Where(), bad), query_where=(0, 0)) == L.ERR_ARGUMENT
    assert "not representable" in L.last_error()
    assert _near_call(wheres=(Where(near=(0.0, 0.0, 1e30)),)) == L.ERR_ARGUMENT


def _grouped_near_call(eng=ENG, where=Where(near=(0.0, 0.0, 1000.0)), per_group=2, top_groups=5, mode=1, n_ids=0):
    q = np.zeros(8, np.float32)
    w = None if where is None else where.to_c_near()
    ids = np.zeros(64, np.uint64)
    sc = np.zeros(64, np.float32)
    gr = np.zeros(64, np.uint64)
    ns = np.zeros(2, np.uint32)
    p = lambda a, t: a.ctypes.data_as(C.POINTER(t))
    return L.lib().wax_vs_search_batch_grouped_where_near(
        eng, p(q, C.c_float), 2, 4, top_groups, per_group, None, n_ids, mode,
        C.cast(C.pointer(w), C.c_void_p) if w is not None else None, p(ids, C.c_uint64), p(sc, C.c_float),
        p(gr, C.c_uint64), 32, p(ns, C.c_uint32))


def test_search_batch_grouped_where_near_argument_checks():
    assert _grouped_near_call(where=None) == L.ERR_NULL
    assert "where is NULL" in L.last_error()
    assert _grouped_near_call(eng=None) == L.ERR_NULL
    assert _grouped_near_call(per_group=0) == L.ERR_ARGUMENT
    assert _grouped_near_call(per_group=L.MAX_PER_GROUP + 1) == L.ERR_ARGUMENT
    assert _grouped_near_call(top_groups=10_000, per_group=2) == L.ERR_ARGUMENT
    assert _grouped_near_call(mode=3) == L.ERR_ARGUMENT
    assert _grouped_near_call(n_ids=3) == L.ERR_NULL
    assert _grouped_near_call(where=Where(near=(0.0, 0.0, float("inf")))) == L.ERR_ARGUMENT


@pytest.mark.parametrize("bad", [float("inf"), 1e23])
def test_python_surface_raises_where_swift_traps(bad):
    from wax_b200 import WaxError
    with pytest.raises(WaxError):
        location_box(0.0, 0.0, bad)
