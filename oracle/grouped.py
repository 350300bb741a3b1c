"""ctypes binding of the grouped-search CPU ORACLE (oracle/wax_oracle_grouped.c).

TEST INFRASTRUCTURE ONLY, like oracle/oracle.py: importable from tests/ and scripts/, never from wax_b200/.  The grouped
oracle is built into its own library together with wax_oracle.c (same flags as oracle/Makefile), so it scores rows with
exactly the frame oracle's arithmetic.  See oracle/wax_oracle_grouped.h for the semantics it restates.
"""
from __future__ import annotations

import ctypes as C
import subprocess
from pathlib import Path

import numpy as np

from . import oracle as _o

_HERE = Path(__file__).resolve().parent
_LIB_PATH = _HERE / "libwax_oracle_grouped.so"
_SOURCES = ("wax_oracle.c", "wax_oracle_grouped.c")
_CFLAGS = ["-O3", "-march=native", "-ffp-contract=off", "-fno-math-errno", "-fPIC", "-pthread", "-Wall", "-Wextra",
           "-std=c11"]


def build(force: bool = False) -> Path:
    """Compile wax_oracle.c + wax_oracle_grouped.c with gcc into libwax_oracle_grouped.so."""
    deps = [_HERE / n for n in (*_SOURCES, "wax_oracle.h", "wax_oracle_grouped.h", "grouped.py")]
    if force or not _LIB_PATH.exists() or _LIB_PATH.stat().st_mtime < max(d.stat().st_mtime for d in deps):
        tmp = _LIB_PATH.with_suffix(".so.tmp")
        subprocess.run(["gcc", *_CFLAGS, "-shared", "-o", str(tmp), *[str(_HERE / s) for s in _SOURCES], "-lm",
                        "-lpthread"], check=True, capture_output=True)
        tmp.replace(_LIB_PATH)
    return _LIB_PATH


_lib = None


def lib() -> C.CDLL:
    global _lib
    if _lib is None:
        build()
        _lib = C.CDLL(str(_LIB_PATH))
        f32p, u64p, u32p, u8p = (C.POINTER(C.c_float), C.POINTER(C.c_uint64), C.POINTER(C.c_uint32),
                                 C.POINTER(C.c_uint8))
        _lib.wax_oracle_search_grouped.restype = C.c_int
        _lib.wax_oracle_search_grouped.argtypes = [C.c_int, C.c_int, f32p, C.c_uint64, C.c_uint32, f32p, u64p, u8p,
                                                   C.c_int64, C.c_uint32, C.c_uint64, C.c_int, u64p, f32p, f32p, u64p,
                                                   u32p]
        _lib.wax_oracle_search_grouped_synth.restype = C.c_int
        _lib.wax_oracle_search_grouped_synth.argtypes = [C.c_int, C.c_int, C.c_uint64, C.c_uint64, C.c_uint64,
                                                         C.c_uint32, C.c_int, f32p, C.c_uint32, u64p, u8p, C.c_int64,
                                                         C.c_uint32, C.c_int, u64p, f32p, f32p, u64p, u32p]
    return _lib


def _p(a: np.ndarray, t):
    return a.ctypes.data_as(C.POINTER(t))


def _mask(allowed, n_rows: int):
    """allowed: None (every row), a bool mask of n_rows, or an array of allowed row indices."""
    if allowed is None:
        return None
    a = np.asarray(allowed)
    if a.dtype == bool and a.size == n_rows:
        return np.ascontiguousarray(a, dtype=np.uint8)
    m = np.zeros(n_rows, np.uint8)
    m[a.astype(np.int64)] = 1
    return m


def _cap(top_groups: int, per_group: int, n_rows: int) -> int:
    return max(1, min(_o.clamp_topk(top_groups) * max(int(per_group), 1), max(n_rows, 1)))


def search_grouped(metric: int, corpus, query, row_group, top_groups: int, per_group: int = 1, allowed=None,
                   mode: int = _o.ACC_F32_SEQ, row_base: int = 0, threads: int = 1):
    """Exact grouped search.  Returns (rows u64[n], distances f32[n], scores f32[n], groups u64[n]), group-major."""
    corpus, query = _o._f32(corpus), _o._f32(query)
    n_rows, dims = (corpus.shape if corpus.ndim == 2 else (0, query.size))
    groups = np.ascontiguousarray(row_group, dtype=np.uint64).reshape(-1)
    assert groups.size == n_rows
    m = _mask(allowed, n_rows)
    cap = _cap(top_groups, per_group, n_rows)
    rows = np.zeros(cap, np.uint64); d = np.zeros(cap, np.float32); s = np.zeros(cap, np.float32)
    g = np.zeros(cap, np.uint64)
    n = C.c_uint32(0)
    rc = lib().wax_oracle_search_grouped(metric, mode, _p(corpus, C.c_float), n_rows, dims, _p(query, C.c_float),
                                         _p(groups, C.c_uint64), None if m is None else _p(m, C.c_uint8),
                                         int(top_groups), int(per_group), row_base, threads, _p(rows, C.c_uint64),
                                         _p(d, C.c_float), _p(s, C.c_float), _p(g, C.c_uint64), C.byref(n))
    if rc != 0:
        raise RuntimeError(f"wax_oracle_search_grouped rc={rc}")
    k = n.value
    return rows[:k].copy(), d[:k].copy(), s[:k].copy(), g[:k].copy()


def search_grouped_synth(metric: int, seed: int, first_row: int, n_rows: int, dims: int, normalize: bool, queries,
                         row_group, top_groups: int, per_group: int = 1, allowed=None, mode: int = _o.ACC_F32_SEQ,
                         threads: int = 1):
    """search_grouped over generator rows, several queries in one streamed pass.  Returns a list of
    (rows, distances, scores, groups) per query."""
    queries = _o._f32(queries).reshape(-1, dims)
    b = queries.shape[0]
    groups = np.ascontiguousarray(row_group, dtype=np.uint64).reshape(-1)
    assert groups.size == n_rows
    m = _mask(allowed, n_rows)
    cap = _cap(top_groups, per_group, n_rows)
    rows = np.zeros((b, cap), np.uint64); d = np.zeros((b, cap), np.float32); s = np.zeros((b, cap), np.float32)
    g = np.zeros((b, cap), np.uint64)
    n = np.zeros(b, np.uint32)
    rc = lib().wax_oracle_search_grouped_synth(metric, mode, seed, first_row, n_rows, dims, int(normalize),
                                               _p(queries, C.c_float), b, _p(groups, C.c_uint64),
                                               None if m is None else _p(m, C.c_uint8), int(top_groups), int(per_group),
                                               threads, _p(rows, C.c_uint64), _p(d, C.c_float), _p(s, C.c_float),
                                               _p(g, C.c_uint64), _p(n, C.c_uint32))
    if rc != 0:
        raise RuntimeError(f"wax_oracle_search_grouped_synth rc={rc}")
    return [(rows[q, :n[q]].copy(), d[q, :n[q]].copy(), s[q, :n[q]].copy(), g[q, :n[q]].copy()) for q in range(b)]
