"""The serial restatement of the reference's vector / halfvec aggregates the GPU aggregate is checked against
(tests/aggregate_oracle.c with the CPU oracle's half conversions, oracle/pgv_distance.c), compiled here at first use into
a directory of the temporary area.  TEST INFRASTRUCTURE ONLY.

The flags are plain IEEE ones (no -ffast-math family, no contraction): the oracle's chains of float8 / fp32 / fp16 adds
must run in the order written, one rounding per add, as the reference's single-add loops do."""
from __future__ import annotations

import ctypes as C
import hashlib
import os
import subprocess
import tempfile

import numpy as np

import oracle as O

HERE = os.path.dirname(os.path.abspath(__file__))
ORACLE = os.path.join(os.path.dirname(HERE), "oracle")
SRC = os.path.join(HERE, "aggregate_oracle.c")
CFLAGS = ["-O2", "-fno-fast-math", "-ffp-contract=off", "-fPIC"]

AVG, SUM = 0, 1
ERRBUF = 256

_lib = None


def lib() -> C.CDLL:
    global _lib
    if _lib is not None:
        return _lib
    h = hashlib.sha1()
    for p in (SRC, os.path.join(ORACLE, "pgv_distance.c"), os.path.join(ORACLE, "pgv_oracle.h")):
        h.update(open(p, "rb").read())
    h.update(O._cpu_stamp().encode())
    d = os.path.join(tempfile.gettempdir(), f"aggregate_oracle_{os.getuid()}_{h.hexdigest()[:16]}")
    so = os.path.join(d, "libaggoracle.so")
    if not os.path.exists(so):
        os.makedirs(d, exist_ok=True)
        tmp = f"{so}.{os.getpid()}.tmp"
        subprocess.run(["gcc", *CFLAGS, "-shared", "-I", ORACLE, "-o", tmp, SRC, os.path.join(ORACLE, "pgv_distance.c"), "-lm"],
                       check=True, capture_output=True)
        os.replace(tmp, so)
    L = C.CDLL(so)
    vp, i32, i64 = C.c_void_p, C.c_int, C.c_int64
    for name, args in [("agg_accum", [i32, vp, i32, i32, i32, vp, i32, vp, vp]),
                       ("agg_combine", [vp, i32, i32, i32, vp, i32, i32, i32, vp, vp, vp]),
                       ("agg_avg", [i32, vp, i32, i32, i32, vp, vp, vp]),
                       ("agg_add", [i32, vp, vp, i32, vp, vp]),
                       ("agg_table", [i32, i32, vp, i64, i32, vp, i32, i64, vp, vp, vp, vp])]:
        getattr(L, name).restype = i32
        getattr(L, name).argtypes = args
    _lib = L
    return L


class AggregateError(Exception):
    """the reference's ERROR, with its message"""


def _p(a):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


def _err(buf):
    raise AggregateError(buf.value.decode())


def _rows(half, rows, dim):
    if half:
        a = np.asarray(rows)
        a = a.view(np.uint16) if a.dtype == np.float16 else (a.astype(np.float32).astype(np.float16).view(np.uint16)
                                                               if a.dtype != np.uint16 else a)
        return np.ascontiguousarray(a, dtype=np.uint16).reshape(-1, dim)
    return np.ascontiguousarray(rows, dtype=np.float32).reshape(-1, dim)


def state_array(lit):
    """a float8[] literal as nested Python lists (None = NULL) -> (ndim, first length, has nulls, float64 data), as the
    ArrayType CheckStateArray inspects; [] is '{}', which has no dimensions"""
    def depth(x):
        return 1 + depth(x[0]) if isinstance(x, list) and x else (1 if isinstance(x, list) else 0)
    nd = depth(lit) if lit != [] else 0
    flat = np.array(lit, dtype=object).ravel().tolist() if lit else []
    hasnull = any(v is None for v in flat)
    data = np.array([0.0 if v is None else float(v) for v in flat] or [0.0], dtype=np.float64)
    return nd, (len(lit) if nd == 1 else (len(lit) if lit else 0)), int(hasnull), data


def accum(half, st, x):
    """vector_accum / halfvec_accum(state literal, row) -> the new state as a list"""
    nd, l0, hn, data = state_array(st)
    x = _rows(half, [x], len(x))[0]
    dim = x.shape[0]
    out = np.empty(dim + 1, dtype=np.float64)
    e = C.create_string_buffer(ERRBUF)
    if lib().agg_accum(int(half), _p(data), nd, l0, hn, _p(x), dim, _p(out), e):
        _err(e)
    return out.tolist()


def combine(s1, s2):
    """vector_combine / halfvec_combine(state literal, state literal) -> the new state as a list"""
    a, b = state_array(s1), state_array(s2)
    out = np.empty(max(a[3].size, b[3].size) + 1, dtype=np.float64)
    olen = C.c_int()
    e = C.create_string_buffer(ERRBUF)
    if lib().agg_combine(_p(a[3]), a[0], a[1], a[2], _p(b[3]), b[0], b[1], b[2], _p(out), C.byref(olen), e):
        _err(e)
    return out[:olen.value].tolist()


def final_avg(half, st):
    """vector_avg / halfvec_avg(state literal) -> float32 / float16 array, or None (SQL NULL)"""
    nd, l0, hn, data = state_array(st)
    out = np.empty(max(l0 - 1, 1), dtype=np.uint16 if half else np.float32)
    is_null = C.c_int()
    e = C.create_string_buffer(ERRBUF)
    if lib().agg_avg(int(half), _p(data), nd, l0, hn, _p(out), C.byref(is_null), e):
        _err(e)
    if is_null.value:
        return None
    return out.view(np.float16) if half else out


def add(half, a, b):
    """vector_add / halfvec_add of two rows of one dimension"""
    a, b = _rows(half, [a], len(a))[0], _rows(half, [b], len(b))[0]
    out = np.empty_like(a)
    e = C.create_string_buffer(ERRBUF)
    if lib().agg_add(int(half), _p(a), _p(b), a.shape[0], _p(out), e):
        _err(e)
    return out.view(np.float16) if half else out


def table_aggregate(half, agg, rows, dim, groups=None, ngroups=1, run_rows=0, state=False):
    """vb_table_aggregate's plan on the CPU: (values [G, dim] float32 / float16, counts [G]) (+ float8 state [G, dim + 1]
    for avg with state=True); raises AggregateError("value out of range: overflow") where the plan overflows"""
    rows = _rows(half, rows, dim)
    n = rows.shape[0]
    g = None if groups is None else np.ascontiguousarray(groups, dtype=np.int32)
    out = np.empty((ngroups, dim), dtype=np.uint16 if half else np.float32)
    counts = np.empty(ngroups, dtype=np.int64)
    st = np.empty((ngroups, dim + 1), dtype=np.float64) if state else None
    e = C.create_string_buffer(ERRBUF)
    if lib().agg_table(int(half), agg, _p(rows), n, dim, _p(g), ngroups, int(run_rows), _p(out), _p(counts), _p(st), e):
        _err(e)
    vals = out.view(np.float16) if half else out
    return (vals, counts, st) if state else (vals, counts)
