"""The btree comparators of vector / halfvec / sparsevec and the order the GPU's vb_order is checked against
(tests/order_oracle.c with the CPU oracle's HalfToFloat4, oracle/pgv_distance.c), compiled here at first use into a
directory of the temporary area.  TEST INFRASTRUCTURE ONLY."""
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
SRC = os.path.join(HERE, "order_oracle.c")
CFLAGS = ["-O2", "-fno-fast-math", "-ffp-contract=off", "-fPIC"]

VECTOR, HALFVEC, SPARSE = 0, 1, 2

_lib = None


def lib() -> C.CDLL:
    global _lib
    if _lib is not None:
        return _lib
    h = hashlib.sha1()
    for p in (SRC, os.path.join(ORACLE, "pgv_distance.c"), os.path.join(ORACLE, "pgv_oracle.h")):
        h.update(open(p, "rb").read())
    h.update(O._cpu_stamp().encode())
    d = os.path.join(tempfile.gettempdir(), f"order_oracle_{os.getuid()}_{h.hexdigest()[:16]}")
    so = os.path.join(d, "liborderoracle.so")
    if not os.path.exists(so):
        os.makedirs(d, exist_ok=True)
        tmp = f"{so}.{os.getpid()}.tmp"
        subprocess.run(["gcc", *CFLAGS, "-shared", "-I", ORACLE, "-o", tmp, SRC, os.path.join(ORACLE, "pgv_distance.c"), "-lm"],
                       check=True, capture_output=True)
        os.replace(tmp, so)
    L = C.CDLL(so)
    vp, i32, i64 = C.c_void_p, C.c_int, C.c_int64
    for name, res, args in [("ord_vector_cmp", i32, [vp, i32, vp, i32]),
                            ("ord_halfvec_cmp", i32, [vp, i32, vp, i32]),
                            ("ord_sparsevec_cmp", i32, [i32, i32, vp, vp, i32, i32, vp, vp]),
                            ("ord_dense_cmp_pairs", None, [i32, vp, vp, i64, i32, vp]),
                            ("ord_sparse_cmp_pairs", None, [i32, i64, vp, vp, vp, vp, vp, vp, vp]),
                            ("ord_order", i64, [i32, i32, vp, vp, vp, vp, i64, vp, vp, vp]),
                            ("ord_bounds", None, [i32, i32, vp, vp, vp, vp, i64, vp, vp, vp, vp, i64, vp, vp])]:
        getattr(L, name).restype = res
        getattr(L, name).argtypes = args
    _lib = L
    return L


def _p(a):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


def half_bits(a):
    """halfvec rows as IEEE binary16 bit patterns (uint16): float16 reinterpreted, other floats rounded"""
    a = np.asarray(a)
    if a.dtype == np.uint16:
        return np.ascontiguousarray(a)
    if a.dtype != np.float16:
        with np.errstate(over="ignore"):
            a = a.astype(np.float16)
    return np.ascontiguousarray(a.view(np.uint16))


def _csr(s):
    return (np.ascontiguousarray(s.row_off, dtype=np.int64), np.ascontiguousarray(s.idx, dtype=np.int32),
            np.ascontiguousarray(s.val, dtype=np.float32))


def vector_cmp(a, b):
    a, b = np.ascontiguousarray(a, np.float32), np.ascontiguousarray(b, np.float32)
    return lib().ord_vector_cmp(_p(a), a.size, _p(b), b.size)


def halfvec_cmp(a, b):
    a, b = half_bits(a), half_bits(b)
    return lib().ord_halfvec_cmp(_p(a), a.size, _p(b), b.size)


def sparsevec_cmp(a, b):
    """a, b: SparseVectors (their own dimensions)"""
    ai, ax = np.ascontiguousarray(a.indices, np.int32), np.ascontiguousarray(a.values, np.float32)
    bi, bx = np.ascontiguousarray(b.indices, np.int32), np.ascontiguousarray(b.values, np.float32)
    return lib().ord_sparsevec_cmp(a.dim, ai.size, _p(ai), _p(ax), b.dim, bi.size, _p(bi), _p(bx))


def dense_cmp_pairs(half, a, b):
    """sign of the comparator for each pair of rows a[k], b[k] ([npairs, dim] each)"""
    a = half_bits(a) if half else np.ascontiguousarray(a, np.float32)
    b = half_bits(b) if half else np.ascontiguousarray(b, np.float32)
    out = np.empty(a.shape[0], np.int32)
    lib().ord_dense_cmp_pairs(int(half), _p(a), _p(b), a.shape[0], a.shape[1], _p(out))
    return out


def sparse_cmp_pairs(a, b):
    """a, b: SparseRows of one dimension and one row count"""
    ao, ai, av = _csr(a)
    bo, bi, bv = _csr(b)
    out = np.empty(a.n, np.int32)
    lib().ord_sparse_cmp_pairs(a.dim, a.n, _p(ao), _p(ai), _p(av), _p(bo), _p(bi), _p(bv), _p(out))
    return out


def _table(kind, rows):
    if kind == SPARSE:
        off, idx, val = _csr(rows)
        return rows.dim, rows.n, None, off, idx, val
    r = half_bits(rows) if kind == HALFVEC else np.ascontiguousarray(rows, np.float32)
    return r.shape[1], r.shape[0], r, None, None, None


def order(kind, rows):
    """(perm int64 [n], group_of_row int32 [n], group_start int64 [groups + 1]) of dense rows [n, dim] or SparseRows"""
    dim, n, r, off, idx, val = _table(kind, rows)
    perm = np.empty(n, np.int64)
    gor = np.empty(n, np.int32)
    gst = np.empty(n + 1, np.int64)
    g = lib().ord_order(kind, dim, _p(r), _p(off), _p(idx), _p(val), n, _p(perm), _p(gor), _p(gst))
    return perm, gor, gst[:g + 1].copy()


def bounds(kind, rows, queries):
    """(lo, hi) per query: rows < q and rows <= q (linear scan)"""
    dim, n, r, off, idx, val = _table(kind, rows)
    if kind == SPARSE:
        qo, qi, qv = _csr(queries)
        q, nq = None, queries.n
    else:
        q = half_bits(queries) if kind == HALFVEC else np.ascontiguousarray(queries, np.float32)
        qo = qi = qv = None
        nq = q.shape[0]
    lo = np.empty(nq, np.int64)
    hi = np.empty(nq, np.int64)
    lib().ord_bounds(kind, dim, _p(r), _p(off), _p(idx), _p(val), n, _p(q), _p(qo), _p(qi), _p(qv), nq, _p(lo), _p(hi))
    return lo, hi
