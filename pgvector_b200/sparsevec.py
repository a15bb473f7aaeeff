"""sparsevec on the device -- host-side mirror of the reference's sparsevec functions (src/sparsevec.c:826-1150) over
the C ABI (vb_sparsevec_* / vb_sparse_table_* / vb_sparse_exact_topk[_filtered]).

A value is ``SparseVector(dim, indices, values)`` with 0-based ascending indices (the on-disk order,
src/sparsevec.h:17-32); the text form '{index:value,...}/dim' is 1-based like the reference's I/O functions.  A batch
of rows is ``SparseRows`` (CSR).  Everything computes on the GPU; nothing here falls back to numpy math.
"""
from __future__ import annotations

import ctypes as C

import numpy as np

from . import _lib
from ._lib import load

L2_SQUARED, NEG_IP, COSINE, L1, L2, IP = 0, 1, 2, 3, 6, 7
SPARSEVEC_MAX_DIM = 1_000_000_000     # src/sparsevec.h:11
SPARSEVEC_MAX_NNZ = 16_000            # src/sparsevec.h:12
HNSW_MAX_NNZ = 1000                   # src/hnsw.h: sparsevec limit of the hnsw opclasses

# hnsw opclasses over sparsevec (sql/vector.sql sparsevec_*_ops): proc-1 metric, normalise?
OPCLASSES = {
    "sparsevec_l2_ops": (L2_SQUARED, False),
    "sparsevec_ip_ops": (NEG_IP, False),
    "sparsevec_cosine_ops": (NEG_IP, True),
    "sparsevec_l1_ops": (L1, False),
}


def _p(a):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


class SparseVector:
    """one sparsevec value; zero values are not stored (sparsevec_in drops them, src/sparsevec.c:322-333)"""

    def __init__(self, dim, indices=(), values=()):
        dim = int(dim)
        if dim < 1:
            raise ValueError("sparsevec must have at least 1 dimension")
        if dim > SPARSEVEC_MAX_DIM:
            raise ValueError(f"sparsevec cannot have more than {SPARSEVEC_MAX_DIM} dimensions")
        idx = np.asarray(indices, dtype=np.int64).ravel()
        val = np.asarray(values, dtype=np.float32).ravel()
        if idx.shape != val.shape:
            raise ValueError("indices and values differ in length")
        if np.isnan(val).any():
            raise ValueError("NaN not allowed in sparsevec")
        if np.isinf(val).any():
            raise ValueError("infinite value not allowed in sparsevec")
        keep = val != 0
        idx, val = idx[keep], val[keep]
        order = np.argsort(idx, kind="stable")
        idx, val = idx[order], val[order]
        if idx.size > SPARSEVEC_MAX_NNZ:
            raise ValueError(f"sparsevec cannot have more than {SPARSEVEC_MAX_NNZ} non-zero elements")
        if idx.size and (idx[0] < 0 or idx[-1] >= dim):
            raise ValueError("sparsevec index out of bounds")
        if idx.size > 1 and (np.diff(idx) == 0).any():
            raise ValueError("sparsevec indices must not contain duplicates")
        self.dim = dim
        self.indices = np.ascontiguousarray(idx, dtype=np.int32)
        self.values = np.ascontiguousarray(val, dtype=np.float32)

    @property
    def nnz(self):
        return int(self.indices.size)

    @classmethod
    def from_text(cls, text):
        """'{1:1.5,3:2}/5' (1-based indices, src/sparsevec.c:215-395)"""
        t = text.strip()
        try:
            body, dim = t.rsplit("/", 1)
            body = body.strip()
            if not (body.startswith("{") and body.endswith("}")):
                raise ValueError
            idx, val = [], []
            inner = body[1:-1].strip()
            if inner:
                for item in inner.split(","):
                    i, v = item.split(":")
                    idx.append(int(i) - 1)
                    val.append(float(v))
            dim = int(dim)
        except ValueError:
            raise ValueError(f'invalid input syntax for type sparsevec: "{text}"') from None
        return cls(dim, idx, val)

    @classmethod
    def from_dense(cls, x):
        x = np.asarray(x, dtype=np.float32).ravel()
        nz = np.nonzero(x)[0]
        return cls(x.size, nz, x[nz])

    def to_dense(self):
        out = np.zeros(self.dim, dtype=np.float32)
        out[self.indices] = self.values
        return out

    def to_text(self):
        def fmt(v):
            s = repr(float(np.float32(v)))
            # shortest float4 text
            for p in range(1, 10):
                c = f"{float(v):.{p}g}"
                if np.float32(c) == np.float32(v):
                    s = c
                    break
            return s
        return "{" + ",".join(f"{int(i) + 1}:{fmt(v)}" for i, v in zip(self.indices, self.values)) + "}/" + str(self.dim)

    def __repr__(self):
        return f"SparseVector({self.to_text()!r})"


class SparseRows:
    """n sparsevec rows of one dimension as CSR (row_off[n + 1], idx, val)"""

    def __init__(self, dim, row_off, idx, val):
        self.dim = int(dim)
        self.row_off = np.ascontiguousarray(row_off, dtype=np.int64)
        self.idx = np.ascontiguousarray(idx, dtype=np.int32)
        self.val = np.ascontiguousarray(val, dtype=np.float32)
        if self.row_off.ndim != 1 or self.row_off.size < 1 or self.idx.shape != self.val.shape:
            raise ValueError("bad CSR arrays")

    @property
    def n(self):
        return int(self.row_off.size - 1)

    @classmethod
    def from_vectors(cls, vectors, dim=None):
        vectors = list(vectors)
        if dim is None:
            if not vectors:
                raise ValueError("dim is required for an empty batch")
            dim = vectors[0].dim
        for v in vectors:
            if v.dim != dim:
                raise ValueError(f"expected {dim} dimensions, not {v.dim}")    # CheckExpectedDim, src/sparsevec.c:56-63
        off = np.zeros(len(vectors) + 1, dtype=np.int64)
        off[1:] = np.cumsum([v.nnz for v in vectors])
        idx = np.concatenate([v.indices for v in vectors]) if vectors else np.empty(0, np.int32)
        val = np.concatenate([v.values for v in vectors]) if vectors else np.empty(0, np.float32)
        return cls(dim, off, idx, val)

    @classmethod
    def from_dense(cls, x):
        x = np.asarray(x, dtype=np.float32)
        if x.ndim == 1:
            x = x.reshape(1, -1)
        r, c = np.nonzero(x)
        off = np.zeros(x.shape[0] + 1, dtype=np.int64)
        off[1:] = np.cumsum(np.bincount(r, minlength=x.shape[0]))
        return cls(x.shape[1], off, c, x[r, c])

    def row(self, r):
        b, e = self.row_off[r], self.row_off[r + 1]
        return SparseVector(self.dim, self.idx[b:e], self.val[b:e])


def _rows(rows):
    if isinstance(rows, SparseRows):
        return rows
    if isinstance(rows, SparseVector):
        return SparseRows.from_vectors([rows])
    return SparseRows.from_vectors(rows)


def distance_batch(metric, q, rows):
    """float8 distances of one query against n rows, as the sparsevec SQL function returns them; ``q=None`` is the
    NULL query (all zeros, src/hnswutils.c:555-556)"""
    rows = _rows(rows)
    out = np.empty(rows.n, dtype=np.float64)
    if q is None:
        rc = load().vb_sparsevec_distance_batch(metric, rows.dim, rows.dim, -1, None, None, rows.n, _p(rows.row_off), _p(rows.idx),
                                                _p(rows.val), _p(out))
    else:
        rc = load().vb_sparsevec_distance_batch(metric, rows.dim, q.dim, q.nnz, _p(q.indices), _p(q.values), rows.n, _p(rows.row_off),
                                                _p(rows.idx), _p(rows.val), _p(out))
    if rc == _lib.EINVAL:
        msg = load().vb_last_error().decode()
        if msg.startswith("different sparsevec dimensions"):
            raise ValueError(msg)
    _lib.check(rc)
    return out


def l2_distance(q, rows):
    return distance_batch(L2, q, rows)


def l2_squared_distance(q, rows):
    return distance_batch(L2_SQUARED, q, rows)


def inner_product(q, rows):
    return distance_batch(IP, q, rows)


def negative_inner_product(q, rows):
    return distance_batch(NEG_IP, q, rows)


def cosine_distance(q, rows):
    return distance_batch(COSINE, q, rows)


def l1_distance(q, rows):
    return distance_batch(L1, q, rows)


def l2_norm(rows):
    rows = _rows(rows)
    out = np.empty(rows.n, dtype=np.float64)
    _lib.check(load().vb_sparsevec_norm_batch(rows.n, _p(rows.row_off), _p(rows.val), _p(out)))
    return out


def l2_normalize(rows):
    """l2_normalize of every row (src/sparsevec.c:1082-1150); raises OverflowError with the reference's text"""
    rows = _rows(rows)
    off = np.empty(rows.n + 1, dtype=np.int64)
    idx = np.empty(max(rows.idx.size, 1), dtype=np.int32)
    val = np.empty(max(rows.val.size, 1), dtype=np.float32)
    rc = load().vb_sparsevec_l2_normalize_batch(rows.n, _p(rows.row_off), _p(rows.idx), _p(rows.val), _p(off), _p(idx), _p(val))
    if rc == _lib.EINVAL and load().vb_last_error().decode() == "value out of range: overflow":
        raise OverflowError("value out of range: overflow")
    _lib.check(rc)
    kept = int(off[-1])
    return SparseRows(rows.dim, off, idx[:kept], val[:kept])


class SparseTable:
    """sparsevec rows resident in HBM; ``exact_topk`` is the sequential-scan plan ORDER BY v <op> q LIMIT k, with
    row filters (``filter``) for a WHERE clause; ``rerank`` orders candidate rows another index fetched"""

    def __init__(self, dim):
        self.dim = int(dim)
        h = C.c_void_p()
        _lib.check(load().vb_sparse_table_create(self.dim, C.byref(h)))
        self.h = h

    def append(self, rows):
        rows = _rows(rows)
        if rows.dim != self.dim:
            raise ValueError(f"expected {self.dim} dimensions, not {rows.dim}")
        _lib.check(load().vb_sparse_table_append(self.h, rows.n, _p(rows.row_off), _p(rows.idx), _p(rows.val)))
        return self

    @property
    def rows(self):
        return int(load().vb_sparse_table_rows(self.h))

    @property
    def nnz(self):
        return int(load().vb_sparse_table_nnz(self.h))

    def filter(self, rows):
        """a row Filter of this table (WHERE <predicate> as the row numbers it allows, numpy int64).  Rows appended
        later are not in it."""
        from . import Filter
        rows = np.ascontiguousarray(rows, dtype=np.int64).reshape(-1)   # host rows only, like the rest of the sparse API
        return Filter._create(self, "vb_sparse_table_filter_create", rows)

    def exact_topk(self, metric, queries, k, filter=None, filter_of_query=None):
        """ORDER BY v <op> q LIMIT k without an index.  filter: a Filter of this table, or a list of them with
        filter_of_query[q] = the index of query q's filter; each query then gets exactly what rerank() returns for its
        filter's rows in ascending order (k <= 2048)."""
        q = _rows(queries)
        k = int(k)
        ids = np.empty((q.n, k), dtype=np.int64)
        dist = np.empty((q.n, k), dtype=np.float64)
        if filter is None:
            rc = load().vb_sparse_exact_topk(self.h, metric, q.dim, q.n, _p(q.row_off), _p(q.idx), _p(q.val), k, _p(ids), _p(dist))
        else:
            from . import _filter_args
            farr, nf, fq = _filter_args(filter, filter_of_query)
            if fq is not None and len(fq) != q.n:
                raise ValueError(f"filter_of_query must have {q.n} entries, got {len(fq)}")
            rc = load().vb_sparse_exact_topk_filtered(self.h, metric, q.dim, q.n, _p(q.row_off), _p(q.idx), _p(q.val), k, farr, nf, _p(fq),
                                                      _p(ids), _p(dist))
        return self._result(rc, ids, dist)

    def rerank(self, metric, queries, candidates, k):
        """ORDER BY v <op> q LIMIT k over each query's own candidate rows: candidates[q] = row numbers of this table
        (-1 = none), typically what a dense or quantized index returned (hybrid search)."""
        q = _rows(queries)
        k = int(k)
        cand = np.asarray(candidates)
        if cand.dtype != np.int64 or cand.ndim != 2 or cand.shape[0] != q.n:
            raise ValueError(f"rerank: candidates must be int64 of shape [{q.n}, c], got {cand.dtype} {cand.shape}")
        cand = np.ascontiguousarray(cand)
        ids = np.empty((q.n, k), dtype=np.int64)
        dist = np.empty((q.n, k), dtype=np.float64)
        rc = load().vb_sparse_table_rerank(self.h, metric, q.dim, q.n, _p(q.row_off), _p(q.idx), _p(q.val), _p(cand), cand.shape[1], k,
                                           _p(ids), _p(dist))
        return self._result(rc, ids, dist)

    @staticmethod
    def _result(rc, ids, dist):
        if rc == _lib.EINVAL:
            msg = load().vb_last_error().decode()
            if msg.startswith("different sparsevec dimensions"):
                raise ValueError(msg)
        _lib.check(rc)
        return ids, dist

    def free(self):
        if self.h:
            load().vb_sparse_table_free(self.h)
            self.h = None

    def __del__(self):
        try:
            self.free()
        except Exception:
            pass
