"""sparsevec on the device -- host-side mirror of the reference's sparsevec functions (src/sparsevec.c:826-1150) over
the C ABI (vb_sparsevec_* / vb_sparse_table_* / vb_sparse_exact_topk[_filtered], their _dev variants, and the casts
vb_dense_to_sparsevec_batch / vb_sparsevec_to_dense_batch).

A value is ``SparseVector(dim, indices, values)`` with 0-based ascending indices (the on-disk order,
src/sparsevec.h:17-32); the text form '{index:value,...}/dim' is 1-based like the reference's I/O functions.  A batch
of rows is ``SparseRows`` (CSR).  Everything computes on the GPU; nothing here falls back to numpy math.

Device CSR: the table calls also take rows and queries that live on the GPU, as a ``torch.sparse_csr_tensor`` [n, dim] or
a ``(row_off, idx, val)`` triple of CUDA tensors, and then return CUDA tensors (int64 ids, float32 distances).  Nothing
goes through host memory; the library checks the CSR on the device.
"""
from __future__ import annotations

import ctypes as C

import numpy as np

from . import _lib
from . import numeric as _numeric
from ._lib import load

VECTOR, HALFVEC = 0, 1
INT32_MAX = 2**31 - 1

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


def _is_cuda(a):
    return a is not None and not isinstance(a, np.ndarray) and hasattr(a, "data_ptr") and bool(getattr(a, "is_cuda", False))


def _device_csr(x, dim):
    """(n, dim, row_off, idx, val) of CUDA CSR input in the layout the _dev entry points read (int64 offsets, int32
    indices, float32 values, contiguous), or None for host input.  x: a torch.sparse_csr_tensor [n, dim] (its dim wins)
    or a (row_off, idx, val) triple of CUDA tensors.  int64 column indices are narrowed with a range check: a value
    outside [0, 2^31) becomes -1, which the library's device check refuses ("sparsevec index out of bounds (row r)")."""
    if isinstance(x, (tuple, list)) and len(x) == 3 and all(_is_cuda(a) for a in x):
        off, idx, val = x
    elif _is_cuda(x) and str(getattr(x, "layout", "")) == "torch.sparse_csr":
        off, idx, val = x.crow_indices(), x.col_indices(), x.values()
        dim = int(x.shape[1])
    else:
        return None
    import torch
    if off.dim() != 1 or idx.dim() != 1 or val.dim() != 1 or idx.shape != val.shape or off.numel() < 1:
        raise ValueError("device CSR: row_off [n + 1], idx [nnz] and val [nnz] must be 1-d, idx and val of one length")
    if idx.dtype == torch.int64:
        idx = torch.where((idx >= 0) & (idx <= INT32_MAX), idx, torch.full_like(idx, -1))
    off = off.to(torch.int64).contiguous()
    idx = idx.to(torch.int32).contiguous()
    val = val.to(torch.float32).contiguous()
    return off.numel() - 1, int(dim), off, idx, val


def _run_dev(fn, *args, tensors=()):
    """a _dev call on tensors torch produced: the library stream waits for torch's, and the results are handed back
    complete (as the dense calls do)"""
    from . import _after_torch, synchronize
    _after_torch(*tensors)
    rc = getattr(load(), fn)(*args)
    if rc == _lib.OK:
        synchronize()
    return rc


def _tp(t):
    return None if t is None else C.c_void_p(t.data_ptr())


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


# ------------------------------------------------------------------------- casts between the dense types and sparsevec

_CAP_ERROR = "non-zero elements, more than cap"


def _to_sparsevec(elem, rows, cap):
    if _is_cuda(rows):
        import torch
        want = torch.float32 if elem == VECTOR else torch.float16
        if rows.dtype != want:
            raise TypeError(f"{'vector' if elem == VECTOR else 'halfvec'} rows must be a {want} CUDA tensor, not {rows.dtype}")
        x = rows.reshape(1, -1) if rows.dim() == 1 else rows
        x = x.contiguous()
        n, dim = int(x.shape[0]), int(x.shape[1])
        off = torch.empty(n + 1, dtype=torch.int64, device=x.device)

        def run(cap):
            idx = torch.empty(max(cap, 1), dtype=torch.int32, device=x.device)
            val = torch.empty(max(cap, 1), dtype=torch.float32, device=x.device)
            rc = _run_dev("vb_dense_to_sparsevec_batch_dev", elem, dim, _tp(x), n, cap, _tp(off), _tp(idx), _tp(val), tensors=(x,))
            return rc, idx, val
        rc, idx, val = run(0 if cap is None else int(cap))
        if cap is None and rc == _lib.EINVAL and _CAP_ERROR in load().vb_last_error().decode():
            rc, idx, val = run(int(off[-1].item()))   # the offsets were written: they size the output
        _lib.check(rc)
        tot = int(off[-1].item())
        return off, idx[:tot], val[:tot]
    if elem == VECTOR:
        x = np.ascontiguousarray(rows, dtype=np.float32)
    else:
        x = np.asarray(rows)
        x = np.ascontiguousarray(x.view(np.uint16) if x.dtype == np.float16 else x, dtype=np.uint16)
    x = x.reshape(1, -1) if x.ndim == 1 else x
    n, dim = x.shape
    off = np.empty(n + 1, dtype=np.int64)

    def run(cap):
        idx = np.empty(max(cap, 1), dtype=np.int32)
        val = np.empty(max(cap, 1), dtype=np.float32)
        return load().vb_dense_to_sparsevec_batch(elem, dim, _p(x), n, cap, _p(off), _p(idx), _p(val)), idx, val
    rc, idx, val = run(0 if cap is None else int(cap))
    if cap is None and rc == _lib.EINVAL and _CAP_ERROR in load().vb_last_error().decode():
        rc, idx, val = run(int(off[-1]))
    _lib.check(rc)
    tot = int(off[-1])
    return SparseRows(dim, off, idx[:tot], val[:tot])


def vector_to_sparsevec(rows, cap=None):
    """vector -> sparsevec (src/sparsevec.c:606-645) of every row: the nonzero elements in index order (-0 is dropped).
    numpy float32 [n, dim] -> SparseRows; a float32 CUDA tensor -> (row_off, idx, val) CUDA tensors.  cap: an upper
    bound of the total nnz, if known (one pass); else the offsets of a first pass size the output."""
    return _to_sparsevec(VECTOR, rows, cap)


def halfvec_to_sparsevec(rows, cap=None):
    """halfvec -> sparsevec (src/sparsevec.c:650-689): numpy float16 (or uint16 bit patterns) [n, dim] -> SparseRows; a
    float16 CUDA tensor -> (row_off, idx, val) CUDA tensors; values widened exactly, zeros of either sign dropped"""
    return _to_sparsevec(HALFVEC, rows, cap)


ARRAY_INT4, ARRAY_FLOAT4, ARRAY_FLOAT8, ARRAY_NUMERIC = 0, 1, 2, 3   # VB_ARRAY_*: integer[], real[], double precision[], numeric[]


class ArrayCastError(ValueError):
    """an error of array_to_sparsevec: the reference's errmsg, with the failing row (.row)"""

    def __init__(self, msg, row):
        super().__init__(msg)
        self.row = row


def _array_check(rc, bad):
    if rc == _lib.EINVAL:
        msg = load().vb_last_error().decode()
        if not msg.startswith("vb_"):   # the reference's texts; argument refusals name the entry point
            raise ArrayCastError(msg, int(bad.value))
    _lib.check(rc)


def array_to_sparsevec(rows, typmod=-1, cap=None):
    """integer[] / real[] / double precision[] / numeric[] :: sparsevec(typmod) of every row (array_to_sparsevec,
    src/sparsevec.c:694-821): the dtype (int32, float32, float64) is the array type, each row one array of dim
    elements, up to 10^9; rows of decimal.Decimal values, or numeric.NumericArrays of numeric_send fields, are
    numeric[].  An element is (float) of the value (numeric: numeric_float4) and is kept when it is not zero (-0 and
    doubles that round to 0 are dropped).  Host rows -> SparseRows; CUDA rows -> (row_off, idx, val) CUDA tensors, as
    vector_to_sparsevec.  cap: an upper bound of the total nnz, if known (one pass); else a first pass sizes the output.
    The reference's errors raise ArrayCastError (a ValueError) with the failing row."""
    bad = C.c_int64(-1)
    in_off = None
    if _numeric.is_numeric_rows(rows):
        A, _ = _numeric.as_numeric_arrays(rows)
        src, n, dim, dev = ARRAY_NUMERIC, A.n, A.dim, A.is_cuda
        x, in_off = A.data, A.off
        if not dev:
            x, in_off = np.ascontiguousarray(x), np.ascontiguousarray(in_off, dtype=np.int64)
    elif _is_cuda(rows):
        import torch
        src, dev = {torch.int32: ARRAY_INT4, torch.float32: ARRAY_FLOAT4, torch.float64: ARRAY_FLOAT8}.get(rows.dtype), True
        if src is None:
            raise ValueError("unsupported array type")
        x = rows.reshape(1, -1) if rows.dim() == 1 else rows
        if x.dim() != 2:
            raise ValueError("array must be 1-D")
        x = x.contiguous()
        n, dim = int(x.shape[0]), int(x.shape[1])
    else:
        x = np.asarray(rows)
        src, dev = {np.dtype(np.int32): ARRAY_INT4, np.dtype(np.float32): ARRAY_FLOAT4, np.dtype(np.float64): ARRAY_FLOAT8}.get(x.dtype), False
        if src is None:
            raise ValueError("unsupported array type")
        x = x.reshape(1, -1) if x.ndim == 1 else x
        if x.ndim != 2:
            raise ValueError("array must be 1-D")
        x = np.ascontiguousarray(x)
        n, dim = x.shape
    if dev:
        import torch
        off = torch.empty(n + 1, dtype=torch.int64, device=x.device)

        def run(cap):
            idx = torch.empty(max(cap, 1), dtype=torch.int32, device=x.device)
            val = torch.empty(max(cap, 1), dtype=torch.float32, device=x.device)
            rc = _run_dev("vb_array_to_sparsevec_batch_dev", src, dim, int(typmod), _tp(x), _tp(in_off), n, cap, _tp(off), _tp(idx),
                          _tp(val), C.byref(bad), tensors=(x,) if in_off is None else (x, in_off))
            return rc, idx, val
        total = lambda: int(off[-1].item())   # noqa: E731
    else:
        off = np.empty(n + 1, dtype=np.int64)

        def run(cap):
            idx = np.empty(max(cap, 1), dtype=np.int32)
            val = np.empty(max(cap, 1), dtype=np.float32)
            rc = load().vb_array_to_sparsevec_batch(src, dim, int(typmod), _p(x), _p(in_off), n, cap, _p(off), _p(idx), _p(val), C.byref(bad))
            return rc, idx, val
        total = lambda: int(off[-1])   # noqa: E731
    rc, idx, val = run(0 if cap is None else int(cap))
    if cap is None and rc == _lib.EINVAL and _CAP_ERROR in load().vb_last_error().decode():
        rc, idx, val = run(total())   # the offsets were written: they size the output
    _array_check(rc, bad)
    tot = total()
    return (off, idx[:tot], val[:tot]) if dev else SparseRows(dim, off, idx[:tot], val[:tot])


def _to_dense(elem, rows, dim):
    d = _device_csr(rows, dim)
    if d is not None:
        import torch
        n, dim, off, idx, val = d
        if dim is None:
            raise ValueError("dim is required for a (row_off, idx, val) triple")
        out = torch.empty((n, dim), dtype=torch.float32 if elem == VECTOR else torch.float16, device=off.device)
        rc = _run_dev("vb_sparsevec_to_dense_batch_dev", elem, dim, n, _tp(off), _tp(idx), _tp(val), _tp(out), tensors=(off, idx, val))
    else:
        r = _rows(rows)
        out = np.empty((r.n, r.dim), dtype=np.float32 if elem == VECTOR else np.float16)
        rc = load().vb_sparsevec_to_dense_batch(elem, r.dim, r.n, _p(r.row_off), _p(r.idx), _p(r.val), _p(out))
    if rc == _lib.EINVAL:
        msg = load().vb_last_error().decode()
        if "is out of range for type halfvec" in msg or "cannot have more than 16000 dimensions" in msg:
            raise ValueError(msg)
    _lib.check(rc)
    return out


def sparsevec_to_vector(rows, dim=None):
    """sparsevec -> vector (src/vector.c:1323-1349) of every row: SparseRows / SparseVectors -> numpy float32 [n, dim];
    device CSR (dim needed for a triple) -> a float32 CUDA tensor.  dim above 16000 raises ValueError (CheckDim)."""
    return _to_dense(VECTOR, rows, dim)


def sparsevec_to_halfvec(rows, dim=None):
    """sparsevec -> halfvec (src/halfvec.c:1199-1225): as sparsevec_to_vector, into float16 by Float4ToHalf; a finite
    value that overflows raises ValueError('"65520" is out of range for type halfvec')"""
    return _to_dense(HALFVEC, rows, dim)


def _order_bounds(order, queries):
    """Order.bounds of a sparse table's order: SparseRows / SparseVectors -> numpy (lo, hi); device CSR -> CUDA tensors"""
    d = _device_csr(queries, order.owner.dim)
    if d is not None:
        import torch
        nq, q_dim, off, idx, val = d
        lo = torch.empty(nq, dtype=torch.int64, device=off.device)
        hi = torch.empty(nq, dtype=torch.int64, device=off.device)
        rc = _run_dev("vb_sparse_order_bounds_dev", order.h, q_dim, nq, _tp(off), _tp(idx), _tp(val), _tp(lo), _tp(hi),
                      tensors=(off, idx, val))
        return SparseTable._result(rc, lo, hi)
    q = _rows(queries)
    lo = np.empty(q.n, dtype=np.int64)
    hi = np.empty(q.n, dtype=np.int64)
    rc = load().vb_sparse_order_bounds(order.h, q.dim, q.n, _p(q.row_off), _p(q.idx), _p(q.val), _p(lo), _p(hi))
    return SparseTable._result(rc, lo, hi)


class SparseTable:
    """sparsevec rows resident in HBM; ``exact_topk`` is the sequential-scan plan ORDER BY v <op> q LIMIT k, with
    row filters (``filter``) for a WHERE clause; ``rerank`` orders candidate rows another index fetched"""

    def __init__(self, dim):
        self.dim = int(dim)
        h = C.c_void_p()
        _lib.check(load().vb_sparse_table_create(self.dim, C.byref(h)))
        self.h = h

    def append(self, rows):
        """append rows: SparseVectors, SparseRows, or device CSR (a torch.sparse_csr_tensor or a (row_off, idx, val)
        triple of CUDA tensors, validated on the device; nothing is appended on any error)"""
        d = _device_csr(rows, self.dim)
        if d is not None:
            n, dim, off, idx, val = d
            if dim != self.dim:
                raise ValueError(f"expected {self.dim} dimensions, not {dim}")
            _lib.check(_run_dev("vb_sparse_table_append_dev", self.h, n, _tp(off), _tp(idx), _tp(val), tensors=(off, idx, val)))
            return self
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
        """a row Filter of this table (WHERE <predicate> as the row numbers it allows: numpy int64, or a 1-d int64 CUDA
        tensor whose values outside [0, rows) are ignored).  Rows appended later are not in it."""
        from . import Filter
        if not _is_cuda(rows):
            rows = np.ascontiguousarray(rows, dtype=np.int64).reshape(-1)
        return Filter._create(self, "vb_sparse_table_filter_create", rows)

    def exact_topk(self, metric, queries, k, filter=None, filter_of_query=None):
        """ORDER BY v <op> q LIMIT k without an index.  filter: a Filter of this table, or a list of them with
        filter_of_query[q] = the index of query q's filter; each query then gets exactly what rerank() returns for its
        filter's rows in ascending order (k <= 2048).  Device CSR queries return CUDA tensors (float32 distances, the
        float of the host call's float8); filter_of_query stays a host array."""
        k = int(k)
        d = _device_csr(queries, self.dim)
        if d is not None:
            import torch
            nq, q_dim, off, idx, val = d
            ids = torch.empty((nq, k), dtype=torch.int64, device=off.device)
            dist = torch.empty((nq, k), dtype=torch.float32, device=off.device)
            qa = (self.h, metric, q_dim, nq, _tp(off), _tp(idx), _tp(val), k)
            if filter is None:
                rc = _run_dev("vb_sparse_exact_topk_dev", *qa, _tp(ids), _tp(dist), tensors=(off, idx, val))
            else:
                from . import _filter_args
                farr, nf, fq = _filter_args(filter, filter_of_query)
                if fq is not None and len(fq) != nq:
                    raise ValueError(f"filter_of_query must have {nq} entries, got {len(fq)}")
                rc = _run_dev("vb_sparse_exact_topk_filtered_dev", *qa, farr, nf, _p(fq), _tp(ids), _tp(dist), tensors=(off, idx, val))
            return self._result(rc, ids, dist)
        q = _rows(queries)
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
        (-1 = none), typically what a dense or quantized index returned (hybrid search).  Device CSR queries take a
        [nq, c] int64 CUDA tensor of candidates (values outside [0, rows) are absent) and return CUDA tensors."""
        k = int(k)
        d = _device_csr(queries, self.dim)
        if d is not None:
            import torch
            nq, q_dim, off, idx, val = d
            if not _is_cuda(candidates) or candidates.dtype != torch.int64 or candidates.dim() != 2 or candidates.shape[0] != nq:
                raise ValueError(f"rerank: candidates of device queries must be an int64 CUDA tensor of shape [{nq}, c]")
            cand = candidates.contiguous()
            ids = torch.empty((nq, k), dtype=torch.int64, device=off.device)
            dist = torch.empty((nq, k), dtype=torch.float32, device=off.device)
            rc = _run_dev("vb_sparse_table_rerank_dev", self.h, metric, q_dim, nq, _tp(off), _tp(idx), _tp(val), _tp(cand),
                          int(cand.shape[1]), k, _tp(ids), _tp(dist), tensors=(off, idx, val, cand))
            return self._result(rc, ids, dist)
        q = _rows(queries)
        cand = np.asarray(candidates)
        if cand.dtype != np.int64 or cand.ndim != 2 or cand.shape[0] != q.n:
            raise ValueError(f"rerank: candidates must be int64 of shape [{q.n}, c], got {cand.dtype} {cand.shape}")
        cand = np.ascontiguousarray(cand)
        ids = np.empty((q.n, k), dtype=np.int64)
        dist = np.empty((q.n, k), dtype=np.float64)
        rc = load().vb_sparse_table_rerank(self.h, metric, q.dim, q.n, _p(q.row_off), _p(q.idx), _p(q.val), _p(cand), cand.shape[1], k,
                                           _p(ids), _p(dist))
        return self._result(rc, ids, dist)

    def order(self):
        """the rows in sparsevec_ops btree order (ORDER BY v, DISTINCT v, GROUP BY v, WHERE v = / < ... $1) as an
        Order; rows appended later are not in it"""
        from . import Order
        return Order._create(self, "vb_sparse_table_order_create", True)

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


# ------------------------------------------------------------------------- type I/O

def sparsevec_in(texts, typmod=-1):
    """sparsevec_in (src/sparsevec.c:203-409) of every literal -> (SparseRows, dims): ascending indices, no zeros;
    SparseRows.dim is the literals' common dimension (0 when they differ).  A (CUDA uint8 text, CUDA int64 offsets)
    pair gives ((row_off, idx, val), dims) as CUDA tensors.  The reference's errors raise TextInputError."""
    from . import _after_torch, _ptr, _raise_text, _text_input
    lib = load()
    text, off, n, dev = _text_input(texts)
    bad = C.c_int64(-1)
    if dev:
        import torch
        new = lambda k, dt: torch.empty(max(k, 1), dtype=dt, device=text.device)  # noqa: E731
        i32, i64, f32 = torch.int32, torch.int64, torch.float32
        fn = lib.vb_text_to_sparsevec_batch_dev
        _after_torch(text, off)
    else:
        new = lambda k, dt: np.empty(max(k, 1), dtype=dt)  # noqa: E731
        i32, i64, f32 = np.int32, np.int64, np.float32
        fn = lib.vb_text_to_sparsevec_batch
    row_off, dims = new(n + 1, i64), new(n, i32)
    row_off[:] = 0      # a refused argument writes no offsets
    rc = fn(typmod, n, _ptr(text), _ptr(off), 0, _ptr(dims), _ptr(row_off), None, None, C.byref(bad))
    bound = int(row_off[n])
    idx, val = new(bound, i32), new(bound, f32)
    if rc == _lib.EINVAL and bound > 0 and bad.value < 0:
        rc = fn(typmod, n, _ptr(text), _ptr(off), bound, _ptr(dims), _ptr(row_off), _ptr(idx), _ptr(val), C.byref(bad))
    _raise_text(rc, bad)
    tot = int(row_off[n])
    dims = dims[:n]
    if dev:
        return (row_off, idx[:tot], val[:tot]), dims
    common = int(dims[0]) if n and (dims == dims[0]).all() else 0
    return SparseRows(common, row_off, idx[:tot], val[:tot]), dims


def sparsevec_out(rows):
    """sparsevec_out (src/sparsevec.c:428-476) of every row: SparseRows give a list of str; device CSR
    ((row_off, idx, val) CUDA tensors, or a torch sparse CSR tensor) with rows.dim given as ((...), dim) gives device
    (text, offsets)."""
    from . import _after_torch
    lib = load()
    if isinstance(rows, tuple) and len(rows) == 2 and isinstance(rows[1], int):
        got = _device_csr(rows[0], rows[1])
        if got is not None:
            import torch
            n, dim, roff, idx, val = got
            out_off = torch.empty(n + 1, dtype=torch.int64, device=roff.device)
            _after_torch(roff, idx, val)
            _lib.check(lib.vb_sparsevec_to_text_batch_dev(dim, n, _tp(roff), _tp(idx), _tp(val), 0, _tp(out_off), None))
            out = torch.empty(max(int(out_off[-1]), 1), dtype=torch.uint8, device=roff.device)
            _lib.check(lib.vb_sparsevec_to_text_batch_dev(dim, n, _tp(roff), _tp(idx), _tp(val), int(out_off[-1]),
                                                          _tp(out_off), _tp(out)))
            return out[:int(out_off[-1])], out_off
    rows = _rows(rows)
    n = rows.n
    nnz = int(rows.row_off[-1] - rows.row_off[0])
    cap = 28 * nnz + 15 * n
    off = np.empty(n + 1, dtype=np.int64)
    out = np.empty(max(cap, 1), dtype=np.uint8)
    roff = np.ascontiguousarray(rows.row_off - rows.row_off[0])
    _lib.check(lib.vb_sparsevec_to_text_batch(rows.dim, n, _p(roff), _p(rows.idx[rows.row_off[0]:]),
                                              _p(rows.val[rows.row_off[0]:]), cap, _p(off), _p(out)))
    blob = out.tobytes()
    return [blob[off[i]:off[i + 1]].decode() for i in range(n)]


def sparsevec_recv(payloads, typmod=-1):
    """sparsevec_recv (src/sparsevec.c:514-562) of every field (a list of bytes, or a (CUDA uint8 payloads, CUDA int64
    offsets) pair), with sparsevec_in's return shapes.  The reference's errors, and PostgreSQL's for a short or
    overlong field, raise TextInputError (a ValueError) with .row."""
    from . import _after_torch, _ptr, _raise_text, _text_input
    lib = load()
    data, off, n, dev = _text_input(payloads)
    bad = C.c_int64(-1)
    if dev:
        import torch
        new = lambda k, dt: torch.empty(max(k, 1), dtype=dt, device=data.device)  # noqa: E731
        i32, i64, f32 = torch.int32, torch.int64, torch.float32
        fn = lib.vb_binary_to_sparsevec_batch_dev
        _after_torch(data, off)
    else:
        new = lambda k, dt: np.empty(max(k, 1), dtype=dt)  # noqa: E731
        i32, i64, f32 = np.int32, np.int64, np.float32
        fn = lib.vb_binary_to_sparsevec_batch
    row_off, dims = new(n + 1, i64), new(n, i32)
    row_off[:] = 0      # a refused argument writes no offsets
    rc = fn(typmod, n, _ptr(data), _ptr(off), 0, _ptr(dims), _ptr(row_off), None, None, C.byref(bad))
    tot = int(row_off[n])
    idx, val = new(tot, i32), new(tot, f32)
    if rc == _lib.EINVAL and tot > 0 and bad.value < 0:
        rc = fn(typmod, n, _ptr(data), _ptr(off), tot, _ptr(dims), _ptr(row_off), _ptr(idx), _ptr(val), C.byref(bad))
    _raise_text(rc, bad)
    dims = dims[:n]
    if dev:
        return (row_off, idx[:tot], val[:tot]), dims
    common = int(dims[0]) if n and (dims == dims[0]).all() else 0
    return SparseRows(common, row_off, idx[:tot], val[:tot]), dims


def sparsevec_send(rows):
    """sparsevec_send (src/sparsevec.c:567-585) of every row: SparseRows give a list of bytes; device CSR given as
    ((row_off, idx, val), dim) gives device (payloads, offsets).  Rows that break the CSR rules raise with the texts
    of sparsevec_out."""
    from . import _after_torch, synchronize
    lib = load()
    if isinstance(rows, tuple) and len(rows) == 2 and isinstance(rows[1], int):
        got = _device_csr(rows[0], rows[1])
        if got is not None:
            import torch
            n, dim, roff, idx, val = got
            out_off = torch.empty(n + 1, dtype=torch.int64, device=roff.device)
            _after_torch(roff, idx, val)
            _lib.check(lib.vb_sparsevec_to_binary_batch_dev(dim, n, _tp(roff), _tp(idx), _tp(val), 0, _tp(out_off), None))
            synchronize()
            total = int(out_off[-1])
            out = torch.empty(max(total, 1), dtype=torch.uint8, device=roff.device)
            _lib.check(lib.vb_sparsevec_to_binary_batch_dev(dim, n, _tp(roff), _tp(idx), _tp(val), total, _tp(out_off),
                                                            _tp(out)))
            synchronize()
            return out[:total], out_off
    rows = _rows(rows)
    n = rows.n
    nnz = int(rows.row_off[-1] - rows.row_off[0])
    cap = 12 * n + 8 * nnz
    off = np.empty(n + 1, dtype=np.int64)
    out = np.empty(max(cap, 1), dtype=np.uint8)
    roff = np.ascontiguousarray(rows.row_off - rows.row_off[0])
    _lib.check(lib.vb_sparsevec_to_binary_batch(rows.dim, n, _p(roff), _p(rows.idx[rows.row_off[0]:]),
                                                _p(rows.val[rows.row_off[0]:]), cap, _p(off), _p(out)))
    blob = out.tobytes()
    return [blob[off[i]:off[i + 1]] for i in range(n)]
