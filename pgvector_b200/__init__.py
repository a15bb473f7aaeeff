"""pgvector_b200 -- host-side mirror of pgvector's distance / index-scan interface
over libvecb200.so (hand-written sm_90a CUDA behind the C ABI of include/vecb200.h).

PostgreSQL is not available in this image, so the reference's C host code
(index AM callbacks) cannot be linked here; the extension-side glue is under
``pgvector_b200/ext`` (written against the PostgreSQL API) and this module is
the thin Python mirror of the same operator / opclass surface that the parity
tests and ``bench.py`` drive.  Names follow the reference: operators
(``l2_distance`` ... ``jaccard_distance``, src/vector.c:576-750,
src/bitvec.c:45-70), opclasses (``vector_l2_ops`` ..., sql/vector.sql:406-446,
819-911), ``IvfflatIndex`` (src/ivfscan.c) and ``HnswIndex`` (src/hnswscan.c).

Everything computes on the GPU through the C ABI; nothing here falls back to
numpy / torch math, and nothing imports the test oracle.
"""
from __future__ import annotations

import ctypes as C

import numpy as np

from . import _lib
from . import numeric as _numeric
from . import sparsevec  # noqa: F401  (sparsevec functions, CSR tables and the exact scan over them)
from ._lib import VecB200Error, load  # noqa: F401
from .sparsevec import SparseRows, SparseTable, SparseVector  # noqa: F401

VECTOR, HALFVEC, BIT = 0, 1, 2
L2_SQUARED, NEG_IP, COSINE, L1, HAMMING, JACCARD, L2, IP, SPHERICAL = range(9)

_NP = {VECTOR: np.float32, HALFVEC: np.uint16, BIT: np.uint8}
_TYPE_NAME = {VECTOR: "vector", HALFVEC: "halfvec", BIT: "bit"}

# opclass -> (element type, proc-1 metric the index evaluates, normalise rows/query?, k-means metric)
# (sql/vector.sql:406-446, 819-866, 894-911; SURVEY Appendix A)
OPCLASSES = {
    "vector_l2_ops": (VECTOR, L2_SQUARED, False, L2),
    "vector_ip_ops": (VECTOR, NEG_IP, False, SPHERICAL),
    "vector_cosine_ops": (VECTOR, NEG_IP, True, SPHERICAL),
    "vector_l1_ops": (VECTOR, L1, False, None),
    "halfvec_l2_ops": (HALFVEC, L2_SQUARED, False, L2),
    "halfvec_ip_ops": (HALFVEC, NEG_IP, False, SPHERICAL),
    "halfvec_cosine_ops": (HALFVEC, NEG_IP, True, SPHERICAL),
    "halfvec_l1_ops": (HALFVEC, L1, False, None),
    "bit_hamming_ops": (BIT, HAMMING, False, HAMMING),
    "bit_jaccard_ops": (BIT, JACCARD, False, None),
}


def init(device: int = 0):
    _lib.check(load().vb_init(device))


def stream_handle() -> int:
    """cudaStream_t of the library (int) -- wrap with torch.cuda.ExternalStream for event timing."""
    return int(load().vb_stream() or 0)


def launch_count() -> int:
    return int(load().vb_launch_count())


PROF_SCAN_ITEMS, PROF_SCAN_LISTS, PROF_TOPK, PROF_ASSIGN, PROF_HNSW, PROF_LIST_TC, PROF_CENTRE_TC = range(7)
# the phases of IvfflatIndex.build
PROF_BUILD_SAMPLE, PROF_BUILD_SEED, PROF_BUILD_LLOYD, PROF_BUILD_DEST, PROF_BUILD_PLACE, PROF_BUILD_ASSIGN = range(8, 14)


def prof_enable(on=True):
    _lib.check(load().vb_prof_enable(1 if on else 0))


def prof_read(kernel):
    """(total milliseconds, launches) of the bracketed kernel class since the last read."""
    ms, n = C.c_double(), C.c_int64()
    _lib.check(load().vb_prof_read(kernel, C.byref(ms), C.byref(n)))
    return ms.value, n.value


def synchronize():
    _lib.check(load().vb_synchronize())


def _after_torch(*tensors):
    """The library launches on its own non-blocking stream: before a call that reads torch CUDA tensors, make that
    stream wait for whatever torch's current stream has enqueued so far (the tensors' producers)."""
    if any(_is_torch(t) and t.is_cuda for t in tensors):
        import torch
        ev = torch.cuda.Event()
        ev.record(torch.cuda.current_stream())
        _lib.check(load().vb_stream_wait_event(C.c_void_p(ev.cuda_event)))


def _host(elem, a):
    """host array in the payload layout of the type.  halfvec rows are IEEE binary16 BIT PATTERNS (uint16): float16
    arrays are reinterpreted, float32/64 arrays are rounded to half (RNE, like the vector -> halfvec cast,
    src/halfvec.c:540-555, without its overflow check) -- never value-cast to integers."""
    a = np.asarray(a)
    if elem == HALFVEC and a.dtype != np.uint16:
        if a.dtype == np.float16:
            a = a.view(np.uint16)
        elif a.dtype in (np.float32, np.float64):
            with np.errstate(over="ignore"):
                a = a.astype(np.float16).view(np.uint16)
        else:
            raise TypeError(f"halfvec rows must be uint16 bit patterns or a float array, not {a.dtype}")
    return np.ascontiguousarray(a, dtype=_NP[elem])


def _ptr(a):
    if a is None:
        return None
    if isinstance(a, np.ndarray):
        return a.ctypes.data_as(C.c_void_p)
    return C.c_void_p(a.data_ptr())  # torch tensor


def _is_torch(a):
    return a is not None and not isinstance(a, np.ndarray) and hasattr(a, "data_ptr")


def _dim_of(elem, a, dim):
    if dim is not None:
        return int(dim)
    return int(a.shape[-1]) * (8 if elem == BIT else 1)


def _check_dims(elem, da, db):
    # CheckDims (src/vector.c:70-77, src/halfvec.c:74-81, src/bitvec.c:33-40)
    if da != db:
        kind = {VECTOR: "vector dimensions", HALFVEC: "halfvec dimensions", BIT: "bit lengths"}[elem]
        raise ValueError(f"different {kind} {da} and {db}")


# --------------------------------------------------------------------- operators

def distance_batch(elem, metric, q, rows, dim=None, q_dim=None):
    """float8 distances of one query against n rows (host arrays), as the fmgr wrapper returns them."""
    rows = _host(elem, rows)
    if rows.ndim == 1:
        rows = rows.reshape(1, -1)
    d = _dim_of(elem, rows, dim)
    if q is not None:
        q = _host(elem, q)
        _check_dims(elem, q_dim if q_dim is not None else _dim_of(elem, q, dim), d)
    out = np.empty(rows.shape[0], dtype=np.float64)
    _lib.check(load().vb_distance_batch(elem, metric, d, _ptr(q), _ptr(rows), rows.shape[0], _ptr(out)))
    return out


def l2_distance(a, rows, elem=VECTOR, **kw):
    return distance_batch(elem, L2, a, rows, **kw)


def l2_squared_distance(a, rows, elem=VECTOR, **kw):
    return distance_batch(elem, L2_SQUARED, a, rows, **kw)


def inner_product(a, rows, elem=VECTOR, **kw):
    return distance_batch(elem, IP, a, rows, **kw)


def negative_inner_product(a, rows, elem=VECTOR, **kw):
    return distance_batch(elem, NEG_IP, a, rows, **kw)


def cosine_distance(a, rows, elem=VECTOR, **kw):
    return distance_batch(elem, COSINE, a, rows, **kw)


def l1_distance(a, rows, elem=VECTOR, **kw):
    return distance_batch(elem, L1, a, rows, **kw)


def spherical_distance(a, rows, elem=VECTOR, **kw):
    return distance_batch(elem, SPHERICAL, a, rows, **kw)


def hamming_distance(a, rows, dim=None, **kw):
    return distance_batch(BIT, HAMMING, a, rows, dim=dim, **kw)


def jaccard_distance(a, rows, dim=None, **kw):
    return distance_batch(BIT, JACCARD, a, rows, dim=dim, **kw)


# --------------------------------------------------------------------- resident table / exact scan

AGG_AVG, AGG_SUM = 0, 1
# Rows per run of Table.avg / Table.sum.  The run kernel has one thread per (run, 128-byte column span of a row), so the
# runs of a table are its parallelism: at 1024 rows, 1M x 1536 fp32 rows are 977 runs x 1536 threads and 2M x 768
# halfvec rows 1954 runs x 384 threads, several waves of a full H100 each, every thread with the next 8 rows' loads in
# flight during its adds (2.3 TB/s for the fp32 shape on an H100 80GB HBM3 at 700 W, DESIGN.md section 5).  Shorter
# runs add run states to write and combine (one float8 per column per run, under 1 % of the rows' bytes here); the
# combine walks a group's runs serially, which stays short next to the row stream at this length.
DEFAULT_RUN_ROWS = 1024


class Table:
    """[n x dim] rows resident in HBM."""

    def __init__(self, elem, dim):
        self.elem, self.dim = elem, int(dim)
        h = C.c_void_p()
        _lib.check(load().vb_table_create(elem, self.dim, C.byref(h)))
        self.h = h

    def append(self, rows):
        if _is_torch(rows):
            _after_torch(rows)
            _lib.check(load().vb_table_append_dev(self.h, _ptr(rows), rows.shape[0]))
        else:
            rows = _host(self.elem, rows)
            _lib.check(load().vb_table_append(self.h, _ptr(rows), rows.shape[0]))
        return self

    def __len__(self):
        return int(load().vb_table_rows(self.h))

    def device_rows(self):
        """(device pointer of row 0, padded row stride in bytes): a read-only view of the resident rows"""
        stride = C.c_size_t()
        p = load().vb_table_device_rows(self.h, C.byref(stride))
        return int(p or 0), int(stride.value)

    def filter(self, rows):
        """a row Filter of this table: the allowed row numbers (numpy array, or a torch CUDA int64 tensor whose values
        outside [0, n) are ignored).  Rows appended later are not in it."""
        return Filter._create(self, "vb_table_filter_create", rows)

    def exact_topk(self, metric, queries, k, filter=None, filter_of_query=None):
        """ORDER BY v <op> q LIMIT k without an index (SURVEY 3.4).  filter: a Filter of this table (WHERE row IN ...),
        or a list of them with filter_of_query[q] = the index of query q's filter; each query then gets exactly what
        rerank() returns for its filter's rows in ascending order (k <= 2048)."""
        if filter is not None:
            return self._exact_topk_filtered(metric, queries, int(k), filter, filter_of_query)
        if _is_torch(queries):
            import torch
            nq = queries.shape[0]
            ids = torch.empty((nq, k), dtype=torch.int64, device=queries.device)
            dist = torch.empty((nq, k), dtype=torch.float32, device=queries.device)
            _after_torch(queries)
            _lib.check(load().vb_exact_topk_dev(self.h, metric, _ptr(queries), nq, k, _ptr(ids), _ptr(dist)))
            synchronize()   # the library runs on its own stream; results are handed back complete
            return ids, dist
        queries = _host(self.elem, queries)
        if queries.ndim == 1:
            queries = queries.reshape(1, -1)
        nq = queries.shape[0]
        ids = np.empty((nq, k), dtype=np.int64)
        dist = np.empty((nq, k), dtype=np.float64)
        _lib.check(load().vb_exact_topk(self.h, metric, _ptr(queries), nq, k, _ptr(ids), _ptr(dist)))
        return ids, dist

    def _exact_topk_filtered(self, metric, queries, k, filter, filter_of_query):
        farr, nf, fq = _filter_args(filter, filter_of_query)
        if _is_torch(queries):
            import torch
            nq = queries.shape[0]
            if fq is not None and len(fq) != nq:
                raise ValueError(f"filter_of_query must have {nq} entries, got {len(fq)}")
            queries = queries.contiguous()
            ids = torch.empty((nq, k), dtype=torch.int64, device=queries.device)
            dist = torch.empty((nq, k), dtype=torch.float32, device=queries.device)
            _after_torch(queries)
            _lib.check(load().vb_exact_topk_filtered_dev(self.h, metric, _ptr(queries), nq, k, farr, nf, _ptr(fq), _ptr(ids), _ptr(dist)))
            synchronize()   # the library runs on its own stream; results are handed back complete
            return ids, dist
        queries = _host(self.elem, queries)
        if queries.ndim == 1:
            queries = queries.reshape(1, -1)
        nq = queries.shape[0]
        if fq is not None and len(fq) != nq:
            raise ValueError(f"filter_of_query must have {nq} entries, got {len(fq)}")
        ids = np.empty((nq, k), dtype=np.int64)
        dist = np.empty((nq, k), dtype=np.float64)
        _lib.check(load().vb_exact_topk_filtered(self.h, metric, _ptr(queries), nq, k, farr, nf, _ptr(fq), _ptr(ids), _ptr(dist)))
        return ids, dist

    def rerank(self, metric, queries, candidates, k):
        """ORDER BY v <op> q LIMIT k over each query's own candidate rows: candidates[q] = row numbers of this table
        (-1 = none), typically what an index on a cheaper form of the vector returned (quantize-then-rerank).
        numpy inputs -> (int64 ids, float64 distances); torch CUDA tensors -> (int64 ids, float32 distances)."""
        k = int(k)
        raw = (self.dim + 7) // 8 if self.elem == BIT else self.dim
        if _is_torch(queries) or _is_torch(candidates):
            import torch
            if not (_is_torch(queries) and _is_torch(candidates) and queries.is_cuda and candidates.is_cuda):
                raise TypeError("rerank: queries and candidates must both be CUDA tensors or both host arrays")
            if queries.dim() != 2 or queries.shape[1] != raw:
                raise ValueError(f"rerank: queries must have shape [nq, {raw}], got {tuple(queries.shape)}")
            nq = queries.shape[0]
            if candidates.dtype != torch.int64 or candidates.dim() != 2 or candidates.shape[0] != nq:
                raise ValueError(f"rerank: candidates must be int64 of shape [{nq}, c], got {candidates.dtype} {tuple(candidates.shape)}")
            queries, candidates = queries.contiguous(), candidates.contiguous()
            ids = torch.empty((nq, k), dtype=torch.int64, device=queries.device)
            dist = torch.empty((nq, k), dtype=torch.float32, device=queries.device)
            _after_torch(queries, candidates)
            _lib.check(load().vb_table_rerank_dev(self.h, metric, _ptr(queries), nq, _ptr(candidates), candidates.shape[1], k,
                                                  _ptr(ids), _ptr(dist)))
            synchronize()   # the library runs on its own stream; results are handed back complete
            return ids, dist
        queries = _host(self.elem, queries)
        if queries.ndim == 1:
            queries = queries.reshape(1, -1)
        if queries.ndim != 2 or queries.shape[1] != raw:
            raise ValueError(f"rerank: queries must have shape [nq, {raw}], got {queries.shape}")
        nq = queries.shape[0]
        candidates = np.asarray(candidates)
        if candidates.dtype != np.int64 or candidates.ndim != 2 or candidates.shape[0] != nq:
            raise ValueError(f"rerank: candidates must be int64 of shape [{nq}, c], got {candidates.dtype} {candidates.shape}")
        candidates = np.ascontiguousarray(candidates)
        ids = np.empty((nq, k), dtype=np.int64)
        dist = np.empty((nq, k), dtype=np.float64)
        _lib.check(load().vb_table_rerank(self.h, metric, _ptr(queries), nq, _ptr(candidates), candidates.shape[1], k,
                                          _ptr(ids), _ptr(dist)))
        return ids, dist

    def avg(self, groups=None, ngroups=None, run_rows=DEFAULT_RUN_ROWS, state=False):
        """avg(v) of the rows, "GROUP BY" groups[i] (-1 = row left out; None = every row in one group): returns
        (values [G, dim] float32 / float16, counts [G]), plus the float8 transition state [G, dim + 1] = n, s_1 .. s_dim
        when state=True.  Each group's rows are aggregated in runs of run_rows consecutive rows whose states are combined
        left to right (0 = one run: the serial plan); the rounding depends on it as the reference's depends on its plan.
        numpy groups (or None) run the host variant and return numpy arrays; a torch CUDA int32 tensor runs the _dev
        variant and returns CUDA tensors.  A group with count 0 is the SQL NULL (its values are zero-filled)."""
        return self._aggregate(AGG_AVG, groups, ngroups, run_rows, state)

    def sum(self, groups=None, ngroups=None, run_rows=DEFAULT_RUN_ROWS):
        """sum(v) of the rows, as avg() groups and splits them: returns (values [G, dim], counts [G]).  An infinite
        element raises VecB200Error ("value out of range: overflow"), as float_overflow_error() does."""
        return self._aggregate(AGG_SUM, groups, ngroups, run_rows, False)

    def _aggregate(self, agg, groups, ngroups, run_rows, state):
        if self.elem not in (VECTOR, HALFVEC):
            raise ValueError(f"{_TYPE_NAME[self.elem]} has no aggregates")
        run_rows = int(run_rows)
        if groups is None:
            ngroups = 1 if ngroups is None else int(ngroups)
        elif ngroups is None:
            ngroups = max(1, int(groups.max()) + 1) if len(groups) else 1
        ngroups = int(ngroups)
        dim = self.dim
        if _is_torch(groups):
            import torch
            if not groups.is_cuda or groups.dtype != torch.int32 or groups.dim() != 1:
                raise TypeError("groups must be a 1-d int32 CUDA tensor or a host array")
            groups = groups.contiguous()
            dev = groups.device
            vals = torch.empty((ngroups, dim), dtype=torch.float32 if self.elem == VECTOR else torch.float16, device=dev)
            counts = torch.empty(ngroups, dtype=torch.int64, device=dev)
            st = torch.empty((ngroups, dim + 1), dtype=torch.float64, device=dev) if state else None
            _after_torch(groups)
            _lib.check(load().vb_table_aggregate_dev(self.h, agg, _ptr(groups), ngroups, run_rows, _ptr(vals), _ptr(counts), _ptr(st)))
            synchronize()   # the library runs on its own stream; results are handed back complete
        else:
            if groups is not None:
                groups = np.ascontiguousarray(groups, dtype=np.int32)
                if groups.shape != (len(self),):
                    raise ValueError(f"groups must have one entry per row ({len(self)}), got shape {groups.shape}")
            vals = np.empty((ngroups, dim), dtype=np.float32 if self.elem == VECTOR else np.float16)
            counts = np.empty(ngroups, dtype=np.int64)
            st = np.empty((ngroups, dim + 1), dtype=np.float64) if state else None
            _lib.check(load().vb_table_aggregate(self.h, agg, _ptr(groups), ngroups, run_rows, _ptr(vals), _ptr(counts), _ptr(st)))
        return (vals, counts, st) if state else (vals, counts)

    def order(self):
        """the rows in vector_ops / halfvec_ops btree order (ORDER BY v, DISTINCT v, GROUP BY v, WHERE v = / < ... $1)
        as an Order; rows appended later are not in it"""
        return Order._create(self, "vb_table_order_create", False)

    def exact_topk_sharded(self, metric, queries_dev, k, id_offset):
        """exact top-k over a row-sharded table (collective over the library's communicator); torch CUDA tensors"""
        import torch
        nq = queries_dev.shape[0]
        ids = torch.empty((nq, k), dtype=torch.int64, device=queries_dev.device)
        dist = torch.empty((nq, k), dtype=torch.float32, device=queries_dev.device)
        _after_torch(queries_dev)
        _lib.check(load().vb_exact_topk_sharded_dev(self.h, metric, _ptr(queries_dev), nq, k, int(id_offset), _ptr(ids), _ptr(dist)))
        synchronize()
        return ids, dist

    def free(self):
        if self.h:
            load().vb_table_free(self.h)
            self.h = None

    def __del__(self):
        try:
            self.free()
        except Exception:
            pass


# --------------------------------------------------------------------- IVFFlat

class IvfflatIndex:
    """Device image of an ivfflat index and its scan (src/ivfscan.c).

    ``probes`` mirrors the ivfflat.probes GUC (src/ivfflat.c:45-47).  For the cosine opclasses (``self.normalize``)
    the reference stores l2_normalize'd rows (src/ivfbuild.c:174-180) and normalises the query once per scan
    (src/ivfscan.c:222-229); this image takes rows and centres as stored, and ``prepare_query`` applies the
    query-side normalisation."""

    def __init__(self, opclass, dim, lists):
        self.opclass = opclass
        self.elem, self.metric, self.normalize, self.kmeans_metric = OPCLASSES[opclass]
        if self.metric not in (L2_SQUARED, NEG_IP, HAMMING):
            raise ValueError(f"operator class {opclass} is not supported by ivfflat")
        self.dim, self.lists = int(dim), int(lists)
        self.probes = 1  # IVFFLAT_DEFAULT_PROBES
        h = C.c_void_p()
        _lib.check(load().vb_ivf_create(self.elem, self.metric, self.dim, self.lists, C.byref(h)))
        self.h = h

    def load(self, centers, list_offsets, rows, ids=None):
        off = np.ascontiguousarray(list_offsets, dtype=np.int64)
        assert off.shape[0] == self.lists + 1
        self._off = off
        if _is_torch(rows):
            self._keep = (centers, rows, ids)
            _after_torch(centers, rows, ids)
            _lib.check(load().vb_ivf_load_dev(self.h, _ptr(centers), _ptr(off), _ptr(rows), _ptr(ids)))
        else:
            centers = _host(self.elem, centers)
            rows = _host(self.elem, rows)
            ids = None if ids is None else np.ascontiguousarray(ids, dtype=np.int64)
            _lib.check(load().vb_ivf_load(self.h, _ptr(centers), _ptr(off), _ptr(rows), _ptr(ids)))
        return self

    def prepare_query(self, q):
        """what ivfflatgettuple does to the ORDER BY value before the scan (src/ivfscan.c:213-231): l2_normalize for
        the cosine opclasses, identity otherwise."""
        return l2_normalize(q, self.elem) if self.normalize else q

    def load_by_list(self, centers, lists):
        """the same image loaded one list at a time: `lists` = iterable of (list number, rows, ids), ascending"""
        centers = _host(self.elem, centers)
        _lib.check(load().vb_ivf_begin_load(self.h, _ptr(centers)))
        off = np.zeros(self.lists + 1, dtype=np.int64)
        for l, rows, ids in lists:
            rows = _host(self.elem, rows)
            ids = np.ascontiguousarray(ids, dtype=np.int64)
            _lib.check(load().vb_ivf_load_list(self.h, int(l), _ptr(rows), _ptr(ids), rows.shape[0]))
            off[l + 1] = rows.shape[0]
        _lib.check(load().vb_ivf_end_load(self.h))
        self._off = np.concatenate([[0], np.cumsum(off[1:])]).astype(np.int64)
        return self

    def replace_list(self, l, rows, ids):
        """swap one list of the loaded image (what an insert into / a vacuum of that list needs)"""
        rows = _host(self.elem, rows)
        ids = np.ascontiguousarray(ids, dtype=np.int64)
        _lib.check(load().vb_ivf_replace_list(self.h, int(l), _ptr(rows), _ptr(ids), rows.shape[0]))
        delta = rows.shape[0] - int(self._off[l + 1] - self._off[l])
        self._off = self._off.copy()
        self._off[l + 1:] += delta
        return self

    def _device_rows(self, rows, n):
        """torch CUDA rows as the _dev entry points read them: [n, cols] of the element's width, contiguous"""
        width = {VECTOR: 4, HALFVEC: 2, BIT: 1}[self.elem]
        cols = self.dim if self.elem != BIT else (self.dim + 7) // 8
        if rows.element_size() != width or rows.dtype.is_complex or tuple(rows.reshape(n, -1).shape) != (n, cols):
            raise TypeError(f"device rows for {self.opclass} must be [n, {cols}] of {width}-byte elements, "
                            f"not {tuple(rows.shape)} {rows.dtype}")
        return rows.reshape(n, -1).contiguous()

    def build(self, rows, ids, seed=42, sample_rows=None, n_samples=None, first_row=None, u=None, max_iter=500, chunk_rows=None):
        """CREATE INDEX on the device (ivfflatbuild, src/ivfbuild.c): samples, k-means++, Lloyd, assign and placement of
        `rows` into a resident image, in one call.  Returns (lists, order, iters): the list of every row (int32 [n]; -1
        for a row of norm 0 under a cosine opclass, which is not indexed), the row number stored at every image row (int64
        [n], -1 past len(index)) and the Lloyd iterations run.  `sample_rows` (row numbers) or `n_samples` rows drawn from
        `seed` train the centres; `first_row` and `u` are the k-means++ draws, as kmeans_pp_init_draws takes them.  numpy
        rows are streamed from the host in chunks of `chunk_rows`; torch CUDA rows are read in place."""
        n = rows.shape[0] if rows.ndim > 1 else 1
        if (first_row is None) != (u is None):
            raise ValueError("first_row and u come together")
        opts = _lib.IvfBuildOpts(seed=int(seed), max_iter=int(max_iter), chunk_rows=int(chunk_rows or 0))
        if sample_rows is not None:
            sample_rows = np.ascontiguousarray(sample_rows, dtype=np.int64).reshape(-1)
            opts.sample_rows, opts.n_samples = sample_rows.ctypes.data, sample_rows.shape[0]
        elif n_samples is not None:
            opts.n_samples = int(n_samples)
        if u is not None:
            u = np.ascontiguousarray(u, dtype=np.float64).reshape(-1)
            if u.shape[0] < self.lists - 1:
                raise ValueError(f"u holds {u.shape[0]} draws, {self.lists - 1} are needed")
            opts.first_row, opts.u = int(first_row), u.ctypes.data
        lists = np.empty(n, dtype=np.int32)
        order = np.empty(n, dtype=np.int64)
        iters = C.c_int()
        if _is_torch(rows) and rows.is_cuda:
            import torch
            rows = self._device_rows(rows, n)
            if ids is not None:
                ids = torch.as_tensor(ids, device=rows.device).to(torch.int64).reshape(n).contiguous()
            _after_torch(rows, ids)
            fn = load().vb_ivf_build_dev
        else:
            if _is_torch(rows):
                rows = rows.numpy()
            if _is_torch(ids):
                ids = ids.cpu().numpy()
            rows = _host(self.elem, rows).reshape(n, -1)
            if rows.shape[1] != (self.dim if self.elem != BIT else (self.dim + 7) // 8):
                raise TypeError(f"rows for {self.opclass} of {self.dim} dimensions must not be {tuple(rows.shape)}")
            ids = None if ids is None else np.ascontiguousarray(ids, dtype=np.int64).reshape(n)
            fn = load().vb_ivf_build
        _lib.check(fn(self.h, _ptr(rows), _ptr(ids), n, 1 if self.normalize else 0, C.byref(opts), _ptr(lists), _ptr(order),
                      C.byref(iters)))
        self._refresh_offsets()
        return lists, order, iters.value

    def centers(self):
        """the centre table of the image, [lists] rows of the element type (what CreateListPages writes)"""
        cols = self.dim if self.elem != BIT else (self.dim + 7) // 8
        out = np.empty((self.lists, cols), dtype=_NP[self.elem])
        _lib.check(load().vb_ivf_centers(self.h, _ptr(out)))
        return out

    def __len__(self):
        return int(load().vb_ivf_rows(self.h))

    def insert(self, rows, ids):
        """INSERT into the resident image without reloading it (InsertTuple, src/ivfinsert.c:72-181, row after row):
        each row is appended to the list FindInsertPage picks.  Returns the lists (int32 [n]).  ids are the rows' heap
        ids.  Cosine opclasses: the rows are l2-normalised here, and a row of norm 0 is skipped with list -1, as
        IvfflatCheckNorm does.  torch CUDA rows take the device path, normalisation included (vector_norm and
        l2_normalize on the device); their ids are taken as int64 on the rows' device."""
        n = rows.shape[0] if rows.ndim > 1 else 1
        out = np.full(n, -1, dtype=np.int32)
        if _is_torch(rows) and rows.is_cuda:
            import torch
            rows = self._device_rows(rows, n)
            ids = torch.as_tensor(ids, device=rows.device).to(torch.int64).reshape(n).contiguous()
            keep = slice(None)
            if self.normalize:
                keep_dev = torch.nonzero(vector_norm(rows, self.elem) > 0).reshape(-1)
                rows = l2_normalize(rows[keep_dev], self.elem) if keep_dev.numel() else rows[keep_dev]
                ids = ids[keep_dev].contiguous()
                keep = keep_dev.cpu().numpy()
            got = np.empty(rows.shape[0], dtype=np.int32)
            _after_torch(rows, ids)
            _lib.check(load().vb_ivf_insert_dev(self.h, _ptr(rows), _ptr(ids), rows.shape[0], _ptr(got)))
            out[keep] = got
        else:
            if _is_torch(rows):
                rows = rows.cpu().numpy()
            if _is_torch(ids):
                ids = ids.cpu().numpy()
            rows = _host(self.elem, rows).reshape(n, -1)
            ids = np.ascontiguousarray(ids, dtype=np.int64).reshape(n)
            keep = slice(None)
            if self.normalize:
                keep = np.flatnonzero(vector_norm(rows, self.elem) > 0)
                rows = l2_normalize(rows[keep], self.elem) if keep.size else rows[keep]
                ids = np.ascontiguousarray(ids[keep])
            got = np.empty(rows.shape[0], dtype=np.int32)
            _lib.check(load().vb_ivf_insert(self.h, _ptr(np.ascontiguousarray(rows)), _ptr(ids), rows.shape[0], _ptr(got)))
            out[keep] = got
        self._refresh_offsets()
        return out

    def delete(self, ids):
        """VACUUM's ivfflatbulkdelete on the resident image: removes every row whose heap id is in `ids` (ids it does not
        hold are ignored); survivors keep their order.  Returns the number of rows removed (tuples_removed)."""
        ids = np.ascontiguousarray(ids, dtype=np.int64).reshape(-1)
        removed = C.c_int64(0)
        _lib.check(load().vb_ivf_delete(self.h, _ptr(ids), ids.shape[0], C.byref(removed)))
        self._refresh_offsets()
        return int(removed.value)

    def list_offsets(self):
        """the image's list offsets [lists + 1]"""
        off = np.empty(self.lists + 1, dtype=np.int64)
        _lib.check(load().vb_ivf_list_offsets(self.h, _ptr(off)))
        return off

    def _refresh_offsets(self):
        self._off = self.list_offsets()

    def scan_lists(self, queries, max_probes=None):
        """GetScanLists: nearest lists per query, ascending."""
        mp = int(max_probes or self.probes)
        if queries is None:
            nq, q = 1, None
        else:
            q = _host(self.elem, queries)
            if q.ndim == 1:
                q = q.reshape(1, -1)
            nq = q.shape[0]
        lists = np.empty((nq, mp), dtype=np.int32)
        dist = np.empty((nq, mp), dtype=np.float64)
        _lib.check(load().vb_ivf_scan_lists(self.h, _ptr(q), nq, mp, _ptr(lists), _ptr(dist)))
        return lists, dist

    def scan_items(self, q, lists, cap=None):
        """GetScanItems for one query: every row of `lists`, sorted by distance."""
        lists = np.ascontiguousarray(lists, dtype=np.int32)
        total = int(sum(self._off[l + 1] - self._off[l] for l in lists))
        cap = total if cap is None else min(int(cap), total)
        ids = np.empty(max(cap, 1), dtype=np.int64)
        dist = np.empty(max(cap, 1), dtype=np.float64)
        n = C.c_int64()
        qh = None if q is None else _host(self.elem, q)
        _lib.check(load().vb_ivf_scan_items(self.h, _ptr(qh), _ptr(lists), len(lists), cap, _ptr(ids), _ptr(dist), C.byref(n)))
        return ids[:cap], dist[:cap], int(n.value)

    def search(self, queries, k, probes=None, filter=None, filter_of_query=None):
        """first batch of ivfflatgettuple for many queries: k nearest of the probed lists.  filter: a Filter of this index,
        or a list of them with filter_of_query[q] = the index of query q's filter: each query then gets the first k of
        its unfiltered order over the probed lists that its filter allows (-1 / +inf padded), WHERE ... ORDER BY ... LIMIT k
        with ivfflat.iterative_scan = off."""
        p = int(probes or self.probes)
        if filter is not None:
            return self._search_filtered(queries, int(k), p, filter, filter_of_query)
        if _is_torch(queries):
            import torch
            nq = queries.shape[0]
            ids = torch.empty((nq, k), dtype=torch.int64, device=queries.device)
            dist = torch.empty((nq, k), dtype=torch.float32, device=queries.device)
            _after_torch(queries)
            _lib.check(load().vb_ivf_search_dev(self.h, _ptr(queries), nq, p, k, _ptr(ids), _ptr(dist)))
            synchronize()   # (search_into is the asynchronous variant)
            return ids, dist
        q = _host(self.elem, queries)
        if q.ndim == 1:
            q = q.reshape(1, -1)
        nq = q.shape[0]
        ids = np.empty((nq, k), dtype=np.int64)
        dist = np.empty((nq, k), dtype=np.float64)
        _lib.check(load().vb_ivf_search(self.h, _ptr(q), nq, p, k, _ptr(ids), _ptr(dist)))
        return ids, dist

    def _search_filtered(self, queries, k, p, filter, filter_of_query):
        farr, nf, fq = _filter_args(filter, filter_of_query)
        if _is_torch(queries):
            import torch
            nq = queries.shape[0]
            if fq is not None and len(fq) != nq:
                raise ValueError(f"filter_of_query must have {nq} entries, got {len(fq)}")
            queries = queries.contiguous()
            ids = torch.empty((nq, k), dtype=torch.int64, device=queries.device)
            dist = torch.empty((nq, k), dtype=torch.float32, device=queries.device)
            _after_torch(queries)
            _lib.check(load().vb_ivf_search_filtered_dev(self.h, _ptr(queries), nq, p, k, farr, nf, _ptr(fq), _ptr(ids), _ptr(dist)))
            synchronize()   # the library runs on its own stream; results are handed back complete
            return ids, dist
        q = _host(self.elem, queries)
        if q.ndim == 1:
            q = q.reshape(1, -1)
        nq = q.shape[0]
        if fq is not None and len(fq) != nq:
            raise ValueError(f"filter_of_query must have {nq} entries, got {len(fq)}")
        ids = np.empty((nq, k), dtype=np.int64)
        dist = np.empty((nq, k), dtype=np.float64)
        _lib.check(load().vb_ivf_search_filtered(self.h, _ptr(q), nq, p, k, farr, nf, _ptr(fq), _ptr(ids), _ptr(dist)))
        return ids, dist

    def filter(self, ids):
        """a row Filter of this index: the allowed heap ids as given at load (numpy array, or a torch CUDA int64
        tensor); ids the index does not hold are ignored.  It is refused once the index changes."""
        return Filter._create(self, "vb_ivf_filter_create", ids)

    def iterative_scan(self, queries, probes=None, max_probes=None, page=100, filter=None, filter_of_query=None):
        """ivfflat.iterative_scan = relaxed_order for a batch of queries: an IvfflatScan whose next_batch() returns the next
        page of every query's sequence (src/ivfscan.c:400-406).  probes / max_probes mirror ivfflat.probes /
        ivfflat.max_probes; max_probes defaults to probes (iterative_scan = off).  Cosine opclasses: pass
        prepare_query(queries).  filter: a Filter of this index, or a list of them with filter_of_query[q] = the index
        of query q's filter: each sequence is then the unfiltered one restricted to the ids its filter allows."""
        p = int(probes or self.probes)
        return IvfflatScan(self, queries, p, int(max_probes or p), int(page), filter=filter, filter_of_query=filter_of_query)

    def search_into(self, queries_dev, k, probes, ids_dev, dist_dev):
        """asynchronous device-resident search into preallocated torch tensors (bench inner loop): enqueued on the
        library stream after torch's current stream; the caller synchronises (pv.synchronize()) before reading."""
        _after_torch(queries_dev)
        _lib.check(load().vb_ivf_search_dev(self.h, _ptr(queries_dev), queries_dev.shape[0], int(probes), int(k),
                                            _ptr(ids_dev), _ptr(dist_dev)))

    def search_sharded_into(self, queries_dev, k, probes, ids_dev, dist_dev):
        """list-sharded search over the library's communicator (collective; every rank gets the full result)"""
        _after_torch(queries_dev)
        _lib.check(load().vb_ivf_search_sharded_dev(self.h, _ptr(queries_dev), queries_dev.shape[0], int(probes), int(k),
                                                    _ptr(ids_dev), _ptr(dist_dev)))

    def search_sharded_host_into(self, queries, k, probes, ids, dist):
        """list-sharded search, host buffers in and out (int64 ids, float64 distances)"""
        _lib.check(load().vb_ivf_search_sharded(self.h, _ptr(queries), queries.shape[0], int(probes), int(k), _ptr(ids), _ptr(dist)))

    def search_host_into(self, queries, k, probes, ids, dist):
        _lib.check(load().vb_ivf_search(self.h, _ptr(queries), queries.shape[0], int(probes), int(k), _ptr(ids), _ptr(dist)))

    def prefetch_queries(self, queries, slot):
        """start the H2D copy of the next batch (pinned host array) into slot 0 / 1; returns at once"""
        _lib.check(load().vb_ivf_prefetch_queries(self.h, _ptr(queries), queries.shape[0], int(slot)))

    def search_prefetched_into(self, slot, k, probes, ids, dist):
        """search the batch prefetched into `slot`; host outputs (int64 ids, float64 distances)"""
        _lib.check(load().vb_ivf_search_prefetched(self.h, int(slot), int(probes), int(k), _ptr(ids), _ptr(dist)))

    def last_scan_bytes(self):
        return int(load().vb_ivf_last_scan_bytes(self.h))

    def last_candidates(self):
        return int(load().vb_ivf_last_candidates(self.h))

    def tc_level0_fallbacks(self):
        """queries the int8 filter level could not certify (only they were searched again, from level 1 on)"""
        return int(load().vb_ivf_tc_level0_fallbacks(self.h))

    def tc_levelp_fallbacks(self):
        """queries the projection lower-bound level could not certify (only they were searched again, from level 0 on)"""
        return int(load().vb_ivf_tc_levelp_fallbacks(self.h))

    def tc_level1_fallbacks(self):
        """queries the hi-plane-only filter level could not certify (their batches were repeated with both planes)"""
        return int(load().vb_ivf_tc_level1_fallbacks(self.h))

    def tc_fallbacks(self):
        """queries re-run exactly because the tensor-core filter could not certify them (scan_impl = 4)"""
        return int(load().vb_ivf_tc_fallbacks(self.h))

    def free(self):
        if self.h:
            load().vb_ivf_free(self.h)
            self.h = None

    def __del__(self):
        try:
            self.free()
        except Exception:
            pass


class IvfflatScan:
    """One ivfflat iterative index scan per query (src/ivfscan.c:360-414): next_batch() returns (ids, distances, counts) of
    the next <= page elements of every query, nearest first within a group of `probes` lists; counts == 0 marks an
    exhausted scan.  Close it (or use it as a context manager) before the index changes or is freed."""

    def __init__(self, index, queries, probes, max_probes, page, filter=None, filter_of_query=None):
        q = None if queries is None else _host(index.elem, queries)   # (NULL queries: the library refuses them)
        if q is not None and q.ndim == 1:
            q = q.reshape(1, -1)
        self.index, self.page = index, page
        self.nq = 0 if q is None else q.shape[0]
        self.h = None
        h = C.c_void_p()
        if filter is None:
            _lib.check(load().vb_ivf_scan_begin(index.h, _ptr(q), self.nq, probes, max_probes, page, C.byref(h)))
        else:
            farr, nf, fq = _filter_args(filter, filter_of_query)
            if fq is not None and len(fq) != self.nq:
                raise ValueError(f"filter_of_query must have {self.nq} entries, got {len(fq)}")
            _lib.check(load().vb_ivf_scan_begin_filtered(index.h, _ptr(q), self.nq, probes, max_probes, page, farr, nf, _ptr(fq),
                                                         C.byref(h)))
        self.h = h

    def next_batch(self):
        ids = np.empty((self.nq, self.page), dtype=np.int64)
        dist = np.empty((self.nq, self.page), dtype=np.float64)
        cnt = np.empty(self.nq, dtype=np.int32)
        _lib.check(load().vb_ivf_scan_next(self.h, _ptr(ids), _ptr(dist), _ptr(cnt)))
        return ids, dist, cnt

    def lists_done(self):
        """per query, the lists scanned so far (the reference's listIndex)"""
        out = np.empty(self.nq, dtype=np.int32)
        _lib.check(load().vb_ivf_scan_lists_done(self.h, _ptr(out)))
        return out

    def tuples_of(self, query=0, limit=None):
        """what ivfflatgettuple hands the executor for one query, in order: (heap id, distance) pairs"""
        out = []
        while limit is None or len(out) < limit:
            ids, dist, cnt = self.next_batch()
            if cnt[query] == 0:
                break
            out.extend((int(ids[query, j]), float(dist[query, j])) for j in range(int(cnt[query])))
        return out if limit is None else out[:limit]

    def close(self):
        if self.h:
            load().vb_ivf_scan_end(self.h)
            self.h = None

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


# --------------------------------------------------------------------- row filters

class Filter:
    """A row filter: the allowed rows of one Table (row numbers), one IvfflatIndex (heap ids) or one HnswIndex (element
    numbers), resident on the device -- what a B-tree or bitmap scan on a filter column yields for WHERE <predicate>
    ORDER BY v <op> q LIMIT k.  Made by Table.filter / IvfflatIndex.filter / HnswIndex.filter; len() = rows allowed.
    Free it (or use it as a context manager) when done."""

    def __init__(self, owner, h):
        self.owner, self.h = owner, h

    @classmethod
    def _create(cls, owner, fn, rows):
        h = C.c_void_p()
        if _is_torch(rows):
            import torch
            if not rows.is_cuda or rows.dtype != torch.int64 or rows.dim() != 1:
                raise TypeError("filter: a tensor of rows must be a 1-d int64 CUDA tensor")
            rows = rows.contiguous()
            _after_torch(rows)
            _lib.check(getattr(load(), fn + "_dev")(owner.h, _ptr(rows), rows.shape[0], C.byref(h)))
        else:
            rows = np.ascontiguousarray(rows, dtype=np.int64).reshape(-1)
            _lib.check(getattr(load(), fn)(owner.h, _ptr(rows), rows.shape[0], C.byref(h)))
        return cls(owner, h)

    def __len__(self):
        return int(load().vb_filter_rows(self.h)) if self.h else 0

    def free(self):
        if self.h:
            load().vb_filter_free(self.h)
            self.h = None

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.free()

    def __del__(self):
        try:
            self.free()
        except Exception:
            pass


class Order:
    """The rows of one Table or SparseTable in the order of its btree operator class (vector_ops, halfvec_ops,
    sparsevec_ops), ties by ascending row number, with the groups of equal rows: perm [n] (row numbers in order),
    group_of_row [n] (dense rank of each row's value, what Table.avg / Table.sum take as groups), group_start
    [groups + 1] (position in perm of each group's first row, then n).  bounds(queries) -> (lo, hi): the rows equal to
    query q are perm[lo[q]:hi[q]].  Made by Table.order / SparseTable.order; free it (or use it as a context manager)
    when done."""

    def __init__(self, owner, h, sparse):
        self.owner, self.h, self.sparse = owner, h, sparse

    @classmethod
    def _create(cls, owner, fn, sparse):
        h = C.c_void_p()
        _lib.check(getattr(load(), fn)(owner.h, C.byref(h)))
        return cls(owner, h, sparse)

    @property
    def rows(self):
        """rows ordered: the table's row count when the order was made"""
        return int(load().vb_order_rows(self.h))

    @property
    def groups(self):
        return int(load().vb_order_groups(self.h))

    @property
    def passes(self):
        """refinement passes the sort took"""
        return int(load().vb_order_passes(self.h))

    def read(self, device=False):
        """(perm int64 [n], group_of_row int32 [n], group_start int64 [groups + 1]): numpy arrays, or CUDA tensors with
        device=True"""
        n, g = self.rows, self.groups
        if device:
            import torch
            perm = torch.empty(n, dtype=torch.int64, device="cuda")
            gor = torch.empty(n, dtype=torch.int32, device="cuda")
            gst = torch.empty(g + 1, dtype=torch.int64, device="cuda")
            _lib.check(load().vb_order_read_dev(self.h, _ptr(perm), _ptr(gor), _ptr(gst)))
            synchronize()   # the library runs on its own stream; results are handed back complete
            return perm, gor, gst
        perm = np.empty(n, dtype=np.int64)
        gor = np.empty(n, dtype=np.int32)
        gst = np.empty(g + 1, dtype=np.int64)
        _lib.check(load().vb_order_read(self.h, _ptr(perm), _ptr(gor), _ptr(gst)))
        return perm, gor, gst

    @property
    def perm(self):
        out = np.empty(self.rows, dtype=np.int64)
        _lib.check(load().vb_order_read(self.h, _ptr(out), None, None))
        return out

    @property
    def group_of_row(self):
        out = np.empty(self.rows, dtype=np.int32)
        _lib.check(load().vb_order_read(self.h, None, _ptr(out), None))
        return out

    @property
    def group_start(self):
        out = np.empty(self.groups + 1, dtype=np.int64)
        _lib.check(load().vb_order_read(self.h, None, None, _ptr(out)))
        return out

    def bounds(self, queries):
        """(lo, hi) per query: the number of ordered rows < q and <= q.  Dense orders take rows of the table's type (numpy,
        or a CUDA tensor of float32 / float16 rows, which returns CUDA tensors); sparse orders take SparseRows /
        SparseVectors or device CSR, as SparseTable.exact_topk does."""
        if self.sparse:
            return sparsevec._order_bounds(self, queries)
        t = self.owner
        if _is_torch(queries):
            import torch
            want = torch.float32 if t.elem == VECTOR else torch.float16
            q = queries.reshape(1, -1) if queries.dim() == 1 else queries
            if not q.is_cuda or q.dtype != want or q.dim() != 2 or q.shape[1] != t.dim:
                raise ValueError(f"bounds: queries must be a {want} CUDA tensor of shape [nq, {t.dim}]")
            q = q.contiguous()
            nq = q.shape[0]
            lo = torch.empty(nq, dtype=torch.int64, device=q.device)
            hi = torch.empty(nq, dtype=torch.int64, device=q.device)
            _after_torch(q)
            _lib.check(load().vb_order_bounds_dev(self.h, _ptr(q), nq, _ptr(lo), _ptr(hi)))
            synchronize()   # the library runs on its own stream; results are handed back complete
            return lo, hi
        q = _host(t.elem, queries)
        if q.ndim == 1:
            q = q.reshape(1, -1)
        if q.ndim != 2 or q.shape[1] != t.dim:
            raise ValueError(f"bounds: queries must have shape [nq, {t.dim}], got {q.shape}")
        nq = q.shape[0]
        lo = np.empty(nq, dtype=np.int64)
        hi = np.empty(nq, dtype=np.int64)
        _lib.check(load().vb_order_bounds(self.h, _ptr(q), nq, _ptr(lo), _ptr(hi)))
        return lo, hi

    def free(self):
        if self.h:
            load().vb_order_free(self.h)
            self.h = None

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.free()

    def __del__(self):
        try:
            self.free()
        except Exception:
            pass


def _filter_args(filter, filter_of_query):
    """(C array of filter handles, count, int32 filter_of_query or None) for the filtered entry points"""
    filters = [filter] if isinstance(filter, Filter) else list(filter)
    if not filters or any(not isinstance(f, Filter) or not f.h for f in filters):
        raise ValueError("filter: a Filter, or a non-empty list of live Filters")
    if filter_of_query is None and len(filters) > 1:
        raise ValueError("filter_of_query is required with more than one filter")
    fq = None if filter_of_query is None else np.ascontiguousarray(filter_of_query, dtype=np.int32).reshape(-1)
    arr = (C.c_void_p * len(filters))(*[f.h.value for f in filters])
    return arr, len(filters), fq


# --------------------------------------------------------------------- IVFFlat build

def make_allreduce(fn):
    """wrap a python callable (ptr, count, dtype_code) -> None as the C hook."""
    def _cb(buf, count, dtype, _ctx):
        try:
            fn(buf, count, dtype)
            return 0
        except Exception:  # pragma: no cover - surfaced as VB error
            return -1
    return _lib.ALLREDUCE_FN(_cb)


def kmeans(samples: Table, kmeans_metric, init_centers, max_iter=500, seed=42, allreduce=None):
    """IvfflatKmeans (src/ivfkmeans.c:553-570) from given initial centres."""
    centers = _host(samples.elem, init_centers).copy()
    k = centers.shape[0]
    iters = C.c_int()
    cb = make_allreduce(allreduce) if allreduce is not None else None
    _lib.check(load().vb_kmeans(samples.h, kmeans_metric, _ptr(centers), k, max_iter, seed,
                                C.cast(cb, C.c_void_p) if cb is not None else None, None, C.byref(iters)))
    return centers, iters.value


def kmeans_pp_init(samples: Table, kmeans_metric, k, seed=42):
    raw = (samples.dim + 7) // 8 if samples.elem == BIT else samples.dim
    centers = np.empty((k, raw), dtype=_NP[samples.elem])
    _lib.check(load().vb_kmeans_pp_init(samples.h, kmeans_metric, _ptr(centers), k, seed))
    return centers


def kmeans_pp_stats():
    """(skipped by the triangle rule, stopped by the bf16 bound, re-scored exactly) of the last k-means++ seeding"""
    out = np.zeros(3, dtype=np.int64)
    _lib.check(load().vb_kmeans_pp_stats(_ptr(out)))
    return tuple(int(x) for x in out)


def kmeans_pp_init_draws(samples: Table, kmeans_metric, k, first_row, u):
    """InitCenters (src/ivfkmeans.c:23-91) with the caller's draws; returns (centres, picked sample rows)."""
    raw = (samples.dim + 7) // 8 if samples.elem == BIT else samples.dim
    centers = np.empty((k, raw), dtype=_NP[samples.elem])
    u = np.ascontiguousarray(u, dtype=np.float64)
    picked = np.empty(k, dtype=np.int64)
    _lib.check(load().vb_kmeans_pp_init_draws(samples.h, kmeans_metric, _ptr(centers), k, int(first_row), _ptr(u), _ptr(picked)))
    return centers, picked


def assign(rows: Table, metric, centers):
    """AddTupleToSort's nearest-centre pass (src/ivfbuild.c:161-219)."""
    if _is_torch(centers):
        import torch
        out = torch.empty(len(rows), dtype=torch.int32, device=centers.device)
        _after_torch(centers)
        _lib.check(load().vb_assign_dev(rows.h, metric, _ptr(centers), centers.shape[0], _ptr(out)))
        return out
    centers = _host(rows.elem, centers)
    out = np.empty(len(rows), dtype=np.int32)
    _lib.check(load().vb_assign(rows.h, metric, _ptr(centers), centers.shape[0], _ptr(out)))
    return out


# --------------------------------------------------------------------- HNSW

# one change record of HnswIndex.insert (vb_hnsw_slot)
HNSW_SLOT_DTYPE = np.dtype([("element", np.int32), ("layer", np.int32), ("slot", np.int32), ("neighbor", np.int32)])


class HnswIndex:
    """Device image of an hnsw index and its scan (src/hnswscan.c, src/hnswutils.c:824-987).

    ``ef_search`` mirrors the hnsw.ef_search GUC (src/hnsw.c:93-95)."""

    def __init__(self, opclass, dim, m=16):
        self.opclass = opclass
        self.elem, self.metric, self.normalize, _ = OPCLASSES[opclass]
        self.dim, self.m = int(dim), int(m)
        self.ef_search = 40  # HNSW_DEFAULT_EF_SEARCH
        h = C.c_void_p()
        _lib.check(load().vb_hnsw_create(self.elem, self.metric, self.dim, self.m, C.byref(h)))
        self.h = h

    def load(self, rows, levels, nbr0, upper_off, upper, entry):
        rows = _host(self.elem, rows)
        levels = np.ascontiguousarray(levels, dtype=np.int32)
        nbr0 = np.ascontiguousarray(nbr0, dtype=np.int32)
        upper_off = np.ascontiguousarray(upper_off, dtype=np.int64)
        upper = np.ascontiguousarray(upper, dtype=np.int32)
        slots = upper.shape[0] if upper.size else 0
        self.n = rows.shape[0]
        _lib.check(load().vb_hnsw_load(self.h, _ptr(rows), rows.shape[0], _ptr(levels), _ptr(nbr0), _ptr(upper_off),
                                       _ptr(upper) if slots else None, slots, int(entry)))
        return self

    def build(self, rows, ef_construction=64, seed=42, levels=None):
        """CREATE INDEX on the device (src/hnswbuild.c:437-480 in batches): row i becomes element i."""
        lv = None if levels is None else np.ascontiguousarray(levels, dtype=np.int32)
        if _is_torch(rows):
            _after_torch(rows)
            self.n = rows.shape[0]
            _lib.check(load().vb_hnsw_build_dev(self.h, _ptr(rows), self.n, int(ef_construction), int(seed), _ptr(lv)))
        else:
            rows = _host(self.elem, rows)
            self.n = rows.shape[0]
            _lib.check(load().vb_hnsw_build(self.h, _ptr(rows), self.n, int(ef_construction), int(seed), _ptr(lv)))
        return self

    def insert(self, rows, ef_construction=64, seed=42, levels=None):
        """INSERT into the resident image (batched HnswInsertTupleOnDisk, src/hnswinsert.c:696-743): row i becomes
        element n_old + i.  Returns (dup_of [n], the element each row was folded into or -1; the change records, a
        structured array of (element, layer, slot, neighbor) sorted by (element, layer, slot): every neighbour-array
        slot whose value changed, with its new value)."""
        lv = None if levels is None else np.ascontiguousarray(levels, dtype=np.int32)
        nchg = C.c_int64(0)
        if _is_torch(rows):
            _after_torch(rows)
            n = rows.shape[0]
            dup = np.empty(n, dtype=np.int32)
            _lib.check(load().vb_hnsw_insert_dev(self.h, _ptr(rows), n, int(ef_construction), int(seed), _ptr(lv), _ptr(dup),
                                                 C.byref(nchg)))
        else:
            rows = _host(self.elem, rows)
            if rows.ndim == 1:
                rows = rows.reshape(1, -1)
            n = rows.shape[0]
            dup = np.empty(n, dtype=np.int32)
            _lib.check(load().vb_hnsw_insert(self.h, _ptr(rows), n, int(ef_construction), int(seed), _ptr(lv), _ptr(dup),
                                             C.byref(nchg)))
        self.n = int(load().vb_hnsw_rows(self.h))
        return dup, self.changes(int(nchg.value))

    def vacuum(self, counts, ef_construction=64):
        """VACUUM's graph work on the resident image (hnswbulkdelete after RemoveHeapTids, src/hnswvacuum.c): counts
        [n] are the heap TIDs each element keeps (0..10; 0 = deleted now or by an earlier vacuum).  Elements that link to
        a deleted one are repaired, the entry point is replaced when it is deleted, and deleted elements lose every
        neighbour; their numbers are not reused.  Returns (the change records, as insert() returns them; the number of
        elements repaired)."""
        counts = np.ascontiguousarray(counts, dtype=np.int32)
        n = int(load().vb_hnsw_rows(self.h))
        if counts.shape != (n,):
            raise ValueError(f"counts must have {n} entries, got {counts.shape}")
        nrep, nchg = C.c_int64(0), C.c_int64(0)
        _lib.check(load().vb_hnsw_vacuum(self.h, _ptr(counts), int(ef_construction), C.byref(nrep), C.byref(nchg)))
        return self.changes(int(nchg.value)), int(nrep.value)

    def changes(self, count):
        """the last insert's or vacuum's change records (count = the number it reported)"""
        out = np.empty(count, dtype=HNSW_SLOT_DTYPE)
        _lib.check(load().vb_hnsw_insert_changes(self.h, _ptr(out), count))
        return out

    def set_heaptid_counts(self, counts):
        """heap TIDs per element as the pages hold them (0..10; 0 = being deleted): they drive the insert's
        RemoveElements, its preference for deleted neighbours and duplicate folding"""
        counts = np.ascontiguousarray(counts, dtype=np.int32)
        n = int(load().vb_hnsw_rows(self.h))
        if counts.shape != (n,):
            raise ValueError(f"counts must have {n} entries, got {counts.shape}")
        _lib.check(load().vb_hnsw_set_heaptid_counts(self.h, _ptr(counts)))

    def export(self):
        """the graph as arrays (the layout load() takes, plus dup_of): what the page writer consumes"""
        n, m = int(load().vb_hnsw_rows(self.h)), self.m
        slots = int(load().vb_hnsw_upper_slots(self.h))
        levels = np.empty(n, dtype=np.int32)
        nbr0 = np.empty((n, 2 * m), dtype=np.int32)
        upper_off = np.empty(n, dtype=np.int64)
        upper = np.full((max(slots, 1), m), -1, dtype=np.int32)
        dup_of = np.empty(n, dtype=np.int32)
        entry = C.c_int64(-1)
        _lib.check(load().vb_hnsw_export(self.h, _ptr(levels), _ptr(nbr0), _ptr(upper_off), _ptr(upper), C.byref(entry), _ptr(dup_of)))
        e = int(entry.value)
        return dict(levels=levels, nbr0=nbr0, upper_off=upper_off, upper=upper[:slots], entry=e,
                    entry_level=int(levels[e]) if e >= 0 else -1, m=m, dup_of=dup_of)

    def search(self, queries, k=None, ef_search=None):
        ef = int(ef_search or self.ef_search)
        k = int(k or ef)
        q = _host(self.elem, queries)
        if q.ndim == 1:
            q = q.reshape(1, -1)
        nq = q.shape[0]
        ids = np.empty((nq, k), dtype=np.int64)
        dist = np.empty((nq, k), dtype=np.float64)
        nd = np.empty(nq, dtype=np.int64)
        _lib.check(load().vb_hnsw_search(self.h, _ptr(q), nq, ef, k, _ptr(ids), _ptr(dist), _ptr(nd)))
        return ids, dist, nd

    def search_into(self, queries_dev, k, ef, ids_dev, dist_dev, nd_dev=None):
        _after_torch(queries_dev)
        _lib.check(load().vb_hnsw_search_dev(self.h, _ptr(queries_dev), queries_dev.shape[0], int(ef), int(k),
                                             _ptr(ids_dev), _ptr(dist_dev), _ptr(nd_dev)))

    def filter(self, elements):
        """an element Filter of this index: the allowed element numbers (numpy array, or a torch CUDA int64 tensor whose
        values outside [0, n) are ignored).  It is refused once the index is loaded or built again."""
        return Filter._create(self, "vb_hnsw_filter_create", elements)

    def iterative_scan(self, queries, ef_search=None, max_scan_tuples=20000, filter=None, filter_of_query=None, page=None):
        """hnsw.iterative_scan for a batch of queries: an HnswScan whose next_batch() mirrors ResumeScanItems
        (src/hnswscan.c:62-87); max_scan_tuples mirrors hnsw.max_scan_tuples (src/hnsw.c:101-105).  filter: a Filter of
        this index, or a list of them with filter_of_query[q] = the index of query q's filter: next_batch() then returns
        the next `page` (default ef_search) elements of each query's sequence that its filter allows."""
        ef = int(ef_search or self.ef_search)
        if filter is None and page is not None:
            raise ValueError("page applies to a filtered scan only (an unfiltered scan returns ef_search per batch)")
        return HnswScan(self, queries, ef, int(max_scan_tuples), filter=filter, filter_of_query=filter_of_query,
                        page=ef if page is None else int(page))

    def free(self):
        if self.h:
            load().vb_hnsw_free(self.h)
            self.h = None

    def __del__(self):
        try:
            self.free()
        except Exception:
            pass


class HnswScan:
    """One iterative index scan per query (src/hnswscan.c:228-340): next_batch() returns (ids, distances, counts) of
    the next <= ef_search elements of every query, nearest first; counts == 0 marks an exhausted scan.  With a filter,
    the next <= page allowed elements, counts < page only once the sequence is exhausted."""

    def __init__(self, index, queries, ef, max_scan_tuples, filter=None, filter_of_query=None, page=None):
        q = _host(index.elem, queries)
        if q.ndim == 1:
            q = q.reshape(1, -1)
        self.index, self.nq, self.ef = index, q.shape[0], ef
        self.h = None
        h = C.c_void_p()
        if filter is None:
            self.width = ef
            _lib.check(load().vb_hnsw_scan_begin(index.h, _ptr(q), self.nq, ef, max_scan_tuples, C.byref(h)))
        else:
            self.width = int(page)
            farr, nf, fq = _filter_args(filter, filter_of_query)
            if fq is not None and len(fq) != self.nq:
                raise ValueError(f"filter_of_query must have {self.nq} entries, got {len(fq)}")
            _lib.check(load().vb_hnsw_scan_begin_filtered(index.h, _ptr(q), self.nq, ef, max_scan_tuples, self.width, farr, nf,
                                                          _ptr(fq), C.byref(h)))
        self.h = h

    def next_batch(self):
        ids = np.empty((self.nq, self.width), dtype=np.int64)
        dist = np.empty((self.nq, self.width), dtype=np.float64)
        cnt = np.empty(self.nq, dtype=np.int32)
        _lib.check(load().vb_hnsw_scan_next(self.h, _ptr(ids), _ptr(dist), _ptr(cnt)))
        return ids, dist, cnt

    def tuples(self):
        t = np.empty(self.nq, dtype=np.int64)
        _lib.check(load().vb_hnsw_scan_tuples(self.h, _ptr(t)))
        return t

    def tuples_of(self, query=0, strict=False, limit=None):
        """what hnswgettuple hands the executor for one query, in order: (element, distance) pairs; strict mirrors
        hnsw.iterative_scan = strict_order (elements nearer than one already returned are skipped, :316-322)"""
        out = []
        prev = -np.inf
        while limit is None or len(out) < limit:
            ids, dist, cnt = self.next_batch()
            if cnt[query] == 0:
                break
            for j in range(int(cnt[query])):
                d = float(dist[query, j])
                if strict:
                    if d < prev:
                        continue
                    prev = d
                out.append((int(ids[query, j]), d))
        return out if limit is None else out[:limit]

    def close(self):
        if self.h:
            load().vb_hnsw_scan_end(self.h)
            self.h = None

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


# --------------------------------------------------------------------- communicator (one process per GPU)

def comm_unique_id() -> bytes:
    """the 128-byte NCCL id one rank creates and the host hands to the others"""
    buf = C.create_string_buffer(128)
    _lib.check(load().vb_comm_unique_id(buf, 128))
    return buf.raw


def comm_init(id_bytes: bytes, rank: int, world: int):
    """collective: create the library's own NCCL communicator on its device"""
    _lib.check(load().vb_comm_init(C.c_char_p(id_bytes), int(rank), int(world)))


def comm_free():
    _lib.check(load().vb_comm_free())


def comm_world() -> int:
    return int(load().vb_comm_world())


def tc_traffic(on=True, read=False):
    """traffic accounting of the tensor-core filter launches; read=True returns and resets the 8 counters"""
    out = np.zeros(8, dtype=np.int64) if read else None
    _lib.check(load().vb_ivf_tc_traffic(1 if on else 0, _ptr(out)))
    return out


def tc_level0_rescored():
    """read and reset the level-0 refine's counters, kept while tc_traffic is on: [rows re-scored exactly, rows the
    global bound would have re-scored, queries refined]"""
    out = np.zeros(3, dtype=np.int64)
    _lib.check(load().vb_ivf_tc_level0_rescored(_ptr(out)))
    return out


def set_tensor_cores(on: bool):
    """False forces the exact fp32 CUDA-core assign kernel (parity tests); True (default) uses the tensor cores (wgmma)."""
    _lib.check(load().vb_set_tensor_cores(1 if on else 0))


def last_assign_rechecked() -> int:
    return int(load().vb_last_assign_rechecked())


def set_option(name: str, value: int):
    """tuning switches of the library: "scan_impl" (0 = LDG kernel, 1 = bulk-copy/TMA kernel), "tensor_cores"."""
    _lib.check(load().vb_set_option(name.encode(), int(value)))


# --------------------------------------------------------------------- row transforms
#
# numpy rows run the host variants and return numpy arrays (halfvec: uint16 bit patterns).  torch CUDA rows run the _dev
# variants, which read the rows where they are, and return CUDA tensors: norms float64, vector rows float32, halfvec rows
# float16 (any 2-byte dtype is read as binary16 bit patterns), bit rows uint8 [n, (dim + 7) // 8].

def _is_cuda(a):
    return _is_torch(a) and a.is_cuda


def _dev_rows(rows, elem):
    """torch CUDA rows as the _dev transforms read them: (2-d contiguous rows, whether a single row was given)"""
    import torch
    if elem == VECTOR and rows.dtype != torch.float32:
        raise TypeError(f"vector rows on the device must be float32, not {rows.dtype}")
    if elem == HALFVEC and (rows.element_size() != 2 or rows.dtype.is_complex):
        raise TypeError(f"halfvec rows on the device must have a 2-byte dtype, not {rows.dtype}")
    if elem not in (VECTOR, HALFVEC):
        raise ValueError(f"elem must be VECTOR or HALFVEC, not {elem}")
    single = rows.dim() == 1
    r2 = rows.reshape(1, -1) if single else rows
    if r2.dim() != 2:
        raise ValueError(f"rows must be 1-d or 2-d, got shape {tuple(rows.shape)}")
    return r2.contiguous(), single


def _dev_call(fn, *args, inputs=()):
    """a _dev transform after torch's pending work on its inputs; the results are complete when it returns"""
    _after_torch(*inputs)
    _lib.check(fn(*args))
    synchronize()   # the library runs on its own stream; results are handed back complete


def vector_norm(rows, elem=VECTOR):
    """vector_norm / l2_norm of every row (src/vector.c:767-780, src/halfvec.c:703-720)."""
    if _is_cuda(rows):
        import torch
        r2, single = _dev_rows(rows, elem)
        out = torch.empty(r2.shape[0], dtype=torch.float64, device=r2.device)
        _dev_call(load().vb_norm_batch_dev, elem, r2.shape[1], _ptr(r2), r2.shape[0], _ptr(out), inputs=(r2,))
        return out[0] if single else out
    rows = _host(elem, rows)
    single = rows.ndim == 1
    r2 = rows.reshape(1, -1) if single else rows
    out = np.empty(r2.shape[0], dtype=np.float64)
    _lib.check(load().vb_norm_batch(elem, r2.shape[1], _ptr(r2), r2.shape[0], _ptr(out)))
    return out[0] if single else out


def l2_normalize(rows, elem=VECTOR):
    """l2_normalize of every row (src/vector.c:785-819, src/halfvec.c:725-759); raises OverflowError like the reference."""
    try:
        if _is_cuda(rows):
            import torch
            r2, single = _dev_rows(rows, elem)
            out = torch.empty(r2.shape, dtype=torch.float32 if elem == VECTOR else torch.float16, device=r2.device)
            _dev_call(load().vb_l2_normalize_batch_dev, elem, r2.shape[1], _ptr(r2), r2.shape[0], _ptr(out), inputs=(r2,))
            return out[0] if single else out
        rows = _host(elem, rows)
        single = rows.ndim == 1
        r2 = np.ascontiguousarray(rows.reshape(1, -1) if single else rows)
        out = np.empty_like(r2)
        _lib.check(load().vb_l2_normalize_batch(elem, r2.shape[1], _ptr(r2), r2.shape[0], _ptr(out)))
        return out[0] if single else out
    except VecB200Error as e:
        if "overflow" in str(e):
            raise OverflowError("value out of range: overflow") from None
        raise


def vector_to_halfvec(rows):
    """vector::halfvec (src/halfvec.c:540-555): RNE to half bit patterns; raises like the reference on overflow"""
    try:
        if _is_cuda(rows):
            import torch
            r2, single = _dev_rows(rows, VECTOR)
            out = torch.empty(r2.shape, dtype=torch.float16, device=r2.device)
            _dev_call(load().vb_vector_to_halfvec_batch_dev, r2.shape[1], _ptr(r2), r2.shape[0], _ptr(out), inputs=(r2,))
            return out[0] if single else out
        rows = _host(VECTOR, rows)
        single = rows.ndim == 1
        r2 = np.ascontiguousarray(rows.reshape(1, -1) if single else rows)
        out = np.empty(r2.shape, dtype=np.uint16)
        _lib.check(load().vb_vector_to_halfvec_batch(r2.shape[1], _ptr(r2), r2.shape[0], _ptr(out)))
        return out[0] if single else out
    except VecB200Error as e:
        if "out of range for type halfvec" in str(e):
            raise ValueError(str(e).split(": ", 1)[1]) from None
        raise


def halfvec_to_vector(rows):
    """halfvec::vector: exact widening"""
    if _is_cuda(rows):
        import torch
        r2, single = _dev_rows(rows, HALFVEC)
        out = torch.empty(r2.shape, dtype=torch.float32, device=r2.device)
        _dev_call(load().vb_halfvec_to_vector_batch_dev, r2.shape[1], _ptr(r2), r2.shape[0], _ptr(out), inputs=(r2,))
        return out[0] if single else out
    rows = _host(HALFVEC, rows)
    single = rows.ndim == 1
    r2 = np.ascontiguousarray(rows.reshape(1, -1) if single else rows)
    out = np.empty(r2.shape, dtype=np.float32)
    _lib.check(load().vb_halfvec_to_vector_batch(r2.shape[1], _ptr(r2), r2.shape[0], _ptr(out)))
    return out[0] if single else out


def binary_quantize(rows, elem=VECTOR):
    """binary_quantize of every row (src/vector.c:952-978): packed bits, MSB first."""
    if _is_cuda(rows):
        import torch
        r2, single = _dev_rows(rows, elem)
        out = torch.empty((r2.shape[0], (r2.shape[1] + 7) // 8), dtype=torch.uint8, device=r2.device)
        _dev_call(load().vb_binary_quantize_batch_dev, elem, r2.shape[1], _ptr(r2), r2.shape[0], _ptr(out), inputs=(r2,))
        return out[0] if single else out
    rows = _host(elem, rows)
    single = rows.ndim == 1
    r2 = np.ascontiguousarray(rows.reshape(1, -1) if single else rows)
    out = np.empty((r2.shape[0], (r2.shape[1] + 7) // 8), dtype=np.uint8)
    _lib.check(load().vb_binary_quantize_batch(elem, r2.shape[1], _ptr(r2), r2.shape[0], _ptr(out)))
    return out[0] if single else out


def subvector(rows, start, count, elem=VECTOR):
    """subvector(v, start, count) of every row (src/vector.c:983-1025, src/halfvec.c:939-981): `count` elements from
    1-based `start`, clipped to the row as the reference clips them.  The reference's errors ("vector must have at least
    1 dimension", ...) raise ValueError."""
    lib = load()
    dev = _is_cuda(rows)
    if dev:
        r2, single = _dev_rows(rows, elem)
        fn = lib.vb_subvector_batch_dev
    else:
        r2 = _host(elem, rows)
        single = r2.ndim == 1
        r2 = np.ascontiguousarray(r2.reshape(1, -1) if single else r2)
        fn = lib.vb_subvector_batch
    n, dim = r2.shape
    d = C.c_int(0)

    def call(src, m, out):
        rc = fn(elem, dim, src, m, int(start), int(count), out, C.byref(d))
        if rc == _lib.EINVAL:
            msg = lib.vb_last_error().decode()
            if msg.endswith(" must have at least 1 dimension") or " cannot have more than " in msg:
                raise ValueError(msg)
        _lib.check(rc)

    call(None, 0, None)   # n = 0 sizes the output
    if dev:
        import torch
        out = torch.empty((n, d.value), dtype=torch.float32 if elem == VECTOR else torch.float16, device=r2.device)
        _after_torch(r2)
        call(_ptr(r2), n, _ptr(out))
        synchronize()   # the library runs on its own stream; results are handed back complete
    else:
        out = np.empty((n, d.value), dtype=_NP[elem])
        call(_ptr(r2), n, _ptr(out))
    return out[0] if single else out


# --------------------------------------------------------------------- + - * || and the array casts
#
# Both operands are numpy arrays (host variants) or both torch CUDA tensors (_dev variants); a 1-d operand is one row,
# used with every row of the other.  The result is one row when both operands are 1-d.

ADD, SUB, MUL = 0, 1, 2
ARRAY_INT4, ARRAY_FLOAT4, ARRAY_FLOAT8 = 0, 1, 2


def _check_reference(rc):
    """the reference's errors as Python ones: "value out of range: ..." raises OverflowError, its other texts
    (dimensions, NaN / infinite elements, halfvec range) ValueError; argument refusals name the entry point."""
    if rc == _lib.EINVAL:
        msg = load().vb_last_error().decode()
        if msg.startswith("value out of range: "):
            raise OverflowError(msg)
        if not msg.startswith("vb_"):
            raise ValueError(msg)
    _lib.check(rc)


def _operands(a, b, elem):
    """(a rows, b rows, whether the result is one row, whether on the device)"""
    dev = _is_cuda(a)
    if dev != _is_cuda(b):
        raise TypeError("both operands must be numpy arrays or both torch CUDA tensors")
    out = []
    for x in (a, b):
        if dev:
            out.append(_dev_rows(x, elem))
        else:
            x = _host(elem, x)
            out.append((np.ascontiguousarray(x.reshape(1, -1) if x.ndim == 1 else x), x.ndim == 1))
    (a2, sa), (b2, sb) = out
    return a2, b2, sa and sb, dev


def _result_rows(a2, b2):
    na, nb = a2.shape[0], b2.shape[0]
    return na if nb == 1 else nb


def _arith(op, a, b, elem):
    lib = load()
    a2, b2, single, dev = _operands(a, b, elem)
    m, dim = _result_rows(a2, b2), a2.shape[1]
    args = (elem, op, a2.shape[1], _ptr(a2), a2.shape[0], b2.shape[1], _ptr(b2), b2.shape[0])
    if dev:
        import torch
        out = torch.empty((m, dim), dtype=a2.dtype if elem == VECTOR else torch.float16, device=a2.device)
        _after_torch(a2, b2)
        _check_reference(lib.vb_arith_batch_dev(*args, _ptr(out)))
        synchronize()
    else:
        out = np.empty((m, dim), dtype=_NP[elem])
        _check_reference(lib.vb_arith_batch(*args, _ptr(out)))
    return out[0] if single else out


def vector_add(a, b, elem=VECTOR):
    """a + b (vector_add, src/vector.c:826-852; halfvec_add, src/halfvec.c:766-798); overflow raises OverflowError."""
    return _arith(ADD, a, b, elem)


def vector_sub(a, b, elem=VECTOR):
    """a - b (vector_sub, src/vector.c:859-885; halfvec_sub, src/halfvec.c:805-837); overflow raises OverflowError."""
    return _arith(SUB, a, b, elem)


def vector_mul(a, b, elem=VECTOR):
    """a * b (vector_mul, src/vector.c:892-921; halfvec_mul, src/halfvec.c:844-879); overflow and underflow raise
    OverflowError."""
    return _arith(MUL, a, b, elem)


def vector_concat(a, b, elem=VECTOR):
    """a || b (vector_concat, src/vector.c:928-947; halfvec_concat, src/halfvec.c:886-903)."""
    lib = load()
    a2, b2, single, dev = _operands(a, b, elem)
    m, da, db = _result_rows(a2, b2), a2.shape[1], b2.shape[1]
    fn = lib.vb_concat_batch_dev if dev else lib.vb_concat_batch
    d = C.c_int(0)
    _check_reference(fn(elem, da, None, 0, db, None, 0, None, C.byref(d)))   # 0 rows size the output
    if dev:
        import torch
        out = torch.empty((m, d.value), dtype=a2.dtype if elem == VECTOR else torch.float16, device=a2.device)
        _after_torch(a2, b2)
    else:
        out = np.empty((m, d.value), dtype=_NP[elem])
    _check_reference(fn(elem, da, _ptr(a2), a2.shape[0], db, _ptr(b2), b2.shape[0], _ptr(out), C.byref(d)))
    if dev:
        synchronize()
    return out[0] if single else out


def _numeric_cast(elem, rows, typmod):
    """numeric[] rows (Decimal values or NumericArrays) through vb_numeric_array_to_rows_batch[_dev]"""
    lib = load()
    A, single = _numeric.as_numeric_arrays(rows)
    bad = C.c_int64(-1)
    if A.is_cuda:
        import torch
        out = torch.empty((A.n, A.dim), dtype=torch.float32 if elem == VECTOR else torch.float16, device=A.data.device)
        _after_torch(A.data, A.off)
        _check_reference(lib.vb_numeric_array_to_rows_batch_dev(elem, A.dim, int(typmod), _ptr(A.data), _ptr(A.off), A.n, _ptr(out),
                                                                C.byref(bad)))
        synchronize()
    else:
        out = np.empty((A.n, A.dim), dtype=_NP[elem])
        _check_reference(lib.vb_numeric_array_to_rows_batch(elem, A.dim, int(typmod), _ptr(np.ascontiguousarray(A.data)),
                                                            _ptr(np.ascontiguousarray(A.off, dtype=np.int64)), A.n, _ptr(out), C.byref(bad)))
    return out[0] if single else out


def _array_cast(elem, rows, typmod):
    if _numeric.is_numeric_rows(rows):
        return _numeric_cast(elem, rows, typmod)
    lib = load()
    dev = _is_cuda(rows)
    if dev:
        import torch
        src = {torch.int32: ARRAY_INT4, torch.float32: ARRAY_FLOAT4, torch.float64: ARRAY_FLOAT8}.get(rows.dtype)
    else:
        rows = np.asarray(rows)
        src = {np.dtype(np.int32): ARRAY_INT4, np.dtype(np.float32): ARRAY_FLOAT4, np.dtype(np.float64): ARRAY_FLOAT8}.get(rows.dtype)
    if src is None:
        raise ValueError("unsupported array type")
    single = rows.ndim == 1
    r2 = rows.reshape(1, -1) if single else rows
    if r2.ndim != 2:
        raise ValueError("array must be 1-D")
    n, dim = r2.shape
    if dev:
        r2 = r2.contiguous()
        out = torch.empty((n, dim), dtype=torch.float32 if elem == VECTOR else torch.float16, device=r2.device)
        _after_torch(r2)
        _check_reference(lib.vb_array_to_rows_batch_dev(elem, src, dim, int(typmod), _ptr(r2), n, _ptr(out)))
        synchronize()
    else:
        r2 = np.ascontiguousarray(r2)
        out = np.empty((n, dim), dtype=_NP[elem])
        _check_reference(lib.vb_array_to_rows_batch(elem, src, dim, int(typmod), _ptr(r2), n, _ptr(out)))
    return out[0] if single else out


def array_to_vector(rows, typmod=-1):
    """integer[] / real[] / double precision[] / numeric[] :: vector(typmod) of every row (src/vector.c:443-512): the
    dtype (int32, float32, float64) is the array type; rows of decimal.Decimal values, or numeric.NumericArrays of
    numeric_send fields (host or CUDA), are numeric[].  The reference's errors raise ValueError."""
    return _array_cast(VECTOR, rows, typmod)


def array_to_halfvec(rows, typmod=-1):
    """the same to halfvec (src/halfvec.c:442-509): binary16 bit patterns (uint16) from numpy rows, float16 on the
    device.  The reference's errors, including "<float>" is out of range for type halfvec, raise ValueError."""
    return _array_cast(HALFVEC, rows, typmod)


# ------------------------------------------------------------------------- type I/O: text in, text out

def _text_input(texts):
    """(bytes, off, n, on the device) of a list of str (text literals) or bytes (binary payloads), or of a (CUDA uint8
    tensor, CUDA int64 offsets) pair"""
    if isinstance(texts, (tuple, list)) and len(texts) == 2 and all(_is_cuda(t) for t in texts):
        import torch
        text, off = texts
        if text.dtype != torch.uint8 or off.dtype != torch.int64 or text.dim() != 1 or off.dim() != 1 or off.numel() < 1:
            raise ValueError("device text: a 1-d uint8 tensor and 1-d int64 offsets [n + 1]")
        return text.contiguous(), off.contiguous(), off.numel() - 1, True
    blobs = [t.encode() if isinstance(t, str) else bytes(t) for t in texts]
    off = np.zeros(len(blobs) + 1, dtype=np.int64)
    off[1:] = np.cumsum([len(b) for b in blobs])
    text = np.frombuffer(b"".join(blobs) or b"\0", dtype=np.uint8)
    return text, off, len(blobs), False


def _raise_text(rc, bad):
    if rc == _lib.EINVAL:
        lib = load()
        msg = lib.vb_last_error().decode()
        if bad.value >= 0:
            raise _lib.TextInputError(msg, lib.vb_last_error_detail().decode(), int(bad.value))
    _lib.check(rc)


def _text_to_rows(elem, texts, typmod):
    lib = load()
    text, off, n, dev = _text_input(texts)
    bad = C.c_int64(-1)
    if dev:
        import torch
        row_off = torch.zeros(n + 1, dtype=torch.int64, device=text.device)   # a refused argument writes none
        fn = lib.vb_text_to_rows_batch_dev
        _after_torch(text, off)
    else:
        row_off = np.zeros(n + 1, dtype=np.int64)
        fn = lib.vb_text_to_rows_batch
    rc = fn(elem, typmod, n, _ptr(text), _ptr(off), 0, _ptr(row_off), None, C.byref(bad))
    total = int(row_off[-1])
    if dev:
        out = torch.empty(0, dtype=torch.float32 if elem == VECTOR else torch.float16, device=text.device)
    else:
        out = np.empty(0, dtype=_NP[elem])
    if rc == _lib.EINVAL and total > 0 and bad.value < 0:
        if dev:
            out = torch.empty(total, dtype=torch.float32 if elem == VECTOR else torch.float16, device=text.device)
        else:
            out = np.empty(total, dtype=_NP[elem])
        rc = fn(elem, typmod, n, _ptr(text), _ptr(off), total, _ptr(row_off), _ptr(out), C.byref(bad))
    _raise_text(rc, bad)
    if dev:
        return out, row_off
    return [out[row_off[i]:row_off[i + 1]] for i in range(n)]


def vector_in(texts, typmod=-1):
    """vector_in (src/vector.c:174-281) of every literal: a list of str gives a list of float32 arrays; a (CUDA uint8
    text, CUDA int64 offsets) pair gives device (values, row offsets).  The reference's errors raise
    TextInputError (a ValueError) with .detail and .row."""
    return _text_to_rows(VECTOR, texts, typmod)


def halfvec_in(texts, typmod=-1):
    """halfvec_in (src/halfvec.c:178-286): rows as binary16 bit patterns (uint16) on the host, float16 on the device."""
    return _text_to_rows(HALFVEC, texts, typmod)


def _rows_to_text(elem, rows):
    lib = load()
    if _is_cuda(rows):
        import torch
        x, _ = _dev_rows(rows, elem)
        n, dim = int(x.shape[0]), int(x.shape[1])
        off = torch.empty(n + 1, dtype=torch.int64, device=x.device)
        _after_torch(x)
        _lib.check(lib.vb_rows_to_text_batch_dev(elem, dim, _ptr(x), n, 0, _ptr(off), None))
        out = torch.empty(max(int(off[-1]), 1), dtype=torch.uint8, device=x.device)
        _lib.check(lib.vb_rows_to_text_batch_dev(elem, dim, _ptr(x), n, int(off[-1]), _ptr(off), _ptr(out)))
        return out[:int(off[-1])], off
    x = _host(elem, rows)
    x = x.reshape(1, -1) if x.ndim == 1 else x
    n, dim = x.shape
    # the reference's own bound: 15 bytes per element, separators and brackets
    cap = n * (dim * 16 + 2)
    off = np.empty(n + 1, dtype=np.int64)
    out = np.empty(max(cap, 1), dtype=np.uint8)
    _lib.check(lib.vb_rows_to_text_batch(elem, dim, _ptr(x), n, cap, _ptr(off), _ptr(out)))
    blob = out.tobytes()
    return [blob[off[i]:off[i + 1]].decode() for i in range(n)]


def vector_out(rows):
    """vector_out (src/vector.c:289-326) of every row: numpy rows give a list of str, CUDA rows device (text, offsets)."""
    return _rows_to_text(VECTOR, rows)


def halfvec_out(rows):
    """halfvec_out (src/halfvec.c:294-335): numpy rows are binary16 bit patterns (uint16) or floats rounded to half."""
    return _rows_to_text(HALFVEC, rows)


# ------------------------------------------------------------------------- type I/O: binary in, binary out

def _binary_to_rows(elem, payloads, typmod):
    lib = load()
    data, off, n, dev = _text_input(payloads)
    bad = C.c_int64(-1)
    if dev:
        import torch
        torch_dt = torch.float32 if elem == VECTOR else torch.float16
        row_off = torch.zeros(n + 1, dtype=torch.int64, device=data.device)   # a refused argument writes none
        fn = lib.vb_binary_to_rows_batch_dev
        _after_torch(data, off)
    else:
        row_off = np.zeros(n + 1, dtype=np.int64)
        fn = lib.vb_binary_to_rows_batch
    rc = fn(elem, typmod, n, _ptr(data), _ptr(off), 0, _ptr(row_off), None, C.byref(bad))
    total = int(row_off[-1])
    if dev:
        out = torch.empty(max(total, 1), dtype=torch_dt, device=data.device)
    else:
        out = np.empty(max(total, 1), dtype=_NP[elem])
    if rc == _lib.EINVAL and bad.value < 0 and total > 0:
        rc = fn(elem, typmod, n, _ptr(data), _ptr(off), total, _ptr(row_off), _ptr(out), C.byref(bad))
    _raise_text(rc, bad)
    out = out[:total]
    if dev:
        return out, row_off
    return [out[row_off[i]:row_off[i + 1]] for i in range(n)]


def vector_recv(payloads, typmod=-1):
    """vector_recv (src/vector.c:376-400) of every field: a list of bytes gives a list of float32 arrays; a (CUDA uint8
    payloads, CUDA int64 offsets) pair gives device (values, row offsets), as vector_in does.  The reference's errors,
    and PostgreSQL's for a short or overlong field, raise TextInputError (a ValueError) with .row."""
    return _binary_to_rows(VECTOR, payloads, typmod)


def halfvec_recv(payloads, typmod=-1):
    """halfvec_recv (src/halfvec.c:373-401): rows as binary16 bit patterns (uint16) on the host, float16 on the device."""
    return _binary_to_rows(HALFVEC, payloads, typmod)


def _rows_to_binary(elem, rows):
    lib = load()
    if _is_cuda(rows):
        import torch
        x, _ = _dev_rows(rows, elem)
        n, dim = int(x.shape[0]), int(x.shape[1])
        off = torch.empty(n + 1, dtype=torch.int64, device=x.device)
        total = n * (4 + dim * x.element_size())
        out = torch.empty(max(total, 1), dtype=torch.uint8, device=x.device)
        _after_torch(x)
        _lib.check(lib.vb_rows_to_binary_batch_dev(elem, dim, _ptr(x), n, total, _ptr(off), _ptr(out)))
        synchronize()
        return out[:total], off
    x = _host(elem, rows)
    x = x.reshape(1, -1) if x.ndim == 1 else x
    n, dim = x.shape
    cap = n * (4 + dim * x.itemsize)
    off = np.empty(n + 1, dtype=np.int64)
    out = np.empty(max(cap, 1), dtype=np.uint8)
    _lib.check(lib.vb_rows_to_binary_batch(elem, dim, _ptr(x), n, cap, _ptr(off), _ptr(out)))
    blob = out.tobytes()
    return [blob[off[i]:off[i + 1]] for i in range(n)]


def vector_send(rows):
    """vector_send (src/vector.c:405-422) of every row: numpy rows give a list of bytes, CUDA rows device (payloads,
    offsets).  The bits go out unchanged."""
    return _rows_to_binary(VECTOR, rows)


def halfvec_send(rows):
    """halfvec_send (src/halfvec.c:406-419): numpy rows are binary16 bit patterns (uint16) or floats rounded to half."""
    return _rows_to_binary(HALFVEC, rows)


from .sparsevec import sparsevec_in, sparsevec_out, sparsevec_recv, sparsevec_send  # noqa: E402,F401
