"""ctypes bindings of the CPU oracle (oracle/liboracle.so) and of the reference's
own kernels compiled verbatim (oracle/_ref/libpgvref.so).

TEST INFRASTRUCTURE ONLY.  Import this package from tests/, from
``__graft_entry__.smoke()`` and from ``bench.py``'s cpu_baseline / ``--impl
reference`` legs -- never from ``pgvector_b200`` (a test greps for that).
"""
from __future__ import annotations

import ctypes as C
import hashlib
import os
import subprocess

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))

VECTOR, HALFVEC, BIT = 0, 1, 2
L2_SQUARED, NEG_IP, COSINE, L1, HAMMING, JACCARD, L2, IP, SPHERICAL = range(9)
TIES_PG, TIES_TOTAL = 0, 1

_NP = {VECTOR: np.float32, HALFVEC: np.uint16, BIT: np.uint8}


def _cpu_stamp() -> str:
    try:
        with open("/proc/cpuinfo") as f:
            for line in f:
                if line.startswith("flags"):
                    return hashlib.sha1(line.encode()).hexdigest()[:16]
    except OSError:
        pass
    return "unknown"


def build(force: bool = False) -> None:
    """(Re)build liboracle.so for THIS host's CPU (-march=native, the reference's
    flag) and, when a pgvector source tree is present, oracle/_ref/ from the reference's
    own sources.  Elsewhere an existing _ref/ is used as it is."""
    so = os.path.join(HERE, "liboracle.so")
    stamp_path = os.path.join(HERE, ".built_for")
    stamp = _cpu_stamp()
    have = os.path.exists(so) and os.path.exists(stamp_path) and open(stamp_path).read() == stamp
    srcs = [os.path.join(HERE, f) for f in os.listdir(HERE) if f.endswith((".c", ".h"))]
    if have and not force and all(os.path.getmtime(s) <= os.path.getmtime(so) for s in srcs):
        if os.path.exists(os.path.join(HERE, "_ref", "libpgvref.so")) or not os.path.exists("/root/reference/src"):
            return
    # several processes (one per GPU under torchrun) may get here together: one builds, the others wait for the lock
    # and find the library up to date; the library is linked beside its final name and renamed
    import fcntl
    with open(os.path.join(HERE, ".build_lock"), "w") as lock:
        fcntl.flock(lock, fcntl.LOCK_EX)
        have = os.path.exists(so) and os.path.exists(stamp_path) and open(stamp_path).read() == stamp
        if have and not force and all(os.path.getmtime(s) <= os.path.getmtime(so) for s in srcs):
            if os.path.exists(os.path.join(HERE, "_ref", "libpgvref.so")) or not os.path.exists("/root/reference/src"):
                return
        tmp = so + ".tmp"
        subprocess.run(["make", "-C", HERE, "-s", "-B", "liboracle.so", "OUT=" + tmp], check=True, capture_output=True)
        os.replace(tmp, so)
        subprocess.run(["make", "-C", HERE, "-s", "ref"], check=True, capture_output=True)
        with open(stamp_path, "w") as f:
            f.write(stamp)


_lib = None
_ref = None


def lib() -> C.CDLL:
    global _lib
    if _lib is None:
        build()
        _lib = C.CDLL(os.path.join(HERE, "liboracle.so"))
        _declare(_lib)
    return _lib


def ref():
    """The reference's own halfutils.c/bitutils.c (None when not built)."""
    global _ref
    if _ref is None:
        p = os.path.join(HERE, "_ref", "libpgvref.so")
        if not os.path.exists(p):
            return None
        r = C.CDLL(p)
        r.ref_half_l2sq.restype = C.c_float
        r.ref_half_ip.restype = C.c_float
        r.ref_half_cos.restype = C.c_double
        r.ref_half_l1.restype = C.c_float
        for f in (r.ref_half_l2sq, r.ref_half_ip, r.ref_half_cos, r.ref_half_l1):
            f.argtypes = [C.c_int, C.c_void_p, C.c_void_p]
        r.ref_bit_hamming.restype = C.c_uint64
        r.ref_bit_hamming.argtypes = [C.c_uint32, C.c_void_p, C.c_void_p]
        r.ref_bit_jaccard.restype = C.c_double
        r.ref_bit_jaccard.argtypes = [C.c_uint32, C.c_void_p, C.c_void_p]
        r.ref_half_to_float.restype = C.c_float
        r.ref_half_to_float.argtypes = [C.c_uint16]
        r.ref_float_to_half.restype = C.c_uint16
        r.ref_float_to_half.argtypes = [C.c_float]
        r.ref_half_batch.restype = None
        r.ref_half_batch.argtypes = [C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_long, C.c_void_p]
        r.ref_bit_batch.restype = None
        r.ref_bit_batch.argtypes = [C.c_int, C.c_uint32, C.c_void_p, C.c_void_p, C.c_long, C.c_void_p]
        _ref = r
    return _ref


class IvfIndex(C.Structure):
    _fields_ = [("elem", C.c_int), ("metric", C.c_int), ("dim", C.c_int), ("lists", C.c_int),
                ("centers", C.c_void_p), ("list_offsets", C.c_void_p), ("rows", C.c_void_p), ("ids", C.c_void_p)]


def _declare(L):
    vp, i32, i64, dbl = C.c_void_p, C.c_int, C.c_int64, C.c_double
    L.pgv_float_to_half.restype = C.c_uint16
    L.pgv_float_to_half.argtypes = [C.c_float]
    L.pgv_half_to_float.restype = C.c_float
    L.pgv_half_to_float.argtypes = [C.c_uint16]
    L.pgv_distance.restype = dbl
    L.pgv_distance.argtypes = [i32, i32, i32, vp, vp]
    L.pgv_distance_f64.restype = dbl
    L.pgv_distance_f64.argtypes = [i32, i32, i32, vp, vp]
    L.pgv_norm.restype = dbl
    L.pgv_norm.argtypes = [i32, i32, vp]
    L.pgv_l2_normalize.restype = i32
    L.pgv_l2_normalize.argtypes = [i32, i32, vp, vp]
    L.pgv_binary_quantize.restype = None
    L.pgv_binary_quantize.argtypes = [i32, i32, vp, vp]
    L.pgv_distance_batch.restype = None
    L.pgv_distance_batch.argtypes = [i32, i32, i32, vp, vp, i64, vp]
    L.pgv_exact_topk.restype = None
    L.pgv_exact_topk.argtypes = [i32, i32, i32, vp, vp, i64, i32, vp, vp]
    P = C.POINTER(IvfIndex)
    L.pgv_ivf_set_tie_mode.restype = None
    L.pgv_ivf_set_tie_mode.argtypes = [i32]
    L.pgv_ivf_scan_lists.restype = i32
    L.pgv_ivf_scan_lists.argtypes = [P, vp, i32, vp, vp]
    L.pgv_ivf_scan_items.restype = i64
    L.pgv_ivf_scan_items.argtypes = [P, vp, vp, i32, i64, vp, vp]
    L.pgv_ivf_search.restype = i64
    L.pgv_ivf_search.argtypes = [P, vp, i32, i32, vp, vp]
    L.pgv_ivf_search_batch.restype = None
    L.pgv_ivf_search_batch.argtypes = [P, vp, i64, i32, i32, i32, vp, vp]
    L.pgv_ivf_assign.restype = None
    L.pgv_ivf_assign.argtypes = [i32, i32, i32, vp, i64, vp, i32, i32, vp]
    for f in (L.pgv_kmeans_elkan, L.pgv_kmeans_lloyd):
        f.restype = i32
        f.argtypes = [i32, i32, i32, vp, i64, vp, i32, i32, C.c_uint64, vp]
    L.pgv_kmeans_pp_init.restype = None
    L.pgv_kmeans_pp_init.argtypes = [i32, i32, i32, vp, i64, vp, i32, C.c_uint64]
    L.pgv_kmeans_pp_init_draws.restype = None
    L.pgv_kmeans_pp_init_draws.argtypes = [i32, i32, i32, vp, i64, vp, i32, i64, vp, vp]
    L.pgv_hnsw_create.restype = vp
    L.pgv_hnsw_create.argtypes = [i32, i32, i32, i32, i32, C.c_uint64]
    L.pgv_hnsw_free.restype = None
    L.pgv_hnsw_free.argtypes = [vp]
    L.pgv_hnsw_build.restype = None
    L.pgv_hnsw_build.argtypes = [vp, vp, i64]
    L.pgv_hnsw_count.restype = i64
    L.pgv_hnsw_count.argtypes = [vp]
    L.pgv_hnsw_entry.restype = i32
    L.pgv_hnsw_entry.argtypes = [vp, vp, vp]
    L.pgv_hnsw_export_layer0.restype = None
    L.pgv_hnsw_export_layer0.argtypes = [vp, vp, vp]
    L.pgv_hnsw_export_upper.restype = i64
    L.pgv_hnsw_export_upper.argtypes = [vp, vp, vp]
    L.pgv_hnsw_export_elements.restype = None
    L.pgv_hnsw_export_elements.argtypes = [vp, vp, vp, vp]
    L.pgv_hnsw_import.restype = vp
    L.pgv_hnsw_import.argtypes = [i32, i32, i32, i32, vp, i64, vp, vp, vp, vp, i64, i32]
    L.pgv_hnsw_search.restype = i32
    L.pgv_hnsw_search.argtypes = [vp, vp, i32, i32, vp, vp, vp]
    L.pgv_hnsw_iter_scan.restype = i64
    L.pgv_hnsw_iter_scan.argtypes = [vp, vp, i32, i32, i64, i64, vp, vp, vp, vp]
    L.pgv_hnsw_search_batch.restype = None
    L.pgv_hnsw_search_batch.argtypes = [vp, vp, i64, i32, i32, i32, i32, vp, vp, vp]

    L.pgv_sparse_distance.restype = dbl
    L.pgv_sparse_distance.argtypes = [i32, i32, vp, vp, i32, vp, vp]
    L.pgv_sparse_distance_f64.restype = dbl
    L.pgv_sparse_distance_f64.argtypes = [i32, i32, vp, vp, i32, vp, vp]
    L.pgv_sparse_l2_norm.restype = dbl
    L.pgv_sparse_l2_norm.argtypes = [i32, vp]
    L.pgv_sparse_l2_normalize.restype = i32
    L.pgv_sparse_l2_normalize.argtypes = [i32, vp, vp, vp, vp]
    L.pgv_sparse_distance_batch.restype = None
    L.pgv_sparse_distance_batch.argtypes = [i32, i32, vp, vp, i64, vp, vp, vp, vp]


# ----------------------------------------------------------------- helpers

def _p(a):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


def _rows(elem, a):
    a = np.ascontiguousarray(a, dtype=_NP[elem])
    return a


def row_dim(elem, a):
    """logical dimension of a row array (bits for BIT rows are passed explicitly)."""
    return a.shape[-1]


def f2h(x):
    """float32 array -> IEEE half bit patterns (uint16), RNE, via the oracle."""
    L = lib()
    x = np.ascontiguousarray(x, dtype=np.float32)
    out = np.empty(x.shape, dtype=np.uint16)
    flat, o = x.ravel(), out.ravel()
    for i in range(flat.size):
        o[i] = L.pgv_float_to_half(float(flat[i]))
    return out


def distance(elem, metric, a, b, dim=None, f64=False):
    L = lib()
    a, b = _rows(elem, a), _rows(elem, b)
    d = dim if dim is not None else a.shape[-1]
    fn = L.pgv_distance_f64 if f64 else L.pgv_distance
    return fn(elem, metric, d, _p(a), _p(b))


def distance_batch(elem, metric, q, rows, dim=None):
    L = lib()
    q, rows = _rows(elem, q), _rows(elem, rows)
    d = dim if dim is not None else rows.shape[-1]
    out = np.empty(rows.shape[0], dtype=np.float64)
    L.pgv_distance_batch(elem, metric, d, _p(q), _p(rows), rows.shape[0], _p(out))
    return out


def norm(elem, a):
    a = _rows(elem, a)
    return lib().pgv_norm(elem, a.shape[-1], _p(a))


def l2_normalize(elem, a):
    a = _rows(elem, a)
    out = np.empty_like(a)
    if a.ndim == 1:
        rc = lib().pgv_l2_normalize(elem, a.shape[0], _p(a), _p(out))
        if rc:
            raise OverflowError("value out of range: overflow")
        return out
    for i in range(a.shape[0]):
        lib().pgv_l2_normalize(elem, a.shape[1], _p(a[i]), C.c_void_p(out[i].ctypes.data))
    return out


def binary_quantize(elem, a):
    a = _rows(elem, a)
    single = a.ndim == 1
    a2 = a.reshape(1, -1) if single else a
    dim = a2.shape[1]
    out = np.zeros((a2.shape[0], (dim + 7) // 8), dtype=np.uint8)
    for i in range(a2.shape[0]):
        lib().pgv_binary_quantize(elem, dim, C.c_void_p(a2[i].ctypes.data), C.c_void_p(out[i].ctypes.data))
    return out[0] if single else out


def exact_topk(elem, metric, q, rows, k, dim=None):
    L = lib()
    q, rows = _rows(elem, q), _rows(elem, rows)
    d = dim if dim is not None else rows.shape[-1]
    ids = np.empty(k, dtype=np.int64)
    dist = np.empty(k, dtype=np.float64)
    L.pgv_exact_topk(elem, metric, d, _p(q), _p(rows), rows.shape[0], k, _p(ids), _p(dist))
    return ids, dist


# ----------------------------------------------------------------- sparsevec (pgv_sparse.c)

def _sp(v):
    """(indices, values) -> contiguous int32 / float32 arrays (indices ascending, 0-based)"""
    idx = np.ascontiguousarray(v[0], dtype=np.int32)
    val = np.ascontiguousarray(v[1], dtype=np.float32)
    assert idx.shape == val.shape and idx.ndim == 1
    return idx, val


def sparse_distance(metric, a, b, f64=False):
    """a, b = (indices, values); the float8 of sparsevec's l2_distance / inner_product / ... (src/sparsevec.c:826-1057)"""
    (ai, ax), (bi, bx) = _sp(a), _sp(b)
    fn = lib().pgv_sparse_distance_f64 if f64 else lib().pgv_sparse_distance
    return fn(metric, ai.size, _p(ai), _p(ax), bi.size, _p(bi), _p(bx))


def sparse_l2_norm(a):
    _, ax = _sp(a)
    return lib().pgv_sparse_l2_norm(ax.size, _p(ax))


def sparse_l2_normalize(a):
    ai, ax = _sp(a)
    oi, ox = np.empty_like(ai), np.empty_like(ax)
    n = lib().pgv_sparse_l2_normalize(ai.size, _p(ai), _p(ax), _p(oi), _p(ox))
    if n < 0:
        raise OverflowError("value out of range: overflow")
    return oi[:n].copy(), ox[:n].copy()


def sparse_distance_batch(metric, q, row_off, idx, val):
    """one query against CSR rows: out[r] = distance(row r, q)"""
    qi, qx = _sp(q)
    row_off = np.ascontiguousarray(row_off, dtype=np.int64)
    idx = np.ascontiguousarray(idx, dtype=np.int32)
    val = np.ascontiguousarray(val, dtype=np.float32)
    n = row_off.size - 1
    out = np.empty(n, dtype=np.float64)
    lib().pgv_sparse_distance_batch(metric, qi.size, _p(qi), _p(qx), n, _p(row_off), _p(idx), _p(val), _p(out))
    return out


def ivf_set_tie_mode(total_order: bool):
    """False: PostgreSQL pairing-heap tie order (reference); True: (distance, list number)."""
    lib().pgv_ivf_set_tie_mode(1 if total_order else 0)


class Ivf:
    """Flat-array IVFFlat index image for the oracle."""

    def __init__(self, elem, metric, centers, list_offsets, rows, ids=None, dim=None):
        self.elem, self.metric = elem, metric
        self.centers = _rows(elem, centers)
        self.rows = _rows(elem, rows)
        self.offsets = np.ascontiguousarray(list_offsets, dtype=np.int64)
        self.ids = None if ids is None else np.ascontiguousarray(ids, dtype=np.int64)
        self.dim = dim if dim is not None else self.rows.shape[-1]
        self.lists = self.centers.shape[0]
        self.c = IvfIndex(elem, metric, self.dim, self.lists, self.centers.ctypes.data, self.offsets.ctypes.data,
                          self.rows.ctypes.data, None if self.ids is None else self.ids.ctypes.data)

    def scan_lists(self, q, max_probes):
        L = lib()
        q = None if q is None else _rows(self.elem, q)
        n = min(max_probes, self.lists)
        out = np.empty(max(n, 1), dtype=np.int32)
        dist = np.empty(max(n, 1), dtype=np.float64)
        c = L.pgv_ivf_scan_lists(C.byref(self.c), _p(q), max_probes, _p(out), _p(dist))
        return out[:c], dist[:c]

    def search(self, q, probes, k=0):
        L = lib()
        q = None if q is None else _rows(self.elem, q)
        cap = k if k > 0 else int(self.rows.shape[0])
        ids = np.empty(max(cap, 1), dtype=np.int64)
        dist = np.empty(max(cap, 1), dtype=np.float64)
        n = L.pgv_ivf_search(C.byref(self.c), _p(q), probes, k, _p(ids), _p(dist))
        m = min(n, cap)
        return ids[:m], dist[:m], n

    def search_batch(self, queries, probes, k, threads=1):
        L = lib()
        queries = _rows(self.elem, queries)
        nq = queries.shape[0]
        ids = np.empty((nq, k), dtype=np.int64)
        dist = np.empty((nq, k), dtype=np.float64)
        L.pgv_ivf_search_batch(C.byref(self.c), _p(queries), nq, probes, k, threads, _p(ids), _p(dist))
        return ids, dist


def ivf_assign(elem, metric, rows, centers, threads=1, dim=None):
    rows, centers = _rows(elem, rows), _rows(elem, centers)
    d = dim if dim is not None else rows.shape[-1]
    out = np.empty(rows.shape[0], dtype=np.int32)
    lib().pgv_ivf_assign(elem, metric, d, _p(rows), rows.shape[0], _p(centers), centers.shape[0], threads, _p(out))
    return out


def kmeans(elem, kmeans_metric, samples, init_centers, max_iter=500, seed=42, algo="elkan", dim=None):
    samples = _rows(elem, samples)
    centers = _rows(elem, init_centers).copy()
    d = dim if dim is not None else samples.shape[-1]
    closest = np.empty(samples.shape[0], dtype=np.int32)
    fn = lib().pgv_kmeans_elkan if algo == "elkan" else lib().pgv_kmeans_lloyd
    it = fn(elem, kmeans_metric, d, _p(samples), samples.shape[0], _p(centers), centers.shape[0], max_iter, seed, _p(closest))
    return centers, closest, it


def kmeans_pp_init(elem, kmeans_metric, samples, k, seed=42, dim=None):
    samples = _rows(elem, samples)
    d = dim if dim is not None else samples.shape[-1]
    centers = np.empty((k,) + samples.shape[1:], dtype=samples.dtype)
    lib().pgv_kmeans_pp_init(elem, kmeans_metric, d, _p(samples), samples.shape[0], _p(centers), k, seed)
    return centers


def kmeans_pp_init_draws(elem, kmeans_metric, samples, k, first, u, dim=None):
    """InitCenters with caller-supplied draws; returns (centres, picked sample rows)."""
    samples = _rows(elem, samples)
    d = dim if dim is not None else samples.shape[-1]
    centers = np.empty((k,) + samples.shape[1:], dtype=samples.dtype)
    u = np.ascontiguousarray(u, dtype=np.float64)
    picked = np.empty(k, dtype=np.int64)
    lib().pgv_kmeans_pp_init_draws(elem, kmeans_metric, d, _p(samples), samples.shape[0], _p(centers), k, int(first), _p(u), _p(picked))
    return centers, picked


class Hnsw:
    def __init__(self, elem, metric, rows, m=16, ef_construction=64, seed=42, dim=None, _handle=None):
        L = lib()
        self.elem, self.metric, self.m = elem, metric, m
        self.rows = _rows(elem, rows)
        self.dim = dim if dim is not None else self.rows.shape[-1]
        if _handle is None:
            self.h = L.pgv_hnsw_create(elem, metric, self.dim, m, ef_construction, seed)
            L.pgv_hnsw_build(self.h, _p(self.rows), self.rows.shape[0])
        else:
            self.h = _handle
        self.n = L.pgv_hnsw_count(self.h)

    def __del__(self):
        try:
            lib().pgv_hnsw_free(self.h)
        except Exception:
            pass

    def export(self):
        """dict of numpy arrays describing the graph (element-indexed)."""
        L = lib()
        n, m = self.n, self.m
        levels = np.empty(n, dtype=np.int32)
        nbr0 = np.empty((n, 2 * m), dtype=np.int32)
        L.pgv_hnsw_export_layer0(self.h, _p(levels), _p(nbr0))
        upper_off = np.empty(n, dtype=np.int64)
        slots = L.pgv_hnsw_export_upper(self.h, _p(upper_off), None)
        upper = np.full((max(slots, 1), m), -1, dtype=np.int32)
        L.pgv_hnsw_export_upper(self.h, _p(upper_off), _p(upper))
        elem_row = np.empty(n, dtype=np.int64)
        nht = np.empty(n, dtype=np.int32)
        ht = np.empty((n, 10), dtype=np.int64)
        L.pgv_hnsw_export_elements(self.h, _p(elem_row), _p(nht), _p(ht))
        entry = C.c_int64()
        el = C.c_int()
        L.pgv_hnsw_entry(self.h, C.byref(entry), C.byref(el))
        return dict(levels=levels, nbr0=nbr0, upper_off=upper_off, upper=upper[:slots], elem_row=elem_row,
                    n_heaptids=nht, heaptids=ht, entry=entry.value, entry_level=el.value, m=m)

    @classmethod
    def from_export(cls, elem, metric, elem_rows, g, dim=None):
        L = lib()
        rows = _rows(elem, elem_rows)
        d = dim if dim is not None else rows.shape[-1]
        levels = np.ascontiguousarray(g["levels"], dtype=np.int32)
        nbr0 = np.ascontiguousarray(g["nbr0"], dtype=np.int32)
        uo = np.ascontiguousarray(g["upper_off"], dtype=np.int64)
        up = np.ascontiguousarray(g["upper"], dtype=np.int32)
        if up.size == 0:
            up = np.full((1, g["m"]), -1, dtype=np.int32)
        h = L.pgv_hnsw_import(elem, metric, d, g["m"], _p(rows), rows.shape[0], _p(levels), _p(nbr0), _p(uo), _p(up),
                              g["entry"], g["entry_level"])
        obj = cls(elem, metric, rows, m=g["m"], dim=d, _handle=h)
        obj._keep = (levels, nbr0, uo, up)
        return obj

    def search(self, q, ef, ties=TIES_PG):
        L = lib()
        q = None if q is None else _rows(self.elem, q)
        ids = np.empty(ef + 2, dtype=np.int64)
        dist = np.empty(ef + 2, dtype=np.float64)
        nd = C.c_int64()
        n = L.pgv_hnsw_search(self.h, _p(q), ef, ties, _p(ids), _p(dist), C.byref(nd))
        return ids[:n], dist[:n], nd.value

    def iter_scan(self, q, ef, max_scan_tuples=20000, max_out=1 << 20, ties=TIES_PG):
        """the element sequence of an iterative scan in relaxed order (src/hnswscan.c:62-87, 228-340):
        (ids, distances, batch number of each output [-1 = the drain after max_scan_tuples], tuples counter)"""
        L = lib()
        q = None if q is None else _rows(self.elem, q)
        max_out = int(min(max_out, max(1, L.pgv_hnsw_count(self.h))))
        ids = np.empty(max_out, dtype=np.int64)
        dist = np.empty(max_out, dtype=np.float64)
        batch = np.empty(max_out, dtype=np.int32)
        nd = C.c_int64()
        n = L.pgv_hnsw_iter_scan(self.h, _p(q), ef, ties, max_scan_tuples, max_out, _p(ids), _p(dist), _p(batch), C.byref(nd))
        return ids[:n], dist[:n], batch[:n], nd.value

    def search_batch(self, queries, ef, k, ties=TIES_PG, threads=1):
        L = lib()
        queries = _rows(self.elem, queries)
        nq = queries.shape[0]
        ids = np.empty((nq, k), dtype=np.int64)
        dist = np.empty((nq, k), dtype=np.float64)
        nd = np.empty(nq, dtype=np.int64)
        L.pgv_hnsw_search_batch(self.h, _p(queries), nq, ef, ties, threads, k, _p(ids), _p(dist), _p(nd))
        return ids, dist, nd
