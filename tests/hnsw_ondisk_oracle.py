"""The serial on-disk HNSW insert the GPU insert is checked against (tests/hnsw_ondisk_oracle.c on top of the CPU
oracle's HNSW, compiled here at first use into a directory of the temporary area, with the oracle's own flags).
TEST INFRASTRUCTURE ONLY."""
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
SRC = os.path.join(HERE, "hnsw_ondisk_oracle.c")
# oracle/Makefile's CFLAGS (the reference's flags)
CFLAGS = ["-O2", "-ftree-vectorize", "-fassociative-math", "-fno-signed-zeros", "-fno-trapping-math", "-ffp-contract=fast",
          "-march=native", "-fPIC", "-fopenmp", "-std=gnu11", "-w"]

_lib = None


def lib() -> C.CDLL:
    global _lib
    if _lib is not None:
        return _lib
    deps = [SRC] + [os.path.join(ORACLE, f) for f in ("pgv_hnsw.c", "pgv_distance.c", "pgv_oracle.h", "pgv_pairingheap.h")]
    h = hashlib.sha1()
    for p in deps:
        h.update(open(p, "rb").read())
    h.update(O._cpu_stamp().encode())
    d = os.path.join(tempfile.gettempdir(), f"hnsw_ondisk_oracle_{os.getuid()}_{h.hexdigest()[:16]}")
    so = os.path.join(d, "libhnswondisk.so")
    if not os.path.exists(so):
        os.makedirs(d, exist_ok=True)
        tmp = f"{so}.{os.getpid()}.tmp"
        subprocess.run(["gcc", *CFLAGS, "-shared", "-I", ORACLE, "-o", tmp, SRC, os.path.join(ORACLE, "pgv_distance.c"), "-lm"],
                       check=True, capture_output=True)
        os.replace(tmp, so)
    L = C.CDLL(so)
    vp, i32, i64 = C.c_void_p, C.c_int, C.c_int64
    L.pgv_hnsw_create.restype = vp
    L.pgv_hnsw_create.argtypes = [i32, i32, i32, i32, i32, C.c_uint64]
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
    L.pgv_hnsw_search.restype = i32
    L.pgv_hnsw_search.argtypes = [vp, vp, i32, i32, vp, vp, vp]
    L.disk_hnsw_wrap.restype = vp
    L.disk_hnsw_wrap.argtypes = [vp, i64]
    L.disk_hnsw_free.restype = None
    L.disk_hnsw_free.argtypes = [vp]
    L.disk_hnsw_insert.restype = None
    L.disk_hnsw_insert.argtypes = [vp, vp, i64, vp]
    L.disk_hnsw_set_heaptid_counts.restype = None
    L.disk_hnsw_set_heaptid_counts.argtypes = [vp, vp]
    L.disk_hnsw_dup_of.restype = None
    L.disk_hnsw_dup_of.argtypes = [vp, vp]
    L.disk_hnsw_graph.restype = vp
    L.disk_hnsw_graph.argtypes = [vp]
    _lib = L
    return L


def _p(a):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


class DiskHnsw:
    """an oracle HNSW graph (the serial in-memory build of `rows`, possibly none) that grows by serial on-disk inserts"""

    def __init__(self, elem, metric, rows, m=16, ef_construction=64, seed=42, dim=None):
        L = lib()
        self.elem, self.metric, self.m = elem, metric, m
        self._rows = O._rows(elem, rows)
        self.dim = dim if dim is not None else self._rows.shape[-1]
        g = L.pgv_hnsw_create(elem, metric, self.dim, m, ef_construction, seed)
        L.pgv_hnsw_build(g, _p(self._rows), self._rows.shape[0])
        self.d = L.disk_hnsw_wrap(g, self._rows.shape[0])
        self.g = L.disk_hnsw_graph(self.d)

    def __del__(self):
        try:
            lib().disk_hnsw_free(self.d)
        except Exception:
            pass

    @property
    def n(self):
        return int(lib().pgv_hnsw_count(self.g))

    def insert_on_disk(self, rows, levels=None):
        """serial INSERT of rows (HnswInsertTupleOnDisk): returns (dup_of of the new rows, the change records)"""
        rows = O._rows(self.elem, rows)
        before = self.export()
        lv = None if levels is None else np.ascontiguousarray(levels, dtype=np.int32)
        n0 = self.n
        lib().disk_hnsw_insert(self.d, _p(rows), rows.shape[0], _p(lv))
        after = self.export()
        return after["dup_of"][n0:], slot_changes(before, after)

    def set_heaptid_counts(self, counts):
        counts = np.ascontiguousarray(counts, dtype=np.int32)
        assert counts.shape == (self.n,)
        lib().disk_hnsw_set_heaptid_counts(self.d, _p(counts))

    def export(self):
        L = lib()
        n, m = self.n, self.m
        levels = np.empty(n, dtype=np.int32)
        nbr0 = np.empty((n, 2 * m), dtype=np.int32)
        L.pgv_hnsw_export_layer0(self.g, _p(levels), _p(nbr0))
        upper_off = np.empty(n, dtype=np.int64)
        slots = L.pgv_hnsw_export_upper(self.g, _p(upper_off), None)
        upper = np.full((max(slots, 1), m), -1, dtype=np.int32)
        L.pgv_hnsw_export_upper(self.g, _p(upper_off), _p(upper))
        elem_row = np.empty(n, dtype=np.int64)
        nht = np.empty(n, dtype=np.int32)
        ht = np.empty((n, 10), dtype=np.int64)
        L.pgv_hnsw_export_elements(self.g, _p(elem_row), _p(nht), _p(ht))
        dup_of = np.empty(n, dtype=np.int32)
        L.disk_hnsw_dup_of(self.d, _p(dup_of))
        entry = C.c_int64()
        el = C.c_int()
        L.pgv_hnsw_entry(self.g, C.byref(entry), C.byref(el))
        return dict(levels=levels, nbr0=nbr0, upper_off=upper_off, upper=upper[:slots], elem_row=elem_row, n_heaptids=nht,
                    heaptids=ht, entry=entry.value, entry_level=el.value, m=m, dup_of=dup_of)

    def search(self, q, ef, ties=O.TIES_PG):
        q = O._rows(self.elem, q)
        ids = np.empty(ef + 2, dtype=np.int64)
        dist = np.empty(ef + 2, dtype=np.float64)
        nd = C.c_int64()
        n = lib().pgv_hnsw_search(self.g, _p(q), ef, ties, _p(ids), _p(dist), C.byref(nd))
        return ids[:n], dist[:n], nd.value


SLOT_DTYPE = np.dtype([("element", np.int32), ("layer", np.int32), ("slot", np.int32), ("neighbor", np.int32)])


def slot_changes(before, after):
    """the neighbour-array slots whose value differs between two exports of one graph (after = before grown by an
    insert): (element, layer, slot, neighbor) records sorted by (element, layer, slot); slot indexes the layer's lm
    entries"""
    m, n0, n1 = after["m"], len(before["levels"]), len(after["levels"])
    old0 = np.full((n1, 2 * m), -1, np.int32)
    old0[:n0] = before["nbr0"]
    e, j = np.nonzero(after["nbr0"] != old0)
    recs = [np.stack([e, np.zeros_like(e), j, after["nbr0"][e, j]], axis=1)]
    old_up = np.full((len(after["upper"]), m), -1, np.int32)
    old_up[:len(before["upper"])] = before["upper"]
    lv, uo = after["levels"], after["upper_off"]
    owner = np.repeat(np.arange(n1), np.maximum(lv, 0))
    if len(owner):
        layer = np.concatenate([np.arange(1, v + 1) for v in lv if v > 0])
        slot = uo[owner] + layer - 1
        s, j = np.nonzero(after["upper"][slot] != old_up[slot])
        recs.append(np.stack([owner[s], layer[s], j, after["upper"][slot][s, j]], axis=1))
    r = np.concatenate(recs).astype(np.int64)
    r = r[np.lexsort((r[:, 2], r[:, 1], r[:, 0]))]
    out = np.empty(len(r), dtype=SLOT_DTYPE)
    for i, k in enumerate(SLOT_DTYPE.names):
        out[k] = r[:, i]
    return out
