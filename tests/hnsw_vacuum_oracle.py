"""The serial HNSW vacuum the GPU vacuum is checked against (tests/hnsw_vacuum_oracle.c, on top of the serial on-disk
insert and the CPU oracle's HNSW, compiled here at first use into a directory of the temporary area, with the oracle's
own flags).  TEST INFRASTRUCTURE ONLY."""
from __future__ import annotations

import ctypes as C
import hashlib
import os
import subprocess
import tempfile

import numpy as np

import oracle as O
from tests.hnsw_ondisk_oracle import CFLAGS, ORACLE, _p, slot_changes

HERE = os.path.dirname(os.path.abspath(__file__))
SRC = os.path.join(HERE, "hnsw_vacuum_oracle.c")

_lib = None


def lib() -> C.CDLL:
    global _lib
    if _lib is not None:
        return _lib
    deps = [SRC, os.path.join(HERE, "hnsw_ondisk_oracle.c")] + [
        os.path.join(ORACLE, f) for f in ("pgv_hnsw.c", "pgv_distance.c", "pgv_oracle.h", "pgv_pairingheap.h")]
    h = hashlib.sha1()
    for p in deps:
        h.update(open(p, "rb").read())
    h.update(O._cpu_stamp().encode())
    d = os.path.join(tempfile.gettempdir(), f"hnsw_vacuum_oracle_{os.getuid()}_{h.hexdigest()[:16]}")
    so = os.path.join(d, "libhnswvacuum.so")
    if not os.path.exists(so):
        os.makedirs(d, exist_ok=True)
        tmp = f"{so}.{os.getpid()}.tmp"
        subprocess.run(["gcc", *CFLAGS, "-shared", "-I", ORACLE, "-I", HERE, "-o", tmp, SRC, os.path.join(ORACLE, "pgv_distance.c"), "-lm"],
                       check=True, capture_output=True)
        os.replace(tmp, so)
    L = C.CDLL(so)
    vp, i32, i64 = C.c_void_p, C.c_int, C.c_int64
    for name, res, args in [("pgv_hnsw_create", vp, [i32, i32, i32, i32, i32, C.c_uint64]), ("pgv_hnsw_build", None, [vp, vp, i64]),
                            ("pgv_hnsw_count", i64, [vp]), ("pgv_hnsw_entry", i32, [vp, vp, vp]),
                            ("pgv_hnsw_export_layer0", None, [vp, vp, vp]), ("pgv_hnsw_export_upper", i64, [vp, vp, vp]),
                            ("pgv_hnsw_export_elements", None, [vp, vp, vp, vp]), ("pgv_hnsw_search", i32, [vp, vp, i32, i32, vp, vp, vp]),
                            ("disk_hnsw_wrap", vp, [vp, i64]), ("disk_hnsw_free", None, [vp]), ("disk_hnsw_insert", None, [vp, vp, i64, vp]),
                            ("disk_hnsw_dup_of", None, [vp, vp]), ("disk_hnsw_graph", vp, [vp]), ("disk_hnsw_vacuum", i64, [vp, vp])]:
        getattr(L, name).restype = res
        getattr(L, name).argtypes = args
    _lib = L
    return L


class VacuumHnsw:
    """an oracle HNSW graph (the serial in-memory build of `rows`) that changes by serial on-disk inserts and serial
    vacuums"""

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

    def vacuum(self, counts):
        """serial graph work of hnswbulkdelete on the heap TID counts left by RemoveHeapTids: returns (the change
        records, the number of repairs)"""
        counts = np.ascontiguousarray(counts, dtype=np.int32)
        assert counts.shape == (self.n,)
        before = self.export()
        nrep = int(lib().disk_hnsw_vacuum(self.d, _p(counts)))
        return slot_changes(before, self.export()), nrep

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
