"""ivfflat.iterative_scan restated on the CPU oracle's IVFFlat bindings, for the tests of the device scan handle.

src/ivfscan.c:268-277 clamps probes and max_probes; ivfflatgettuple (:400-406) then calls GetScanItems for the next
`probes` lists of the probe order whenever the sorted batch runs dry.  iter_scan runs GetScanLists
(pgv_ivf_scan_lists) once for max(max_probes, probes) lists and GetScanItems (pgv_ivf_scan_items, fully sorted) once per
group of `probes` consecutive lists."""
import ctypes as C

import numpy as np

import oracle as O

_DTYPE = {O.VECTOR: np.float32, O.HALFVEC: np.uint16, O.BIT: np.uint8}


def _ptr(a):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


def iter_scan(oix, q, probes, max_probes):
    """every group's (ids, distances) of one query on an oracle.Ivf image, empty groups included; their concatenation is
    what ivfflatgettuple hands the executor"""
    p = min(probes, oix.lists)
    P = min(max(max_probes, probes), oix.lists)
    lists, _ = oix.scan_lists(q, P)
    qq = None if q is None else np.ascontiguousarray(q, dtype=_DTYPE[oix.elem])
    groups = []
    for g0 in range(0, len(lists), p):
        g = np.ascontiguousarray(lists[g0:g0 + p], dtype=np.int32)
        total = int(sum(oix.offsets[l + 1] - oix.offsets[l] for l in g))
        ids = np.empty(max(total, 1), dtype=np.int64)
        dist = np.empty(max(total, 1), dtype=np.float64)
        n = O.lib().pgv_ivf_scan_items(C.byref(oix.c), _ptr(qq), _ptr(g), len(g), total, _ptr(ids), _ptr(dist))
        groups.append((ids[:n], dist[:n]))
    return groups
