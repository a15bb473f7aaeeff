"""FindInsertPage, the list an IVFFlat insert goes to (tests/ivf_insert_oracle.c against the CPU oracle's distance
functions, compiled here at first use into a directory of the temporary area, with the oracle's own flags).
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
SRC = os.path.join(HERE, "ivf_insert_oracle.c")
# oracle/Makefile's CFLAGS (the reference's flags)
CFLAGS = ["-O2", "-ftree-vectorize", "-fassociative-math", "-fno-signed-zeros", "-fno-trapping-math", "-ffp-contract=fast",
          "-march=native", "-fPIC", "-std=gnu11", "-w"]

_lib = None


def lib() -> C.CDLL:
    global _lib
    if _lib is not None:
        return _lib
    deps = [SRC] + [os.path.join(ORACLE, f) for f in ("pgv_distance.c", "pgv_oracle.h")]
    h = hashlib.sha1()
    for p in deps:
        h.update(open(p, "rb").read())
    h.update(O._cpu_stamp().encode())
    d = os.path.join(tempfile.gettempdir(), f"ivf_insert_oracle_{os.getuid()}_{h.hexdigest()[:16]}")
    so = os.path.join(d, "libivfinsert.so")
    if not os.path.exists(so):
        os.makedirs(d, exist_ok=True)
        tmp = f"{so}.{os.getpid()}.tmp"
        subprocess.run(["gcc", *CFLAGS, "-shared", "-I", ORACLE, "-o", tmp, SRC, os.path.join(ORACLE, "pgv_distance.c"), "-lm"],
                       check=True, capture_output=True)
        os.replace(tmp, so)
    L = C.CDLL(so)
    L.pgv_ivf_insert_lists.restype = None
    L.pgv_ivf_insert_lists.argtypes = [C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_int64, C.c_void_p, C.c_int, C.c_void_p]
    _lib = L
    return L


def insert_lists(elem, metric, rows, centers, dim=None):
    """FindInsertPage's list for every row (rows and centres in the oracle's payload layout)"""
    rows = np.ascontiguousarray(rows)
    centers = np.ascontiguousarray(centers)
    d = int(dim) if dim is not None else rows.shape[1] * (8 if elem == O.BIT else 1)
    out = np.empty(rows.shape[0], dtype=np.int32)
    lib().pgv_ivf_insert_lists(elem, metric, d, rows.ctypes.data_as(C.c_void_p), rows.shape[0], centers.ctypes.data_as(C.c_void_p),
                               centers.shape[0], out.ctypes.data_as(C.c_void_p))
    return out
