"""The reference's type I/O restated on the CPU for the tests of the device text calls: the three _in loops over
glibc strtof / strtol in the C locale (tests/text_io_oracle.c, compiled here at first use into a directory of the
temporary area), and float_to_shortest_decimal_bufn in Python: the shortest digits that strtof reads back, the nearest
among them (ties to the even digit), computed exactly with fractions.  TEST INFRASTRUCTURE ONLY."""
from __future__ import annotations

import ctypes as C
import hashlib
import os
import subprocess
import tempfile
from fractions import Fraction

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
SRC = os.path.join(HERE, "text_io_oracle.c")
MSG = 300000

_lib = None


def lib() -> C.CDLL:
    global _lib
    if _lib is not None:
        return _lib
    h = hashlib.sha1(open(SRC, "rb").read()).hexdigest()[:16]
    d = os.path.join(tempfile.gettempdir(), f"text_io_oracle_{os.getuid()}_{h}")
    so = os.path.join(d, "libtextiooracle.so")
    if not os.path.exists(so):
        os.makedirs(d, exist_ok=True)
        tmp = f"{so}.{os.getpid()}.tmp"
        subprocess.run(["gcc", "-O2", "-fPIC", "-shared", "-o", tmp, SRC, "-lm"], check=True, capture_output=True)
        os.replace(tmp, so)
    L = C.CDLL(so)
    L.text_dense_in.argtypes = [C.c_int, C.c_char_p, C.c_int32, C.c_void_p, C.POINTER(C.c_int), C.c_char_p, C.c_char_p]
    L.text_sparse_in.argtypes = [C.c_char_p, C.c_int32, C.c_void_p, C.c_void_p, C.POINTER(C.c_int), C.POINTER(C.c_int),
                                 C.c_char_p, C.c_char_p]
    L.text_strtof.argtypes = [C.c_char_p, C.POINTER(C.c_int), C.POINTER(C.c_int)]
    L.text_strtof.restype = C.c_uint32
    _lib = L
    return L


def _cstr(lit):
    b = lit.encode() if isinstance(lit, str) else bytes(lit)
    return b.split(b"\0", 1)[0]


def strtof(s):
    """(float32 bits, bytes consumed, ERANGE) of glibc strtof"""
    end, er = C.c_int(), C.c_int()
    u = lib().text_strtof(_cstr(s), C.byref(end), C.byref(er))
    return int(u), end.value, bool(er.value)


def dense_in(half, lit, typmod=-1):
    """(row, None, None) or (None, errmsg, errdetail); half: rows are uint16 bit patterns"""
    b = _cstr(lit)
    out = np.empty(16000, dtype=np.uint16 if half else np.float32)
    dim = C.c_int()
    msg, det = C.create_string_buffer(MSG), C.create_string_buffer(256)
    if lib().text_dense_in(int(half), b, typmod, out.ctypes.data, C.byref(dim), msg, det):
        return None, msg.value.decode(errors="replace"), det.value.decode()
    return out[:dim.value].copy(), None, None


def sparse_in(lit, typmod=-1):
    """((dim, idx, val), None, None) or (None, errmsg, errdetail)"""
    b = _cstr(lit)
    n = b.count(b",") + 1
    idx, val = np.empty(max(n, 1), np.int32), np.empty(max(n, 1), np.float32)
    nnz, dim = C.c_int(), C.c_int()
    msg, det = C.create_string_buffer(MSG), C.create_string_buffer(256)
    if lib().text_sparse_in(b, typmod, idx.ctypes.data, val.ctypes.data, C.byref(nnz), C.byref(dim), msg, det):
        return None, msg.value.decode(errors="replace"), det.value.decode()
    return (dim.value, idx[:nnz.value].copy(), val[:nnz.value].copy()), None, None


def _reads_back(digits, exp10, bits):
    return strtof(f"{digits}e{exp10}")[0] == bits


def shortest(f):
    """float_to_shortest_decimal_bufn of a float32: the digits and the exponent of the first digit"""
    f = np.float32(f)
    bits = int(f.view(np.uint32))
    x = Fraction(abs(float(f)))
    X = 0
    # exact X: 10^X <= x < 10^(X+1)
    while Fraction(10) ** X > x:
        X -= 1
    while Fraction(10) ** (X + 1) <= x:
        X += 1
    for p in range(1, 10):
        t = X - p + 1
        scale = Fraction(10) ** t
        lo = int(x / scale)
        cands = []
        for d in (lo, lo + 1):
            if d > 0 and _reads_back(d, t, bits & 0x7fffffff):
                cands.append(d)
        if cands:
            if len(cands) == 2:
                a, b = abs(cands[0] * scale - x), abs(cands[1] * scale - x)
                # a tie (the value ends in 5 one digit further) goes to the even digit, as Ryu's does
                d = cands[0] if a < b or (a == b and cands[0] % 2 == 0) else cands[1]
            else:
                d = cands[0]
            s = str(d).rstrip("0")
            return s, t + len(str(d)) - 1
    raise AssertionError("no 9-digit decimal reads back")


def format_float4(f):
    f = np.float32(f)
    if np.isnan(f):
        return "NaN"
    if np.isinf(f):
        return "-Infinity" if f < 0 else "Infinity"
    sign = "-" if np.signbit(f) else ""
    if f == 0:
        return sign + "0"
    s, X = shortest(f)
    return layout(sign, s, X)


def layout(sign, s, X):
    """the layout of digits s with first-digit exponent X: fixed for X in [-4, 6), else d[.ddd]e+-XX"""
    if -4 <= X < 6:
        if X < 0:
            body = "0." + "0" * (-X - 1) + s
        else:
            body = (s + "0" * (X + 1))[:X + 1] + ("." + s[X + 1:] if len(s) > X + 1 else "")
    else:
        body = s[0] + ("." + s[1:] if len(s) > 1 else "") + "e" + ("-" if X < 0 else "+") + f"{abs(X):02d}"
    return sign + body


def format_float4_numpy(f):
    """format_float4 with numpy's shortest digits (fast: for sweeps of many values; shortest() is the exact one)"""
    f = np.float32(f)
    if np.isnan(f) or np.isinf(f) or f == 0:
        return format_float4(f)
    s, X = numpy_digits(f)
    return layout("-" if np.signbit(f) else "", s, X)


def numpy_digits(f):
    """numpy's shortest unique digits and exponent, the cross-check of shortest()"""
    m, e = np.format_float_scientific(np.float32(abs(f)), unique=True, trim="-").split("e")
    return m.replace(".", "").rstrip("0") or "0", int(e)


def vector_out(row, half=False):
    vals = np.asarray(row, dtype=np.uint16).view(np.float16).astype(np.float32) if half else np.asarray(row, np.float32)
    return "[" + ",".join(format_float4(v) for v in vals) + "]"


def sparsevec_out(dim, idx, val):
    return "{" + ",".join(f"{int(i) + 1}:{format_float4(v)}" for i, v in zip(idx, val)) + "}/" + str(dim)
