"""numpy restatement of array_to_sparsevec (src/sparsevec.c:694-821) for integer[] / real[] / double precision[]
sources, batched as vb_array_to_sparsevec_batch is: n rows of dim elements, the error of the lowest failing row.

Per row, in the reference's order: each element becomes (float) of the int32 or double (numpy's astype rounds to
nearest even, as the C cast does) or the real as is; it is kept when v != 0 (so -0 and a double that rounds to 0 are
dropped, NaN and the infinities kept); CheckNnz; then CheckElement over the kept values in index order.
"""
from __future__ import annotations

import json
import os

import numpy as np

MAX_DIM = 1_000_000_000   # SPARSEVEC_MAX_DIM (src/sparsevec.h:11)
MAX_NNZ = 16_000          # SPARSEVEC_MAX_NNZ (src/sparsevec.h:12)
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "array_cast_kat.json")
DTYPES = {"int4": np.int32, "float4": np.float32, "float8": np.float64}


class CastError(ValueError):
    """the reference's errmsg, with the failing row (-1 for the checks before any work)"""

    def __init__(self, msg, row=-1):
        super().__init__(msg)
        self.row = row


def to_float4(rows):
    """the float each element becomes"""
    with np.errstate(over="ignore"):
        return np.asarray(rows).astype(np.float32)


def array_to_sparsevec(rows, typmod=-1):
    """rows: [n, dim] int32 / float32 / float64 -> (row_off int64 [n + 1], idx int32, val float32), or CastError"""
    rows = np.asarray(rows)
    if rows.ndim == 1:
        rows = rows.reshape(1, -1)
    n, dim = rows.shape
    if dim < 1:
        raise CastError("sparsevec must have at least 1 dimension")
    if dim > MAX_DIM:
        raise CastError(f"sparsevec cannot have more than {MAX_DIM} dimensions")
    if typmod != -1 and typmod != dim:
        raise CastError(f"expected {typmod} dimensions, not {dim}")
    f = to_float4(rows)
    keep = f != 0
    cnt = keep.sum(axis=1)
    special = keep & ~np.isfinite(f)
    over = np.nonzero(cnt > MAX_NNZ)[0]
    spec_rows = np.nonzero(special.any(axis=1))[0]
    first = min([int(r) for r in over[:1]] + [int(r) for r in spec_rows[:1]], default=-1)
    if first >= 0:
        if cnt[first] > MAX_NNZ:
            raise CastError(f"sparsevec cannot have more than {MAX_NNZ} non-zero elements", first)
        i = int(np.argmax(special[first]))
        raise CastError("NaN not allowed in sparsevec" if np.isnan(f[first, i]) else "infinite value not allowed in sparsevec", first)
    r, c = np.nonzero(keep)
    off = np.zeros(n + 1, dtype=np.int64)
    off[1:] = np.cumsum(cnt)
    return off, c.astype(np.int32), f[r, c]


def format_row(dim, idx, val):
    """sparsevec_out of one row with integral values ('{1:1,3:2}/6', 1-based), enough for the known answers"""
    return "{" + ",".join(f"{int(i) + 1}:{np.format_float_positional(np.float32(v), trim='-')}" for i, v in zip(idx, val)) + f"}}/{dim}"


def kat_cases():
    with open(GOLDEN) as f:
        return json.load(f)["cases"]


def kat_rows(case):
    """the case's array as a [1, dim] numpy row of its source type (numeric[]: a list with one row of Decimal values)"""
    e = case["elems"]
    if case["src"] == "numeric":
        import decimal
        return [[decimal.Decimal(x) for x in e]]
    if isinstance(e, dict):
        lo, hi = e["range"]
        e = list(range(lo, hi))
    vals = [float(x) if isinstance(x, str) else x for x in e]
    return np.array(vals, dtype=DTYPES[case["src"]]).reshape(1, -1)


# ------------------------------------------------------------------------------- numeric[] sources
# PostgreSQL core's rules (numeric.c: numeric_recv, numeric_out, numeric_float4; float.c: float4in), restated: a field is
# numeric_send's bytes; numeric_float4 is float4in(numeric_out(x)), and float4in is glibc strtof (called here through
# ctypes, as float4in calls it) plus its range rule.

import ctypes as _C
import errno as _errno
import math as _math
import struct as _struct

_libc = _C.CDLL("libc.so.6", use_errno=True)
_libc.strtof.restype = _C.c_float
_libc.strtof.argtypes = [_C.c_char_p, _C.POINTER(_C.c_char_p)]

FIELD_ERRORS = {"short": "insufficient data left in message", "sign": 'invalid sign in external "numeric" value',
                "scale": 'invalid scale in external "numeric" value', "digit": 'invalid digit in external "numeric" value',
                "trailing": "incorrect binary data format"}
SIGNS = (0x0000, 0x4000, 0xC000, 0xD000, 0xF000)


class FieldError(ValueError):
    """a malformed field: numeric_recv's text, with the field number (.field)"""

    def __init__(self, msg, field):
        super().__init__(msg)
        self.field = field


def field_check(f):
    """numeric_recv's first failing read or check of the field bytes f, as a FIELD_ERRORS key, or None"""
    if len(f) < 6:
        return "short"
    nd, _, sign = _struct.unpack(">HhH", f[:6])
    if sign not in SIGNS:
        return "sign"
    if len(f) < 8:
        return "short"
    if _struct.unpack(">H", f[6:8])[0] & ~0x3FFF:
        return "scale"
    for i in range(nd):
        if len(f) < 8 + 2 * (i + 1):
            return "short"
        if _struct.unpack(">H", f[8 + 2 * i:10 + 2 * i])[0] >= 10000:
            return "digit"
    return "trailing" if len(f) > 8 + 2 * nd else None


def numeric_out(f):
    """numeric_out of a finite field numeric_recv accepts: its digits truncated to dscale fraction digits (trunc_var),
    leading zero groups stripped (make_result), then get_str_from_var"""
    nd, weight, sign, dscale = _struct.unpack(">HhHH", f[:8])
    digits = list(_struct.unpack(f">{nd}H", f[8:8 + 2 * nd]))
    keep = max(0, min(nd, weight + 1 + (dscale + 3) // 4))
    digits = digits[:keep]
    if digits and keep == weight + 1 + (dscale + 3) // 4 and dscale % 4:
        cut = 10 ** (4 - dscale % 4)
        digits[-1] -= digits[-1] % cut
    while digits and digits[0] == 0:
        digits.pop(0)
        weight -= 1
    if not digits:
        weight, sign = 0, 0
    g = lambda i: digits[i] if 0 <= i < len(digits) else 0   # noqa: E731
    s = "-" if sign == 0x4000 else ""
    if weight < 0:
        s += "0"
        i = weight + 1
    else:
        s += str(g(0)) + "".join(f"{g(i):04d}" for i in range(1, weight + 1))
        i = weight + 1
    if dscale > 0:
        frac = ""
        while len(frac) < dscale:
            frac += f"{g(i):04d}"
            i += 1
        s += "." + frac[:dscale]
    return s


def float4in(text):
    """float4in of a numeric_out text: glibc strtof, and "out of range for type real" when it sets ERANGE with a result
    of 0 or infinity"""
    _C.set_errno(0)
    v = _libc.strtof(text.encode(), None)
    if _C.get_errno() == _errno.ERANGE and (v == 0 or _math.isinf(v)):
        raise CastError(f'"{text}" is out of range for type real')
    return np.float32(v)


def numeric_float4(f):
    """numeric_float4 of a field numeric_recv accepts"""
    sign = _struct.unpack(">H", f[4:6])[0]
    if sign == 0xC000:
        return np.float32("nan")
    if sign in (0xD000, 0xF000):
        return np.float32("inf") if sign == 0xD000 else np.float32("-inf")
    return float4in(numeric_out(f))


def _fields(data, off, n, dim):
    data = bytes(np.asarray(data, dtype=np.uint8).tobytes())
    off = np.asarray(off, dtype=np.int64)
    return [[data[off[r * dim + i]:off[r * dim + i + 1]] for i in range(dim)] for r in range(n)]


def _check_fields(rows):
    for r, row in enumerate(rows):
        for i, f in enumerate(row):
            bad = field_check(f)
            if bad:
                raise FieldError(FIELD_ERRORS[bad], r * len(row) + i)


def numeric_to_rows(elem, rows, typmod=-1):
    """numeric[] :: vector (elem "vector") or halfvec ("halfvec") of rows of field bytes: float32 rows or binary16 bit
    patterns (uint16), or CastError (FieldError for a malformed field, before any data error)"""
    n, dim = len(rows), (len(rows[0]) if rows else 0)
    if dim < 1:
        raise CastError(f"{elem} must have at least 1 dimension")
    if dim > 16000:
        raise CastError(f"{elem} cannot have more than 16000 dimensions")
    if typmod != -1 and typmod != dim:
        raise CastError(f"expected {typmod} dimensions, not {dim}")
    _check_fields(rows)
    out = np.zeros((n, dim), dtype=np.float32 if elem == "vector" else np.uint16)
    for r, row in enumerate(rows):
        try:
            if elem == "vector":
                v = np.array([numeric_float4(f) for f in row], dtype=np.float32)      # the whole row, then CheckElement
                for x in v:
                    if not np.isfinite(x):
                        raise CastError(f"{'NaN' if np.isnan(x) else 'infinite value'} not allowed in vector")
                out[r] = v
            else:
                h = np.zeros(dim, dtype=np.uint16)
                for i, f in enumerate(row):                                             # numeric_float4, Float4ToHalf
                    x = numeric_float4(f)
                    with np.errstate(over="ignore"):
                        h[i] = np.float32(x).astype(np.float16).view(np.uint16)
                    if (h[i] & 0x7FFF) == 0x7C00 and np.isfinite(x):
                        raise CastError(f'"{_pg_float4(x)}" is out of range for type halfvec')
                for b in h:                                                             # CheckElement
                    if (b & 0x7C00) == 0x7C00:
                        raise CastError(f"{'NaN' if b & 0x3FF else 'infinite value'} not allowed in halfvec")
                out[r] = h
        except CastError as e:
            raise CastError(str(e), r) from None
    return out


def numeric_to_sparsevec(rows, typmod=-1):
    """numeric[] :: sparsevec of rows of field bytes: (row_off, idx, val), or CastError"""
    n, dim = len(rows), (len(rows[0]) if rows else 0)
    if dim < 1:
        raise CastError("sparsevec must have at least 1 dimension")
    if typmod != -1 and typmod != dim:
        raise CastError(f"expected {typmod} dimensions, not {dim}")
    _check_fields(rows)
    f = np.zeros((n, dim), dtype=np.float32)
    for r, row in enumerate(rows):
        try:
            f[r] = [numeric_float4(x) for x in row]                                   # the count loop's conversions
        except CastError as e:
            raise CastError(str(e), r) from None
        try:
            array_to_sparsevec(f[r:r + 1])
        except CastError as e:
            raise CastError(str(e), r) from None
    return array_to_sparsevec(f)


def _pg_float4(v):
    """float_to_shortest_decimal_buf: the shortest digits that read back, fixed notation for exponents -4 .. 14"""
    s = np.format_float_scientific(np.float32(v), unique=True, trim="-")
    mant, e = s.split("e")
    e = int(e)
    if -4 <= e < 15:
        return np.format_float_positional(np.float32(v), unique=True, trim="-")
    return f"{mant}e{'-' if e < 0 else '+'}{abs(e):02d}"


def fields_of(values):
    """rows of numeric_send bytes of rows of Decimal values (or of raw bytes, kept as they are)"""
    from pgvector_b200.numeric import numeric_send
    return [[v if isinstance(v, bytes) else numeric_send(v) for v in row] for row in values]


def pack(rows):
    """(data uint8, off int64) of rows of field bytes"""
    flat = [f for row in rows for f in row]
    off = np.zeros(len(flat) + 1, dtype=np.int64)
    off[1:] = np.cumsum([len(f) for f in flat])
    return np.frombuffer(b"".join(flat) + b"\0", dtype=np.uint8).copy(), off


def format_dense(elem, row):
    """vector_out / halfvec_out of one row (halfvec: binary16 bit patterns)"""
    f = np.asarray(row).view(np.float16).astype(np.float32) if elem == "halfvec" else np.asarray(row, dtype=np.float32)
    return "[" + ",".join(_pg_float4(x) for x in f) + "]"


def kat_answer(case):
    """the restatement's answer to a known-answer case: the value's text, or CastError"""
    rows = kat_rows(case)
    if case["src"] == "numeric":
        fields = fields_of(rows)
        if case["type"] == "sparsevec":
            off, idx, val = numeric_to_sparsevec(fields, case["typmod"])
            return format_row(len(rows[0]), idx, val)
        return format_dense(case["type"], numeric_to_rows(case["type"], fields, case["typmod"])[0])
    off, idx, val = array_to_sparsevec(rows, case["typmod"])
    return format_row(rows.shape[1], idx, val)
