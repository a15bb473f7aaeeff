"""numeric[] elements for the array casts: PostgreSQL's numeric_send encoding of decimal.Decimal values, and
NumericArrays, a batch of encoded rows (host or device) that array_to_vector, array_to_halfvec and
sparsevec.array_to_sparsevec take like a numpy or torch array.

A field is numeric_send's (src/backend/utils/adt/numeric.c): big-endian int16 ndigits, int16 weight, uint16 sign,
uint16 dscale, then ndigits base-10000 int16 digits, with no leading or trailing zero digits (make_result strips
them) and dscale = the digits after the decimal point the value was written with."""
from __future__ import annotations

import decimal
import struct

import numpy as np

NUMERIC_POS, NUMERIC_NEG, NUMERIC_NAN, NUMERIC_PINF, NUMERIC_NINF = 0x0000, 0x4000, 0xC000, 0xD000, 0xF000


def numeric_send(x) -> bytes:
    """the numeric_send bytes of a Decimal (or anything Decimal() takes), as PostgreSQL writes that value"""
    d = x if isinstance(x, decimal.Decimal) else decimal.Decimal(x)
    if d.is_nan():
        return struct.pack(">hhHH", 0, 0, NUMERIC_NAN, 0)
    if d.is_infinite():
        return struct.pack(">hhHH", 0, 0, NUMERIC_NINF if d < 0 else NUMERIC_PINF, 0)
    sign, digits, exp = d.as_tuple()
    dscale = max(0, -exp)
    n = int("".join(map(str, digits)) or "0")
    e0 = (exp // 4) * 4                                  # the exponent of the last group: a multiple of 4
    n *= 10 ** (exp - e0)
    groups = []
    while n:
        n, g = divmod(n, 10000)
        groups.append(g)
    if not groups:                                       # zero: no digits, weight 0, positive
        return struct.pack(">hhHH", 0, 0, NUMERIC_POS, dscale)
    groups.reverse()
    weight = e0 // 4 + len(groups) - 1
    while groups[-1] == 0:
        groups.pop()
    return struct.pack(f">hhHH{len(groups)}h", len(groups), weight, NUMERIC_NEG if sign else NUMERIC_POS, dscale, *groups)


class NumericArrays:
    """n rows of dim numeric elements as numeric_send fields: field e = r * dim + i is data[off[e] .. off[e + 1]).
    data (uint8) and off (int64, n * dim + 1 entries) are numpy arrays, or both CUDA tensors for the _dev calls."""

    def __init__(self, data, off, dim):
        self.data, self.off, self.dim = data, off, int(dim)
        total = int(off.shape[0]) - 1
        if self.dim < 0 or total < 0 or (self.dim and total % self.dim) or (not self.dim and total):
            raise ValueError("off must have n * dim + 1 entries")
        self.n = total // self.dim if self.dim else 0

    @property
    def is_cuda(self):
        return bool(getattr(self.data, "is_cuda", False))

    @classmethod
    def from_rows(cls, rows):
        """from an [n, dim] nesting of Decimal values (or one row)"""
        rows = [list(r) for r in rows]
        dim = len(rows[0]) if rows else 0
        if any(len(r) != dim for r in rows):
            raise ValueError("array must be 1-D")       # rows of different lengths are not one array type per row
        fields = [numeric_send(x) for r in rows for x in r]
        off = np.zeros(len(fields) + 1, dtype=np.int64)
        off[1:] = np.cumsum([len(f) for f in fields])
        data = np.frombuffer(b"".join(fields) or b"\0", dtype=np.uint8).copy()
        return cls(data, off, dim)

    def cuda(self):
        import torch
        return NumericArrays(torch.from_numpy(np.ascontiguousarray(self.data)).cuda(), torch.from_numpy(self.off).cuda(), self.dim)


def is_numeric_rows(rows):
    """rows of Decimal values (a list nesting, or a numpy object array), or NumericArrays"""
    if isinstance(rows, NumericArrays):
        return True
    if isinstance(rows, np.ndarray):
        return rows.dtype == object and rows.size > 0 and isinstance(rows.flat[0], decimal.Decimal)
    if isinstance(rows, (list, tuple)) and rows:
        first = rows[0]
        if isinstance(first, (list, tuple, np.ndarray)) and len(first):
            first = first[0]
        return isinstance(first, decimal.Decimal)
    return False


def as_numeric_arrays(rows):
    """(NumericArrays, whether the input was one row)"""
    if isinstance(rows, NumericArrays):
        return rows, False
    if isinstance(rows, np.ndarray):
        single = rows.ndim == 1
        return NumericArrays.from_rows(rows.reshape(1, -1).tolist() if single else rows.tolist()), single
    single = not isinstance(rows[0], (list, tuple, np.ndarray))
    return NumericArrays.from_rows([list(rows)] if single else rows), single
