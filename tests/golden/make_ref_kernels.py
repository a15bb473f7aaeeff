#!/usr/bin/env python3
"""Record what pgvector's own half / bit kernels (oracle/_ref/libpgvref.so, compiled from a pgvector source tree by
oracle.build()) return on seeded inputs, into ref_kernels.npz.  test_oracle_golden compares the oracle with these
values, so the comparison runs where no pgvector tree is present.

    python3 tests/golden/make_ref_kernels.py
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))

import oracle as O  # noqa: E402
from tests.util import f32_to_half_bits  # noqa: E402

HALF_DIMS = (1, 3, 8, 9, 64, 100, 768, 1537)
BIT_LENGTHS = (0, 1, 7, 8, 52, 63, 64, 65, 513, 1024, 4099)


def conversion_inputs():
    rng = np.random.default_rng(0)
    return np.concatenate([
        rng.standard_normal(2000).astype(np.float32) * 10,
        np.float32([0, -0.0, 1, -1, 65504, 65520, 65519.99, 1e-8, 5.96e-8, 2.98e-8, 2.9802322e-8, 6.1e-5, 6.0975552e-5,
                    1e5, -1e5, np.inf, -np.inf, 0.1, 0.33325195, 1.0009766, 1.00048828125, 1.0014648]),
        (rng.standard_normal(500) * 1e-6).astype(np.float32),
    ])


def kernel_inputs():
    """(half rows a, b per dimension, bit strings a, b per bit length), seeded"""
    rng = np.random.default_rng(1)
    half = {dim: (f32_to_half_bits(rng.standard_normal(dim)), f32_to_half_bits(rng.standard_normal(dim))) for dim in HALF_DIMS}
    bits = {}
    for nbits in BIT_LENGTHS:
        nbytes = (nbits + 7) // 8
        a = rng.integers(0, 256, size=max(nbytes, 1), dtype=np.uint8)[:nbytes].copy()
        b = rng.integers(0, 256, size=max(nbytes, 1), dtype=np.uint8)[:nbytes].copy()
        if nbits % 8 and nbytes:
            mask = (0xFF << (8 - nbits % 8)) & 0xFF
            a[-1] &= mask
            b[-1] &= mask
        bits[nbits] = (np.ascontiguousarray(a), np.ascontiguousarray(b))
    return half, bits


def main():
    R = O.ref()
    if R is None:
        sys.exit("oracle/_ref/libpgvref.so is not built (oracle.build() needs a pgvector source tree)")
    out = {}
    xs = conversion_inputs()
    out["f2h"] = np.array([R.ref_float_to_half(float(x)) for x in xs], dtype=np.uint16)
    out["h2f"] = np.array([R.ref_half_to_float(h) for h in range(0, 65536, 7)], dtype=np.float32)
    half, bits = kernel_inputs()
    for dim, (a, b) in half.items():
        pa, pb = a.ctypes.data, b.ctypes.data
        out[f"half_{dim}"] = np.array([R.ref_half_l2sq(dim, pa, pb), R.ref_half_ip(dim, pa, pb), R.ref_half_l1(dim, pa, pb),
                                       R.ref_half_cos(dim, pa, pb)], dtype=np.float64)
    for nbits, (a, b) in bits.items():
        nbytes = (nbits + 7) // 8
        pa = a.ctypes.data if nbytes else None
        pb = b.ctypes.data if nbytes else None
        out[f"bit_{nbits}"] = np.array([R.ref_bit_hamming(nbytes, pa, pb), R.ref_bit_jaccard(nbytes, pa, pb)], dtype=np.float64)
    np.savez_compressed(os.path.join(HERE, "ref_kernels.npz"), **out)


if __name__ == "__main__":
    main()
