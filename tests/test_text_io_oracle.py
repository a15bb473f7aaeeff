"""The CPU restatement of the type I/O (tests/text_io_oracle) against the reference's regression outputs and the
layout rule of float_to_shortest_decimal_bufn."""
import numpy as np
import pytest

from tests import text_io_oracle as T


@pytest.mark.parametrize("lit,want", [
    ("[1,2,3]", [1, 2, 3]), (" [ 1,  2 ,    3  ] ", [1, 2, 3]), ("[1.23456]", [1.23456]), ("[1e-46,1]", [0, 1]),
])
def test_vector_in_values(lit, want):
    row, msg, _ = T.dense_in(0, lit)
    assert msg is None and np.array_equal(row, np.array(want, np.float32))


@pytest.mark.parametrize("half,lit,msg,detail", [
    (0, "[hello,1]", 'invalid input syntax for type vector: "[hello,1]"', ""),
    (0, "[NaN,1]", "NaN not allowed in vector", ""),
    (0, "[Infinity,1]", "infinite value not allowed in vector", ""),
    (0, "[4e38,1]", '"4e38" is out of range for type vector', ""),
    (0, "[1,2,3", 'invalid input syntax for type vector: "[1,2,3"', ""),
    (0, "[1,2,3]9", 'invalid input syntax for type vector: "[1,2,3]9"', "Junk after closing right brace."),
    (0, "1,2,3", 'invalid input syntax for type vector: "1,2,3"', 'Vector contents must start with "[".'),
    (0, "[]", "vector must have at least 1 dimension", ""),
    (1, "[65520]", '"65520" is out of range for type halfvec', ""),
])
def test_vector_in_errors(half, lit, msg, detail):
    row, m, d = T.dense_in(half, lit)
    assert row is None and (m, d) == (msg, detail)


@pytest.mark.parametrize("lit,msg,detail", [
    ("{1:1e-46}/1", '"1e-46" is out of range for type sparsevec', ""),
    ("{1:1,2:1}/", 'invalid input syntax for type sparsevec: "{1:1,2:1}/"', ""),
    ("{1:1,2:1", 'invalid input syntax for type sparsevec: "{1:1,2:1"', ""),
    ("{1:1,2:1} 3", 'invalid input syntax for type sparsevec: "{1:1,2:1} 3"', "Unexpected end of input."),
    ("{1:1}/2a", 'invalid input syntax for type sparsevec: "{1:1}/2a"', "Junk after closing."),
    ("{1:1,1:1}/2", "sparsevec indices must not contain duplicates", ""),
    ("{0:1}/3", "sparsevec index out of bounds", ""),
    ("{}/0", "sparsevec must have at least 1 dimension", ""),
])
def test_sparsevec_in_errors(lit, msg, detail):
    row, m, d = T.sparse_in(lit)
    assert row is None and (m, d) == (msg, detail)


def test_sparsevec_in_drops_zeros_and_sorts():
    (dim, idx, val), m, _ = T.sparse_in("{5:0,3:2,1:1}/3")
    assert m is None and dim == 3 and list(idx) == [0, 2] and list(val) == [1, 2]


def test_float_layout_rule():
    # fixed notation for a first-digit exponent in [-4, 6), else d[.ddd]e+-XX with two or more exponent digits
    for v, s in ((1e6, "1e+06"), (999999, "999999"), (1.6777216e7, "1.6777216e+07"), (1e-4, "0.0001"), (1e-5, "1e-05"),
                 (150000, "150000"), (1.5e-38, "1.5e-38"), (1e-45, "1e-45"), (-0.0, "-0"), (1.23456, "1.23456"),
                 (np.inf, "Infinity"), (-np.inf, "-Infinity"), (np.nan, "NaN")):
        assert T.format_float4(np.float32(v)) == s


def test_shortest_digits_agree_with_numpy():
    rng = np.random.default_rng(1)
    bits = rng.integers(1, 0x7f800000, 3000, dtype=np.uint32)
    for v in bits.view(np.float32):
        assert T.shortest(v) == T.numpy_digits(v)


def test_shortest_digit_ties_go_to_even():
    # 2729066.75 lies exactly between the 8-digit decimals 2729066.7 and 2729066.8, and both read back: the even
    # digit wins, as in Ryu (PostgreSQL's f2s) and numpy
    assert T.shortest(np.float32(2729066.75)) == ("27290668", 6)
    assert T.numpy_digits(np.float32(2729066.75)) == ("27290668", 6)
    assert T.format_float4(np.float32(2729066.75)) == "2.7290668e+06"


def test_known_answers():
    import json
    import os
    kat = json.load(open(os.path.join(os.path.dirname(__file__), "golden", "text_io_kat.json")))["cases"]
    assert len(kat) >= 120
    for c in kat:
        if c.get("typmod_in"):
            continue
        if c["type"] == "sparsevec":
            r, m, d = T.sparse_in(c["literal"], c["typmod"])
            got = T.sparsevec_out(*r) if r else None
        else:
            r, m, d = T.dense_in(c["type"] == "halfvec", c["literal"], c["typmod"])
            got = T.vector_out(r, c["type"] == "halfvec") if r is not None else None
        if "error" in c:
            assert r is None and (m, d) == (c["error"], c["detail"]), c
        else:
            assert got == c["output"], c
