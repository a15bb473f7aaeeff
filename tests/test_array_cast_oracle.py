"""The restatement of array_to_sparsevec and of the numeric[] casts (tests/array_cast_oracle.py) against the
reference's known answers (cast.out: tests/golden/array_cast_kat.json), the order of their checks, and the numeric_send
encoder.  No GPU needed."""
import decimal
import struct

import numpy as np
import pytest

from tests import array_cast_oracle as A

CASES = A.kat_cases()


@pytest.mark.parametrize("case", CASES, ids=[c["source"] for c in CASES])
def test_known_answers(case):
    if "error" in case:
        with pytest.raises(A.CastError) as e:
            A.kat_answer(case)
        assert str(e.value) == case["error"]
    else:
        assert A.kat_answer(case) == case["expected"]


def test_kept_values():
    # -0 and doubles that round to 0 are dropped; subnormals, int32 extremes and values rounded by (float) are kept
    x = np.array([[0.0, -0.0, 1e-46, -1e-46, 1e-40, 0.1, 2.0**-149, -(2.0**-149) * 0.75]])
    off, idx, val = A.array_to_sparsevec(x)
    assert idx.tolist() == [4, 5, 6, 7]
    assert val.tolist() == [np.float32(1e-40), np.float32(0.1), np.float32(2.0**-149), -np.float32(2.0**-149)]
    i = np.array([[0, 2**31 - 1, -2**31, 16777217]], dtype=np.int32)
    off, idx, val = A.array_to_sparsevec(i)
    assert val.tolist() == [2.0**31, -2.0**31, 16777216.0]


def test_error_order():
    nan, inf = float("nan"), float("inf")
    # within a row: CheckNnz before CheckElement, then the first special value in index order
    row = np.ones((1, 16001))
    row[0, 5] = nan
    with pytest.raises(A.CastError, match="non-zero elements"):
        A.array_to_sparsevec(row)
    with pytest.raises(A.CastError, match="infinite"):
        A.array_to_sparsevec(np.array([[0, inf, nan]], dtype=np.float32))
    with pytest.raises(A.CastError, match="NaN"):
        A.array_to_sparsevec(np.array([[0, nan, inf]], dtype=np.float32))
    # across rows: the lowest failing row wins, whatever its error
    rows = np.zeros((3, 16001))
    rows[2] = 1
    rows[1, 7] = 4e38
    with pytest.raises(A.CastError) as e:
        A.array_to_sparsevec(rows)
    assert (e.value.row, str(e.value)) == (1, "infinite value not allowed in sparsevec")
    # the dimension checks come before any element
    with pytest.raises(A.CastError, match="expected 3 dimensions, not 2"):
        A.array_to_sparsevec(np.array([[nan, 1.0]]), typmod=3)


# ------------------------------------------------------------------------------- numeric[]

D = decimal.Decimal
EXACT = decimal.Context(prec=400)   # enough for the exact expansion of any float32 and of its halfway points


def test_numeric_send_round_trip():
    from pgvector_b200.numeric import numeric_send
    cases = {"0": "0", "0.000": "0.000", "-0": "0", "1": "1", "1.0": "1.0", "-0.00012": "-0.00012", "1E+5": "100000",
             "12345.678": "12345.678", "1.23E-7": "0.000000123", "10000": "10000", "0.0001": "0.0001",
             "123456789.123456789": "123456789.123456789"}
    for lit, text in cases.items():
        f = numeric_send(D(lit))
        assert A.field_check(f) is None
        assert A.numeric_out(f) == text, lit
    # the layout of one value: ndigits, weight, sign, dscale, base-10000 digits without leading or trailing zero groups
    assert numeric_send(D("-12345.678")) == struct.pack(">hhHH3h", 3, 1, 0x4000, 3, 1, 2345, 6780)
    assert numeric_send(D("NaN"))[4:6] == b"\xc0\x00" and numeric_send(D("-Infinity"))[4:6] == b"\xf0\x00"
    rng = np.random.default_rng(1)
    for _ in range(300):
        d = D(int(rng.integers(-10**12, 10**12))).scaleb(int(rng.integers(-30, 30)))
        assert D(A.numeric_out(numeric_send(d))) == d


def test_exact_float32_expansions_read_back():
    from pgvector_b200.numeric import numeric_send
    rng = np.random.default_rng(2)
    bits = rng.integers(0, 0x7F800000, size=400, dtype=np.int64).astype(np.uint32)
    bits[:4] = [1, 0x007FFFFF, 0x00800000, 0x7F7FFFFF]
    for b in bits:
        x = np.uint32(b).view(np.float32)
        for s in (1, -1):
            assert A.numeric_float4(numeric_send(EXACT.multiply(D(float(x)), s))).view(np.uint32) == (x * s).view(np.uint32)


def test_numeric_rules():
    from pgvector_b200.numeric import numeric_send
    f4 = lambda s: A.numeric_float4(numeric_send(D(s)))   # noqa: E731
    # the 2^-150 boundary: exactly half the least subnormal rounds to 0 and fails; above it is 2^-149
    half = EXACT.power(D(2), -150)
    with pytest.raises(A.CastError, match="out of range for type real"):
        f4(format(half, "f"))
    assert f4(format(EXACT.add(half, D("1e-200")), "f")).view(np.uint32) == 1
    assert f4("1e-40") == np.float32(1e-40)
    # FLT_MAX plus half an ulp rounds up to infinity and fails; one unit below it stays FLT_MAX
    top = EXACT.subtract(EXACT.power(D(2), 128), EXACT.power(D(2), 103))
    with pytest.raises(A.CastError, match='^"340282356779733661637539395458142568448" is out of range for type real$'):
        f4(top)
    assert f4(EXACT.subtract(top, 1)) == np.finfo(np.float32).max
    # zero with the negative sign is +0; digits past dscale are truncated
    neg_zero = struct.pack(">hhHH1h", 1, 0, 0x4000, 0, 0)
    assert A.numeric_float4(neg_zero).view(np.uint32) == 0
    trunc = struct.pack(">hhHH2h", 2, 0, 0x0000, 2, 1, 2399)   # 1.2399 printed with dscale 2: 1.23
    assert A.numeric_out(trunc) == "1.23" and A.numeric_float4(trunc) == np.float32("1.23")


def test_numeric_error_order():
    from pgvector_b200.numeric import numeric_send
    big, nan = numeric_send(D("1e39")), numeric_send(D("NaN"))
    one = numeric_send(D(1))
    # vector: the whole row converts first, so a range error at element 2 beats a NaN at element 1
    with pytest.raises(A.CastError, match="out of range for type real"):
        A.numeric_to_rows("vector", [[one, nan, big]])
    # halfvec: element by element, so its range error at element 1 beats the real range error at element 2
    with pytest.raises(A.CastError, match='^"65520" is out of range for type halfvec$'):
        A.numeric_to_rows("halfvec", [[one, numeric_send(D(65520)), big]])
    # sparsevec: the count loop's range error beats an earlier NaN; CheckNnz beats a NaN
    with pytest.raises(A.CastError, match="out of range for type real"):
        A.numeric_to_sparsevec([[nan, big]])
    with pytest.raises(A.CastError, match="non-zero elements"):
        A.numeric_to_sparsevec([[nan] + [one] * 16000])
    # a malformed field wins over every data error, in any row
    with pytest.raises(A.FieldError) as e:
        A.numeric_to_rows("vector", [[big, one], [one, one[:-1]]])
    assert (str(e.value), e.value.field) == ("insufficient data left in message", 3)
    for f, text in ((one + b"\0", "incorrect binary data format"), (one[:4] + b"\x12\x34" + one[6:], 'invalid sign in external "numeric" value'),
                    (one[:6] + b"\x40\x00" + one[8:], 'invalid scale in external "numeric" value'),
                    (one[:8] + b"\x27\x10", 'invalid digit in external "numeric" value')):
        assert A.FIELD_ERRORS[A.field_check(f)] == text
