"""array_to_sparsevec on the device (vb_array_to_sparsevec_batch[_dev], pgvector_b200.sparsevec.array_to_sparsevec):
integer[] / real[] / double precision[] / numeric[] rows to sparsevec CSR; and numeric[] rows to vector and halfvec
(vb_numeric_array_to_rows_batch[_dev], array_to_vector / array_to_halfvec of Decimal rows or NumericArrays).

Both variants are checked bit for bit against the numpy restatement (tests/array_cast_oracle.py), which itself
reproduces the reference's answers (cast.out: tests/golden/array_cast_kat.json).  The first tests need no device."""
import ctypes as C
import decimal
import os
import struct

import numpy as np
import pytest

from tests import array_cast_oracle as A

EINVAL = -1
gpu = pytest.mark.gpu
SOURCES = [np.int32, np.float32, np.float64]


def test_the_new_symbols_are_exported_and_bound():
    from pgvector_b200 import _lib
    if not os.path.exists(_lib.LIB_PATH):
        import __graft_entry__
        __graft_entry__.build()
    lib = C.CDLL(_lib.LIB_PATH)
    for name in ("vb_array_to_sparsevec_batch", "vb_array_to_sparsevec_batch_dev", "vb_numeric_array_to_rows_batch",
                 "vb_numeric_array_to_rows_batch_dev"):
        assert hasattr(lib, name), name
        assert name in _lib.SIGNATURES, name


# ------------------------------------------------------------------------------- helpers

@pytest.fixture(scope="module")
def pv():
    import pgvector_b200 as pv
    pv.init(0)
    return pv


def _bits(a):
    return np.ascontiguousarray(a, dtype=np.float32).view(np.int32)


def _same(got, want):
    off, idx, val = got
    assert np.array_equal(off, want[0])
    assert np.array_equal(idx, want[1])
    assert np.array_equal(_bits(val), _bits(want[2]))


def _host(pv, x, typmod=-1, cap=None):
    R = pv.sparsevec.array_to_sparsevec(x, typmod, cap)
    return R.row_off, R.idx, R.val


def _device(pv, x, typmod=-1, cap=None):
    import torch
    off, idx, val = pv.sparsevec.array_to_sparsevec(torch.from_numpy(np.ascontiguousarray(x)).cuda(), typmod, cap)
    return off.cpu().numpy(), idx.cpu().numpy(), val.cpu().numpy()


def _both(pv, x, typmod=-1):
    """both variants against the restatement: the same CSR bits, or the same error text and row"""
    try:
        want = A.array_to_sparsevec(x, typmod)
    except A.CastError as e:
        for run in (_host, _device):
            with pytest.raises(pv.sparsevec.ArrayCastError) as got:
                run(pv, x, typmod)
            assert (str(got.value), got.value.row) == (str(e), e.row), run.__name__
        return None
    _same(_host(pv, x, typmod), want)
    _same(_device(pv, x, typmod), want)
    return want


def _rows(rng, dtype, n, dim, density):
    """n rows with about density of their elements non-zero, of values that stay finite as float"""
    mask = rng.random((n, dim)) < density
    if dtype == np.int32:
        v = rng.integers(-2**31, 2**31 - 1, size=(n, dim), dtype=np.int64).astype(np.int32)
        v[v == 0] = 7
    else:
        v = (rng.standard_normal((n, dim)) * 10.0 ** rng.integers(-30, 30, size=(n, dim))).astype(dtype)
        v[v == 0] = 1
    return np.where(mask, v, 0).astype(dtype)


# ------------------------------------------------------------------------------- the reference's answers

@gpu
@pytest.mark.parametrize("case", A.kat_cases(), ids=[c["source"] for c in A.kat_cases()])
def test_known_answers(pv, case):
    rows = A.kat_rows(case)
    typ = case["type"]
    for dev in (False, True):
        if case["src"] == "numeric":
            data, off = A.pack(A.fields_of(rows))
            x = pv.numeric.NumericArrays(data, off, len(rows[0]))
            x = x.cuda() if dev else x
        else:
            import torch
            x = torch.from_numpy(rows).cuda() if dev else rows
        run = {"sparsevec": lambda: pv.sparsevec.array_to_sparsevec(x, case["typmod"]),
               "vector": lambda: pv.array_to_vector(x, case["typmod"]), "halfvec": lambda: pv.array_to_halfvec(x, case["typmod"])}[typ]
        if "error" in case:
            with pytest.raises(ValueError) as e:
                run()
            assert str(e.value) == case["error"]
            continue
        got = run()
        if typ == "sparsevec":
            off_, idx, val = (got.row_off, got.idx, got.val) if not dev else (t.cpu().numpy() for t in got)
            assert A.format_row(len(rows[0]), idx, val) == case["expected"]
        else:
            g = got.cpu().numpy() if dev else got
            assert A.format_dense(typ, g[0].view(np.uint16) if typ == "halfvec" else g[0]) == case["expected"]


# ------------------------------------------------------------------------------- bit identity with the restatement

@gpu
@pytest.mark.parametrize("dtype", SOURCES, ids=["int4", "float4", "float8"])
@pytest.mark.parametrize("dim", [1, 31, 32, 33, 16001, 30522, 250000])
@pytest.mark.parametrize("density", [0.0, 0.01, 0.5, 1.0])
def test_random_rows(pv, dtype, dim, density):
    rng = np.random.default_rng(dim * 7 + int(density * 100))
    n = max(1, min(2000, 2_000_000 // dim))
    x = _rows(rng, dtype, n, dim, density)
    if dim > 16000 and density >= 0.5:
        # rows over the limit fail at the first of them; then only the last row can
        _both(pv, x)
        x[: n - 1] = 0
    _both(pv, x)


@gpu
@pytest.mark.parametrize("dtype", SOURCES, ids=["int4", "float4", "float8"])
def test_many_rows(pv, dtype):
    rng = np.random.default_rng(5)
    _both(pv, _rows(rng, dtype, 100_000, 32, 0.3))
    _both(pv, _rows(rng, dtype, 20_000, 768, 0.05))


@gpu
def test_four_long_rows(pv):
    # 4 rows of 50M elements: too few rows to fill the device, so each is split; on the host each row is a chunk
    rng = np.random.default_rng(11)
    dim = 50_000_000
    x = np.zeros((4, dim), dtype=np.float32)
    for r in range(4):
        at = rng.choice(dim, size=4000 + 3000 * r, replace=False)
        x[r, at] = rng.standard_normal(at.size).astype(np.float32) + 3
    _both(pv, x)
    x[2, rng.choice(dim, size=16001 - 10000, replace=False)] = 1.5   # row 2 over the limit (and row 3 still under)
    x[3, 17] = np.nan
    _both(pv, x)


@gpu
def test_special_values(pv):
    nan, inf = float("nan"), float("inf")
    tiny = [2.0**-149, -(2.0**-149), 2.0**-126 * 0.5, 1e-40, -1e-40]
    _both(pv, np.array([[0.0, -0.0] + tiny], dtype=np.float32))
    _both(pv, np.array([[0.0, -0.0, 1e-46, -1e-46, 2.0**-150, 2.0**-150 * 1.0000001, 3.4028235677973366e38] + tiny]))
    _both(pv, np.array([[0, 1, -1, 2**31 - 1, -2**31, 16777217, -16777219]], dtype=np.int32))
    for dtype in (np.float32, np.float64):
        for v in (nan, inf, -inf):
            _both(pv, np.array([[0, 1, v, 0]], dtype=dtype))
    _both(pv, np.array([[4e38, 0], [-4e38, 0]]))


# ------------------------------------------------------------------------------- errors

@gpu
@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_error_order_with_several_offenders(pv, dtype):
    nan, inf = float("nan"), float("inf")
    dim = 16005
    x = np.zeros((6, dim), dtype=dtype)
    x[1, 100], x[1, 50] = nan, inf          # row 1: the infinity comes first in index order
    x[2, :16001] = 1                        # row 2: CheckNnz ...
    x[2, 3] = nan                           # ... beats its earlier NaN
    x[4, 9] = nan
    _both(pv, x)                            # row 1, infinite
    x[1] = 0
    _both(pv, x)                            # row 2, CheckNnz
    x[2] = 0
    _both(pv, x)                            # row 4, NaN
    # the same in long rows that are split across warps
    y = np.zeros((3, 250_000), dtype=dtype)
    y[1, 200_000] = nan
    y[1, 240_000] = inf
    y[2, ::15] = 1                          # 16667 kept in row 2
    _both(pv, y)
    y[1] = 0
    _both(pv, y)


@gpu
def test_dimension_checks_and_refusals(pv):
    S = pv.sparsevec
    lib = pv._lib.load()
    for run in (_host, _device):
        with pytest.raises(ValueError, match="^expected 7 dimensions, not 6$"):
            run(pv, np.full((2, 6), np.nan, np.float32), 7)
        with pytest.raises(ValueError, match="^sparsevec must have at least 1 dimension$"):
            run(pv, np.zeros((3, 0), np.float32))
    with pytest.raises(ValueError, match="unsupported array type"):
        S.array_to_sparsevec(np.zeros((1, 3), np.int64))
    off = np.zeros(2, np.int64)
    bad = C.c_int64(5)
    x = np.ones((1, 3), np.float32)
    p = lambda a: a.ctypes.data_as(C.c_void_p)
    assert lib.vb_array_to_sparsevec_batch(4, 3, -1, p(x), None, 1, 0, p(off), None, None, C.byref(bad)) == EINVAL
    assert "bad source type 4" in lib.vb_last_error().decode() and bad.value == -1
    assert lib.vb_array_to_sparsevec_batch(3, 3, -1, p(x), None, 1, 0, p(off), None, None, C.byref(bad)) == EINVAL
    assert "in_off is required for numeric[]" in lib.vb_last_error().decode()
    assert lib.vb_array_to_sparsevec_batch(1, 1_000_000_001, -1, p(x), None, 1, 0, p(off), None, None, C.byref(bad)) == EINVAL
    assert lib.vb_last_error().decode() == "sparsevec cannot have more than 1000000000 dimensions"
    # the refused array_to_vector source stays refused
    out = np.zeros(3, np.float32)
    assert lib.vb_array_to_rows_batch(0, 3, 3, -1, p(x), 1, p(out)) == EINVAL


@gpu
def test_cap_and_sizing(pv):
    import torch
    lib = pv._lib.load()
    rng = np.random.default_rng(3)
    x = _rows(rng, np.float64, 500, 3000, 0.02)
    want = A.array_to_sparsevec(x)
    total = int(want[0][-1])
    n, dim = x.shape
    p = lambda a: a.ctypes.data_as(C.c_void_p)
    xd = torch.from_numpy(x).cuda()
    torch.cuda.synchronize()   # the raw calls below run on the library stream
    bad = C.c_int64(0)
    for dev in (False, True):
        fn = lib.vb_array_to_sparsevec_batch_dev if dev else lib.vb_array_to_sparsevec_batch
        tp = (lambda t: C.c_void_p(t.data_ptr())) if dev else p
        mk = (lambda k, dt: torch.empty(k, dtype=dt, device="cuda")) if dev else (lambda k, dt: np.empty(k, dt))
        src = xd if dev else x
        off = mk(n + 1, torch.int64 if dev else np.int64)
        # a sizing call writes the offsets and names the total
        assert fn(2, dim, -1, tp(src), None, n, 0, tp(off), None, None, C.byref(bad)) == EINVAL
        assert f"the rows have {total} non-zero elements, more than cap = 0" in lib.vb_last_error().decode()
        pv.synchronize()
        got_off = off.cpu().numpy() if dev else off
        assert np.array_equal(got_off, want[0]) and bad.value == -1
        # one short of the total fails the same way; the exact total succeeds
        idx, val = mk(total, torch.int32 if dev else np.int32), mk(total, torch.float32 if dev else np.float32)
        assert fn(2, dim, -1, tp(src), None, n, total - 1, tp(off), tp(idx), tp(val), C.byref(bad)) == EINVAL
        assert fn(2, dim, -1, tp(src), None, n, total, tp(off), tp(idx), tp(val), C.byref(bad)) == 0
        pv.synchronize()
        if dev:
            idx, val = idx.cpu().numpy(), val.cpu().numpy()
        _same((got_off, idx, val), want)
    # a data error wins over the cap check, so a sizing call already raises it
    y = x.copy()
    y[321, 5] = np.inf
    for run in (_host, _device):
        with pytest.raises(pv.sparsevec.ArrayCastError) as e:
            run(pv, y, cap=0)
        assert (str(e.value), e.value.row) == ("infinite value not allowed in sparsevec", 321)


@gpu
def test_host_chunks(pv):
    # about 32 MB of source per chunk: 1200 rows of 30522 doubles are 9 chunks; the error sits in the last one
    rng = np.random.default_rng(9)
    x = _rows(rng, np.float64, 1200, 30522, 0.01)
    _same(_host(pv, x), A.array_to_sparsevec(x))
    x[1150, 30000] = np.nan
    x[1190, 3] = np.inf
    _both(pv, x)


@gpu
def test_no_rows_launch_nothing(pv):
    import torch
    before = pv.launch_count()
    for dtype in SOURCES:
        R = pv.sparsevec.array_to_sparsevec(np.zeros((0, 5), dtype))
        assert R.row_off.tolist() == [0] and R.idx.size == 0
        off, idx, val = pv.sparsevec.array_to_sparsevec(torch.zeros((0, 5), dtype=getattr(torch, np.dtype(dtype).name), device="cuda"))
        assert off.cpu().tolist() == [0] and idx.numel() == 0
    assert pv.launch_count() == before


@gpu
def test_device_pipeline_equals_the_host_path(pv):
    # float64 model output -> sparsevec -> resident table -> exact top-k, all on the device, against the host path
    import torch
    S = pv.sparsevec
    rng = np.random.default_rng(21)
    dim = 30522
    x = _rows(rng, np.float64, 1000, dim, 0.004)
    q = _rows(rng, np.float64, 16, dim, 0.01)
    host_t = S.SparseTable(dim).append(S.array_to_sparsevec(x))
    dev_t = S.SparseTable(dim).append(S.array_to_sparsevec(torch.from_numpy(x).cuda()))
    Q = S.array_to_sparsevec(q)
    Qd = S.array_to_sparsevec(torch.from_numpy(q).cuda())
    for metric in (0, 1, 2):
        want = host_t.exact_topk(metric, Q, 10)
        got = dev_t.exact_topk(metric, Qd, 10)
        assert np.array_equal(got[0].cpu().numpy(), want[0])
        assert np.array_equal(_bits(got[1].cpu().numpy()), _bits(want[1].astype(np.float32)))


# ------------------------------------------------------------------------------- numeric[]

D = decimal.Decimal
EXACT = decimal.Context(prec=5000)


def _num_run(pv, typ, x, typmod=-1):
    if typ == "sparsevec":
        got = pv.sparsevec.array_to_sparsevec(x, typmod)
        return (got.row_off, got.idx, got.val) if isinstance(got, pv.sparsevec.SparseRows) else tuple(t.cpu().numpy() for t in got)
    got = (pv.array_to_vector if typ == "vector" else pv.array_to_halfvec)(x, typmod)
    g = got if isinstance(got, np.ndarray) else got.cpu().numpy()
    return g.view(np.uint16) if typ == "halfvec" else g


def _num_both(pv, typ, fields, typmod=-1):
    """rows of numeric field bytes through the host and _dev variants against the restatement: the same bits, or the
    same error (a malformed field: the library's refusal naming it)"""
    from pgvector_b200 import VecB200Error
    data, off = A.pack(fields)
    x = pv.numeric.NumericArrays(data, off, len(fields[0]))
    try:
        want = A.numeric_to_sparsevec(fields, typmod) if typ == "sparsevec" else A.numeric_to_rows(typ, fields, typmod)
    except A.FieldError as e:
        for arg in (x, x.cuda()):
            with pytest.raises(VecB200Error) as got:
                _num_run(pv, typ, arg, typmod)
            assert str(got.value).endswith(f"numeric field {e.field}: {e}"), str(got.value)
        return None
    except A.CastError as e:
        for arg in (x, x.cuda()):
            with pytest.raises(ValueError) as got:
                _num_run(pv, typ, arg, typmod)
            assert str(got.value) == str(e)
            if typ == "sparsevec":
                assert got.value.row == e.row
        return None
    for arg in (x, x.cuda()):
        got = _num_run(pv, typ, arg, typmod)
        if typ == "sparsevec":
            _same(got, want)
        else:
            assert np.array_equal(got.view(np.uint32 if typ == "vector" else np.uint16), want.view(np.uint32 if typ == "vector" else np.uint16))
    return want


def _random_decimals(rng, n, lo=-37, hi=37):
    """decimals of 1 to 40 significant digits, magnitudes 10^lo .. 10^hi, either sign, some zero"""
    out = []
    for _ in range(n):
        k = int(rng.integers(1, 41))
        digits = "".join(str(int(d)) for d in rng.integers(0, 10, size=k))
        d = D(("-" if rng.random() < 0.5 else "") + "0." + digits).scaleb(int(rng.integers(lo, hi)) + 1, EXACT)
        out.append(D(0) if rng.random() < 0.05 else d)
    return out


def _midpoints(rng, n):
    """exact float32 midpoints between neighbours (normal and subnormal), each one, and each +- 10^-k of its ulp"""
    out = []
    for b in rng.integers(1, 0x7F7FFFFF, size=n, dtype=np.int64):
        x = np.uint32(b).view(np.float32)
        y = np.nextafter(x, np.float32(np.inf))
        m = EXACT.divide(EXACT.add(D(float(x)), D(float(y))), 2)
        ulp = EXACT.subtract(D(float(y)), D(float(x)))
        out.append(m)
        for k in (1, 5, 20, 60, 200, 2000):
            d = EXACT.multiply(ulp, D(10) ** -k)
            out += [EXACT.add(m, d), EXACT.subtract(m, d)]
    return out


@gpu
@pytest.mark.parametrize("typ", ["vector", "halfvec", "sparsevec"])
def test_numeric_random_decimals(pv, typ):
    rng = np.random.default_rng({"vector": 1, "halfvec": 2, "sparsevec": 3}[typ])
    hi = 4 if typ == "halfvec" else 37
    for dim in (1, 31, 33):
        vals = _random_decimals(rng, 60 * dim, hi=hi)
        _num_both(pv, typ, A.fields_of([vals[r * dim:(r + 1) * dim] for r in range(60)]))


@gpu
@pytest.mark.parametrize("typ", ["vector", "sparsevec"])
def test_numeric_midpoints_and_long_digit_strings(pv, typ):
    rng = np.random.default_rng(4)
    vals = _midpoints(rng, 40)
    dim = 13
    vals += [D(0)] * (-len(vals) % dim)
    fields = A.fields_of([vals[i:i + dim] for i in range(0, len(vals), dim)])
    assert max(len(f) for row in fields for f in row) > 1000          # thousands of digits
    _num_both(pv, typ, fields)


@gpu
def test_numeric_boundaries_and_specials(pv):
    top = EXACT.subtract(EXACT.power(D(2), 128), EXACT.power(D(2), 103))     # FLT_MAX plus half an ulp
    tiny = EXACT.power(D(2), -150)                                         # half the least subnormal
    ok = [EXACT.subtract(top, 1), EXACT.minus(EXACT.subtract(top, 1)), EXACT.add(tiny, D("1e-300")), D("1e-40"), D("-1e-45"), D(0),
          D("0.000")]
    neg_zero = struct.pack(">hhHH", 0, 0, 0x4000, 2)
    for typ in ("vector", "sparsevec"):
        _num_both(pv, typ, A.fields_of([ok + [neg_zero]]))
        for bad in (top, EXACT.minus(top), tiny, EXACT.minus(tiny), D("1e39"), D("1e-46"), D("NaN"), D("Infinity"), D("-Infinity")):
            _num_both(pv, typ, A.fields_of([[D(1)] * 3, [D(2), bad, D(3)]]))
    _num_both(pv, "halfvec", A.fields_of([[D("65519.99"), D("-65504"), D("1e-8"), neg_zero]]))
    for bad in (D("65520"), D("1e39"), D("NaN"), D("-Infinity")):
        _num_both(pv, "halfvec", A.fields_of([[D(1), bad]]))


@gpu
def test_numeric_error_order(pv):
    one, nan, big, inf = D(1), D("NaN"), D("1e39"), D("Infinity")
    # vector: a range error after a NaN in the row wins (the row converts first); across rows the lowest row
    _num_both(pv, "vector", A.fields_of([[one] * 12, [one, nan, one, one, one, one, one, one, one, big, one, one]]))
    _num_both(pv, "vector", A.fields_of([[one, inf, one], [big, one, one], [nan, one, one]]))
    # halfvec: element by element, so its range error beats a later numeric range error, and an earlier one wins
    _num_both(pv, "halfvec", A.fields_of([[one, nan, D(70000), big]]))
    _num_both(pv, "halfvec", A.fields_of([[one, big, D(70000)]]))
    # sparsevec: the count loop's range error beats an earlier NaN; CheckNnz beats a NaN; the lowest row first
    _num_both(pv, "sparsevec", A.fields_of([[nan, one, big]]))
    _num_both(pv, "sparsevec", A.fields_of([[nan] + [one] * 16000, [big] * 16001]))
    _num_both(pv, "sparsevec", A.fields_of([[one] * 16001, [big] * 16001]))


@gpu
def test_numeric_malformed_fields_are_refused_first(pv):
    one = A.fields_of([[D(1)]])[0][0]
    big = A.fields_of([[D("1e39")]])[0][0]
    bad = [one[:-1], one[:5], one + b"\0", one[:4] + b"\x12\x34" + one[6:], one[:6] + b"\x40\x00" + one[8:], one[:8] + b"\x27\x10",
           one[:8] + b"\xff\xff"]
    for f in bad:
        for typ in ("vector", "halfvec", "sparsevec"):
            _num_both(pv, typ, [[big, one], [one, one], [one, f]])   # the data error in row 0 loses to the field in row 2


@gpu
def test_numeric_host_chunks(pv):
    # 2600 rows of 768 fields of 12 bytes plus 8 offset bytes: two host chunks of about 32 MB; the host result equals
    # the _dev one (one pass over all rows), and sampled rows equal the restatement
    rng = np.random.default_rng(8)
    n, dim = 2600, 768
    m = n * dim
    hdr = np.zeros((m, 12), dtype=np.uint8)
    sign = np.where(rng.random(m) < 0.5, 0x40, 0x00).astype(np.uint8)
    d0, d1 = rng.integers(0, 10000, size=m), rng.integers(0, 10000, size=m)
    hdr[:, 1] = 2                          # ndigits 2, weight 0, dscale 4
    hdr[:, 4] = sign
    hdr[:, 7] = 4
    hdr[:, 8], hdr[:, 9] = d0 >> 8, d0 & 0xFF
    hdr[:, 10], hdr[:, 11] = d1 >> 8, d1 & 0xFF
    data = hdr.reshape(-1).copy()
    off = np.arange(m + 1, dtype=np.int64) * 12
    x = pv.numeric.NumericArrays(data, off, dim)
    for typ in ("vector", "sparsevec"):
        host, dev = _num_run(pv, typ, x), _num_run(pv, typ, x.cuda())
        if typ == "vector":
            assert np.array_equal(host.view(np.uint32), dev.view(np.uint32))
            rows = [[bytes(hdr[r * dim + i]) for i in range(dim)] for r in (0, 1300, n - 1)]
            want = A.numeric_to_rows("vector", rows)
            assert np.array_equal(host[[0, 1300, n - 1]].view(np.uint32), want.view(np.uint32))
        else:
            _same(host, dev)
    # an error in the last chunk names its row
    hdr[(n - 2) * dim + 5, 4] = 0xC0     # NaN
    x = pv.numeric.NumericArrays(hdr.reshape(-1).copy(), off, dim)
    for arg in (x, x.cuda()):
        with pytest.raises(pv.sparsevec.ArrayCastError) as e:
            pv.sparsevec.array_to_sparsevec(arg)
        assert (str(e.value), e.value.row) == ("NaN not allowed in sparsevec", n - 2)
        with pytest.raises(ValueError, match="^NaN not allowed in vector$"):
            pv.array_to_vector(arg)


@gpu
def test_numeric_decimal_rows_and_empty_batches(pv):
    import torch
    rows = [[D("1.5"), D("-0.25"), D("0")], [D("1e-3"), D("2"), D("0.1")]]
    assert np.array_equal(pv.array_to_vector(rows), np.array([[1.5, -0.25, 0], [1e-3, 2, 0.1]], dtype=np.float32))
    assert np.array_equal(pv.array_to_vector(rows[0]), np.array([1.5, -0.25, 0], dtype=np.float32))
    assert pv.sparsevec.array_to_sparsevec(rows).idx.tolist() == [0, 1, 0, 1, 2]
    before = pv.launch_count()
    empty = pv.numeric.NumericArrays(np.zeros(1, np.uint8), np.zeros(1, np.int64), 4)
    assert pv.array_to_vector(empty).shape == (0, 4)
    assert pv.sparsevec.array_to_sparsevec(empty).row_off.tolist() == [0]
    e2 = empty.cuda()
    assert tuple(pv.array_to_halfvec(e2).shape) == (0, 4)
    assert pv.sparsevec.array_to_sparsevec(e2)[0].cpu().tolist() == [0]
    assert pv.launch_count() == before
