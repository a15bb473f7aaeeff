"""The operators + - * || of vector and halfvec and the array casts (integer[] / real[] / double precision[] to vector /
halfvec) over batches of rows, host and device.

A numpy restatement of the six reference functions (row-by-row semantics, including which error a batch raises first)
reproduces the reference's answers (vector_type.out, halfvec.out, cast.out: tests/golden/row_arith_kat.json) without a
device.  On the device every result is compared with the restatement bit for bit (bit patterns, so NaN and -0 count);
numpy's float32 arithmetic and astype conversions round to nearest even, so the restatement is exact."""
import ctypes as C
import json
import os

import numpy as np
import pytest

EINVAL, ENODEVICE = -1, -2
VECTOR, HALFVEC = 0, 1
ADD, SUB, MUL = 0, 1, 2
INT4, FLOAT4, FLOAT8 = 0, 1, 2
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "row_arith_kat.json")
NEW_SYMBOLS = ["vb_arith_batch", "vb_arith_batch_dev", "vb_concat_batch", "vb_concat_batch_dev", "vb_array_to_rows_batch",
               "vb_array_to_rows_batch_dev"]
NAME = {VECTOR: "vector", HALFVEC: "halfvec"}
OPS = {"add": ADD, "sub": SUB, "mul": MUL}
SRC = {"int4": INT4, "float4": FLOAT4, "float8": FLOAT8}
SRC_DTYPE = {INT4: np.int32, FLOAT4: np.float32, FLOAT8: np.float64}


# ------------------------------------------------------------------------------- the restatement

def _f(elem, x):
    """element values as float32 (halfvec rows are binary16 bit patterns)"""
    return x.view(np.float16).astype(np.float32) if elem == HALFVEC else x


def _half_bits(f):
    with np.errstate(over="ignore"):
        return f.astype(np.float16).view(np.uint16)


def _first(mask, kinds, passes=None):
    """(row, kind) of the first offender in the reference's order: row, then pass, then element; None if none"""
    n, dim = mask.shape
    if not mask.any():
        return None
    key = np.where(mask, (np.arange(n)[:, None] * 2 + (0 if passes is None else passes)) * dim + np.arange(dim)[None, :], np.iinfo(np.int64).max)
    i = np.unravel_index(int(np.argmin(key)), key.shape)
    return i, kinds[i]


def arith_ref(elem, op, a, b):
    """a op b of rows a [na, dim] and b [nb, dim] (one of the counts may be 1): (out, None) or (None, error text)"""
    if a.shape[1] != b.shape[1]:
        return None, f"different {NAME[elem]} dimensions {a.shape[1]} and {b.shape[1]}"
    x, y = _f(elem, a), _f(elem, b)
    with np.errstate(all="ignore"):
        r = x + y if op == ADD else x - y if op == SUB else x * y
    if elem == VECTOR:
        out, inf, zero = r, np.isinf(r), r == 0
        nz = (x != 0) & (y != 0)
    else:
        out = _half_bits(r)
        inf, zero = (out & 0x7FFF) == 0x7C00, (out & 0x7FFF) == 0
        nz = ((a & 0x7FFF) != 0) & ((b & 0x7FFF) != 0)
    under = zero & nz if op == MUL else np.zeros_like(inf)
    bad = _first(inf | under, np.where(inf, "overflow", "underflow"))
    if bad is not None:
        return None, f"value out of range: {bad[1]}"
    return out, None


def concat_ref(elem, a, b):
    if a.shape[1] + b.shape[1] > 16000:
        return None, f"{NAME[elem]} cannot have more than 16000 dimensions"
    m = a.shape[0] if b.shape[0] == 1 else b.shape[0]
    return np.concatenate([np.broadcast_to(a, (m, a.shape[1])), np.broadcast_to(b, (m, b.shape[1]))], axis=1), None


def pg_float4(v):
    """float_to_shortest_decimal_buf: the shortest digits that read back, fixed notation for exponents -4 .. 14"""
    s = np.format_float_scientific(np.float32(v), unique=True, trim="-")
    mant, e = s.split("e")
    e = int(e)
    if -4 <= e < 15:
        return np.format_float_positional(np.float32(v), unique=True, trim="-")
    return f"{mant}e{'-' if e < 0 else '+'}{abs(e):02d}"


def array_cast_ref(elem, src, rows, typmod=-1):
    """array_to_vector / array_to_halfvec of rows [n, dim] of int32 / float32 / float64"""
    dim = rows.shape[1]
    name = NAME[elem]
    if dim < 1:
        return None, f"{name} must have at least 1 dimension"
    if dim > 16000:
        return None, f"{name} cannot have more than 16000 dimensions"
    if typmod != -1 and typmod != dim:
        return None, f"expected {typmod} dimensions, not {dim}"
    with np.errstate(over="ignore"):
        f = rows.astype(np.float32)
    if elem == VECTOR:
        bad = _first(~np.isfinite(f), np.where(np.isnan(f), "NaN", "infinite value"))
        return (f, None) if bad is None else (None, f"{bad[1]} not allowed in vector")
    h = _half_bits(f)
    hinf = (h & 0x7C00) == 0x7C00
    over = hinf & np.isfinite(f)
    check = hinf & ~over
    bad = _first(over | check, np.where(over, "range", np.where((h & 0x7FFF) != 0x7C00, "NaN", "infinite value")), np.where(over, 0, 1))
    if bad is None:
        return h, None
    (r, c), kind = bad
    if kind == "range":
        return None, f'"{pg_float4(f[r, c])}" is out of range for type halfvec'
    return None, f"{kind} not allowed in halfvec"


# ------------------------------------------------------------------------------- the fixture

def _cases():
    return json.load(open(GOLDEN))["cases"]


def _row(elem, text):
    x = np.array([float(v) for v in text.strip("[]").split(",")], np.float32)
    return (_half_bits(x) if elem == HALFVEC else x).reshape(1, -1)


def _array(src, text):
    body = text.strip("{}")
    vals = [v for v in body.split(",") if v] if body else []
    if src == INT4:
        return np.array([int(v) for v in vals], np.int32).reshape(1, -1)
    return np.array([float(v) for v in vals], SRC_DTYPE[src]).reshape(1, -1)


def _text(elem, out):
    return "[" + ",".join(f"{float(v):g}" for v in _f(elem, np.ascontiguousarray(out)).ravel()) + "]"


def _case_args(c):
    elem = VECTOR if c["type"] == "vector" else HALFVEC
    if c["fn"].startswith("array_to_"):
        return elem, ("cast", SRC[c["src"]], _array(SRC[c["src"]], c["input"]), c["typmod"])
    a = np.zeros((1, c["a_zeros"]), np.float32 if elem == VECTOR else np.uint16) if "a_zeros" in c else _row(elem, c["a"])
    return elem, (c["fn"], a, _row(elem, c["b"]))


def _ref(elem, args):
    if args[0] == "cast":
        return array_cast_ref(elem, args[1], args[2], args[3])
    if args[0] == "concat":
        return concat_ref(elem, args[1], args[2])
    return arith_ref(elem, OPS[args[0]], args[1], args[2])


def test_the_fixture_reads():
    cases = _cases()
    assert len(cases) == 56
    assert all(("expected" in c) != ("error" in c) for c in cases)
    assert all(c["source"].startswith("test/expected/") for c in cases)
    for fn in ("add", "sub", "mul", "concat", "array_to_vector", "array_to_halfvec"):
        assert sum(c["fn"] == fn for c in cases) >= 4, fn


def test_the_restatement_reproduces_every_known_answer():
    for c in _cases():
        elem, args = _case_args(c)
        out, err = _ref(elem, args)
        if "error" in c:
            assert err == c["error"], c["sql"]
        else:
            assert err is None and _text(elem, out) == c["expected"], c["sql"]


def test_the_restated_check_order():
    """the rules the batch follows, on the restatement: lowest row; in a * row the first element; in a halfvec cast a
    range error beats an earlier NaN of its row, and a NaN in an earlier row beats a later range error"""
    a = np.array([[1, 1e-30, 1e30], [1e30, 1, 1]], np.float32)
    b = np.array([[1, 1e-30, 1e30], [1e30, 1, 1]], np.float32)
    assert arith_ref(VECTOR, MUL, a, b)[1] == "value out of range: underflow"
    assert arith_ref(VECTOR, MUL, a[:, ::-1].copy(), b[:, ::-1].copy())[1] == "value out of range: overflow"
    rows = np.array([[1, np.nan, 70000.0], [1, 1, 1]], np.float64)
    assert array_cast_ref(HALFVEC, FLOAT8, rows)[1] == '"70000" is out of range for type halfvec'
    assert array_cast_ref(VECTOR, FLOAT8, rows)[1] == "NaN not allowed in vector"
    rows = np.array([[1, 1, 1], [np.nan, 1, 1], [1, 1, 70000.0]], np.float64)
    assert array_cast_ref(HALFVEC, FLOAT8, rows)[1] == "NaN not allowed in halfvec"
    assert pg_float4(np.float32(65520.0000001)) == "65520" and pg_float4(np.float32(3e38)) == "3e+38"


def test_every_new_symbol_is_exported_and_bound():
    from pgvector_b200 import _lib
    if not os.path.exists(_lib.LIB_PATH):
        import __graft_entry__
        __graft_entry__.build()
    lib = C.CDLL(_lib.LIB_PATH)
    for name in NEW_SYMBOLS:
        assert hasattr(lib, name), name
        assert name in _lib.SIGNATURES, name


def test_without_a_device_every_new_entry_point_is_an_error():
    import torch
    if torch.cuda.is_available():
        pytest.skip("a device is visible")
    import pgvector_b200 as pv
    lib = pv._lib.load()
    d = C.c_int(0)
    assert lib.vb_arith_batch(VECTOR, ADD, 3, None, 0, 3, None, 0, None) == ENODEVICE
    assert lib.vb_arith_batch_dev(HALFVEC, MUL, 3, None, 0, 3, None, 0, None) == ENODEVICE
    assert lib.vb_concat_batch(VECTOR, 3, None, 0, 2, None, 0, None, C.byref(d)) == ENODEVICE
    assert lib.vb_concat_batch_dev(HALFVEC, 3, None, 0, 2, None, 0, None, C.byref(d)) == ENODEVICE
    assert lib.vb_array_to_rows_batch(VECTOR, FLOAT8, 3, -1, None, 0, None) == ENODEVICE
    assert lib.vb_array_to_rows_batch_dev(HALFVEC, INT4, 3, -1, None, 0, None) == ENODEVICE
    assert d.value == 0
    with pytest.raises(pv.VecB200Error) as e:
        pv.vector_add(np.ones(3, np.float32), np.ones(3, np.float32))
    assert e.value.code == ENODEVICE


def test_unsupported_array_types_are_refused_before_the_library():
    import pgvector_b200 as pv
    for dt in (np.int64, np.float16, np.uint8):
        with pytest.raises(ValueError, match="unsupported array type"):
            pv.array_to_vector(np.ones((2, 3), dt))


# ------------------------------------------------------------------------------- helpers

gpu = pytest.mark.gpu


@pytest.fixture(scope="module")
def pv():
    import pgvector_b200 as pv
    pv.init(0)
    return pv


def _bits(a):
    a = a.cpu().numpy() if hasattr(a, "cpu") else np.asarray(a)
    a = np.ascontiguousarray(a)
    return a.view({8: np.uint64, 4: np.uint32, 2: np.uint16, 1: np.uint8}[a.itemsize])


def _same(got, want):
    assert tuple(got.shape) == tuple(np.shape(want)), (tuple(got.shape), np.shape(want))
    assert np.array_equal(_bits(got), _bits(want))


def _cuda(x):
    import torch
    x = np.ascontiguousarray(x)
    return torch.from_numpy(x.view(np.float16) if x.dtype == np.uint16 else x).cuda()


def _special(rng, n, dim, elem):
    """rows with +-0, subnormals, values next to FLT_MAX / 65504 and NaN, no infinities"""
    x = (rng.standard_normal((n, dim)) * 4).astype(np.float32)
    u = rng.random((n, dim))
    if elem == VECTOR:
        big = np.float32(3.4028235e38)
        x[u < 0.02] = -0.0
        x[(u >= 0.02) & (u < 0.04)] = 0.0
        sub = (u >= 0.04) & (u < 0.07)
        x[sub] = (rng.standard_normal(int(sub.sum())) * 1e-39).astype(np.float32)
        near = (u >= 0.07) & (u < 0.09)
        x[near] = np.where(rng.random(int(near.sum())) < 0.5, big, -np.nextafter(big, np.float32(0)))
        tiny = (u >= 0.09) & (u < 0.11)
        x[tiny] = (rng.standard_normal(int(tiny.sum())) * 1e-20).astype(np.float32)
        x[(u >= 0.11) & (u < 0.115)] = np.nan
        return x
    h = _half_bits(x)
    h[u < 0.02] = 0x8000
    h[(u >= 0.02) & (u < 0.04)] = 0
    sub = (u >= 0.04) & (u < 0.07)
    h[sub] = rng.integers(1, 0x400, int(sub.sum())).astype(np.uint16) | (rng.integers(0, 2, int(sub.sum())).astype(np.uint16) << 15)
    near = (u >= 0.07) & (u < 0.09)
    h[near] = np.where(rng.random(int(near.sum())) < 0.5, 0x7BFF, 0xFBFE).astype(np.uint16)   # 65504, -65472
    h[(u >= 0.11) & (u < 0.115)] = 0x7E00
    return h


def _no_errors(elem, op, a, b):
    """patch the operand that is not broadcast with 0 where a result would raise, so the whole output is defined"""
    full_a = a.shape[0] > 1 or b.shape[0] == 1
    for _ in range(2):
        x, y = _f(elem, a), _f(elem, b)
        with np.errstate(all="ignore"):
            r = x + y if op == ADD else x - y if op == SUB else x * y
        if elem == VECTOR:
            bad = np.isinf(r) | ((r == 0) & (x != 0) & (y != 0) if op == MUL else False)
        else:
            h = _half_bits(r)
            bad = ((h & 0x7FFF) == 0x7C00) | (((h & 0x7FFF) == 0) & ((a & 0x7FFF) != 0) & ((b & 0x7FFF) != 0) if op == MUL else False)
        bad = np.broadcast_to(bad, r.shape)
        if not bad.any():
            return a, b
        if full_a and not (b.shape[0] > 1 and a.shape[0] == 1):
            a = a.copy()
            a[bad] = 0
        else:
            b = b.copy()
            b[bad] = 0
    return a, b


def _arith_both(pv, elem, op, a, b):
    """(host result, device result) of the library"""
    fn = {ADD: pv.vector_add, SUB: pv.vector_sub, MUL: pv.vector_mul}[op]
    return fn(a, b, elem), fn(_cuda(a), _cuda(b), elem)


# ------------------------------------------------------------------------------- the known answers

@gpu
@pytest.mark.parametrize("device", [False, True])
def test_every_known_answer(pv, device):
    for c in _cases():
        elem, args = _case_args(c)
        conv = _cuda if device else (lambda x: x)
        try:
            if args[0] == "cast":
                fn = pv.array_to_vector if elem == VECTOR else pv.array_to_halfvec
                got = fn(conv(args[2]), args[3])
            elif args[0] == "concat":
                got = pv.vector_concat(conv(args[1]), conv(args[2]), elem)
            else:
                got = {"add": pv.vector_add, "sub": pv.vector_sub, "mul": pv.vector_mul}[args[0]](conv(args[1]), conv(args[2]), elem)
        except (ValueError, OverflowError) as e:
            assert "error" in c, c["sql"]
            assert str(e) == c["error"], c["sql"]
            assert isinstance(e, OverflowError) == c["error"].startswith("value out of range"), c["sql"]
            continue
        assert "expected" in c, c["sql"]
        got = got.cpu().numpy() if device else got
        if elem == HALFVEC and got.dtype == np.float16:
            got = got.view(np.uint16)
        assert _text(elem, got) == c["expected"], c["sql"]


# ------------------------------------------------------------------------------- bit identity

DIMS = [1, 3, 8, 17, 768, 1536, 16000]


@gpu
@pytest.mark.parametrize("elem", [VECTOR, HALFVEC])
@pytest.mark.parametrize("op", [ADD, SUB, MUL])
def test_arith_equals_the_restatement(pv, elem, op):
    rng = np.random.default_rng(100 + 10 * elem + op)
    shapes = [(n, dim) for dim in DIMS for n in (0, 1, 1000) if n * dim <= 4_000_000] + [(100_000, 17), (100_000, 768)]
    for n, dim in shapes:
        for mode in ("pair", "bcast_a", "bcast_b"):
            na = 1 if mode == "bcast_a" else n
            nb = 1 if mode == "bcast_b" else n
            a, b = _special(rng, na, dim, elem), _special(rng, nb, dim, elem)
            a, b = _no_errors(elem, op, a, b)
            want, err = arith_ref(elem, op, a, b)
            assert err is None
            host, dev = _arith_both(pv, elem, op, a, b)
            _same(host, want)
            _same(dev, want)


@gpu
@pytest.mark.parametrize("elem", [VECTOR, HALFVEC])
def test_concat_equals_the_restatement(pv, elem):
    rng = np.random.default_rng(7 + elem)
    for da, db in [(1, 1), (3, 5), (8, 8), (17, 3), (768, 768), (1536, 17), (15999, 1), (1, 15999)]:
        for n in (0, 1, 1000):
            for na, nb in ((n, n), (1, n), (n, 1)):
                if n * (da + db) > 4_000_000:
                    continue
                a, b = _special(rng, na, da, elem), _special(rng, nb, db, elem)
                want, _ = concat_ref(elem, a, b)
                _same(pv.vector_concat(a, b, elem), want)
                _same(pv.vector_concat(_cuda(a), _cuda(b), elem), want)


@gpu
@pytest.mark.parametrize("elem", [VECTOR, HALFVEC])
@pytest.mark.parametrize("src", [INT4, FLOAT4, FLOAT8])
def test_array_casts_equal_the_restatement(pv, elem, src):
    rng = np.random.default_rng(3 + 3 * elem + src)
    fn = pv.array_to_vector if elem == VECTOR else pv.array_to_halfvec
    for dim in DIMS:
        for n in (0, 1, 1000, 100_000):
            if n * dim > 4_000_000:
                continue
            if src == INT4:
                lim = 60000 if elem == HALFVEC else 2**31 - 1
                x = rng.integers(-lim, lim, (n, dim), dtype=np.int64).astype(np.int32)
            else:
                x = rng.standard_normal((n, dim)) * (1e4 if elem == HALFVEC else 1e30)
                u = rng.random((n, dim))
                x[u < 0.02] = -0.0
                x[(u >= 0.02) & (u < 0.05)] *= 1e-42 if elem == VECTOR else 1e-9   # float / half subnormals and underflow
                if elem == VECTOR:
                    x[(u >= 0.05) & (u < 0.06)] = 3.4028235e38
                else:
                    x[(u >= 0.05) & (u < 0.06)] = 65519.99
                x = x.astype(SRC_DTYPE[src])
            want, err = array_cast_ref(elem, src, x)
            assert err is None, err
            _same(fn(x), want)
            _same(fn(_cuda(x)), want)


@gpu
def test_narrow_word_paths(pv):
    """odd halfvec dims and device pointers one element off their alignment reach the 2- and 4-byte words"""
    import torch
    rng = np.random.default_rng(5)
    lib = pv._lib.load()
    for elem in (VECTOR, HALFVEC):
        es = 4 if elem == VECTOR else 2
        for dim in (3, 17, 1535):
            n = 500
            a, b = _special(rng, n, dim, elem), _special(rng, n, dim, elem)
            a, b = _no_errors(elem, ADD, a, b)
            want, _ = arith_ref(elem, ADD, a, b)
            buf_a = torch.zeros(n * dim * es + 64, dtype=torch.uint8, device="cuda")
            buf_b = torch.zeros_like(buf_a)
            out = torch.zeros(2 * n * dim * es + 64, dtype=torch.uint8, device="cuda")   # room for a || b
            buf_a[es:es + a.nbytes].copy_(torch.from_numpy(a.view(np.uint8).ravel()).cuda())
            buf_b[es:es + b.nbytes].copy_(torch.from_numpy(b.view(np.uint8).ravel()).cuda())
            pa, pb, po = buf_a.data_ptr() + es, buf_b.data_ptr() + es, out.data_ptr() + es
            assert lib.vb_arith_batch_dev(elem, ADD, dim, C.c_void_p(pa), n, dim, C.c_void_p(pb), n, C.c_void_p(po)) == 0
            pv.synchronize()
            _same(out[es:es + a.nbytes].cpu().numpy().view(a.dtype).reshape(n, dim), want)
            d = C.c_int(0)
            assert lib.vb_concat_batch_dev(elem, dim, C.c_void_p(pa), n, dim, C.c_void_p(pb), n, C.c_void_p(po), C.byref(d)) == 0
            pv.synchronize()
            _same(out[es:es + 2 * a.nbytes].cpu().numpy().view(a.dtype).reshape(n, 2 * dim), np.concatenate([a, b], 1))
        for src in (FLOAT4, FLOAT8):
            x = rng.standard_normal((n, 17)).astype(SRC_DTYPE[src])
            want, _ = array_cast_ref(elem, src, x)
            xs = np.dtype(SRC_DTYPE[src]).itemsize
            buf = torch.zeros(x.nbytes + 64, dtype=torch.uint8, device="cuda")
            buf[xs:xs + x.nbytes].copy_(torch.from_numpy(x.view(np.uint8).ravel()).cuda())
            assert lib.vb_array_to_rows_batch_dev(elem, src, 17, -1, C.c_void_p(buf.data_ptr() + xs), n, C.c_void_p(po)) == 0
            pv.synchronize()
            _same(out[es:es + want.nbytes].cpu().numpy().view(want.dtype).reshape(n, 17), want)


@gpu
def test_in_place_arithmetic_equals_out_of_place(pv):
    rng = np.random.default_rng(9)
    lib = pv._lib.load()
    for elem in (VECTOR, HALFVEC):
        for op in (ADD, SUB, MUL):
            n, dim = 3000, 768
            a, b = _no_errors(elem, op, _special(rng, n, dim, elem), _special(rng, n, dim, elem))
            want, _ = arith_ref(elem, op, a, b)
            da, db = _cuda(a), _cuda(b)
            assert lib.vb_arith_batch_dev(elem, op, dim, pv._ptr(da), n, dim, pv._ptr(db), n, pv._ptr(da)) == 0   # out = a
            pv.synchronize()
            _same(da, want.view(np.float16) if elem == HALFVEC else want)
            da = _cuda(a)
            b1 = np.ascontiguousarray(b[:1])
            want1, _ = arith_ref(elem, op, a, b1)
            if want1 is not None:
                db1 = _cuda(b1)
                assert lib.vb_arith_batch_dev(elem, op, dim, pv._ptr(da), n, dim, pv._ptr(db1), 1, pv._ptr(da)) == 0
                pv.synchronize()
                _same(da, want1.view(np.float16) if elem == HALFVEC else want1)
            # in place over the broadcast operand is an overlap, refused
            db1 = _cuda(b1)
            assert lib.vb_arith_batch_dev(elem, op, dim, pv._ptr(_cuda(a)), n, dim, pv._ptr(db1), 1, pv._ptr(db1)) == EINVAL


# ------------------------------------------------------------------------------- error order

def _raises(fn, text, exc):
    with pytest.raises(exc) as e:
        fn()
    assert str(e.value) == text


@gpu
@pytest.mark.parametrize("device", [False, True])
def test_the_first_offender_decides(pv, device):
    conv = _cuda if device else (lambda x: x)
    n, dim = 2000, 64
    one = np.ones((n, dim), np.float32)
    # lowest row: an underflow in row 700 beats an overflow in row 1500, wherever the elements are
    a, b = one.copy(), one.copy()
    a[1500, 3], b[1500, 3] = 3e38, 3e38
    a[700, 60], b[700, 60] = 1e-30, 1e-30
    _raises(lambda: pv.vector_mul(conv(a), conv(b)), "value out of range: underflow", OverflowError)
    a[300, 10], b[300, 10] = 3e38, 3e38
    _raises(lambda: pv.vector_mul(conv(a), conv(b)), "value out of range: overflow", OverflowError)
    # within a * row, the first element decides between overflow and underflow
    a, b = one.copy(), one.copy()
    a[5, 40], b[5, 40] = 3e38, 3e38
    a[5, 41], b[5, 41] = 1e-30, 1e-30
    _raises(lambda: pv.vector_mul(conv(a), conv(b)), "value out of range: overflow", OverflowError)
    a[5, 2], b[5, 2] = 1e-30, 1e-30
    _raises(lambda: pv.vector_mul(conv(a), conv(b)), "value out of range: underflow", OverflowError)
    # halfvec: -0 results count as zero; underflow of a broadcast operand
    h = _half_bits(one)
    w = _half_bits(np.full((1, dim), 1e-4, np.float32))
    hh = h.copy()
    hh[9, 1] = _half_bits(np.float32(-1e-4))
    _raises(lambda: pv.vector_mul(conv(hh), conv(w), HALFVEC), "value out of range: underflow", OverflowError)
    hh[9, 0] = 0x7BFF
    _raises(lambda: pv.vector_add(conv(hh), conv(hh), HALFVEC), "value out of range: overflow", OverflowError)
    # halfvec cast: a range error beats an earlier NaN in its row ...
    x = np.ones((n, dim), np.float64)
    x[800, 5] = np.nan
    x[800, 50] = 65520.0000001
    _raises(lambda: pv.array_to_halfvec(conv(x)), '"65520" is out of range for type halfvec', ValueError)
    # ... and a NaN in an earlier row beats a range error in a later one
    x[400, 63] = np.nan
    _raises(lambda: pv.array_to_halfvec(conv(x)), "NaN not allowed in halfvec", ValueError)
    x[100, 7] = np.inf
    _raises(lambda: pv.array_to_halfvec(conv(x)), "infinite value not allowed in halfvec", ValueError)
    # the text shows the converted float
    x = np.full((3, 5), 2.0, np.float64)
    x[2, 4] = 1e20
    _raises(lambda: pv.array_to_halfvec(conv(x)), '"1e+20" is out of range for type halfvec', ValueError)
    xi = np.full((3, 5), 2, np.int32)
    xi[1, 1] = 70000
    _raises(lambda: pv.array_to_halfvec(conv(xi)), '"70000" is out of range for type halfvec', ValueError)
    # vector cast: the whole row is converted, then the first non-finite element
    x = np.ones((n, dim), np.float64)
    x[20, 30] = 4e38
    x[20, 31] = np.nan
    _raises(lambda: pv.array_to_vector(conv(x)), "infinite value not allowed in vector", ValueError)
    x[20, 29] = np.nan
    _raises(lambda: pv.array_to_vector(conv(x)), "NaN not allowed in vector", ValueError)


# ------------------------------------------------------------------------------- refusals and asynchrony

@gpu
def test_refused_and_empty_calls_launch_nothing(pv):
    import torch
    lib = pv._lib.load()
    x = torch.ones((4, 8), dtype=torch.float32, device="cuda")
    y = torch.ones((3, 8), dtype=torch.float32, device="cuda")
    o = torch.empty((8, 16), dtype=torch.float32, device="cuda")
    p = pv._ptr
    d = C.c_int(-7)
    before = pv.launch_count()
    refused = [
        lib.vb_arith_batch_dev(2, ADD, 8, p(x), 4, 8, p(x), 4, p(o)),                # bad elem
        lib.vb_arith_batch_dev(VECTOR, 3, 8, p(x), 4, 8, p(x), 4, p(o)),             # bad op
        lib.vb_arith_batch_dev(VECTOR, ADD, 0, p(x), 4, 0, p(x), 4, p(o)),           # dim 0
        lib.vb_arith_batch_dev(VECTOR, ADD, 8, p(x), -1, 8, p(x), 4, p(o)),          # negative count
        lib.vb_arith_batch_dev(VECTOR, ADD, 8, p(x), 4, 8, p(y), 3, p(o)),           # 4 and 3 rows
        lib.vb_arith_batch_dev(VECTOR, ADD, 8, p(x), 4, 4, p(x), 4, p(o)),           # different dimensions
        lib.vb_arith_batch_dev(VECTOR, ADD, 8, None, 4, 8, p(x), 4, p(o)),           # NULL
        lib.vb_arith_batch_dev(VECTOR, ADD, 8, p(x), 4, 8, p(y), 1, p(x[1:])),        # overlap, not in place
        lib.vb_arith_batch(VECTOR, ADD, 8, None, 4, 8, None, 4, None),
        lib.vb_concat_batch_dev(VECTOR, 8, p(x), 4, 8, p(x), 4, p(x), C.byref(d)),   # overlap
        lib.vb_concat_batch_dev(VECTOR, 8000, p(x), 0, 8001, p(x), 0, None, C.byref(d)),   # 16001 dimensions
        lib.vb_concat_batch(HALFVEC, 8, p(x), 4, 8, p(y), 3, p(o), C.byref(d)),      # counts
        lib.vb_concat_batch_dev(VECTOR, 8, p(x), 4, 8, p(x), 4, p(o), None),         # NULL out_dim
        lib.vb_array_to_rows_batch_dev(VECTOR, 3, 8, -1, p(x), 4, p(o)),             # bad src
        lib.vb_array_to_rows_batch_dev(VECTOR, FLOAT4, 0, -1, p(x), 4, p(o)),        # CheckDim
        lib.vb_array_to_rows_batch_dev(VECTOR, FLOAT4, 16001, -1, p(x), 4, p(o)),
        lib.vb_array_to_rows_batch_dev(HALFVEC, FLOAT4, 8, 7, p(x), 4, p(o)),        # CheckExpectedDim
        lib.vb_array_to_rows_batch_dev(VECTOR, FLOAT4, 8, -1, p(x), 4, p(x)),        # overlap
        lib.vb_array_to_rows_batch(VECTOR, FLOAT8, 8, -1, None, 4, None),
    ]
    assert refused == [EINVAL] * len(refused)
    assert d.value == -7
    assert lib.vb_array_to_rows_batch_dev(HALFVEC, FLOAT4, 8, 7, p(x), 4, p(o)) == EINVAL
    assert lib.vb_last_error().decode() == "expected 7 dimensions, not 8"
    assert lib.vb_array_to_rows_batch_dev(HALFVEC, FLOAT4, 0, 7, p(x), 4, p(o)) == EINVAL
    assert lib.vb_last_error().decode() == "halfvec must have at least 1 dimension"
    assert lib.vb_concat_batch_dev(HALFVEC, 8000, p(x), 0, 8001, p(x), 0, None, C.byref(d)) == EINVAL
    assert lib.vb_last_error().decode() == "halfvec cannot have more than 16000 dimensions"
    assert lib.vb_arith_batch_dev(HALFVEC, SUB, 8, p(x), 4, 4, p(x), 4, p(o)) == EINVAL
    assert lib.vb_last_error().decode() == "different halfvec dimensions 8 and 4"
    # 0 result rows: nothing launched, concat sizes the output
    assert lib.vb_arith_batch_dev(VECTOR, ADD, 8, None, 0, 8, p(x), 1, None) == 0
    assert lib.vb_arith_batch(VECTOR, MUL, 8, p(x), 1, 8, None, 0, None) == 0
    assert lib.vb_array_to_rows_batch_dev(VECTOR, INT4, 8, 8, None, 0, None) == 0
    assert lib.vb_concat_batch_dev(VECTOR, 8, None, 0, 5, None, 0, None, C.byref(d)) == 0 and d.value == 13
    assert lib.vb_concat_batch(HALFVEC, 8, None, 1, 5, None, 0, None, C.byref(d)) == 0 and d.value == 13
    assert pv.launch_count() == before
    with pytest.raises(TypeError):
        pv.vector_add(x, np.ones(8, np.float32))


@gpu
def test_concat_replays_from_a_cuda_graph(pv):
    import torch
    lib = pv._lib.load()
    p = pv._ptr
    rng = np.random.default_rng(12)
    n = 4000
    a = _cuda(_special(rng, n, 768, HALFVEC))
    b = _cuda(_special(rng, 1, 513, HALFVEC))
    out = torch.empty((n, 768 + 513), dtype=torch.float16, device="cuda")
    d = C.c_int(0)

    def call():
        assert lib.vb_concat_batch_dev(HALFVEC, 768, p(a), n, 513, p(b), 1, p(out), C.byref(d)) == 0

    torch.cuda.synchronize()
    call()
    pv.synchronize()
    eager = out.clone()
    out.fill_(7)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=torch.cuda.ExternalStream(pv.stream_handle())):
        call()
    out.fill_(3)
    torch.cuda.synchronize()
    g.replay()
    torch.cuda.synchronize()
    _same(out, eager.cpu())
    assert d.value == 768 + 513


# ------------------------------------------------------------------------------- the centring recipe

@gpu
def test_centring_on_the_device_equals_the_host_pipeline(pv):
    """v - (SELECT avg(v) FROM t) on device tensors: Table.avg with CUDA groups, broadcast vector_sub, append to a new
    table and exact top-k there; the same pipeline through the host variants gives the same bits"""
    import torch
    rng = np.random.default_rng(31)
    n, dim, nq, k = 50_000, 256, 32, 10
    rows = (rng.standard_normal((n, dim)) + 3).astype(np.float32)
    q = rng.standard_normal((nq, dim)).astype(np.float32)
    rows_d = torch.from_numpy(rows).cuda()
    t = pv.Table(VECTOR, dim).append(rows_d)
    mean_d, cnt_d = t.avg(torch.zeros(n, dtype=torch.int32, device="cuda"), 1)
    mean_h, cnt_h = t.avg(np.zeros(n, np.int32), 1)
    assert mean_d.is_cuda
    _same(mean_d, mean_h)
    got = pv.vector_sub(rows_d, mean_d[0])
    want = pv.vector_sub(rows, mean_h[0])
    assert got.is_cuda
    _same(got, want)
    tg = pv.Table(VECTOR, dim).append(got)
    th = pv.Table(VECTOR, dim).append(want)
    qd = torch.from_numpy(q).cuda()
    for metric in (pv.L2, pv.COSINE):
        ids, dist = tg.exact_topk(metric, qd, k)
        wids, wdist = th.exact_topk(metric, qd, k)
        _same(ids, wids.cpu())
        _same(dist, wdist.cpu())
    for x in (t, tg, th):
        x.free()
