"""vector_in / halfvec_in / sparsevec_in and the three _out functions on the device, host and _dev variants, compared
exactly (values bitwise, text bytewise, errmsg, errdetail, row) with the CPU restatement in tests/text_io_oracle."""
import random

import numpy as np
import pytest

from tests import text_io_oracle as T

pytestmark = pytest.mark.gpu

CASES = [
    "[1,2,3]", "[-1,-2,-3]", "[1.,2.,3.]", " [ 1,  2 ,    3  ] ", "[1.23456]", "[hello,1]", "[NaN,1]", "[Infinity,1]",
    "[-Infinity,1]", "[1.5e38,-1.5e38]", "[1.5e+38,-1.5e+38]", "[1.5e-38,-1.5e-38]", "[4e38,1]", "[-4e38,1]",
    "[1e-46,1]", "[-1e-46,1]", "[1,2,3", "[1,2,3]9", "1,2,3", "", "[", "[ ", "[,", "[]", "[ ]", "[,]", "[1,]", "[1a]",
    "[1,,3]", "[1, ,3]", "[0x1.8p3]", "[0x]", "[1e]", "[.]", "[-]", "[+1]", "[ nan(abc) ]", "[inf]", "[INFINITY]",
    "[infin]", "[1\t,\n2\r]\f\v", "[65504]", "[65520]", "[65519.99]", "[-65520]", "[6e-8]", "[1e-8]",
    "[3.4028235e38]", "[3.4028236e38]", "[3.40282357e38]", "[1.17549435e-38]", "[1.4e-45]", "[7e-46]", "[7.1e-46]",
    "[0.000000000000000000000000000000000000000000000700649232162408535461864791644958065640130970938257885878534141944895541342930300743319094181060791015625]",
    "[0.000000000000000000000000000000000000000000000700649232162408535461864791644958065640130970938257885878534141944895541342930300743319094181060791015626]",
    "[1.00000005960464477539062500000000000000000000001]", "[1.000000059604644775390625]", "[1.0000000596046447753906249999]",
    "[" + "1" * 40 + "]", "[0." + "0" * 30 + "1" + "5" * 500 + "]", "[123456789012345678901234567890e-10]",
]
SPARSE = [
    "{1:1.5,3:3.5}/5", "{1:-2,3:-4}/5", "{1:2.,3:4.}/5", " { 1 : 1.5 ,  3  :  3.5  } / 5 ", "{1:1.23456}/1",
    "{1:hello,2:1}/2", "{1:NaN,2:1}/2", "{1:Infinity,2:1}/2", "{1:4e38}/1", "{1:1e-46}/1", "{}/5", "{}/0", "{}/-1",
    "{}/1000000001", "{}/1000000000", "{1:0}/1", "{5:0}/3", "{5:1}/3", "{0:1}/3", "{-1:1}/3", "{2:1,1:1}/2",
    "{1:1,1:1}/2", "{1:1,2:1", "{1:1,2:1}/", "{1:1}/2a", "1:1}/2", "{}", "{:1}/1", "{1:}/1", "{1}/1", "{1:1,}/1",
    "{1:1}}/1", "{3:1,2:2,1:3}/3", "{9999999999:1}/3", "{-9999999999:1}/3", "{1:1}/99999999999", "{2:1,2:2,9:1}/3",
    "{9:1,2:1,2:2}/3", "{1:1}/ 2 ", "{1 :1}/2",
]


@pytest.fixture(scope="module")
def pv():
    import pgvector_b200 as pv
    pv.init(0)
    return pv


def _want_dense(half, lits, typmod=-1):
    rows = []
    for i, lit in enumerate(lits):
        row, msg, det = T.dense_in(half, lit, typmod)
        if row is None:
            return None, (msg, det, i)
        rows.append(row)
    return rows, None


def _got(fn, *args):
    from pgvector_b200._lib import TextInputError
    try:
        return fn(*args), None
    except TextInputError as e:
        return None, (str(e), e.detail, e.row)


def _dev_text(lits):
    import torch
    blobs = [x.encode() for x in lits]
    off = np.zeros(len(blobs) + 1, np.int64)
    off[1:] = np.cumsum([len(b) for b in blobs])
    text = torch.tensor(list(b"".join(blobs) or b"\0"), dtype=torch.uint8, device="cuda")
    return text, torch.tensor(off, device="cuda")


def _check_dense(pv, half, lits, typmod=-1):
    fn = pv.halfvec_in if half else pv.vector_in
    want, werr = _want_dense(half, lits, typmod)
    got, gerr = _got(fn, lits, typmod)
    assert gerr == werr, (lits, gerr, werr)
    dgot, derr = _got(fn, _dev_text(lits), typmod)
    assert derr == werr, (lits, derr, werr)
    if want is None:
        return
    dt = np.uint16 if half else np.uint32
    for g, w in zip(got, want):
        assert np.array_equal(np.asarray(g).view(dt), w.view(dt)), (lits, g, w)
    vals, off = dgot
    vals = vals.cpu().numpy().view(dt)
    off = off.cpu().numpy()
    for i, w in enumerate(want):
        assert np.array_equal(vals[off[i]:off[i + 1]], w.view(dt))


@pytest.mark.parametrize("half", [0, 1])
def test_known_literals_one_by_one(pv, half):
    for lit in CASES:
        _check_dense(pv, half, [lit])


def test_sparse_literals_one_by_one(pv):
    for lit in SPARSE:
        want, msg, det = T.sparse_in(lit)
        got, gerr = _got(pv.sparsevec_in, [lit])
        dgot, derr = _got(pv.sparsevec_in, _dev_text([lit]))
        if want is None:
            assert gerr == (msg, det, 0), (lit, gerr, msg)
            assert derr == (msg, det, 0), (lit, derr, msg)
            continue
        assert gerr is None and derr is None, (lit, gerr, derr)
        rows, dims = got
        assert int(dims[0]) == want[0]
        assert np.array_equal(rows.idx, want[1]) and np.array_equal(rows.val.view(np.uint32), want[2].view(np.uint32)), lit
        (roff, idx, val), ddims = dgot
        assert int(ddims[0].item()) == want[0]
        assert np.array_equal(idx.cpu().numpy(), want[1]) and np.array_equal(val.cpu().numpy().view(np.uint32), want[2].view(np.uint32))


def _token(rng):
    kind = rng.random()
    sign = rng.choice(["", "", "-", "+"])
    if kind < 0.45:
        return sign + repr(float(np.float32(rng.uniform(-2, 2) * 10 ** rng.randint(-40, 38))))
    if kind < 0.6:
        digits = "".join(rng.choice("0123456789") for _ in range(rng.randint(20, 200)))
        return sign + digits[: rng.randint(0, 5)] + "." + digits + (f"e{rng.randint(-60, 40)}" if rng.random() < 0.5 else "")
    if kind < 0.72:
        # a decimal halfway point between adjacent floats, and +-1 in its last digit
        f = np.float32(rng.uniform(0.5, 2) * 10 ** rng.randint(-44, 37))
        from fractions import Fraction
        a = Fraction(float(f))
        b = Fraction(float(np.nextafter(f, np.float32(np.inf))))
        h = (a + b) / 2
        s = _fraction_decimal(h)
        adj = rng.choice([0, 0, 1, -1])
        if adj:
            s = _bump(s, adj)
        return sign + s
    if kind < 0.8:
        return sign + rng.choice(["inf", "Infinity", "INF", "nan", "NaN", "nan(x_1)", "nan(", "infinit", "0x1.8p3", "0x.8p-1",
                                  "0x1p-150", "0x1p128", "0x1.fffffep127", "0x", "1e", "1e+", ".", "", "0x1p", "1e-50",
                                  "1e50", "65504", "65520", "65519.998", "6e-8", "3e-8", "1.4e-45", "7e-46", "3.4028235e38",
                                  "3.4028236e38", "1.1754942e-38"])
    return sign + str(rng.randint(0, 100000)) + rng.choice(["", ".5", "e3", "e-3", "E+1"])


def _fraction_decimal(h):
    """exact decimal text of a dyadic fraction"""
    num, den = h.numerator, h.denominator
    k = den.bit_length() - 1
    digits = num * 5 ** k
    s = str(digits).rjust(k + 1, "0")
    return (s[:-k] + "." + s[-k:]) if k else s


def _bump(s, d):
    intpart, _, frac = s.partition(".")
    n = int(intpart + frac) + d
    t = str(n).rjust(len(intpart + frac), "0")
    return t[: len(intpart)] + ("." + t[len(intpart):] if frac else "")


def _literal(rng, n):
    ws = lambda: rng.choice(["", "", " ", "\t", "\n ", "\r\f\v"])  # noqa: E731
    body = "".join((ws() + _token(rng) + ws() + ("," if i < n - 1 else "")) for i in range(n))
    lit = ws() + "[" + body + "]" + ws()
    if rng.random() < 0.05:
        lit = lit + rng.choice(["x", ",", "]"])
    return lit


@pytest.mark.parametrize("half", [0, 1])
def test_fuzzed_literals_match_the_oracle(pv, half):
    rng = random.Random(7 + half)
    for _ in range(300):
        _check_dense(pv, half, [_literal(rng, rng.randint(1, 6))])


def test_fuzzed_tokens_parse_bit_exactly(pv):
    rng = random.Random(11)
    toks = [_token(rng) for _ in range(20000)]
    good = []
    for t in toks:
        u, end, er = T.strtof(t)
        if end == len(t.encode()) and end > 0 and not er and (u & 0x7f800000) != 0x7f800000:
            good.append(t)
    got = pv.vector_in([f"[{t}]" for t in good])
    want = np.array([T.strtof(t)[0] for t in good], np.uint32)
    assert np.array_equal(np.concatenate(got).view(np.uint32), want)


def test_batch_reports_first_bad_literal(pv):
    rng = random.Random(3)
    for _ in range(5):
        lits = [_literal(random.Random(i), 4) for i in range(200)]
        lits = [l for l in lits if T.dense_in(0, l)[0] is not None][:150]
        bad = rng.randrange(len(lits))
        lits[bad] = "[1,2,x]"
        _check_dense(pv, 0, lits)


def test_typmod(pv):
    _check_dense(pv, 0, ["[1,2,3]", "[1,2]"], 3)
    _check_dense(pv, 1, ["[1,2,3]"], 3)
    _check_dense(pv, 0, ["[1,2,3]"], 2)
    for lit, tm in (("{1:1}/3", 3), ("{1:1}/3", 2)):
        want, msg, det = T.sparse_in(lit, tm)
        got, gerr = _got(pv.sparsevec_in, [lit], tm)
        assert (gerr is None) == (want is not None)
        if gerr:
            assert gerr == (msg, det, 0)


def test_dimension_limits(pv):
    big = "[" + ",".join(["1.25"] * 16000) + "]"
    _check_dense(pv, 0, [big])
    _check_dense(pv, 1, [big])
    _check_dense(pv, 0, ["[" + ",".join(["1"] * 16001) + "]"])
    _check_dense(pv, 0, ["[" + ",".join(["1"] * 16000) + ",x"])
    sp = "{" + ",".join(f"{i}:1" for i in range(1, 16001)) + "}/16000"
    want, _, _ = T.sparse_in(sp)
    (rows, _), _ = _got(pv.sparsevec_in, [sp])
    assert np.array_equal(rows.idx, want[1])
    sp2 = "{" + ",".join(f"{i}:1" for i in range(1, 16002)) + "}/16001"
    _, gerr = _got(pv.sparsevec_in, [sp2])
    assert gerr[0] == "sparsevec cannot have more than 16000 non-zero elements"


def test_nul_ends_a_literal(pv):
    _check_dense(pv, 0, ["[1,2]\0,3]", "[1]\0"])


def _kat():
    import json
    import os
    return json.load(open(os.path.join(os.path.dirname(__file__), "golden", "text_io_kat.json")))["cases"]


def test_known_answers(pv):
    """every SELECT '<literal>'::type of the reference's regression outputs: printed text, or ERROR and DETAIL"""
    from pgvector_b200._lib import VecB200Error
    for c in _kat():
        typ, lit, tm = c["type"], c["literal"], c["typmod"]
        if c.get("typmod_in"):
            # a modifier out of range never reaches the input function; the batch calls refuse it as an argument
            fn = pv.sparsevec_in if typ == "sparsevec" else pv.halfvec_in if typ == "halfvec" else pv.vector_in
            with pytest.raises(VecB200Error):
                fn([lit], tm)
            continue
        for texts in ([lit], _dev_text([lit])):
            if typ == "sparsevec":
                got, err = _got(pv.sparsevec_in, texts, tm)
            else:
                got, err = _got(pv.halfvec_in if typ == "halfvec" else pv.vector_in, texts, tm)
            if "error" in c:
                assert err == (c["error"], c["detail"], 0), (c, err)
                continue
            assert err is None, (c, err)
            if typ == "sparsevec":
                if isinstance(texts, list):
                    rows, dims = got
                    out = pv.sparsevec_out(pv.SparseRows(int(dims[0]), rows.row_off, rows.idx, rows.val))
                else:
                    (roff, idx, val), dims = got
                    t, o = pv.sparsevec_out(((roff, idx, val), int(dims[0].item())))
                    out = [t.cpu().numpy().tobytes().decode()]
            else:
                out_fn = pv.halfvec_out if typ == "halfvec" else pv.vector_out
                if isinstance(texts, list):
                    out = out_fn(got[0].reshape(1, -1))
                else:
                    vals, _ = got
                    t, o = out_fn(vals.reshape(1, -1))
                    out = [t.cpu().numpy().tobytes().decode()]
            assert out == [c["output"]], (c, out)


def test_sparse_output_refuses_bad_indices(pv):
    """rows the sparse table calls refuse are refused before any text is formatted"""
    from pgvector_b200._lib import VecB200Error
    for idx in ([-5], [3], [1, 0], [1, 1]):
        rows = pv.SparseRows(3, np.array([0, len(idx)]), np.array(idx, np.int32), np.ones(len(idx), np.float32))
        with pytest.raises(VecB200Error):
            pv.sparsevec_out(rows)


def test_empty_batches(pv):
    import torch
    assert pv.vector_in([]) == []
    vals, off = pv.vector_in((torch.zeros(1, dtype=torch.uint8, device="cuda"), torch.zeros(1, dtype=torch.int64, device="cuda")))
    assert vals.numel() == 0 and off.tolist() == [0]


def test_format_against_the_oracle(pv):
    import torch
    # every 4096th bit pattern against numpy's shortest digits (tests/test_text_io_oracle.py checks those against the
    # exact ones), the edges below against the exact oracle
    pats = np.arange(0, 1 << 32, 4096, dtype=np.uint64).astype(np.uint32)
    pv_vals = pats.view(np.float32)
    pv_vals = pv_vals[np.isfinite(pv_vals)]
    got = pv.vector_out(pv_vals.reshape(-1, 1))
    want = ["[" + T.format_float4_numpy(v) + "]" for v in pv_vals]
    bad = [(g, w) for g, w in zip(got, want) if g != w]
    assert not bad, bad[:10]
    pats = np.arange(0, 1 << 32, 4096 * 37, dtype=np.uint64).astype(np.uint32)
    specials = []
    for e in range(-45, 39):
        f = np.float32(10.0 ** e)
        specials += [f, np.nextafter(f, np.float32(0)), np.nextafter(f, np.float32(np.inf))]
    for e in range(-149, 128):
        f = np.float32(2.0 ** e)
        specials += [f, np.nextafter(f, np.float32(0)), np.nextafter(f, np.float32(np.inf))]
    specials += [1e6, 999999, 1.6777216e7, 1e-4, 1e-5, 0.0, -0.0, np.inf, -np.inf, np.nan, 150000, 123456]
    vals = np.concatenate([pats.view(np.float32), np.array(specials, np.float32)])
    vals = vals[~np.isnan(vals)]
    got = pv.vector_out(vals.reshape(-1, 1))
    want = ["[" + T.format_float4(v) + "]" for v in vals]
    bad = [(g, w) for g, w in zip(got, want) if g != w]
    assert not bad, bad[:10]
    text, off = pv.vector_out(torch.tensor(vals.reshape(-1, 1), device="cuda"))
    blob = text.cpu().numpy().tobytes()
    off = off.cpu().numpy()
    assert [blob[off[i]:off[i + 1]].decode() for i in range(len(vals))] == want
    assert T.format_float4(np.float32(1e6)) == "1e+06"
    assert T.format_float4(np.float32(999999)) == "999999"
    assert T.format_float4(np.float32(1.6777216e7)) == "1.6777216e+07"
    assert T.format_float4(np.float32(1e-4)) == "0.0001"
    assert T.format_float4(np.float32(1e-5)) == "1e-05"


def test_every_half_formats(pv):
    h = np.arange(65536, dtype=np.uint32).astype(np.uint16)
    h = h[(h & 0x7c00) != 0x7c00]
    got = pv.halfvec_out(h.reshape(-1, 1))
    want = ["[" + T.format_float4(np.float32(v)) + "]" for v in h.view(np.float16)]
    assert got == want


def test_round_trip(pv):
    rng = np.random.default_rng(5)
    x = (rng.standard_normal((300, 37)) * 10.0 ** rng.integers(-30, 30, (300, 1))).astype(np.float32)
    text = pv.vector_out(x)
    assert text == [T.vector_out(r) for r in x]
    back = np.stack(pv.vector_in(text))
    assert np.array_equal(back.view(np.uint32), x.view(np.uint32))
    assert pv.vector_out(back) == text


def test_sparse_rows_and_append(pv):
    import torch
    rng = random.Random(9)
    lits = []
    for _ in range(200):
        dim = rng.randint(1, 50)
        ids = rng.sample(range(1, dim + 1), rng.randint(0, min(dim, 8)))
        lits.append("{" + ",".join(f"{i}:{rng.choice(['0', '1.5', '-2e-3', '7'])}" for i in ids) + f"}}/{dim}")
    want = [T.sparse_in(l)[0] for l in lits]
    (rows, dims) = pv.sparsevec_in(lits)
    for i, w in enumerate(want):
        b, e = rows.row_off[i], rows.row_off[i + 1]
        assert dims[i] == w[0] and np.array_equal(rows.idx[b:e], w[1]) and np.array_equal(rows.val[b:e], w[2])
    same = [l for l, w in zip(lits, want) if w[0] == 50]
    if same:
        (r2, _) = pv.sparsevec_in(same)
        out = pv.sparsevec_out(r2)
        assert out == [T.sparsevec_out(50, *T.sparse_in(l)[0][1:]) for l in same]
        (roff, idx, val), _ = pv.sparsevec_in(_dev_text(same))
        t = pv.SparseTable(50)
        from pgvector_b200._lib import load
        from pgvector_b200.sparsevec import _tp
        assert load().vb_sparse_table_append_dev(t.h, len(same), _tp(roff), _tp(idx), _tp(val)) == 0
        assert int(load().vb_sparse_table_rows(t.h)) == len(same)


def test_sizing_call_reports_the_bound(pv):
    from pgvector_b200._lib import load
    import ctypes as C
    lits = [b"[1,2,3]", b"[4, 5]"]
    off = np.array([0, 7, 13], np.int64)
    text = np.frombuffer(b"".join(lits), np.uint8)
    row_off = np.zeros(3, np.int64)
    bad = C.c_int64(0)
    rc = load().vb_text_to_rows_batch(0, -1, 2, text.ctypes.data, off.ctypes.data, 0, row_off.ctypes.data, None, C.byref(bad))
    assert rc == -1 and list(row_off) == [0, 3, 5] and bad.value == -1
    assert "5" in load().vb_last_error().decode()
