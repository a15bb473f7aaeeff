"""vector_recv / halfvec_recv / sparsevec_recv and the three _send functions on the device, host and _dev variants,
compared exactly (values bitwise, payloads bytewise, errmsg, failing field) with the restatement in
tests/binary_io_oracle."""
import ctypes as C
import json
import os

import numpy as np
import pytest

from tests import binary_io_oracle as O

pytestmark = pytest.mark.gpu

KAT = json.load(open(os.path.join(os.path.dirname(__file__), "golden", "binary_io_kat.json")))["cases"]


@pytest.fixture(scope="module")
def pv():
    import pgvector_b200 as pv
    pv.init(0)
    return pv


def _dev(payloads, gaps=None):
    """a (CUDA uint8, CUDA int64 offsets) pair; gaps[i] junk bytes before field i move it to any offset mod 16"""
    import torch
    parts, off, pos = [], [0], 0
    ends = []
    for i, p in enumerate(payloads):
        g = gaps[i] if gaps is not None else 0
        parts.append(b"\xa5" * g + p)
        pos += g
        off.append(pos)
        pos += len(p)
        ends.append(pos)
    blob = b"".join(parts) or b"\0"
    data = torch.frombuffer(bytearray(blob), dtype=torch.uint8).cuda()
    # with gaps the fields are not adjacent: (data, starts, ends) instead of one offsets array
    starts = np.array(off[1:], np.int64)
    if gaps is None:
        o = np.zeros(len(payloads) + 1, np.int64)
        o[1:] = np.cumsum([len(p) for p in payloads])
        return data, torch.from_numpy(o).cuda()
    return data, starts, np.array(ends, np.int64)


def _run(fn, *args):
    from pgvector_b200._lib import TextInputError
    try:
        return fn(*args), None
    except TextInputError as e:
        return None, (e.row, str(e))


def _recv(pv, kind, payloads, typmod=-1, dev=False):
    fn = {"vector": pv.vector_recv, "halfvec": pv.halfvec_recv, "sparsevec": pv.sparsevec_recv}[kind]
    return _run(fn, _dev(payloads) if dev else payloads, typmod)


def _dense_rows(got, dev, n):
    if not dev:
        return [np.asarray(r) for r in got]
    vals, off = got
    v = vals.cpu().numpy()
    o = off.cpu().numpy()
    return [v[o[i]:o[i + 1]] for i in range(n)]


def _bits(row, half):
    return np.asarray(row).view(np.uint16 if half else np.uint32)


def _check_batch(pv, kind, payloads, typmod=-1):
    want, err = O.recv_batch(payloads, typmod, kind)
    for dev in (False, True):
        got, gerr = _recv(pv, kind, payloads, typmod, dev)
        assert gerr == err, (dev, gerr, err)
        if err:
            continue
        if kind == "sparsevec":
            if dev:
                (roff, idx, val), dims = got
                roff, idx, val, dims = roff.cpu().numpy(), idx.cpu().numpy(), val.cpu().numpy(), dims.cpu().numpy()
            else:
                rows, dims = got
                roff, idx, val = rows.row_off, rows.idx, rows.val
            for i, (d, wi, wv) in enumerate(want):
                assert dims[i] == d
                assert np.array_equal(idx[roff[i]:roff[i + 1]], wi)
                assert np.array_equal(val[roff[i]:roff[i + 1]].view(np.uint32), wv)
        else:
            rows = _dense_rows(got, dev, len(payloads))
            for r, w in zip(rows, want):
                assert np.array_equal(_bits(r, kind == "halfvec"), w)


@pytest.mark.parametrize("i", range(len(KAT)))
def test_known_answer(pv, i):
    c = KAT[i]
    p = bytes.fromhex(c["payload"])
    for dev in (False, True):
        got, err = _recv(pv, c["type"], [p], c["typmod"], dev)
        if "error" in c:
            assert err == (0, c["error"]), dev
            continue
        assert err is None
        if c["type"] == "sparsevec":
            rows, dims = got
            if dev:
                (roff, idx, val) = rows
                idx, val = idx.cpu().numpy()[:len(c["indices"])], val.cpu().numpy()[:len(c["indices"])]
                assert int(dims[0]) == c["dim"]
            else:
                idx, val = rows.idx, rows.val
                assert pv.sparsevec_out(rows) == [c["text"]]
                assert pv.sparsevec_send(rows) == [p]
            assert idx.tolist() == c["indices"] and val.view(np.uint32).tolist() == c["bits"]
        else:
            half = c["type"] == "halfvec"
            row = _dense_rows(got, dev, 1)[0]
            assert _bits(row, half).tolist() == c["bits"]
            if not dev:
                out = pv.halfvec_out if half else pv.vector_out
                send = pv.halfvec_send if half else pv.vector_send
                assert out(row[None]) == [c["text"]]
                assert send(row[None]) == [p]


def test_fuzzed_dense_batches(pv):
    rng = np.random.default_rng(5)
    special = np.array([0x0000, 0x8000, 0x0001, 0x03ff, 0x0400, 0x7bff, 0xfbff, 0x3c00], np.uint16)
    for kind in ("vector", "halfvec"):
        half = kind == "halfvec"
        dims = list(rng.integers(1, 64, 40)) + [1, 15, 16, 17, 768, 1536, 4097, 16000]
        rows = []
        for d in dims:
            if half:
                b = rng.integers(0, 0x7c00, d).astype(np.uint16) | (rng.integers(0, 2, d) << 15).astype(np.uint16)
                m = rng.random(d) < 0.2
                b[m] = rng.choice(special, int(m.sum()))
            else:
                b = rng.standard_normal(d).astype(np.float32).view(np.uint32)
                b[rng.random(d) < 0.05] = 0x80000000
                b[rng.random(d) < 0.05] = 0x00000001
            rows.append(b)
        payloads = [O.send_dense(b, half) for b in rows]
        _check_batch(pv, kind, payloads)
        # every field offset mod 16 on the device
        gaps = [int(g) for g in rng.integers(0, 16, len(payloads))]
        data, starts, ends = _dev(payloads, gaps)
        _check_gapped(pv, kind, data, starts, ends, rows, half)


def _check_gapped(pv, kind, data, starts, ends, rows, half):
    """fields at arbitrary byte offsets of one buffer: one device call per field, off = [start, end]"""
    import torch
    lib = pv._lib.load()
    elem = 1 if half else 0
    for s, e, w in zip(starts, ends, rows):
        off = torch.tensor([s, e], dtype=torch.int64, device="cuda")
        roff = torch.zeros(2, dtype=torch.int64, device="cuda")
        out = torch.empty(len(w) + 1, dtype=torch.float16 if half else torch.float32, device="cuda")
        bad = C.c_int64(0)
        rc = lib.vb_binary_to_rows_batch_dev(elem, -1, 1, data.data_ptr(), off.data_ptr(), len(w), roff.data_ptr(),
                                             out.data_ptr(), C.byref(bad))
        assert rc == 0, lib.vb_last_error()
        got = out[:len(w)].cpu().numpy().view(np.uint16 if half else np.uint32)
        assert np.array_equal(got, w)


def test_fuzzed_sparse_batches(pv):
    rng = np.random.default_rng(6)
    payloads = []
    for nnz in list(rng.integers(0, 200, 60)) + [0, 1, 3, 4, 5, 16000]:
        dim = int(rng.integers(max(nnz, 1), 100000))
        idx = np.sort(rng.choice(dim, nnz, replace=False)).astype(np.int32)
        val = rng.standard_normal(nnz).astype(np.float32).view(np.uint32)
        val[val & 0x7fffffff == 0] = 0x3f800000
        payloads.append(O.send_sparse(dim, idx, val))
    _check_batch(pv, "sparsevec", payloads)


def test_first_offender_by_row_then_step(pv):
    f = lambda *v: O.send_dense(np.array(v, np.float32).view(np.uint32))  # noqa: E731
    good = f(1, 2, 3)
    cases = [
        [good, f(1, np.nan, 3), good[:-1], f(np.inf, 1, 1)],
        [good, good[:-1], f(1, np.nan, 3)],
        [good, f(1, 2, 3, np.inf, np.nan)[:-3], good],
        [good] * 500 + [good + b"\0"] + [good[:3]] * 10,
        [good] * 3000 + [f(*([1.0] * 2000 + [np.nan]))] + [f(np.inf)] * 5,
    ]
    for payloads in cases:
        _check_batch(pv, "vector", payloads)
        _check_batch(pv, "vector", payloads, 3)
    s = O.send_sparse
    one = lambda *v: np.array(v, np.float32).view(np.uint32)  # noqa: E731
    sp = [s(5, [0, 2], one(1, 2)), s(5, [0, 2], one(0, np.nan)), s(5, [2, 2], one(np.nan, 1)), s(5, [9], one(1))[:-2]]
    _check_batch(pv, "sparsevec", sp)
    _check_batch(pv, "sparsevec", sp[:1] + sp[2:])
    _check_batch(pv, "sparsevec", sp[:1] + sp[3:])
    _check_batch(pv, "sparsevec", [s(5, [0], one(1)), s(6, [0], one(1)), s(5, [0], one(1))], 5)


def test_typmod_sizes_and_refusals(pv):
    import torch
    lib = pv._lib.load()
    p = [O.send_dense(np.ones(4, np.float32).view(np.uint32))] * 3
    rows, off = pv.vector_recv(_dev(p), 4)
    assert off.cpu().tolist() == [0, 4, 8, 12] and rows.shape == (12,)
    blob = np.frombuffer(b"".join(p) + b"\x00\x01", np.uint8)
    o = np.array([0, 20, 40, 60, 62], np.int64)
    row_off = np.zeros(5, np.int64)
    bad = C.c_int64(0)
    # sizing: the bound offsets, a cap refusal naming the total, nothing else written
    rc = lib.vb_binary_to_rows_batch(0, -1, 4, blob.ctypes.data, o.ctypes.data, 0, row_off.ctypes.data, None, C.byref(bad))
    assert rc == -1 and row_off.tolist() == [0, 4, 8, 12, 12] and bad.value == -1
    assert "12" in lib.vb_last_error().decode()
    for fn in (lib.vb_binary_to_rows_batch, lib.vb_binary_to_rows_batch_dev):
        assert fn(0, -1, 0, None, None, 0, row_off.ctypes.data if fn is lib.vb_binary_to_rows_batch else
                  torch.zeros(1, dtype=torch.int64, device="cuda").data_ptr(), None, C.byref(bad)) == 0
        assert fn(0, -1, 2, None, None, 0, None, None, C.byref(bad)) == -1
        assert fn(0, 0, 0, None, None, 0, None, None, C.byref(bad)) == -1
        assert fn(2, -1, 0, None, None, 0, None, None, C.byref(bad)) == -1
    for fn in (lib.vb_binary_to_sparsevec_batch, lib.vb_binary_to_sparsevec_batch_dev):
        assert fn(-1, 2, None, None, 0, None, None, None, None, C.byref(bad)) == -1
    out_off = np.zeros(3, np.int64)
    x = np.ones((2, 3), np.float32)
    assert lib.vb_rows_to_binary_batch(0, 3, x.ctypes.data, 2, 0, out_off.ctypes.data, None) == 0
    assert out_off.tolist() == [0, 16, 32]
    buf = np.zeros(32, np.uint8)
    assert lib.vb_rows_to_binary_batch(0, 3, x.ctypes.data, 2, 31, out_off.ctypes.data, buf.ctypes.data) == -1
    assert "32" in lib.vb_last_error().decode()
    assert lib.vb_rows_to_binary_batch(0, 0, x.ctypes.data, 2, 31, out_off.ctypes.data, None) == -1
    assert lib.vb_rows_to_binary_batch(0, 3, None, 2, 31, out_off.ctypes.data, None) == -1
    assert pv.vector_recv([]) == [] and pv.vector_send(np.zeros((0, 3), np.float32)) == []


def test_copy_stream_round_trip(pv):
    """copy.sql: COPY t TO ... (FORMAT binary) then COPY t2 FROM it, with the payloads cut out of a PGCOPY stream"""
    import torch
    rows = np.array([[0, 0, 0], [1, 2, 3], [1, 1, 1]], np.float32)
    for kind, send, recv in (("vector", pv.vector_send, pv.vector_recv), ("halfvec", pv.halfvec_send, pv.halfvec_recv)):
        sent = send(rows)
        stream, spans = O.copy_stream(sent[:1] + [None] + sent[1:])
        assert spans[0][0] == 25
        data = torch.frombuffer(bytearray(stream), dtype=torch.uint8).cuda()
        # the fields are not adjacent (length words between them): one call per contiguous run, here each field
        for (a, b), want in zip(spans, sent):
            got, _ = recv((data[a:b].contiguous(), torch.tensor([0, b - a], device="cuda")), 3)
            half = kind == "halfvec"
            assert O.send_dense(got.cpu().numpy().view(np.uint16 if half else np.uint32), half) == want
        back = recv([stream[a:b] for a, b in spans], 3)
        assert send(np.stack(back)) == sent
    from pgvector_b200.sparsevec import SparseRows
    (r, _) = pv.sparsevec_in(["{}/3", "{1:1,2:2,3:3}/3", "{1:1,2:1,3:1}/3"])
    sent = pv.sparsevec_send(r)
    stream, spans = O.copy_stream([sent[0], None, sent[1], sent[2]])
    back, dims = pv.sparsevec_recv([stream[a:b] for a, b in spans], 3)
    assert isinstance(back, SparseRows) and pv.sparsevec_out(back) == ["{}/3", "{1:1,2:2,3:3}/3", "{1:1,2:1,3:1}/3"]


def test_text_to_binary_and_back(pv):
    rng = np.random.default_rng(8)
    x = rng.standard_normal((300, 97)).astype(np.float32)
    text = pv.vector_out(x)
    rows = np.stack(pv.vector_in(text))
    back = pv.vector_recv(pv.vector_send(rows))
    assert np.array_equal(np.stack(back).view(np.uint32), rows.view(np.uint32))
    assert pv.vector_out(np.stack(back)) == text
    import torch
    payload, off = pv.vector_send(torch.from_numpy(rows).cuda())
    vals, roff = pv.vector_recv((payload, off))
    assert np.array_equal(vals.cpu().numpy().view(np.uint32), rows.reshape(-1).view(np.uint32))


def test_send_copies_bits_unchanged(pv):
    import torch
    bits = np.array([0x7fc00001, 0xffbfffff, 0x7f800001, 0x80000000, 0x00000001, 0x807fffff, 0x7f800000, 0xff800000],
                    np.uint32)
    for dim in (8, 13):
        b = np.resize(bits, (5, dim)).astype(np.uint32)
        want = [O.send_dense(r) for r in b]
        assert pv.vector_send(b.view(np.float32)) == want
        p, off = pv.vector_send(torch.from_numpy(b.view(np.float32)).cuda())
        blob = p.cpu().numpy().tobytes()
        o = off.cpu().tolist()
        assert [blob[o[i]:o[i + 1]] for i in range(5)] == want
        h = np.resize(np.array([0x7e01, 0xfc00, 0x7c00, 0x8000, 0x0001, 0x03ff, 0xfe7f], np.uint16), (3, dim))
        assert pv.halfvec_send(h) == [O.send_dense(r, True) for r in h]


def test_sparse_send_refuses_bad_rows(pv):
    import torch
    from pgvector_b200.sparsevec import SparseRows
    for roff, idx, msg in (([0, 2], [1, 1], "ascending order (row 0)"), ([0, 1, 2], [0, 7], "out of bounds (row 1)")):
        rows = SparseRows(5, np.array(roff, np.int64), np.array(idx, np.int32), np.ones(len(idx), np.float32))
        with pytest.raises(Exception) as e1:
            pv.sparsevec_out(rows)
        with pytest.raises(Exception) as e2:
            pv.sparsevec_send(rows)
        dev = tuple(torch.tensor(a, dtype=t, device="cuda") for a, t in
                    ((roff, torch.int64), (idx, torch.int32), (np.ones(len(idx)), torch.float32)))
        with pytest.raises(Exception) as e3:
            pv.sparsevec_send((dev, 5))
        assert msg in str(e1.value) and msg in str(e2.value) and msg in str(e3.value)


def test_dense_send_replays_from_a_cuda_graph(pv):
    import torch
    lib = pv._lib.load()
    rng = np.random.default_rng(12)
    n, dim = 3000, 257
    x = torch.from_numpy(rng.standard_normal((n, dim)).astype(np.float32)).cuda()
    total = n * (4 + 4 * dim)
    out = torch.empty(total, dtype=torch.uint8, device="cuda")
    off = torch.empty(n + 1, dtype=torch.int64, device="cuda")

    def call():
        assert lib.vb_rows_to_binary_batch_dev(0, dim, x.data_ptr(), n, total, off.data_ptr(), out.data_ptr()) == 0

    torch.cuda.synchronize()
    call()
    pv.synchronize()
    eager = out.clone()
    out.fill_(7)
    off.fill_(-1)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=torch.cuda.ExternalStream(pv.stream_handle())):
        call()
    torch.cuda.synchronize()
    g.replay()
    torch.cuda.synchronize()
    assert torch.equal(out, eager)
    assert off[-1].item() == total


def test_device_load_equals_host_load(pv):
    """recv_dev -> table append -> exact top-k equals the same load through the host variants"""
    import torch
    from pgvector_b200.sparsevec import _tp
    lib = pv._lib.load()
    rng = np.random.default_rng(21)
    n, dim, nq, k = 20000, 128, 16, 10
    x = rng.standard_normal((n, dim)).astype(np.float32)
    payloads = pv.vector_send(x)
    q = rng.standard_normal((nq, dim)).astype(np.float32)
    vals, _ = pv.vector_recv(_dev(payloads), dim)
    td = pv.Table(0, dim).append(vals.reshape(n, dim))
    th = pv.Table(0, dim).append(np.stack(pv.vector_recv(payloads, dim)))
    for metric in (pv.L2, pv.COSINE):
        a, da = td.exact_topk(metric, q, k)
        b, db = th.exact_topk(metric, q, k)
        assert np.array_equal(np.asarray(a), np.asarray(b)) and np.array_equal(np.asarray(da), np.asarray(db))
    td.free()
    th.free()
    sp = []
    for _ in range(2000):
        nnz = int(rng.integers(0, 40))
        idx = np.sort(rng.choice(1000, nnz, replace=False)).astype(np.int32)
        sp.append(O.send_sparse(1000, idx, (rng.random(nnz).astype(np.float32) + 0.5).view(np.uint32)))
    (roff, idx, val), _ = pv.sparsevec_recv(_dev(sp), 1000)
    t1 = pv.SparseTable(1000)
    assert lib.vb_sparse_table_append_dev(t1.h, len(sp), _tp(roff), _tp(idx), _tp(val)) == 0
    rows, _ = pv.sparsevec_recv(sp, 1000)
    t2 = pv.SparseTable(1000)
    t2.append(rows)
    qs = rows.__class__(1000, rows.row_off[:5].copy(), rows.idx[:rows.row_off[4]], rows.val[:rows.row_off[4]])
    a, da = t1.exact_topk(pv.L2, qs, k)
    b, db = t2.exact_topk(pv.L2, qs, k)
    assert np.array_equal(a, b) and np.array_equal(da, db)
