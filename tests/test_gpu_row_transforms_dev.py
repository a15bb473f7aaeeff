"""The dense row transforms on device buffers: the _dev variants of vector_norm, l2_normalize, binary_quantize and the
vector <-> halfvec casts, and subvector (host and device), the value of the README's subvector-indexing recipe.

Every _dev result is compared with the host variant's bit for bit (bit patterns, so NaN and -0 count).  subvector is
checked against the reference's answers (vector_type.out, halfvec.out: tests/golden/subvector_kat.json), a numpy
restatement of its dimension rule and numpy slicing.  The three README recipes run end to end on device tensors and must
equal the same pipelines fed with host-transformed rows.  The first tests need no device."""
import ctypes as C
import json
import os

import numpy as np
import pytest

EINVAL, ENODEVICE = -1, -2
VECTOR, HALFVEC, BIT = 0, 1, 2
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "subvector_kat.json")
NEW_SYMBOLS = ["vb_norm_batch_dev", "vb_l2_normalize_batch_dev", "vb_binary_quantize_batch_dev", "vb_vector_to_halfvec_batch_dev",
               "vb_halfvec_to_vector_batch_dev", "vb_subvector_batch", "vb_subvector_batch_dev"]
INT32_MAX, INT32_MIN = 2**31 - 1, -2**31


def subvector_rule(dim, start, count, name):
    """subvector's dimension rule restated (src/vector.c:995-1018): (first element, 0-based; result dimension), or the
    error text.  Python ints do not overflow, and the reference only forms start + count where it cannot either."""
    err = f"{name} must have at least 1 dimension"
    if count < 1:
        return err
    end = dim + 1 if start > dim - count else start + count
    if start < 1:
        start = 1
    elif start > dim:
        return err
    d = end - start
    if d < 1:
        return err
    if d > 16000:
        return f"{name} cannot have more than 16000 dimensions"
    return start - 1, d


def _text(x):
    return "[" + ",".join(f"{float(v):g}" for v in x) + "]"


def _cases():
    return json.load(open(GOLDEN))["cases"]


# ------------------------------------------------------------------------------- anywhere

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
    assert lib.vb_norm_batch_dev(VECTOR, 3, None, 1, None) == ENODEVICE
    assert lib.vb_l2_normalize_batch_dev(VECTOR, 3, None, 1, None) == ENODEVICE
    assert lib.vb_binary_quantize_batch_dev(HALFVEC, 3, None, 1, None) == ENODEVICE
    assert lib.vb_vector_to_halfvec_batch_dev(3, None, 1, None) == ENODEVICE
    assert lib.vb_halfvec_to_vector_batch_dev(3, None, 1, None) == ENODEVICE
    assert lib.vb_subvector_batch(VECTOR, 3, None, 0, 1, 2, None, C.byref(d)) == ENODEVICE
    assert lib.vb_subvector_batch_dev(HALFVEC, 3, None, 0, 1, 2, None, C.byref(d)) == ENODEVICE
    with pytest.raises(pv.VecB200Error) as e:
        pv.subvector(np.ones((2, 5), np.float32), 1, 3)
    assert e.value.code == ENODEVICE


def test_the_subvector_fixture_reads():
    cases = _cases()
    assert len(cases) == 20
    for t in ("vector", "halfvec"):
        mine = [c for c in cases if c["type"] == t]
        assert sum("expected" in c for c in mine) == 6 and sum("error" in c for c in mine) == 4
    assert all(("expected" in c) != ("error" in c) for c in cases)
    assert all(c["source"].startswith("test/expected/") for c in cases)


def test_the_restated_dimension_rule_reproduces_the_fixture():
    for c in _cases():
        x = np.array(json.loads(c["input"]), np.float32)
        got = subvector_rule(x.size, c["start"], c["count"], c["type"])
        if "error" in c:
            assert got == c["error"], c["sql"]
        else:
            first, d = got
            assert _text(x[first:first + d]) == c["expected"], c["sql"]


# ------------------------------------------------------------------------------- helpers

gpu = pytest.mark.gpu


@pytest.fixture(scope="module")
def pv():
    import pgvector_b200 as pv
    pv.init(0)
    return pv


def _bits(a):
    """the bit patterns of a numpy array or a tensor, as unsigned integers of its width"""
    a = a.cpu().numpy() if hasattr(a, "cpu") else np.asarray(a)
    a = np.ascontiguousarray(a)
    return a.view({8: np.uint64, 4: np.uint32, 2: np.uint16, 1: np.uint8}[a.itemsize])


def _same(dev, host):
    assert tuple(dev.shape) == tuple(np.shape(host))
    assert np.array_equal(_bits(dev), _bits(host))


def _special_rows(rng, n, dim, half):
    """n rows with a zero row, -0, subnormals, +-inf and NaN (halfvec: uint16 bit patterns)"""
    x = rng.standard_normal((n, dim), dtype=np.float32)
    if half:
        b = x.astype(np.float16).view(np.uint16)
        sub = rng.random((n, dim)) < 0.02
        b[sub] = rng.integers(1, 0x400, int(sub.sum())).astype(np.uint16) | (rng.integers(0, 2, int(sub.sum())).astype(np.uint16) << 15)
        b[rng.random((n, dim)) < 0.01] = 0x8000
        specials = [0x0000, 0x8000, 0x0001, 0x83FF, 0x7C00, 0xFC00, 0x7E00, 0x7C01]
        rows = b
    else:
        sub = rng.random((n, dim)) < 0.02
        x[sub] = (rng.standard_normal(int(sub.sum())) * 1e-39).astype(np.float32)
        x[rng.random((n, dim)) < 0.01] = -0.0
        specials = [0.0, -0.0, 1e-45, -1e-40, np.inf, -np.inf, np.nan]
        rows = x
    if n >= 10:
        rows[0] = 0                                       # a zero row: stays zero, norm 0
        rows[1] = 0x8000 if half else -0.0                # all -0
        rows[2] = (np.arange(dim) % 0x3FF + 1) if half else np.float32(1e-42) * (np.arange(dim) % 7 + 1)   # subnormals only
        rows[3, dim // 2] = 0x7C00 if half else np.inf
        rows[4, 0] = 0xFC00 if half else -np.inf
        rows[5, dim - 1] = 0x7E00 if half else np.nan
        k = min(dim, len(specials))
        rows[6, :k] = np.array(specials[:k], rows.dtype)
        rows[7, :] = rows[3, :]
        rows[7, 0] = 0x7C00 if half else np.inf           # inf and inf: inf / inf = NaN
    elif n == 1:
        rows[0, 0] = 0x8000 if half else -0.0
    return rows


def _to_dev(rows, half):
    import torch
    return torch.from_numpy(np.ascontiguousarray(rows.view(np.float16) if half else rows)).cuda()


SHAPES = [(VECTOR, 3), (VECTOR, 1536), (VECTOR, 2000), (HALFVEC, 9), (HALFVEC, 768)]


# ------------------------------------------------------------------------------- bit identity with the host calls

@gpu
@pytest.mark.parametrize("elem,dim", SHAPES)
@pytest.mark.parametrize("n", [0, 1, 100_000])
def test_dev_transforms_equal_the_host_transforms(pv, elem, dim, n):
    import torch
    half = elem == HALFVEC
    rng = np.random.default_rng(dim * 7 + n)
    rows = _special_rows(rng, n, dim, half)
    r = _to_dev(rows, half)
    _same(pv.vector_norm(r, elem), pv.vector_norm(rows, elem))
    want = pv.l2_normalize(rows, elem)
    got = pv.l2_normalize(r, elem)
    assert got.dtype == (torch.float16 if half else torch.float32)
    _same(got, want)
    _same(pv.binary_quantize(r, elem), pv.binary_quantize(rows, elem))
    if half:
        _same(pv.halfvec_to_vector(r), pv.halfvec_to_vector(rows))
        # any 2-byte dtype is read as binary16 bit patterns
        r16 = torch.from_numpy(rows.view(np.int16)).cuda()
        _same(pv.l2_normalize(r16, elem), want)
        _same(pv.halfvec_to_vector(r16), pv.halfvec_to_vector(rows))
    else:
        _same(pv.vector_to_halfvec(r), pv.vector_to_halfvec(rows))
    for start, count in ((1, max(1, dim // 2)), (2, dim - 1 or 1), (dim, 5)):
        _same(pv.subvector(r, start, count, elem), pv.subvector(rows, start, count, elem))
    # in place gives what out of place gives
    lib = pv._lib.load()
    inplace = r.clone()
    pv._after_torch(inplace)
    assert lib.vb_l2_normalize_batch_dev(elem, dim, pv._ptr(inplace), n, pv._ptr(inplace)) == 0
    pv.synchronize()
    _same(inplace, want)


@gpu
def test_a_single_row_and_no_rows(pv):
    import torch
    x = np.array([3.0, -4.0, 0.0], np.float32)
    r = torch.from_numpy(x).cuda()
    assert float(pv.vector_norm(r)) == 5.0 and pv.vector_norm(r).dim() == 0
    _same(pv.l2_normalize(r), pv.l2_normalize(x))
    _same(pv.subvector(r, 2, 5), pv.subvector(x, 2, 5))
    e = torch.empty((0, 7), dtype=torch.float32, device="cuda")
    before = pv.launch_count()
    assert pv.vector_norm(e).shape == (0,) and pv.l2_normalize(e).shape == (0, 7)
    assert pv.binary_quantize(e).shape == (0, 1) and pv.vector_to_halfvec(e).shape == (0, 7)
    assert pv.subvector(e, 2, 3).shape == (0, 3)
    assert pv.launch_count() == before                  # n = 0 launches nothing


# ------------------------------------------------------------------------------- errors

@gpu
def test_halfvec_overflow_texts_name_the_first_offender(pv):
    import torch
    for x, text in ((np.array([[1.0, 2.0], [65520.0, -65520.0]], np.float32), '"65520" is out of range for type halfvec'),
                    (np.array([1.0, -3e38, 7e4], np.float32), '"-3e+38" is out of range for type halfvec'),
                    (np.array([1e5], np.float32), '"100000" is out of range for type halfvec'),
                    (np.array([[1.0, 7e4], [-3e38, 1.0]], np.float32), '"70000" is out of range for type halfvec')):
        for arg in (x, torch.from_numpy(x).cuda()):
            with pytest.raises(ValueError) as e:
                pv.vector_to_halfvec(arg)
            assert str(e.value) == text
    # many rows: the offender with the lowest row-major index, wherever the threads that see them run
    big = np.random.default_rng(5).standard_normal((100_000, 768)).astype(np.float32)
    big[99_000, 3] = 1e30
    big[61_234, 700] = -70_000.0
    big[61_235, 0] = 65_520.0
    with pytest.raises(ValueError, match='^"-70000" is out of range for type halfvec$'):
        pv.vector_to_halfvec(torch.from_numpy(big).cuda())


@gpu
def test_refused_dev_calls(pv):
    import torch
    lib = pv._lib.load()
    p = pv._ptr
    x = torch.ones((4, 8), dtype=torch.float32, device="cuda")
    out = torch.full((4, 8), 7.0, dtype=torch.float32, device="cuda")
    norms = torch.full((4,), 7.0, dtype=torch.float64, device="cuda")
    bits = torch.full((4, 1), 7, dtype=torch.uint8, device="cuda")
    for call in (lambda: lib.vb_norm_batch_dev(BIT, 8, p(x), 4, p(norms)),
                 lambda: lib.vb_norm_batch_dev(VECTOR, 0, p(x), 4, p(norms)),
                 lambda: lib.vb_l2_normalize_batch_dev(VECTOR, 8, p(x), -1, p(out)),
                 lambda: lib.vb_l2_normalize_batch_dev(VECTOR, 8, None, 4, p(out)),
                 lambda: lib.vb_binary_quantize_batch_dev(VECTOR, 8, p(x), 4, None),
                 lambda: lib.vb_vector_to_halfvec_batch_dev(-3, p(x), 4, p(out)),
                 lambda: lib.vb_halfvec_to_vector_batch_dev(8, None, 1, p(out)),
                 # overlapping input and output (only l2_normalize may run exactly in place)
                 lambda: lib.vb_l2_normalize_batch_dev(VECTOR, 8, p(x), 4, C.c_void_p(x.data_ptr() + 4)),
                 lambda: lib.vb_halfvec_to_vector_batch_dev(8, p(out), 4, p(out)),
                 lambda: lib.vb_norm_batch_dev(VECTOR, 8, p(out), 4, C.c_void_p(out.data_ptr() + 64))):
        assert call() == EINVAL
    pv.synchronize()
    assert torch.all(out == 7.0) and torch.all(norms == 7.0) and torch.all(bits == 7)
    for n in (0, 4):   # n = 0 is validated too
        assert lib.vb_norm_batch_dev(3, 8, p(x), n, p(norms)) == EINVAL
        assert "elem must be VB_VECTOR or VB_HALFVEC" in lib.vb_last_error().decode()


# ------------------------------------------------------------------------------- subvector

@gpu
@pytest.mark.parametrize("device", [False, True])
def test_subvector_against_the_reference_answers(pv, device):
    import torch
    for c in _cases():
        elem = VECTOR if c["type"] == "vector" else HALFVEC
        x = np.array(json.loads(c["input"]), np.float32 if elem == VECTOR else np.float16)
        arg = torch.from_numpy(x).cuda() if device else x
        if "error" in c:
            with pytest.raises(ValueError) as e:
                pv.subvector(arg, c["start"], c["count"], elem)
            assert str(e.value) == c["error"], c["sql"]
            continue
        got = pv.subvector(arg, c["start"], c["count"], elem)
        got = got.cpu().numpy() if device else got
        if elem == HALFVEC:
            got = got.view(np.float16)
        assert _text(got) == c["expected"], c["sql"]


@gpu
@pytest.mark.parametrize("elem,dim", [(VECTOR, 5), (VECTOR, 1536), (VECTOR, 37), (HALFVEC, 9), (HALFVEC, 768), (HALFVEC, 7)])
def test_subvector_sweep_against_numpy_slicing(pv, elem, dim):
    """start / count around every edge (negative, 0, past the end, INT32 limits), odd halfvec offsets, and device rows
    whose base address is only element-aligned; host and device give numpy's slice or the restated rule's error"""
    import torch
    half = elem == HALFVEC
    name = "halfvec" if half else "vector"
    rng = np.random.default_rng(dim)
    n = 3001
    rows = _special_rows(rng, n, dim, half)
    dt = np.float16 if half else np.float32
    # device rows 1 element past an aligned allocation: the widest word the kernel may use is then the element
    store = torch.empty(n * dim + 1, dtype=torch.float16 if half else torch.float32, device="cuda")
    store[1:] = torch.from_numpy(rows.view(dt).reshape(-1)).cuda()
    shifted = store[1:].view(n, dim)
    aligned = _to_dev(rows, half)
    starts = [INT32_MIN, -2**31 + 3, -5, -1, 0, 1, 2, 3, 4, 5, dim // 2, dim - 1, dim, dim + 1, INT32_MAX]
    counts = [INT32_MIN, -1, 0, 1, 2, 3, 4, 255, 256, dim - 1, dim, dim + 5, INT32_MAX]
    for start in starts:
        for count in counts:
            want = subvector_rule(dim, start, count, name)
            if isinstance(want, str):
                for arg in (rows, aligned):
                    with pytest.raises(ValueError) as e:
                        pv.subvector(arg, start, count, elem)
                    assert str(e.value) == want, (start, count)
                continue
            first, d = want
            sl = rows[:, first:first + d]
            _same(pv.subvector(rows, start, count, elem), sl)
            _same(pv.subvector(aligned, start, count, elem), sl)
            _same(pv.subvector(shifted, start, count, elem), sl)


@gpu
def test_a_refused_subvector_leaves_out_and_out_dim_untouched(pv):
    import torch
    lib = pv._lib.load()
    p = pv._ptr
    x = torch.arange(40, dtype=torch.float32, device="cuda").reshape(4, 10)
    xh = np.arange(40, dtype=np.float32).reshape(4, 10)
    out = torch.full((4, 10), 7.0, dtype=torch.float32, device="cuda")
    oh = np.full((4, 10), 7.0, np.float32)
    for elem, start, count, text in ((VECTOR, 1, 0, "vector must have at least 1 dimension"),
                                     (HALFVEC, 11, 1, "halfvec must have at least 1 dimension"),
                                     (VECTOR, -1, 2, "vector must have at least 1 dimension"),
                                     (BIT, 1, 3, "elem must be VB_VECTOR or VB_HALFVEC")):
        for fn, src, dst in ((lib.vb_subvector_batch_dev, p(x), p(out)), (lib.vb_subvector_batch, p(xh), p(oh))):
            d = C.c_int(12345)
            assert fn(elem, 10, src, 4, start, count, dst, C.byref(d)) == EINVAL
            assert text in lib.vb_last_error().decode()
            assert d.value == 12345
    # rows and output that overlap are refused the same way
    d = C.c_int(12345)
    assert lib.vb_subvector_batch_dev(VECTOR, 10, p(x), 4, 1, 5, C.c_void_p(x.data_ptr() + 8), C.byref(d)) == EINVAL
    assert d.value == 12345
    pv.synchronize()
    assert torch.all(out == 7.0) and np.all(oh == 7.0)
    assert torch.equal(x, torch.arange(40, dtype=torch.float32, device="cuda").reshape(4, 10))
    # n = 0 sizes the output, with no rows and no output
    d = C.c_int(0)
    assert lib.vb_subvector_batch_dev(HALFVEC, 10, None, 0, 4, 100, None, C.byref(d)) == 0 and d.value == 7


# ------------------------------------------------------------------------------- asynchrony

@gpu
def test_the_read_free_calls_replay_from_a_cuda_graph(pv):
    """norm, binary_quantize, halfvec_to_vector and subvector _dev read nothing back: they can be captured on vb_stream()
    and replayed, and the replay writes what the eager calls wrote"""
    import torch
    lib = pv._lib.load()
    p = pv._ptr
    n, dim = 5000, 768
    rng = np.random.default_rng(11)
    x = torch.from_numpy(_special_rows(rng, n, dim, False)).cuda()
    xh = torch.from_numpy(_special_rows(rng, n, dim, True).view(np.float16)).cuda()
    outs = [torch.empty(n, dtype=torch.float64, device="cuda"), torch.empty((n, dim // 8), dtype=torch.uint8, device="cuda"),
            torch.empty((n, dim), dtype=torch.float32, device="cuda"), torch.empty((n, 255), dtype=torch.float16, device="cuda")]
    d = C.c_int(0)

    def calls():
        assert lib.vb_norm_batch_dev(VECTOR, dim, p(x), n, p(outs[0])) == 0
        assert lib.vb_binary_quantize_batch_dev(HALFVEC, dim, p(xh), n, p(outs[1])) == 0
        assert lib.vb_halfvec_to_vector_batch_dev(dim, p(xh), n, p(outs[2])) == 0
        assert lib.vb_subvector_batch_dev(HALFVEC, dim, p(xh), n, 2, 255, p(outs[3]), C.byref(d)) == 0

    torch.cuda.synchronize()
    calls()
    pv.synchronize()
    eager = [o.clone() for o in outs]
    for o in outs:
        o.fill_(7)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=torch.cuda.ExternalStream(pv.stream_handle())):
        calls()
    for o in outs:
        o.fill_(3)
    torch.cuda.synchronize()
    g.replay()
    torch.cuda.synchronize()
    for o, e in zip(outs, eager):
        _same(o, e.cpu())
    assert d.value == 255


# ------------------------------------------------------------------------------- the README recipes on device tensors

@gpu
def test_half_precision_indexing_on_the_device(pv):
    """embedding::halfvec(n): fp32 rows -> vector_to_halfvec -> halfvec table -> exact top-k"""
    import torch
    rng = np.random.default_rng(21)
    n, dim, nq, k = 50_000, 512, 64, 10
    rows = rng.standard_normal((n, dim)).astype(np.float32)
    q = rng.standard_normal((nq, dim)).astype(np.float32)
    got_t = pv.Table(HALFVEC, dim).append(pv.vector_to_halfvec(torch.from_numpy(rows).cuda()))
    want_t = pv.Table(HALFVEC, dim).append(pv.vector_to_halfvec(rows))
    qd = pv.vector_to_halfvec(torch.from_numpy(q).cuda())
    qh = torch.from_numpy(pv.vector_to_halfvec(q).view(np.float16)).cuda()
    for metric in (pv.L2, pv.COSINE, pv.NEG_IP):
        ids, dist = got_t.exact_topk(metric, qd, k)
        wids, wdist = want_t.exact_topk(metric, qh, k)
        _same(ids, wids.cpu())
        _same(dist, wdist.cpu())
    got_t.free()
    want_t.free()


@gpu
def test_binary_quantization_with_rerank_on_the_device(pv):
    """binary_quantize(embedding)::bit(n): bit table top-20 by Hamming, re-ranked by <=> on the fp32 rows"""
    import torch
    rng = np.random.default_rng(22)
    n, dim, nq, c, k = 50_000, 1024, 64, 20, 10
    rows = rng.standard_normal((n, dim)).astype(np.float32)
    q = rng.standard_normal((nq, dim)).astype(np.float32)
    rows_d, q_d = torch.from_numpy(rows).cuda(), torch.from_numpy(q).cuda()
    full = pv.Table(VECTOR, dim).append(rows_d)
    got_b = pv.Table(BIT, dim).append(pv.binary_quantize(rows_d))
    want_b = pv.Table(BIT, dim).append(pv.binary_quantize(rows))
    cand, _ = got_b.exact_topk(pv.HAMMING, pv.binary_quantize(q_d), c)
    wcand, _ = want_b.exact_topk(pv.HAMMING, torch.from_numpy(pv.binary_quantize(q)).cuda(), c)
    _same(cand, wcand.cpu())
    ids, dist = full.rerank(pv.COSINE, q_d, cand, k)
    wids, wdist = full.rerank(pv.COSINE, q_d, wcand, k)
    _same(ids, wids.cpu())
    _same(dist, wdist.cpu())
    for t in (full, got_b, want_b):
        t.free()


@gpu
def test_subvector_indexing_on_the_device(pv):
    """subvector(embedding, 1, 256)::vector(256) under vector_cosine_ops: build from the device subvectors; queries
    through subvector -> l2_normalize -> search -> re-rank against the full rows"""
    import torch
    rng = np.random.default_rng(23)
    n, dim, sub, nq, lists, probes, c, k = 20_000, 1536, 256, 64, 40, 8, 40, 10
    rows = rng.standard_normal((n, dim)).astype(np.float32)
    rows[17] = 0                                          # norm 0: not indexed
    q = rng.standard_normal((nq, dim)).astype(np.float32)
    rows_d, q_d = torch.from_numpy(rows).cuda(), torch.from_numpy(q).cuda()
    full = pv.Table(VECTOR, dim).append(rows_d)
    results = []
    for rows_sub, q_norm in ((pv.subvector(rows_d, 1, sub), pv.l2_normalize(pv.subvector(q_d, 1, sub))),
                             (torch.from_numpy(pv.subvector(rows, 1, sub)).cuda(),
                              torch.from_numpy(pv.l2_normalize(pv.subvector(q, 1, sub))).cuda())):
        ix = pv.IvfflatIndex("vector_cosine_ops", sub, lists)
        lists_of_row, order, _ = ix.build(rows_sub, np.arange(n), seed=9)
        assert lists_of_row[17] == -1
        cand, _ = ix.search(q_norm, c, probes=probes)
        ids, dist = full.rerank(pv.COSINE, q_d, cand, k)
        results.append((lists_of_row, order, ix.centers(), _bits(q_norm), cand.cpu(), ids.cpu(), dist.cpu()))
        ix.free()
    for a, b in zip(*results):
        _same(a, b)
    full.free()


# ------------------------------------------------------------------------------- IvfflatIndex.insert, cosine

@gpu
@pytest.mark.parametrize("opclass", ["vector_cosine_ops", "halfvec_cosine_ops"])
def test_cosine_insert_of_device_rows_equals_the_host_path(pv, opclass):
    import torch
    half = opclass.startswith("halfvec")
    rng = np.random.default_rng(24 + half)
    n, m, dim, lists = 6000, 1500, 96, 24
    base = rng.standard_normal((n, dim)).astype(np.float32)
    new = rng.standard_normal((m, dim)).astype(np.float32)
    new[[3, 700, 1499]] = 0                               # norm 0: skipped, list -1
    new[5, 7] = np.nan                                    # norm NaN: skipped too
    new[9] *= 1e-3
    if half:
        base, new = base.astype(np.float16), new.astype(np.float16)
    host_ix, dev_ix = pv.IvfflatIndex(opclass, dim, lists), pv.IvfflatIndex(opclass, dim, lists)
    for ix in (host_ix, dev_ix):
        ix.build(base, np.arange(n), seed=4)
    ids = np.arange(m) + 10_000
    want = host_ix.insert(new, ids)
    got = dev_ix.insert(torch.from_numpy(new).cuda(), torch.from_numpy(ids).cuda())
    assert np.array_equal(got, want)
    assert (want[[3, 5, 700, 1499]] == -1).all() and (np.delete(want, [3, 5, 700, 1499]) >= 0).all()
    assert np.array_equal(dev_ix.list_offsets(), host_ix.list_offsets())
    # the images hold the same rows in the same places: every row's distance to the queries, in order
    q = rng.standard_normal((8, dim)).astype(np.float16 if half else np.float32)
    qn = torch.from_numpy(host_ix.prepare_query(q).view(np.float16) if half else host_ix.prepare_query(q)).cuda()
    a = dev_ix.search(qn, 1000, probes=lists)
    b = host_ix.search(qn, 1000, probes=lists)
    _same(a[0], b[0].cpu())
    _same(a[1], b[1].cpu())
    host_ix.free()
    dev_ix.free()
