"""sparsevec on device buffers: the _dev variants of the sparse table calls (append, exact top-k, filtered top-k, re-rank,
filter creation), the device CSR check they share, and the casts between vector / halfvec and sparsevec.

Every _dev result is compared with the host variant's on the same table: ids equal, distances the float of the host
float8 bit for bit.  The casts are checked against the reference's answers (cast.out, tests/golden/sparsevec_casts.json)
and a numpy restatement.  The first tests need no device."""
import ctypes as C
import json
import os

import numpy as np
import pytest

import oracle as O
from tests.test_oracle_sparse import random_sparse

EINVAL, ENODEVICE = -1, -2
METRICS = [O.L2, O.L2_SQUARED, O.NEG_IP, O.COSINE, O.L1]
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "sparsevec_casts.json")
NEW_SYMBOLS = ["vb_sparse_table_append_dev", "vb_sparse_exact_topk_dev", "vb_sparse_table_filter_create_dev",
               "vb_sparse_exact_topk_filtered_dev", "vb_sparse_table_rerank_dev", "vb_dense_to_sparsevec_batch",
               "vb_dense_to_sparsevec_batch_dev", "vb_sparsevec_to_dense_batch", "vb_sparsevec_to_dense_batch_dev"]


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
    S = pv.sparsevec
    for fn, arg in ((S.vector_to_sparsevec, np.ones((2, 3), np.float32)), (S.halfvec_to_sparsevec, np.ones((2, 3), np.float16)),
                    (S.sparsevec_to_vector, [S.SparseVector(3, [1], [2.0])]), (S.sparsevec_to_halfvec, [S.SparseVector(3, [1], [2.0])])):
        with pytest.raises(pv.VecB200Error) as e:
            fn(arg)
        assert e.value.code == ENODEVICE, fn.__name__
    lib = pv._lib.load()
    h = C.c_void_p()
    assert lib.vb_sparse_table_append_dev(None, 1, None, None, None) == ENODEVICE
    assert lib.vb_sparse_exact_topk_dev(None, O.L2, 3, 1, None, None, None, 1, None, None) == ENODEVICE
    assert lib.vb_sparse_table_filter_create_dev(None, None, 0, C.byref(h)) == ENODEVICE
    assert lib.vb_sparse_exact_topk_filtered_dev(None, O.L2, 3, 1, None, None, None, 1, None, 1, None, None, None) == ENODEVICE
    assert lib.vb_sparse_table_rerank_dev(None, O.L2, 3, 1, None, None, None, None, 1, 1, None, None) == ENODEVICE
    assert lib.vb_dense_to_sparsevec_batch_dev(0, 3, None, 1, 0, None, None, None) == ENODEVICE
    assert lib.vb_sparsevec_to_dense_batch_dev(0, 3, 1, None, None, None, None) == ENODEVICE


def test_the_cast_fixture_reads():
    cases = json.load(open(GOLDEN))["cases"]
    assert {c["cast"] for c in cases} == {"vector_to_sparsevec", "halfvec_to_sparsevec", "sparsevec_to_vector", "sparsevec_to_halfvec"}
    assert all(("expected" in c) != ("error" in c) for c in cases)


# ------------------------------------------------------------------------------- helpers

gpu = pytest.mark.gpu


@pytest.fixture(scope="module")
def pv():
    import pgvector_b200 as pv
    pv.init(0)
    return pv


def _dev(R):
    """SparseRows -> (row_off, idx, val) CUDA tensors"""
    import torch
    return (torch.from_numpy(R.row_off).cuda(), torch.from_numpy(R.idx.astype(np.int32)).cuda(),
            torch.from_numpy(R.val.astype(np.float32)).cuda())


def _rows(pv, rng, dim, n, lo=1, hi=150, zero_every=0):
    S = pv.sparsevec
    rows = [random_sparse(rng, dim, int(rng.integers(lo, hi))) for _ in range(n)]
    if zero_every:
        for r in range(0, n, zero_every):
            rows[r] = S.SparseVector(dim)
    return rows


def _f32_bits(a):
    return np.ascontiguousarray(a, dtype=np.float32).view(np.int32)


def _same_as_host(got, want):
    """_dev result (CUDA tensors) against the host result (int64, float8): ids equal, distances (float) of the float8"""
    ids, dist = got[0].cpu().numpy(), got[1].cpu().numpy()
    assert np.array_equal(ids, want[0])
    w = want[1].astype(np.float32)
    assert np.array_equal(np.isnan(dist), np.isnan(w))
    ok = ~np.isnan(w)
    assert np.array_equal(_f32_bits(dist)[ok], _f32_bits(w)[ok])


def _mixed_table(pv, dim, rows, split):
    """one host append, then one _dev append"""
    S = pv.sparsevec
    t = S.SparseTable(dim).append(rows[:split])
    t.append(_dev(S.SparseRows.from_vectors(rows[split:], dim)))
    return t


# ------------------------------------------------------------------------------- bit identity with the host calls

@gpu
@pytest.mark.parametrize("metric", METRICS)
def test_dev_calls_equal_the_host_calls(pv, metric):
    S = pv.sparsevec
    rng = np.random.default_rng(metric + 300)
    dim, n, nq, k, c = 5000, 1500, 40, 20, 64
    rows = _rows(pv, rng, dim, n, zero_every=97)          # zero-norm rows: cosine NaN
    queries = [random_sparse(rng, dim, int(rng.integers(1, 120))) for _ in range(nq)]
    queries[3] = S.SparseVector(dim)                       # a zero-nnz query
    queries[5] = rows[10]
    Q = S.SparseRows.from_vectors(queries, dim)
    Qd = _dev(Q)
    t = _mixed_table(pv, dim, rows, 700)
    ref = S.SparseTable(dim).append(rows[:700]).append(rows[700:])
    assert (t.rows, t.nnz) == (ref.rows, ref.nnz)
    want = t.exact_topk(metric, Q, k)
    # the _dev append stored what the host append stores
    w2 = ref.exact_topk(metric, Q, k)
    assert np.array_equal(want[0], w2[0]) and np.array_equal(want[1].view(np.int64), w2[1].view(np.int64))
    _same_as_host(t.exact_topk(metric, Qd, k), want)
    # filtered: several filters (one made on the device), filter_of_query
    allowed = [np.sort(rng.choice(n, size=s, replace=False)) for s in (3, 50, 800)]
    import torch
    filters = [t.filter(allowed[0]), t.filter(torch.from_numpy(allowed[1]).cuda()), t.filter(allowed[2])]
    fq = (np.arange(nq) % 3).astype(np.int32)
    _same_as_host(t.exact_topk(metric, Qd, k, filter=filters, filter_of_query=fq),
                  t.exact_topk(metric, Q, k, filter=filters, filter_of_query=fq))
    _same_as_host(t.exact_topk(metric, Qd, k, filter=filters[2]), t.exact_topk(metric, Q, k, filter=filters[2]))
    # re-rank, with -1 and a duplicate
    cand = rng.integers(-1, n, size=(nq, c)).astype(np.int64)
    cand[:, 7] = cand[:, 1]
    _same_as_host(t.rerank(metric, Qd, torch.from_numpy(cand).cuda(), k), t.rerank(metric, Q, cand, k))
    for f in filters:
        f.free()
    t.free()
    ref.free()


@gpu
def test_an_empty_table_and_no_queries(pv):
    import torch
    S = pv.sparsevec
    t = S.SparseTable(50)
    Q = S.SparseRows.from_vectors([S.SparseVector(50, [3], [1.0]), S.SparseVector(50)], 50)
    ids, dist = t.exact_topk(O.L2, _dev(Q), 3)
    assert ids.is_cuda and dist.is_cuda and dist.dtype == torch.float32
    assert torch.all(ids == -1) and torch.all(torch.isinf(dist))
    z = S.SparseRows(50, np.zeros(1, np.int64), np.empty(0, np.int32), np.empty(0, np.float32))
    ids, dist = t.exact_topk(O.L2, _dev(z), 3)
    assert ids.shape == (0, 3)
    t.append(_dev(z))
    assert t.rows == 0
    t.free()


@gpu
def test_sub_batches(pv):
    """more than 65535 queries, and a table whose key runs split at 1 GiB: the host call's answer"""
    import torch
    S = pv.sparsevec
    rng = np.random.default_rng(31)
    dim, n, nq, k = 500, 40, 65_535 + 1234, 3
    t = _mixed_table(pv, dim, _rows(pv, rng, dim, n, hi=20), 25)
    nnz = rng.integers(0, 6, nq)
    off = np.zeros(nq + 1, np.int64)
    off[1:] = np.cumsum(nnz)
    idx = np.concatenate([np.sort(rng.choice(dim, size=m, replace=False)) for m in nnz]).astype(np.int32)
    Q = S.SparseRows(dim, off, idx, rng.standard_normal(idx.size).astype(np.float32))
    Qd = _dev(Q)
    _same_as_host(t.exact_topk(O.L2, Qd, k), t.exact_topk(O.L2, Q, k))
    with t.filter(np.arange(n)) as f:
        _same_as_host(t.exact_topk(O.L2, Qd, k, filter=f), t.exact_topk(O.L2, Q, k, filter=f))
    cand = np.tile(np.arange(n, dtype=np.int64), (nq, 1))
    _same_as_host(t.rerank(O.L2, Qd, torch.from_numpy(cand).cuda(), k), t.rerank(O.L2, Q, cand, k))
    t.free()
    # 300k rows: the exact scan takes 894 queries per sub-batch, a filter of every row splits at 2^28 distances
    n2, nq2 = 300_000, 2000
    nn = rng.integers(0, 4, n2)
    off2 = np.zeros(n2 + 1, np.int64)
    off2[1:] = np.cumsum(nn)
    first = np.repeat(rng.integers(0, dim - 3, n2), nn)                  # runs of consecutive indices
    idx2 = (first + np.arange(off2[-1]) - np.repeat(off2[:-1], nn)).astype(np.int32)
    R = S.SparseRows(dim, off2, idx2, rng.standard_normal(idx2.size).astype(np.float32))
    big = S.SparseTable(dim).append(_dev(R))
    Q2 = S.SparseRows(dim, off[:nq2 + 1], idx[:off[nq2]], Q.val[:off[nq2]])
    _same_as_host(big.exact_topk(O.NEG_IP, _dev(Q2), k), big.exact_topk(O.NEG_IP, Q2, k))
    with big.filter(np.arange(n2)) as f:
        _same_as_host(big.exact_topk(O.NEG_IP, _dev(Q2), k, filter=f), big.exact_topk(O.NEG_IP, Q2, k, filter=f))
    big.free()


# ------------------------------------------------------------------------------- validation

def _defects(dim):
    """(name, row_off, idx, bad row) of CSR defects; values follow idx"""
    M = 16_000
    return [
        ("first offset", [1, 2, 3], [0, 1, 2], 0),
        ("decreasing", [0, 2, 1, 3], [0, 1, 2], 1),
        ("nnz above the limit", [0, 1, 1 + M + 1], [0] + list(range(M + 1)), 1),
        ("index below 0", [0, 1, 3], [0, 1, -1], 1),
        ("index at dim", [0, 2, 3], [0, dim, 2], 0),
        ("equal indices", [0, 1, 2, 4], [0, 1, 3, 3], 2),
        ("descending indices", [0, 1, 3], [4, 5, 2], 1),
    ]


@gpu
@pytest.mark.parametrize("case", range(7))
def test_csr_defects_are_refused_with_the_host_text_and_the_row(pv, case):
    import torch
    S = pv.sparsevec
    lib = pv._lib.load()
    dim = 20_000
    name, off, idx, bad_row = _defects(dim)[case]
    off = np.array(off, np.int64)
    idx = np.array(idx, np.int32)
    val = np.ones(idx.size, np.float32)
    n = off.size - 1
    p = S._p
    rng = np.random.default_rng(case)
    t = S.SparseTable(dim).append(_rows(pv, rng, dim, 30, hi=10))
    # the host variant's text, plus the row where it does not name one
    assert lib.vb_sparse_table_append(t.h, n, p(off), p(idx), p(val)) == EINVAL
    host = lib.vb_last_error().decode()
    want = host if "(row" in host or "start at 0" in host else f"{host} (row {bad_row})"
    assert f"(row {bad_row})" in want or "start at 0" in want
    d_off, d_idx, d_val = (torch.from_numpy(a).cuda() for a in (off, idx, val))
    tp = S._tp
    q = [random_sparse(rng, dim, 5) for _ in range(3)]
    before = t.exact_topk(O.L1, q, 4)
    rows_nnz = (t.rows, t.nnz)
    assert lib.vb_sparse_table_append_dev(t.h, n, tp(d_off), tp(d_idx), tp(d_val)) == EINVAL
    assert lib.vb_last_error().decode() == want
    assert (t.rows, t.nnz) == rows_nnz
    after = t.exact_topk(O.L1, q, 4)
    assert np.array_equal(before[0], after[0]) and np.array_equal(before[1], after[1])
    # the same CSR as queries: the text names "queries", nothing is written
    assert lib.vb_sparse_exact_topk(t.h, O.L2, dim, n, p(off), p(idx), p(val), 2, p(np.empty((n, 2), np.int64)),
                                    p(np.empty((n, 2), np.float64))) == EINVAL
    qhost = lib.vb_last_error().decode()
    qwant = qhost if "(row" in qhost or "start at 0" in qhost else f"{qhost} (row {bad_row})"
    ids = torch.full((n, 2), 12345, dtype=torch.int64, device="cuda")
    dist = torch.full((n, 2), 6.5, dtype=torch.float32, device="cuda")
    cand = torch.zeros((n, 4), dtype=torch.int64, device="cuda")
    with t.filter([1, 2]) as f:
        farr = (C.c_void_p * 1)(f.h.value)
        calls = [
            lambda: lib.vb_sparse_exact_topk_dev(t.h, O.L2, dim, n, tp(d_off), tp(d_idx), tp(d_val), 2, tp(ids), tp(dist)),
            lambda: lib.vb_sparse_exact_topk_filtered_dev(t.h, O.L2, dim, n, tp(d_off), tp(d_idx), tp(d_val), 2, farr, 1, None, tp(ids),
                                                          tp(dist)),
            lambda: lib.vb_sparse_table_rerank_dev(t.h, O.L2, dim, n, tp(d_off), tp(d_idx), tp(d_val), tp(cand), 4, 2, tp(ids), tp(dist)),
        ]
        for call in calls:
            assert call() == EINVAL
            assert lib.vb_last_error().decode() == qwant
            pv.synchronize()
            assert torch.all(ids == 12345) and torch.all(dist == 6.5)
    # and the casts to dense check the same way
    out = torch.full((n, 16_000), 7.0, dtype=torch.float32, device="cuda")
    assert lib.vb_sparsevec_to_dense_batch_dev(0, 16_000, n, tp(d_off), tp(d_idx), tp(d_val), tp(out)) == EINVAL
    assert "start at 0" in lib.vb_last_error().decode() or f"(row {bad_row})" in lib.vb_last_error().decode()
    pv.synchronize()
    assert torch.all(out == 7.0)
    t.free()


@gpu
def test_rerank_dev_candidates_outside_the_table_are_absent(pv):
    import torch
    S = pv.sparsevec
    rng = np.random.default_rng(41)
    dim, n, nq, c, k = 2000, 200, 16, 30, 12
    t = _mixed_table(pv, dim, _rows(pv, rng, dim, n, zero_every=17), 90)
    Q = S.SparseRows.from_vectors([random_sparse(rng, dim, 30) for _ in range(nq)], dim)
    cand = rng.integers(-5, n + 5, size=(nq, c)).astype(np.int64)
    cand[0, :] = n                                       # nothing valid at all
    cand[1, 3] = 2**40
    cand[2, 4] = -2**40
    host = np.where((cand >= 0) & (cand < n), cand, -1)
    _same_as_host(t.rerank(O.COSINE, _dev(Q), torch.from_numpy(cand).cuda(), k), t.rerank(O.COSINE, Q, host, k))
    t.free()


@gpu
def test_device_filters_equal_host_filters(pv):
    import torch
    S = pv.sparsevec
    rng = np.random.default_rng(43)
    dim, n = 3000, 500
    t = _mixed_table(pv, dim, _rows(pv, rng, dim, n), 200)
    rows = np.array([5, 499, 5, 7, -1, 500, 10**12, 7, 0], np.int64)
    fd = t.filter(torch.from_numpy(rows).cuda())
    fh = t.filter([0, 5, 7, 499])
    assert len(fd) == len(fh) == 4
    Q = S.SparseRows.from_vectors([random_sparse(rng, dim, 40) for _ in range(5)], dim)
    a = t.exact_topk(O.L2, Q, 6, filter=fd)
    b = t.exact_topk(O.L2, Q, 6, filter=fh)
    assert np.array_equal(a[0], b[0]) and np.array_equal(a[1].view(np.int64), b[1].view(np.int64))
    with t.filter(torch.empty(0, dtype=torch.int64, device="cuda")) as e:
        assert len(e) == 0
    fd.free()
    fh.free()
    t.free()


# ------------------------------------------------------------------------------- casts

def _dense_text(x):
    return "[" + ",".join(f"{float(v):g}" for v in x) + "]"


@gpu
@pytest.mark.parametrize("device", [False, True])
def test_casts_against_the_reference_answers(pv, device):
    import torch
    S = pv.sparsevec
    for case in json.load(open(GOLDEN))["cases"]:
        fn = getattr(S, case["cast"])
        if case["cast"].endswith("_to_sparsevec"):
            x = np.array(json.loads(case["input"]), np.float32 if case["cast"].startswith("vector") else np.float16)
            if device:
                off, idx, val = fn(torch.from_numpy(x).cuda())
                R = S.SparseRows(x.size, off.cpu().numpy(), idx.cpu().numpy(), val.cpu().numpy())
            else:
                R = fn(x)
            assert R.row(0).to_text() == case["expected"], case["sql"]
            continue
        v = S.SparseVector.from_text(case["input"])
        arg = S.SparseRows.from_vectors([v])
        if device:
            arg = (*_dev(arg),)
        if "error" in case:
            with pytest.raises(ValueError) as e:
                fn(arg, dim=v.dim) if device else fn(arg)
            assert str(e.value) == case["error"], case["sql"]
            continue
        out = fn(arg, dim=v.dim) if device else fn(arg)
        out = out.cpu().numpy() if device else out
        assert _dense_text(out[0]) == case["expected"], case["sql"]


def _random_dense(rng, n, dim, half):
    x = rng.standard_normal((n, dim)).astype(np.float32)
    x[rng.random((n, dim)) < 0.7] = 0.0
    x[rng.random((n, dim)) < 0.05] = -0.0
    if half:
        h = x.astype(np.float16)
        b = h.view(np.uint16)
        sub = rng.random((n, dim)) < 0.05
        b[sub] = rng.integers(1, 0x400, int(sub.sum())).astype(np.uint16) | (rng.integers(0, 2, int(sub.sum())).astype(np.uint16) << 15)
        b[:, 0] = 0x8000                                     # -0 is dropped
        return h
    x[:, 0] = -0.0
    x[0, :] = 0.0                                           # a row with nothing kept
    return x


@gpu
@pytest.mark.parametrize("half", [False, True])
def test_casts_on_random_rows(pv, half):
    import torch
    S = pv.sparsevec
    rng = np.random.default_rng(7 + half)
    n, dim = 700, 1537
    x = _random_dense(rng, n, dim, half)
    to_sparse = S.halfvec_to_sparsevec if half else S.vector_to_sparsevec
    to_dense = S.sparsevec_to_halfvec if half else S.sparsevec_to_vector
    # numpy restatement: kept = nonzero bit pattern outside the sign, in index order, values widened
    bits = x.view(np.uint16) & 0x7FFF if half else (x != 0)
    keep = bits != 0
    r, c = np.nonzero(keep)
    want_off = np.zeros(n + 1, np.int64)
    want_off[1:] = np.cumsum(keep.sum(1))
    want_val = x[r, c].astype(np.float32)
    R = to_sparse(x)
    assert np.array_equal(R.row_off, want_off) and np.array_equal(R.idx, c.astype(np.int32))
    assert np.array_equal(R.val.view(np.int32), want_val.view(np.int32))
    off, idx, val = to_sparse(torch.from_numpy(x).cuda())
    assert np.array_equal(off.cpu().numpy(), R.row_off) and np.array_equal(idx.cpu().numpy(), R.idx)
    assert np.array_equal(val.cpu().numpy().view(np.int32), R.val.view(np.int32))
    off2, idx2, val2 = to_sparse(torch.from_numpy(x).cuda(), cap=int(want_off[-1]))
    assert torch.equal(off2, off) and torch.equal(idx2, idx) and torch.equal(val2, val)
    # back: the identity up to the dropped -0
    back = to_dense(R)
    xz = np.where(keep, x, np.zeros_like(x))
    assert np.array_equal(back.view(np.uint16 if half else np.int32), xz.view(np.uint16 if half else np.int32))
    back_d = to_dense((off, idx, val), dim=dim)
    assert np.array_equal(back_d.cpu().numpy().view(np.uint16 if half else np.int32), back.view(np.uint16 if half else np.int32))
    # cap too small: offsets written, nothing else, the count named
    lib = pv._lib.load()
    o = np.empty(n + 1, np.int64)
    assert lib.vb_dense_to_sparsevec_batch(int(half), dim, S._p(np.ascontiguousarray(x)), n, 5, S._p(o), None, None) == EINVAL
    assert f"{int(want_off[-1])} non-zero elements, more than cap = 5" in lib.vb_last_error().decode()
    assert np.array_equal(o, want_off)


@gpu
def test_sparse_to_halfvec_rounding_and_overflow(pv):
    import torch
    S = pv.sparsevec
    dim = 6
    vals = np.array([1e-8, -1e-8, 65504.0, 1e-6, 3.14159], np.float32)
    R = S.SparseRows(dim, np.array([0, 2, 5], np.int64), np.array([0, 5, 1, 2, 3], np.int32), vals)
    h = S.sparsevec_to_halfvec(R)
    want = np.zeros((2, dim), np.float16)
    want[0, 0], want[0, 5], want[1, 1], want[1, 2], want[1, 3] = vals.astype(np.float16)
    assert np.array_equal(h.view(np.uint16), want.view(np.uint16))
    assert np.array_equal(S.sparsevec_to_halfvec(_dev(R), dim=dim).cpu().numpy().view(np.uint16), want.view(np.uint16))
    over = S.SparseRows(dim, np.array([0, 1, 3], np.int64), np.array([2, 0, 4], np.int32), np.array([1.0, 70000.0, 65520.0], np.float32))
    for arg, kw in ((over, {}), (_dev(over), {"dim": dim})):
        with pytest.raises(ValueError, match='^"70000" is out of range for type halfvec$'):
            S.sparsevec_to_halfvec(arg, **kw)
    assert torch.equal(S.sparsevec_to_vector(_dev(over), dim=dim).cpu(), torch.from_numpy(S.sparsevec_to_vector(over)))


# ------------------------------------------------------------------------------- a pipeline on device buffers

@gpu
def test_dense_candidates_reranked_by_the_sparse_column_on_the_device(pv):
    """vb_exact_topk_dev ids -> vb_sparse_table_rerank_dev on a sparse table whose row numbers are the dense table's,
    with the inputs made on another torch stream: the host path's answer"""
    import torch
    S = pv.sparsevec
    rng = np.random.default_rng(53)
    n, ddim, sdim, nq, c, k = 4000, 64, 3000, 32, 100, 10
    dense = rng.standard_normal((n, ddim)).astype(np.float32)
    srows = S.SparseRows.from_vectors(_rows(pv, rng, sdim, n, hi=60), sdim)
    qd = rng.standard_normal((nq, ddim)).astype(np.float32)
    qs = S.SparseRows.from_vectors([random_sparse(rng, sdim, 40) for _ in range(nq)], sdim)
    T = pv.Table(O.VECTOR, ddim).append(dense)
    st = S.SparseTable(sdim).append(srows)
    want_c, _ = T.exact_topk(O.L2, qd, c)
    want = st.rerank(O.NEG_IP, qs, want_c, k)
    side = torch.cuda.Stream()
    with torch.cuda.stream(side):
        q_dev = torch.from_numpy(qd).cuda().clone()   # produced on the side stream
        qs_dev = tuple(a.clone() for a in _dev(qs))
        cand, _ = T.exact_topk(O.L2, q_dev, c)
        got = st.rerank(O.NEG_IP, qs_dev, cand, k)
    side.synchronize()
    assert np.array_equal(cand.cpu().numpy(), want_c)
    _same_as_host(got, want)
    T.free()
    st.free()
