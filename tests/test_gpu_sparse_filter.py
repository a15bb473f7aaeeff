"""Filtered and re-ranked sparsevec queries over a resident CSR table (vb_sparse_table_filter_create,
vb_sparse_exact_topk_filtered, vb_sparse_table_rerank): the plan of WHERE <predicate> ORDER BY v <op> q LIMIT k with a
B-tree or bitmap scan on the filter column, and the re-rank of another index's candidates by the sparse column.

Against the oracle (oracle/pgv_sparse.c) over the allowed rows, bit for bit against vb_sparse_exact_topk and against each
other, on the reference's tiny orderings (hnsw_sparsevec.out), at the edges, and on every refused call (outputs left
untouched).  The first test needs no device."""
import ctypes as C
import math

import numpy as np
import pytest

import oracle as O
from tests.test_oracle_sparse import OPS, ORDERINGS, random_sparse, sv

RTOL = 1e-5   # as tests/test_gpu_sparse.py
EINVAL, ENODEVICE = -1, -2
METRICS = [O.L2, O.L2_SQUARED, O.NEG_IP, O.COSINE, O.L1]


# ------------------------------------------------------------------------------- anywhere

def test_without_a_device_every_new_entry_point_is_an_error():
    import torch
    if torch.cuda.is_available():
        pytest.skip("a device is visible")
    import pgvector_b200 as pv
    S = pv.sparsevec
    t = object.__new__(S.SparseTable)      # the constructor itself needs a device
    t.dim, t.h = 5, None
    q = [S.SparseVector(5, [0], [1.0])]
    with pytest.raises(pv.VecB200Error) as e:
        t.filter([0])
    assert e.value.code == ENODEVICE
    buf = C.create_string_buffer(256)
    f = pv.Filter(t, C.c_void_p(C.addressof(buf)))
    try:
        with pytest.raises(pv.VecB200Error) as e:
            t.exact_topk(O.L2, q, 1, filter=f)
        assert e.value.code == ENODEVICE
    finally:
        f.h = None
    with pytest.raises(pv.VecB200Error) as e:
        t.rerank(O.L2, q, np.zeros((1, 1), np.int64), 1)
    assert e.value.code == ENODEVICE


# ------------------------------------------------------------------------------- on the GPU

gpu = pytest.mark.gpu


@pytest.fixture(scope="module")
def pv():
    import pgvector_b200 as pv
    pv.init(0)
    return pv


def _rows(pv, rng, dim, n, lo=1, hi=150, zero_every=0):
    S = pv.sparsevec
    rows = [random_sparse(rng, dim, int(rng.integers(lo, hi))) for _ in range(n)]
    if zero_every:
        for r in range(0, n, zero_every):
            rows[r] = S.SparseVector(dim)
    return rows


def _table(pv, dim, rows, split=None):
    t = pv.sparsevec.SparseTable(dim)
    split = len(rows) // 2 if split is None else split
    t.append(rows[:split]).append(rows[split:])      # two appends: offsets are rebased on the device
    return t


def _bits(a):
    return np.ascontiguousarray(a, dtype=np.float64).view(np.int64)


def _same(got, want):
    assert np.array_equal(got[0], want[0])
    assert np.array_equal(_bits(got[1]), _bits(want[1]))


def _check_against_oracle(ids, dist, d, allowed, k):
    """ids / dist of one query against the oracle distances d over all rows, restricted to `allowed` (ascending)"""
    take = min(k, allowed.size)
    assert np.all(ids[take:] == -1) and np.all(np.isinf(dist[take:]))
    if take == 0:
        return
    order = allowed[np.argsort(d[allowed], kind="stable")[:take]]
    got = ids[:take]
    assert np.isin(got, allowed).all()
    if not np.array_equal(got, order):
        cut = d[order[-1]]
        for i in set(got.tolist()) ^ set(order.tolist()):
            assert abs(d[i] - cut) <= 2 * RTOL * max(abs(cut), 1e-30)
    assert np.all(np.abs(dist[:take] - d[got]) <= 2 * RTOL * np.maximum(np.abs(d[got]), 1e-6))


@gpu
@pytest.mark.parametrize("metric", METRICS)
def test_filtered_topk_matches_the_oracle(pv, metric):
    S = pv.sparsevec
    rng = np.random.default_rng(metric + 40)
    dim, n, nq, k = 30_000, 6000, 48, 10
    rows = _rows(pv, rng, dim, n)
    queries = [random_sparse(rng, dim, int(rng.integers(1, 200))) for _ in range(nq)]
    t = _table(pv, dim, rows, 2500)
    allowed = [np.sort(rng.choice(n, size=s, replace=False)) for s in (6, 60, 900, 4000)]
    filters = [t.filter(a) for a in allowed]
    assert [len(f) for f in filters] == [a.size for a in allowed]
    fq = rng.integers(0, len(filters), nq).astype(np.int32)
    ids, dist = t.exact_topk(metric, queries, k, filter=filters, filter_of_query=fq)
    R = S.SparseRows.from_vectors(rows, dim)
    for qi, q in enumerate(queries):
        d = O.sparse_distance_batch(metric, sv(q), R.row_off, R.idx, R.val)
        _check_against_oracle(ids[qi], dist[qi], d, allowed[fq[qi]], k)
    # one shared filter, given alone
    ids1, dist1 = t.exact_topk(metric, queries, k, filter=filters[2])
    for qi, q in enumerate(queries[:8]):
        d = O.sparse_distance_batch(metric, sv(q), R.row_off, R.idx, R.val)
        _check_against_oracle(ids1[qi], dist1[qi], d, allowed[2], k)
    for f in filters:
        f.free()
    t.free()


@gpu
@pytest.mark.parametrize("metric", METRICS)
def test_bit_identity_with_the_exact_scan_and_the_rerank(pv, metric):
    """on a table built by two appends, with zero-nnz rows and queries (cosine NaN): a filter of every row gives
    vb_sparse_exact_topk; each filtered result is the re-rank of its filter's rows in ascending order; a re-rank of every
    row in order gives vb_sparse_exact_topk"""
    S = pv.sparsevec
    rng = np.random.default_rng(metric + 70)
    dim, n, nq, k = 5000, 1500, 24, 20
    rows = _rows(pv, rng, dim, n, zero_every=97)
    queries = [random_sparse(rng, dim, int(rng.integers(1, 120))) for _ in range(nq)]
    queries[3] = S.SparseVector(dim)
    # queries sharing entries with rows: real matches, and ties at equal distances
    queries[5] = rows[10]
    t = _table(pv, dim, rows, 700)
    want = t.exact_topk(metric, queries, k)
    every = t.filter(np.arange(n))
    _same(t.exact_topk(metric, queries, k, filter=every), want)
    cand = np.tile(np.arange(n, dtype=np.int64), (nq, 1))
    _same(t.rerank(metric, queries, cand, k), want)
    # and with k = n: every row's distance
    if n <= 2048:
        full = t.exact_topk(metric, queries, n)
        _same(t.exact_topk(metric, queries, n, filter=every), full)
        _same(t.rerank(metric, queries, cand, n), full)
    allowed = [np.sort(rng.choice(n, size=s, replace=False)) for s in (3, 50, 800)]
    filters = [t.filter(a) for a in allowed]
    fq = (np.arange(nq) % 3).astype(np.int32)
    got = t.exact_topk(metric, queries, k, filter=filters, filter_of_query=fq)
    for j in range(3):
        sel = np.flatnonzero(fq == j)
        sub = [queries[i] for i in sel]
        c = np.tile(allowed[j].astype(np.int64), (sel.size, 1))
        _same((got[0][sel], got[1][sel]), t.rerank(metric, sub, c, k))
    for f in filters + [every]:
        f.free()
    t.free()


@gpu
@pytest.mark.parametrize("block", ORDERINGS, ids=[b["index"]["opclass"] for b in ORDERINGS])
def test_tiny_orderings_through_a_filter_and_a_rerank(pv, block):
    S = pv.sparsevec
    vals = [v for grp in block["rows"] for v in grp["values"] if v is not None]
    t = S.SparseTable(block["dim"]).append([S.SparseVector.from_text(v) for v in vals])
    every = t.filter(np.arange(len(vals)))
    for qd in block["queries"]:
        q = [S.SparseVector.from_text(qd["query"])]
        for ids, dist in (t.exact_topk(OPS[qd["op"]], q, len(vals), filter=every),
                          t.rerank(OPS[qd["op"]], q, np.arange(len(vals), dtype=np.int64)[None, :], len(vals))):
            got = [vals[i] for i, d in zip(ids[0], dist[0]) if not math.isnan(d)]
            assert got == qd["expected"]
    every.free()
    t.free()


@gpu
def test_empty_filter_and_padding(pv):
    S = pv.sparsevec
    rng = np.random.default_rng(5)
    dim, n = 2000, 400
    rows = _rows(pv, rng, dim, n)
    t = _table(pv, dim, rows)
    q = [random_sparse(rng, dim, 40) for _ in range(3)]
    with t.filter(np.empty(0, np.int64)) as f:
        assert len(f) == 0
        ids, dist = t.exact_topk(O.L2, q, 5, filter=f)
        assert np.all(ids == -1) and np.all(np.isinf(dist))
    # k above the allowed rows, duplicates collapse
    with t.filter([7, 3, 7, 399, 3]) as f:
        assert len(f) == 3
        ids, dist = t.exact_topk(O.L1, q, 6, filter=f)
        assert np.all(ids[:, 3:] == -1) and np.all(np.isinf(dist[:, 3:]))
        assert all(sorted(r.tolist()) == [3, 7, 399] for r in ids[:, :3])
        full = t.exact_topk(O.L1, q, n)
        for qi in range(3):
            by_row = dict(zip(full[0][qi].tolist(), full[1][qi].tolist()))
            assert [by_row[i] for i in ids[qi, :3]] == dist[qi, :3].tolist()
    # an empty table: every filter is empty
    e = S.SparseTable(dim)
    with e.filter([]) as f:
        ids, dist = e.exact_topk(O.COSINE, q, 2, filter=f)
        assert np.all(ids == -1) and np.all(np.isinf(dist))
    ids, dist = e.rerank(O.COSINE, q, np.full((3, 4), -1, np.int64), 2)
    assert np.all(ids == -1) and np.all(np.isinf(dist))
    e.free()
    t.free()


@gpu
@pytest.mark.parametrize("metric", [O.COSINE, O.L2])
def test_rerank_duplicates_absent_candidates_and_nan(pv, metric):
    S = pv.sparsevec
    rng = np.random.default_rng(9)
    dim, n, nq, c, k = 3000, 300, 12, 40, 25
    rows = _rows(pv, rng, dim, n, zero_every=23)       # zero-norm rows: cosine NaN
    queries = [random_sparse(rng, dim, int(rng.integers(1, 60))) for _ in range(nq)]
    queries[0] = S.SparseVector(dim)                      # zero query: every cosine distance is NaN
    t = _table(pv, dim, rows)
    full_ids, full_d = t.exact_topk(metric, queries, n)
    cand = rng.integers(-1, n, size=(nq, c)).astype(np.int64)
    cand[:, 5] = cand[:, 2]                               # a row listed twice
    cand[1, :] = -1                                       # no candidate at all
    ids, dist = t.rerank(metric, queries, cand, k)
    for qi in range(nq):
        d_of = dict(zip(full_ids[qi].tolist(), _bits(full_d[qi]).tolist()))
        dv = dict(zip(full_ids[qi].tolist(), full_d[qi].tolist()))
        valid = [(j, r) for j, r in enumerate(cand[qi].tolist()) if r >= 0]
        # ascending distance, NaN after every number, ties to the earlier candidate position
        order = sorted(valid, key=lambda jr: (math.isnan(dv[jr[1]]), 0.0 if math.isnan(dv[jr[1]]) else dv[jr[1]], jr[0]))[:k]
        want_ids = [r for _, r in order] + [-1] * (k - len(order))
        assert ids[qi].tolist() == want_ids
        assert _bits(dist[qi][:len(order)]).tolist() == [d_of[r] for _, r in order]
        assert np.all(np.isinf(dist[qi][len(order):]))
    t.free()


@gpu
def test_more_queries_than_one_launch_holds(pv):
    """nq above 65535: sub-batches, bit-identical to the unfiltered scan (which sub-batches too)"""
    S = pv.sparsevec
    rng = np.random.default_rng(13)
    dim, n, nq, k = 500, 40, 65_535 + 1234, 3
    rows = _rows(pv, rng, dim, n, hi=20)
    t = _table(pv, dim, rows)
    nnz = rng.integers(0, 6, nq)
    off = np.zeros(nq + 1, np.int64)
    off[1:] = np.cumsum(nnz)
    idx = np.concatenate([np.sort(rng.choice(dim, size=m, replace=False)) for m in nnz]).astype(np.int32)
    val = rng.standard_normal(idx.size).astype(np.float32)
    Q = S.SparseRows(dim, off, idx, val)
    want = t.exact_topk(O.L2, Q, k)
    with t.filter(np.arange(n)) as f:
        _same(t.exact_topk(O.L2, Q, k, filter=f), want)
    _same(t.rerank(O.L2, Q, np.tile(np.arange(n, dtype=np.int64), (nq, 1)), k), want)
    t.free()


@gpu
def test_filter_made_before_an_append_stays_valid(pv):
    S = pv.sparsevec
    rng = np.random.default_rng(17)
    dim = 4000
    rows = _rows(pv, rng, dim, 900)
    t = S.SparseTable(dim).append(rows[:500])
    allowed = np.sort(rng.choice(500, size=120, replace=False))
    q = [random_sparse(rng, dim, 50) for _ in range(6)]
    with t.filter(allowed) as f:
        before = t.exact_topk(O.NEG_IP, q, 10, filter=f)
        t.append(rows[500:])
        assert t.rows == 900 and len(f) == 120
        after = t.exact_topk(O.NEG_IP, q, 10, filter=f)
        _same(after, before)
        _same(after, t.rerank(O.NEG_IP, q, np.tile(allowed.astype(np.int64), (6, 1)), 10))
    t.free()


# ------------------------------------------------------------------------------- refused calls

def _raw_topk(pv, t, metric, q, k, filters, fq=None, q_dim=None):
    """the C call with sentinel-filled outputs: (rc, message, outputs untouched?)"""
    lib = pv._lib.load()
    Q = pv.sparsevec._rows(q)
    ids = np.full((Q.n, max(k, 1)), 12345, np.int64)
    dist = np.full((Q.n, max(k, 1)), 6.5, np.float64)
    farr = (C.c_void_p * len(filters))(*[f.h.value for f in filters])
    p = pv.sparsevec._p
    rc = lib.vb_sparse_exact_topk_filtered(t.h, metric, Q.dim if q_dim is None else q_dim, Q.n, p(Q.row_off), p(Q.idx), p(Q.val), k, farr,
                                           len(filters), p(fq), p(ids), p(dist))
    return rc, lib.vb_last_error().decode(), bool(np.all(ids == 12345) and np.all(dist == 6.5))


def _raw_rerank(pv, t, metric, q, cand, k, q_dim=None):
    lib = pv._lib.load()
    Q = pv.sparsevec._rows(q)
    ids = np.full((Q.n, max(k, 1)), 12345, np.int64)
    dist = np.full((Q.n, max(k, 1)), 6.5, np.float64)
    p = pv.sparsevec._p
    cand = np.ascontiguousarray(cand, np.int64)
    rc = lib.vb_sparse_table_rerank(t.h, metric, Q.dim if q_dim is None else q_dim, Q.n, p(Q.row_off), p(Q.idx), p(Q.val), p(cand),
                                    cand.shape[1], k, p(ids), p(dist))
    return rc, lib.vb_last_error().decode(), bool(np.all(ids == 12345) and np.all(dist == 6.5))


@gpu
def test_sparse_and_dense_filters_do_not_mix(pv):
    S = pv.sparsevec
    rng = np.random.default_rng(21)
    dim = 64
    t = _table(pv, dim, _rows(pv, rng, dim, 50, hi=10))
    sf = t.filter(np.arange(10))
    # a sparse filter on the dense calls
    dense = pv.Table(O.VECTOR, 4).append(np.ones((50, 4), np.float32))
    with pytest.raises(pv.VecB200Error, match="made for another table or index") as e:
        dense.exact_topk(O.L2, np.zeros((1, 4), np.float32), 1, filter=sf)
    assert e.value.code == EINVAL
    ix = pv.IvfflatIndex("vector_l2_ops", 4, 2).load(np.zeros((2, 4), np.float32), np.array([0, 25, 50], np.int64),
                                                     np.ones((50, 4), np.float32), np.arange(50, dtype=np.int64))
    with pytest.raises(pv.VecB200Error, match="made for another table or index") as e:
        ix.search(np.zeros((1, 4), np.float32), k=1, probes=1, filter=sf)
    assert e.value.code == EINVAL
    gi = pv.HnswIndex("vector_l2_ops", 3)
    gi.load(np.array([[1, 2, 3]], np.float32), np.zeros(1, np.int32), np.full((1, 32), -1, np.int32), np.full(1, -1, np.int64),
            np.zeros((0, 16), np.int32), 0)
    with pytest.raises(pv.VecB200Error, match="made for another table or index") as e:
        gi.iterative_scan(np.zeros((1, 3), np.float32), filter=sf)
    assert e.value.code == EINVAL
    # a dense filter on the sparse calls
    q = [random_sparse(rng, dim, 5)]
    with dense.filter(np.arange(5)) as df:
        rc, msg, untouched = _raw_topk(pv, t, O.L2, q, 1, [df])
        assert rc == EINVAL and "made for another table or index" in msg and untouched
    # another sparse table's filter, and a filter that outlived its table (a new table may take its address)
    t2 = _table(pv, dim, _rows(pv, rng, dim, 50, hi=10))
    rc, msg, untouched = _raw_topk(pv, t2, O.L2, q, 1, [sf])
    assert rc == EINVAL and "made for another table or index" in msg and untouched
    t.free()
    t3 = _table(pv, dim, _rows(pv, rng, dim, 50, hi=10))
    rc, msg, untouched = _raw_topk(pv, t3, O.L2, q, 1, [sf])
    assert rc == EINVAL and "made for another table or index" in msg and untouched
    sf.free()
    for x in (t2, t3):
        x.free()


@gpu
def test_argument_errors_name_the_value_and_write_nothing(pv):
    S = pv.sparsevec
    rng = np.random.default_rng(23)
    dim, n = 5, 30
    t = _table(pv, dim, _rows(pv, rng, dim, n, hi=4))
    q = [S.SparseVector(dim, [0, 3], [1.0, -2.0]) for _ in range(3)]
    with pytest.raises(pv.VecB200Error) as e:
        t.filter([0, 30])
    assert e.value.code == EINVAL and "rows[1] = 30 is not a row of the table (0..29)" in str(e.value)
    with pytest.raises(pv.VecB200Error) as e:
        t.filter([-1])
    assert e.value.code == EINVAL and "rows[0] = -1" in str(e.value)
    f0, f1 = t.filter([1, 2]), t.filter([3])
    rc, msg, untouched = _raw_topk(pv, t, O.L2, q, 2, [f0, f1], np.array([0, 1, 2], np.int32))
    assert rc == EINVAL and "filter_of_query[2] = 2, not in 0..1" in msg and untouched
    rc, msg, untouched = _raw_topk(pv, t, O.L2, q, 2, [f0, f1], None)
    assert rc == EINVAL and "filter_of_query may only be NULL with one filter" in msg and untouched
    rc, msg, untouched = _raw_rerank(pv, t, O.L2, q, np.array([[0, 1], [2, -1], [4, 30]]), 2)
    assert rc == EINVAL and "candidate 1 of query 2 is 30, not a row of the table (-1 or 0..29)" in msg and untouched
    rc, msg, untouched = _raw_rerank(pv, t, O.L2, q, np.array([[0, 1], [-2, 1], [4, 3]]), 2)
    assert rc == EINVAL and "candidate 0 of query 1 is -2" in msg and untouched
    for k in (0, 2049):
        rc, msg, untouched = _raw_topk(pv, t, O.L2, q, k, [f0])
        assert rc == EINVAL and msg == "k must be in 1..2048" and untouched
        rc, msg, untouched = _raw_rerank(pv, t, O.L2, q, np.zeros((3, 2)), k)
        assert rc == EINVAL and msg == "k must be in 1..2048" and untouched
    rc, msg, untouched = _raw_topk(pv, t, O.IP, q, 1, [f0])
    assert rc == EINVAL and untouched
    rc, msg, untouched = _raw_rerank(pv, t, O.IP, q, np.zeros((3, 2)), 1)
    assert rc == EINVAL and untouched
    # CheckDims' text (src/sparsevec.c:44-51), the row's dimension first
    rc, msg, untouched = _raw_topk(pv, t, O.L2, q, 1, [f0], q_dim=4)
    assert rc == EINVAL and msg == "different sparsevec dimensions 5 and 4" and untouched
    rc, msg, untouched = _raw_rerank(pv, t, O.L2, q, np.zeros((3, 2)), 1, q_dim=4)
    assert rc == EINVAL and msg == "different sparsevec dimensions 5 and 4" and untouched
    with pytest.raises(ValueError, match="different sparsevec dimensions 5 and 4"):
        t.exact_topk(O.L2, [S.SparseVector(4, [0], [1.0])], 1, filter=f0)
    with pytest.raises(ValueError, match="different sparsevec dimensions 5 and 4"):
        t.rerank(O.L2, [S.SparseVector(4, [0], [1.0])], np.zeros((1, 1), np.int64), 1)
    # and the library keeps working
    ids, _ = t.exact_topk(O.L2, q, 2, filter=[f0, f1], filter_of_query=[0, 1, 0])
    assert sorted(ids[0].tolist()) == [1, 2] and ids[1].tolist() == [3, -1]
    f0.free()
    f1.free()
    t.free()
