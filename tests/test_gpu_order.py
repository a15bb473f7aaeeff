"""The btree order on the GPU (vb_order): btree.out's orderings and equality lookups for vector, halfvec and sparsevec;
perm, group_of_row, group_start, groups and bounds equal to the CPU oracle's for tables of 0 .. 200 000 rows and for
adversarial data (all rows equal, repeated values, -0 / +0, +-inf, deep shared prefixes, the one-hot staircase, halfvec
subnormals, sparse rows with nnz 0 / stored zeros / 16 000 entries) with the pass bounds; NaN rows; appends and table
growth; refusals; the _dev variants and their CUDA graph replay; GROUP BY v through Table.avg."""
import json
import os

import numpy as np
import pytest

from tests import order_oracle as OO

pytestmark = pytest.mark.gpu
EINVAL = -1
HERE = os.path.dirname(os.path.abspath(__file__))
KAT = json.load(open(os.path.join(HERE, "golden", "btree_kat.json")))


@pytest.fixture(scope="module")
def pv():
    import pgvector_b200 as pv
    pv.init(0)
    return pv


def dense_table(pv, half, rows):
    t = pv.Table(pv.HALFVEC if half else pv.VECTOR, rows.shape[1])
    if rows.shape[0]:
        t.append(rows)
    return t


def sparse_table(pv, rows):
    t = pv.SparseTable(rows.dim)
    if rows.n:
        t.append(rows)
    return t


def check_against_oracle(o, kind, rows, queries, passes_max=None):
    perm, gor, gst = o.read()
    wp, wg, ws = OO.order(kind, rows)
    np.testing.assert_array_equal(perm, wp)
    np.testing.assert_array_equal(gor, wg)
    np.testing.assert_array_equal(gst, ws)
    assert o.groups == len(ws) - 1 and o.rows == len(wp)
    lo, hi = o.bounds(queries)
    wlo, whi = OO.bounds(kind, rows, queries)
    np.testing.assert_array_equal(lo, wlo)
    np.testing.assert_array_equal(hi, whi)
    if passes_max is not None:
        assert o.passes <= passes_max


def dense_queries(rng, rows, m=64):
    """half present in the table, half perturbed copies"""
    if rows.shape[0] == 0:
        return np.zeros((4, rows.shape[1]), rows.dtype)
    pick = rows[rng.integers(0, rows.shape[0], m)].copy()
    pick[m // 2:, -1] = pick[m // 2:, -1] + 1
    return pick


def sparse_queries(rng, rows, m=32):
    from pgvector_b200.sparsevec import SparseRows
    if rows.n == 0:
        return SparseRows(rows.dim, [0, 0], [], [])
    return SparseRows.from_vectors([rows.row(int(r)) for r in rng.integers(0, rows.n, m)], rows.dim)


def random_sparse(rng, n, dim, nnz, vals=None):
    from pgvector_b200.sparsevec import SparseRows
    counts = rng.integers(0, nnz + 1, n)
    off = np.zeros(n + 1, np.int64)
    off[1:] = np.cumsum(counts)
    idx = np.concatenate([np.sort(rng.choice(dim, c, replace=False)) for c in counts]) if n else np.empty(0)
    val = rng.choice(vals, off[-1]) if vals is not None else rng.standard_normal(off[-1])
    return SparseRows(dim, off, idx.astype(np.int32), val.astype(np.float32))


# ------------------------------------------------------------------ btree.out

@pytest.mark.parametrize("case", KAT["btree"], ids=lambda c: c["type"])
def test_btree_out(pv, case):
    from pgvector_b200.sparsevec import SparseRows, SparseVector
    texts = [t for t in case["rows"] if t is not None]
    want = [t for t in case["order"] if t is not None]
    if case["type"] == "sparsevec":
        t = sparse_table(pv, SparseRows.from_vectors([SparseVector.from_text(x) for x in texts], case["dim"]))
        q = SparseRows.from_vectors([SparseVector.from_text(case["eq"]["query"])], case["dim"])
    else:
        rows = np.array([json.loads(x) for x in texts], np.float32)
        t = dense_table(pv, case["type"] == "halfvec", rows.astype(np.float16) if case["type"] == "halfvec" else rows)
        q = np.array([json.loads(case["eq"]["query"])], np.float32)
        q = q.astype(np.float16) if case["type"] == "halfvec" else q
    with t.order() as o:
        perm = o.perm
        assert [texts[i] for i in perm] == want
        lo, hi = o.bounds(q)
        assert [texts[i] for i in perm[lo[0]:hi[0]]] == case["eq"]["rows"]


# ------------------------------------------------------------------ parity with the oracle

@pytest.mark.parametrize("n", [0, 1, 1000, 200000])
@pytest.mark.parametrize("half,dim", [(False, 1), (False, 3), (False, 64), (True, 3), (True, 64)])
def test_dense_parity(pv, n, half, dim):
    rng = np.random.default_rng(n + dim)
    levels = 3 if dim <= 3 else 2   # few levels: many ties and long shared prefixes at every size
    rows = rng.integers(-levels, levels + 1, (n, dim)).astype(np.float16 if half else np.float32)
    t = dense_table(pv, half, rows)
    with t.order() as o:
        check_against_oracle(o, OO.HALFVEC if half else OO.VECTOR, rows, dense_queries(rng, rows),
                             passes_max=(dim if not half else (dim + 1) // 2) + 1)


@pytest.mark.parametrize("n", [0, 1, 1000, 200000])
@pytest.mark.parametrize("dim,nnz", [(5, 3), (1000, 20)])
def test_sparse_parity(pv, n, dim, nnz):
    rng = np.random.default_rng(7 * n + dim)
    rows = random_sparse(rng, n, dim, nnz, vals=np.array([-1.0, 0.5, 1.0], np.float32))
    t = sparse_table(pv, rows)
    with t.order() as o:
        check_against_oracle(o, OO.SPARSE, rows, sparse_queries(rng, rows), passes_max=nnz + 2)


# ------------------------------------------------------------------ adversarial data

@pytest.mark.parametrize("half", [False, True])
def test_all_rows_equal_take_two_passes(pv, half):
    rows = np.tile(np.linspace(-1, 1, 300, dtype=np.float32), (5000, 1)).astype(np.float16 if half else np.float32)
    with dense_table(pv, half, rows).order() as o:
        check_against_oracle(o, OO.HALFVEC if half else OO.VECTOR, rows, rows[:2], passes_max=2)
        assert o.groups == 1


def test_sparse_all_rows_equal_take_two_passes(pv):
    from pgvector_b200.sparsevec import SparseRows, SparseVector
    v = SparseVector(100, np.arange(0, 100, 3), np.linspace(-1, 1, 34))
    rows = SparseRows.from_vectors([v] * 3000, 100)
    with sparse_table(pv, rows).order() as o:
        check_against_oracle(o, OO.SPARSE, rows, SparseRows.from_vectors([v], 100), passes_max=2)
        assert o.groups == 1


@pytest.mark.parametrize("half", [False, True])
def test_values_repeated_k_times_shuffled(pv, half):
    rng = np.random.default_rng(3)
    base = rng.standard_normal((2000, 96)).astype(np.float32)
    rows = np.repeat(base, 8, axis=0)[rng.permutation(16000)].astype(np.float16 if half else np.float32)
    with dense_table(pv, half, rows).order() as o:
        check_against_oracle(o, OO.HALFVEC if half else OO.VECTOR, rows, dense_queries(rng, rows))
        assert o.groups == len(np.unique(rows.view(np.uint16 if half else np.uint32), axis=0))


@pytest.mark.parametrize("half", [False, True])
def test_signed_zeros_and_infinities(pv, half):
    rng = np.random.default_rng(4)
    vals = np.array([-0.0, 0.0, np.inf, -np.inf, 1.0], np.float32)
    rows = rng.choice(vals, (3000, 4)).astype(np.float16 if half else np.float32)
    with dense_table(pv, half, rows).order() as o:
        check_against_oracle(o, OO.HALFVEC if half else OO.VECTOR, rows, rows[:50])
        gor = o.group_of_row
    z = np.where(rows == 0, 0, rows).astype(np.float32)   # -0 and +0 in one group
    _, inv = np.unique(z.view(np.uint32), axis=0, return_inverse=True)
    pairs = set(zip(inv.reshape(-1).tolist(), gor.tolist()))
    assert len(pairs) == len(set(inv.reshape(-1).tolist())) == gor.max() + 1


@pytest.mark.parametrize("half", [False, True])
def test_rows_sharing_all_but_the_last_element(pv, half):
    rng = np.random.default_rng(5)
    dim = 257
    rows = np.tile(rng.standard_normal(dim).astype(np.float32), (4000, 1))
    rows[:, -1] = rng.integers(0, 50, 4000)
    rows = rows.astype(np.float16 if half else np.float32)
    with dense_table(pv, half, rows).order() as o:
        check_against_oracle(o, OO.HALFVEC if half else OO.VECTOR, rows, dense_queries(rng, rows), passes_max=2)


@pytest.mark.parametrize("half", [False, True])
def test_one_hot_staircase(pv, half):
    dim = 200
    rows = np.vstack([np.eye(dim), np.eye(dim)[::-1]]).astype(np.float16 if half else np.float32)
    with dense_table(pv, half, rows).order() as o:
        check_against_oracle(o, OO.HALFVEC if half else OO.VECTOR, rows, rows[::7],
                             passes_max=(dim if not half else (dim + 1) // 2) + 1)
        assert o.passes > 3


def test_halfvec_subnormals(pv):
    rng = np.random.default_rng(6)
    sub = np.arange(0, 1024, dtype=np.uint16)
    bits = rng.choice(np.concatenate([sub, sub | 0x8000]), (5000, 9)).astype(np.uint16)
    rows = bits.view(np.float16)
    with dense_table(pv, True, rows).order() as o:
        check_against_oracle(o, OO.HALFVEC, rows, rows[:40])


def test_sparse_adversarial_rows(pv):
    """nnz 0, stored zeros of both signs, a negative entry at a smaller index than a positive one, 16 000 entries"""
    from pgvector_b200.sparsevec import SparseRows
    rng = np.random.default_rng(8)
    dim = 40000
    vecs = []
    for _ in range(300):
        k = rng.integers(0, 4)
        idx = np.sort(rng.choice(6, k, replace=False))
        vecs.append((idx, rng.choice(np.array([-1.0, -0.0, 0.0, 1.0], np.float32), k)))
    big = np.sort(rng.choice(dim, 16000, replace=False))
    vecs += [(big, np.ones(16000, np.float32)), (big, np.ones(16000, np.float32)),
             (big, np.concatenate([np.ones(15999, np.float32), [2.0]]))]
    vecs += [(np.array([0]), np.array([-1.0])), (np.array([1]), np.array([1.0])), (np.array([], np.int64), np.array([]))]
    off = np.zeros(len(vecs) + 1, np.int64)
    off[1:] = np.cumsum([len(i) for i, _ in vecs])
    rows = SparseRows(dim, off, np.concatenate([i for i, _ in vecs]).astype(np.int32), np.concatenate([v for _, v in vecs]).astype(np.float32))
    with sparse_table(pv, rows).order() as o:
        check_against_oracle(o, OO.SPARSE, rows, SparseRows(dim, off[:9] - off[0], rows.idx[:off[8]], rows.val[:off[8]]),
                             passes_max=16000 + 2)


# ------------------------------------------------------------------ NaN, lifetime, refusals

@pytest.mark.parametrize("half", [False, True])
def test_nan_rows_give_a_permutation(pv, half):
    rng = np.random.default_rng(9)
    rows = rng.integers(-2, 3, (5000, 8)).astype(np.float32)
    rows[rng.random((5000, 8)) < 0.05] = np.nan
    rows = rows.astype(np.float16 if half else np.float32)
    with dense_table(pv, half, rows).order() as o:
        perm = o.perm
        np.testing.assert_array_equal(np.sort(perm), np.arange(5000))
        lo, hi = o.bounds(rows[:10])
        assert (lo <= hi).all() and (hi <= 5000).all()


def test_appends_after_creation_and_growth(pv):
    rng = np.random.default_rng(10)
    rows = rng.integers(-2, 3, (1000, 16)).astype(np.float32)
    t = dense_table(pv, False, rows)
    o = t.order()
    t.append(rng.integers(-2, 3, (300000, 16)).astype(np.float32))   # grows (and moves) the table's buffer
    assert o.rows == 1000 and len(t) == 301000
    check_against_oracle(o, OO.VECTOR, rows, dense_queries(rng, rows))
    np.testing.assert_array_equal(np.sort(o.perm), np.arange(1000))
    o.free()
    srows = random_sparse(rng, 500, 50, 5)
    st = sparse_table(pv, srows)
    so = st.order()
    st.append(random_sparse(rng, 200000, 50, 5))
    check_against_oracle(so, OO.SPARSE, srows, sparse_queries(rng, srows))
    so.free()


def test_refusals_leave_outputs_untouched(pv):
    import ctypes as C
    from pgvector_b200 import _lib
    from pgvector_b200.sparsevec import SparseRows
    lib = _lib.load()
    bt = pv.Table(pv.BIT, 64)
    bt.append(np.zeros((4, 8), np.uint8))
    with pytest.raises(pv.VecB200Error, match="bit_ops") as e:
        bt.order()
    assert e.value.code == EINVAL
    rows = np.arange(12, dtype=np.float32).reshape(4, 3)
    t = dense_table(pv, False, rows)
    srows = SparseRows(3, [0, 1, 2], [0, 1], [1.0, 2.0])
    st = sparse_table(pv, srows)
    o, so = t.order(), st.order()
    lo = np.full(1, -7, np.int64)
    hi = np.full(1, -7, np.int64)
    # dense order given to the sparse call and the reverse
    rc = lib.vb_sparse_order_bounds(o.h, 3, 1, srows.row_off.ctypes.data_as(C.c_void_p), srows.idx.ctypes.data_as(C.c_void_p),
                                    srows.val.ctypes.data_as(C.c_void_p), lo.ctypes.data_as(C.c_void_p), hi.ctypes.data_as(C.c_void_p))
    assert rc == EINVAL and (lo == -7).all() and (hi == -7).all()
    q = rows[:1].copy()
    rc = lib.vb_order_bounds(so.h, q.ctypes.data_as(C.c_void_p), 1, lo.ctypes.data_as(C.c_void_p), hi.ctypes.data_as(C.c_void_p))
    assert rc == EINVAL and (lo == -7).all() and (hi == -7).all()
    # q_dim mismatch: CheckDims' text
    with pytest.raises(ValueError, match="different sparsevec dimensions 3 and 4"):
        so.bounds(SparseRows(4, [0, 1], [0], [1.0]))
    # freed tables
    t.free()
    st.free()
    rc = lib.vb_order_bounds(o.h, q.ctypes.data_as(C.c_void_p), 1, lo.ctypes.data_as(C.c_void_p), hi.ctypes.data_as(C.c_void_p))
    assert rc == EINVAL and "freed" in lib.vb_last_error().decode() and (lo == -7).all() and (hi == -7).all()
    rc = lib.vb_sparse_order_bounds(so.h, 3, 1, srows.row_off.ctypes.data_as(C.c_void_p), srows.idx.ctypes.data_as(C.c_void_p),
                                    srows.val.ctypes.data_as(C.c_void_p), lo.ctypes.data_as(C.c_void_p), hi.ctypes.data_as(C.c_void_p))
    assert rc == EINVAL and (lo == -7).all() and (hi == -7).all()
    np.testing.assert_array_equal(np.sort(o.perm), np.arange(4))   # reads need only the order
    o.free()
    so.free()


# ------------------------------------------------------------------ _dev variants, graph capture, GROUP BY

@pytest.mark.parametrize("half", [False, True])
def test_dev_variants_equal_host_and_replay_in_a_graph(pv, half):
    import torch
    rng = np.random.default_rng(11)
    rows = rng.integers(-2, 3, (20000, 24)).astype(np.float16 if half else np.float32)
    t = dense_table(pv, half, rows)
    with t.order() as o:
        perm, gor, gst = o.read()
        dp, dg, ds = o.read(device=True)
        np.testing.assert_array_equal(dp.cpu().numpy(), perm)
        np.testing.assert_array_equal(dg.cpu().numpy(), gor)
        np.testing.assert_array_equal(ds.cpu().numpy(), gst)
        q = dense_queries(rng, rows, 256)
        lo, hi = o.bounds(q)
        qd = torch.from_numpy(q).cuda()
        dlo, dhi = o.bounds(qd)
        np.testing.assert_array_equal(dlo.cpu().numpy(), lo)
        np.testing.assert_array_equal(dhi.cpu().numpy(), hi)
        # capture the read-free _dev calls on the library stream and replay them
        from pgvector_b200 import _lib
        import ctypes as C
        lib = _lib.load()
        s = torch.cuda.ExternalStream(pv.stream_handle())
        glo = torch.full_like(dlo, -1)
        ghi = torch.full_like(dhi, -1)
        gp = torch.full_like(dp, -1)
        torch.cuda.synchronize()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, stream=s):
            assert lib.vb_order_bounds_dev(o.h, C.c_void_p(qd.data_ptr()), qd.shape[0], C.c_void_p(glo.data_ptr()),
                                           C.c_void_p(ghi.data_ptr())) == 0
            assert lib.vb_order_read_dev(o.h, C.c_void_p(gp.data_ptr()), None, None) == 0
        g.replay()
        torch.cuda.synchronize()
        np.testing.assert_array_equal(glo.cpu().numpy(), lo)
        np.testing.assert_array_equal(ghi.cpu().numpy(), hi)
        np.testing.assert_array_equal(gp.cpu().numpy(), perm)


def test_sparse_dev_bounds_equal_host(pv):
    import torch
    rng = np.random.default_rng(12)
    rows = random_sparse(rng, 20000, 300, 6, vals=np.array([-1.0, 1.0, 2.0], np.float32))
    with sparse_table(pv, rows).order() as o:
        q = sparse_queries(rng, rows, 128)
        lo, hi = o.bounds(q)
        dq = (torch.from_numpy(q.row_off).cuda(), torch.from_numpy(q.idx).cuda(), torch.from_numpy(q.val).cuda())
        dlo, dhi = o.bounds(dq)
        np.testing.assert_array_equal(dlo.cpu().numpy(), lo)
        np.testing.assert_array_equal(dhi.cpu().numpy(), hi)


@pytest.mark.parametrize("half", [False, True])
def test_group_by_v_through_avg(pv, half):
    rng = np.random.default_rng(13)
    base = rng.standard_normal((500, 32)).astype(np.float32)
    rows = base[rng.integers(0, 500, 8000)].astype(np.float16 if half else np.float32)
    t = dense_table(pv, half, rows)
    with t.order() as o:
        perm, gor, gst = o.read()
        vals, counts = t.avg(groups=o.group_of_row, ngroups=o.groups)
    np.testing.assert_array_equal(counts, np.diff(gst))
    first = rows[perm[gst[:-1]]]
    np.testing.assert_array_equal(vals.view(np.uint16 if half else np.uint32), first.view(np.uint16 if half else np.uint32))
