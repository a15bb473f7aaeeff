"""The batched IVFFlat search with row filters (vb_ivf_search_filtered / _dev, IvfflatIndex.search(filter=...)):
WHERE <predicate> ORDER BY v <op> q LIMIT k with ivfflat.iterative_scan = off, for a batch of queries.

1. against the oracle: GetScanLists + GetScanItems over the probes, restricted to the allowed ids, first k;
2. a filter of every row: bit-identical to vb_ivf_search for every scan_impl, level 0 on and off, batched or not;
3. against the filtered handle's first page (scan_impl 0), and the unfiltered search's distance of every row (scan_impl 3);
4. per-query filters: equal to one call per filter, filters freed after the call, host = device;
5. the level-0 / level-1 fallbacks with filters;
6. padding, allowed rows at +inf and NaN, rejected rows never returned;
7. argument, ownership and staleness errors, the host output untouched;
8. the data and predicates of the reference's test/t/009_ivfflat_filtering.pl."""
import ctypes as C
import os

import numpy as np
import pytest

import oracle as O
from tests.ivf_iter_oracle import iter_scan
from tests.test_gpu_ivf_iterative import LISTS, OPCLASSES, data_for, make_index
from tests.util import mixture

pytestmark = pytest.mark.gpu
RTOL = 1e-5
SCAN_IMPL = int(os.environ.get("VB_TEST_SCAN_IMPL", "2"))


@pytest.fixture(scope="module")
def pv():
    import pgvector_b200 as pv
    pv.init(0)
    pv.set_option("scan_impl", 2)
    O.ivf_set_tie_mode(True)
    yield pv
    O.ivf_set_tie_mode(False)
    pv.set_option("scan_impl", SCAN_IMPL)


def bits_equal(a, b):
    a, b = np.asarray(a), np.asarray(b)
    return a.shape == b.shape and np.array_equal(a.view(np.uint8), b.view(np.uint8))


def dim_of(opclass):
    return 64 if opclass.startswith("bit") else 24


@pytest.fixture(scope="module")
def indexes(pv):
    out = {}
    for i, opclass in enumerate(OPCLASSES):
        dim = dim_of(opclass)
        rows, centers, _ = data_for(opclass, 3000, dim, LISTS, seed=70 + i)
        queries = data_for(opclass, 400, dim, LISTS, seed=170 + i)[0][:80]
        gix, oix = make_index(pv, opclass, rows, centers, dim)
        out[opclass] = (gix, oix, queries)
    yield out
    for gix, _, _ in out.values():
        gix.free()


def allowed_of(rng, ids, sel):
    ids = np.asarray(ids)
    if sel == 0:
        return np.zeros(0, np.int64)
    if sel == 1:
        return np.sort(ids).astype(np.int64)
    return np.sort(rng.choice(ids, max(1, int(len(ids) * sel)), replace=False)).astype(np.int64)


def sequences(oix, queries, probes):
    """per query, the full sorted sequence of its probed lists (GetScanLists + GetScanItems)"""
    return [iter_scan(oix, q, probes, probes)[0] for q in queries]


def expect(seq, allowed, k):
    ids, dist = seq
    keep = np.isin(ids, allowed)
    return ids[keep][:k], dist[keep][:k], dict(zip(ids[keep].tolist(), dist[keep].tolist()))


def assert_matches(gi, gd, want):
    """ids equal up to near-ties, distances within RTOL, -1 / +inf padding after the expected rows"""
    wi, wd, d_of = want
    n = len(wi)
    assert np.all(gi[n:] == -1) and np.all(np.isposinf(gd[n:])), (gi[n:], gd[n:])
    gi, gd = gi[:n], gd[:n]
    assert np.all(gi >= 0)
    # (absolute near 0: inner products cancel, so the fp32 sums' error scales with the largest distances of the run)
    fin = np.isfinite(wd)
    atol = RTOL * max(1.0, float(np.abs(wd[fin]).max())) if fin.any() else 0.0
    assert np.allclose(gd, wd, rtol=RTOL, atol=atol, equal_nan=True)
    for j in np.nonzero(gi != wi)[0]:
        assert int(gi[j]) in d_of, (j, gi[j])
        assert abs(d_of[int(gi[j])] - wd[j]) <= RTOL * abs(wd[j]) + atol, (j, gi[j], wi[j])


# ---------------------------------------------------------------------------------------------- 1. oracle parity


@pytest.mark.parametrize("opclass", OPCLASSES)
def test_filtered_search_is_the_oracle_restricted(pv, indexes, opclass):
    gix, oix, queries = indexes[opclass]
    rng = np.random.default_rng(5)
    for probes in (1, 3, 7):
        seqs = sequences(oix, queries, probes)
        for sel in (1, 0.5, 0.1, 0.01, 0):
            allowed = allowed_of(rng, oix.ids, sel)
            with gix.filter(allowed) as f:
                for k in (1, 10, 100, 2500):
                    gi, gd = gix.search(queries, k=k, probes=probes, filter=f)
                    for q in range(len(queries)):
                        assert_matches(gi[q], gd[q], expect(seqs[q], allowed, k))


# ---------------------------------------------------------------------------------------------- 2. a filter of every row


@pytest.mark.parametrize("opclass", OPCLASSES)
def test_full_filter_is_bit_identical_to_search(pv, indexes, opclass):
    gix, oix, _ = indexes[opclass]
    dim = dim_of(opclass)
    queries = data_for(opclass, 400, dim, LISTS, seed=11)[0]
    try:
        with gix.filter(np.asarray(oix.ids)) as f:
            for scan_impl in (0, 2, 3, 4):
                pv.set_option("scan_impl", scan_impl)
                for level0 in (0, 1):
                    pv.set_option("tc_level0", level0)
                    for nq in (300, 40, 12):   # 300 x 3 probes takes the batched kernels, 40 x 3 does not, 12 <= 16
                        q = queries[:nq]
                        pv.set_option("one_query", 0)
                        wi, wd = gix.search(q, k=10, probes=3)
                        pv.set_option("one_query", 1)
                        gi, gd = gix.search(q, k=10, probes=3, filter=f)
                        assert np.array_equal(gi, wi) and bits_equal(gd, wd), (scan_impl, level0, nq)
    finally:
        pv.set_option("scan_impl", 2)
        pv.set_option("tc_level0", 1)
        pv.set_option("one_query", 1)


# ---------------------------------------------------------------------------------------------- 3. against the handle


@pytest.mark.parametrize("opclass", OPCLASSES)
def test_equals_the_filtered_handle_first_page(pv, indexes, opclass):
    gix, oix, queries = indexes[opclass]
    rng = np.random.default_rng(8)
    try:
        for sel in (0.5, 0.1):
            allowed = allowed_of(rng, oix.ids, sel)
            with gix.filter(allowed) as f:
                pv.set_option("scan_impl", 0)
                for probes, k in ((3, 10), (7, 100)):
                    gi, gd = gix.search(queries, k=k, probes=probes, filter=f)
                    with gix.iterative_scan(queries, probes=probes, max_probes=probes, page=k, filter=f) as s:
                        hi, hd, _ = s.next_batch()
                    assert np.array_equal(gi, hi) and bits_equal(gd, hd)
                pv.set_option("scan_impl", 3)
                gi, gd = gix.search(queries, k=10, probes=7, filter=f)
                ui, ud = gix.search(queries, k=2500, probes=7)
                for q in range(len(queries)):
                    d_of = dict(zip(ui[q].tolist(), ud[q].tolist()))
                    for i, d in zip(gi[q].tolist(), gd[q].tolist()):
                        if i >= 0:
                            assert i in set(allowed.tolist())
                            assert np.float64(d).tobytes() == np.float64(d_of[i]).tobytes()
    finally:
        pv.set_option("scan_impl", 2)


# ---------------------------------------------------------------------------------------------- 4. per-query filters


@pytest.mark.parametrize("nfilters", [4, 64])
def test_per_query_filters_equal_one_call_per_filter(pv, indexes, nfilters):
    import torch
    from pgvector_b200 import _lib
    gix, oix, _ = indexes["vector_l2_ops"]
    queries = data_for("vector_l2_ops", 400, 24, LISTS, seed=23)[0][:256]
    rng = np.random.default_rng(nfilters)
    allowed = [allowed_of(rng, oix.ids, s) for s in rng.choice([0.5, 0.1, 0.02, 0.0], nfilters)]
    fq = rng.integers(0, nfilters, len(queries)).astype(np.int32)
    filters = [gix.filter(a) for a in allowed]
    try:
        for scan_impl in (0, 3):
            pv.set_option("scan_impl", scan_impl)
            gi, gd = gix.search(queries, k=20, probes=5, filter=filters, filter_of_query=fq)
            for i, f in enumerate(filters):
                wi, wd = gix.search(queries, k=20, probes=5, filter=f)
                sel = fq == i
                assert np.array_equal(gi[sel], wi[sel]) and bits_equal(gd[sel], wd[sel])
            # device queries and outputs, with one filter freed right after the call returns
            extra = gix.filter(allowed[0])
            fl = filters[1:] + [extra]
            fq_dev = np.where(fq == 0, nfilters - 1, fq - 1).astype(np.int32)
            arr = (C.c_void_p * nfilters)(*[f.h.value for f in fl])
            tq = torch.from_numpy(queries).cuda()
            ids = torch.empty((len(queries), 20), dtype=torch.int64, device="cuda")
            dist = torch.empty((len(queries), 20), dtype=torch.float32, device="cuda")
            torch.cuda.synchronize()
            _lib.check(_lib.load().vb_ivf_search_filtered_dev(gix.h, tq.data_ptr(), len(queries), 5, 20, arr, nfilters,
                                                              fq_dev.ctypes.data_as(C.c_void_p), ids.data_ptr(), dist.data_ptr()))
            extra.free()
            pv.synchronize()
            assert np.array_equal(ids.cpu().numpy(), gi) and bits_equal(dist.cpu().numpy(), gd.astype(np.float32))
    finally:
        pv.set_option("scan_impl", 2)
        for f in filters:
            f.free()


# ---------------------------------------------------------------------------------------------- 5. fallbacks


@pytest.mark.parametrize("latent", [0, 8])
def test_level_fallbacks_keep_filtered_results(pv, latent):
    from tests.test_gpu_ivfflat import make_index as make_l2_index
    rng = np.random.default_rng(41)
    if latent:
        frame = np.linalg.qr(rng.standard_normal((64, latent)))[0].astype(np.float32)
        x = (rng.standard_normal((20000, latent)).astype(np.float32) @ frame.T + 0.01 * rng.standard_normal((20000, 64))).astype(np.float32)
        q = (rng.standard_normal((400, latent)).astype(np.float32) @ frame.T + 0.01 * rng.standard_normal((400, 64))).astype(np.float32)
        c = x[rng.choice(20000, 40, replace=False)].copy()
    else:
        x, c = mixture(20000, 64, 40, seed=42)
        q, _ = mixture(400, 64, 40, seed=43)
    gix, oix = make_l2_index(pv, "vector_l2_ops", x, c)
    seqs = sequences(oix, q, 6)
    try:
        pv.set_option("scan_impl", 4)
        l0, l1 = gix.tc_level0_fallbacks(), gix.tc_level1_fallbacks()
        for sel in (1, 0.5, 0.1):
            allowed = allowed_of(rng, oix.ids, sel)
            with gix.filter(allowed) as f:
                gi, gd = gix.search(q, k=10, probes=6, filter=f)
                for i in range(len(q)):
                    assert_matches(gi[i], gd[i], expect(seqs[i], allowed, 10))
        grew = (gix.tc_level0_fallbacks() - l0, gix.tc_level1_fallbacks() - l1)
        print("level-0 / level-1 fallbacks", grew)
        assert sum(grew) > 0
    finally:
        pv.set_option("scan_impl", 2)
        gix.free()


# ---------------------------------------------------------------------------------------------- 6. padding, +inf and NaN


def test_padding_infinite_and_nan_rows(pv):
    rng = np.random.default_rng(3)
    dim, lists = 8, 4
    centers = rng.standard_normal((lists, dim)).astype(np.float32)
    rows = rng.standard_normal((400, dim)).astype(np.float32)
    rows[[10, 20, 30]] = 3e38                      # L2 to any query overflows to +inf
    off = np.array([0, 100, 200, 300, 400], dtype=np.int64)
    ids = np.arange(400, dtype=np.int64)
    q = rng.standard_normal((6, dim)).astype(np.float32)
    gix = pv.IvfflatIndex("vector_l2_ops", dim, lists).load(centers, off, rows, ids)
    oix = O.Ivf(O.VECTOR, pv.OPCLASSES["vector_l2_ops"][1], centers, off, rows, ids, dim=dim)
    seqs = sequences(oix, q, 2)
    for allowed in (np.array([10, 20, 55, 150, 250, 399]), np.array([10, 30]), np.arange(0, 400, 3)):
        with gix.filter(allowed) as f:
            gi, gd = gix.search(q, k=50, probes=2, filter=f)
        for i in range(len(q)):
            want = expect(seqs[i], allowed, 50)
            assert_matches(gi[i], gd[i], want)
            assert set(gi[i][gi[i] >= 0].tolist()) <= set(allowed.tolist())
            assert np.array_equal(gi[i][:len(want[0])], want[0])   # +inf rows in scan order, at the end
    gix.free()
    # cosine against zero rows is NaN: allowed NaN rows follow every other allowed row, in scan order
    rows = rng.standard_normal((400, dim)).astype(np.float32)
    rows /= np.linalg.norm(rows, axis=1, keepdims=True)
    rows[[5, 50, 105, 160, 240, 330]] = 0
    gix = pv.IvfflatIndex("vector_cosine_ops", dim, lists).load(centers, off, rows, ids)
    oix = O.Ivf(O.VECTOR, pv.OPCLASSES["vector_cosine_ops"][1], centers, off, rows, ids, dim=dim)
    qn = q / np.linalg.norm(q, axis=1, keepdims=True)
    seqs = sequences(oix, qn, 3)
    for allowed in (np.array([50, 160, 240, 7, 8, 9]), np.arange(0, 400, 2), np.arange(400)):
        with gix.filter(allowed) as f:
            gi, gd = gix.search(qn, k=300, probes=3, filter=f)
        for i in range(len(q)):
            want = expect(seqs[i], allowed, 300)
            assert_matches(gi[i], gd[i], want)
            nan = np.isnan(want[1])
            assert np.array_equal(gi[i][:len(want[0])][nan], want[0][nan])
    gix.free()


# ---------------------------------------------------------------------------------------------- 7. errors


def test_errors_leave_the_host_output_untouched(pv):
    from pgvector_b200 import _lib
    rng = np.random.default_rng(9)
    dim, lists = 8, 4
    centers = rng.standard_normal((lists, dim)).astype(np.float32)
    rows = rng.standard_normal((200, dim)).astype(np.float32)
    off = np.array([0, 50, 100, 150, 200], dtype=np.int64)
    q = rng.standard_normal((3, dim)).astype(np.float32)
    L = _lib.load()

    def call(ix, filters, fq=None):
        ids = np.full((3, 5), 77, np.int64)
        dist = np.full((3, 5), 7.0)
        arr = (C.c_void_p * len(filters))(*[f.h.value for f in filters])
        rc = L.vb_ivf_search_filtered(ix.h, q.ctypes.data_as(C.c_void_p), 3, 2, 5, arr, len(filters),
                                      None if fq is None else np.asarray(fq, np.int32).ctypes.data_as(C.c_void_p),
                                      ids.ctypes.data_as(C.c_void_p), dist.ctypes.data_as(C.c_void_p))
        assert np.all(ids == 77) and np.all(dist == 7.0)
        return rc, (L.vb_last_error() or b"").decode()

    def load():
        return pv.IvfflatIndex("vector_l2_ops", dim, lists).load(centers, off, rows, np.arange(200, dtype=np.int64))

    a, b = load(), load()
    fa, fb = a.filter(np.arange(0, 200, 3)), b.filter(np.arange(0, 200, 2))
    rc, msg = call(a, [fb])
    assert rc == -1 and "another table or index" in msg
    rc, msg = call(a, [fa, fa], [0, 2, 1])
    assert rc == -1 and "filter_of_query[1] = 2" in msg
    b.free()
    rc, msg = call(a, [fb])
    assert rc == -1 and "another table or index" in msg
    fb.free()
    a.replace_list(2, rng.standard_normal((7, dim)).astype(np.float32), np.arange(1000, 1007, dtype=np.int64))
    rc, msg = call(a, [fa])
    assert rc == -5 and "index changed since the filter was created" in msg
    fa.free()
    fa = a.filter(np.arange(0, 200, 3))
    a.insert(rng.standard_normal((5, dim)).astype(np.float32), np.arange(2000, 2005, dtype=np.int64))
    rc, msg = call(a, [fa])
    assert rc == -5 and "index changed since the filter was created" in msg
    fa.free()
    fa = a.filter(np.arange(0, 200, 3))
    a.delete(np.array([3, 6], np.int64))
    rc, msg = call(a, [fa])
    assert rc == -5 and "index changed since the filter was created" in msg
    fa.free()
    u = pv.IvfflatIndex("vector_l2_ops", dim, lists)
    fa = a.filter(np.arange(0, 200, 3))
    rc, msg = call(u, [fa])
    assert rc == -5 and "not loaded" in msg
    fa.free()
    u.free()
    a.free()


# ---------------------------------------------------------------------------------------------- 8. TAP 009


def test_tap_009_predicates_in_one_call(pv):
    rng = np.random.default_rng(9)
    n, lists = 10_000, 100
    x = rng.random((n, 3), dtype=np.float32)
    kmetric = pv.OPCLASSES["vector_l2_ops"][3]
    ts = pv.Table(pv.VECTOR, 3).append(x[:50 * lists])
    centers, _ = pv.kmeans(ts, kmetric, pv.kmeans_pp_init(ts, kmetric, lists, seed=42), max_iter=100)
    ts.free()
    gix, oix = make_index(pv, "vector_l2_ops", x, np.ascontiguousarray(centers, np.float32), 3)
    c = (np.arange(n) + 1) % 50          # i % 50 of the TAP test's rows i = 1 .. n (id = i - 1)
    c0 = int(rng.integers(50))
    preds = [c == c0, c != c0, c >= 1, c < 1]
    allowed = [np.nonzero(p)[0].astype(np.int64) for p in preds]
    filters = [gix.filter(a) for a in allowed]
    queries = rng.random((64, 3), dtype=np.float32)
    fq = (np.arange(len(queries)) % 4).astype(np.int32)
    try:
        for probes in (1, 10):
            gi, gd = gix.search(queries, k=20, probes=probes, filter=filters, filter_of_query=fq)
            seqs = sequences(oix, queries, probes)
            for i in range(len(queries)):
                assert_matches(gi[i], gd[i], expect(seqs[i], allowed[fq[i]], 20))
    finally:
        for f in filters:
            f.free()
        gix.free()
