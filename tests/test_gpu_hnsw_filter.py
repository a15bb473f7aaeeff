"""Filtered hnsw.iterative_scan on the device (vb_hnsw_scan_begin_filtered): element filters of an HNSW image, and pages
of the allowed elements of each query's sequence.  The filtered sequence is the unfiltered handle's sequence restricted to
the allowed elements -- same order, same element numbers, same float8 distances bit for bit -- so it is checked against
the unfiltered handle on the same GPU, which makes the comparison exact even in long scans."""
import ctypes as C

import numpy as np
import pytest

import oracle as O
from tests.util import f32_to_half_bits, mixture

pytestmark = pytest.mark.gpu

EF = 40


@pytest.fixture(scope="module")
def pv():
    import pgvector_b200 as pv
    pv.init(0)
    return pv


OPCLASS_DIMS = {"vector_l2_ops": 16, "vector_ip_ops": 16, "vector_cosine_ops": 16, "vector_l1_ops": 16,
                "halfvec_l2_ops": 24, "bit_hamming_ops": 64, "bit_jaccard_ops": 64}
_GRAPHS = {}


def graph(pv, opclass, n=2000, nq=16):
    """a device-built graph of `opclass` and its queries (cached per module run)"""
    if opclass not in _GRAPHS:
        elem, _, normalize, _ = pv.OPCLASSES[opclass]
        dim = OPCLASS_DIMS[opclass]
        x, _ = mixture(n, dim, 20, seed=71)
        q, _ = mixture(nq, dim, 20, seed=72)
        if elem == O.HALFVEC:
            x, q = f32_to_half_bits(x), f32_to_half_bits(q)
        elif elem == O.BIT:
            x, q = O.binary_quantize(O.VECTOR, x), O.binary_quantize(O.VECTOR, q)
        if normalize:
            x, q = O.l2_normalize(elem, x), O.l2_normalize(elem, q)
        gi = pv.HnswIndex(opclass, dim, m=8).build(x, ef_construction=32, seed=3)
        _GRAPHS[opclass] = (gi, q)
    return _GRAPHS[opclass]


def unfiltered(gi, queries, ef, mst):
    """per query: element ids, distances, the batch of each element, and tuples after every batch (the last = at exhaustion)"""
    nq = len(queries)
    ids, dist, batch, tup = ([[] for _ in range(nq)] for _ in range(4))
    with gi.iterative_scan(queries, ef_search=ef, max_scan_tuples=mst) as sc:
        b = 0
        while True:
            bi, bd, cnt = sc.next_batch()
            t = sc.tuples()
            for q in range(nq):
                c = int(cnt[q])
                ids[q].extend(bi[q, :c].tolist())
                dist[q].extend(bd[q, :c].tolist())
                batch[q].extend([b] * c)
                tup[q].append(int(t[q]))
            b += 1
            if not cnt.any():
                break
    return [(np.array(ids[q], np.int64), np.array(dist[q], np.float64), np.array(batch[q], np.int64), np.array(tup[q]))
            for q in range(nq)]


def filtered(gi, queries, ef, mst, filt, page, filter_of_query=None, free_after_begin=False, max_calls=100000):
    """per call: (ids [nq x page], distances, counts, tuples), until every query returned 0 twice"""
    calls = []
    with gi.iterative_scan(queries, ef_search=ef, max_scan_tuples=mst, filter=filt, filter_of_query=filter_of_query,
                           page=page) as sc:
        if free_after_begin:
            for f in (filt if isinstance(filt, list) else [filt]):
                f.free()
        zeros = 0
        for _ in range(max_calls):
            bi, bd, cnt = sc.next_batch()
            assert bi.shape == (len(queries), page)
            calls.append((bi, bd, cnt, sc.tuples()))
            zeros = zeros + 1 if not cnt.any() else 0
            if zeros == 2:
                break
    return calls


def check_query(ref, allowed, calls, q, page):
    """the filtered pages of query q against the unfiltered sequence restricted to `allowed` (a boolean mask)"""
    uid, ud, ub, ut = ref
    keep = allowed[uid]
    want_ids, want_d, want_b = uid[keep], ud[keep], ub[keep]
    got_ids, got_d = [], []
    done = False
    at = 0
    for bi, bd, cnt, tup in calls:
        c = int(cnt[q])
        assert np.all(bi[q, c:] == -1) and np.all(np.isinf(bd[q, c:]))
        if done:
            assert c == 0                                            # 0 stays 0
            assert int(tup[q]) == ut[-1]
            continue
        got_ids.extend(bi[q, :c].tolist())
        got_d.extend(bd[q, :c].tolist())
        at += c
        if c == page:
            # the call stopped at the batch of its last element
            assert int(tup[q]) == ut[want_b[at - 1]], (q, at)
        else:
            done = True                                              # fewer than page: the sequence is exhausted
            assert int(tup[q]) == ut[-1]
    assert done
    assert np.array_equal(np.array(got_ids, np.int64), want_ids)
    assert np.array_equal(np.array(got_d, np.float64).view(np.int64), want_d.view(np.int64))   # bit for bit


def allowed_mask(n, sel, seed):
    if sel >= 1:
        return np.ones(n, bool)
    return np.random.default_rng(seed).random(n) < sel


@pytest.mark.parametrize("mst", [300, 3000, 10 ** 9])
@pytest.mark.parametrize("opclass", list(OPCLASS_DIMS))
def test_filtered_sequence_is_the_unfiltered_one_restricted(pv, opclass, mst):
    gi, queries = graph(pv, opclass)
    n = gi.n
    refs = unfiltered(gi, queries, EF, mst)
    exhausted_at = set()
    for si, sel in enumerate((1, 0.1, 0.01, 0.001, 0)):
        allowed = allowed_mask(n, sel, seed=100 + si)
        with gi.filter(np.flatnonzero(allowed)) as f:
            assert len(f) == int(allowed.sum())
            for page in (1, 7, EF, 3 * EF + 1):
                if page == 1 and allowed.sum() > 600:
                    continue            # (a call per allowed element: covered by the selective filters)
                calls = filtered(gi, queries, EF, mst, f, page)
                for q in range(len(queries)):
                    check_query(refs[q], allowed, calls, q, page)
                    exhausted_at.add(next(i for i, c in enumerate(calls) if c[2][q] < page))
    assert len(exhausted_at) > 1        # queries ran out at different calls


@pytest.mark.parametrize("mst", [300, 3000])
def test_per_query_filters_and_filters_freed_after_begin(pv, mst):
    """4 filters over 32 queries in one handle: each query's pages equal its filter's single-filter run.  At
    max_scan_tuples 300 every query reaches the drain, whose first step compacts each query's discarded array by its
    own filter."""
    gi, _ = graph(pv, "vector_l2_ops")
    queries, _ = mixture(32, 16, 20, seed=73)
    n = gi.n
    masks = [allowed_mask(n, s, seed=200 + i) for i, s in enumerate((0.5, 0.1, 0.02, 0.005))]
    fq = np.arange(32) % 4
    page = 9
    single = []
    for m in masks:
        with gi.filter(np.flatnonzero(m)) as f:
            single.append(filtered(gi, queries, EF, mst, f, page))
    filters = [gi.filter(np.flatnonzero(m)) for m in masks]
    calls = filtered(gi, queries, EF, mst, filters, page, filter_of_query=fq, free_after_begin=True)
    assert all(not f.h for f in filters)
    refs = unfiltered(gi, queries, EF, mst)
    if mst == 300:      # batches ran after the budget was spent: the drain
        assert all(np.any(ut[:-1] >= mst) and np.argmax(ut >= mst) < ub.max() for _, _, ub, ut in refs)
    for q in range(32):
        check_query(refs[q], masks[fq[q]], calls, q, page)
        mine = np.concatenate([c[0][q, :c[2][q]] for c in calls])
        alone = np.concatenate([c[0][q, :c[2][q]] for c in single[fq[q]]])
        assert np.array_equal(mine, alone)


def test_reference_where_mod_50_limit_11(pv):
    """the WHERE i % 50 = 0 ... LIMIT 11 shape of test/t/043_hnsw_iterative_scan.pl with the filter on the device: the 11
    rows equal the oracle's iterative scan restricted to the allowed elements (total order, short scans), and the
    nearest allowed rows are found"""
    rng = np.random.default_rng(5)
    rows = rng.random((20000, 3)).astype(np.float32)
    og = O.Hnsw(O.VECTOR, O.L2_SQUARED, rows, m=8, ef_construction=32, seed=7)
    g = og.export()
    er = g["elem_row"]
    gi = pv.HnswIndex("vector_l2_ops", 3, m=8).load(rows[er], g["levels"], g["nbr0"], g["upper_off"], g["upper"], g["entry"])
    allowed = er % 50 == 0
    queries = rows[[7, 101, 2024, 9999, 15000, 19998]]
    with gi.filter(np.flatnonzero(allowed)) as f:
        with gi.iterative_scan(queries, ef_search=40, max_scan_tuples=20000, filter=f, page=11) as sc:
            ids, dist, cnt = sc.next_batch()
    assert np.all(cnt == 11)
    same = 0
    for i, q in enumerate(queries):
        wi, wd, _, _ = og.iter_scan(q, 40, max_scan_tuples=20000, max_out=4000, ties=O.TIES_TOTAL)
        want = wi[allowed[wi]][:11]
        same += int(np.array_equal(ids[i], want))
        hits = set(er[ids[i]].tolist())
        d = ((rows[::50] - q) ** 2).sum(1)
        exact = set((np.argsort(d)[:5] * 50).tolist())
        assert len(exact & hits) >= 4
    assert same >= len(queries) - 1, same


def test_construction_counts_and_errors(pv):
    import torch
    gi, queries = graph(pv, "vector_l2_ops")
    n = gi.n
    with gi.filter(np.array([0, 5, 5, 9, n - 1])) as f:
        assert len(f) == 4                                           # duplicates collapse
    with gi.filter(np.array([], np.int64)) as f:
        assert len(f) == 0
    with pytest.raises(pv.VecB200Error) as e:
        gi.filter(np.array([3, n + 2]))
    assert e.value.code == -1 and f"elements[1] = {n + 2}" in str(e.value)
    with pytest.raises(pv.VecB200Error):
        gi.filter(np.array([-1]))
    dev = torch.tensor([-1, 3, n, 3, 7, 10 ** 12], dtype=torch.int64, device="cuda")
    with gi.filter(dev) as fd, gi.filter(np.array([3, 7])) as fh:
        assert len(fd) == 2                                          # out-of-range values ignored on the device
        a = filtered(gi, queries, EF, 3000, fd, 5)
        b = filtered(gi, queries, EF, 3000, fh, 5)
        assert len(a) == len(b) and all(np.array_equal(x[0], y[0]) for x, y in zip(a, b))


def test_cross_kind_and_stale_filters_are_refused(pv):
    gi, queries = graph(pv, "vector_l2_ops")
    x, _ = mixture(500, 16, 5, seed=74)
    other = pv.HnswIndex("vector_l2_ops", 16, m=8).build(x, ef_construction=32)
    t = pv.Table(pv.VECTOR, 16).append(x)
    ivf = pv.IvfflatIndex("vector_l2_ops", 16, 1).load(x[:1], np.array([0, 500]), x, np.arange(500))

    def code(fn):
        with pytest.raises(pv.VecB200Error) as e:
            fn()
        return e.value.code

    with gi.filter(np.arange(10)) as fh, t.filter(np.arange(10)) as ft, ivf.filter(np.arange(10)) as fi, \
            other.filter(np.arange(10)) as fo:
        assert code(lambda: gi.iterative_scan(queries, ef_search=EF, filter=ft)) == -1
        assert code(lambda: gi.iterative_scan(queries, ef_search=EF, filter=fi)) == -1
        assert code(lambda: gi.iterative_scan(queries, ef_search=EF, filter=fo)) == -1
        assert code(lambda: t.exact_topk(pv.L2_SQUARED, queries, 5, filter=fh)) == -1
        assert code(lambda: ivf.iterative_scan(queries, probes=1, filter=fh)) == -1
        assert code(lambda: gi.iterative_scan(queries, ef_search=EF, filter=[fh, fh], filter_of_query=[0, 2] + [0] * 14)) == -1
        assert code(lambda: gi.iterative_scan(queries, ef_search=EF, filter=fh, page=2049)) == -1
        assert code(lambda: gi.iterative_scan(queries, ef_search=EF, filter=fh, page=0)) == -1
    with pytest.raises(ValueError):
        gi.iterative_scan(queries, ef_search=EF, page=10)          # page without a filter
    # a filter whose index was freed is refused by a new index, whatever its address
    tmp = pv.HnswIndex("vector_l2_ops", 16, m=8).build(x, ef_construction=32)
    ft = tmp.filter(np.arange(10))
    tmp.free()
    again = pv.HnswIndex("vector_l2_ops", 16, m=8).build(x, ef_construction=32)
    assert code(lambda: again.iterative_scan(queries, ef_search=EF, filter=ft)) == -1
    ft.free()
    # a rebuild or a reload changes the image: its earlier filters are refused at begin
    for change in ("build", "load"):
        f = again.filter(np.arange(10))
        if change == "build":
            again.build(x, ef_construction=32)
        else:
            ex = again.export()
            again.load(x, ex["levels"], ex["nbr0"], ex["upper_off"], ex["upper"], ex["entry"])
        with pytest.raises(pv.VecB200Error) as e:
            again.iterative_scan(queries, ef_search=EF, filter=f)
        assert e.value.code == -5 and "index changed since the filter was created" in str(e.value)
        f.free()


def test_next_after_reload_fails_and_writes_nothing(pv):
    x, _ = mixture(800, 16, 5, seed=75)
    q, _ = mixture(4, 16, 5, seed=76)
    gi = pv.HnswIndex("vector_l2_ops", 16, m=8).build(x, ef_construction=32)
    with gi.filter(np.arange(0, 800, 3)) as f:
        sc = gi.iterative_scan(q, ef_search=EF, filter=f, page=6)
    ids, dist, cnt = sc.next_batch()
    assert np.all(cnt == 6)
    ex = gi.export()
    gi.load(x, ex["levels"], ex["nbr0"], ex["upper_off"], ex["upper"], ex["entry"])
    ids = np.full((4, 6), 123, np.int64)
    dist = np.full((4, 6), 4.5)
    cnt = np.full(4, 77, np.int32)
    p = lambda a: a.ctypes.data_as(C.c_void_p)
    rc = pv.load().vb_hnsw_scan_next(sc.h, p(ids), p(dist), p(cnt))
    assert rc == -5 and b"index changed" in pv.load().vb_last_error()
    assert np.all(ids == 123) and np.all(dist == 4.5) and np.all(cnt == 77)
    sc.close()


def test_empty_index(pv):
    gi = pv.HnswIndex("vector_l2_ops", 3)
    gi.load(np.zeros((0, 3), np.float32), np.zeros(0, np.int32), np.zeros((0, 32), np.int32), np.zeros(0, np.int64),
            np.zeros((0, 16), np.int32), -1)
    with gi.filter(np.array([], np.int64)) as f:
        assert len(f) == 0
        with gi.iterative_scan(np.ones((2, 3), np.float32), ef_search=10, filter=f, page=4) as sc:
            for _ in range(2):
                ids, dist, cnt = sc.next_batch()
                assert ids.shape == (2, 4) and np.all(ids == -1) and np.all(np.isinf(dist)) and np.all(cnt == 0)
