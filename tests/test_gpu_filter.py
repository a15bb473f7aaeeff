"""Row filters on the device (vb_table_filter_create / vb_ivf_filter_create, vb_exact_topk_filtered,
vb_ivf_scan_begin_filtered): "WHERE <predicate> ORDER BY v <op> q LIMIT k" where the allowed rows are never read.

- construction: allowed counts = |allowed ∩ image ids| with duplicates, absent ids, empty and full sets; device filters
  equal host ones; argument, ownership and staleness errors;
- exact: bit-identical to Table.rerank over the allowed rows in ascending order for every element type and metric at
  several selectivities, against the oracle, equal to vb_exact_topk (scan_impl 0) for the full set, ties, padding,
  rows appended later, per-query filters, host = device;
- IVFFlat iterative scan: the unfiltered handle's sequence restricted to the allowed ids, group by group, bit for bit, for
  six opclasses and the probes / max_probes / page grid of test_gpu_ivf_iterative.py; empty and per-query filters,
  filters freed after begin, refusal after replace_list;
- the reference's TAP tests 041 and 042 with the filter on the device."""
import numpy as np
import pytest

import oracle as O
from tests.test_gpu_distance import _random_rows
from tests.test_gpu_ivf_iterative import LISTS, MAX_LISTS, OPCLASSES, data_for, drain, groups_of, kmeans_index, make_index
from tests.test_gpu_rerank import check_against_reference

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def pv():
    import pgvector_b200 as pv
    pv.init(0)
    pv.set_option("scan_impl", 2)
    O.ivf_set_tie_mode(True)
    yield pv
    O.ivf_set_tie_mode(False)


def bits_equal(a, b):
    return np.array_equal(np.asarray(a).view(np.uint64), np.asarray(b).view(np.uint64))


# ---------------------------------------------------------------------------------------------- construction


@pytest.fixture(scope="module")
def ivf_small(pv):
    rows, centers, q = data_for("vector_l2_ops", 1500, 24, LISTS, seed=3)
    gix, oix = make_index(pv, "vector_l2_ops", rows, centers, 24)
    yield gix, oix, q
    gix.free()


def test_filter_rows_count_allowed_ids(pv, ivf_small):
    import torch
    gix, oix, _ = ivf_small
    image_ids = np.asarray(oix.ids)
    rng = np.random.default_rng(1)
    cases = [np.zeros(0, np.int64), image_ids.copy(), image_ids[rng.choice(len(image_ids), 40)],   # with duplicates
             np.concatenate([image_ids[::7], image_ids[::7], np.arange(10_000, 10_050), [-5, 2**40]]),  # absent ids too
             rng.permutation(image_ids)[:300]]
    for ids in cases:
        want = int(np.isin(image_ids, ids).sum())
        with gix.filter(ids) as f:
            assert len(f) == want
        with gix.filter(torch.from_numpy(np.ascontiguousarray(ids, dtype=np.int64)).cuda()) as f:
            assert len(f) == want
    t = pv.Table(pv.VECTOR, 4).append(np.zeros((100, 4), np.float32))
    for rows in (np.zeros(0, np.int64), np.arange(100), np.array([5, 5, 7, 99, 0, 7])):
        with t.filter(rows) as f:
            assert len(f) == len(set(rows.tolist()))
    with t.filter(torch.tensor([3, -1, 100, 3, 50], dtype=torch.int64, device="cuda")) as f:
        assert len(f) == 2   # values outside [0, n) are ignored on the device path
    t.free()


def test_filter_errors(pv, ivf_small):
    gix, oix, q = ivf_small
    t = pv.Table(pv.VECTOR, 24).append(np.zeros((10, 24), np.float32))
    t2 = pv.Table(pv.VECTOR, 24).append(np.zeros((10, 24), np.float32))
    with pytest.raises(pv.VecB200Error) as e:
        t.filter(np.array([1, 2, 10]))
    assert e.value.code == -1 and "rows[2] = 10" in str(e.value)
    with pytest.raises(pv.VecB200Error) as e:
        t.filter(np.array([-1]))
    assert e.value.code == -1 and "rows[0] = -1" in str(e.value)
    f2 = t2.filter(np.arange(3))
    fi = gix.filter(np.asarray(oix.ids)[:50])
    for f in (f2, fi):
        with pytest.raises(pv.VecB200Error) as e:
            t.exact_topk(pv.L2, q[:2], 5, filter=f)
        assert e.value.code == -1 and "another table or index" in str(e.value)
    with pytest.raises(pv.VecB200Error) as e:
        gix.iterative_scan(q, probes=2, max_probes=4, page=5, filter=t.filter(np.arange(3)))
    assert e.value.code == -1 and "another table or index" in str(e.value)
    with pytest.raises(pv.VecB200Error) as e:
        t.exact_topk(pv.L2, q[:2], 5, filter=[t.filter(np.arange(3)), t.filter(np.arange(4))], filter_of_query=[0, 2])
    assert e.value.code == -1 and "filter_of_query[1] = 2" in str(e.value)
    for f in (f2, fi):
        f.free()
    t.free()
    t2.free()


def test_ivf_filter_is_refused_after_replace_list(pv):
    rng = np.random.default_rng(9)
    dim, lists = 8, 4
    centers = rng.standard_normal((lists, dim)).astype(np.float32)
    rows = rng.standard_normal((200, dim)).astype(np.float32)
    off = np.array([0, 50, 100, 150, 200], dtype=np.int64)
    gix = pv.IvfflatIndex("vector_l2_ops", dim, lists).load(centers, off, rows, np.arange(200, dtype=np.int64))
    q = rng.standard_normal((3, dim)).astype(np.float32)
    f = gix.filter(np.arange(0, 200, 3))
    s = gix.iterative_scan(q, probes=1, max_probes=lists, page=5, filter=f)
    s.next_batch()
    gix.replace_list(2, rng.standard_normal((7, dim)).astype(np.float32), np.arange(1000, 1007, dtype=np.int64))
    with pytest.raises(pv.VecB200Error) as e:
        s.next_batch()
    assert e.value.code == -5 and "index changed since the scan began" in str(e.value)
    s.close()
    with pytest.raises(pv.VecB200Error) as e:
        gix.iterative_scan(q, probes=1, max_probes=lists, page=5, filter=f)
    assert e.value.code == -5 and "index changed since the filter was created" in str(e.value)
    f.free()
    gix.free()


def test_repeated_image_ids_and_device_filters_scan_alike(pv):
    """an id the image holds on several rows allows every one of them; a filter built from device ids scans exactly like
    the one built from host ids"""
    import torch
    rng = np.random.default_rng(12)
    dim, lists = 8, 4
    centers = rng.standard_normal((lists, dim)).astype(np.float32)
    rows = rng.standard_normal((300, dim)).astype(np.float32)
    off = np.array([0, 60, 150, 220, 300], dtype=np.int64)
    ids = np.arange(300, dtype=np.int64) % 97   # every id on three or four rows, spread over the lists
    gix = pv.IvfflatIndex("vector_l2_ops", dim, lists).load(centers, off, rows, ids)
    q = rng.standard_normal((5, dim)).astype(np.float32)
    with gix.iterative_scan(q, probes=1, max_probes=lists, page=7) as s:
        full, _ = drain(s)
    allowed = np.array([7, 7, 40, 96, 500], dtype=np.int64)
    with gix.filter(np.array([7])) as f:
        assert len(f) == int((ids == 7).sum()) == 4
    results = []
    for made in (gix.filter(allowed), gix.filter(torch.from_numpy(allowed).cuda())):
        assert len(made) == int(np.isin(ids, allowed).sum())
        with made as f, gix.iterative_scan(q, probes=1, max_probes=lists, page=7, filter=f) as s:
            pages, _ = drain(s)
        for i in range(len(q)):
            assert_groups_identical(groups_of(pages[i]), restricted(groups_of(full[i]), allowed))
        results.append(pages)
    for a, b in zip(*results):
        assert_groups_identical(groups_of(a), groups_of(b))
    gix.free()


def test_filter_of_a_freed_table_is_refused(pv):
    t = pv.Table(pv.VECTOR, 4).append(np.zeros((10, 4), np.float32))
    f = t.filter(np.arange(10))
    t.free()
    t2 = pv.Table(pv.VECTOR, 4).append(np.zeros((5, 4), np.float32))
    with pytest.raises(pv.VecB200Error) as e:
        t2.exact_topk(pv.L2, np.zeros((1, 4), np.float32), 3, filter=f)
    assert e.value.code == -1 and "another table or index" in str(e.value)
    f.free()
    t2.free()


# ---------------------------------------------------------------------------------------------- filtered exact top-k

EXACT = [(O.VECTOR, O.L2, 64), (O.VECTOR, O.L2_SQUARED, 17), (O.VECTOR, O.IP, 128), (O.VECTOR, O.NEG_IP, 32),
         (O.VECTOR, O.COSINE, 48), (O.VECTOR, O.L1, 20), (O.HALFVEC, O.L2, 96), (O.HALFVEC, O.NEG_IP, 40),
         (O.HALFVEC, O.COSINE, 64), (O.HALFVEC, O.L1, 24), (O.HALFVEC, O.IP, 16), (O.HALFVEC, O.L2_SQUARED, 8),
         (O.BIT, O.HAMMING, 1024), (O.BIT, O.JACCARD, 200)]
SELECTIVITY = ["none", "one", "0.1%", "10%", "all"]


def allowed_rows(rng, n, sel):
    if sel == "none":
        return np.zeros(0, np.int64)
    if sel == "one":
        return np.array([int(rng.integers(n))], np.int64)
    if sel == "all":
        return np.arange(n, dtype=np.int64)
    frac = {"0.1%": 0.001, "10%": 0.1}[sel]
    return np.sort(rng.choice(n, max(1, int(n * frac)), replace=False)).astype(np.int64)


@pytest.mark.parametrize("sel", SELECTIVITY)
@pytest.mark.parametrize("elem,metric,dim", EXACT)
def test_exact_filtered_is_the_rerank_and_the_oracle(pv, elem, metric, dim, sel):
    rng = np.random.default_rng(dim * 11 + metric * 5 + elem + len(sel))
    n, nq, k = 5000, 6, 10
    rows = _random_rows(elem, n, dim, rng)
    queries = _random_rows(elem, nq, dim, rng)
    t = pv.Table(elem, dim).append(rows)
    allowed = allowed_rows(rng, n, sel)
    # shuffled and repeated: the filter holds the set
    with t.filter(np.concatenate([rng.permutation(allowed), allowed[: len(allowed) // 3]])) as f:
        assert len(f) == len(allowed)
        gi, gd = t.exact_topk(metric, queries, k, filter=f)
        cand = np.tile(allowed, (nq, 1))
        wi, wd = t.rerank(metric, queries, cand, k)
        assert np.array_equal(gi, wi) and bits_equal(gd, wd)
        check_against_reference(elem, metric, rows, queries, cand, gi, gd, k, dim)
    t.free()


@pytest.mark.parametrize("elem,metric,dim", [(O.VECTOR, O.L2, 1536), (O.HALFVEC, O.NEG_IP, 96), (O.BIT, O.HAMMING, 512),
                                             (O.VECTOR, O.COSINE, 24)])
def test_full_filter_is_the_exact_scan(pv, elem, metric, dim):
    rng = np.random.default_rng(dim + metric)
    n = 3000
    rows = _random_rows(elem, n, dim, rng)
    queries = _random_rows(elem, 70, dim, rng)   # >= 64 queries: vb_exact_topk would tile under scan_impl 2
    t = pv.Table(elem, dim).append(rows)
    pv.set_option("scan_impl", 0)
    try:
        with t.filter(np.arange(n)) as f:
            for k in (1, 100, 2048):
                wi, wd = t.exact_topk(metric, queries, k)
                gi, gd = t.exact_topk(metric, queries, k, filter=f)
                assert np.array_equal(gi, wi) and bits_equal(gd, wd), k
    finally:
        pv.set_option("scan_impl", 2)
    t.free()


def test_ties_padding_appends_and_device_path(pv):
    import torch
    rows = np.ones((60, 4), np.float32)
    rows[10:20] = 3.0
    t = pv.Table(O.VECTOR, 4).append(rows)
    q = np.zeros((2, 4), np.float32)
    allowed = np.arange(0, 60, 2, dtype=np.int64)
    f = t.filter(allowed[::-1].copy())
    ids, _ = t.exact_topk(O.L2, q, 27, filter=f)
    assert list(ids[0]) == [i for i in allowed if not 10 <= i < 20] + [10, 12]
    # fewer allowed rows than k: the re-rank's padding
    ids, dist = t.exact_topk(O.L2, q, 40, filter=f)
    wi, wd = t.rerank(O.L2, q, np.tile(allowed, (2, 1)), 40)
    assert np.array_equal(ids, wi) and bits_equal(dist, wd)
    assert np.all(ids[:, 30:] == -1)
    # rows appended after the filter was made are never returned, even when nearer
    t.append(np.zeros((50, 4), np.float32))
    ids2, dist2 = t.exact_topk(O.L2, q, 40, filter=f)
    assert np.array_equal(ids2, ids) and bits_equal(dist2, dist)
    # device queries and outputs: the host results
    di, dd = t.exact_topk(O.L2, torch.from_numpy(q).cuda(), 40, filter=f)
    assert np.array_equal(di.cpu().numpy(), ids) and np.array_equal(dd.cpu().numpy(), dist.astype(np.float32))
    f.free()
    t.free()


@pytest.mark.parametrize("elem,metric,dim", [(O.VECTOR, O.L2, 64), (O.HALFVEC, O.COSINE, 32), (O.BIT, O.JACCARD, 256)])
def test_per_query_filters_equal_one_call_per_filter(pv, elem, metric, dim):
    import torch
    rng = np.random.default_rng(77 + metric)
    n, nq, nf, k = 4000, 256, 16, 12
    rows = _random_rows(elem, n, dim, rng)
    queries = _random_rows(elem, nq, dim, rng)
    t = pv.Table(elem, dim).append(rows)
    filters = [t.filter(np.nonzero(np.arange(n) % nf == i)[0]) for i in range(nf - 1)] + [t.filter(np.zeros(0, np.int64))]
    fq = rng.integers(0, nf, nq).astype(np.int32)
    gi, gd = t.exact_topk(metric, queries, k, filter=filters, filter_of_query=fq)
    for i in range(nf):
        sel = np.nonzero(fq == i)[0]
        if len(sel):
            wi, wd = t.exact_topk(metric, queries[sel], k, filter=filters[i])
            assert np.array_equal(gi[sel], wi) and bits_equal(gd[sel], wd), i
    qd = torch.from_numpy(np.ascontiguousarray(queries)).cuda()
    di, dd = t.exact_topk(metric, qd, k, filter=filters, filter_of_query=fq)
    assert np.array_equal(di.cpu().numpy(), gi) and np.array_equal(dd.cpu().numpy(), gd.astype(np.float32))
    for f in filters:
        f.free()
    t.free()


def test_per_query_filters_with_a_scan_launch_per_filter(pv):
    """filters whose queries fill the scan grid get a scan launch each: still one call per filter's results"""
    rng = np.random.default_rng(5)
    n, dim, nq, nf, k = 20000, 1536, 64, 4, 20
    rows = rng.standard_normal((n, dim)).astype(np.float32)
    queries = rng.standard_normal((nq, dim)).astype(np.float32)
    t = pv.Table(O.VECTOR, dim).append(rows)
    filters = [t.filter(np.nonzero(np.arange(n) % nf == i)[0]) for i in range(nf)]
    fq = (np.arange(nq) * 7 % nf).astype(np.int32)
    gi, gd = t.exact_topk(O.L2, queries, k, filter=filters, filter_of_query=fq)
    for i in range(nf):
        sel = np.nonzero(fq == i)[0]
        wi, wd = t.rerank(O.L2, queries[sel], np.tile(np.nonzero(np.arange(n) % nf == i)[0], (len(sel), 1)), k)
        assert np.array_equal(gi[sel], wi) and bits_equal(gd[sel], wd), i
    for f in filters:
        f.free()
    t.free()


# ---------------------------------------------------------------------------------------------- filtered iterative scan


@pytest.fixture(scope="module")
def indexes(pv):
    out = {}
    for i, opclass in enumerate(OPCLASSES):
        dim = 64 if opclass.startswith("bit") else 24
        rows, centers, q = data_for(opclass, 1500, dim, LISTS, seed=10 + i)
        gix, oix = make_index(pv, opclass, rows, centers, dim)
        out[opclass] = (gix, oix, q)
    yield out
    for gix, _, _ in out.values():
        gix.free()


def restricted(groups, allowed):
    """the unfiltered groups of one query restricted to the allowed ids, groups left empty dropped"""
    out = []
    for done, ids, dist in groups:
        keep = np.isin(ids, allowed)
        if keep.any():
            out.append((done, ids[keep], dist[keep]))
    return out


def assert_groups_identical(got, want):
    assert [g[0] for g in got] == [w[0] for w in want]
    for (_, gi, gd), (_, wi, wd) in zip(got, want):
        assert np.array_equal(gi, wi) and bits_equal(gd, wd)


@pytest.mark.parametrize("page", [1, 10, 2048])
@pytest.mark.parametrize("mp", ["p", "2p+1", "lists"])
@pytest.mark.parametrize("probes", [1, 3, 7])
@pytest.mark.parametrize("opclass", OPCLASSES)
def test_filtered_sequences_are_the_unfiltered_ones_restricted(pv, indexes, opclass, probes, mp, page):
    gix, oix, q = indexes[opclass]
    max_probes = {"p": probes, "2p+1": 2 * probes + 1, "lists": LISTS}[mp]
    ids = np.asarray(oix.ids)
    allowed = ids[np.random.default_rng(probes * 31 + page).random(len(ids)) < 0.1]
    with gix.iterative_scan(q, probes=probes, max_probes=max_probes, page=page) as s:
        full, _ = drain(s)
    with gix.filter(allowed) as f, gix.iterative_scan(q, probes=probes, max_probes=max_probes, page=page, filter=f) as s:
        pages, history = drain(s)
        assert s.lists_done().tolist() == [min(max_probes, LISTS)] * len(q)
    for i in range(len(q)):
        assert_groups_identical(groups_of(pages[i]), restricted(groups_of(full[i]), allowed))


def test_empty_per_query_and_freed_filters(pv, indexes):
    gix, oix, q = indexes["vector_l2_ops"]
    probes, max_probes, page = 2, 9, 7
    ids = np.asarray(oix.ids)
    with gix.iterative_scan(q, probes=probes, max_probes=max_probes, page=page) as s:
        full, _ = drain(s)
    # an empty filter: the first next returns all zero counts
    with gix.filter(np.zeros(0, np.int64)) as f, gix.iterative_scan(q, probes=probes, max_probes=max_probes, page=page, filter=f) as s:
        _, _, cnt = s.next_batch()
        assert not cnt.any()
        assert s.lists_done().tolist() == [max_probes] * len(q)
    # per-query filters, freed right after begin
    sets = [ids[ids % 4 == r] for r in range(4)]
    filters = [gix.filter(a) for a in sets]
    fq = np.arange(len(q), dtype=np.int32) % 4
    s = gix.iterative_scan(q, probes=probes, max_probes=max_probes, page=page, filter=filters, filter_of_query=fq)
    for f in filters:
        f.free()
    pages, _ = drain(s)
    s.close()
    for i in range(len(q)):
        assert_groups_identical(groups_of(pages[i]), restricted(groups_of(full[i]), sets[fq[i]]))


def test_iterative_scan_off_first_page_is_the_limit_answer(pv, indexes):
    gix, oix, q = indexes["halfvec_l2_ops"]
    probes, k = 3, 10
    ids = np.asarray(oix.ids)
    allowed = ids[ids % 5 == 0]
    with gix.iterative_scan(q, probes=probes, max_probes=probes, page=1000) as s:
        full, _ = drain(s)
    with gix.filter(allowed) as f, gix.iterative_scan(q, probes=probes, max_probes=probes, page=k, filter=f) as s:
        got, _, cnt = s.next_batch()
    for i in range(len(q)):
        want = [t for t in np.concatenate([p[1] for p in full[i]]) if t in set(allowed.tolist())][:k]
        assert got[i, :cnt[i]].tolist() == [int(t) for t in want]


# ---------------------------------------------------------------------------------------------- the reference's TAP tests


@pytest.fixture(scope="module")
def uniform3():
    rng = np.random.default_rng(41)
    return rng.random((100_000, 3), dtype=np.float32)


def limit_of(scan, limit):
    got = [[] for _ in range(scan.nq)]
    live = np.ones(scan.nq, dtype=bool)
    while live.any():
        ids, _, cnt = scan.next_batch()
        for q in np.nonzero(live)[0]:
            if cnt[q] == 0:
                live[q] = False
                continue
            got[q].extend(int(t) for t in ids[q, :cnt[q]])
            if len(got[q]) >= limit:
                got[q] = got[q][:limit]
                live[q] = False
    return got


def test_tap_041_filtered_counts_on_the_device(pv, uniform3):
    x = uniform3
    ix = kmeans_index(pv, "vector_l2_ops", x, 100)
    ids = np.arange(1, len(x) + 1)
    with ix.filter(ids[ids % 10000 == 0]) as f:
        with ix.iterative_scan(x[:1], probes=10, max_probes=MAX_LISTS, page=100, filter=f) as s:
            assert len(limit_of(s, 11)[0]) == 10
        for max_probes in (30, 50, 70):
            with ix.iterative_scan(x[:20], probes=10, max_probes=max_probes, page=100, filter=f) as s:
                avg = np.mean([len(g) for g in limit_of(s, 11)])
            assert max_probes / 10 - 2 < avg < max_probes / 10 + 2, (max_probes, avg)
    ix.free()


@pytest.mark.parametrize("opclass,metric", [("vector_l2_ops", "l2"), ("vector_cosine_ops", "cosine")])
def test_tap_042_recall_on_the_device(pv, uniform3, opclass, metric):
    x = uniform3
    rng = np.random.default_rng(42)
    queries = rng.random((20, 3), dtype=np.float32)
    ix = kmeans_index(pv, opclass, x, 100)
    q = ix.prepare_query(queries)
    ids_all = np.arange(1, len(x) + 1)
    table = pv.Table(pv.VECTOR, 3).append(x)
    floors = {100: {1: 0.57, 10: 0.98}, 1000: {1: 0.80 if metric == "l2" else 0.88}}
    for c, by_probes in floors.items():
        sel = ids_all % c == 0
        # the truth: the filtered exact top-20 on the device (row r holds id r + 1), ties within 1e-6 counted
        with table.filter(np.nonzero(sel)[0]) as tf:
            tids, tdist = table.exact_topk(pv.L2 if metric == "l2" else pv.COSINE, queries, 20, filter=tf)
        xs = x[sel].astype(np.float64)
        if metric == "l2":
            d = np.sqrt(((xs[None] - queries[:, None].astype(np.float64)) ** 2).sum(-1))
        else:
            qn = queries / np.linalg.norm(queries, axis=1, keepdims=True)
            d = 1 - (xs @ qn.T.astype(np.float64)).T / np.linalg.norm(xs, axis=1)[None]
        truth = [set((tids[i] + 1).tolist()) | set(ids_all[sel][d[i] <= tdist[i, 19] + 1e-6].tolist()) for i in range(len(queries))]
        with ix.filter(ids_all[sel]) as f:
            for probes, floor in by_probes.items():
                with ix.iterative_scan(q, probes=probes, max_probes=MAX_LISTS, page=100, filter=f) as s:
                    got = limit_of(s, 20)
                recall = sum(len(set(g) & truth[i]) for i, g in enumerate(got)) / (20 * len(queries))
                assert recall >= floor, (c, probes, recall)
    table.free()
    ix.free()
