"""ivfflat.iterative_scan on the device (vb_ivf_scan_begin / _next / _lists_done / _end) against the oracle's
restatement (tests/ivf_iter_oracle.py), the per-scan path (vb_ivf_scan_items) and the reference's TAP tests
test/t/041_ivfflat_iterative_scan.pl and test/t/042_ivfflat_iterative_scan_recall.pl."""
import numpy as np
import pytest

import oracle as O
from tests.ivf_iter_oracle import iter_scan
from tests.util import assert_same_neighbours, build_ivf_arrays, f32_to_half_bits

pytestmark = pytest.mark.gpu
RTOL = 1e-5
MAX_LISTS = 32768   # IVFFLAT_MAX_LISTS, the default of ivfflat.max_probes


@pytest.fixture(scope="module")
def pv():
    import pgvector_b200 as pv
    pv.init(0)
    pv.set_option("scan_impl", 2)
    O.ivf_set_tie_mode(True)   # equal centre distances: smaller list number first, as on the device
    yield pv
    O.ivf_set_tie_mode(False)


def drain(scan, max_calls=1_000_000):
    """every page of every query until all are exhausted: per query [(lists_done after the call, ids, dist)], and the
    lists_done of every call"""
    pages = [[] for _ in range(scan.nq)]
    history = []
    for _ in range(max_calls):
        ids, dist, cnt = scan.next_batch()
        done = scan.lists_done()
        history.append((cnt.copy(), done.copy()))
        for q in range(scan.nq):
            c = int(cnt[q])
            assert np.all(ids[q, c:] == -1) and np.all(np.isinf(dist[q, c:]))
            if c:
                pages[q].append((int(done[q]), ids[q, :c].copy(), dist[q, :c].copy()))
        if not cnt.any():
            return pages, history
    raise AssertionError("scan did not end")


def groups_of(pages):
    """pages of one query -> [(listIndex after the group, ids, dist)]: a page never spans two groups"""
    out = []
    for done, ids, dist in pages:
        if out and out[-1][0] == done:
            out[-1] = (done, np.concatenate([out[-1][1], ids]), np.concatenate([out[-1][2], dist]))
        else:
            out.append((done, ids, dist))
    return out


def oracle_groups(oix, q, probes, max_probes):
    p = min(probes, oix.lists)
    P = min(max(max_probes, probes), oix.lists)
    return [(min((g + 1) * p, P), ids, dist) for g, (ids, dist) in enumerate(iter_scan(oix, q, probes, max_probes)) if len(ids)]


def assert_groups_match(got, want, exact):
    assert [g[0] for g in got] == [g[0] for g in want]
    for (_, gi, gd), (_, wi, wd) in zip(got, want):
        assert len(gi) == len(wi) and set(gi.tolist()) == set(wi.tolist())
        if exact:
            assert np.array_equal(gi, wi) and np.array_equal(gd, wd)
        else:
            # distances within 1e-5 (absolute near 0: inner products of unit vectors cancel), ids equal up to near-ties:
            # where the orders differ, the id the device put there carries the oracle's distance of that position
            assert np.allclose(gd, wd, rtol=RTOL, atol=1e-6)
            d_of = dict(zip(wi.tolist(), wd.tolist()))
            for j in np.nonzero(gi != wi)[0]:
                assert abs(d_of[int(gi[j])] - wd[j]) <= RTOL * abs(wd[j]) + 1e-6, (j, gi[j], wi[j])


# ---------------------------------------------------------------------------------------------- indexes


def data_for(opclass, n, dim, lists, seed):
    """rows, centres and queries in the payload layout of the opclass (cosine: normalised, as the index stores them)"""
    rng = np.random.default_rng(seed)
    x = rng.standard_normal((n, dim)).astype(np.float32)
    q = rng.standard_normal((8, dim)).astype(np.float32)
    if opclass.startswith("bit"):
        pack = lambda a: np.packbits(a > 0, axis=1)
        rows = pack(x)
        return rows, rows[rng.choice(n, lists, replace=False)].copy(), pack(q)
    if "cosine" in opclass:
        x /= np.linalg.norm(x, axis=1, keepdims=True)
        q /= np.linalg.norm(q, axis=1, keepdims=True)
    centers = x[rng.choice(n, lists, replace=False)] + 0.1 * rng.standard_normal((lists, dim)).astype(np.float32)
    if opclass.startswith("halfvec"):
        return f32_to_half_bits(x), f32_to_half_bits(centers), f32_to_half_bits(q)
    return x, centers, q


def make_index(pv, opclass, rows, centers, dim):
    elem, metric, _, _ = pv.OPCLASSES[opclass]
    lists = centers.shape[0]
    assign = O.ivf_assign(elem, metric, rows, centers, threads=8, dim=dim)
    grouped, ids, offsets = build_ivf_arrays(rows, assign, lists)
    gix = pv.IvfflatIndex(opclass, dim, lists).load(centers, offsets, grouped, ids)
    oix = O.Ivf(elem, metric, centers, offsets, grouped, ids, dim=dim)
    return gix, oix


OPCLASSES = ["vector_l2_ops", "vector_ip_ops", "vector_cosine_ops", "halfvec_l2_ops", "halfvec_cosine_ops", "bit_hamming_ops"]
LISTS = 16


@pytest.fixture(scope="module")
def indexes(pv):
    out = {}
    for i, opclass in enumerate(OPCLASSES):
        dim = 64 if opclass.startswith("bit") else 24
        rows, centers, q = data_for(opclass, 1500, dim, LISTS, seed=10 + i)
        gix, oix = make_index(pv, opclass, rows, centers, dim)
        out[opclass] = (gix, oix, q)
    return out


# ---------------------------------------------------------------------------------------------- 1. the regression output


def three_rows(pv, rows):
    centers = np.array([[0, 0, 0], [1, 2, 3], [1, 1, 1]], dtype=np.float32)
    off = np.arange(4, dtype=np.int64) if len(rows) else np.zeros(4, dtype=np.int64)
    return pv.IvfflatIndex("vector_l2_ops", 3, 3).load(centers, off, rows.reshape(-1, 3), np.arange(len(rows), dtype=np.int64)), centers


@pytest.mark.parametrize("max_probes,want", [(MAX_LISTS, [[1, 2, 3], [1, 1, 1], [0, 0, 0]]), (1, [[1, 2, 3]]), (2, [[1, 2, 3], [1, 1, 1]])])
def test_regression_output_orderings(pv, max_probes, want):
    ix, rows = three_rows(pv, np.array([[0, 0, 0], [1, 2, 3], [1, 1, 1]], dtype=np.float32))
    with ix.iterative_scan(np.array([3, 3, 3], dtype=np.float32), probes=1, max_probes=max_probes, page=10) as s:
        assert [rows[i].tolist() for i, _ in s.tuples_of(0)] == want
    ix.free()


def test_regression_output_empty_index(pv):
    ix, _ = three_rows(pv, np.zeros((0, 3), dtype=np.float32))
    with ix.iterative_scan(np.array([3, 3, 3], dtype=np.float32), probes=1, max_probes=MAX_LISTS, page=10) as s:
        assert s.tuples_of(0) == []
        assert s.lists_done().tolist() == [3]
    ix.free()


# ---------------------------------------------------------------------------------------------- 2. sequences = the oracle's


@pytest.mark.parametrize("page", [1, 10, 2048])
@pytest.mark.parametrize("mp", ["p", "2p+1", "lists"])
@pytest.mark.parametrize("probes", [1, 3, 7])
@pytest.mark.parametrize("opclass", OPCLASSES)
def test_sequences_match_oracle(pv, indexes, opclass, probes, mp, page):
    gix, oix, q = indexes[opclass]
    max_probes = {"p": probes, "2p+1": 2 * probes + 1, "lists": LISTS}[mp]
    with gix.iterative_scan(q, probes=probes, max_probes=max_probes, page=page) as s:
        pages, _ = drain(s)
    for i in range(len(q)):
        assert_groups_match(groups_of(pages[i]), oracle_groups(oix, q[i], probes, max_probes), exact=opclass.startswith("bit"))


# ---------------------------------------------------------------------------------------------- 3. bit-identical to the per-scan path


@pytest.mark.parametrize("scan_impl", [2, 0])
@pytest.mark.parametrize("opclass", ["vector_l2_ops", "vector_ip_ops", "halfvec_l2_ops", "bit_hamming_ops"])
def test_sequences_equal_scan_items(pv, indexes, opclass, scan_impl):
    gix, _, q = indexes[opclass]
    probes, max_probes = 3, 10
    pv.set_option("scan_impl", scan_impl)
    try:
        with gix.iterative_scan(q, probes=probes, max_probes=max_probes, page=37) as s:
            pages, _ = drain(s)
        lists, _ = gix.scan_lists(q, max_probes)
        for i in range(len(q)):
            want = []
            for g0 in range(0, max_probes, probes):
                ids, dist, n = gix.scan_items(q[i], lists[i, g0:g0 + probes])
                if n:
                    want.append((min(g0 + probes, max_probes), ids, dist))
            got = groups_of(pages[i])
            assert [g[0] for g in got] == [w[0] for w in want]
            for (_, gi, gd), (_, wi, wd) in zip(got, want):
                assert np.array_equal(gi, wi) and np.array_equal(gd, wd)
    finally:
        pv.set_option("scan_impl", 2)


# ---------------------------------------------------------------------------------------------- 4. queries progress independently


@pytest.mark.parametrize("page", [1, 10])
def test_skewed_index_queries_in_different_groups(pv, page):
    rng = np.random.default_rng(5)
    dim, lists = 16, 8
    centers = rng.standard_normal((lists, dim)).astype(np.float32)
    sizes = [900, 0, 0, 50, 40, 30, 30, 30]          # one giant list, two empty ones; list 4 is emptied below
    rows = np.concatenate([centers[l] + 0.3 * rng.standard_normal((n, dim)).astype(np.float32) for l, n in enumerate(sizes)])
    off = np.concatenate([[0], np.cumsum(sizes)]).astype(np.int64)
    ids = np.arange(len(rows), dtype=np.int64) + 1000
    gix = pv.IvfflatIndex("vector_l2_ops", dim, lists).load(centers, off, rows, ids)
    gix.replace_list(4, np.zeros((0, dim), dtype=np.float32), np.zeros(0, dtype=np.int64))
    keep = np.r_[0:off[4], off[5]:off[-1]]
    off2 = off.copy()
    off2[5:] -= sizes[4]
    oix = O.Ivf(O.VECTOR, O.L2_SQUARED, centers, off2, rows[keep], ids[keep])
    q = rng.standard_normal((12, dim)).astype(np.float32) * 2
    probes, max_probes = 2, lists
    with gix.iterative_scan(q, probes=probes, max_probes=max_probes, page=page) as s:
        assert s.lists_done().tolist() == [0] * len(q)
        pages, history = drain(s)
    mixed = False
    for cnt, done in history:
        live = done[cnt > 0]
        mixed |= len(set(live.tolist())) > 1
    assert mixed, "every call had all queries in the same group"
    for i in range(len(q)):
        want = oracle_groups(oix, q[i], probes, max_probes)
        assert_groups_match(groups_of(pages[i]), want, exact=False)
        # listIndex per call: the end of the group the page came from; max_probes once exhausted
        ends = [d for d, _, _ in pages[i]]
        assert ends == sorted(ends)
        assert history[-1][1][i] == max_probes


# ---------------------------------------------------------------------------------------------- 5. exhaustion


def test_exhaustion_totals_and_first_group(pv, indexes):
    gix, oix, q = indexes["vector_l2_ops"]
    probes, max_probes = 3, 9
    lists, _ = gix.scan_lists(q, max_probes)
    with gix.iterative_scan(q, probes=probes, max_probes=max_probes, page=64) as s:
        pages, _ = drain(s)
        for _ in range(2):
            assert not s.next_batch()[2].any()
        assert s.lists_done().tolist() == [max_probes] * len(q)
    for i in range(len(q)):
        assert sum(len(p[1]) for p in pages[i]) == sum(int(oix.offsets[l + 1] - oix.offsets[l]) for l in lists[i])
    # max_probes = probes (iterative_scan = off): exactly the first group, whose first page is vb_ivf_search's top page
    page = 10
    with gix.iterative_scan(q, probes=probes, max_probes=probes, page=page) as s:
        first = s.next_batch()
        pages, _ = drain(s)
    for i in range(len(q)):
        assert {d for d, _, _ in pages[i]} <= {probes}
    ids, dist = gix.search(q, k=page, probes=probes)
    assert_same_neighbours(first[0], first[1], ids, dist, RTOL)


# ---------------------------------------------------------------------------------------------- 6-7. the reference's TAP tests


def kmeans_index(pv, opclass, x, lists, seed=42):
    elem, metric, normalize, kmetric = pv.OPCLASSES[opclass]
    rows = (x / np.linalg.norm(x, axis=1, keepdims=True)).astype(np.float32) if normalize else x
    ts = pv.Table(elem, rows.shape[1]).append(rows[:50 * lists])
    centers, _ = pv.kmeans(ts, kmetric, pv.kmeans_pp_init(ts, kmetric, lists, seed=seed), max_iter=100)
    ts.free()
    ta = pv.Table(elem, rows.shape[1]).append(rows)
    assign = pv.assign(ta, metric, centers)
    ta.free()
    grouped, order, offsets = build_ivf_arrays(rows, assign.astype(np.int64), lists)
    return pv.IvfflatIndex(opclass, rows.shape[1], lists).load(centers, offsets, grouped, order + 1)   # ids: i = 1..n


def filtered(scan, keep, limit):
    """per query, the ids the executor keeps (keep(id)) until LIMIT or the end of the scan"""
    got = [[] for _ in range(scan.nq)]
    live = np.ones(scan.nq, dtype=bool)
    while live.any():
        ids, _, cnt = scan.next_batch()
        for q in np.nonzero(live)[0]:
            if cnt[q] == 0:
                live[q] = False
                continue
            got[q].extend(int(t) for t in ids[q, :cnt[q]] if keep(int(t)))
            if len(got[q]) >= limit:
                got[q] = got[q][:limit]
                live[q] = False
    return got


@pytest.fixture(scope="module")
def uniform3(pv):
    rng = np.random.default_rng(41)
    return rng.random((100_000, 3), dtype=np.float32)


def test_tap_041_filtered_counts(pv, uniform3):
    x = uniform3
    ix = kmeans_index(pv, "vector_l2_ops", x, 100)
    keep = lambda i: i % 10000 == 0
    with ix.iterative_scan(x[:1], probes=10, max_probes=MAX_LISTS, page=100) as s:
        assert len(filtered(s, keep, 11)[0]) == 10
    for max_probes in (30, 50, 70):
        with ix.iterative_scan(x[:20], probes=10, max_probes=max_probes, page=100) as s:
            avg = np.mean([len(g) for g in filtered(s, keep, 11)])
        assert max_probes / 10 - 2 < avg < max_probes / 10 + 2, (max_probes, avg)
    ix.free()


@pytest.mark.parametrize("opclass,metric", [("vector_l2_ops", "l2"), ("vector_cosine_ops", "cosine")])
def test_tap_042_recall(pv, uniform3, opclass, metric):
    x = uniform3
    rng = np.random.default_rng(42)
    queries = rng.random((20, 3), dtype=np.float32)
    ix = kmeans_index(pv, opclass, x, 100)
    q = ix.prepare_query(queries)
    ids_all = np.arange(1, len(x) + 1)
    floors = {100: {1: 0.57, 10: 0.98}, 1000: {1: 0.80 if metric == "l2" else 0.88}}
    for c, by_probes in floors.items():
        sel = ids_all % c == 0
        t = pv.Table(pv.VECTOR, 3).append(x[sel])
        tids, tdist = t.exact_topk(pv.L2 if metric == "l2" else pv.COSINE, queries, 20)
        t.free()
        xs = x[sel].astype(np.float64)
        if metric == "l2":
            d = np.sqrt(((xs[None] - queries[:, None].astype(np.float64)) ** 2).sum(-1))
        else:
            qn = queries / np.linalg.norm(queries, axis=1, keepdims=True)
            d = 1 - (xs @ qn.T.astype(np.float64)).T / np.linalg.norm(xs, axis=1)[None]
        # the test's truth: every filtered row no further than the 20th filtered distance (the float64 distances here
        # and the device's float32 ones differ by rounding: the 20 nearest always count, ties within 1e-6 too)
        truth = [set(ids_all[sel][tids[i]].tolist()) | set(ids_all[sel][d[i] <= tdist[i, 19] + 1e-6].tolist()) for i in range(len(queries))]
        for probes, floor in by_probes.items():
            with ix.iterative_scan(q, probes=probes, max_probes=MAX_LISTS, page=100) as s:
                got = filtered(s, lambda i: i % c == 0, 20)
            recall = sum(len(set(g) & truth[i]) for i, g in enumerate(got)) / (20 * len(queries))
            assert recall >= floor, (c, probes, recall)
    ix.free()


# ---------------------------------------------------------------------------------------------- 8-10. isolation, changes, errors


def test_interleaved_handles_and_searches_do_not_change_sequences(pv, indexes):
    gix, _, q = indexes["vector_l2_ops"]
    table = pv.Table(pv.VECTOR, q.shape[1]).append(np.random.default_rng(3).standard_normal((5000, q.shape[1])).astype(np.float32))
    args = [dict(probes=3, max_probes=9, page=10), dict(probes=2, max_probes=LISTS, page=7)]
    alone = []
    for a, qq in zip(args, (q[:4], q[4:])):
        with gix.iterative_scan(qq, **a) as s:
            alone.append(drain(s)[0])
    sa, sb = gix.iterative_scan(q[:4], **args[0]), gix.iterative_scan(q[4:], **args[1])
    got = [[[] for _ in range(4)], [[] for _ in range(4)]]
    live = [True, True]
    step = 0
    while any(live):
        for h, s in enumerate((sa, sb)):
            if not live[h]:
                continue
            ids, dist, cnt = s.next_batch()
            done = s.lists_done()
            live[h] = bool(cnt.any())
            for i in range(4):
                if cnt[i]:
                    got[h][i].append((int(done[i]), ids[i, :cnt[i]].copy(), dist[i, :cnt[i]].copy()))
            if step % 2:
                gix.search(q, k=50, probes=5)
            else:
                table.exact_topk(pv.L2_SQUARED, q, 30)
            step += 1
    sa.close()
    sb.close()
    table.free()
    for h in range(2):
        for i in range(4):
            assert len(got[h][i]) == len(alone[h][i])
            for (d1, i1, x1), (d2, i2, x2) in zip(got[h][i], alone[h][i]):
                assert d1 == d2 and np.array_equal(i1, i2) and np.array_equal(x1, x2)


def test_replace_list_between_calls_is_refused(pv):
    rng = np.random.default_rng(9)
    dim, lists = 8, 4
    centers = rng.standard_normal((lists, dim)).astype(np.float32)
    rows = rng.standard_normal((200, dim)).astype(np.float32)
    off = np.array([0, 50, 100, 150, 200], dtype=np.int64)
    gix = pv.IvfflatIndex("vector_l2_ops", dim, lists).load(centers, off, rows, np.arange(200, dtype=np.int64))
    q = rng.standard_normal((3, dim)).astype(np.float32)
    s = gix.iterative_scan(q, probes=1, max_probes=lists, page=5)
    s.next_batch()
    new_rows = rng.standard_normal((7, dim)).astype(np.float32)
    gix.replace_list(2, new_rows, np.arange(1000, 1007, dtype=np.int64))
    with pytest.raises(pv.VecB200Error) as e:
        s.next_batch()
    assert e.value.code == -5 and "index changed since the scan began" in str(e.value)
    s.close()
    assert s.h is None
    with gix.iterative_scan(q, probes=1, max_probes=lists, page=5) as s2:
        seen = set()
        for i in range(3):
            seen |= {t for t, _ in s2.tuples_of(i)}
    assert set(range(1000, 1007)) <= seen and not (set(range(100, 150)) & seen)
    gix.free()


def test_argument_errors(pv, indexes):
    gix, _, q = indexes["vector_l2_ops"]
    for probes, max_probes, page in ((0, 2, 10), (1, 0, 10), (1, 2, 0), (1, 2, 2049)):
        with pytest.raises(pv.VecB200Error) as e:
            pv.IvfflatScan(gix, q, probes, max_probes, page)
        assert e.value.code == -1 and "vb_ivf_scan_begin" in str(e.value)
    with pytest.raises(pv.VecB200Error) as e:
        gix.iterative_scan(None, probes=1, max_probes=2, page=10)
    assert e.value.code == -1 and "NULL" in str(e.value)
    empty = pv.IvfflatIndex("vector_l2_ops", q.shape[1], 4)
    with pytest.raises(pv.VecB200Error) as e:
        empty.iterative_scan(q, probes=1, page=10)
    assert e.value.code == -5 and "not loaded" in str(e.value)
    empty.free()
