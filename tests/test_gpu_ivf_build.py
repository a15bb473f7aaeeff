"""CREATE INDEX ... USING ivfflat in one call (vb_ivf_build / vb_ivf_build_dev = ivfflatbuild, src/ivfbuild.c): the
image equals, bit for bit, what the separate entry points (k-means++ seeding, Lloyd, assign, load) give on the same samples
and draws; the cosine opclasses drop rows of norm 0 and store the others normalised; the reference's recall floors hold on
built indexes; and the image takes inserts, deletes, filters and scans like a loaded one.  The expected-array model the GPU
tests compare with is pinned by the tests at the top, which need no device."""
import numpy as np
import pytest

import oracle as O
from tests.util import build_ivf_arrays, f32_to_half_bits, mixture, recall_at_k

gpu = pytest.mark.gpu
EINVAL, ENODEVICE, ESTATE = -1, -2, -5


def expected_arrays(rows, ids, lists_of_row, lists):
    """tests.util.build_ivf_arrays over the indexed rows (list >= 0): (rows grouped, ids grouped, offsets, order), order =
    the call's row number at every image row"""
    kept = np.flatnonzero(lists_of_row >= 0)
    grouped, order, off = build_ivf_arrays(rows[kept], lists_of_row[kept], lists)
    return grouped, np.asarray(ids)[kept][order], off, kept[order]


# ------------------------------------------------------------------------------- anywhere

def test_expected_arrays_are_stable_inside_a_list_and_drop_skipped_rows():
    rows = np.arange(8, dtype=np.float32).reshape(8, 1)
    lists_of_row = np.array([2, 0, -1, 2, 0, 1, -1, 0], dtype=np.int32)
    grouped, ids, off, order = expected_arrays(rows, np.arange(100, 108), lists_of_row, 4)
    assert order.tolist() == [1, 4, 7, 5, 0, 3]
    assert off.tolist() == [0, 3, 4, 6, 6]
    assert ids.tolist() == [101, 104, 107, 105, 100, 103]
    assert grouped[:, 0].tolist() == [1, 4, 7, 5, 0, 3]
    # nothing skipped: the plain model
    grouped, ids, off, order = expected_arrays(rows, np.arange(8), np.array([1, 0, 1, 0, 1, 0, 1, 0], dtype=np.int32), 2)
    assert order.tolist() == [1, 3, 5, 7, 0, 2, 4, 6] and off.tolist() == [0, 4, 8]
    # every row skipped: an empty image
    grouped, ids, off, order = expected_arrays(rows, np.arange(8), np.full(8, -1, dtype=np.int32), 3)
    assert grouped.shape[0] == 0 and off.tolist() == [0, 0, 0, 0] and order.size == 0


def test_build_without_a_device_is_an_error():
    import torch
    if torch.cuda.is_available():
        pytest.skip("a device is visible")
    import pgvector_b200 as pv
    with pytest.raises(pv.VecB200Error) as e:
        pv.IvfflatIndex("vector_l2_ops", 4, 2).build(np.zeros((8, 4), np.float32), np.arange(8))
    assert e.value.code == ENODEVICE


# ------------------------------------------------------------------------------- on the GPU

@pytest.fixture(scope="module")
def pv():
    import pgvector_b200 as pv
    pv.init(0)
    return pv


def data(pv, opclass, n, dim, lists, seed, zeros=0):
    """rows of the opclass's element type; `zeros` of them (vector / halfvec) have norm 0"""
    elem = pv.OPCLASSES[opclass][0]
    x, _ = mixture(n, dim, lists, seed=seed)
    if zeros:
        x[np.random.default_rng(seed).choice(n, zeros, replace=False)] = 0
    if elem == O.HALFVEC:
        return f32_to_half_bits(x)
    if elem == O.BIT:
        return np.packbits(x > 0, axis=1)
    return x


def composed(pv, opclass, rows, dim, lists, sample_rows, first_row, u, seed):
    """the build from the separate entry points: (centres, lists of the rows with -1 for skipped ones, stored rows)"""
    elem, metric, normalize, km = pv.OPCLASSES[opclass]
    samples = rows[sample_rows]
    if km == pv.SPHERICAL:
        samples = samples[pv.vector_norm(samples, elem) > 0]
        samples = pv.l2_normalize(samples, elem)
    t = pv.Table(elem, dim).append(samples)
    init, _ = pv.kmeans_pp_init_draws(t, km, lists, first_row, u)
    centers, iters = pv.kmeans(t, km, init, seed=seed)
    stored, skip = rows, np.zeros(rows.shape[0], dtype=bool)
    if normalize:
        skip = ~(pv.vector_norm(rows, elem) > 0)
        stored = pv.l2_normalize(rows, elem)
    lists_of_row = pv.assign(pv.Table(elem, dim).append(stored), metric, centers)
    lists_of_row[skip] = -1
    return centers, lists_of_row, stored, iters


def same_image(pv, ix, twin, queries, lists, k=10):
    """ids and distances of search, of one query over all lists (row order inside lists), and of an iterative scan"""
    assert np.array_equal(ix.list_offsets(), twin.list_offsets())
    for probes in (1, 4):
        a, b = ix.search(queries, k, probes=probes), twin.search(queries, k, probes=probes)
        assert np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1], equal_nan=True), probes
    a, b = ix.scan_items(queries[0], np.arange(lists)), twin.scan_items(queries[0], np.arange(lists))
    assert a[2] == b[2] and np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1], equal_nan=True)
    for l in range(lists):
        assert np.array_equal(ix.scan_items(None, [l])[0], twin.scan_items(None, [l])[0]), l
    with ix.iterative_scan(queries[:16], probes=2, max_probes=5, page=30) as s, \
            twin.iterative_scan(queries[:16], probes=2, max_probes=5, page=30) as t:
        for _ in range(3):
            x, y = s.next_batch(), t.next_batch()
            for p, q in zip(x, y):
                assert np.array_equal(p, q, equal_nan=True)


CASES = [("vector_l2_ops", 20000, 96, 64), ("vector_ip_ops", 12000, 64, 40), ("vector_cosine_ops", 12000, 64, 40),
         ("halfvec_l2_ops", 12000, 200, 48), ("halfvec_cosine_ops", 12000, 72, 32), ("bit_hamming_ops", 12000, 1024, 24),
         ("bit_hamming_ops", 6000, 52, 16), ("vector_l2_ops", 6000, 3, 50)]


@gpu
@pytest.mark.parametrize("opclass,n,dim,lists", CASES)
def test_build_equals_the_composition_of_the_entry_points(pv, opclass, n, dim, lists):
    import torch
    elem, metric, normalize, km = pv.OPCLASSES[opclass]
    zeros = 25 if elem != O.BIT and km == pv.SPHERICAL else 0
    rows = data(pv, opclass, n, dim, lists, seed=n + dim, zeros=zeros)
    ids = np.arange(n, dtype=np.int64) * 3 + 11
    rng = np.random.default_rng(dim)
    sample_rows = rng.permutation(n)[:max(20 * lists, 2000)]
    if zeros:   # some of the rows of norm 0 are samples
        sample_rows[:5] = np.flatnonzero(pv.vector_norm(rows, elem) == 0)[:5]
        sample_rows = np.unique(sample_rows)[rng.permutation(np.unique(sample_rows).size)]
    first_row, u, seed = 17, rng.random(lists - 1), 9
    centers, want_lists, stored, want_iters = composed(pv, opclass, rows, dim, lists, sample_rows, first_row, u, seed)
    grouped, gids, off, order = expected_arrays(stored, ids, want_lists, lists)
    twin = pv.IvfflatIndex(opclass, dim, lists).load(centers, off, grouped, gids)
    queries = twin.prepare_query(data(pv, opclass, 48, dim, lists, seed=5))
    kw = dict(seed=seed, sample_rows=sample_rows, first_row=first_row, u=u)
    raw = rows if elem != O.HALFVEC else rows.view(np.float16)
    variants = [("host", rows, {}), ("host, 3 chunks and a ragged one", rows, dict(chunk_rows=n // 3 - 7)),
                ("device", torch.from_numpy(raw).cuda(), {})]
    for name, r, extra in variants:
        ix = pv.IvfflatIndex(opclass, dim, lists)
        got_lists, got_order, iters = ix.build(r, ids, **kw, **extra)
        assert iters == want_iters, name
        assert np.array_equal(ix.centers(), centers), name
        assert np.array_equal(got_lists, want_lists), (name, np.flatnonzero(got_lists != want_lists)[:5])
        assert len(ix) == order.size == n - int((want_lists < 0).sum())
        assert np.array_equal(got_order[:order.size], order) and np.all(got_order[order.size:] == -1), name
        same_image(pv, ix, twin, queries, lists)
        ix.free()
    twin.free()


@gpu
def test_exact_kernel_assign_gives_the_same_build(pv):
    rows = data(pv, "vector_l2_ops", 8000, 48, 32, seed=2)
    kw = dict(seed=4, sample_rows=np.arange(0, 8000, 4), first_row=3, u=np.random.default_rng(1).random(31))
    a = pv.IvfflatIndex("vector_l2_ops", 48, 32)
    la, oa, _ = a.build(rows, np.arange(8000), **kw)
    pv.set_tensor_cores(False)
    try:
        b = pv.IvfflatIndex("vector_l2_ops", 48, 32)
        lb, ob, _ = b.build(rows, np.arange(8000), **kw)
    finally:
        pv.set_tensor_cores(True)
    assert np.array_equal(la, lb) and np.array_equal(oa, ob) and np.array_equal(a.centers(), b.centers())


def _assign_agreement(elem, metric, rows, centers, got, dim=None):
    """the rule of tests/test_gpu_kmeans.py: a disagreement with the oracle must be an fp32 near-tie of the two centres"""
    want = O.ivf_assign(elem, metric, rows, centers, threads=8, dim=dim)
    diff = np.nonzero(got != want)[0]
    for i in diff[:50]:
        d_g = O.distance(elem, metric, rows[i], centers[got[i]], dim=dim, f64=True)
        d_w = O.distance(elem, metric, rows[i], centers[want[i]], dim=dim, f64=True)
        assert abs(d_g - d_w) <= 1e-5 * max(abs(d_w), 1.0), (i, d_g, d_w)
    return 1.0 - len(diff) / len(want)


@gpu
@pytest.mark.parametrize("opclass,dim,lists", [("vector_l2_ops", 24, 20), ("halfvec_l2_ops", 40, 16), ("vector_cosine_ops", 32, 12),
                                               ("bit_hamming_ops", 128, 10)])
def test_build_against_the_oracle(pv, opclass, dim, lists):
    elem, metric, normalize, km = pv.OPCLASSES[opclass]
    n = 6000
    rows = data(pv, opclass, n, dim, lists, seed=77)
    sample_rows = np.arange(0, n, 2)
    ix = pv.IvfflatIndex(opclass, dim, lists)
    rng = np.random.default_rng(5)
    first_row, u = int(rng.integers(0, sample_rows.size)), rng.random(lists - 1)
    got_lists, _, iters = ix.build(rows, np.arange(n), sample_rows=sample_rows, first_row=first_row, u=u)
    stored = O.l2_normalize(elem, rows) if normalize else rows
    samples = O.l2_normalize(elem, rows[sample_rows]) if km == O.SPHERICAL else rows[sample_rows]
    centers = ix.centers()
    agree = _assign_agreement(elem, metric, stored, centers, got_lists, dim=dim)
    assert agree >= (1.0 if elem == O.BIT else 0.9995), agree
    # Lloyd against Elkan from the shared seeding (the seeding itself is pinned against the oracle's by test_gpu_kmeans)
    t = pv.Table(elem, dim).append(samples)
    init, _ = pv.kmeans_pp_init_draws(t, km, lists, first_row, u)
    want_c, _, want_it = O.kmeans(elem, km, samples, init, algo="elkan", dim=dim)
    assert abs(iters - want_it) <= 2
    if elem == O.BIT:
        assert (np.unpackbits(centers) != np.unpackbits(want_c)).mean() < 0.01
    elif elem == O.HALFVEC:
        assert np.allclose(centers.view(np.float16).astype(np.float32), want_c.view(np.float16).astype(np.float32), rtol=2e-3, atol=2e-3)
    else:
        assert np.allclose(centers, want_c, rtol=1e-4, atol=1e-4)


@gpu
def test_duplicated_rows_go_to_the_first_nearest_list_in_call_order(pv):
    """strict < keeps the first minimum (src/ivfbuild.c:186-190): the bit rows of two patterns sit at equal Hamming
    distances from several centres, and every copy of a pattern lands in the lowest-numbered of its nearest lists"""
    rng = np.random.default_rng(4)
    patterns = np.packbits(rng.random((2, 64)) < 0.5, axis=1)
    rows = np.concatenate([patterns[rng.integers(0, 2, 400)], np.packbits(rng.random((400, 64)) < 0.5, axis=1)])
    ix = pv.IvfflatIndex("bit_hamming_ops", 64, 24)
    lists_of_row, order, _ = ix.build(rows, np.arange(800) + 1000, sample_rows=np.arange(300, 800), seed=2)
    centers = ix.centers()
    ties = 0
    for i in range(800):
        d = O.distance_batch(O.BIT, O.HAMMING, rows[i], centers, dim=64)
        assert lists_of_row[i] == int(np.argmin(d)), i   # (argmin returns the first minimum)
        ties += int((d == d.min()).sum() > 1)
    assert ties > 20 and len(ix) == 800
    for l in np.unique(lists_of_row):
        got = ix.scan_items(None, [l])[0]
        assert np.array_equal(got, np.flatnonzero(lists_of_row == l) + 1000)   # call order inside the list
    assert np.array_equal(order, np.argsort(lists_of_row, kind="stable"))


@gpu
@pytest.mark.parametrize("opclass", ["vector_cosine_ops", "halfvec_cosine_ops", "vector_ip_ops"])
def test_cosine_build_rules(pv, opclass):
    elem, metric, normalize, km = pv.OPCLASSES[opclass]
    n, dim, lists = 5000, 16, 16
    rows = data(pv, opclass, n, dim, lists, seed=31, zeros=60)
    zero = pv.vector_norm(rows, elem) == 0
    assert zero.sum() == 60
    ix = pv.IvfflatIndex(opclass, dim, lists)
    ids = np.arange(n, dtype=np.int64)
    sample_rows = np.concatenate([np.flatnonzero(zero)[:10], np.flatnonzero(~zero)[:1500]])
    lists_of_row, order, _ = ix.build(rows, ids, sample_rows=sample_rows, first_row=5, u=np.random.default_rng(2).random(lists - 1))
    # the centres come from unit samples whatever the opclass stores
    c = ix.centers()
    cf = c.view(np.float16).astype(np.float32) if elem == O.HALFVEC else c
    assert np.allclose(np.linalg.norm(cf, axis=1), 1.0, atol=2e-3 if elem == O.HALFVEC else 1e-6)
    if normalize:
        assert np.array_equal(lists_of_row == -1, zero) and len(ix) == n - 60
        stored = pv.l2_normalize(rows, elem)
    else:
        assert np.all(lists_of_row >= 0) and len(ix) == n
        stored = rows
    # the stored rows, read back as their inner products with the basis vectors (exact: one non-zero product per row)
    got = np.zeros((n, dim), dtype=np.float64)
    for j in range(dim):
        e = np.zeros(dim, dtype=np.float32)
        e[j] = 1
        i, d, cnt = ix.scan_items(f32_to_half_bits(e) if elem == O.HALFVEC else e, np.arange(lists))
        assert cnt == len(ix)
        got[i, j] = -d
    want = stored.view(np.float16).astype(np.float64) if elem == O.HALFVEC else stored.astype(np.float64)
    keep = lists_of_row >= 0
    assert np.array_equal(got[keep], want[keep])
    assert not got[~keep].any()


def _tap_data(elem, n, seed):
    rng = np.random.default_rng(seed)
    if elem == O.BIT:
        return np.packbits(rng.random((n, 56)) < 0.5, axis=1) & np.array([255] * 6 + [0xF0], np.uint8), 52
    x = rng.random((n, 3)).astype(np.float32)
    return (f32_to_half_bits(x) if elem == O.HALFVEC else x), 3


@gpu
@pytest.mark.parametrize("opclass", ["vector_l2_ops", "vector_cosine_ops", "halfvec_l2_ops", "halfvec_cosine_ops", "bit_hamming_ops"])
@pytest.mark.parametrize("device_rows", [False, True])
def test_recall_floors_of_the_reference_on_built_indexes(pv, opclass, device_rows):
    """test/t/003, 032, 035 (uniform 3-d, lists = 100, LIMIT 20, scaled to 20k rows; bit(52)): probes 1 >= 0.71, 10 >= 0.95,
    lists -> 1.00 (cosine 0.9925), with samples drawn by the library; 005: every indexed row finds itself at probes = 1"""
    import torch
    elem, metric, normalize, km = pv.OPCLASSES[opclass]
    n, lists, k = 20000, 100, 20
    rows, dim = _tap_data(elem, n, seed=3)
    queries, _ = _tap_data(elem, 20, seed=4)
    r = rows if not device_rows else torch.from_numpy(rows if elem != O.HALFVEC else rows.view(np.float16)).cuda()
    sets = []
    for seed in (1, 2):
        ix = pv.IvfflatIndex(opclass, dim, lists)
        lists_of_row, order, iters = ix.build(r, np.arange(n), seed=seed, n_samples=5000)
        assert 1 <= iters <= 500 and len(ix) == n
        sets.append(lists_of_row)
        q = ix.prepare_query(queries)
        stored = pv.l2_normalize(rows, elem) if normalize else rows
        exact = pv.Table(elem, dim).append(stored)
        ti, td = exact.exact_topk(metric, q, k)
        floors = ((1, 0.71), (10, 0.95), (lists, 0.9925 if normalize else 1.0)) if elem != O.BIT else ((lists, 1.0),)
        for probes, floor in floors:
            gi, gd = ix.search(q, k, probes=probes)
            # tie-aware: a returned row counts when it is no farther than the k-th true neighbour
            hit = np.mean([(np.isin(g, t) | (d <= dd[-1])).mean() for g, t, d, dd in zip(gi, ti, gd, td)])
            assert hit >= floor, (probes, hit)
            assert elem == O.BIT or probes != lists or recall_at_k(gi, ti) >= floor - 0.01
        # a row is in the list of its nearest centre, so probes = 1 finds it, at distance 0 (under the inner product a
        # stored row need not be its own nearest neighbour: rounded unit vectors differ in length)
        if not normalize:
            some = np.random.default_rng(seed).choice(n, 300, replace=False)
            gi, gd = ix.search(stored[some], 1, probes=1)
            assert np.all(gd[:, 0] == 0)
        ix.free()
    assert not np.array_equal(sets[0], sets[1])   # another seed, another sample set, other centres


@gpu
def test_library_drawn_samples_are_distinct_and_follow_the_seed(pv):
    """the draw is observable through the centres of a build with lists = n_samples and no Lloyd movement: with as many
    lists as samples, k-means++ picks every distinct sample once"""
    n, dim, lists = 3000, 8, 64
    rows = data(pv, "vector_l2_ops", n, dim, 16, seed=8)
    seen = []
    for seed in (1, 1, 2):
        ix = pv.IvfflatIndex("vector_l2_ops", dim, lists)
        ix.build(rows, np.arange(n), seed=seed, n_samples=lists, max_iter=1)
        c = ix.centers()
        picked = sorted(int(np.flatnonzero((rows == ci).all(axis=1))[0]) for ci in c if (rows == ci).all(axis=1).any())
        assert len(set(picked)) == lists   # (the rows are distinct, so a repeated draw would leave fewer centres than lists)
        seen.append((picked, c))
    assert np.array_equal(seen[0][1], seen[1][1]) and seen[0][0] == seen[1][0]
    assert seen[0][0] != seen[2][0]


@gpu
@pytest.mark.parametrize("n", [4 ** 6 + 3, 4 ** 6, 4 ** 6 - 1, 1500])
def test_a_draw_of_every_row_is_a_permutation_of_the_rows(pv, n):
    """n_samples = n: the draw, sorted, must be 0 .. n - 1, so the build equals the one given sample_rows = arange(n).  Just
    above a power of four the Feistel domain is almost four times n and most draws walk the cycle"""
    rows = data(pv, "vector_l2_ops", n, 8, 16, seed=n)
    a, b = pv.IvfflatIndex("vector_l2_ops", 8, 16), pv.IvfflatIndex("vector_l2_ops", 8, 16)
    la, oa, ia = a.build(rows, np.arange(n), seed=5, n_samples=n)
    lb, ob, ib = b.build(rows, np.arange(n), seed=5, sample_rows=np.arange(n))
    assert np.array_equal(a.centers(), b.centers()) and np.array_equal(la, lb) and np.array_equal(oa, ob) and ia == ib


FIRST_CALL = r"""
import sys
import numpy as np
import pgvector_b200 as pv
opclass, chunk_rows = sys.argv[1], int(sys.argv[2])
elem, metric, normalize, km = pv.OPCLASSES[opclass]
n, dim, lists = 3000, 24, 12
rng = np.random.default_rng(1)
rows = (rng.standard_normal((lists, dim))[rng.integers(0, lists, n)] + 0.3 * rng.standard_normal((n, dim))).astype(np.float32)
rows[::97] = 0
ids = np.arange(n, dtype=np.int64) * 5 + 2
ix = pv.IvfflatIndex(opclass, dim, lists)
lists_of_row, order, _ = ix.build(rows, ids, seed=3, chunk_rows=chunk_rows or None)   # the process's first library call
centers = ix.centers()
stored = pv.l2_normalize(rows, elem) if normalize else rows
want = pv.assign(pv.Table(elem, dim).append(stored), metric, centers)
if normalize:
    want[~(pv.vector_norm(rows, elem) > 0)] = -1
assert np.array_equal(lists_of_row, want)
kept = np.flatnonzero(want >= 0)
o = kept[np.argsort(want[kept], kind="stable")]
off = np.concatenate([[0], np.cumsum(np.bincount(want[kept], minlength=lists))]).astype(np.int64)
assert np.array_equal(order[:o.size], o) and np.array_equal(ix.list_offsets(), off)
twin = pv.IvfflatIndex(opclass, dim, lists).load(centers, off, np.ascontiguousarray(stored[o]), ids[o])
q = twin.prepare_query(rows[1:40])
for a, b in ((ix.search(q, 10, probes=3), twin.search(q, 10, probes=3)),
             (ix.scan_items(q[0], np.arange(lists))[:2], twin.scan_items(q[0], np.arange(lists))[:2])):
    assert np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1])
print("first call ok")
"""


@gpu
@pytest.mark.parametrize("opclass,chunk_rows", [("vector_l2_ops", 0), ("vector_l2_ops", 900), ("vector_cosine_ops", 0)])
def test_a_host_build_as_the_first_call_of_a_process(opclass, chunk_rows):
    """nothing has sized the library's pinned staging buffers before the build: the k-means' own uploads grow them between
    the build's passes over the host rows"""
    import os
    import subprocess
    import sys
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    r = subprocess.run([sys.executable, "-c", FIRST_CALL, opclass, str(chunk_rows)], cwd=root, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0 and "first call ok" in r.stdout, r.stdout[-2000:] + r.stderr[-4000:]


@gpu
def test_same_inputs_and_seed_give_the_same_build(pv):
    rows = data(pv, "halfvec_l2_ops", 9000, 40, 30, seed=6)
    out = []
    for _ in range(2):
        ix = pv.IvfflatIndex("halfvec_l2_ops", 40, 30)
        l, o, it = ix.build(rows, np.arange(9000), seed=7)
        out.append((ix.centers(), l, o, it))
        ix.free()
    for a, b in zip(*out):
        assert np.array_equal(a, b)


@gpu
def test_a_built_image_takes_inserts_deletes_filters_and_rebuilds(pv):
    opclass, n, dim, lists = "vector_l2_ops", 10000, 32, 40
    rows = data(pv, opclass, n, dim, lists, seed=12)
    ids = np.arange(n, dtype=np.int64) + 500
    ix = pv.IvfflatIndex(opclass, dim, lists)
    lists_of_row, order, _ = ix.build(rows, ids, seed=3)
    grouped, gids, off, _ = expected_arrays(rows, ids, lists_of_row, lists)
    twin = pv.IvfflatIndex(opclass, dim, lists).load(ix.centers(), off, grouped, gids)
    queries = data(pv, opclass, 48, dim, lists, seed=13)
    more = 1.2 * data(pv, opclass, 700, dim, lists, seed=14)
    assert np.array_equal(ix.insert(more, np.arange(700) + 10 ** 6), twin.insert(more, np.arange(700) + 10 ** 6))
    same_image(pv, ix, twin, queries, lists)
    gone = np.concatenate([ids[::7], np.arange(0, 700, 3) + 10 ** 6])
    assert ix.delete(gone) == twin.delete(gone) == gone.size
    same_image(pv, ix, twin, queries, lists)
    flt, tflt = ix.filter(ids[1::2]), twin.filter(ids[1::2])
    a, b = ix.search(queries, 10, probes=5, filter=flt), twin.search(queries, 10, probes=5, filter=tflt)
    assert np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1])

    # a rebuild on the same handle: handles made before it are refused, the second build's image answers
    scan = ix.iterative_scan(queries[:4], probes=2, max_probes=4, page=10)
    rows2 = data(pv, opclass, 4000, dim, lists, seed=15)
    lists2, _, _ = ix.build(rows2, np.arange(4000), seed=4)
    assert len(ix) == 4000
    with pytest.raises(pv.VecB200Error) as e:
        scan.next_batch()
    assert e.value.code == ESTATE
    scan.close()
    with pytest.raises(pv.VecB200Error) as e:
        ix.search(queries, 10, probes=5, filter=flt)
    assert e.value.code == ESTATE
    grouped, gids, off, _ = expected_arrays(rows2, np.arange(4000), lists2, lists)
    twin2 = pv.IvfflatIndex(opclass, dim, lists).load(ix.centers(), off, grouped, gids)
    same_image(pv, ix, twin2, queries, lists)

    # refused calls leave that image answering as before
    before = ix.search(queries, 10, probes=5)
    bad = [dict(rows=rows2[:lists - 1], ids=np.arange(lists - 1)),                                   # fewer rows than lists
           dict(rows=rows2, ids=None),                                                                # no heap ids
           dict(rows=rows2, ids=np.arange(4000), sample_rows=np.array([0, 1, 4000] + list(range(2, 60)))),   # out of range
           dict(rows=rows2, ids=np.arange(4000), sample_rows=np.array([5, 5] + list(range(6, 60)))),  # repeated
           dict(rows=rows2, ids=np.arange(4000), sample_rows=np.arange(lists - 1))]                  # fewer samples than lists
    import torch
    for kw in bad:
        r, i = kw.pop("rows"), kw.pop("ids")
        for r_ in (r, torch.from_numpy(r).cuda()):   # vb_ivf_build and vb_ivf_build_dev
            with pytest.raises(pv.VecB200Error) as e:
                ix.build(r_, i, **kw)
            assert e.value.code == EINVAL, kw
    zero_samples = np.zeros((4000, dim), np.float32)
    zero_samples[:lists - 1] = rows2[:lists - 1]
    cx = pv.IvfflatIndex("vector_cosine_ops", dim, lists)
    cx.build(rows2, np.arange(4000), seed=1)
    cbefore = cx.search(cx.prepare_query(queries), 10, probes=5)
    with pytest.raises(pv.VecB200Error) as e:
        cx.build(zero_samples, np.arange(4000), seed=1)
    assert e.value.code == EINVAL and "usable samples" in str(e.value)
    cafter = cx.search(cx.prepare_query(queries), 10, probes=5)
    assert np.array_equal(cbefore[0], cafter[0]) and np.array_equal(cbefore[1], cafter[1])
    after = ix.search(queries, 10, probes=5)
    assert np.array_equal(before[0], after[0]) and np.array_equal(before[1], after[1])
    same_image(pv, ix, twin2, queries, lists)
