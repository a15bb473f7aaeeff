"""INSERT and VACUUM on a resident IVFFlat image (vb_ivf_insert = InsertTuple / FindInsertPage, src/ivfinsert.c;
vb_ivf_delete = ivfflatbulkdelete, src/ivfvacuum.c): the lists the inserts choose, the stored order of every list, and
search outputs -- ids, distances and counters, for every scan implementation and filter level, and iterative scans --
bit for bit equal to those of a fresh load of the expected arrays, through the in-place re-pack of the tensor-core
planes, table growth, norm changes that move the certificates' bounds, and empty lists and images."""
import ctypes as C

import numpy as np
import pytest

import oracle as O
from tests.ivf_insert_oracle import insert_lists
from tests.util import assert_same_neighbours, build_ivf_arrays, f32_to_half_bits, mixture

pytestmark = pytest.mark.gpu
EINVAL, ESTATE = -1, -5


@pytest.fixture(scope="module")
def pv():
    import pgvector_b200 as pv
    pv.init(0)
    return pv


OPCLASSES = ["vector_l2_ops", "vector_ip_ops", "vector_cosine_ops", "halfvec_l2_ops", "halfvec_ip_ops", "halfvec_cosine_ops",
             "bit_hamming_ops"]


def small_image(pv, opclass, n=6000, dim=32, lists=128, seed=5):
    elem, metric, normalize, _ = pv.OPCLASSES[opclass]
    x, c = mixture(n, dim, lists, seed=seed)
    if normalize:
        x, c = O.l2_normalize(O.VECTOR, x), O.l2_normalize(O.VECTOR, c)
    if elem == O.HALFVEC:
        x, c = f32_to_half_bits(x), f32_to_half_bits(c)
    elif elem == O.BIT:
        x, c = np.packbits(x > 0, axis=1), np.packbits(c > 0, axis=1)
    assign = O.ivf_assign(elem, metric, x, c, dim=dim)
    grouped, ids, off = build_ivf_arrays(x, assign, lists)
    return pv.IvfflatIndex(opclass, dim, lists).load(c, off, grouped, ids), c, elem, metric, normalize


def new_rows(opclass, pv, m, dim, seed):
    elem, _, _, _ = pv.OPCLASSES[opclass]
    x, _ = mixture(m, dim, 128, seed=seed)
    x = 1.5 * x
    if elem == O.HALFVEC:
        return f32_to_half_bits(x)
    if elem == O.BIT:
        return np.packbits(x > 0, axis=1)
    return x


@pytest.mark.parametrize("opclass", OPCLASSES)
def test_insert_lists_are_the_support1_probe_and_find_insert_page(pv, opclass):
    ix, c, elem, metric, normalize = small_image(pv, opclass)
    dim, nid, n_clear = 32, 10 ** 6, 0
    for m, seed in ((1, 1), (7, 2), (300, 3)):
        x = new_rows(opclass, pv, m, dim, seed)
        stored = pv.l2_normalize(x, elem) if normalize else x
        want, _ = ix.scan_lists(stored, 1)
        got = ix.insert(x, np.arange(nid, nid + m))
        nid += m
        assert np.array_equal(got, want[:, 0]), (m, np.flatnonzero(got != want[:, 0])[:5])
        ref = insert_lists(elem, metric, stored, c, dim=dim)
        d = np.stack([O.distance_batch(elem, metric, r, c, dim=dim) for r in stored])
        two = np.sort(d, axis=1)[:, :2]
        clear = (two[:, 1] - two[:, 0]) > 1e-5 * np.maximum(np.abs(two).max(axis=1), 1e-30)
        assert np.array_equal(got[clear], ref[clear])
        n_clear += int(clear.sum())
    assert n_clear > 100


def test_nan_distance_to_centre_zero_stays_in_list_zero(pv):
    dim, lists = 4, 128
    rng = np.random.default_rng(0)
    c = rng.standard_normal((lists, dim)).astype(np.float32)
    c[0] = [3e38, 3e38, 0, 0]
    x = rng.standard_normal((2000, dim)).astype(np.float32)
    assign = O.ivf_assign(O.VECTOR, O.NEG_IP, x, c)
    grouped, ids, off = build_ivf_arrays(x, assign, lists)
    ix = pv.IvfflatIndex("vector_ip_ops", dim, lists).load(c, off, grouped, ids)
    for m in (1, 300):
        r = rng.standard_normal((m, dim)).astype(np.float32)
        r[0] = [3e38, -3e38, 1, 0]
        assert np.isnan(O.distance(O.VECTOR, O.NEG_IP, r[0], c[0]))
        want, _ = ix.scan_lists(r, 1)
        got = ix.insert(r, np.arange(10 ** 6, 10 ** 6 + m) + m)
        assert got[0] == 0
        assert np.array_equal(got[1:], want[1:, 0])
        # FindInsertPage where every distance is finite (near the overflow of the products with centre 0 the device's
        # and the oracle's summation orders may round to different infinities)
        d = np.stack([O.distance_batch(O.VECTOR, O.NEG_IP, x_, c) for x_ in r])
        fin = np.isfinite(d).all(axis=1)
        fin[0] = True
        assert np.array_equal(got[fin], insert_lists(O.VECTOR, O.NEG_IP, r, c)[fin])


# ------------------------------------------------------------------------------- identity with a fresh load

DIM, LISTS, N0 = 1536, 256, 100_000
SETTINGS = [(impl, l0, l1) for impl in (0, 2, 3, 4) for l0 in (0, 1) for l1 in (0, 1)]


class Model:
    """the expected arrays: rows and ids grouped by list, in stored order"""

    def __init__(self, centers, rows, ids, off, opclass="vector_l2_ops", dim=DIM, lists=LISTS):
        self.centers, self.rows, self.ids, self.off = centers, rows, ids, off
        self.opclass, self.dim, self.lists = opclass, dim, lists

    def labels(self):
        return np.repeat(np.arange(self.lists), np.diff(self.off))

    def insert(self, rows, ids, lists):
        lab = np.concatenate([self.labels(), lists])
        order = np.argsort(lab, kind="stable")
        self.rows = np.ascontiguousarray(np.concatenate([self.rows, rows])[order])
        self.ids = np.concatenate([self.ids, ids])[order]
        self.off = np.concatenate([[0], np.cumsum(np.bincount(lab, minlength=self.lists))]).astype(np.int64)

    def delete(self, ids):
        keep = ~np.isin(self.ids, ids)
        lab = self.labels()[keep]
        self.rows, self.ids = np.ascontiguousarray(self.rows[keep]), self.ids[keep]
        self.off = np.concatenate([[0], np.cumsum(np.bincount(lab, minlength=self.lists))]).astype(np.int64)
        return int((~keep).sum())

    def fresh(self, pv):
        return pv.IvfflatIndex(self.opclass, self.dim, self.lists).load(self.centers, self.off, self.rows, self.ids)


def outputs(pv, ix, queries, k=10, probes=8):
    out = []
    for impl, l0, l1 in SETTINGS:
        pv.set_option("scan_impl", impl)
        pv.set_option("tc_level0", l0)
        pv.set_option("tc_level1", l1)
        c0 = (ix.tc_fallbacks(), ix.tc_level1_fallbacks(), ix.tc_level0_fallbacks())
        for q in (queries, queries[:3]):
            i, d = ix.search(q, k, probes=probes)
            c1 = (ix.tc_fallbacks(), ix.tc_level1_fallbacks(), ix.tc_level0_fallbacks())
            out.append((i, d, tuple(b - a for a, b in zip(c0, c1)), ix.last_candidates()))
            c0 = c1
    pv.set_option("scan_impl", 2)
    pv.set_option("tc_level0", 1)
    pv.set_option("tc_level1", 1)
    with ix.iterative_scan(queries[:64], probes=2, max_probes=6, page=40) as s:
        for _ in range(4):
            i, d, n = s.next_batch()
            out.append((i.copy(), d.copy(), n.copy(), 0))
    return out


def assert_identical(pv, ix, model, queries, check_oracle=False):
    off = ix.list_offsets()
    assert np.array_equal(off, model.off)
    for l in range(model.lists):
        got, _, n = ix.scan_items(None, [l])
        assert n == off[l + 1] - off[l]
        assert np.array_equal(got, model.ids[off[l]:off[l + 1]]), l
    e = model.fresh(pv)
    try:
        a, b = outputs(pv, ix, queries), outputs(pv, e, queries)
    finally:
        e.free()
    for j, (x, y) in enumerate(zip(a, b)):
        assert np.array_equal(x[0], y[0]), j
        assert np.array_equal(x[1], y[1], equal_nan=True), j
        # With filter level 1 on, which level a batch starts at also depends on the image's search history (a level that
        # failed rests for the next 64 batches), which a fresh load does not share: there ids and distances must agree,
        # and the fallback counters and candidate counts are compared where level 1 is off.
        if j < 2 * len(SETTINGS) and SETTINGS[j // 2][2] == 0:
            assert np.array_equal(np.asarray(x[2]), np.asarray(y[2])) and x[3] == y[3], (j, x[2], y[2], x[3], y[3])
    if check_oracle and model.rows.shape[0]:
        oix = O.Ivf(O.VECTOR, O.L2_SQUARED, model.centers, model.off, model.rows, model.ids)
        wi, wd = oix.search_batch(queries[:64], 8, 10)
        assert_same_neighbours(a[0][0][:64], a[0][1][:64], wi, wd, rtol=1e-5)


@pytest.fixture(scope="module")
def big(pv):
    x, c = mixture(N0, DIM, LISTS, seed=21)
    assign = O.ivf_assign(O.VECTOR, O.L2_SQUARED, x, c, threads=8)
    grouped, ids, off = build_ivf_arrays(x, assign, LISTS)
    ids = ids * 7 + 3   # heap ids unlike row numbers
    q, _ = mixture(512, DIM, LISTS, seed=22)
    return Model(c, grouped, ids, off), q


def test_inserts_and_deletes_give_the_outputs_of_a_fresh_load(pv, big):
    m0, q = big
    model = Model(m0.centers, m0.rows.copy(), m0.ids.copy(), m0.off.copy())
    ix = model.fresh(pv)
    rng = np.random.default_rng(7)
    nid = [10 ** 9]

    def ins(rows):
        ids = np.arange(nid[0], nid[0] + rows.shape[0], dtype=np.int64)
        nid[0] += rows.shape[0]
        lists = ix.insert(rows, ids)
        model.insert(rows, ids, lists)
        return ids, lists

    def dele(ids):
        assert ix.delete(ids) == model.delete(ids)

    # before any batched search: no planes yet (and the first growth of a loaded table)
    ins(mixture(500, DIM, LISTS, seed=30)[0])
    assert_identical(pv, ix, model, q, check_oracle=True)
    # the planes and the int8 plane exist now: re-packed in place
    ins(mixture(300, DIM, LISTS, seed=31)[0])
    assert_identical(pv, ix, model, q)
    # past capacity, with planes: the table and the plane buffers grow
    ins(mixture(60_000, DIM, LISTS, seed=32)[0])
    assert_identical(pv, ix, model, q)
    # a row whose norm raises xmax / rmax, and deleting it again
    spike = (40 * model.rows[rng.integers(0, model.rows.shape[0])]).reshape(1, -1)
    sid, _ = ins(spike)
    assert_identical(pv, ix, model, q)
    dele(sid)
    assert_identical(pv, ix, model, q)
    # a row with an Inf norm (the filter's bound is lost: finite becomes false) and deleting it
    inf = np.full((1, DIM), 1e37, np.float32)
    iid, _ = ins(inf)
    assert_identical(pv, ix, model, q)
    dele(iid)
    assert_identical(pv, ix, model, q)
    # all rows into one list, and into the last list
    _, l1 = ins(np.repeat(model.centers[5:6], 50, axis=0))
    assert set(l1.tolist()) == {5}
    _, l2 = ins(np.repeat(model.centers[LISTS - 1:], 20, axis=0) + 1e-3)
    assert set(l2.tolist()) == {LISTS - 1}
    assert_identical(pv, ix, model, q)
    # deletes: absent ids, a whole list, random rows
    assert ix.delete(np.array([-5, 10 ** 12], np.int64)) == 0
    dele(model.ids[model.off[3]:model.off[4]].copy())
    dele(rng.choice(model.ids, 1000, replace=False))
    assert_identical(pv, ix, model, q, check_oracle=True)
    # insert after delete
    ins(mixture(700, DIM, LISTS, seed=33)[0])
    assert_identical(pv, ix, model, q)
    # everything, then an insert into the empty image
    dele(model.ids.copy())
    assert ix.list_offsets()[-1] == 0
    assert_identical(pv, ix, model, q[:64])
    ins(mixture(400, DIM, LISTS, seed=34)[0])
    assert_identical(pv, ix, model, q, check_oracle=True)
    ix.free()


def test_filters_and_scan_handles_made_before_a_change_are_refused(pv):
    ix, c, elem, metric, _ = small_image(pv, "vector_l2_ops")
    q = mixture(8, 32, 128, seed=9)[0]
    f = ix.filter(np.arange(100))
    s = ix.iterative_scan(q, probes=2, page=10)
    s.next_batch()
    ix.insert(new_rows("vector_l2_ops", pv, 5, 32, 4), np.arange(10 ** 6, 10 ** 6 + 5))
    with pytest.raises(pv.VecB200Error) as e:
        s.next_batch()
    assert e.value.code == ESTATE
    s.close()
    with pytest.raises(pv.VecB200Error) as e:
        ix.iterative_scan(q, probes=2, page=10, filter=f).next_batch()
    assert e.value.code == ESTATE
    f.free()
    f = ix.filter(np.arange(100))
    assert ix.delete(np.array([1, 2, 3])) == 3
    with pytest.raises(pv.VecB200Error) as e:
        ix.iterative_scan(q, probes=2, page=10, filter=f).next_batch()
    assert e.value.code == ESTATE
    f.free()


def test_refused_calls_leave_the_image_as_it_was(pv):
    L = pv.load()
    ix, c, elem, metric, _ = small_image(pv, "vector_l2_ops")
    q = mixture(300, 32, 128, seed=9)[0]
    before = ix.search(q, 10, probes=4)
    off = ix.list_offsets()
    x = new_rows("vector_l2_ops", pv, 4, 32, 4)
    ids = np.arange(4, dtype=np.int64)
    out = np.empty(4, np.int32)
    p = lambda a: a.ctypes.data_as(C.c_void_p)
    assert L.vb_ivf_insert(ix.h, p(x), None, 4, p(out)) == EINVAL
    assert L.vb_ivf_insert(ix.h, None, p(ids), 4, p(out)) == EINVAL
    assert L.vb_ivf_insert(ix.h, p(x), p(ids), -1, p(out)) == EINVAL
    assert L.vb_ivf_delete(ix.h, None, 3, None) == EINVAL
    assert L.vb_ivf_insert(ix.h, p(x), p(ids), 0, p(out)) == 0
    assert np.array_equal(ix.list_offsets(), off)
    after = ix.search(q, 10, probes=4)
    assert np.array_equal(before[0], after[0]) and np.array_equal(before[1], after[1])
    # an image that is not loaded, and one loaded without heap ids
    h = pv.IvfflatIndex("vector_l2_ops", 32, 128)
    assert L.vb_ivf_insert(h.h, p(x), p(ids), 4, p(out)) == ESTATE
    assert L.vb_ivf_delete(h.h, p(ids), 4, None) == ESTATE
    h.load(c, off, np.zeros((off[-1], 32), np.float32))
    assert L.vb_ivf_insert(h.h, p(x), p(ids), 4, p(out)) == ESTATE
    assert L.vb_ivf_delete(h.h, p(ids), 4, None) == ESTATE
    h.free()


def test_device_rows_and_cosine_zero_rows(pv):
    import torch
    ix, c, elem, metric, _ = small_image(pv, "vector_l2_ops")
    x = new_rows("vector_l2_ops", pv, 300, 32, 6)
    ids = np.arange(10 ** 6, 10 ** 6 + 300)
    want, _ = ix.scan_lists(x, 1)
    got = ix.insert(torch.from_numpy(x).cuda(), torch.from_numpy(ids).cuda())
    assert np.array_equal(got, want[:, 0])
    for l in np.unique(got):
        g, _, _ = ix.scan_items(None, [int(l)])
        assert np.array_equal(g[-int((got == l).sum()):], ids[got == l])
    cx, _, _, _, _ = small_image(pv, "vector_cosine_ops")
    x = new_rows("vector_l2_ops", pv, 6, 32, 7)
    x[2] = 0
    got = cx.insert(x, np.arange(6) + 10 ** 6)
    assert got[2] == -1 and (np.delete(got, 2) >= 0).all()
    assert cx.list_offsets()[-1] == 6000 + 5


@pytest.mark.parametrize("opclass", ["halfvec_l2_ops", "halfvec_ip_ops"])
def test_halfvec_inserts_and_deletes_repack_in_place(pv, opclass):
    """the halfvec packing paths of the in-place re-pack: planes and the int8 plane built, then changes whose first
    changed row lies inside the table (a non-zero start tile), compared with a fresh load bit for bit"""
    dim, lists, n = 96, 128, 30_000
    elem, metric, _, _ = pv.OPCLASSES[opclass]
    x, c = mixture(n, dim, lists, seed=41)
    x, c = f32_to_half_bits(x), f32_to_half_bits(c)
    assign = O.ivf_assign(elem, metric, x, c, dim=dim)
    grouped, ids, off = build_ivf_arrays(x, assign, lists)
    model = Model(c, grouped, ids.astype(np.int64) * 5 + 1, off, opclass=opclass, dim=dim, lists=lists)
    ix = model.fresh(pv)
    q = f32_to_half_bits(mixture(512, dim, lists, seed=42)[0])
    ix.search(q, 10, probes=8)          # builds the bf16 planes and the int8 plane
    nid = 10 ** 9
    for m, seed in ((2000, 43), (40, 44)):   # the first grows table and plane buffers, the second re-packs from its tile
        rows = f32_to_half_bits(mixture(m, dim, lists, seed=seed)[0])
        new_ids = np.arange(nid, nid + m, dtype=np.int64)
        nid += m
        model.insert(rows, new_ids, ix.insert(rows, new_ids))
        assert_identical(pv, ix, model, q)
    victims = np.random.default_rng(45).choice(model.ids[model.off[lists // 2]:], 300, replace=False)
    assert ix.delete(victims) == model.delete(victims)
    assert_identical(pv, ix, model, q)
    ix.free()
