"""GPU parity at the HEADLINE SHAPE (BASELINE config B scaled in rows, not in dimension): 1536-d fp32 rows,
lists = 100, probes = 10, k = 10 through the tensor-core filter (scan_impl 4) at filter level 1 and level 2, on both
synthetic laws bench.py reports (intrinsic dimension 16, and SURVEY 8(d)'s isotropic Gaussian mixture), against the
oracle port of src/ivfscan.c:47-187 -- plus near-tie sets at dim 1536 and at IVFFLAT_MAX_DIM = 2000
(src/ivfflat.h:37) whose neighbour gaps sit around the certificate's error bound, where a wrong dimension term in
the bound (vb_list_tc.cu lc_make_bound) would certify wrong neighbours."""
import os

import numpy as np
import pytest

import oracle as O
from tests.util import assert_same_neighbours, build_ivf_arrays, mixture

pytestmark = pytest.mark.gpu
RTOL = 1e-5
DIM, LISTS, PROBES, K = 1536, 100, 10, 10


@pytest.fixture(scope="module")
def pv():
    import pgvector_b200 as pv
    pv.init(0)
    O.ivf_set_tie_mode(True)
    yield pv
    O.ivf_set_tie_mode(False)
    pv.set_option("scan_impl", int(os.environ.get("VB_TEST_SCAN_IMPL", "2")))
    pv.set_option("tc_level1", 1)


def low_rank(n, dim, latent, seed, noise=0.02, frame_seed=3):
    """bench.py's default law: x = Q z + noise * eps with Q a dim x latent orthonormal frame"""
    frame = np.linalg.qr(np.random.default_rng(frame_seed).standard_normal((dim, latent)))[0].astype(np.float32)
    rng = np.random.default_rng(seed)
    z = rng.standard_normal((n, latent)).astype(np.float32)
    return (z @ frame.T + noise * rng.standard_normal((n, dim)).astype(np.float32)).astype(np.float32)


def build(pv, rows, lists, seed):
    """k-means centres from the library itself (shared with the oracle), assignment by the oracle"""
    n, dim = rows.shape
    rng = np.random.default_rng(seed)
    samp = rows[rng.choice(n, min(n, lists * 50), replace=False)]
    t = pv.Table(pv.VECTOR, dim).append(samp)
    init = samp[rng.choice(len(samp), lists, replace=False)].copy()
    centers, _ = pv.kmeans(t, pv.L2, init, max_iter=20)
    t.free()
    assign = O.ivf_assign(O.VECTOR, O.L2_SQUARED, rows, centers, threads=os.cpu_count() or 8)
    grouped, ids, offsets = build_ivf_arrays(rows, assign, lists)
    gix = pv.IvfflatIndex("vector_l2_ops", dim, lists).load(centers, offsets, grouped, ids)
    oix = O.Ivf(O.VECTOR, O.L2_SQUARED, centers, offsets, grouped, ids)
    return gix, oix


@pytest.fixture(scope="module", params=["rank16", "mixture"])
def headline(request, pv):
    n = 100_000
    if request.param == "rank16":
        rows, queries = low_rank(n, DIM, 16, seed=3), low_rank(512, DIM, 16, seed=4)
    else:
        rows, _ = mixture(n, DIM, LISTS, seed=3)
        queries, _ = mixture(512, DIM, LISTS, seed=4)
    gix, oix = build(pv, rows, LISTS, seed=42)
    want = oix.search_batch(queries, PROBES, K, threads=os.cpu_count() or 8)
    return request.param, gix, oix, queries, want


@pytest.mark.parametrize("level", [1, 2])
def test_headline_shape_matches_oracle(pv, headline, level):
    law, gix, oix, queries, (wi, wd) = headline
    pv.set_option("scan_impl", 4)
    pv.set_option("tc_level1", 1 if level == 1 else 0)
    try:
        f0, l0 = gix.tc_fallbacks(), gix.tc_level1_fallbacks()
        ids, dist = gix.search(queries, k=K, probes=PROBES)
        exact_fallbacks, l1_fallbacks = gix.tc_fallbacks() - f0, gix.tc_level1_fallbacks() - l0
        lists, ldist = gix.scan_lists(queries, PROBES)
    finally:
        pv.set_option("tc_level1", 1)
        pv.set_option("scan_impl", int(os.environ.get("VB_TEST_SCAN_IMPL", "2")))
    assert np.allclose(dist, wd, rtol=RTOL, atol=0)
    assert_same_neighbours(ids, dist, wi, wd, RTOL, min_positional=0.999)
    assert exact_fallbacks == 0, "the filter must certify this workload (no exact re-run)"
    if level == 2:
        assert l1_fallbacks == 0
    if law == "rank16" and level == 1:
        assert l1_fallbacks == 0, "well separated neighbours certify at level 1"
    # GetScanLists at the same shape (centre table through the filter: 512 queries x 100 centres < 128 -> exact tiles;
    # either way the probed lists equal the oracle's)
    for i in range(0, 512, 37):
        wl, wld = oix.scan_lists(queries[i], PROBES)
        assert np.array_equal(lists[i], wl), i
        assert np.allclose(ldist[i], wld, rtol=RTOL)


def test_headline_shape_every_scan_kernel_agrees(pv, headline):
    """the five scan formulations return the same neighbours at 1536 dimensions (per-query LDG / TMA bulk kernels,
    list-major fp32, tensor-core filter); the filter re-scores with the per-query arithmetic: bit-identical to it"""
    law, gix, oix, queries, (wi, wd) = headline
    got = {}
    try:
        for impl in (0, 1, 3, 4):
            pv.set_option("scan_impl", impl)
            got[impl] = gix.search(queries[:256], k=K, probes=PROBES)
    finally:
        pv.set_option("scan_impl", int(os.environ.get("VB_TEST_SCAN_IMPL", "2")))
    for impl in (0, 1, 3, 4):
        assert np.allclose(got[impl][1], wd[:256], rtol=RTOL, atol=0), impl
        assert_same_neighbours(got[impl][0], got[impl][1], wi[:256], wd[:256], RTOL, min_positional=0.999)
    assert np.array_equal(got[4][1], got[0][1]) and np.array_equal(got[4][0], got[0][0])


@pytest.mark.parametrize("dim", [1536, 2000])
@pytest.mark.parametrize("gap", [3e-3, 1e-4, 1e-6])
def test_near_ties_at_long_rows(pv, dim, gap):
    """Clusters of near-duplicates: every query has ~40 candidates whose distances differ by `gap` relative -- above
    the level-1 bound (2^-7), between the two bounds, and below the level-2 bound (2^-12..).  Whatever level
    certifies (or none: exact re-run), ids and distances must equal the per-query fp32 scan bit for bit, and the
    oracle within tolerance.  dim = 2000 = IVFFLAT_MAX_DIM exercises the accumulation term of the bound."""
    rng = np.random.default_rng(dim + int(1 / gap))
    n_base, dup, lists = 60, 40, 12
    base = rng.standard_normal((n_base, dim)).astype(np.float32)
    # duplicates at geometrically spaced tiny offsets along one random direction per base vector
    dirs = rng.standard_normal((n_base, dim)).astype(np.float32)
    dirs /= np.linalg.norm(dirs, axis=1, keepdims=True)
    scale = (np.linalg.norm(base, axis=1) * gap)[:, None, None] * np.arange(1, dup + 1, dtype=np.float32)[None, :, None]
    rows = (base[:, None, :] + scale * dirs[:, None, :]).reshape(-1, dim).astype(np.float32)
    filler, _ = mixture(6000, dim, lists, seed=7)
    rows = np.concatenate([rows, filler]).astype(np.float32)
    perm = rng.permutation(len(rows))
    rows = rows[perm]
    centers = rows[rng.choice(len(rows), lists, replace=False)].copy()
    queries = (base[rng.integers(0, n_base, 300)] + 1e-3 * rng.standard_normal((300, dim))).astype(np.float32)
    assign = O.ivf_assign(O.VECTOR, O.L2_SQUARED, rows, centers, threads=os.cpu_count() or 8)
    grouped, ids, offsets = build_ivf_arrays(rows, assign, lists)
    gix = pv.IvfflatIndex("vector_l2_ops", dim, lists).load(centers, offsets, grouped, ids)
    oix = O.Ivf(O.VECTOR, O.L2_SQUARED, centers, offsets, grouped, ids)
    try:
        pv.set_option("scan_impl", 0)
        i0, d0 = gix.search(queries, k=K, probes=6)
        pv.set_option("scan_impl", 3)
        i3, d3 = gix.search(queries, k=K, probes=6)
        pv.set_option("scan_impl", 4)
        pv.set_option("tc_level1", 1)
        f0 = gix.tc_fallbacks()
        i1, d1 = gix.search(queries, k=K, probes=6)
        f1 = gix.tc_fallbacks()
        pv.set_option("tc_level1", 0)
        i2, d2 = gix.search(queries, k=K, probes=6)
        f2 = gix.tc_fallbacks()
    finally:
        pv.set_option("tc_level1", 1)
        pv.set_option("scan_impl", int(os.environ.get("VB_TEST_SCAN_IMPL", "2")))
    # A certified batch carries the re-scored distances = the per-query scan's arithmetic (impl 0), bit for bit; a batch
    # no level could certify (more near-duplicates than candidates kept: 40 > k' = 32 at level 2) is re-run on the
    # exact list-major kernel (impl 3), bit for bit.  Nothing else may come back.
    for name, (ii, dd), fell_back in (("level1", (i1, d1), f1 > f0), ("level2", (i2, d2), f2 > f1)):
        if fell_back:
            assert np.array_equal(dd, d3) and np.array_equal(ii, i3), name
        else:
            assert np.array_equal(dd, d0) and np.array_equal(ii, i0), name
    wi, wd = oix.search_batch(queries, 6, K, threads=os.cpu_count() or 8)
    for dd in (d0, d3):
        assert np.allclose(dd, wd, rtol=RTOL, atol=1e-9)
    if gap >= 1e-4:   # above fp32 summation noise the order is the oracle's too
        assert_same_neighbours(i0, d0, wi, wd, RTOL, min_positional=0.98, boundary=4)
        assert_same_neighbours(i3, d3, wi, wd, RTOL, min_positional=0.98, boundary=4)


@pytest.mark.parametrize("k,probes", [(10, 10), (1, 3), (40, 10), (24, 7)])
def test_refine_of_preselected_candidates_equals_the_slab_selecting_refine(pv, headline, k, probes):
    """The one-CTA-per-query refine selects the k' nearest from the slab minima itself (slab_select 1) or takes them from
    the full selection kernel (slab_select 0): both routes return bit for bit the same neighbours, distances, probe lists
    and counters at both filter levels, and where no batch fell back to the exact kernels, what the per-query LDG scan
    (scan_impl 0) returns.  Each route runs on a fresh copy of the index, so both start from the same filter-level state
    (a level-1 failure rests level 1 for the next batches of that index), and level 0 -- which needs slab minima -- is off."""
    law, gix, oix, queries, _ = headline
    out = {}
    try:
        pv.set_option("scan_impl", 0)
        want = gix.search(queries, k=k, probes=probes)
        pv.set_option("scan_impl", 4)
        pv.set_option("tc_level0", 0)
        for level1 in (1, 0):
            pv.set_option("tc_level1", level1)
            for slab in (1, 0):
                pv.set_option("slab_select", slab)
                ix = pv.IvfflatIndex("vector_l2_ops", DIM, LISTS).load(oix.centers, oix.offsets, oix.rows, oix.ids)
                ids, dist = ix.search(queries, k=k, probes=probes)
                lists, ldist = ix.scan_lists(queries[:300], probes)
                out[level1, slab] = (ids, dist, lists, ldist, ix.tc_fallbacks(), ix.tc_level1_fallbacks())
                ix.free()
    finally:
        pv.set_option("slab_select", 1)
        pv.set_option("tc_level0", 1)
        pv.set_option("tc_level1", 1)
        pv.set_option("scan_impl", int(os.environ.get("VB_TEST_SCAN_IMPL", "2")))
    for level1 in (1, 0):
        a, b = out[level1, 1], out[level1, 0]
        for x, y in zip(a[:4], b[:4]):
            assert np.array_equal(x, y), (level1, k, probes)
        assert a[4:] == b[4:]
        if a[4] == 0:
            assert np.array_equal(a[0], want[0]) and np.array_equal(a[1], want[1]), (level1, k, probes)


@pytest.mark.parametrize("k,probes", [(10, 10), (1, 3), (40, 20)])
def test_slab_selection_equals_the_full_selection(pv, headline, k, probes):
    """The filter's epilogue stores the minimum d~ of every 32-row slab; the k' nearest are then selected from the slabs
    whose minimum is under the k'-th smallest slab minimum (vb_scan.cu slab_select_kernel) instead of a radix selection
    over the whole candidate run.  Same candidates, same order: outputs are bit-identical, at both filter levels."""
    law, ix, oix, queries, _ = headline
    qs = queries[:300]
    out = {}
    try:
        pv.set_option("scan_impl", 4)
        for level1 in (1, 0):
            pv.set_option("tc_level1", level1)
            for slab in (0, 1):
                pv.set_option("slab_select", slab)
                f0 = ix.tc_fallbacks()
                out[(level1, slab)] = ix.search(qs, k=k, probes=probes) + (ix.tc_fallbacks() - f0,)
    finally:
        pv.set_option("slab_select", 1)
        pv.set_option("tc_level1", 1)
        pv.set_option("scan_impl", int(os.environ.get("VB_TEST_SCAN_IMPL", "2")))
    for level1 in (1, 0):
        i0, d0, f0 = out[(level1, 0)]
        i1, d1, f1 = out[(level1, 1)]
        assert np.array_equal(i0, i1) and np.array_equal(d0, d1) and f0 == f1


def test_selection_from_slab_minima_with_ties_by_the_thousand(pv):
    """5000 copies of one row: every slab minimum ties, more candidates qualify than the selection's buffer holds, and the
    flagged queries go through the full selection (the CTA-per-query kernel reports them as uncertified and the batch is
    repeated on the selection kernels) -- results still equal the exact scan's (ids by position order)"""
    rng = np.random.default_rng(11)
    dim = 64
    base = rng.standard_normal((3000, dim)).astype(np.float32)
    dup = np.repeat(base[:1], 5000, axis=0)
    rows = np.concatenate([dup, base])
    ix, oix = build(pv, rows, 4, seed=2)
    qs = np.concatenate([base[:1] + 0.01, base[5:105]]).astype(np.float32)     # 101 queries x 4 probes: a batched scan
    try:
        pv.set_option("scan_impl", 4)
        got_i, got_d = ix.search(qs, k=10, probes=4)
        pv.set_option("scan_impl", 3)
        want_i, want_d = ix.search(qs, k=10, probes=4)
    finally:
        pv.set_option("scan_impl", int(os.environ.get("VB_TEST_SCAN_IMPL", "2")))
    assert np.allclose(got_d, want_d, rtol=1e-5, atol=1e-6)
    # among exact ties the order is by position in the list; both paths apply it
    assert np.array_equal(got_i[1:], want_i[1:])
    assert set(got_i[0].tolist()) <= set(range(5000))
