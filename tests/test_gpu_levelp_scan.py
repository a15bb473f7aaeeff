"""The level-P list scan (vb_list_proj.cu lp_scan_kernel: one CTA per (list, 128-row table tile) unit, projected distances,
lower bounds and slab minima in one pass) on the layouts it has to get right: list boundaries off the 32-row slabs, lists
of 1 to 31 rows and empty lists, one list probed by every query of a batch (more queries than one staged chunk), r above
16 and r at its cap dim / 8 (the rows' tile then needs more than 48 KiB of shared memory), a batch of more than 131 072
(query, probe) pairs (the multi-kernel grouping) and a row filter.  Each case searches with level P (tc_levelp 1) and
without it (level 0) and must return the same ids and distances bit for bit, and level P must have run: no int8 filter
launch, or the queries it could not certify counted as its fallbacks."""
import os

import numpy as np
import pytest

import oracle as O
from tests.test_gpu_headline import low_rank
from tests.util import build_ivf_arrays

pytestmark = pytest.mark.gpu
# 250 k rows in 128 lists: level P pays for batches of up to ~1400 queries at r = 16 (ivf_levelp_pays)
DIM, LISTS, PROBES, K, NQ, N = 256, 128, 8, 10, 256, 250_000


@pytest.fixture(scope="module")
def pv():
    import pgvector_b200 as pv
    pv.init(0)
    O.ivf_set_tie_mode(True)
    yield pv
    O.ivf_set_tie_mode(False)
    pv.set_option("tc_levelp", 1)
    pv.set_option("scan_impl", int(os.environ.get("VB_TEST_SCAN_IMPL", "2")))


def centres_and_assign(pv, rows, lists, seed=42):
    """k-means centres from the library, assignment by the oracle (as tests/test_gpu_headline.py builds)"""
    n, dim = rows.shape
    rng = np.random.default_rng(seed)
    samp = rows[rng.choice(n, min(n, lists * 50), replace=False)]
    t = pv.Table(pv.VECTOR, dim).append(samp)
    init = samp[rng.choice(len(samp), lists, replace=False)].copy()
    centers, _ = pv.kmeans(t, pv.L2, init, max_iter=20)
    t.free()
    return centers, O.ivf_assign(O.VECTOR, O.L2_SQUARED, rows, centers, threads=os.cpu_count() or 8)


def load(pv, rows, centers, assign):
    grouped, ids, offsets = build_ivf_arrays(rows, assign, len(centers))
    return pv.IvfflatIndex("vector_l2_ops", rows.shape[1], len(centers)).load(centers, offsets, grouped, ids), offsets


def arms(pv, ix, queries, probes=PROBES, **kw):
    """{levelp: (ids, dist, level-P fallbacks, tensor-core filter launches)} with level P on and off"""
    out = {}
    try:
        pv.set_option("scan_impl", 2)
        for lp in (1, 0):
            pv.set_option("tc_levelp", lp)
            f0 = ix.tc_levelp_fallbacks()
            pv.tc_traffic(True, read=True)
            i, d = ix.search(queries, k=K, probes=probes, **kw)
            out[lp] = (i, d, ix.tc_levelp_fallbacks() - f0, int(pv.tc_traffic(False, read=True)[3]))
    finally:
        pv.set_option("tc_levelp", 1)
        pv.set_option("scan_impl", int(os.environ.get("VB_TEST_SCAN_IMPL", "2")))
    return out


def check(out, certified=True):
    assert np.array_equal(out[1][0], out[0][0])
    assert np.array_equal(out[1][1], out[0][1])
    assert out[0][3] > 0 and out[0][2] == 0                  # level 0 ran in the arm without level P
    assert out[1][3] == 0 or out[1][2] > 0, out[1][2:]      # level P ran (its failed queries re-run from level 0)
    if certified:
        assert out[1][2] == 0 and out[1][3] == 0, out[1][2:]


@pytest.fixture(scope="module")
def big(pv):
    """250 k rank-8 rows of dimension 256, k-means centres of 128 lists and the oracle's assignment"""
    rows, queries = low_rank(N, DIM, 8, seed=3), low_rank(NQ, DIM, 8, seed=4)
    centers, assign = centres_and_assign(pv, rows, LISTS)
    return rows, centers, assign, queries


def fresh(pv, big, assign=None):
    """an index of its own (a batch whose failures rest level P must not decide another case's route), with its level-P
    basis built (r = 16) by a first batch that every case checks"""
    rows, centers, a, queries = big
    ix, offsets = load(pv, rows, centers, a if assign is None else assign)
    check(arms(pv, ix, queries), certified=assign is None)
    return ix, offsets


def test_spread_batch(pv, big):
    _, offsets = fresh(pv, big)
    assert (offsets[1:-1] % 32 != 0).sum() > LISTS // 2   # most list boundaries fall inside a slab


def test_small_and_empty_lists(pv, big):
    rows, centers, assign, queries = big
    a = assign.copy()
    # lists 0 .. 30 keep 1 .. 31 of their rows, lists 31 .. 35 none: the rest go to lists 64 .. 99
    for l in range(36):
        members = np.flatnonzero(a == l)
        a[members[l + 1 if l < 31 else 0:]] = l + 64
    # the queries probe them
    d2 = ((queries[:, None, :] - centers[None, :, :]) ** 2).sum(-1)
    probed = np.argsort(d2, axis=1, kind="stable")[:, :PROBES]
    assert np.isin(probed, np.arange(31)).any() and np.isin(probed, np.arange(31, 36)).any()
    _, offsets = fresh(pv, big, a)
    sizes = np.diff(offsets)
    assert list(sizes[:31]) == list(range(1, 32)) and not sizes[31:36].any()


def test_one_list_probed_by_every_query(pv, big):
    _, centers, _, queries = big
    ix, _ = fresh(pv, big)
    rng = np.random.default_rng(21)
    # 512 queries about one centre (all probe its list: 528 queries in its group, 17 staged chunks) beside the spread batch
    near = (centers[5] + 0.01 * rng.standard_normal((512, DIM))).astype(np.float32)
    d2 = ((near[:, None, :] - centers[None, :, :]) ** 2).sum(-1)
    assert (d2.argmin(1) == 5).all()
    check(arms(pv, ix, np.concatenate([queries, near])), certified=False)


def test_more_pairs_than_one_grouping_kernel(pv, big):
    # 520 queries x 256 probes = 133 120 (query, probe) pairs: build_query_groups counts and scatters them in three
    # kernels.  With 1024 lists of ~244 rows a query's candidates keep the whole batch in one sub-batch (the
    # candidate-distance buffer stays under 1 GiB), where 128 lists would split it; the batch is the index's first, so
    # it pays with r taken at its cap and builds the basis itself.
    rows, _, _, _ = big
    centers, assign = centres_and_assign(pv, rows, 1024)
    ix, _ = load(pv, rows, centers, assign)
    check(arms(pv, ix, low_rank(520, DIM, 8, seed=22), probes=256), certified=False)


def test_filtered(pv, big):
    ix, _ = fresh(pv, big)
    rng = np.random.default_rng(23)
    allowed = np.sort(rng.choice(N, N // 3, replace=False)).astype(np.int64)
    with ix.filter(allowed) as f:
        check(arms(pv, ix, big[3], filter=f), certified=False)


@pytest.mark.parametrize("dim,latent", [(512, 24), (512, 40), (1024, 136)], ids=["r32", "r48", "r128-cap"])
def test_wide_projections(pv, dim, latent):
    # r = the smallest multiple of 16 holding 90 % of the energy: 32 and 48 for 24 and 40 latent directions; 136 of them in
    # 1024 dimensions need more than 112, so r = dim / 8 = 128 (83 KiB of rows' tile in shared memory)
    rows, queries = low_rank(80_000, dim, latent, seed=24), low_rank(NQ, dim, latent, seed=25)
    centers, assign = centres_and_assign(pv, rows, LISTS)
    ix, _ = load(pv, rows, centers, assign)
    check(arms(pv, ix, queries), certified=False)
