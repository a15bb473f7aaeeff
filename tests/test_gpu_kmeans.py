"""GPU parity of the IVFFlat build path: nearest-centre assign (src/ivfbuild.c:161-219), Lloyd k-means
with the reference's centre rules (src/ivfkmeans.c:179-236, 246-485) and k-means++ seeding (:23-91)."""
import numpy as np
import pytest

import oracle as O
from tests.util import f32_to_half_bits, mixture

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def pv():
    import pgvector_b200 as pv
    pv.init(0)
    return pv


def _data(elem, n, dim, k, seed, unit=False):
    x, c = mixture(n, dim, k, seed=seed)
    if elem == O.BIT:
        return O.binary_quantize(O.VECTOR, x), O.binary_quantize(O.VECTOR, c)
    if elem == O.HALFVEC:
        x, c = f32_to_half_bits(x), f32_to_half_bits(c)
    if unit:
        x, c = O.l2_normalize(elem, x), O.l2_normalize(elem, c)
    return x, c


def _assign_agreement(elem, metric, rows, centers, got, dim=None):
    want = O.ivf_assign(elem, metric, rows, centers, threads=8, dim=dim)
    diff = np.nonzero(got != want)[0]
    # any disagreement must be a genuine fp32 near-tie between the two chosen centres
    for i in diff[:50]:
        d_g = O.distance(elem, metric, rows[i], centers[got[i]], dim=dim, f64=True)
        d_w = O.distance(elem, metric, rows[i], centers[want[i]], dim=dim, f64=True)
        assert abs(d_g - d_w) <= 1e-5 * max(abs(d_w), 1.0), (i, d_g, d_w)
    return 1.0 - len(diff) / len(want)


@pytest.mark.parametrize("tensor_cores", [False, True])
@pytest.mark.parametrize("elem,metric,n,dim,k", [
    (O.VECTOR, O.L2_SQUARED, 5000, 96, 37),
    (O.VECTOR, O.L2_SQUARED, 20000, 1536, 300),
    (O.VECTOR, O.NEG_IP, 6000, 64, 100),
    (O.HALFVEC, O.L2_SQUARED, 6000, 200, 129),
    (O.HALFVEC, O.NEG_IP, 4000, 768, 64),
    (O.VECTOR, O.L2_SQUARED, 3000, 3, 100),       # the reference's own test shape (3-d, lists=100): tiny margins
    (O.BIT, O.HAMMING, 5000, 1024, 50),
    (O.BIT, O.HAMMING, 3000, 52, 20),
])
def test_assign_matches_oracle(pv, tensor_cores, elem, metric, n, dim, k):
    if dim == 3:
        rng = np.random.default_rng(3)
        rows, centers = rng.random((n, 3)).astype(np.float32), rng.random((k, 3)).astype(np.float32)
    else:
        rows, centers = _data(elem, n, dim, k, seed=n + k, unit=(metric == O.NEG_IP))
    pv.set_tensor_cores(tensor_cores)
    try:
        t = pv.Table(elem, dim).append(rows)
        got = pv.assign(t, metric, centers)
        rechecked = pv.last_assign_rechecked()
    finally:
        pv.set_tensor_cores(True)
    agree = _assign_agreement(elem, metric, rows, centers, got, dim=dim)
    assert agree >= (1.0 if elem == O.BIT else 0.9995), agree
    if tensor_cores and elem != O.BIT and n >= 1024 and k >= 16:
        assert rechecked >= 0            # the tensor-core path ran
        assert rechecked <= 0.2 * n      # and only a minority of rows needed the exact kernel
    else:
        assert rechecked == -1


def test_assign_first_minimum_wins_on_exact_ties(pv):
    """duplicate centres: strict < keeps the first (src/ivfbuild.c:186-190)"""
    rng = np.random.default_rng(0)
    c = rng.standard_normal((40, 16)).astype(np.float32)
    centers = np.concatenate([c, c])          # centre i == centre i + 40
    rows = (c[rng.integers(0, 40, 3000)] + 0.01 * rng.standard_normal((3000, 16))).astype(np.float32)
    for tc in (False, True):
        pv.set_tensor_cores(tc)
        got = pv.assign(pv.Table(O.VECTOR, 16).append(rows), O.L2_SQUARED, centers)
        pv.set_tensor_cores(True)
        assert got.max() < 40
        assert np.array_equal(got, O.ivf_assign(O.VECTOR, O.L2_SQUARED, rows, centers))


@pytest.mark.parametrize("elem,km,dim,k,unit", [(O.VECTOR, O.L2, 24, 20, False), (O.HALFVEC, O.L2, 40, 16, False),
                                                (O.VECTOR, O.SPHERICAL, 32, 12, True), (O.BIT, O.HAMMING, 128, 10, False)])
def test_kmeans_matches_elkan_oracle_from_shared_centres(pv, elem, km, dim, k, unit):
    rows, _ = _data(elem, 4000, dim, k, seed=77, unit=unit)
    init = O.kmeans_pp_init(elem, km, rows, k, seed=5, dim=dim)
    want_c, want_a, want_it = O.kmeans(elem, km, rows, init, algo="elkan", dim=dim)
    t = pv.Table(elem, dim).append(rows)
    got_c, got_it = pv.kmeans(t, km, init)
    proc1 = {O.L2: O.L2_SQUARED, O.SPHERICAL: O.NEG_IP, O.HAMMING: O.HAMMING}[km]
    got_a = pv.assign(t, proc1, got_c)
    assert abs(got_it - want_it) <= 2
    # Hamming distances tie constantly; Elkan's bound updates and a dense Lloyd pass can settle equal-distance
    # samples on different (equally near) centres, so the bit case is held to a looser agreement
    assert (got_a == want_a).mean() > (0.97 if elem == O.BIT else 0.995)
    if elem == O.BIT:
        assert (np.unpackbits(got_c) != np.unpackbits(want_c)).mean() < 0.01
    elif elem == O.HALFVEC:
        a, b = got_c.view(np.float16).astype(np.float32), want_c.view(np.float16).astype(np.float32)
        assert np.allclose(a, b, rtol=2e-3, atol=2e-3)
    else:
        assert np.allclose(got_c, want_c, rtol=1e-4, atol=1e-4)
        if unit:
            assert np.allclose(np.linalg.norm(got_c, axis=1), 1.0, atol=1e-6)


def test_kmeans_single_iteration_centres_are_bit_identical_sums(pv):
    """one Lloyd step: per-cluster fp32 sums are accumulated in ascending sample order like SumCenters"""
    rows, _ = _data(O.VECTOR, 3000, 20, 8, seed=9)
    init = rows[:8].copy()
    got_c, it = pv.kmeans(pv.Table(O.VECTOR, 20).append(rows), O.L2, init, max_iter=1)
    want_c, _, _ = O.kmeans(O.VECTOR, O.L2, rows, init, max_iter=1, algo="lloyd")
    assert it == 1
    assert np.array_equal(got_c, want_c)


def test_kmeans_pp_init_picks_samples_and_spreads(pv):
    rows, true_c = _data(O.VECTOR, 5000, 16, 25, seed=13)
    t = pv.Table(O.VECTOR, 16).append(rows)
    c = pv.kmeans_pp_init(t, O.L2, 25, seed=1)
    # every centre is one of the samples
    for ci in c:
        assert np.any(np.all(rows == ci, axis=1))
    # D^2 seeding covers (almost) every mixture component
    owner = O.ivf_assign(O.VECTOR, O.L2_SQUARED, c, true_c)
    assert len(set(owner)) >= 20


def test_allreduce_hook_is_called_with_sums_counts_and_changes(pv):
    import torch
    rows, _ = _data(O.VECTOR, 2000, 8, 5, seed=3)
    calls = []

    def hook(ptr, count, dtype):
        calls.append((count, dtype))     # single process: identity reduction

    t = pv.Table(O.VECTOR, 8).append(rows)
    c1, it1 = pv.kmeans(t, O.L2, rows[:5].copy(), max_iter=3, allreduce=hook)
    c2, it2 = pv.kmeans(t, O.L2, rows[:5].copy(), max_iter=3)
    assert np.array_equal(c1, c2) and it1 == it2
    assert (5 * 8, 0) in calls and (5, 1) in calls and (1, 1) in calls


@pytest.mark.parametrize("elem,km,n,dim,k,unit", [(O.VECTOR, O.L2, 6000, 64, 60, False), (O.VECTOR, O.L2, 3000, 3, 100, False),
                                                  (O.HALFVEC, O.L2, 4000, 200, 40, False), (O.VECTOR, O.SPHERICAL, 4000, 48, 30, True),
                                                  (O.BIT, O.HAMMING, 4000, 256, 25, False)])
def test_kmeans_pp_picks_the_oracles_rows_from_shared_draws(pv, elem, km, n, dim, k, unit):
    """InitCenters (src/ivfkmeans.c:23-91): fed the same first row and the same RandomDouble() draws, the GPU seeding
    (distance scan + weight update + prefix sum + pick per round) chooses the same sample rows as the oracle's
    sequential loop.  A pick may differ only when the draw lands within rounding of a boundary of the cumulative
    weights (the GPU adds the doubles in scan order, the reference subtracts them one by one); every later pick then
    differs too, so the comparison is the common prefix."""
    if dim == 3:
        rows = np.random.default_rng(3).random((n, 3)).astype(np.float32)
    else:
        rows, _ = _data(elem, n, dim, k, seed=n + dim, unit=unit)
    rng = np.random.default_rng(k)
    first = int(rng.integers(0, n))
    u = rng.random(k - 1)
    want_c, want_p = O.kmeans_pp_init_draws(elem, km, rows, k, first, u, dim=dim)
    t = pv.Table(elem, dim).append(rows)
    got_c, got_p = pv.kmeans_pp_init_draws(t, km, k, first, u)
    same = got_p == want_p
    prefix = k if same.all() else int(np.argmin(same))
    assert prefix >= (k if elem != O.BIT else 1), (prefix, got_p[:prefix + 2], want_p[:prefix + 2])
    assert np.array_equal(got_c[:prefix], want_c[:prefix])
    if elem == O.BIT and prefix < k:
        # Hamming weights are small integers: equal cumulative sums are ordinary, and a draw exactly on a boundary is
        # resolved the same way by both ("choice <= 0" = first j with cum >= choice) -- a mismatch needs explaining
        j, a, b = prefix, int(got_p[prefix]), int(want_p[prefix])
        assert abs(a - b) <= 1, (j, a, b)


def test_assign_tolerance_grows_with_the_row_length(pv):
    """halfvec rows of 4000 dimensions (HNSW_MAX_DIM * 2, the ivfflat limit for halfvec, src/ivfflat.h:37-38 via
    halfvec.h): the split-bf16 product's accumulation error exceeds the 2^-13 constant of shorter rows, so the margin
    test must use the dimension-dependent bound -- tensor-core assign == exact fp32 assign == oracle."""
    n, dim, k = 4096, 4000, 64
    rng = np.random.default_rng(4000)
    c = rng.standard_normal((k, dim)).astype(np.float32)
    # rows sit between pairs of centres so best / second-best margins are small
    a, b = rng.integers(0, k, n), rng.integers(0, k, n)
    w = rng.random((n, 1)).astype(np.float32) * 0.02 + 0.49
    x = (w * c[a] + (1 - w) * c[b] + 0.05 * rng.standard_normal((n, dim))).astype(np.float32)
    rows, centers = f32_to_half_bits(x), f32_to_half_bits(c)
    t = pv.Table(O.HALFVEC, dim).append(rows)
    pv.set_tensor_cores(False)
    try:
        exact = pv.assign(t, O.L2_SQUARED, centers)
    finally:
        pv.set_tensor_cores(True)
    got = pv.assign(t, O.L2_SQUARED, centers)
    assert pv.last_assign_rechecked() >= 0
    assert np.array_equal(got, exact)
    assert _assign_agreement(O.HALFVEC, O.L2_SQUARED, rows, centers, got, dim=dim) >= 0.999


@pytest.mark.parametrize("law", ["mixture", "low_rank"])
def test_filtered_seeding_picks_exactly_what_the_full_pass_picks(pv, law):
    """k-means++ with the triangle-inequality and bf16 filters in front of the exact distances (option pp_filter):
    the weights are those of the full pass, so from the same draws the same rows are picked -- equal to the unfiltered
    GPU pass and to the oracle -- while most samples are never re-scored."""
    n, dim, k = 30000, 128, 96
    rng = np.random.default_rng(17)
    if law == "mixture":
        rows, _ = _data(O.VECTOR, n, dim, k, seed=5)
    else:
        frame = np.linalg.qr(rng.standard_normal((dim, 8)))[0].astype(np.float32)
        rows = (rng.standard_normal((n, 8)).astype(np.float32) @ frame.T + 0.02 * rng.standard_normal((n, dim))).astype(np.float32)
    first = int(rng.integers(0, n))
    u = rng.random(k - 1)
    t = pv.Table(O.VECTOR, dim).append(rows)
    try:
        pv.set_option("pp_filter", 0)
        c0, p0 = pv.kmeans_pp_init_draws(t, O.L2, k, first, u)
        assert pv.kmeans_pp_stats() == (0, 0, 0)
        pv.set_option("pp_filter", 2)
        c2, p2 = pv.kmeans_pp_init_draws(t, O.L2, k, first, u)
        skipped, stopped, exact = pv.kmeans_pp_stats()
    finally:
        pv.set_option("pp_filter", 1)
    assert np.array_equal(p2, p0) and np.array_equal(c2, c0)
    assert skipped + stopped + exact == n * (k - 1)
    assert exact < 0.5 * n * (k - 1), (skipped, stopped, exact)
    want_c, want_p = O.kmeans_pp_init_draws(O.VECTOR, O.L2, rows, k, first, u)
    assert np.array_equal(p2, want_p)
