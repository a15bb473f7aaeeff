"""The level-0 refine's per-row re-score rule (vb_list_tc.cu cta_refine_body, LIST): phase 1 re-scores the k smallest d~,
phase 2 the candidates with d~ - E_i <= (k-th exact distance), E_i the bound of the candidate's own row.  It must return
what the search returns without level 0 (option tc_level0 = 0) and what the per-query fp32 scan returns, while
re-scoring fewer rows than the global bound (d~ <= k-th d~ + 2 eps) would; and a few spike rows, which widen the
global bound of every query, must no longer make level 0 give up."""
import os

import numpy as np
import pytest

import oracle as O
from tests.test_gpu_headline import build, low_rank
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
    pv.set_option("tc_level0", 1)
    pv.set_option("scan_impl", int(os.environ.get("VB_TEST_SCAN_IMPL", "2")))


def search_arms(pv, ix, queries, k=K, probes=PROBES):
    """{1: (ids, dist, level-0 fallbacks, refine counters), 0: the same without level 0, "impl0": per-query scan}"""
    out = {}
    try:
        pv.set_option("scan_impl", 4)
        for l0 in (1, 0):
            pv.set_option("tc_level0", l0)
            f0 = ix.tc_level0_fallbacks()
            pv.tc_traffic(True, read=True)
            pv.tc_level0_rescored()
            i, d = ix.search(queries, k=k, probes=probes)
            pv.tc_traffic(False, read=True)
            out[l0] = (i, d, ix.tc_level0_fallbacks() - f0, pv.tc_level0_rescored())
        pv.set_option("tc_level0", 1)
        pv.set_option("scan_impl", 0)
        out["impl0"] = ix.search(queries, k=k, probes=probes)
    finally:
        pv.set_option("tc_level0", 1)
        pv.set_option("scan_impl", int(os.environ.get("VB_TEST_SCAN_IMPL", "2")))
    return out


def same(a, b):
    return np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1])


def rows_per_query(out):
    rescored, global_rule, queries = (int(v) for v in out[1][3])
    assert queries > 0, "the level-0 refine did not run"
    assert out[0][3][2] == 0, "level 0 off: its refine must not run"
    return rescored / queries, global_rule / queries


@pytest.mark.parametrize("law", ["rank16", "mixture"])
def test_rowbound_headline_matches_level1_and_the_oracle(pv, law):
    n = 100_000
    if law == "rank16":
        rows, queries = low_rank(n, DIM, 16, seed=3), low_rank(2048, DIM, 16, seed=4)
    else:
        rows, _ = mixture(n, DIM, LISTS, seed=3)
        queries, _ = mixture(2048, DIM, LISTS, seed=4)
    gix, oix = build(pv, rows, LISTS, seed=42)
    out = search_arms(pv, gix, queries)
    assert same(out[1], out[0]), law
    assert same(out[1], out["impl0"]), law
    wi, wd = oix.search_batch(queries[:512], PROBES, K, threads=os.cpu_count() or 8)
    assert np.allclose(out[1][1][:512], wd, rtol=RTOL, atol=0)
    assert_same_neighbours(out[1][0][:512], out[1][1][:512], wi, wd, RTOL, min_positional=0.999)
    new, old = rows_per_query(out)
    print(f"{law}: rows re-scored per query {new:.2f} (global bound: {old:.2f}), fallbacks {out[1][2]}")
    assert K <= new < old
    if law == "rank16":
        assert out[1][2] <= 2048 // 16


@pytest.mark.parametrize("opclass", ["vector_ip_ops", "halfvec_l2_ops", "halfvec_ip_ops"])
def test_rowbound_inner_product_and_halfvec(pv, opclass):
    elem = pv.HALFVEC if opclass.startswith("halfvec") else pv.VECTOR
    metric = O.NEG_IP if "_ip_" in opclass else O.L2_SQUARED
    rows = low_rank(40_000, DIM, 16, seed=5)
    queries = low_rank(1024, DIM, 16, seed=6)
    if elem == pv.HALFVEC:
        rows, queries = rows.astype(np.float16).astype(np.float32), queries.astype(np.float16).astype(np.float32)
    lists = 64
    rng = np.random.default_rng(1)
    centers = rows[rng.choice(len(rows), lists, replace=False)].copy()
    assign = O.ivf_assign(O.VECTOR, metric, rows, centers, threads=os.cpu_count() or 8)
    grouped, ids, offsets = build_ivf_arrays(rows, assign, lists)
    if elem == pv.HALFVEC:
        ix = pv.IvfflatIndex(opclass, DIM, lists).load(centers.astype(np.float16).view(np.uint16), offsets,
                                                         grouped.astype(np.float16).view(np.uint16), ids)
        q = queries.astype(np.float16).view(np.uint16)
    else:
        ix = pv.IvfflatIndex(opclass, DIM, lists).load(centers, offsets, grouped, ids)
        q = queries
    out = search_arms(pv, ix, q, probes=8)
    assert same(out[1], out[0]), opclass
    assert same(out[1], out["impl0"]), opclass
    new, old = rows_per_query(out)
    assert new <= old, opclass


def test_rowbound_spike_rows_widen_only_their_own_bound(pv):
    """a handful of rows with one spike coordinate, sized to double the table's largest int8 residual: the global bound
    of every query doubles, and only the spike rows' own bounds widen.  Level 0 still certifies nearly every query,
    with the oracle's results."""
    rng = np.random.default_rng(17)
    rows = low_rank(30_000, DIM, 16, seed=13)
    amax = np.abs(rows).max(axis=1)
    sx = amax / 127.0
    res = np.sqrt(((rows - sx[:, None] * np.clip(np.rint(rows / sx[:, None]), -127, 127)) ** 2).sum(1))
    spikes = rng.choice(len(rows), 6, replace=False)
    # a spike of height S quantises the rest of its row with step S / 127, so its residual grows about linearly with S:
    # measure it at a trial height and scale that to twice the table's largest residual
    trial = rows[spikes[0]].copy()
    trial[0] = 20.0 * amax.max()
    st = abs(trial[0]) / 127.0
    r_trial = np.sqrt(((trial - st * np.clip(np.rint(trial / st), -127, 127)) ** 2).sum())
    height = trial[0] * 2.0 * res.max() / r_trial
    rows[spikes, rng.integers(0, DIM, len(spikes))] = height
    queries = low_rank(1024, DIM, 16, seed=14)
    ix, oix = build(pv, rows, 32, seed=5)
    out = search_arms(pv, ix, queries, probes=6)
    assert out[1][2] <= len(queries) // 8, out[1][2]
    assert same(out[1], out[0])
    wi, wd = oix.search_batch(queries, 6, K, threads=os.cpu_count() or 8)
    assert np.allclose(out[1][1], wd, rtol=RTOL, atol=1e-6)
    assert_same_neighbours(out[1][0], out[1][1], wi, wd, RTOL, min_positional=0.999)
