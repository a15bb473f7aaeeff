"""Filter level 0 of the batched IVFFlat list scan (int8 rows and queries, vb_list_tc.cu list_tc_l0_kernel): at the
headline shape it must return bit for bit what the search returns without it (option tc_level0 = 0) and what the
per-query fp32 scan returns, for both laws bench.py reports, L2 and inner product, vector and halfvec rows.  Rows that
make its bound useless (one dominant coordinate, huge norms) and near-duplicate sets larger than its k' make level 0
fail for some or all queries of a batch: only those queries are searched again, the others keep their certified
results, and the level-0 counter rises."""
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


def search_arms(pv, ix, queries, k=K, probes=PROBES, impls=(0,)):
    """(ids, dist, level-0 fallbacks, list-scan traffic counters) with level 0 on, with it off, and the per-query scans
    of `impls`"""
    out = {}
    try:
        pv.set_option("scan_impl", 4)
        for l0 in (1, 0):
            pv.set_option("tc_level0", l0)
            f0 = ix.tc_level0_fallbacks()
            pv.tc_traffic(True, read=True)
            i, d = ix.search(queries, k=k, probes=probes)
            out[l0] = (i, d, ix.tc_level0_fallbacks() - f0, pv.tc_traffic(False, read=True))
        pv.set_option("tc_level0", 1)
        for impl in impls:
            pv.set_option("scan_impl", impl)
            out["impl%d" % impl] = ix.search(queries, k=k, probes=probes)
    finally:
        pv.set_option("tc_level0", 1)
        pv.set_option("scan_impl", int(os.environ.get("VB_TEST_SCAN_IMPL", "2")))
    return out


def same(a, b):
    return np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1])


def assert_level0_ran(out):
    """the level-0 arm really scanned at level 0: without fallbacks its launch read exactly half the distinct row bytes
    of the level-1 arm's (1 byte per element instead of 2, same tiles); with fallbacks, the re-run added launches"""
    t0, t1 = out[1][3], out[0][3]
    if out[1][2] == 0:
        assert t0[3] == t1[3] and 2 * t0[1] == t1[1], (t0, t1)
    else:
        assert t0[3] > t1[3], (t0, t1)


@pytest.fixture(scope="module", params=["rank16", "mixture"])
def headline(request, pv):
    n = 100_000
    if request.param == "rank16":
        rows, queries = low_rank(n, DIM, 16, seed=3), low_rank(2048, DIM, 16, seed=4)
    else:
        rows, _ = mixture(n, DIM, LISTS, seed=3)
        queries, _ = mixture(2048, DIM, LISTS, seed=4)
    gix, oix = build(pv, rows, LISTS, seed=42)
    return request.param, gix, oix, queries


def test_level0_headline_matches_level1_and_the_oracle(pv, headline):
    law, gix, oix, queries = headline
    out = search_arms(pv, gix, queries)
    assert_level0_ran(out)
    assert same(out[1], out[0]), law
    assert same(out[1], out["impl0"]), law
    wi, wd = oix.search_batch(queries[:512], PROBES, K, threads=os.cpu_count() or 8)
    assert np.allclose(out[1][1][:512], wd, rtol=RTOL, atol=0)
    assert_same_neighbours(out[1][0][:512], out[1][1][:512], wi, wd, RTOL, min_positional=0.999)
    if law == "rank16":
        assert out[1][2] <= 2048 // 16, "level 0 certifies nearly every query of this law"


@pytest.mark.parametrize("opclass", ["vector_ip_ops", "halfvec_l2_ops", "halfvec_ip_ops"])
def test_level0_inner_product_and_halfvec(pv, opclass):
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
    assert_level0_ran(out)
    assert same(out[1], out[0]), opclass
    assert same(out[1], out["impl0"]), opclass


def test_level0_dominant_coordinate_rows_fail_and_are_repaired(pv):
    """rows with one huge coordinate: the int8 residual of the others is of the order of the distances, every query fails
    level 0, and the search still returns the level-1 results"""
    rng = np.random.default_rng(9)
    rows = low_rank(30_000, DIM, 16, seed=7)
    spikes = rng.choice(len(rows), 300, replace=False)
    rows[spikes, rng.integers(0, DIM, 300)] = 1e4
    rows[rng.choice(len(rows), 50, replace=False)] = 0.0                   # zero rows
    rows[rng.choice(len(rows), 50, replace=False)] *= 1e3                  # large norms
    queries = low_rank(600, DIM, 16, seed=8)
    ix, oix = build(pv, rows, 32, seed=2)
    out = search_arms(pv, ix, queries, probes=6)
    assert out[1][2] > 0, "level 0 must fail here"
    assert same(out[1], out[0])
    wi, wd = oix.search_batch(queries, 6, K, threads=os.cpu_count() or 8)
    assert np.allclose(out[1][1], wd, rtol=RTOL, atol=1e-6)


@pytest.mark.parametrize("dim", [1536, 2000])
def test_level0_partial_failure_repairs_only_the_failed_queries(pv, dim):
    """clusters of 200 near-duplicates (more than level 0's k' = 128 inside its bound) beside ordinary rows: the queries
    aimed at a cluster fail level 0 and are searched again; the others stay certified at level 0.  The results equal
    the search without level 0 bit for bit, and the oracle's within tolerance."""
    rng = np.random.default_rng(dim)
    base = rng.standard_normal((8, dim)).astype(np.float32)
    dirs = rng.standard_normal((8, dim)).astype(np.float32)
    dirs /= np.linalg.norm(dirs, axis=1, keepdims=True)
    steps = (np.linalg.norm(base, axis=1) * 2e-3)[:, None, None] * np.arange(1, 201, dtype=np.float32)[None, :, None]
    dups = (base[:, None, :] + steps * dirs[:, None, :]).reshape(-1, dim)
    filler = low_rank(20_000, dim, 16, seed=dim + 1) * 3.0
    rows = np.concatenate([dups, filler]).astype(np.float32)
    queries = np.concatenate([base + 1e-3 * rng.standard_normal((8, dim)).astype(np.float32),
                              low_rank(500, dim, 16, seed=dim + 2) * 3.0]).astype(np.float32)
    ix, oix = build(pv, rows, 24, seed=4)
    out = search_arms(pv, ix, queries, probes=4)
    assert 0 < out[1][2] < len(queries), "some, not all, queries must fail level 0"
    assert same(out[1], out[0])
    wi, wd = oix.search_batch(queries, 4, K, threads=os.cpu_count() or 8)
    assert np.allclose(out[1][1], wd, rtol=RTOL, atol=1e-6)


def test_level0_device_search_repairs_in_place(pv):
    """search_into (device queries and results) with failed queries: the repaired rows land at their own positions"""
    import torch
    rng = np.random.default_rng(21)
    rows = low_rank(30_000, DIM, 16, seed=11)
    rows[rng.choice(len(rows), 200, replace=False), rng.integers(0, DIM, 200)] = 5e3
    queries = low_rank(700, DIM, 16, seed=12)
    ix, _ = build(pv, rows, 32, seed=3)
    dev = torch.device("cuda", 0)
    q = torch.from_numpy(queries).to(dev)
    got = {}
    try:
        pv.set_option("scan_impl", 4)
        for l0 in (1, 0):
            pv.set_option("tc_level0", l0)
            i = torch.empty((len(queries), K), dtype=torch.int64, device=dev)
            d = torch.empty((len(queries), K), dtype=torch.float32, device=dev)
            f0 = ix.tc_level0_fallbacks()
            ix.search_into(q, K, 6, i, d)
            pv.synchronize()
            got[l0] = (i.cpu().numpy(), d.cpu().numpy(), ix.tc_level0_fallbacks() - f0)
    finally:
        pv.set_option("tc_level0", 1)
        pv.set_option("scan_impl", int(os.environ.get("VB_TEST_SCAN_IMPL", "2")))
    assert got[1][2] > 0
    assert same(got[1], got[0])
