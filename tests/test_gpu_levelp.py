"""Filter level P of the batched IVFFlat list scan (vb_list_proj.cu: a lower bound from the rows' projection on their
principal directions, in front of level 0).  On a low-rank law it must return bit for bit what the search returns
without it (option tc_levelp = 0), read no int8 plane (no tensor-core filter launch) and certify every query; on an
isotropic law no basis holds 90 % of the energy and level 0 runs as before; where near-duplicate sets outnumber its k'
the queries it cannot certify are searched again from level 0 and still match; after inserts and deletes, under row filters
and with non-finite rows (the exact path, in both arms) it still matches the search without it; and where a batch is too
small for it to pay, or the tensor-core filter is asked for (scan_impl 4), level 0 runs."""
import os

import numpy as np
import pytest

import oracle as O
from tests.test_gpu_headline import build, low_rank

pytestmark = pytest.mark.gpu
# (NQ queries over 70 k - 80 k rows in 128 lists: level P pays -- the int8 bytes it saves, taken at r = dim / 8 before the
# basis exists, exceed the rows its refine adds: ivf_levelp_pays)
DIM, LISTS, PROBES, K, NQ = 256, 128, 8, 10, 256


@pytest.fixture(scope="module")
def pv():
    import pgvector_b200 as pv
    pv.init(0)
    O.ivf_set_tie_mode(True)
    yield pv
    O.ivf_set_tie_mode(False)
    pv.set_option("tc_levelp", 1)
    pv.set_option("scan_impl", int(os.environ.get("VB_TEST_SCAN_IMPL", "2")))


def arms(pv, ix, queries, **kw):
    """{levelp: (ids, dist, level-P fallbacks, tensor-core filter launches)} with level P on and off"""
    out = {}
    try:
        pv.set_option("scan_impl", 2)
        for lp in (1, 0):
            pv.set_option("tc_levelp", lp)
            f0 = ix.tc_levelp_fallbacks()
            pv.tc_traffic(True, read=True)
            i, d = ix.search(queries, k=K, probes=PROBES, **kw)
            out[lp] = (i, d, ix.tc_levelp_fallbacks() - f0, int(pv.tc_traffic(False, read=True)[3]))
    finally:
        pv.set_option("tc_levelp", 1)
        pv.set_option("scan_impl", int(os.environ.get("VB_TEST_SCAN_IMPL", "2")))
    return out


def assert_same(out):
    assert np.array_equal(out[1][0], out[0][0])
    assert np.array_equal(out[1][1], out[0][1])


@pytest.fixture(scope="module")
def lowrank(pv):
    rows, queries = low_rank(80_000, DIM, 8, seed=3), low_rank(NQ, DIM, 8, seed=4)
    gix, oix = build(pv, rows, LISTS, seed=42)
    return rows, gix, queries


def test_low_rank_matches_level0_without_the_int8_plane(pv, lowrank):
    _, gix, queries = lowrank
    out = arms(pv, gix, queries)
    assert_same(out)
    assert out[1][2] == 0 and out[1][3] == 0, out[1][2:]   # every query certified at level P, no int8 scan
    assert out[0][3] > 0


def test_isotropic_law_builds_no_level_p(pv):
    rng = np.random.default_rng(5)
    rows = rng.standard_normal((80_000, DIM)).astype(np.float32)
    queries = rng.standard_normal((NQ, DIM)).astype(np.float32)
    gix, _ = build(pv, rows, LISTS, seed=42)
    out = arms(pv, gix, queries)
    assert_same(out)
    assert out[1][3] > 0 and out[1][2] == 0   # level 0 ran as without level P


def test_failed_queries_cascade_into_level0(pv):
    rows, queries = low_rank(70_000, DIM, 8, seed=6), low_rank(NQ, DIM, 8, seed=7)
    rng = np.random.default_rng(8)
    # 300 rows within the bound's slack of each of the first 16 queries: their 128 smallest bounds cannot separate them
    dup = np.concatenate([q + 0.02 * rng.standard_normal((300, DIM)).astype(np.float32) for q in queries[:16]])
    rows = np.concatenate([rows, dup]).astype(np.float32)
    gix, _ = build(pv, rows, LISTS, seed=42)
    out = arms(pv, gix, queries)
    assert_same(out)
    assert 0 < out[1][2] < len(queries), out[1][2]


def test_insert_delete_keep_the_plane_current(pv):
    rows, queries = low_rank(80_000, DIM, 8, seed=14), low_rank(NQ, DIM, 8, seed=15)
    gix, _ = build(pv, rows, LISTS, seed=42)
    arms(pv, gix, queries)                                   # the level-P image exists before the change
    gix.insert(low_rank(3000, DIM, 8, seed=11), np.arange(10_000_000, 10_003_000, dtype=np.int64))
    gix.delete(np.arange(0, 80_000, 7, dtype=np.int64))
    # a plane left behind by the moved rows would bound other rows than the ones re-scored: the results would differ
    out = arms(pv, gix, queries)
    assert_same(out)
    assert out[1][3] == 0 or out[1][2] > 0   # level P ran: no int8 scan but the re-run of its failed queries


def test_filtered_matches_unfiltered_then_filtered(pv, lowrank):
    _, gix, queries = lowrank
    rng = np.random.default_rng(9)
    allowed = np.sort(rng.choice(80_000, 60_000, replace=False)).astype(np.int64)
    with gix.filter(allowed) as f:
        out = arms(pv, gix, queries, filter=f)
    assert_same(out)


def test_non_finite_rows_take_no_level_p(pv):
    rows, queries = low_rank(80_000, DIM, 8, seed=12), low_rank(NQ, DIM, 8, seed=13)
    gix, _ = build(pv, rows, LISTS, seed=42)
    bad = low_rank(2, DIM, 8, seed=16)
    bad[0, 3], bad[1, 0] = np.inf, np.nan
    gix.insert(bad, np.array([20_000_000, 20_000_001], dtype=np.int64))
    out = arms(pv, gix, queries)
    assert_same(out)
    assert out[1][3] == 0 and out[1][2] == 0   # no error bound holds: the exact kernels, in both arms


def test_small_batches_and_forced_tensor_cores_keep_level0(pv, lowrank):
    _, gix, queries = lowrank
    for qs in (low_rank(2048, DIM, 8, seed=17),   # 2048 queries over 80 k rows: the refine's extra rows outweigh the bytes saved
               queries[:128]):                  # fewer than 256 queries
        out = arms(pv, gix, qs)
        assert_same(out)
        assert out[1][3] > 0 and out[1][2] == 0
    pv.set_option("scan_impl", 4)
    try:
        pv.tc_traffic(True, read=True)
        gix.search(queries, k=K, probes=PROBES)
        assert int(pv.tc_traffic(False, read=True)[3]) > 0
    finally:
        pv.set_option("scan_impl", int(os.environ.get("VB_TEST_SCAN_IMPL", "2")))
