"""VACUUM of a resident HNSW image on the GPU (vb_hnsw_vacuum = the graph part of hnswbulkdelete, src/hnswvacuum.c):
serial parity with the oracle's vacuum, the change records as the exact slot diff, loaded and built images alike, the
reference's vacuum tests (test/t/011, 014, 022, 026), no tombstone in any result or live list, and what a vacuum does
to filters and scan handles."""
import ctypes as C

import numpy as np
import pytest

import oracle as O
from tests.hnsw_vacuum_oracle import VacuumHnsw
from tests.test_gpu_hnsw_insert import check_records, make_rows
from tests.test_hnsw_vacuum_oracle import _rows_011, dead_hold_links, live_links_to_dead

pytestmark = pytest.mark.gpu
EINVAL, ESTATE = -1, -5


@pytest.fixture(scope="module")
def pv():
    import pgvector_b200 as pv
    pv.init(0)
    return pv


def with_export_counts(ex, counts):
    ex = dict(ex)
    ex["n_heaptids"] = counts
    return ex


def vacuum(pv, gi, counts, efc=64, fraction=64):
    try:
        pv.set_option("hnsw_build_fraction", fraction)
        return gi.vacuum(counts, ef_construction=efc)
    finally:
        pv.set_option("hnsw_build_fraction", 64)


# (opclass, dim, m, ef_construction, rows): besides m = 8 / ef_construction = 40, the repair kernel at m = 100 /
# ef_construction = 1000, on both sides of its lanes-per-row split at 32 words (vector(123) and (125)), where R of
# ef_construction + 1 entries fits in shared memory but four times that does not (vector(3) at ef_construction 1000,
# vector(2000) at 620, halfvec(4000) at 300: a shared R between the two), and where not even ef_construction + 1 entries
# fit (halfvec(4000) at 1000: R in global memory from the start)
SERIAL_VACUUM_SHAPES = [("vector_l2_ops", 24, 8, 40, 3000, "vector_l2_ops"), ("halfvec_ip_ops", 32, 8, 40, 3000, "halfvec_ip_ops"),
                        ("vector_l2_ops", 24, 100, 1000, 1500, "vector_l2_ops-m100-efc1000"),
                        ("vector_l2_ops", 123, 8, 40, 3000, "vector_l2_ops-dim123"),
                        ("vector_l2_ops", 125, 8, 40, 3000, "vector_l2_ops-dim125"),
                        ("vector_l2_ops", 3, 16, 1000, 2000, "vector_l2_ops-dim3-efc1000"),
                        ("vector_l2_ops", 2000, 16, 620, 800, "vector_l2_ops-dim2000-efc620"),
                        ("halfvec_ip_ops", 4000, 16, 300, 600, "halfvec_ip_ops-dim4000-efc300"),
                        ("halfvec_ip_ops", 4000, 16, 1000, 600, "halfvec_ip_ops-dim4000-efc1000")]


def repair_shared_cap(opclass, dim, m, efc):
    """R's capacity in shared memory as vb_hnsw_vacuum picks it (hb_insert_smem / hb_insert_shared_cap, vb_hnsw_build.cu):
    the largest in [ef + 1, 4 (ef + 1)] whose 4-warp CTA fits in 200 KiB, or 0: R in global memory"""
    words = ((4 if opclass.startswith("vector") else 2) * dim + 15) // 16
    qvec = 2 * words if opclass.startswith("halfvec") else words   # (a halfvec row image is widened to fp32)

    def cta(cap):
        b = qvec * 16 * 2 + cap * 2 * 8 + 32 * 8 + cap * 2 * 4 + 32 * 4 * 2 + 2 * m * 4 + cap * 2 + cap
        return ((b + 15) & ~15) * 4
    efv = efc + 1
    return next((c for c in range(4 * efv, efv - 1, -1) if cta(c) <= 200 * 1024), 0)


def test_vacuum_shapes_take_the_routes_they_name():
    cap = {i: (repair_shared_cap(o, d, m, efc), efc + 1) for o, d, m, efc, n, i in SERIAL_VACUUM_SHAPES}
    for i in ("vector_l2_ops-dim3-efc1000", "vector_l2_ops-dim2000-efc620", "halfvec_ip_ops-dim4000-efc300"):
        c, efv = cap[i]
        assert efv <= c < 4 * efv, (i, c)
    assert cap["vector_l2_ops"][0] == 4 * 41 and cap["halfvec_ip_ops-dim4000-efc1000"][0] == 0


SERIAL_VACUUM_CASES = [pytest.param(o, d, m, efc, n, dl, id=f"{i}-{dl}") for o, d, m, efc, n, i in SERIAL_VACUUM_SHAPES
                       for dl in (0.10, 0.75, 0.99)]


@pytest.mark.parametrize("opclass,dim,m,efc,n,deleted", SERIAL_VACUUM_CASES)
def test_one_element_batches_are_the_serial_vacuum(pv, opclass, dim, m, efc, n, deleted):
    """batches of one element: the GPU vacuum is the oracle's serial vacuum (tests/hnsw_vacuum_oracle.c).  At 99 %
    deleted a repair's candidate list outgrows the shared-memory one and is rerun in global memory."""
    elem, metric, x, dim = make_rows(opclass, n, 41, dim=dim)
    og = VacuumHnsw(elem, metric, x, m=m, ef_construction=efc, seed=3, dim=dim)
    ge = og.export()
    gi = pv.HnswIndex(opclass, dim, m=m).load(x, ge["levels"], ge["nbr0"], ge["upper_off"], ge["upper"], ge["entry"])
    counts = np.ones(n, np.int32)
    counts[np.random.default_rng(int(deleted * 100)).choice(n, int(n * deleted), replace=False)] = 0
    recs, nrep = vacuum(pv, gi, counts, efc=efc, fraction=1 << 30)
    orecs, onrep = og.vacuum(counts)
    g, oe = gi.export(), og.export()
    assert g["entry"] == oe["entry"] and counts[g["entry"]] == 1
    assert nrep == onrep and nrep > 0
    touched = np.union1d(recs["element"][recs["layer"] == 0], orecs["element"][orecs["layer"] == 0])
    touched = touched[counts[touched] > 0]
    same = np.all(g["nbr0"][touched] == oe["nbr0"][touched], axis=1)
    assert len(touched) > 0 and same.mean() >= 0.98, same.mean()
    assert live_links_to_dead(with_export_counts(g, counts)) == 0 and dead_hold_links(with_export_counts(g, counts)) == 0


@pytest.mark.parametrize("fraction", [64, 1 << 30])
def test_records_are_the_slot_diff(pv, fraction):
    elem, metric, x, dim = make_rows("vector_l2_ops", 4000, 5)
    gi = pv.HnswIndex("vector_l2_ops", dim, m=8).build(x, ef_construction=40, seed=1)
    before = gi.export()
    counts = np.ones(4000, np.int32)
    counts[np.random.default_rng(2).choice(4000, 400, replace=False)] = 0
    recs, nrep = vacuum(pv, gi, counts, efc=40, fraction=fraction)
    after = gi.export()
    assert nrep > 0 and np.any(recs["neighbor"] == -1)
    check_records(before, after, recs)
    # a second call reports its own records only
    counts2 = counts.copy()
    counts2[np.random.default_rng(3).choice(np.nonzero(counts)[0], 100, replace=False)] = 0
    recs2, _ = vacuum(pv, gi, counts2, efc=40, fraction=fraction)
    check_records(after, gi.export(), recs2)
    assert live_links_to_dead(with_export_counts(gi.export(), counts2)) == 0


def test_loaded_and_built_images_vacuum_alike(pv):
    elem, metric, x, dim = make_rows("vector_l2_ops", 5000, 6)
    gb = pv.HnswIndex("vector_l2_ops", dim).build(x, seed=4)
    ex = gb.export()
    gl = pv.HnswIndex("vector_l2_ops", dim).load(x, ex["levels"], ex["nbr0"], ex["upper_off"], ex["upper"], ex["entry"])
    counts = np.ones(5000, np.int32)
    counts[np.random.default_rng(7).choice(5000, 500, replace=False)] = 0
    r1, n1 = gb.vacuum(counts)
    r2, n2 = gl.vacuum(counts)
    assert n1 == n2 and n1 > 0 and np.array_equal(r1, r2)
    assert gb.export()["entry"] == gl.export()["entry"]


def vacuum_recall(pv, opclass, rows, queries, dim, ef, tie_aware=False):
    elem, metric, _, _ = pv.OPCLASSES[opclass]
    gi = pv.HnswIndex(opclass, dim, m=4).build(rows, ef_construction=8, seed=1)
    keep = np.arange(1, len(rows) + 1) <= 2500
    counts = keep.astype(np.int32)
    recs, nrep = gi.vacuum(counts, ef_construction=8)
    assert nrep > 0 and live_links_to_dead(with_export_counts(gi.export(), counts)) == 0
    live = np.nonzero(keep)[0]
    ids, dist, _ = gi.search(queries, k=20, ef_search=ef)
    hit = tot = 0
    for qi, q in enumerate(queries):
        got = ids[qi][ids[qi] >= 0]
        assert np.all(counts[got] > 0)
        if tie_aware:
            kth = O.exact_topk(elem, metric, q, rows[live], 20, dim=dim)[1][-1]
            hit += int(np.sum(dist[qi][:len(got)] <= kth))
        else:
            truth = live[O.exact_topk(elem, metric, q, rows[live], 20, dim=dim)[0]]
            hit += len(set(got.tolist()) & set(truth.tolist()))
        tot += 20
    return hit / tot


def test_014_vector_vacuum_recall(pv):
    rng = np.random.default_rng(14)
    rows = rng.random((10000, 3)).astype(np.float32)
    queries = rng.random((20, 3)).astype(np.float32)
    r = vacuum_recall(pv, "vector_l2_ops", rows, queries, 3, 20)
    assert r >= 0.95, r


def test_022_bit_vacuum_recall(pv):
    rng = np.random.default_rng(22)
    rows = np.packbits(rng.integers(0, 2, (10000, 52), dtype=np.uint8), axis=1)
    queries = np.packbits(rng.integers(0, 2, (20, 52), dtype=np.uint8), axis=1)
    r = vacuum_recall(pv, "bit_hamming_ops", rows, queries, 52, 100, tie_aware=True)
    assert r >= 0.80, r


def test_026_halfvec_vacuum_recall(pv):
    from tests.util import f32_to_half_bits
    rng = np.random.default_rng(26)
    rows = f32_to_half_bits(rng.random((10000, 3)).astype(np.float32))
    queries = f32_to_half_bits(rng.random((20, 3)).astype(np.float32))
    r = vacuum_recall(pv, "halfvec_l2_ops", rows, queries, 3, 20)
    assert r >= 0.95, r


def test_011_delete_all_but_one_then_all_then_insert(pv):
    rows = _rows_011()
    gi = pv.HnswIndex("vector_l2_ops", 3).build(rows, seed=11)
    keep = np.zeros(len(rows), np.int32)
    keep[122] = 1
    gi.vacuum(keep)
    assert gi.export()["entry"] == 122
    ids, _, _ = gi.search(np.zeros((1, 3), np.float32), k=10, ef_search=40)
    assert ids[0][ids[0] >= 0].tolist() == [122]
    gi.vacuum(np.zeros(len(rows), np.int32))
    ex = gi.export()
    assert ex["entry"] == -1 and dead_hold_links(with_export_counts(ex, np.zeros(len(rows), np.int32))) == 0
    # the next insert's first row becomes the entry point
    n0 = len(rows)
    lv = np.zeros(100, np.int32)
    gi.insert(rows[:100], levels=lv)
    ex = gi.export()
    assert ex["entry"] == n0
    ids, dist, _ = gi.search(rows[:20], k=1, ef_search=40)
    assert np.all(ids[:, 0] >= n0) and np.all(dist[:, 0] == 0)


def test_no_tombstone_in_results_or_live_lists(pv):
    elem, metric, x, dim = make_rows("vector_l2_ops", 20000, 9)
    gi = pv.HnswIndex("vector_l2_ops", dim).build(x, seed=2)
    counts = np.ones(20000, np.int32)
    counts[np.random.default_rng(4).choice(20000, 2000, replace=False)] = 0
    gi.vacuum(counts)
    q = x[np.random.default_rng(5).choice(20000, 2000, replace=False)] + 0.01
    ids, _, _ = gi.search(q, k=10, ef_search=40)
    got = ids[ids >= 0]
    assert len(got) == 2000 * 10 and np.all(counts[got] > 0)
    ex = with_export_counts(gi.export(), counts)
    assert live_links_to_dead(ex) == 0 and dead_hold_links(ex) == 0


def test_state_filters_handles_and_bad_arguments(pv):
    elem, metric, x, dim = make_rows("vector_l2_ops", 3000, 8)
    gi = pv.HnswIndex("vector_l2_ops", dim).build(x)
    f = gi.filter(np.arange(0, 3000, 3))
    fs = gi.iterative_scan(x[:4], ef_search=20, max_scan_tuples=200, filter=f, page=10)
    us = gi.iterative_scan(x[:4], ef_search=20, max_scan_tuples=200)
    fs.next_batch()
    us.next_batch()
    snap = gi.export()
    L = pv._lib.load()
    nrep, nchg = C.c_int64(0), C.c_int64(0)
    good = np.ones(3000, np.int32)
    for counts, efc in [(np.full(3000, 11, np.int32), 64), (np.full(3000, -1, np.int32), 64), (good, 16), (good, 2000), (None, 64)]:
        ptr = None if counts is None else counts.ctypes.data_as(C.c_void_p)
        assert L.vb_hnsw_vacuum(gi.h, ptr, efc, C.byref(nrep), C.byref(nchg)) == EINVAL
        after = gi.export()
        assert all(np.array_equal(snap[k], after[k]) for k in ("levels", "nbr0", "upper_off", "upper", "dup_of"))
        assert snap["entry"] == after["entry"]
    with pytest.raises(ValueError):
        gi.vacuum(np.ones(10, np.int32))
    counts = good.copy()
    counts[::7] = 0
    recs, nrep = gi.vacuum(counts)
    out = np.empty(len(recs), dtype=pv.HNSW_SLOT_DTYPE)
    assert L.vb_hnsw_insert_changes(gi.h, out.ctypes.data_as(C.c_void_p), len(recs)) == 0
    assert np.array_equal(out, recs)
    with pytest.raises(pv.VecB200Error) as e:
        fs.next_batch()
    assert e.value.code == ESTATE
    with pytest.raises(pv.VecB200Error) as e:
        gi.iterative_scan(x[:4], ef_search=20, filter=f, page=10)
    assert e.value.code == ESTATE
    ids, _, cnt = us.next_batch()
    assert cnt.min() > 0
    fs.close()
    us.close()
