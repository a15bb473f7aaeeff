"""The serial vacuum (tests/hnsw_vacuum_oracle.c: hnswbulkdelete's RepairGraphEntryPoint, RepairGraph and MarkDeleted,
src/hnswvacuum.c) that the GPU vacuum is checked against: the recall floors of the reference's vacuum tests (test/t/014,
022, 026), deleting everything or all but one row (011), and rounds of inserts, deletes and vacuums (047)."""
import numpy as np
import pytest

import oracle as O
from tests.hnsw_vacuum_oracle import VacuumHnsw
from tests.util import f32_to_half_bits


def live_links_to_dead(ex):
    """number of neighbour slots of live elements that name an element with no heap TIDs"""
    cnt = ex["n_heaptids"]
    live = cnt > 0
    bad = int(np.sum((ex["nbr0"][live] >= 0) & (cnt[np.maximum(ex["nbr0"][live], 0)] == 0)))
    lv, uo = ex["levels"], ex["upper_off"]
    for e in np.nonzero(live & (lv > 0))[0]:
        s = ex["upper"][uo[e]:uo[e] + lv[e]]
        bad += int(np.sum((s >= 0) & (cnt[np.maximum(s, 0)] == 0)))
    return bad


def dead_hold_links(ex):
    cnt = ex["n_heaptids"]
    dead = cnt == 0
    n = int(np.sum(ex["nbr0"][dead] >= 0))
    lv, uo = ex["levels"], ex["upper_off"]
    for e in np.nonzero(dead & (lv > 0))[0]:
        n += int(np.sum(ex["upper"][uo[e]:uo[e] + lv[e]] >= 0))
    return n


def recall_after_delete(elem, metric, rows, queries, keep, ef, dim=None, k=20, tie_aware=False):
    g = VacuumHnsw(elem, metric, rows, m=4, ef_construction=8, dim=dim)
    counts = keep.astype(np.int32)
    recs, nrep = g.vacuum(counts)
    ex = g.export()
    assert live_links_to_dead(ex) == 0 and dead_hold_links(ex) == 0
    assert nrep > 0 and len(recs) > 0
    live = np.nonzero(keep)[0]
    hit = tot = 0
    for q in queries:
        ids, dist, _ = g.search(q, ef, ties=O.TIES_TOTAL)
        assert np.all(counts[ids] > 0)
        if tie_aware:
            kth = O.exact_topk(elem, metric, q, rows[live], k, dim=dim)[1][-1]
            hit += int(np.sum(dist[:k] <= kth))
        else:
            truth = live[O.exact_topk(elem, metric, q, rows[live], k, dim=dim)[0]]
            hit += len(set(ids[:k].tolist()) & set(truth.tolist()))
        tot += k
    return hit / tot


def test_014_vector_vacuum_recall():
    """10 000 random 3-d vectors, m 4, ef_construction 8, rows i > 2500 deleted: LIMIT 20 at ef_search 20 >= 0.95"""
    rng = np.random.default_rng(14)
    rows = rng.random((10000, 3)).astype(np.float32)
    queries = rng.random((20, 3)).astype(np.float32)
    keep = np.arange(1, 10001) <= 2500
    assert recall_after_delete(O.VECTOR, O.L2_SQUARED, rows, queries, keep, 20) >= 0.95


def test_022_bit_vacuum_recall():
    """10 000 random bit(52), m 4, ef_construction 8, rows i > 2500 deleted: within the true 20th distance >= 0.80"""
    rng = np.random.default_rng(22)
    rows = np.packbits(rng.integers(0, 2, (10000, 52), dtype=np.uint8), axis=1)
    queries = np.packbits(rng.integers(0, 2, (20, 52), dtype=np.uint8), axis=1)
    keep = np.arange(1, 10001) <= 2500
    r = recall_after_delete(O.BIT, O.HAMMING, rows, queries, keep, 100, dim=52, tie_aware=True)
    assert r >= 0.80, r


def test_026_halfvec_vacuum_recall():
    """026: the 014 shape as halfvec(3) with halfvec_l2_ops: >= 0.95"""
    rng = np.random.default_rng(26)
    rows = f32_to_half_bits(rng.random((10000, 3)).astype(np.float32))
    queries = f32_to_half_bits(rng.random((20, 3)).astype(np.float32))
    keep = np.arange(1, 10001) <= 2500
    assert recall_after_delete(O.HALFVEC, O.L2_SQUARED, rows, queries, keep, 20) >= 0.95


def _rows_011():
    i = np.arange(1, 10001)
    rng = np.random.default_rng(11)
    mods = rng.integers(1, 1001, 3)
    return np.stack([i % v for v in mods], axis=1).astype(np.float32)


def test_011_delete_all_but_one_then_all_then_insert():
    rows = _rows_011()
    g = VacuumHnsw(O.VECTOR, O.L2_SQUARED, rows, m=16, ef_construction=64)
    keep = np.zeros(len(rows), np.int32)
    keep[122] = 1   # i = 123
    _, nrep = g.vacuum(keep)
    ex = g.export()
    assert ex["entry"] == 122 and dead_hold_links(ex) == 0
    ids, _, _ = g.search(np.zeros(3, np.float32), 40, ties=O.TIES_TOTAL)
    assert ids.tolist() == [122]
    # delete the last one: the entry point becomes -1
    g.vacuum(np.zeros(len(rows), np.int32))
    ex = g.export()
    assert ex["entry"] == -1 and dead_hold_links(ex) == 0
    ids, _, _ = g.search(np.zeros(3, np.float32), 40, ties=O.TIES_TOTAL)
    assert len(ids) == 0
    # an insert makes its first row the entry point
    n0 = g.n
    g.insert_on_disk(rows[:100], levels=np.zeros(100, np.int32))
    ex = g.export()
    assert ex["entry"] == n0
    ids, _, _ = g.search(rows[5], 40, ties=O.TIES_TOTAL)
    assert len(ids) > 0 and np.all(ids >= n0)
    assert live_links_to_dead(ex) == 0


def test_047_rounds_of_insert_delete_vacuum():
    """rounds of inserts, deletes and vacuums, with searches between: no live element ever links to a deleted one"""
    rng = np.random.default_rng(47)
    g = VacuumHnsw(O.VECTOR, O.L2_SQUARED, rng.random((1000, 3)).astype(np.float32), m=16, ef_construction=64)
    for _ in range(6):
        g.insert_on_disk(rng.random((200, 3)).astype(np.float32))
        counts = g.export()["n_heaptids"].copy()
        live = np.nonzero(counts > 0)[0]
        counts[rng.choice(live, size=len(live) // 5, replace=False)] = 0
        g.vacuum(counts)
        ex = g.export()
        assert live_links_to_dead(ex) == 0 and dead_hold_links(ex) == 0
        assert ex["entry"] >= 0 and counts[ex["entry"]] > 0
        for q in rng.random((5, 3)).astype(np.float32):
            ids, _, _ = g.search(q, 40, ties=O.TIES_TOTAL)
            assert len(ids) > 0 and np.all(counts[ids] > 0)


def test_vacuum_records_are_the_slot_diff_and_repairs_are_needed_ones():
    """a vacuum with nothing deleted repairs only elements whose layer-0 list is not full; a second vacuum of the same
    counts repairs no element that links to a deleted one"""
    rng = np.random.default_rng(5)
    rows = rng.random((2000, 8)).astype(np.float32)
    g = VacuumHnsw(O.VECTOR, O.L2_SQUARED, rows, m=8, ef_construction=32)
    ex = g.export()
    not_full = int(np.sum(ex["nbr0"][:, -1] < 0)) - int(ex["nbr0"][ex["entry"], -1] < 0)
    recs, nrep = g.vacuum(np.ones(len(rows), np.int32))
    assert nrep == not_full
    counts = np.ones(len(rows), np.int32)
    counts[rng.choice(len(rows), 200, replace=False)] = 0
    recs, nrep = g.vacuum(counts)
    assert nrep > 0 and np.any(recs["neighbor"] == -1)
    ex = g.export()
    assert live_links_to_dead(ex) == 0 and dead_hold_links(ex) == 0
