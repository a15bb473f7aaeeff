"""The serial on-disk insert (tests/hnsw_ondisk_oracle.c = HnswInsertTupleOnDisk, src/hnswinsert.c:696-743),
which the GPU insert is checked against: the recall floors of the reference's insert tests (test/t/013, 021, 025) on
graphs grown from an empty index, duplicate folding (015), and the rules for elements being deleted
(RemoveElements, GetUpdateIndex)."""
import numpy as np
import pytest

import oracle as O
from tests.hnsw_ondisk_oracle import DiskHnsw
from tests.util import f32_to_half_bits, mixture


def grown(elem, metric, rows, dim=None, m=16, efc=64, levels=None):
    """an empty oracle index and then every row inserted one at a time"""
    d = dim if dim is not None else rows.shape[1]
    g = DiskHnsw(elem, metric, rows[:0], m=m, ef_construction=efc, dim=d)
    dup, chg = g.insert_on_disk(rows, levels=levels)
    return g, dup, chg


def recall_floor(g, elem, metric, rows, queries, ef, dim=None, k=20):
    hit = tot = 0
    for q in queries:
        ids, dist, _ = g.search(q, ef, ties=O.TIES_TOTAL)
        truth = O.exact_topk(elem, metric, q, rows, k, dim=dim)[0]
        hit += len(set(ids[:k].tolist()) & set(truth.tolist()))
        tot += k
    return hit / tot


@pytest.mark.parametrize("opclass", ["l2", "ip", "cosine", "l1"])
def test_013_vector_insert_recall(opclass):
    """10 000 3-d vectors of random() * random() inserted into an empty index, ef_search 40, LIMIT 20: >= 0.99 (<#>: 0.97)"""
    rng = np.random.default_rng(13)
    rows = (rng.random((10000, 3)) * rng.random((10000, 3))).astype(np.float32)
    queries = rng.random((20, 3)).astype(np.float32)
    metric = {"l2": O.L2_SQUARED, "ip": O.NEG_IP, "cosine": O.NEG_IP, "l1": O.L1}[opclass]
    if opclass == "cosine":
        rows, queries = O.l2_normalize(O.VECTOR, rows), O.l2_normalize(O.VECTOR, queries)
    g, dup, _ = grown(O.VECTOR, metric, rows)
    assert np.all(dup == -1)
    r = recall_floor(g, O.VECTOR, metric, rows, queries, 40)
    assert r >= (0.97 if opclass == "ip" else 0.99), r


@pytest.mark.parametrize("metric,floor", [(O.HAMMING, 0.98), (O.JACCARD, 0.95)])
def test_021_bit_insert_recall_tie_aware(metric, floor):
    """10 000 random bit(52), ef_search 100, LIMIT 20; a result counts when it is within the true 20th distance"""
    rng = np.random.default_rng(21)
    rows = np.packbits(rng.integers(0, 2, (10000, 52), dtype=np.uint8), axis=1)
    queries = np.packbits(rng.integers(0, 2, (20, 52), dtype=np.uint8), axis=1)
    g, dup, _ = grown(O.BIT, metric, rows, dim=52)
    keep = dup < 0
    hit = tot = 0
    for q in queries:
        _, dist, _ = g.search(q, 100, ties=O.TIES_TOTAL)
        kth = O.exact_topk(O.BIT, metric, q, rows[keep], 20, dim=52)[1][-1]
        hit += int(np.sum(dist[:20] <= kth))
        tot += 20
    assert hit / tot >= floor, hit / tot


@pytest.mark.parametrize("opclass", ["l2", "ip", "cosine", "l1"])
def test_025_halfvec_insert_recall(opclass):
    """10 000 halfvec(10) of 2 * random() * random(), ef_search 40, LIMIT 20: >= 0.98"""
    rng = np.random.default_rng(25)
    x = (2 * rng.random((10000, 10)) * rng.random((10000, 10))).astype(np.float32)
    q = rng.random((20, 10)).astype(np.float32)
    rows, queries = f32_to_half_bits(x), f32_to_half_bits(q)
    metric = {"l2": O.L2_SQUARED, "ip": O.NEG_IP, "cosine": O.NEG_IP, "l1": O.L1}[opclass]
    if opclass == "cosine":
        rows, queries = O.l2_normalize(O.HALFVEC, rows), O.l2_normalize(O.HALFVEC, queries)
    g, _, _ = grown(O.HALFVEC, metric, rows)
    r = recall_floor(g, O.HALFVEC, metric, rows, queries, 40)
    assert r >= 0.98, r


def test_015_duplicates_fold_into_ten_heap_tids():
    """20 copies of [1,1,1] inserted one at a time: the first element takes 10 heap TIDs, so a scan at ef_search 1
    returns 10 rows; the 11th copy becomes an element of its own (the first one is full)"""
    g = DiskHnsw(O.VECTOR, O.L2_SQUARED, np.zeros((0, 3), np.float32))
    dups = []
    for _ in range(20):
        d, _ = g.insert_on_disk(np.ones((1, 3), np.float32))
        dups.append(int(d[0]))
    assert dups == [-1] + [0] * 9 + [-1] + [10] * 9
    ex = g.export()
    assert ex["n_heaptids"][0] == 10 and ex["n_heaptids"][10] == 10
    ids, _, _ = g.search(np.ones(3, np.float32), 1)
    assert len(ids) == 1 and ex["n_heaptids"][ids[0]] == 10


def test_deleted_neighbours_are_never_chosen_and_go_first():
    """RemoveElements: no new list names an element being deleted; GetUpdateIndex: a full list that holds such an
    element loses its first one (then the next, as more updates arrive)"""
    x, _ = mixture(2600, 8, 12, seed=4)
    g, _, _ = grown(O.VECTOR, O.L2_SQUARED, x[:2000], m=4, efc=16)
    counts = np.ones(2000, np.int32)
    counts[::7] = 0
    g.set_heaptid_counts(counts)
    before = g.export()
    _, chg = g.insert_on_disk(x[2000:])
    after = g.export()
    cnt = np.concatenate([counts, np.ones(600, np.int32)])
    new0 = after["nbr0"][2000:]
    assert np.all(cnt[new0[new0 >= 0]] == 1)
    lm = 8
    checked = 0
    old0 = chg[(chg["element"] < 2000) & (chg["layer"] == 0)]
    for e in np.unique(old0["element"]):
        lst = before["nbr0"][e]
        if np.any(lst < 0):
            continue
        z = np.nonzero(counts[lst] == 0)[0]
        if len(z) == 0:
            continue
        c = np.sort(old0["slot"][old0["element"] == e])
        if len(c) <= len(z):
            assert np.array_equal(c, z[:len(c)]), (e, c, z)
        else:
            assert set(z) <= set(c)
        checked += 1
    assert checked > 20, checked
    assert lm == 2 * before["m"]
