"""INSERT into a resident HNSW image on the GPU (vb_hnsw_insert = batched HnswInsertTupleOnDisk,
src/hnswinsert.c:696-743): serial parity with the oracle's on-disk insert, the change records as the exact slot diff,
loaded and built images alike, the reference's insert recall floors (test/t/013, 015, 016, 021, 025), the entry point,
and what an insert does to filters and scan handles."""
import ctypes as C

import numpy as np
import pytest

import oracle as O
from tests.hnsw_ondisk_oracle import DiskHnsw, slot_changes
from tests.util import f32_to_half_bits, mixture, recall_at_k

pytestmark = pytest.mark.gpu
EINVAL, ESTATE = -1, -5


@pytest.fixture(scope="module")
def pv():
    import pgvector_b200 as pv
    pv.init(0)
    return pv


def draw_levels(n, m, seed):
    """HnswInitElement's law: floor(-ln(U) * 1 / ln(m))"""
    u = np.random.default_rng(seed).random(n)
    return np.floor(-np.log1p(-u) / np.log(m)).astype(np.int32)


def apply_changes(before, n1, slots1):
    """the page writer's view: a pre-insert export grown by the new elements, with the records applied"""
    m = before["m"]
    nbr0 = np.full((n1, 2 * m), -1, np.int32)
    nbr0[:len(before["nbr0"])] = before["nbr0"]
    up = np.full((slots1, m), -1, np.int32)
    up[:len(before["upper"])] = before["upper"]
    return nbr0, up


def check_records(before, after, recs):
    nbr0, up = apply_changes(before, len(after["levels"]), len(after["upper"]))
    for r in recs:
        if r["layer"] == 0:
            nbr0[r["element"], r["slot"]] = r["neighbor"]
        else:
            up[after["upper_off"][r["element"]] + r["layer"] - 1, r["slot"]] = r["neighbor"]
    assert np.array_equal(nbr0, after["nbr0"]) and np.array_equal(up, after["upper"])
    want = slot_changes(before, after)     # exactly the slots that differ: no other slot changed
    assert np.array_equal(recs, want.astype(recs.dtype))
    keys = recs["element"].astype(np.int64) << 16 | recs["layer"].astype(np.int64) << 8 | recs["slot"]
    assert np.all(np.diff(keys) > 0)


def make_rows(kind, n, seed, dim=None):
    """mixture rows of a vector_l2_ops or a halfvec opclass (24 and 32 dimensions unless given)"""
    if kind == "vector_l2_ops":
        dim = dim or 24
        x, _ = mixture(n, dim, 16, seed=seed)
        return O.VECTOR, O.L2_SQUARED, x, dim
    dim = dim or 32
    x, _ = mixture(n, dim, 16, seed=seed)
    return O.HALFVEC, O.NEG_IP, f32_to_half_bits(x), dim


# (opclass, dim, m, ef_construction, rows before the insert): the insert kernel at m = 100 / ef_construction = 1000, on both
# sides of its lanes-per-row split at 32 words (vector(123) and (125)), and on halfvec(4000) rows, whose R of 1000 entries
# lives in global memory
SERIAL_INSERT_CASES = [
    pytest.param("vector_l2_ops", 24, 8, 40, 1500, id="vector_l2_ops"),
    pytest.param("halfvec_ip_ops", 32, 8, 40, 1500, id="halfvec_ip_ops"),
    pytest.param("vector_l2_ops", 24, 100, 1000, 800, id="vector_l2_ops-m100-efc1000"),
    pytest.param("vector_l2_ops", 123, 8, 40, 1500, id="vector_l2_ops-dim123"),
    pytest.param("vector_l2_ops", 125, 8, 40, 1500, id="vector_l2_ops-dim125"),
    pytest.param("halfvec_ip_ops", 4000, 16, 1000, 400, id="halfvec_ip_ops-dim4000-efc1000"),
]


@pytest.mark.parametrize("opclass,dim,m,efc,n0", SERIAL_INSERT_CASES)
def test_one_row_batches_are_the_serial_on_disk_insert(pv, opclass, dim, m, efc, n0):
    """batches of one row and the oracle's level draws: the GPU insert is the serial on-disk insert (tests/hnsw_ondisk_oracle.c), including elements
    being deleted (heap TID count 0).  (Bit Hamming is not compared list for list: its integer distances tie almost
    everywhere, the oracle's search breaks ties in pairing-heap order and the GPU's by element number, and one different
    tie sends the serial inserts apart; measured on an H100, 26 % of the lists were identical and 63 % had the same
    distances.  Its inserts are held to the 021 recall floors instead.)"""
    elem, metric, x, dim = make_rows(opclass, 2 * n0, 31, dim=dim)
    og = DiskHnsw(elem, metric, x[:n0], m=m, ef_construction=efc, seed=3, dim=dim)
    ge = og.export()
    assert len(ge["levels"]) == n0
    counts = np.ones(n0, np.int32)
    counts[np.random.default_rng(1).choice(n0, n0 // 20, replace=False)] = 0
    og.set_heaptid_counts(counts)
    gi = pv.HnswIndex(opclass, dim, m=m).load(x[:n0], ge["levels"], ge["nbr0"], ge["upper_off"], ge["upper"], ge["entry"])
    gi.set_heaptid_counts(counts)
    lv = draw_levels(n0, m, 8)
    try:
        pv.set_option("hnsw_build_fraction", 1 << 30)
        dup, recs = gi.insert(x[n0:], ef_construction=efc, levels=lv)
    finally:
        pv.set_option("hnsw_build_fraction", 64)
    odup, orecs = og.insert_on_disk(x[n0:], levels=lv)
    g, oe = gi.export(), og.export()
    assert g["entry"] == oe["entry"]
    assert np.array_equal(dup, odup)
    touched = np.union1d(recs["element"][recs["layer"] == 0], orecs["element"][orecs["layer"] == 0])
    same = np.all(g["nbr0"][touched] == oe["nbr0"][touched], axis=1)
    assert len(touched) > n0 and same.mean() > 0.98, same.mean()
    assert not np.isin(g["nbr0"][n0:], np.nonzero(counts == 0)[0]).any()


@pytest.mark.parametrize("fraction", [64, 1 << 30])
def test_records_are_the_slot_diff(pv, fraction):
    x, _ = mixture(4000, 16, 20, seed=5)
    gi = pv.HnswIndex("vector_l2_ops", 16, m=8).build(x[:3000], ef_construction=40, seed=1)
    before = gi.export()
    try:
        pv.set_option("hnsw_build_fraction", fraction)
        dup, recs = gi.insert(x[3000:], ef_construction=40, seed=2)
    finally:
        pv.set_option("hnsw_build_fraction", 64)
    after = gi.export()
    assert np.all(dup == -1) and len(after["levels"]) == 4000
    assert np.array_equal(after["nbr0"][:3000][before["nbr0"] >= 0] >= 0, np.ones(int((before["nbr0"] >= 0).sum()), bool))
    check_records(before, after, recs)
    # a second call: the records are that call's alone
    before2 = after
    _, recs2 = gi.insert(x[:50] + 0.5, ef_construction=40, seed=3)
    check_records(before2, gi.export(), recs2)


def test_loaded_and_built_images_insert_alike(pv):
    """the on-disk update never reads a stored distance: a built image and vb_hnsw_load of its export give the same
    records"""
    x, _ = mixture(5000, 32, 20, seed=6)
    gb = pv.HnswIndex("vector_l2_ops", 32).build(x[:4000], seed=4)
    ex = gb.export()
    gl = pv.HnswIndex("vector_l2_ops", 32).load(x[:4000], ex["levels"], ex["nbr0"], ex["upper_off"], ex["upper"], ex["entry"])
    lv = draw_levels(1000, 16, 9)
    d1, r1 = gb.insert(x[4000:], levels=lv)
    d2, r2 = gl.insert(x[4000:], levels=lv)
    assert np.array_equal(d1, d2) and np.array_equal(r1, r2) and len(r1) > 1000 * 16


def gpu_grown(pv, opclass, rows, dim, batch=None):
    gi = pv.HnswIndex(opclass, dim)
    gi.build(rows[:0])
    if batch is None:
        gi.insert(rows)
    else:
        for i in range(0, len(rows), batch):
            gi.insert(rows[i:i + batch], seed=i)
    return gi


@pytest.mark.parametrize("opclass", ["vector_l2_ops", "vector_ip_ops", "vector_cosine_ops", "vector_l1_ops"])
def test_013_recall_on_a_gpu_grown_graph(pv, opclass):
    rng = np.random.default_rng(13)
    rows = (rng.random((10000, 3)) * rng.random((10000, 3))).astype(np.float32)
    queries = rng.random((20, 3)).astype(np.float32)
    elem, metric, normalize, _ = pv.OPCLASSES[opclass]
    if normalize:
        rows, queries = O.l2_normalize(O.VECTOR, rows), O.l2_normalize(O.VECTOR, queries)
    gi = gpu_grown(pv, opclass, rows, 3)
    ids, _, _ = gi.search(queries, k=20, ef_search=40)
    truth = [O.exact_topk(O.VECTOR, metric, q, rows, 20)[0] for q in queries]
    assert recall_at_k(ids, truth) >= (0.97 if opclass == "vector_ip_ops" else 0.99)


@pytest.mark.parametrize("opclass,floor", [("bit_hamming_ops", 0.98), ("bit_jaccard_ops", 0.95)])
def test_021_recall_on_a_gpu_grown_graph(pv, opclass, floor):
    elem, metric, _, _ = pv.OPCLASSES[opclass]
    rng = np.random.default_rng(21)
    rows = np.packbits(rng.integers(0, 2, (10000, 52), dtype=np.uint8), axis=1)
    queries = np.packbits(rng.integers(0, 2, (20, 52), dtype=np.uint8), axis=1)
    gi = gpu_grown(pv, opclass, rows, 52)
    _, dist, _ = gi.search(queries, k=20, ef_search=100)
    hit = 0
    for q, d in zip(queries, dist):
        hit += int(np.sum(d <= O.exact_topk(elem, metric, q, rows, 20, dim=52)[1][-1]))
    assert hit / (20 * len(queries)) >= floor


@pytest.mark.parametrize("opclass", ["halfvec_l2_ops", "halfvec_ip_ops", "halfvec_cosine_ops", "halfvec_l1_ops"])
def test_025_recall_on_a_gpu_grown_graph(pv, opclass):
    rng = np.random.default_rng(25)
    rows = f32_to_half_bits((2 * rng.random((10000, 10)) * rng.random((10000, 10))).astype(np.float32))
    queries = f32_to_half_bits(rng.random((20, 10)).astype(np.float32))
    elem, metric, normalize, _ = pv.OPCLASSES[opclass]
    if normalize:
        rows, queries = O.l2_normalize(O.HALFVEC, rows), O.l2_normalize(O.HALFVEC, queries)
    gi = gpu_grown(pv, opclass, rows, 10)
    ids, _, _ = gi.search(queries, k=20, ef_search=40)
    truth = [O.exact_topk(O.HALFVEC, metric, q, rows, 20)[0] for q in queries]
    assert recall_at_k(ids, truth) >= 0.98


def test_016_inserts_of_ten_rows(pv):
    """1900-d L2, rows arriving ten at a time: the first ten are all reachable at ef_search 40, and after 1000 rows a
    scan at ef_search 1000 reaches >= 997 of them"""
    rng = np.random.default_rng(16)
    rows = rng.random((1000, 1900)).astype(np.float32)
    gi = pv.HnswIndex("vector_l2_ops", 1900)
    gi.build(rows[:0])
    gi.insert(rows[:10])
    ids, _, _ = gi.search(rng.random((1, 1900)).astype(np.float32), k=40, ef_search=40)
    assert sorted(ids[0][ids[0] >= 0].tolist()) == list(range(10))
    for i in range(10, 1000, 10):
        gi.insert(rows[i:i + 10], seed=i)
    ids, _, _ = gi.search(rng.random((1, 1900)).astype(np.float32), k=1000, ef_search=1000)
    assert len(set(ids[0][ids[0] >= 0].tolist())) >= 997


def test_015_duplicates_one_at_a_time(pv):
    gi = pv.HnswIndex("vector_l2_ops", 3)
    gi.build(np.zeros((0, 3), np.float32))
    dups = [int(gi.insert(np.ones((1, 3), np.float32))[0][0]) for _ in range(20)]
    og = DiskHnsw(O.VECTOR, O.L2_SQUARED, np.zeros((0, 3), np.float32))
    odups = [int(og.insert_on_disk(np.ones((1, 3), np.float32))[0][0]) for _ in range(20)]
    assert dups == odups
    ids, _, _ = gi.search(np.ones(3, np.float32), k=1, ef_search=1)
    e = int(ids[0, 0])
    assert 1 + int(np.sum(gi.export()["dup_of"] == e)) == 10


def test_growing_a_build_keeps_its_recall(pv):
    # low intrinsic dimension (the benchmarks' law): a graph index on it has a meaningful recall
    rng = np.random.default_rng(40)
    frame = np.linalg.qr(rng.standard_normal((64, 16)))[0]
    x = (rng.standard_normal((40000, 16)) @ frame.T + 0.02 * rng.standard_normal((40000, 64))).astype(np.float32)
    q = (rng.standard_normal((200, 16)) @ frame.T + 0.02 * rng.standard_normal((200, 64))).astype(np.float32)
    truth = [O.exact_topk(O.VECTOR, O.L2_SQUARED, qq, x, 10)[0] for qq in q]
    full = pv.HnswIndex("vector_l2_ops", 64).build(x, seed=1)
    grown = pv.HnswIndex("vector_l2_ops", 64).build(x[:20000], seed=1)
    grown.insert(x[20000:], seed=2)
    r_full = recall_at_k(full.search(q, k=10, ef_search=40)[0], truth)
    r_grown = recall_at_k(grown.search(q, k=10, ef_search=40)[0], truth)
    assert r_grown >= r_full - 0.02, (r_grown, r_full)


def test_entry_point_and_levels(pv):
    rng = np.random.default_rng(5)
    rows = rng.standard_normal((3000, 16)).astype(np.float32)
    base_lv = np.zeros(2000, np.int32)
    base_lv[7] = 1
    gi = pv.HnswIndex("vector_l2_ops", 16).build(rows[:2000], levels=base_lv)
    assert gi.export()["entry"] == 7
    new = rows[2000:].copy()
    new[50] = rows[5]                    # folded into element 5: never the entry point, whatever its level
    lv = np.zeros(1000, np.int32)
    lv[50] = 300
    lv[100] = 3
    lv[500] = 200
    lv[600] = 2                          # not above the entry level by then: the entry point stays
    dup, _ = gi.insert(new, levels=lv)
    cap = min((8192 - 24 - 8 - 4 - 4) // 6 // 16 - 2, 63)
    g = gi.export()
    assert dup[50] == 5 and np.sum(dup >= 0) == 1
    assert np.array_equal(g["levels"][2000:], np.minimum(lv, cap))
    assert g["entry"] == 2500 and g["entry_level"] == cap
    ids, dist, _ = gi.search(rows[2000:2040], k=1, ef_search=40)
    assert np.all(dist[:, 0] == 0)


def test_state_filters_handles_and_bad_arguments(pv):
    x, _ = mixture(3000, 16, 10, seed=8)
    gi = pv.HnswIndex("vector_l2_ops", 16).build(x[:2000])
    f = gi.filter(np.arange(0, 2000, 3))
    fs = gi.iterative_scan(x[:4], ef_search=20, max_scan_tuples=200, filter=f, page=10)
    us = gi.iterative_scan(x[:4], ef_search=20, max_scan_tuples=200)
    fs.next_batch()
    us.next_batch()
    snap = gi.export()
    L = pv._lib.load()
    rows = np.ascontiguousarray(x[2000:2100])
    nchg = C.c_int64(0)
    bad = [(rows.ctypes.data_as(C.c_void_p), 100, 16, None),            # ef_construction < 2 * m
           (rows.ctypes.data_as(C.c_void_p), 100, 2000, None),          # ef_construction > 1000
           (rows.ctypes.data_as(C.c_void_p), 100, 64, np.full(100, -1, np.int32)),   # negative level
           (None, 100, 64, None)]
    for ptr, n, efc, lv in bad:
        rc = L.vb_hnsw_insert(gi.h, ptr, n, efc, 1, None if lv is None else lv.ctypes.data_as(C.c_void_p), None, C.byref(nchg))
        assert rc == EINVAL
        after = gi.export()
        assert all(np.array_equal(snap[k], after[k]) for k in ("levels", "nbr0", "upper_off", "upper", "dup_of"))
        assert snap["entry"] == after["entry"]
    with pytest.raises(pv.VecB200Error):
        gi.insert(rows, ef_construction=10)
    dup, recs = gi.insert(rows)
    out = np.empty(len(recs), dtype=pv.HNSW_SLOT_DTYPE)
    assert L.vb_hnsw_insert_changes(gi.h, out.ctypes.data_as(C.c_void_p), len(recs) - 1) == EINVAL
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
    # a filter made after the insert covers the new elements
    f2 = gi.filter(np.arange(2000, 2100))
    with gi.iterative_scan(x[2000:2004], ef_search=20, filter=f2, page=5) as s2:
        ids, _, cnt = s2.next_batch()
    assert np.all(cnt == 5) and np.all((ids >= 2000) & (ids < 2100))
