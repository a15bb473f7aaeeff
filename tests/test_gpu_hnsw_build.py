"""HNSW build on the GPU (vb_hnsw_build = the in-memory build of src/hnswbuild.c:437-480 in batches).

The graph a build produces depends on PRNG level draws and on insertion concurrency (the reference's own parallel
build is not reproducible run to run), so parity is what the reference's tests check: the recall floors of
test/t/012_hnsw_vector_build_recall.pl (>= 0.99 for every vector opclass) and 020_hnsw_bit_build_recall.pl
(>= 0.98 Hamming, >= 0.95 Jaccard) on GPU-built graphs -- plus, on the SAME exported graph, exact equality of the
GPU search with the oracle's search (so the graph arrays mean the same thing to both), structural invariants of
the reference's data structure, and a side-by-side with the oracle's serial build on the same rows."""
import numpy as np
import pytest

import oracle as O
from tests.util import f32_to_half_bits, mixture, recall_at_k

pytestmark = pytest.mark.gpu
RTOL = 1e-5


@pytest.fixture(scope="module")
def pv():
    import pgvector_b200 as pv
    pv.init(0)
    return pv


def gpu_build(pv, opclass, rows, dim=None, m=16, efc=64, seed=7, levels=None):
    d = dim if dim is not None else rows.shape[1]
    gi = pv.HnswIndex(opclass, d, m=m).build(rows, ef_construction=efc, seed=seed, levels=levels)
    return gi, gi.export()


def check_structure(g, n, m):
    """invariants of the reference's graph (src/hnsw.h:150-187, hnswutils.c:1169-1179, 1184-1231)"""
    levels, nbr0, uo, up, dup = g["levels"], g["nbr0"], g["upper_off"], g["upper"], g["dup_of"]
    assert nbr0.shape == (n, 2 * m)
    elem = dup < 0
    # compact lists: a -1 is followed only by -1
    valid = nbr0 >= 0
    assert np.all(valid[:, :-1] | ~valid[:, 1:])
    ids = nbr0[valid]
    assert ids.max() < n and np.all(elem[ids]), "neighbours are elements, never folded duplicates"
    rows_i = np.nonzero(valid)[0]
    assert np.all(ids != rows_i), "no self loops"
    # no repeated neighbour inside a list
    srt = np.sort(np.where(valid, nbr0, np.arange(-1, -1 - 2 * m, -1)[None, :]), axis=1)
    assert np.all(srt[:, 1:] != srt[:, :-1])
    # duplicates carry no connections and never the entry point
    assert not valid[~elem].any()
    assert dup[g["entry"]] < 0 and levels[g["entry"]] == levels[elem].max()
    # upper layers: slots exist exactly for level >= 1 and only reference elements of at least that level
    assert np.all((uo >= 0) == (levels > 0))
    for e in np.nonzero(levels > 0)[0][:2000]:
        for lc in range(1, levels[e] + 1):
            lst = up[uo[e] + lc - 1]
            lst = lst[lst >= 0]
            assert np.all(levels[lst] >= lc) and np.all(lst != e)
    deg = valid.sum(axis=1)[elem]
    return deg


def test_uniform_3d_recall_floor_on_a_gpu_built_graph(pv):
    """test/t/012_hnsw_vector_build_recall.pl: 10k x 3-d, random() * random() per coordinate, defaults (m = 16,
    ef_construction = 64), ef_search = 40, LIMIT 20 -> recall >= 0.99 for <->, <#>, <=>, <+>"""
    rng = np.random.default_rng(12)
    rows = (rng.random((10000, 3)) * rng.random((10000, 3))).astype(np.float32)
    queries = rng.random((20, 3)).astype(np.float32)
    for opclass, metric in (("vector_l2_ops", O.L2_SQUARED), ("vector_ip_ops", O.NEG_IP), ("vector_cosine_ops", O.NEG_IP),
                            ("vector_l1_ops", O.L1)):
        x, q = rows, queries
        if opclass == "vector_cosine_ops":
            keep = np.linalg.norm(rows, axis=1) > 0
            x, q = O.l2_normalize(O.VECTOR, rows[keep]), O.l2_normalize(O.VECTOR, queries)
        gi, g = gpu_build(pv, opclass, x)
        deg = check_structure(g, len(x), 16)
        assert deg.mean() > 8
        ids, _, _ = gi.search(q, k=20, ef_search=40)
        truth = [O.exact_topk(O.VECTOR, metric, qq, x, 20)[0] for qq in q]
        r = recall_at_k(ids, truth)
        assert r >= 0.99, (opclass, r)


@pytest.mark.parametrize("opclass,floor", [("bit_hamming_ops", 0.98), ("bit_jaccard_ops", 0.95)])
def test_bit52_recall_floor_on_a_gpu_built_graph(pv, opclass, floor):
    """test/t/020_hnsw_bit_build_recall.pl: 10k random bit(52), ef_search = 100, LIMIT 20, tie-aware recall
    (a result counts when its distance is within the true k-th distance, :85-91)"""
    elem, metric, _, _ = pv.OPCLASSES[opclass]
    rng = np.random.default_rng(20)
    bits = rng.integers(0, 2, (10000, 52), dtype=np.uint8)
    rows = np.packbits(bits, axis=1)
    queries = np.packbits(rng.integers(0, 2, (20, 52), dtype=np.uint8), axis=1)
    gi, g = gpu_build(pv, opclass, rows, dim=52)
    check_structure(g, 10000, 16)
    ids, dist, _ = gi.search(queries, k=20, ef_search=100)
    hit = tot = 0
    for qq, di in zip(queries, dist):
        kth = O.exact_topk(elem, metric, qq, rows, 20, dim=52)[1][-1]
        hit += int(np.sum(di <= kth))
        tot += 20
    assert hit / tot >= floor, hit / tot


@pytest.mark.parametrize("opclass,dim,n,m,efc", [("vector_l2_ops", 48, 20000, 16, 64), ("halfvec_cosine_ops", 768, 6000, 16, 64),
                                                ("vector_l2_ops", 32, 8000, 8, 40), ("vector_ip_ops", 24, 6000, 40, 100),
                                                ("bit_hamming_ops", 1024, 12000, 16, 64)])
def test_gpu_and_oracle_agree_on_the_gpu_built_graph(pv, opclass, dim, n, m, efc):
    """export -> oracle import: both sides walk the SAME graph, so results are equal query by query (bit-exact for
    bit metrics) and so are the distance-evaluation counts; recall next to the oracle's own serial build of the
    same rows is equal within noise."""
    elem, metric, normalize, _ = pv.OPCLASSES[opclass]
    x, _ = mixture(n, dim, 40, seed=n + dim)
    q, _ = mixture(200, dim, 40, seed=n + dim + 1)
    if elem == O.BIT:
        x, q = O.binary_quantize(O.VECTOR, x), O.binary_quantize(O.VECTOR, q)
    elif elem == O.HALFVEC:
        x, q = f32_to_half_bits(x), f32_to_half_bits(q)
    if normalize:
        x, q = O.l2_normalize(elem, x), O.l2_normalize(elem, q)
    gi, g = gpu_build(pv, opclass, x, dim=dim, m=m, efc=efc)
    deg = check_structure(g, n, m)
    og = O.Hnsw.from_export(elem, metric, x, g, dim=dim)
    ef, k = 80, 10
    ids, dist, nd = gi.search(q, k=k, ef_search=ef)
    wi, wd, wnd = og.search_batch(q, ef, k, ties=O.TIES_TOTAL, threads=8)
    if elem == O.BIT:
        assert np.array_equal(dist, wd) and np.array_equal(ids, wi) and np.array_equal(nd, wnd)
    else:
        assert np.allclose(dist, wd, rtol=RTOL, atol=1e-6)
        same_q = np.all(ids == wi, axis=1)
        assert same_q.mean() > 0.95
        assert np.array_equal(nd[same_q], wnd[same_q])
    # quality next to the reference's serial build (oracle restatement) on the same rows WITH THE SAME LEVEL DRAWS
    # (recall moves by a few points between level draws; measured with shared levels, 8000 x 32, m = 8:
    # serial 0.6945, batches of 1/64 of the graph 0.6955, 1/8 0.6475, one element at a time 0.6945 = the serial build)
    truth = [O.exact_topk(elem, metric, qq, x, k, dim=dim)[0] for qq in q]
    ob = O.Hnsw(elem, metric, x, m=m, ef_construction=efc, seed=7, dim=dim)
    ge = ob.export()
    oi, _, _ = ob.search_batch(q, ef, k, ties=O.TIES_TOTAL, threads=8)
    r_cpu = recall_at_k(ge["elem_row"][np.maximum(oi, 0)], truth)
    if len(ge["levels"]) == n:        # no folded duplicates: element numbers are row numbers
        gi2, g2 = gpu_build(pv, opclass, x, dim=dim, m=m, efc=efc, levels=ge["levels"])
        ids2, _, _ = gi2.search(q, k=k, ef_search=ef)
        r_gpu = recall_at_k(ids2, truth)
        if elem != O.BIT:   # (bit rows tie on distance: id recall is not meaningful; the 52-bit floor test is tie-aware)
            assert r_gpu >= r_cpu - 0.03, (r_gpu, r_cpu)
    # same mean degree as the serial build within a few percent: the heuristic prunes alike
    o_deg = (ge["nbr0"] >= 0).sum(axis=1).mean()
    assert abs(deg.mean() - o_deg) <= 0.15 * o_deg, (deg.mean(), o_deg)


def test_one_element_at_a_time_is_the_serial_build(pv):
    """with batches of one element (option hnsw_build_fraction huge) and the oracle's level draws, the GPU build IS the
    reference's serial build: the same graph, list for list (the restatement of HnswFindElementNeighbors /
    SelectNeighbors / HnswUpdateConnection is exact; only batching changes the graph)"""
    x, _ = mixture(1500, 24, 10, seed=99)
    ob = O.Hnsw(O.VECTOR, O.L2_SQUARED, x, m=8, ef_construction=40, seed=3)
    ge = ob.export()
    assert len(ge["levels"]) == len(x)
    try:
        pv.set_option("hnsw_build_fraction", 1 << 30)
        gi, g = gpu_build(pv, "vector_l2_ops", x, m=8, efc=40, levels=ge["levels"])
    finally:
        pv.set_option("hnsw_build_fraction", 64)
    assert g["entry"] == ge["entry"]
    same0 = np.all(np.sort(g["nbr0"], axis=1) == np.sort(ge["nbr0"], axis=1), axis=1)
    assert same0.mean() > 0.98, same0.mean()        # (fp32 near-ties in the heuristic may differ on a few elements)


def test_caller_supplied_levels_and_first_elements(pv):
    """levels drawn by the caller (the extension passes pg_prng's draws) are used as given, capped at
    HnswGetMaxLevel(m) (src/hnsw.h:133); the entry point is the first element of the highest level
    (src/hnswbuild.c:428-430: replaced only by a strictly higher one)"""
    rng = np.random.default_rng(5)
    rows = rng.standard_normal((3000, 16)).astype(np.float32)
    levels = np.zeros(3000, np.int32)
    levels[[10, 500, 700]] = [2, 3, 3]
    levels[100:130] = 1
    levels[2999] = 200          # capped
    gi, g = gpu_build(pv, "vector_l2_ops", rows, levels=levels)
    cap = min((8192 - 24 - 8 - 4 - 4) // 6 // 16 - 2, 63)
    want = np.minimum(levels, cap)
    assert np.array_equal(g["levels"], want)
    assert g["entry"] == 2999 and g["entry_level"] == cap
    check_structure(g, 3000, 16)
    # the last element only reaches down through the layers that existed before it
    top = g["upper"][g["upper_off"][2999] + 3:g["upper_off"][2999] + cap]
    assert np.all(top == -1)
    ids, dist, _ = gi.search(rows[:50], k=1, ef_search=40)
    assert np.array_equal(ids[:, 0], np.arange(50)) and np.all(dist[:, 0] == 0)


def test_duplicate_rows_are_folded_like_the_reference(pv):
    """FindDuplicateInMemory (src/hnswbuild.c:343-364): a row equal to one of its chosen layer-0 neighbours rides on
    that element (up to HNSW_HEAPTIDS = 10 heap tids per element), it is not inserted"""
    rng = np.random.default_rng(9)
    base = rng.standard_normal((400, 12)).astype(np.float32)
    rows = np.concatenate([base, base[:100], base[:100], rng.standard_normal((600, 12)).astype(np.float32)])
    gi, g = gpu_build(pv, "vector_l2_ops", rows)
    dup = g["dup_of"]
    check_structure(g, len(rows), 16)
    folded = np.nonzero(dup >= 0)[0]
    assert len(folded) >= 150, len(folded)             # (rows of one batch do not see each other: a few become elements)
    assert np.all(folded >= 400) and np.all(folded < 600)
    for e in folded:
        assert np.array_equal(rows[e], rows[dup[e]]) and dup[dup[e]] < 0
    assert np.bincount(dup[folded]).max() <= 9          # 10 heap tids per element including its own
    # every row is still found through its element
    ids, dist, _ = gi.search(rows[400:600], k=1, ef_search=40)
    assert np.all(dist[:, 0] == 0)


def test_tiny_indexes(pv):
    for n in (1, 2, 5, 40):
        rows = np.random.default_rng(n).standard_normal((n, 4)).astype(np.float32)
        gi, g = gpu_build(pv, "vector_l2_ops", rows, m=4, efc=16)
        check_structure(g, n, 4) if n > 1 else None
        ids, dist, _ = gi.search(rows, k=1, ef_search=10)
        assert np.array_equal(ids[:, 0], np.arange(n))
    with pytest.raises(pv.VecB200Error):
        gpu_build(pv, "vector_l2_ops", rows, m=16, efc=16)      # ef_construction < 2 * m is rejected (src/hnswbuild.c:713-716)
