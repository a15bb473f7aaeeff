"""The HNSW kernels at the edges of their route choices, against the oracle.

Three tables pick a kernel instantiation from V, the number of 16-byte words of a table row:
  search (vb_hnsw.cu hnsw_launch_t)          lanes per row 32 for V >= 32, 4 for V 16..31, 8 (one word per lane) for
                                             V == 8, 2 for V 9..15, 1 below 8;
  iterative scan (vb_hnsw_iter.cu)           32 / 4 / 1, split at 32 and 8;
  build, insert, vacuum (vb_hnsw_build.cu)   32 / 8 / 1, split at 32 and 8.
hnsw_score_batch walks a row in steps of LPR words with two steps in flight and a tail for the last one or two, so a
lane-mapping or tail mistake changes the distances of some rows at some widths only.  The widths below sit on both sides
of every split: V = 1, 7, 8, 9, 15, 16, 31, 32, 33, 97 and 500 (vector(2000), halfvec(4000), bit(64000): the largest rows an
index takes).  Neighbour lists are read in chunks of 32 (layer 0 holds 2m, upper layers m entries): m = 2, 16, 17, 32, 33
and 100 cover one chunk, exactly 32 entries, 33, and several chunks.  ef_search and k go to 1 and to 1000, and
ef_construction to 1000.

Searches run on graphs the oracle built (or the GPU built and exported), loaded on both sides, so both walk the same
graph.  Rows and queries are multiples of 1/16 in [-2, 2]: every product, square, absolute difference and partial sum of
a distance is then an exact fp32 value (below 2^24 steps of 1/256 up to 4000 dimensions), exact in half precision too,
and every summation order gives the oracle's distance bit for bit.  So ids, fp32 distances and the distance-evaluation
counts are compared for equality, query by query.  Grid rows tie often; the total order (distance, element) decides
those on both sides.  Cosine is left to the tolerance tests of test_gpu_hnsw.py: normalised grid rows are not exact.
"""
import os

import numpy as np
import pytest

import oracle as O
from tests.test_gpu_hnsw import scan_all
from tests.test_gpu_hnsw_build import check_structure
from tests.test_gpu_hnsw_insert import check_records
from tests.util import f32_to_half_bits, mixture

pytestmark = pytest.mark.gpu
THREADS = os.cpu_count() or 8


@pytest.fixture(scope="module")
def pv():
    import pgvector_b200 as pv
    pv.init(0)
    return pv


def row_words(elem, dim):
    raw = 4 * dim if elem == O.VECTOR else 2 * dim if elem == O.HALFVEC else (dim + 7) // 8
    return (raw + 15) // 16


def grid(elem, n, dim, seed):
    """n rows of multiples of 1/16 in [-2, 2] (bit: random bits, the padding bits of the last byte zero)"""
    rng = np.random.default_rng(seed)
    if elem == O.BIT:
        return np.packbits(rng.integers(0, 2, (n, dim), dtype=np.uint8), axis=1)
    x = rng.integers(-32, 33, (n, dim)).astype(np.float32) / 16
    return f32_to_half_bits(x) if elem == O.HALFVEC else x


_GRAPHS = {}


def oracle_graph(elem, dim, n, m=16, efc=64, seed=1):
    """an oracle-built graph over grid rows (built with L2 / Hamming; a search under another metric walks it all the same):
    (rows in element order, the export)"""
    key = (elem, dim, n, m, efc, seed)
    if key not in _GRAPHS:
        rows = grid(elem, n, dim, seed)
        og = O.Hnsw(elem, O.HAMMING if elem == O.BIT else O.L2_SQUARED, rows, m=m, ef_construction=efc, seed=seed, dim=dim)
        g = og.export()
        _GRAPHS[key] = (rows[g["elem_row"]], g)
    return _GRAPHS[key]


def pair(pv, opclass, erows, g, dim):
    elem, metric, _, _ = pv.OPCLASSES[opclass]
    og = O.Hnsw.from_export(elem, metric, erows, g, dim=dim)
    gi = pv.HnswIndex(opclass, dim, m=g["m"]).load(erows, g["levels"], g["nbr0"], g["upper_off"], g["upper"], g["entry"])
    return og, gi


def assert_same_search(og, gi, queries, ef, k, what):
    ids, dist, nd = gi.search(queries, k=k, ef_search=ef)
    wi, wd, wnd = og.search_batch(queries, ef, k, ties=O.TIES_TOTAL, threads=THREADS)
    bad = np.nonzero(~(np.all(ids == wi, axis=1) & np.all(dist == wd, axis=1) & (nd == wnd)))[0]
    assert len(bad) == 0, f"{what}: {len(bad)} of {len(queries)} queries differ, first {bad[:8].tolist()}"
    assert np.all(ids[:, 0] >= 0)
    return ids


def assert_same_scan(og, gi, queries, ef, max_scan_tuples, what):
    """hnsw.iterative_scan: every batch, element for element, with the oracle's distances and tuples counter"""
    ids, dist, sizes, tuples = scan_all(gi, queries, ef, max_scan_tuples)
    for q in range(len(queries)):
        wi, wd, wb, wt = og.iter_scan(queries[q], ef, max_scan_tuples=max_scan_tuples, ties=O.TIES_TOTAL)
        assert ids[q] == wi.tolist(), f"{what}: query {q}"
        assert np.array_equal(np.array(dist[q]), wd), f"{what}: query {q}"
        assert int(tuples[q]) == wt, f"{what}: query {q}"
        searched = [int((wb == b).sum()) for b in range(int(wb.max()) + 1)] if len(wb) else []
        assert sizes[q][:len(searched)] == searched, f"{what}: query {q}"


# ------------------------------------------------------------------------------------------------ every row width

VECTOR_DIMS = [3, 27, 29, 32, 33, 59, 61, 123, 125, 128, 129, 387, 2000]
HALFVEC_DIMS = [5, 55, 57, 72, 120, 128, 248, 256, 257, 775, 4000]
BIT_DIMS = [52, 833, 1024, 1025, 1920, 2048, 3968, 4096, 4097, 12400, 64000]
L1_DIMS = {29, 61, 125, 2000, 57, 128, 256, 4000}
WIDTHS = [("vector", d) for d in VECTOR_DIMS] + [("halfvec", d) for d in HALFVEC_DIMS] + [("bit", d) for d in BIT_DIMS]
ELEMS = {"vector": O.VECTOR, "halfvec": O.HALFVEC, "bit": O.BIT}


def width_rows(elem, dim):
    return 2000 if row_words(elem, dim) <= 64 else 1200


@pytest.mark.parametrize("kind,dim", WIDTHS)
def test_search_is_exact_at_every_row_width(pv, kind, dim):
    """search of every opclass of the type (cosine excepted) at ef_search 64, k 20 and at ef_search 1, k 1: the same ids,
    fp32 distances and tuples counts as the oracle for every query"""
    elem = ELEMS[kind]
    V = row_words(elem, dim)
    erows, g = oracle_graph(elem, dim, width_rows(elem, dim))
    queries = grid(elem, 96, dim, seed=1000 + dim)
    if elem == O.BIT:
        opclasses = ["bit_hamming_ops", "bit_jaccard_ops"]
    else:
        opclasses = [f"{kind}_l2_ops", f"{kind}_ip_ops"] + ([f"{kind}_l1_ops"] if dim in L1_DIMS else [])
    for opclass in opclasses:
        og, gi = pair(pv, opclass, erows, g, dim)
        for ef, k in ((64, 20), (1, 1)):
            assert_same_search(og, gi, queries, ef, k, f"{opclass}({dim}) V={V} ef={ef} k={k}")


@pytest.mark.parametrize("kind,dim", [("vector", 2000), ("halfvec", 4000), ("bit", 64000)])
def test_search_at_ef_1000_on_the_largest_rows(pv, kind, dim):
    """k = ef_search = 1000 (and k = 1 at ef_search 1000) on the widest rows: R and the query image at their largest"""
    elem = ELEMS[kind]
    erows, g = oracle_graph(elem, dim, 1500, seed=2)
    queries = grid(elem, 16, dim, seed=2000 + dim)
    opclass = "bit_hamming_ops" if elem == O.BIT else f"{kind}_l2_ops"
    og, gi = pair(pv, opclass, erows, g, dim)
    for k in (1000, 1):
        assert_same_search(og, gi, queries, 1000, k, f"{opclass}({dim}) ef=1000 k={k}")


# ------------------------------------------------------------------------------------------------ neighbour lists

LIST_M = [2, 16, 17, 32, 33, 100]


@pytest.mark.parametrize("m", LIST_M)
@pytest.mark.parametrize("dim", [27, 129])
def test_search_reads_every_chunk_of_long_neighbour_lists(pv, m, dim):
    """layer-0 lists of 2m and upper lists of m entries, read 32 at a time: ef_search 1 and 1000, k 1 and ef, on a narrow
    (V = 7) and a wide (V = 33) row"""
    n = 1500 if m == 100 else 3000
    erows, g = oracle_graph(O.VECTOR, dim, n, m=m, efc=max(64, 2 * m), seed=3)
    full0 = (g["nbr0"] >= 0).sum(axis=1)
    assert full0.max() == 2 * m                      # (lists as long as the layer allows)
    if m <= 33:
        assert (g["upper"] >= 0).sum(axis=1).max() == m
    queries = grid(O.VECTOR, 32, dim, seed=3000 + dim)
    og, gi = pair(pv, "vector_l2_ops", erows, g, dim)
    for ef, k in ((1, 1), (1000, 1), (1000, 1000)):
        assert_same_search(og, gi, queries, ef, k, f"m={m} vector({dim}) ef={ef} k={k}")


# ------------------------------------------------------------------------------------------------ iterative scan

@pytest.mark.parametrize("dim", [27, 29, 123, 125])
def test_iterative_scan_is_exact_at_its_splits(pv, dim):
    """the iterative scan's lanes-per-row splits (V = 7 / 8 and 31 / 32)"""
    erows, g = oracle_graph(O.VECTOR, dim, width_rows(O.VECTOR, dim))
    queries = grid(O.VECTOR, 12, dim, seed=4000 + dim)
    for opclass in ("vector_l2_ops", "vector_ip_ops"):
        og, gi = pair(pv, opclass, erows, g, dim)
        assert_same_scan(og, gi, queries, 40, 1000, f"{opclass}({dim})")


@pytest.mark.parametrize("kind,dim", [("vector", 2000), ("halfvec", 4000), ("bit", 64000)])
def test_iterative_scan_at_ef_1000_on_the_largest_rows(pv, kind, dim):
    elem = ELEMS[kind]
    erows, g = oracle_graph(elem, dim, 1500, seed=2)
    queries = grid(elem, 4, dim, seed=5000 + dim)
    opclass = "bit_hamming_ops" if elem == O.BIT else f"{kind}_l2_ops"
    og, gi = pair(pv, opclass, erows, g, dim)
    assert_same_scan(og, gi, queries, 1000, 1400, f"{opclass}({dim})")


def test_iterative_scan_with_m_100(pv):
    erows, g = oracle_graph(O.VECTOR, 27, 1500, m=100, efc=200, seed=3)
    queries = grid(O.VECTOR, 8, 27, seed=6000)
    og, gi = pair(pv, "vector_l2_ops", erows, g, 27)
    assert_same_scan(og, gi, queries, 100, 1200, "m=100")


# ------------------------------------------------------------------------------------------------ build and insert

@pytest.mark.parametrize("opclass,dim,n,m,efc", [
    ("vector_l2_ops", 24, 1500, 100, 1000),
    ("vector_l2_ops", 2000, 1000, 16, 64),
    ("halfvec_l2_ops", 4000, 800, 16, 1000),     # R of 1000 entries does not fit beside two 16 KB row images: global R
    ("halfvec_ip_ops", 4000, 800, 100, 663),
    ("bit_hamming_ops", 64000, 1000, 16, 64),
])
def test_build_and_insert_at_the_limits(pv, opclass, dim, n, m, efc):
    """a GPU build and a GPU insert at m = 100 / ef_construction = 1000 and on the largest rows: the graph keeps the
    reference's invariants, the insert's records are the exact slot diff, and the GPU and the oracle search the exported
    graph alike"""
    elem, metric, _, _ = pv.OPCLASSES[opclass]
    rows = grid(elem, n + n // 4, dim, seed=7 + dim)
    gi = pv.HnswIndex(opclass, dim, m=m).build(rows[:n], ef_construction=efc, seed=5)
    g = gi.export()
    deg = check_structure(g, n, m)
    assert deg.mean() > min(m, 8)
    before = g
    dup, recs = gi.insert(rows[n:], ef_construction=efc, seed=6)
    g = gi.export()
    check_structure(g, len(rows), m)
    check_records(before, g, recs)
    erows = rows
    og = O.Hnsw.from_export(elem, metric, erows, g, dim=dim)
    gi2 = pv.HnswIndex(opclass, dim, m=m).load(erows, g["levels"], g["nbr0"], g["upper_off"], g["upper"], g["entry"])
    queries = grid(elem, 32, dim, seed=8 + dim)
    for ef, k in ((64, 10), (1000, 1000)):
        assert_same_search(og, gi2, queries, ef, k, f"{opclass}({dim}) m={m} efc={efc} ef={ef}")
    # the built image searches like its own export
    ids, dist, nd = gi.search(queries, k=10, ef_search=64)
    ids2, dist2, nd2 = gi2.search(queries, k=10, ef_search=64)
    assert np.array_equal(ids, ids2) and np.array_equal(dist, dist2) and np.array_equal(nd, nd2)


@pytest.mark.parametrize("dim", [27, 29, 123, 125, 129])
def test_one_element_at_a_time_is_the_serial_build_at_every_split(pv, dim):
    """the build's lanes-per-row splits (V = 7 / 8, 31 / 32 / 33): batches of one element with the oracle's level draws
    are the oracle's serial build, list for list (the bar of test_one_element_at_a_time_is_the_serial_build: float rows,
    a near tie may send a few lists apart)"""
    x, _ = mixture(1500, dim, 10, seed=99 + dim)
    ob = O.Hnsw(O.VECTOR, O.L2_SQUARED, x, m=8, ef_construction=40, seed=3)
    ge = ob.export()
    assert len(ge["levels"]) == len(x)
    try:
        pv.set_option("hnsw_build_fraction", 1 << 30)
        gi = pv.HnswIndex("vector_l2_ops", dim, m=8).build(x, ef_construction=40, levels=ge["levels"])
    finally:
        pv.set_option("hnsw_build_fraction", 64)
    g = gi.export()
    assert g["entry"] == ge["entry"]
    same0 = np.all(np.sort(g["nbr0"], axis=1) == np.sort(ge["nbr0"], axis=1), axis=1)
    assert same0.mean() > 0.98, same0.mean()
