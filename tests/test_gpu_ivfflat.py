"""GPU parity of the IVFFlat scan path (GetScanLists / GetScanItems, src/ivfscan.c) vs the oracle."""
import numpy as np
import pytest

import oracle as O
from tests.util import assert_same_neighbours, build_ivf_arrays, f32_to_half_bits, load_golden, mixture, parse_vector, recall_at_k

pytestmark = pytest.mark.gpu
RTOL = 1e-5


@pytest.fixture(scope="module")
def pv():
    import pgvector_b200 as pv
    pv.init(0)
    import os
    pv.set_option("scan_impl", int(os.environ.get("VB_TEST_SCAN_IMPL", "2")))
    # equal centre distances are broken by list number on the GPU; put the oracle in the same
    # deterministic instance (the pairing-heap order is compared by recall, see test_tie_modes_agree_on_recall)
    O.ivf_set_tie_mode(True)
    yield pv
    O.ivf_set_tie_mode(False)


def make_index(pv, opclass, rows, centers, dim=None):
    elem, metric, _, _ = pv.OPCLASSES[opclass]
    lists = centers.shape[0]
    assign = O.ivf_assign(elem, metric, rows, centers, threads=8, dim=dim)
    grouped, ids, offsets = build_ivf_arrays(rows, assign, lists)
    d = dim if dim is not None else rows.shape[1]
    gix = pv.IvfflatIndex(opclass, d, lists).load(centers, offsets, grouped, ids)
    oix = O.Ivf(elem, metric, centers, offsets, grouped, ids, dim=d)
    return gix, oix


@pytest.fixture(scope="module")
def l2_index(pv):
    rows, centers = mixture(30000, 96, 64, seed=3)
    queries, _ = mixture(200, 96, 64, seed=4)
    gix, oix = make_index(pv, "vector_l2_ops", rows, centers)
    return gix, oix, rows, queries


def test_scan_lists_matches_oracle(l2_index):
    gix, oix, rows, queries = l2_index
    for mp in (1, 5, 64, 100):
        lists, dist = gix.scan_lists(queries[:50], mp)
        for i in range(50):
            wl, wd = oix.scan_lists(queries[i], mp)
            n = len(wl)
            assert np.array_equal(lists[i][:n], wl), (mp, i)
            assert np.allclose(dist[i][:n], wd, rtol=RTOL)
            assert np.all(lists[i][n:] == -1)


def test_scan_items_full_sort_matches_oracle(l2_index):
    gix, oix, rows, queries = l2_index
    for i in range(5):
        wl, _ = oix.scan_lists(queries[i], 7)
        ids, dist, n = gix.scan_items(queries[i], wl)
        wi, wd, wn = oix.search(queries[i], 7, 0)
        assert n == wn == len(ids)
        assert np.allclose(dist, wd, rtol=RTOL)
        assert np.all(np.diff(dist) >= 0)
        # same multiset of heap ids; order equal except fp near-ties
        assert sorted(ids) == sorted(wi)
        assert (ids == wi).mean() > 0.995
        # cap smaller than the candidate count: a sorted prefix
        ids2, dist2, n2 = gix.scan_items(queries[i], wl, cap=17)
        assert n2 == wn and np.array_equal(ids2, ids[:17])


def test_scan_items_null_query_returns_everything_at_zero(l2_index):
    gix, oix, rows, queries = l2_index
    ids, dist, n = gix.scan_items(None, [3, 9])
    wi, wd, wn = oix.search(None, 2, 0)   # oracle: first two lists by its tie rule differ; compare counts/zeros
    assert n == len(ids) and np.all(dist == 0)
    lo = sorted(int(x) for x in ids)
    assert lo == sorted(int(x) for x in np.concatenate([oix.ids[oix.offsets[3]:oix.offsets[4]], oix.ids[oix.offsets[9]:oix.offsets[10]]]))


@pytest.mark.parametrize("probes,k", [(1, 10), (8, 10), (64, 100), (5, 1), (10, 3000)])
def test_search_matches_oracle(l2_index, probes, k):
    gix, oix, rows, queries = l2_index
    ids, dist = gix.search(queries, k=k, probes=probes)
    wi, wd = oix.search_batch(queries, probes, k, threads=8)
    finite = np.isfinite(wd)
    assert np.array_equal(np.isfinite(dist), finite)
    assert np.allclose(dist[finite], wd[finite], rtol=RTOL)
    # ranks may swap only between candidates whose distances agree to rounding (k = 3000 of ~4700 candidates
    # has neighbouring gaps of 1e-4 relative; fp32 summation order moves a distance by ~1e-6)
    assert_same_neighbours(ids, dist, wi, wd, RTOL, min_positional=0.998 if k <= 100 else 0.99)
    assert np.array_equal(ids < 0, wi < 0)
    # recall is identical to the oracle's at the same probes (north_star)
    kk = min(k, 10)
    truth = [O.exact_topk(O.VECTOR, O.L2_SQUARED, q, rows, kk)[0] for q in queries[:50]]
    r_gpu = recall_at_k(ids[:50, :kk], truth)
    r_cpu = recall_at_k(wi[:50, :kk], truth)
    assert abs(r_gpu - r_cpu) < 1e-3


def test_probes_equal_lists_is_exact(l2_index):
    """test/t/003_ivfflat_vector_build_recall.pl:114-116: probes = lists gives recall 1.0"""
    gix, oix, rows, queries = l2_index
    ids, dist = gix.search(queries[:40], k=10, probes=64)
    truth = [O.exact_topk(O.VECTOR, O.L2_SQUARED, q, rows, 10)[0] for q in queries[:40]]
    assert recall_at_k(ids, truth) >= 0.999


def test_self_query_recall_is_100_percent(l2_index):
    """test/t/005_ivfflat_query_recall.pl:23-32: a stored row is its own nearest neighbour at probes=1...lists"""
    gix, oix, rows, queries = l2_index
    pick = rows[::1500][:20]
    ids, dist = gix.search(pick, k=1, probes=64)
    assert np.all(dist[:, 0] == 0)
    assert np.array_equal(ids[:, 0], np.arange(0, 30000, 1500)[:20])


@pytest.mark.parametrize("opclass,dim", [("vector_ip_ops", 40), ("vector_cosine_ops", 40), ("halfvec_l2_ops", 72),
                                         ("halfvec_cosine_ops", 768), ("bit_hamming_ops", 52), ("bit_hamming_ops", 1024)])
def test_other_opclasses(pv, opclass, dim):
    elem, metric, normalize, _ = pv.OPCLASSES[opclass]
    lists = 20
    x, c = mixture(6000, dim, lists, seed=11)
    q, _ = mixture(60, dim, lists, seed=12)
    if elem == O.BIT:
        rows, centers, queries = O.binary_quantize(O.VECTOR, x), O.binary_quantize(O.VECTOR, c), O.binary_quantize(O.VECTOR, q)
    else:
        if elem == O.HALFVEC:
            x, c, q = f32_to_half_bits(x), f32_to_half_bits(c), f32_to_half_bits(q)
        rows, centers, queries = x, c, q
        if normalize or metric == O.NEG_IP:
            # cosine opclasses index normalised rows and normalise the query (src/ivfscan.c:222-229);
            # ip k-means centres are unit vectors too (src/ivfkmeans.c:233-235)
            rows, centers, queries = O.l2_normalize(elem, rows), O.l2_normalize(elem, centers), O.l2_normalize(elem, queries)
    gix, oix = make_index(pv, opclass, rows, centers, dim=dim)
    ids, dist = gix.search(queries, k=10, probes=4)
    wi, wd = oix.search_batch(queries, 4, 10, threads=8)
    if elem == O.BIT:
        assert np.array_equal(dist, wd)
        # Hamming ties are constant: identical ids are required only up to equal-distance groups
        for i in range(len(queries)):
            assert sorted(zip(dist[i], ids[i])) == sorted(zip(wd[i], wi[i])) or set(dist[i]) == set(wd[i])
        assert np.array_equal(ids, wi)   # both sides break ties by scan order
    else:
        assert np.allclose(dist, wd, rtol=RTOL, atol=1e-6)
        assert (ids == wi).mean() > 0.99


@pytest.mark.parametrize("opclass,dim", [("vector_l2_ops", 3), ("vector_l2_ops", 96), ("vector_ip_ops", 40), ("vector_cosine_ops", 50),
                                         ("halfvec_l2_ops", 72), ("halfvec_ip_ops", 130), ("halfvec_cosine_ops", 768)])
def test_list_major_scan_equals_per_query_scan(pv, opclass, dim):
    """The batched (list-major) scan writes the same candidate runs as the per-query scans: several row tiles per
    list (one of them partial), query groups larger than one 32-query sub-tile, dimensions that end inside a
    16-element staging step."""
    elem, metric, normalize, _ = pv.OPCLASSES[opclass]
    lists = 12
    x, c = mixture(9000, dim, lists, seed=21)
    q, _ = mixture(300, dim, lists, seed=22)
    if elem == O.HALFVEC:
        x, c, q = f32_to_half_bits(x), f32_to_half_bits(c), f32_to_half_bits(q)
    if normalize or metric == O.NEG_IP:
        x, c, q = O.l2_normalize(elem, x), O.l2_normalize(elem, c), O.l2_normalize(elem, q)
    gix, oix = make_index(pv, opclass, x, c, dim=dim)
    got = {}
    try:
        for impl in (0, 1, 3, 4):
            pv.set_option("scan_impl", impl)
            got[impl] = gix.search(q, k=10, probes=5)
            got[impl, 1] = gix.search(q[:3], k=7, probes=12)      # tiny batch, every list probed
    finally:
        import os
        pv.set_option("scan_impl", int(os.environ.get("VB_TEST_SCAN_IMPL", "2")))
    wi, wd = oix.search_batch(q, 5, 10, threads=8)
    for impl in (0, 1, 3, 4):
        ids, dist = got[impl]
        assert np.allclose(dist, wd, rtol=RTOL, atol=1e-6), impl
        assert (ids == wi).mean() > 0.99, impl
    # the tensor-core filter re-scores with the per-query scan arithmetic: same values as the streaming kernels
    assert np.allclose(got[4][1], got[1][1], rtol=RTOL, atol=1e-6)
    assert (got[4][0] == got[1][0]).mean() > 0.995
    assert np.allclose(got[3][1], got[1][1], rtol=RTOL, atol=1e-6)
    assert (got[3][0] == got[1][0]).mean() > 0.995
    assert np.allclose(got[3, 1][1], got[0, 1][1], rtol=RTOL, atol=1e-6)
    assert (got[3, 1][0] == got[0, 1][0]).mean() > 0.99


@pytest.mark.parametrize("lists", [160, 3000, 5000])
@pytest.mark.parametrize("opclass", ["vector_l2_ops", "vector_cosine_ops", "halfvec_l2_ops"])
def test_probe_selection_through_the_tensor_core_filter(pv, opclass, lists):
    """GetScanLists for a query batch over >= 128 centres runs the filter + exact re-score + certificate: the probed
    lists and their order equal the exact kernels' and the oracle's.  Up to 4096 centres the refine kernel selects the
    run of centre distances itself; 5000 are selected by a launch of their own first."""
    import os
    elem, metric, normalize, _ = pv.OPCLASSES[opclass]
    dim = 48
    x, c = mixture(16000, dim, lists, seed=31)
    q, _ = mixture(320, dim, lists, seed=32)
    if elem == O.HALFVEC:
        x, c, q = f32_to_half_bits(x), f32_to_half_bits(c), f32_to_half_bits(q)
    if normalize:
        x, c, q = O.l2_normalize(elem, x), O.l2_normalize(elem, c), O.l2_normalize(elem, q)
    gix, oix = make_index(pv, opclass, x, c, dim=dim)
    try:
        pv.set_option("scan_impl", 3)
        l3, d3 = gix.scan_lists(q, 7)
        i3, s3 = gix.search(q, k=10, probes=7)
        pv.set_option("scan_impl", 4)
        l4, d4 = gix.scan_lists(q, 7)
        i4, s4 = gix.search(q, k=10, probes=7)
    finally:
        pv.set_option("scan_impl", int(os.environ.get("VB_TEST_SCAN_IMPL", "2")))
    assert np.array_equal(l3, l4)
    assert np.allclose(d3, d4, rtol=RTOL, atol=1e-6)
    for i in range(0, 320, 16):
        wl, wd = oix.scan_lists(q[i], 7)
        assert np.array_equal(l4[i][:len(wl)], wl), i
        assert np.allclose(d4[i][:len(wl)], wd, rtol=RTOL, atol=1e-6)
    assert np.allclose(s3, s4, rtol=RTOL, atol=1e-6)
    assert (i3 == i4).mean() > 0.995


@pytest.mark.parametrize("latent", [0, 8])
def test_filter_levels_return_identical_results(pv, latent):
    """Level 1 (hi plane of the rows only) and level 2 (both planes) of the tensor-core filter end in the same exact
    re-score, so whatever level certifies a batch the output is bit-identical.  Isotropic data (latent = 0) has
    neighbour gaps below the level-1 bound -> escalation to level 2; low intrinsic dimension certifies at level 1."""
    import os
    rng = np.random.default_rng(41)
    if latent:
        frame = np.linalg.qr(rng.standard_normal((64, latent)))[0].astype(np.float32)
        x = (rng.standard_normal((20000, latent)).astype(np.float32) @ frame.T + 0.01 * rng.standard_normal((20000, 64))).astype(np.float32)
        q = (rng.standard_normal((400, latent)).astype(np.float32) @ frame.T + 0.01 * rng.standard_normal((400, 64))).astype(np.float32)
        c = x[rng.choice(20000, 40, replace=False)].copy()
    else:
        x, c = mixture(20000, 64, 40, seed=42)
        q, _ = mixture(400, 64, 40, seed=43)
    gix, oix = make_index(pv, "vector_l2_ops", x, c)
    try:
        pv.set_option("scan_impl", 4)
        pv.set_option("tc_level1", 0)
        i2, d2 = gix.search(q, k=10, probes=6)
        before = gix.tc_level1_fallbacks()
        pv.set_option("tc_level1", 1)
        i1, d1 = gix.search(q, k=10, probes=6)
        l1_failed = gix.tc_level1_fallbacks() - before
        i1b, d1b = gix.search(q, k=10, probes=6)          # while level 1 rests after a failure
    finally:
        pv.set_option("tc_level1", 1)
        pv.set_option("scan_impl", int(os.environ.get("VB_TEST_SCAN_IMPL", "2")))
    assert np.array_equal(i1, i2) and np.array_equal(d1, d2)
    assert np.array_equal(i1b, i2) and np.array_equal(d1b, d2)
    if latent:
        assert l1_failed == 0          # well separated neighbours: the cheap level is enough
    wi, wd = oix.search_batch(q, 6, 10, threads=8)
    assert np.allclose(d1, wd, rtol=RTOL, atol=1e-6)
    assert (i1 == wi).mean() > 0.99


def test_prefetched_search_equals_search(pv, l2_index):
    """The pipelined host path (copy of batch i + 1 on a second stream while batch i computes) returns exactly what
    vb_ivf_search returns; dimensions that are not a multiple of 4 are refused."""
    import torch
    gix, oix, rows, queries = l2_index
    batches = [torch.from_numpy(np.ascontiguousarray(queries[i * 50:(i + 1) * 50])).pin_memory().numpy() for i in range(4)]
    want = [gix.search(b, k=10, probes=8) for b in batches]
    ids = np.empty((50, 10), dtype=np.int64)
    dist = np.empty((50, 10), dtype=np.float64)
    gix.prefetch_queries(batches[0], 0)
    for i in range(4):
        if i + 1 < 4:
            gix.prefetch_queries(batches[i + 1], (i + 1) % 2)
        gix.search_prefetched_into(i % 2, 10, 8, ids, dist)
        assert np.array_equal(ids, want[i][0]), i
        assert np.array_equal(dist, want[i][1]), i
    with pytest.raises(pv.VecB200Error):
        gix.search_prefetched_into(0, 10, 8, ids, dist)      # slot already consumed
    x, c = mixture(500, 6, 4, seed=51)
    odd, _ = make_index(pv, "vector_l2_ops", x, c)
    with pytest.raises(pv.VecB200Error):
        odd.prefetch_queries(x[:8], 0)                       # dim % 4 != 0


def test_tensor_core_filter_falls_back_when_it_cannot_certify(pv):
    """More duplicates of the nearest row than candidates kept per query put the k-th and the k'-th candidate at
    the same approximate distance, so no filter level can certify: those batches must come back from the exact
    kernel, identical to the other scan settings, and be counted."""
    import os
    rng = np.random.default_rng(5)
    base = rng.standard_normal((40, 64)).astype(np.float32)
    rows = np.repeat(base, 200, axis=0)                      # 8000 rows, every vector 200 times (> the 128 candidates kept)
    centers = base[:8].copy()
    q = (base[rng.integers(0, 40, 300)] + 0.01 * rng.standard_normal((300, 64))).astype(np.float32)
    gix, oix = make_index(pv, "vector_l2_ops", rows, centers)
    try:
        pv.set_option("scan_impl", 3)
        ids3, d3 = gix.search(q, k=10, probes=8)
        before = gix.tc_fallbacks()
        pv.set_option("scan_impl", 4)
        ids4, d4 = gix.search(q, k=10, probes=8)
        assert gix.tc_fallbacks() > before
    finally:
        pv.set_option("scan_impl", int(os.environ.get("VB_TEST_SCAN_IMPL", "2")))
    assert np.array_equal(ids3, ids4)
    assert np.array_equal(d3, d4)
    wi, wd = oix.search_batch(q, 8, 10, threads=8)
    assert np.allclose(d4, wd, rtol=RTOL, atol=1e-6)


def test_tie_modes_agree_on_recall(pv):
    """Hamming centre distances tie constantly: the reference's pairing-heap order and the GPU's
    (distance, list) order may probe different lists among equals, never worse ones"""
    x, c = mixture(6000, 52, 20, seed=11)
    q, _ = mixture(60, 52, 20, seed=12)
    rows, centers, queries = O.binary_quantize(O.VECTOR, x), O.binary_quantize(O.VECTOR, c), O.binary_quantize(O.VECTOR, q)
    gix, oix = make_index(pv, "bit_hamming_ops", rows, centers, dim=52)
    ids, dist = gix.search(queries, k=10, probes=4)
    O.ivf_set_tie_mode(False)
    try:
        wi, wd = oix.search_batch(queries, 4, 10, threads=8)
        ll, ld = oix.scan_lists(queries[0], 4)
    finally:
        O.ivf_set_tie_mode(True)
    gl, gd = gix.scan_lists(queries[:1], 4)
    assert np.array_equal(gd[0], ld)                      # same probe distances, possibly different equal-distance lists
    assert abs(dist[:, -1].mean() - wd[:, -1].mean()) < 0.5   # k-th distance statistically the same


def test_reference_index_orderings(pv):
    """tiny-table orderings of test/expected/ivfflat_*.out (no ties in them)"""
    blocks = [b for b in load_golden("index_orderings.json")["blocks"] if b["index"]["am"] == "ivfflat"]
    assert len(blocks) >= 7
    ELEMS = {"vector": O.VECTOR, "halfvec": O.HALFVEC, "bit": O.BIT}
    for b in blocks:
        elem = ELEMS[b["type"]]
        opclass = b["index"]["opclass"]
        _, metric, normalize, _ = pv.OPCLASSES[opclass]
        lists = int(b["index"]["options"].split("=")[1]) if "lists" in b["index"]["options"] else 100
        texts = [v for grp in b["rows"] for v in grp["values"] if v is not None]
        rows = np.stack([parse_vector(t, elem)[0] for t in texts])
        keep = np.ones(len(texts), bool)
        stored = rows
        if normalize:
            keep = np.array([O.norm(elem, r) > 0 for r in rows])      # zero vectors are not indexed
            stored = O.l2_normalize(elem, rows[keep])
        dim = b["dim"]
        # lists = 1: the single centre is irrelevant for the ordering; lists = 3: one row per list
        if lists == 1:
            centers = stored[:1].copy()
        else:
            centers = stored[:lists].copy()
        gix, oix = make_index(pv, opclass, stored, centers, dim=dim)
        kept_texts = [t for t, kp in zip(texts, keep) if kp]
        qry = b["queries"][0]
        qv = parse_vector(qry["query"], elem)[0]
        if normalize:
            qv = O.l2_normalize(elem, qv)
        ids, dist, n = gix.scan_items(qv, list(range(lists)))
        got = [kept_texts[i] for i in ids]
        want = qry["expected"]
        assert got[:len(want)] == want, (b["source"], got, want)


def test_device_pointer_variants_match_host_variants(pv, l2_index):
    """vb_ivf_load_dev / vb_ivf_search_dev / vb_exact_topk_dev (torch CUDA tensors in, out) == host-buffer calls"""
    import torch
    gix, oix, rows, queries = l2_index
    dev = torch.device("cuda", 0)
    centers_t = torch.from_numpy(oix.centers).to(dev)
    rows_t = torch.from_numpy(oix.rows).to(dev)
    ids_t = torch.from_numpy(oix.ids).to(dev)
    q_t = torch.from_numpy(queries).to(dev)
    torch.cuda.synchronize()
    dix = pv.IvfflatIndex("vector_l2_ops", 96, 64).load(centers_t, oix.offsets, rows_t, ids_t)
    ids_d, dist_d = dix.search(q_t, k=10, probes=8)
    ids_h, dist_h = gix.search(queries, k=10, probes=8)
    assert np.array_equal(ids_d.cpu().numpy(), ids_h)
    assert np.allclose(dist_d.cpu().numpy(), dist_h, rtol=1e-6)
    assert dix.last_candidates() > 0 and dix.last_scan_bytes() == (len(queries) * 64 + dix.last_candidates()) * 96 * 4
    t = pv.Table(O.VECTOR, 96).append(rows_t)
    e_ids, e_dist = t.exact_topk(O.L2_SQUARED, q_t[:20].contiguous(), 5)
    h_ids, h_dist = pv.Table(O.VECTOR, 96).append(oix.rows).exact_topk(O.L2_SQUARED, queries[:20], 5)
    assert np.array_equal(e_ids.cpu().numpy(), h_ids)
    assert np.allclose(e_dist.cpu().numpy(), h_dist, rtol=1e-6)


def test_list_at_a_time_load_and_replace_list(pv):
    """vb_ivf_begin_load / vb_ivf_load_list / vb_ivf_end_load build the image vb_ivf_load builds, and
    vb_ivf_replace_list swaps one list (growing, shrinking, emptying it) -- every scan kernel sees the new rows"""
    import os
    rows, centers = mixture(12000, 64, 24, seed=61)
    queries, _ = mixture(300, 64, 24, seed=62)
    assign = O.ivf_assign(O.VECTOR, O.L2_SQUARED, rows, centers, threads=8)
    grouped, ids, offsets = build_ivf_arrays(rows, assign, 24)
    whole = pv.IvfflatIndex("vector_l2_ops", 64, 24).load(centers, offsets, grouped, ids)
    parts = [(l, grouped[offsets[l]:offsets[l + 1]], ids[offsets[l]:offsets[l + 1]]) for l in range(24) if offsets[l + 1] > offsets[l]]
    piece = pv.IvfflatIndex("vector_l2_ops", 64, 24).load_by_list(centers, parts)
    for impl in (0, 3, 4):
        pv.set_option("scan_impl", impl)
        a, b = whole.search(queries, k=10, probes=5), piece.search(queries, k=10, probes=5)
        assert np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1]), impl
    # replace three lists: one grows (rows moved in from list 9), list 9 shrinks accordingly, list 3 becomes empty
    g2, i2, off2 = grouped.copy(), ids.copy(), offsets.copy()
    cur = {l: (g2[off2[l]:off2[l + 1]].copy(), i2[off2[l]:off2[l + 1]].copy()) for l in range(24)}
    take = len(cur[9][0]) // 2
    cur[5] = (np.concatenate([cur[5][0], cur[9][0][:take]]), np.concatenate([cur[5][1], cur[9][1][:take]]))
    cur[9] = (cur[9][0][take:], cur[9][1][take:])
    moved3 = cur[3]
    cur[3] = (cur[3][0][:0], cur[3][1][:0])
    cur[4] = (np.concatenate([cur[4][0], moved3[0]]), np.concatenate([cur[4][1], moved3[1]]))
    try:
        pv.set_option("scan_impl", 4)
        piece.search(queries, k=10, probes=5)          # the packed planes exist before the swap
        for l in (5, 9, 3, 4):
            piece.replace_list(l, cur[l][0], cur[l][1])
        new_rows = np.concatenate([cur[l][0] for l in range(24)])
        new_ids = np.concatenate([cur[l][1] for l in range(24)])
        new_off = np.concatenate([[0], np.cumsum([len(cur[l][0]) for l in range(24)])]).astype(np.int64)
        fresh = pv.IvfflatIndex("vector_l2_ops", 64, 24).load(centers, new_off, new_rows, new_ids)
        oix = O.Ivf(O.VECTOR, O.L2_SQUARED, centers, new_off, new_rows, new_ids)
        for impl in (0, 1, 3, 4):
            pv.set_option("scan_impl", impl)
            a, b = fresh.search(queries, k=10, probes=5), piece.search(queries, k=10, probes=5)
            assert np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1]), impl
        wi, wd = oix.search_batch(queries, 5, 10, threads=8)
        assert np.allclose(b[1], wd, rtol=RTOL) and (b[0] == wi).mean() > 0.99
    finally:
        pv.set_option("scan_impl", int(os.environ.get("VB_TEST_SCAN_IMPL", "2")))
    with pytest.raises(pv.VecB200Error):
        pv._lib.check(pv.load().vb_ivf_load_list(piece.h, 0, None, None, 0))      # outside begin / end
