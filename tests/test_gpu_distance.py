"""GPU parity (through the C ABI): batched distance operators and exact top-k vs the oracle
and vs the reference's known-answer outputs."""
import math

import numpy as np
import pytest

import oracle as O
from tests.util import f32_to_half_bits, load_golden, mixture, parse_vector

pytestmark = pytest.mark.gpu

ELEM = {"vector": O.VECTOR, "halfvec": O.HALFVEC, "bit": O.BIT}
METRIC = {"l2_distance": O.L2, "inner_product": O.IP, "negative_inner_product": O.NEG_IP,
          "cosine_distance": O.COSINE, "l1_distance": O.L1, "hamming_distance": O.HAMMING,
          "jaccard_distance": O.JACCARD}
KAT = [c for c in load_golden("distance_kat.json")["cases"] if c["fn"] in METRIC]

RTOL = 1e-5   # north_star: L2/IP/cosine distances within 1e-5 relative


@pytest.fixture(scope="module")
def pv():
    import os
    import pgvector_b200 as pv
    pv.init(0)
    # VB_TEST_SCAN_IMPL=1 re-runs the suite on the bulk-copy (TMA) scan kernel
    pv.set_option("scan_impl", int(os.environ.get("VB_TEST_SCAN_IMPL", "2")))
    return pv


@pytest.mark.parametrize("case", KAT, ids=[c["source"].split("/")[-1] for c in KAT])
def test_known_answers_on_gpu(pv, case):
    """the reference's regression outputs (test/expected/*.out) reproduced by the CUDA path"""
    elem = ELEM[case["type"]]
    (a, da), (b, db) = [parse_vector(x, elem) for x in case["args"]]
    if case["error"]:
        with pytest.raises(ValueError) as e:
            pv.distance_batch(elem, METRIC[case["fn"]], a, b.reshape(1, -1), dim=db, q_dim=da)
        assert str(e.value) == case["error"]
        return
    got = pv.distance_batch(elem, METRIC[case["fn"]], a, b.reshape(1, -1), dim=da)[0]
    want = float(case["expected"].replace("Infinity", "inf")) if case["expected"] != "NaN" else math.nan
    if math.isnan(want):
        assert math.isnan(got)
    else:
        assert got == want, (case, got)


def _random_rows(elem, n, dim, rng):
    if elem == O.BIT:
        nb = (dim + 7) // 8
        r = rng.integers(0, 256, size=(n, nb), dtype=np.uint8)
        if dim % 8:
            r[:, -1] &= (0xFF << (8 - dim % 8)) & 0xFF
        return r
    x = rng.standard_normal((n, dim)).astype(np.float32)
    return f32_to_half_bits(x) if elem == O.HALFVEC else x


CASES = [(O.VECTOR, m, d) for m in (O.L2_SQUARED, O.L2, O.NEG_IP, O.IP, O.COSINE, O.L1, O.SPHERICAL)
         for d in (1, 3, 4, 17, 128, 1000, 1536, 2000)]
CASES += [(O.HALFVEC, m, d) for m in (O.L2_SQUARED, O.L2, O.NEG_IP, O.COSINE, O.L1) for d in (1, 3, 8, 9, 100, 768, 4000)]
CASES += [(O.BIT, m, d) for m in (O.HAMMING, O.JACCARD) for d in (1, 3, 8, 52, 64, 65, 513, 1024, 4099, 64000)]


@pytest.mark.parametrize("elem,metric,dim", CASES)
def test_distance_batch_matches_oracle(pv, elem, metric, dim):
    rng = np.random.default_rng(dim * 31 + metric)
    n = 777
    rows = _random_rows(elem, n, dim, rng)
    q = _random_rows(elem, 1, dim, rng)[0]
    if metric == O.SPHERICAL:   # expects unit vectors
        rows = O.l2_normalize(elem, rows)
        q = O.l2_normalize(elem, q)
    got = pv.distance_batch(elem, metric, q, rows, dim=dim)
    want = O.distance_batch(elem, metric, q, rows, dim=dim)
    if elem == O.BIT:
        assert np.array_equal(got, want)           # bit-exact Hamming / Jaccard
        return
    truth = np.array([O.distance(elem, metric, rows[i], q, f64=True) for i in range(n)])
    if metric in (O.NEG_IP, O.IP, O.COSINE, O.SPHERICAL):
        # cancellation: tolerance relative to the magnitude of the summands (|a|.|b|)
        a32 = rows.view(np.float16).astype(np.float32) if elem == O.HALFVEC else rows
        q32 = q.view(np.float16).astype(np.float32) if elem == O.HALFVEC else q
        scale = np.abs(a32) @ np.abs(q32)
        if metric in (O.COSINE, O.SPHERICAL):
            scale = np.ones(n)
        assert np.all(np.abs(got - truth) <= RTOL * np.maximum(scale, 1e-30) + 1e-6 * (metric == O.SPHERICAL))
        assert np.all(np.abs(want - truth) <= RTOL * np.maximum(scale, 1e-30) + 1e-6 * (metric == O.SPHERICAL))
    else:
        assert np.all(np.abs(got - truth) <= RTOL * np.abs(truth))
        assert np.all(np.abs(want - truth) <= RTOL * np.abs(truth))


def test_null_query_is_zero_distance(pv):
    rows = np.ones((5, 4), np.float32)
    assert np.array_equal(pv.distance_batch(O.VECTOR, O.L2, None, rows), np.zeros(5))


def _check_topk(elem, metric, rows, queries, got_ids, got_dist, k, dim=None):
    """ids equal the oracle's except where fp32 summation order can flip near-ties; distances within RTOL"""
    bad = 0
    for qi in range(queries.shape[0]):
        wi, wd = O.exact_topk(elem, metric, queries[qi], rows, k, dim=dim)
        scale = np.maximum(np.abs(wd), 1e-30)
        if elem == O.BIT:
            assert np.array_equal(got_dist[qi], wd), qi
            assert np.array_equal(got_ids[qi], wi), qi
            continue
        assert np.all(np.abs(got_dist[qi] - wd) <= 2 * RTOL * np.maximum(scale, np.abs(wd).max() * 1e-2)), qi
        if not np.array_equal(got_ids[qi], wi):
            # allowed only if the differing ids are within tolerance of each other in the oracle
            d_all = O.distance_batch(elem, metric, queries[qi], rows, dim=dim)
            for j in range(k):
                if got_ids[qi][j] != wi[j]:
                    assert abs(d_all[got_ids[qi][j]] - wd[j]) <= 2 * RTOL * max(abs(wd[j]), np.abs(wd).max() * 1e-2), (qi, j)
            bad += 1
    return bad


def test_config_a_exact_l2_10k_by_128(pv):
    """BASELINE config A: exact L2 <-> scan of 10k x 128 fp32, k = 10, 1000 queries"""
    rng = np.random.default_rng(1)
    rows = rng.standard_normal((10000, 128)).astype(np.float32)
    queries = np.random.default_rng(2).standard_normal((1000, 128)).astype(np.float32)
    t = pv.Table(O.VECTOR, 128).append(rows)
    ids, dist = t.exact_topk(O.L2, queries, 10)
    flips = _check_topk(O.VECTOR, O.L2, rows, queries[:200], ids, dist, 10)
    assert flips <= 2
    # sortedness + membership properties on the full batch
    assert np.all(np.diff(dist, axis=1) >= 0)
    assert ids.min() >= 0 and ids.max() < 10000


@pytest.mark.parametrize("elem,metric,dim,n,k", [
    (O.VECTOR, O.NEG_IP, 33, 5000, 7),
    (O.VECTOR, O.COSINE, 64, 3000, 10),
    (O.VECTOR, O.L1, 20, 3000, 5),
    (O.HALFVEC, O.L2, 96, 4000, 10),
    (O.HALFVEC, O.NEG_IP, 768, 2000, 10),
    (O.BIT, O.HAMMING, 52, 6000, 20),
    (O.BIT, O.HAMMING, 1024, 3000, 10),
    (O.VECTOR, O.L2_SQUARED, 16, 9000, 3000),    # k > 2048: segmented sort path
    (O.VECTOR, O.L2, 8, 100, 200),               # k > n: -1 padding
])
def test_exact_topk_matches_oracle(pv, elem, metric, dim, n, k):
    rng = np.random.default_rng(n + k)
    rows = _random_rows(elem, n, dim, rng)
    queries = _random_rows(elem, 6, dim, rng)
    t = pv.Table(elem, dim).append(rows)
    ids, dist = t.exact_topk(metric, queries, k)
    kk = min(k, n)
    _check_topk(elem, metric, rows, queries, ids[:, :kk], dist[:, :kk], kk, dim=dim)
    if k > n:
        assert np.all(ids[:, n:] == -1)


def test_exact_topk_ties_smaller_row_first(pv):
    rows = np.zeros((300, 4), np.float32)
    rows[::3] = 1.0
    t = pv.Table(O.VECTOR, 4).append(rows)
    ids, dist = t.exact_topk(O.L2, np.zeros((1, 4), np.float32), 250)
    zero = [i for i in range(300) if i % 3]
    assert list(ids[0][:200]) == zero
    assert list(ids[0][200:]) == list(range(0, 150, 3))


def test_table_append_is_incremental(pv):
    rng = np.random.default_rng(5)
    rows = rng.standard_normal((1000, 10)).astype(np.float32)
    t = pv.Table(O.VECTOR, 10)
    for lo in range(0, 1000, 137):
        t.append(rows[lo:lo + 137])
    assert len(t) == 1000
    q = rng.standard_normal((3, 10)).astype(np.float32)
    ids, dist = t.exact_topk(O.L2, q, 5)
    _check_topk(O.VECTOR, O.L2, rows, q, ids, dist, 5)
