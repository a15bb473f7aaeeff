"""GPU re-rank of per-query candidate rows (vb_table_rerank[_dev]): the outer "ORDER BY v <op> q LIMIT k" over an index
scan's result, pgvector's quantize-then-rerank pattern.

- with the LDG scan, reranking every row in order is vb_exact_topk bit for bit (same per-row arithmetic, same selection);
- random candidate sets (absent entries, repeated rows, c past the 2048 of one selection) against the oracle's distances
  and a stable sort by (distance, candidate position);
- edge cases: ties in candidate order, NaN distances before padding, short and empty candidate sets, argument errors,
  out-of-range ids on the device path, torch results equal to the host results;
- the README's three flows end to end on the device (binary quantization, subvector, half precision)."""
import os

import numpy as np
import pytest

import oracle as O
from tests.test_gpu_distance import CASES, _random_rows

pytestmark = pytest.mark.gpu
RTOL = 1e-5


@pytest.fixture(scope="module")
def pv():
    import pgvector_b200 as pv
    pv.init(0)
    return pv


@pytest.fixture
def ldg(pv):
    """the rerank always runs the LDG scan kernel; vb_exact_topk does too with scan_impl 0"""
    pv.set_option("scan_impl", 0)
    yield pv
    pv.set_option("scan_impl", int(os.environ.get("VB_TEST_SCAN_IMPL", "2")))


WIDTHS = {O.VECTOR: (1, 17, 1536), O.HALFVEC: (1, 17, 1536, 4000), O.BIT: (1, 513, 1024, 64000)}
PAIRS = sorted({(e, m) for e, m, _ in CASES if m != O.SPHERICAL})
IDENTITY = [(e, m, d) for e, m in PAIRS for d in WIDTHS[e]]


@pytest.mark.parametrize("elem,metric,dim", IDENTITY)
def test_all_rows_in_order_is_the_exact_scan(ldg, elem, metric, dim):
    pv = ldg
    rng = np.random.default_rng(dim * 7 + metric * 3 + elem)
    n, nq = 600, 5
    rows = _random_rows(elem, n, dim, rng)
    queries = _random_rows(elem, nq, dim, rng)
    t = pv.Table(elem, dim).append(rows)
    cand = np.tile(np.arange(n, dtype=np.int64), (nq, 1))
    for k in (10, 300):
        wi, wd = t.exact_topk(metric, queries, k)
        gi, gd = t.rerank(metric, queries, cand, k)
        assert np.array_equal(gi, wi), k
        assert np.array_equal(gd.view(np.uint64), wd.view(np.uint64)), k


def reference(elem, metric, q, rows, cand, k, dim):
    """the outer sort on the host: oracle distances of the listed rows, stable by candidate position.  As in
    vb_exact_topk, VB_IP ranks by the negative inner product (largest first) and reports the inner product."""
    valid = cand[cand >= 0]
    if valid.size == 0:
        return np.full(k, -1, np.int64), np.full(k, np.inf)
    d = O.distance_batch(elem, metric, q, rows[valid], dim=dim)
    order = np.argsort(-d if metric == O.IP else d, kind="stable")[:k]
    ids = np.full(k, -1, np.int64)
    dist = np.full(k, np.inf)
    ids[:order.size] = valid[order]
    dist[:order.size] = d[order]
    return ids, dist


def tolerance(elem, metric, rows, q, ids, want):
    """2 x 1e-5 relative; for inner products relative to the magnitude of the summands (|a|.|q|: cancellation), for
    cosine absolute (its value is bounded by 2)"""
    if metric in (O.NEG_IP, O.IP):
        a32 = rows[ids].view(np.float16).astype(np.float32) if elem == O.HALFVEC else rows[ids]
        q32 = q.view(np.float16).astype(np.float32) if elem == O.HALFVEC else q
        return 2 * RTOL * np.maximum(np.abs(a32) @ np.abs(q32), 1e-30)
    if metric == O.COSINE:
        return np.full(len(ids), 2 * RTOL)
    return 2 * RTOL * np.abs(want)


def check_against_reference(elem, metric, rows, queries, cand, got_ids, got_dist, k, dim):
    for qi in range(queries.shape[0]):
        wi, wd = reference(elem, metric, queries[qi], rows, cand[qi], k, dim)
        real = wi >= 0
        assert np.array_equal(got_ids[qi] >= 0, real), qi
        if elem == O.BIT and metric == O.HAMMING:
            assert np.array_equal(got_ids[qi], wi), qi
            assert np.array_equal(got_dist[qi], wd), qi
            continue
        tol = tolerance(elem, metric, rows, queries[qi], wi[real], wd[real])
        assert np.all(np.abs(got_dist[qi][real] - wd[real]) <= tol), qi
        # ids may differ only where the oracle puts the two rows within tolerance of each other
        for j in np.nonzero(got_ids[qi] != wi)[0]:
            r = got_ids[qi][j]
            dj = O.distance_batch(elem, metric, queries[qi], rows[r:r + 1], dim=dim)[0]
            assert abs(dj - wd[j]) <= tol[j] + tolerance(elem, metric, rows, queries[qi], np.array([r]), np.array([dj]))[0], (qi, j)


def random_candidates(rng, nq, c, n):
    """row numbers with repeats and interleaved -1 (about a fifth of the entries)"""
    cand = rng.integers(0, n, size=(nq, c)).astype(np.int64)
    cand[rng.random((nq, c)) < 0.2] = -1
    return cand


@pytest.mark.parametrize("elem,metric,dim", [
    (O.VECTOR, O.L2, 128), (O.VECTOR, O.COSINE, 64), (O.VECTOR, O.IP, 1536), (O.VECTOR, O.L1, 20),
    (O.HALFVEC, O.NEG_IP, 96), (O.HALFVEC, O.L2_SQUARED, 768),
    (O.BIT, O.HAMMING, 1024), (O.BIT, O.JACCARD, 200),
])
@pytest.mark.parametrize("c,k", [(1, 10), (37, 10), (300, 10), (5000, 10), (5000, 2048)])
def test_random_candidate_sets_match_the_oracle(pv, elem, metric, dim, c, k):
    rng = np.random.default_rng(c * 13 + k + metric * 101 + dim)
    n, nq = 3000, 4
    rows = _random_rows(elem, n, dim, rng)
    queries = _random_rows(elem, nq, dim, rng)
    cand = random_candidates(rng, nq, c, n)
    t = pv.Table(elem, dim).append(rows)
    ids, dist = t.rerank(metric, queries, cand, k)
    check_against_reference(elem, metric, rows, queries, cand, ids, dist, k, dim)


def test_ties_come_back_in_candidate_order(pv):
    rows = np.ones((50, 4), np.float32)
    rows[10:20] = 3.0
    t = pv.Table(O.VECTOR, 4).append(rows)
    q = np.zeros((1, 4), np.float32)
    fwd = np.arange(50, dtype=np.int64)[None, :]
    rev = fwd[:, ::-1].copy()
    ids, _ = t.rerank(O.L2, q, fwd, 45)
    assert list(ids[0]) == [i for i in range(50) if not 10 <= i < 20] + list(range(10, 15))
    ids, _ = t.rerank(O.L2, q, rev, 45)
    assert list(ids[0]) == [i for i in range(49, -1, -1) if not 10 <= i < 20] + list(range(19, 14, -1))


def test_nan_distances_rank_last_but_before_padding(pv):
    rng = np.random.default_rng(3)
    rows = rng.standard_normal((20, 8)).astype(np.float32)
    rows[::4] = 0.0                                           # cosine against a zero row is NaN
    t = pv.Table(O.VECTOR, 8).append(rows)
    q = rng.standard_normal((1, 8)).astype(np.float32)
    cand = np.array([[0, -1, 1, 4, -1, 2, 8, 3, 12, 5, -1]], np.int64)
    ids, dist = t.rerank(O.COSINE, q, cand, 15)
    valid = cand[0][cand[0] >= 0]
    assert np.all(ids[0, :valid.size] >= 0) and np.all(ids[0, valid.size:] == -1)
    zero = [i for i in valid if i % 4 == 0]
    assert list(ids[0, valid.size - len(zero):valid.size]) == zero   # NaNs last, in candidate order
    assert np.all(np.isnan(dist[0, valid.size - len(zero):valid.size]))
    assert not np.isnan(dist[0, :valid.size - len(zero)]).any()


def test_short_and_empty_candidate_sets(pv):
    rng = np.random.default_rng(4)
    rows = rng.standard_normal((100, 16)).astype(np.float32)
    t = pv.Table(O.VECTOR, 16).append(rows)
    q = rng.standard_normal((3, 16)).astype(np.float32)
    cand = np.array([[5, 7, -1], [-1, -1, -1], [1, 2, 3]], np.int64)
    ids, dist = t.rerank(O.L2, q, cand, 5)
    assert sorted(ids[0, :2]) == [5, 7] and np.all(ids[0, 2:] == -1)
    assert np.all(ids[1] == -1)
    assert sorted(ids[2, :3]) == [1, 2, 3] and np.all(ids[2, 3:] == -1)
    ids, _ = t.rerank(O.L2, q, np.empty((3, 0), np.int64), 4)
    assert ids.shape == (3, 4) and np.all(ids == -1)


def test_argument_errors(pv):
    rows = np.random.default_rng(5).standard_normal((1000, 8)).astype(np.float32)
    t = pv.Table(O.VECTOR, 8).append(rows)
    q = np.zeros((2, 8), np.float32)
    cand = np.zeros((2, 4), np.int64)
    with pytest.raises(pv.VecB200Error) as e:
        t.rerank(O.L2, q, cand, 2049)
    assert e.value.code == -1 and "k must be in 1..2048" in str(e.value)
    bad = cand.copy()
    bad[1, 3] = 1000
    with pytest.raises(pv.VecB200Error) as e:
        t.rerank(O.L2, q, bad, 2)
    assert e.value.code == -1 and "candidate 3 of query 1 is 1000" in str(e.value)
    bad[1, 3] = -2
    with pytest.raises(pv.VecB200Error) as e:
        t.rerank(O.L2, q, bad, 2)
    assert "candidate 3 of query 1 is -2" in str(e.value)
    with pytest.raises(ValueError):
        t.rerank(O.L2, q, cand.astype(np.int32), 2)
    with pytest.raises(ValueError):
        t.rerank(O.L2, q, cand[:1], 2)


def test_device_path_equals_host_and_drops_out_of_range_ids(pv):
    import torch
    rng = np.random.default_rng(6)
    n, dim, nq, c, k = 2000, 96, 40, 150, 20
    rows = rng.standard_normal((n, dim)).astype(np.float32)
    queries = rng.standard_normal((nq, dim)).astype(np.float32)
    t = pv.Table(O.VECTOR, dim).append(rows)
    cand = random_candidates(rng, nq, c, n)
    for metric in (O.L2, O.IP, O.COSINE):
        hi, hd = t.rerank(metric, queries, cand, k)
        di, dd = t.rerank(metric, torch.from_numpy(queries).cuda(), torch.from_numpy(cand).cuda(), k)
        assert np.array_equal(di.cpu().numpy(), hi)
        assert np.array_equal(dd.cpu().numpy(), hd.astype(np.float32))
    # ids outside [0, n) are absent on the device path
    wild = cand.copy()
    wild[:, ::7] = n + 5
    wild[:, 3::11] = -9
    wild[0, 0] = 1 << 40
    tame = np.where((wild >= 0) & (wild < n), wild, -1)
    hi, hd = t.rerank(O.L2, queries, tame, k)
    di, dd = t.rerank(O.L2, torch.from_numpy(queries).cuda(), torch.from_numpy(wild).cuda(), k)
    assert np.array_equal(di.cpu().numpy(), hi)
    assert np.array_equal(dd.cpu().numpy(), hd.astype(np.float32))


# ----------------------------------------------------------------------------- the README's flows


def low_dim_rows(n, nq, dim, seed):
    """rows of low intrinsic dimension (as in the benchmarks): a graph index on them has a meaningful recall"""
    rng = np.random.default_rng(seed)
    frame = np.linalg.qr(rng.standard_normal((dim, 8)))[0].astype(np.float32)
    x = rng.standard_normal((n, 8)).astype(np.float32) @ frame.T + 0.05 * rng.standard_normal((n, dim)).astype(np.float32)
    q = rng.standard_normal((nq, 8)).astype(np.float32) @ frame.T + 0.05 * rng.standard_normal((nq, dim)).astype(np.float32)
    return x.astype(np.float32), q.astype(np.float32)


def expand_duplicates(ids, dup_of):
    """an element's heap tids include the rows folded into it: list them too, -1 padded to a rectangle"""
    members = {}
    for r in np.nonzero(dup_of >= 0)[0]:
        members.setdefault(int(dup_of[r]), []).append(int(r))
    lists = [[r for e in row if e >= 0 for r in [int(e)] + members.get(int(e), [])] for row in ids]
    out = np.full((len(lists), max(1, max(len(x) for x in lists))), -1, np.int64)
    for i, x in enumerate(lists):
        out[i, :len(x)] = x
    return out


def check_flow(pv, rows, queries, index_ids, cand, metric, k):
    """rerank against the oracle, and recall against the full-precision truth: reranked = candidate-set recall (the k
    nearest rows the candidates hold are found exactly) >= the index's own recall"""
    dim = rows.shape[1]
    t = pv.Table(O.VECTOR, dim).append(rows)
    ids, dist = t.rerank(metric, queries, cand, k)
    check_against_reference(O.VECTOR, metric, rows, queries, cand, ids, dist, k, dim)
    truth, tdist = t.exact_topk(metric, queries, k + 1)
    hits_rr = hits_cand = hits_ix = used = 0
    for qi in range(queries.shape[0]):
        if abs(tdist[qi, k] - tdist[qi, k - 1]) <= RTOL * max(abs(tdist[qi, k]), 1e-30):
            continue   # a near-tie at the k-th place: which of the two is "truth" is arbitrary
        tr = set(truth[qi, :k].tolist())
        hits_rr += len(tr & set(ids[qi].tolist()))
        hits_cand += len(tr & set(cand[qi].tolist()))
        hits_ix += len(tr & set(index_ids[qi, :k].tolist()))
        used += 1
    assert used >= queries.shape[0] // 2
    assert hits_rr == hits_cand
    assert hits_rr >= hits_ix


def test_binary_quantize_flow(ldg):
    pv = ldg
    rows, queries = low_dim_rows(5000, 40, 64, seed=11)
    bits = pv.binary_quantize(rows)
    ix = pv.HnswIndex("bit_hamming_ops", 64, m=16).build(bits, ef_construction=64, seed=3)
    ef, k = 40, 10
    eids, _, _ = ix.search(pv.binary_quantize(queries), k=ef, ef_search=ef)
    cand = expand_duplicates(eids, ix.export()["dup_of"])
    check_flow(pv, rows, queries, eids, cand, O.COSINE, k)


def test_subvector_flow(ldg):
    pv = ldg
    rows, queries = low_dim_rows(5000, 40, 64, seed=12)
    sub, qsub = O.l2_normalize(O.VECTOR, rows[:, :16].copy()), O.l2_normalize(O.VECTOR, queries[:, :16].copy())
    ix = pv.HnswIndex("vector_cosine_ops", 16, m=16).build(sub, ef_construction=64, seed=3)
    ef, k = 40, 10
    eids, _, _ = ix.search(qsub, k=ef, ef_search=ef)
    cand = expand_duplicates(eids, ix.export()["dup_of"])
    check_flow(pv, rows, queries, eids, cand, O.COSINE, k)


def test_half_precision_flow(ldg):
    pv = ldg
    rows, queries = low_dim_rows(5000, 40, 64, seed=13)
    ix = pv.HnswIndex("halfvec_l2_ops", 64, m=16).build(pv.vector_to_halfvec(rows), ef_construction=64, seed=3)
    ef, k = 40, 10
    eids, _, _ = ix.search(pv.vector_to_halfvec(queries), k=ef, ef_search=ef)
    cand = expand_duplicates(eids, ix.export()["dup_of"])
    check_flow(pv, rows, queries, eids, cand, O.L2, k)
