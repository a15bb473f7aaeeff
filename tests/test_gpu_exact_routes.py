"""The exact top-k (Table.exact_topk) at the edges of its route choices, against a restatement and the oracle.

exact_topk_impl (vb_ivf.cu) cuts the queries into sub-batches of bq = 2^30 / (4 n), so the fp32 distance matrix of one
sub-batch stays under 1 GiB, and computes the distances of each sub-batch in one of three ways:
  tiled      m >= 64 queries, 128 <= n <= 65535 * 128 rows, vector or bit rows, an L2 / inner product / Hamming key and
             scan_impl != 0: assign_exact_kernel in matrix mode (vb_kmeans.cu), 128 x 128 tiles in K steps of 16 words;
  bulk copy  the streamed scan with TMA row stages (vb_scan_bulk.cu) for rows of >= 512 B whose query image is <= 64 KiB
             and for which two stages fit; at scan_impl 1 whenever it can, at scan_impl 2 for tables over 50 MiB;
  LDG        the streamed scan of vb_scan.cu otherwise: LPR lanes per row (32 / 16 / 8 / 4 / 2 / 1 from V, the 16-byte
             words of a row), in chunks of 32 .. 4096 rows.
One CTA per query then radix-selects and bitonic-sorts the k <= 2048 smallest (key, row) pairs; k > 2048 sorts every row
with CUB.  distance_batch, the filtered scan and the re-rank share the per-row arithmetic (the f64-output and the gather
instantiations of the scan).  No counter tells the three distance routes apart, so the file restates the choice on the host
and checks that every case sits where its name says; launch counts show the sub-batches and the selection path.

Rows and queries are multiples of 1/16 in [-2, 2] ([-1/2, 1/2] past 4000 dimensions): every product, square and partial
sum of a distance is an exact fp32 value (below 2^24 steps of 1/256), exact in half precision too, so every route and
every summation order gives the same key.  `reference` restates the selection in float64 numpy, which is exact on these
rows and is itself checked against the oracle's exact_topk and distance_batch.  Ids and distances are compared for
equality, query by query: that pins the tie rule (the smaller row first) and the -1 padding.  Cosine is not exact on grid
rows and is held to the fp32 intervals of test_gpu_hostile_values.
"""
import os

import numpy as np
import pytest

import oracle as O
from tests.test_gpu_hostile_values import _table_laws, check_topk, exact_query, intervals, same_as_returned

gpu = pytest.mark.gpu
DEFAULT_SCAN_IMPL = int(os.environ.get("VB_TEST_SCAN_IMPL", "2"))
ELEMS = {"vector": O.VECTOR, "halfvec": O.HALFVEC, "bit": O.BIT}

# ------------------------------------------------------------------------------ the route choices, restated on the host
# (vb_ivf.cu exact_topk_impl, vb_kmeans.cu launch_distance_matrix, vb_scan.cu launch_scan_t / scan_rows_per_chunk /
# use_bulk_scan, vb_scan_bulk.cu bulk_shape, vb_common.cuh require_scannable_rows)

TILE, K_STEP, MATRIX_MAX_N = 128, 16, 65535 * 128
SCRATCH_BYTES, L2_BYTES = 1 << 30, 50 << 20
SMEM_MAX = 227 * 1024
KEY = {O.L2: O.L2_SQUARED, O.IP: O.NEG_IP}
TILED_KEYS = (O.L2_SQUARED, O.NEG_IP, O.HAMMING)


def raw_bytes(elem, dim):
    return 4 * dim if elem == O.VECTOR else 2 * dim if elem == O.HALFVEC else (dim + 7) // 8


def stride(elem, dim):
    return (raw_bytes(elem, dim) + 15) & ~15


def qimage(elem, dim):
    """bytes of one query's image (halfvec widened to fp32)"""
    return 2 * stride(elem, dim) if elem == O.HALFVEC else stride(elem, dim)


def words(elem, dim):
    """V: 16-byte words of a row"""
    return stride(elem, dim) // 16


def sub_batches(nq, n):
    bq = max(1, min(nq, SCRATCH_BYTES // (4 * max(n, 1))))
    return [min(bq, nq - q0) for q0 in range(0, nq, bq)]


def tiled(elem, metric, m, n, impl):
    return m >= 64 and TILE <= n <= MATRIX_MAX_N and elem != O.HALFVEC and impl != 0 and KEY.get(metric, metric) in TILED_KEYS


def lpr(V):
    return next((l for l in (32, 16, 8, 4, 2) if V >= l), 1)


def rows_per_step(V):
    """G * RPI: rows one CTA of the LDG scan walks per step"""
    return (128 // lpr(V)) * (4 if lpr(V) >= 8 else 8)


def bulk_stages(elem, dim):
    s = stride(elem, dim)
    rpw = max(1, min(48 * 1024 // (8 * s), 8))
    stage_bytes = (8 * rpw * s + 127) & ~127
    fixed = ((qimage(elem, dim) + 127) & ~127) + 2 * 4 * 8 + 256
    return max(0, min((220 * 1024 - fixed) // stage_bytes, 4))


def bulk_supported(elem, dim):
    return stride(elem, dim) >= 512 and qimage(elem, dim) <= 64 * 1024 and bulk_stages(elem, dim) >= 2


def route(elem, metric, m, n, impl, dim):
    if tiled(elem, metric, m, n, impl):
        return "tiled"
    if impl != 0 and bulk_supported(elem, dim) and (impl == 1 or n * stride(elem, dim) > L2_BYTES):
        return "bulk"
    return "ldg"


def chunk_rows(elem, dim):
    return min(max((128 * 1024 // stride(elem, dim)) // 32 * 32, 32), 4096)


def launches(elem, dim, nq, n, k):
    """per sub-batch: the query repack (halfvec, or rows not a multiple of 16 bytes), the distances, the segments, the
    selection (four launches for the sorted path: keys, two CUB passes, emit) and the finish"""
    repack = elem == O.HALFVEC or raw_bytes(elem, dim) != stride(elem, dim)
    return (int(repack) + 4 + (3 if k > 2048 else 0)) * len(sub_batches(nq, n))


# ------------------------------------------------------------------------------------------------------------ the cases

LPR_WIDTHS = ([("vector", d) for d in (4, 5, 12, 13, 28, 29, 60, 61, 124, 125)]
              + [("halfvec", d) for d in (8, 9, 24, 25, 56, 57, 120, 121, 248, 249)]
              + [("bit", d) for d in (128, 129, 384, 385, 896, 897, 1920, 1921, 3968, 3969)])
WIDE = [("vector", 2000), ("halfvec", 4000), ("vector", 16000), ("halfvec", 16000), ("bit", 64000)]
WIDTHS = LPR_WIDTHS + WIDE
K_STEP_WIDTHS = [("vector", 16), ("vector", 17), ("vector", 32), ("vector", 33), ("bit", 512), ("bit", 513),
                 ("vector", 2000), ("vector", 16000), ("bit", 64000)]
N_SIZES = [127, 128, 129, 255, 256, 257]
NQ_SIZES = [63, 64, 65, 127, 128, 129, 1000]
K_STEPS = [1, 2, 3, 255, 256, 257, 1024, 1025, 2047, 2048, 2049]
MILLION, FOUR_MILLION = 1 << 20, 4 * 1024 * 1024
# the widest rows whose query image fits the scan's shared memory
IMAGE_LIMIT = {O.VECTOR: 58112, O.HALFVEC: 58112, O.BIT: 1859584}


def test_route_model_puts_every_case_where_its_name_says():
    for kind, e in ELEMS.items():
        dims = [d for k, d in LPR_WIDTHS if k == kind]
        assert [words(e, d) for d in dims] == [1, 2, 3, 4, 7, 8, 15, 16, 31, 32], kind
        for lo, hi in zip(dims[::2], dims[1::2]):     # each pair straddles one lanes-per-row split
            assert lpr(words(e, lo)) < lpr(words(e, hi)) == words(e, hi), (kind, lo, hi)
        # 31 -> 32 words is also the bulk-copy stride threshold
        assert not bulk_supported(e, dims[-2]) and bulk_supported(e, dims[-1]), kind
    # the matrix kernel's K step of 16 four-byte words: a whole number of steps, or a partial last one
    for kind, d in K_STEP_WIDTHS:
        partial = (stride(ELEMS[kind], d) // 4) % K_STEP != 0
        assert partial == (d in (17, 33, 513)), (kind, d)
    for kind, d in (("vector", 2000), ("halfvec", 4000), ("bit", 64000)):
        assert bulk_supported(ELEMS[kind], d), (kind, d)
    for kind in ("vector", "halfvec"):        # an image over 48 KiB, and fewer than two bulk stages
        assert qimage(ELEMS[kind], 16000) > 48 * 1024 and bulk_stages(ELEMS[kind], 16000) < 2
        assert not bulk_supported(ELEMS[kind], 16000)
    # the tiled route: m >= 64, n >= 128, vector / bit, L2 / inner product / Hamming keys, scan_impl != 0
    for n in N_SIZES:
        for nq in NQ_SIZES:
            for metric in (O.L2, O.L2_SQUARED, O.IP, O.NEG_IP):
                assert tiled(O.VECTOR, metric, nq, n, 1) == (nq >= 64 and n >= 128)
                assert not tiled(O.VECTOR, metric, nq, n, 0)
            assert tiled(O.BIT, O.HAMMING, nq, n, 2) == (nq >= 64 and n >= 128)
            for e, metric in ((O.VECTOR, O.COSINE), (O.VECTOR, O.L1), (O.BIT, O.JACCARD), (O.HALFVEC, O.L2_SQUARED)):
                assert not tiled(e, metric, nq, n, 2)
    # 50 MiB of vector(128) rows at scan_impl 2: LDG at 102400 rows, bulk copy one row later (streamed: nq < 64)
    assert 102400 * stride(O.VECTOR, 128) == L2_BYTES
    assert route(O.VECTOR, O.L2_SQUARED, 8, 102400, 2, 128) == "ldg"
    assert route(O.VECTOR, O.L2_SQUARED, 8, 102401, 2, 128) == "bulk"
    # sub-batches: 2^20 rows take 256 queries at a time; 4 Mi rows 64, one row more 63 (never tiled)
    assert sub_batches(576, MILLION) == [256, 256, 64] and sub_batches(575, MILLION) == [256, 256, 63]
    assert [tiled(O.VECTOR, O.L2_SQUARED, m, MILLION, 2) for m in sub_batches(575, MILLION)] == [True, True, False]
    assert sub_batches(64, FOUR_MILLION) == [64] and sub_batches(64, FOUR_MILLION + 1) == [63, 1]
    assert tiled(O.VECTOR, O.L2_SQUARED, 64, FOUR_MILLION, 2)
    assert launches(O.VECTOR, 4, 576, MILLION, 10) == 12 and launches(O.VECTOR, 4, 575, MILLION, 2049) == 21
    # chunk rows at the clamps
    assert chunk_rows(O.VECTOR, 4) == 4096 and chunk_rows(O.BIT, 64000) == 32 and chunk_rows(O.VECTOR, 125) == 256
    # the query image limit of the scan
    for e, d in IMAGE_LIMIT.items():
        assert qimage(e, d) == SMEM_MAX and qimage(e, d + 1) > SMEM_MAX


# ---------------------------------------------------------------------------------------------- data and restatement

def grid(elem, n, dim, seed):
    """n rows of multiples of 1/16 in [-2, 2] ([-1/2, 1/2] past 4000 dimensions), in the payload layout (bit: random
    bits, the padding bits of the last byte zero)"""
    rng = np.random.default_rng(seed)
    if elem == O.BIT:
        bits = rng.integers(0, 2, (n, dim), dtype=np.uint8)
        return np.packbits(bits, axis=1)
    r = 32 if dim <= 4000 else 8
    x = rng.integers(-r, r + 1, (n, dim)).astype(np.float32) / 16
    return x.astype(np.float16).view(np.uint16) if elem == O.HALFVEC else x


def values(elem, a):
    return (a.view(np.float16) if elem == O.HALFVEC else a).astype(np.float64)


def keys(elem, metric, Q, X, dim):
    """[nq, n] float64 keys the kernels rank by, exact on grid rows: the L2 square, the negative inner product, L1,
    Hamming; Jaccard as the float32 the scan stores"""
    metric = KEY.get(metric, metric)
    if elem == O.BIT:
        a = np.bitwise_count(X).sum(axis=1, dtype=np.int64)
        out = np.empty((len(Q), len(X)))
        for j, q in enumerate(Q):
            both = np.bitwise_count(X & q).sum(axis=1, dtype=np.int64)
            if metric == O.HAMMING:
                out[j] = a + int(np.bitwise_count(q).sum()) - 2 * both
            else:
                with np.errstate(invalid="ignore", divide="ignore"):
                    jac = np.where(both == 0, 1.0, 1.0 - both / (a + int(np.bitwise_count(q).sum()) - both))
                out[j] = jac.astype(np.float32)
        return out
    x, q = values(elem, X), values(elem, Q)
    if metric == O.L1:
        return np.stack([np.abs(x - v).sum(axis=1) for v in q])
    ip = q @ x.T
    if metric == O.NEG_IP:
        return -ip
    return (x * x).sum(axis=1)[None, :] + (q * q).sum(axis=1)[:, None] - 2 * ip


def select(kv, k):
    """the k smallest (key, row) pairs of every row of kv: (rows -1 padded, keys +inf padded)"""
    nq, n = kv.shape
    m = min(k, n)
    ids = np.full((nq, k), -1, np.int64)
    out = np.full((nq, k), np.inf)
    for j in range(nq):
        key = kv[j]
        if m == n:
            order = np.argsort(key, kind="stable")
        else:
            t = np.partition(key, m - 1)[m - 1]
            below = np.flatnonzero(key < t)
            order = np.concatenate([below[np.argsort(key[below], kind="stable")], np.flatnonzero(key == t)[: m - len(below)]])
        ids[j, :m] = order
        out[j, :m] = key[order]
    return ids, out


def finish(metric, kv):
    """the operator's float8 from the key (finish_value): the padding key +inf goes through it as well"""
    if metric == O.L2:
        return np.sqrt(kv)
    if metric == O.IP:
        return -kv
    return kv


def reference(metric, kv, k):
    ids, key = select(kv, k)
    return ids, finish(metric, key)


def assert_same(ids, dist, wi, wd, what):
    bad = np.flatnonzero(~(np.all(ids == wi, axis=1) & np.all(dist == wd, axis=1)))
    assert len(bad) == 0, f"{what}: {len(bad)} of {len(ids)} queries differ, first {bad[:8].tolist()}: " \
                          f"{ids[bad[0]][:8].tolist()} {dist[bad[0]][:8].tolist()} want {wi[bad[0]][:8].tolist()} {wd[bad[0]][:8].tolist()}"


ORACLE_RANKED = (O.L2, O.L2_SQUARED, O.NEG_IP, O.L1, O.HAMMING)   # the oracle ranks IP and Jaccard otherwise


def assert_oracle_agrees(elem, metric, Q, X, dim, k, wi, wd, queries):
    """the restatement is the oracle's exact_topk on these queries"""
    if metric not in ORACLE_RANKED:
        return
    for j in queries:
        oi, od = O.exact_topk(elem, metric, Q[j], X, k, dim=dim)
        assert np.array_equal(oi, wi[j]) and np.array_equal(od, wd[j]), (elem, metric, dim, k, j)


@pytest.fixture(scope="module")
def pv():
    import pgvector_b200 as pv
    pv.init(0)
    yield pv
    pv.set_option("scan_impl", DEFAULT_SCAN_IMPL)


class scan_impl:
    def __init__(self, pv, impl):
        self.pv, self.impl = pv, impl

    def __enter__(self):
        self.pv.set_option("scan_impl", self.impl)

    def __exit__(self, *exc):
        self.pv.set_option("scan_impl", DEFAULT_SCAN_IMPL)


def run(pv, t, metric, Q, k, impl):
    """exact_topk under scan_impl `impl`: (ids, dist, launches)"""
    with scan_impl(pv, impl):
        before = pv.launch_count()
        ids, dist = t.exact_topk(metric, Q, k)
        return ids, dist, pv.launch_count() - before


def check_run(pv, t, elem, dim, metric, Q, kv, k, impl, what):
    ids, dist, used = run(pv, t, metric, Q, k, impl)
    n = kv.shape[1]
    assert used == launches(elem, dim, len(Q), n, k), (what, used)
    wi, wd = reference(metric, kv, k)
    assert_same(ids, dist, wi, wd, f"{what} {route(elem, metric, len(Q), n, impl, dim)} k={k}")
    return wi, wd


# ------------------------------------------------------------------------------------------- tiled against streamed

@gpu
@pytest.mark.parametrize("impl", [0, 1, 2])
@pytest.mark.parametrize("n", N_SIZES)
def test_tiled_and_streamed_batches_equal_the_restatement(pv, n, impl):
    """batches of 63 .. 1000 queries over 127 .. 257 rows: the tiled route from 64 queries and 128 rows at scan_impl
    1 and 2 (vector L2, L2 square, inner product, negative inner product; bit Hamming), the streamed scan below that,
    at scan_impl 0 and for the metrics and types that never tile (L1, Jaccard, halfvec, cosine).  Partial query and
    row tiles, and a partial last K step (vector(33): 36 words; bit(513): 20 words)."""
    cases = (("vector", 33, [O.L2, O.L2_SQUARED, O.IP, O.NEG_IP, O.L1]), ("bit", 513, [O.HAMMING, O.JACCARD]),
             ("halfvec", 33, [O.L2_SQUARED, O.NEG_IP, O.L1]))
    for kind, dim, metrics in cases:
        e = ELEMS[kind]
        X, Q = grid(e, n, dim, seed=n), grid(e, max(NQ_SIZES), dim, seed=n + 7)
        t = pv.Table(e, dim).append(X)
        for metric in metrics:
            kv = keys(e, metric, Q, X, dim)
            for nq in NQ_SIZES:
                for k in (10, n + 1):
                    wi, wd = check_run(pv, t, e, dim, metric, Q[:nq], kv[:nq], k, impl, f"{kind}({dim}) n={n} nq={nq} m={metric}")
            assert_oracle_agrees(e, metric, Q, X, dim, n + 1, wi, wd, (0, 999))
        if e != O.BIT:        # cosine: inside the fp32 intervals, in an order they allow
            xf, qf = values(e, X).astype(np.float32), values(e, Q).astype(np.float32)
            bounds = {}
            for nq in NQ_SIZES:
                ids, dist, _ = run(pv, t, O.COSINE, Q[:nq], 10, impl)
                for j in [j for j in range(nq) if j < 129 or j % 50 == 0]:
                    if j not in bounds:
                        bounds[j] = intervals(O.COSINE, xf, qf[j])
                    check_topk(ids[j], dist[j], *bounds[j], 10, f32=True)
        t.free()


@gpu
def test_config_a_shape_is_exact_for_every_query(pv):
    """bench.py config A: 10 000 vector(128) rows, 1000 queries, k = 10, L2 -- one tiled sub-batch, every query equal"""
    e, dim, n, nq, k = O.VECTOR, 128, 10000, 1000, 10
    X, Q = grid(e, n, dim, seed=10), grid(e, nq, dim, seed=11)
    assert route(e, O.L2, nq, n, DEFAULT_SCAN_IMPL, dim) == ("ldg" if DEFAULT_SCAN_IMPL == 0 else "tiled")
    t = pv.Table(e, dim).append(X)
    wi, wd = check_run(pv, t, e, dim, O.L2, Q, keys(e, O.L2, Q, X, dim), k, DEFAULT_SCAN_IMPL, "config A")
    assert_oracle_agrees(e, O.L2, Q, X, dim, k, wi, wd, (0, 500, 999))
    t.free()


@gpu
@pytest.mark.parametrize("kind,dim", K_STEP_WIDTHS)
def test_tiled_route_at_every_k_step_and_the_widest_rows(pv, kind, dim):
    """129 queries over 257 rows (a partial query tile and a partial row tile) at whole and partial K steps and on the
    widest rows, tiled (scan_impl 2) and streamed (scan_impl 0)"""
    e = ELEMS[kind]
    n, nq = 257, 129
    X, Q = grid(e, n, dim, seed=dim), grid(e, nq, dim, seed=dim + 1)
    t = pv.Table(e, dim).append(X)
    for metric in ((O.HAMMING,) if e == O.BIT else (O.L2_SQUARED, O.NEG_IP)):
        kv = keys(e, metric, Q, X, dim)
        for impl in (2, 0):
            assert route(e, metric, nq, n, impl, dim) == ("tiled" if impl else "ldg")
            for k in (10, n + 1):
                wi, wd = check_run(pv, t, e, dim, metric, Q, kv, k, impl, f"{kind}({dim}) m={metric} impl={impl}")
        assert_oracle_agrees(e, metric, Q, X, dim, n + 1, wi, wd, (0, 128))
    t.free()


@gpu
def test_hostile_laws_through_the_tiled_route(pv):
    """the hostile laws (NaN, infinite and overflowing distances, common offsets, ties) at 64 queries: tiled at
    scan_impl 2, streamed at 0; inside the fp32 intervals, and the oracle's bit for bit where the result is exact"""
    dim, n, nq = 128, 1000, 64
    for name, (x, q) in _table_laws(O.VECTOR, dim, n, nq).items():
        t = pv.Table(O.VECTOR, dim).append(x)
        for metric in (O.L2, O.NEG_IP):
            bounds = [intervals(metric, x, q[j]) for j in range(nq)]
            for impl in (2, 0):
                assert route(O.VECTOR, metric, nq, n, impl, dim) == ("tiled" if impl else "ldg")
                for k in (10, n + 5):
                    ids, dist, _ = run(pv, t, metric, q, k, impl)
                    for j in range(nq):
                        lo, hi = bounds[j]
                        check_topk(ids[j], dist[j], lo, hi, k)
                        if exact_query(lo, hi, np.arange(n)):
                            wi, wd = O.exact_topk(O.VECTOR, metric, q[j], x, k)
                            assert np.array_equal(ids[j], wi) and same_as_returned(metric, dist[j], wd), (name, metric, impl, k, j)
        t.free()


# ------------------------------------------------------------------------------------------- streamed widths and chunks

STREAM_METRICS = {O.VECTOR: [O.L2_SQUARED, O.NEG_IP, O.L1], O.HALFVEC: [O.L2_SQUARED, O.NEG_IP, O.L1], O.BIT: [O.HAMMING, O.JACCARD]}
DIST_METRICS = {O.VECTOR: [O.L2, O.L2_SQUARED, O.IP, O.NEG_IP, O.L1], O.HALFVEC: [O.L2, O.L2_SQUARED, O.IP, O.NEG_IP, O.L1],
                O.BIT: [O.HAMMING, O.JACCARD]}


def stream_sizes(elem, dim):
    """n = 1, one LDG step of rows +- 1, one chunk +- 1, and two chunks and a row"""
    g, cr = rows_per_step(words(elem, dim)), chunk_rows(elem, dim)
    return sorted({1, g - 1, g, g + 1, cr - 1, cr, cr + 1, 2 * cr + 1} - {0})


@gpu
@pytest.mark.parametrize("kind,dim", WIDTHS)
def test_streamed_scan_at_every_row_width(pv, kind, dim):
    """8 queries (never tiled) at scan_impl 0 (LDG) and 1 (bulk copy where the row allows it), the table grown through
    n = 1, one LDG step of rows +- 1 and one chunk +- 1 to two chunks and a row; k = 10 and n + 1 (every row's distance
    in order); then distance_batch, the f64 instantiation, against the oracle"""
    e = ELEMS[kind]
    sizes = stream_sizes(e, dim)
    X, Q = grid(e, sizes[-1], dim, seed=dim), grid(e, 8, dim, seed=dim + 1)
    kvs = {m: keys(e, m, Q, X, dim) for m in STREAM_METRICS[e]}
    t = pv.Table(e, dim)
    for n in sizes:
        t.append(X[len(t):n])
        for impl in (0, 1):
            assert route(e, STREAM_METRICS[e][0], len(Q), n, impl, dim) == ("bulk" if impl and bulk_supported(e, dim) else "ldg")
            for metric, kv in kvs.items():
                for k in (10, n + 1):
                    check_run(pv, t, e, dim, metric, Q, kv[:, :n], k, impl, f"{kind}({dim}) n={n} impl={impl} m={metric}")
    t.free()
    n = sizes[-1]
    for metric, kv in kvs.items():     # the restated keys are the oracle's distances
        want = O.distance_batch(e, metric, Q[0], X, dim=dim)
        assert np.array_equal(kv[0], want.astype(np.float32) if metric == O.JACCARD else want), (kind, dim, metric)
        wi, wd = reference(metric, kv, n + 1)
        assert_oracle_agrees(e, metric, Q, X, dim, n + 1, wi, wd, (0, 7))
    for impl in (0, 1):
        with scan_impl(pv, impl):
            for metric in DIST_METRICS[e]:
                got = pv.distance_batch(e, metric, Q[3], X, dim=dim)
                assert np.array_equal(got, O.distance_batch(e, metric, Q[3], X, dim=dim)), (kind, dim, metric, impl)


@gpu
@pytest.mark.parametrize("kind,dim", WIDTHS)
def test_filtered_scan_and_rerank_at_every_row_width(pv, kind, dim):
    """the gather instantiation of the scan: a filter of every third row and the last, and candidate lists in random
    order with holes (-1), over two chunks and a row; k = 10 and past the allowed rows (padding)"""
    e = ELEMS[kind]
    n = stream_sizes(e, dim)[-1]
    X, Q = grid(e, n, dim, seed=dim + 2), grid(e, 8, dim, seed=dim + 3)
    allowed = np.union1d(np.arange(0, n, 3), [n - 1])
    rng = np.random.default_rng(dim)
    c = min(n, 300)
    cand = np.stack([rng.permutation(n)[:c] for _ in range(len(Q))]).astype(np.int64)
    cand[:, 5::7] = -1
    t = pv.Table(e, dim).append(X)
    f = t.filter(allowed)
    for metric in STREAM_METRICS[e]:
        kv = keys(e, metric, Q, X, dim)
        for k in (10, min(len(allowed) + 1, 2048)):
            ids, dist = t.exact_topk(metric, Q, k, filter=f)
            wi, wd = reference(metric, kv[:, allowed], k)
            assert_same(ids, dist, np.where(wi >= 0, allowed[np.maximum(wi, 0)], -1), wd, f"filter {kind}({dim}) m={metric} k={k}")
        for k in (10, c + 1):
            ids, dist = t.rerank(metric, Q, cand, k)
            for j in range(len(Q)):
                valid = cand[j][cand[j] >= 0]
                wi, wd = reference(metric, kv[j:j + 1, valid], k)
                assert_same(ids[j:j + 1], dist[j:j + 1], np.where(wi >= 0, valid[np.maximum(wi, 0)], -1), wd,
                            f"rerank {kind}({dim}) m={metric} k={k} query {j}")
    f.free()
    t.free()


@gpu
@pytest.mark.parametrize("n", [102400, 102401])
def test_bulk_copy_threshold_at_50_mib(pv, n):
    """scan_impl 2 streams a table of exactly 50 MiB with the LDG scan and one row more with the bulk copy; 8 queries,
    k = 10 and every row"""
    e, dim = O.VECTOR, 128
    X, Q = grid(e, n, dim, seed=12), grid(e, 8, dim, seed=13)
    t = pv.Table(e, dim).append(X)
    for metric in (O.L2_SQUARED, O.NEG_IP):
        assert route(e, metric, len(Q), n, 2, dim) == ("bulk" if n > 102400 else "ldg")
        kv = keys(e, metric, Q, X, dim)
        for k in (10, n + 1):
            wi, wd = check_run(pv, t, e, dim, metric, Q, kv, k, 2, f"n={n} m={metric}")
        assert_oracle_agrees(e, metric, Q, X, dim, n + 1, wi, wd, (0,))
    t.free()


# ------------------------------------------------------------------------------------------------------ sub-batches

def million_reference(X, Q, k):
    """select() over a large table, a block of queries at a time"""
    ids, kv = [], []
    block = max(1, (1 << 25) // len(X))
    for j in range(0, len(Q), block):
        i, v = select(keys(O.VECTOR, O.L2_SQUARED, Q[j:j + block], X, 4), k)
        ids.append(i)
        kv.append(v)
    return np.concatenate(ids), np.concatenate(kv)


@gpu
def test_sub_batches_of_a_million_rows(pv):
    """2^20 vector(4) rows: 256 queries per sub-batch.  576 queries are three tiled sub-batches; 575 end on a streamed
    one of 63.  k = 10 and 2049 (the sorted path in every sub-batch); the device variant's floats are the host's doubles
    rounded.  Grid rows of 4 dimensions tie by the hundred thousand."""
    import torch
    X, Q = grid(O.VECTOR, MILLION, 4, seed=20), grid(O.VECTOR, 576, 4, seed=21)
    wi, wk = million_reference(X, Q, 2049)      # (the top 10 are its first 10)
    for j in (0, 575):
        oi, od = O.exact_topk(O.VECTOR, O.L2_SQUARED, Q[j], X, 2049)
        assert np.array_equal(oi, wi[j]) and np.array_equal(od, wk[j]), j
    t = pv.Table(O.VECTOR, 4).append(X)
    for nq in (576, 575):
        for k in (10, 2049):
            ids, dist, used = run(pv, t, O.L2_SQUARED, Q[:nq], k, 2)
            assert used == launches(O.VECTOR, 4, nq, MILLION, k), (nq, k, used)
            assert_same(ids, dist, wi[:nq, :k], wk[:nq, :k], f"nq={nq} k={k}")
    Qd = torch.from_numpy(Q[:575]).cuda()
    before = pv.launch_count()
    with scan_impl(pv, 2):
        ids, dist = t.exact_topk(O.L2_SQUARED, Qd, 10)
    assert pv.launch_count() - before == launches(O.VECTOR, 4, 575, MILLION, 10)
    assert np.array_equal(ids.cpu().numpy(), wi[:575, :10])
    assert np.array_equal(dist.cpu().numpy(), wk[:575, :10].astype(np.float32))
    t.free()


@gpu
@pytest.mark.parametrize("n", [FOUR_MILLION, FOUR_MILLION + 1])
def test_sub_batch_size_at_four_million_rows(pv, n):
    """4 Mi rows take 64 queries per sub-batch (one tiled sub-batch of 64); one row more takes 63 (two streamed ones)"""
    X, Q = grid(O.VECTOR, n, 4, seed=22), grid(O.VECTOR, 64, 4, seed=23)
    wi, wk = million_reference(X, Q, 257)
    oi, od = O.exact_topk(O.VECTOR, O.L2_SQUARED, Q[63], X, 257)
    assert np.array_equal(oi, wi[63]) and np.array_equal(od, wk[63])
    assert route(O.VECTOR, O.L2_SQUARED, sub_batches(64, n)[0], n, 2, 4) == ("tiled" if n == FOUR_MILLION else "ldg")
    t = pv.Table(O.VECTOR, 4).append(X)
    for k in (10, 257):
        ids, dist, used = run(pv, t, O.L2_SQUARED, Q, k, 2)
        assert used == launches(O.VECTOR, 4, 64, n, k) == 4 * len(sub_batches(64, n)), (k, used)
        assert_same(ids, dist, wi[:, :k], wk[:, :k], f"n={n} k={k}")
    t.free()


# ------------------------------------------------------------------------------------------------------ selection

_SELECTION = {}


def selection_case(n):
    """vector(4) grid rows (ties by the thousand) and 72 queries, with the restated top 2049"""
    if n not in _SELECTION:
        X, Q = grid(O.VECTOR, n, 4, seed=30 + n), grid(O.VECTOR, 72, 4, seed=31)
        _SELECTION[n] = (X, Q) + select(keys(O.VECTOR, O.L2_SQUARED, Q, X, 4), max(2049, n + 1))
    return _SELECTION[n]


@gpu
@pytest.mark.parametrize("k", K_STEPS)
def test_selection_at_every_k_step(pv, k):
    """k across every power of two of the bitonic sort and past 2048 (the sorted path), 72 queries over 100 000 rows:
    tiled (scan_impl 2) and streamed (scan_impl 0)"""
    n = 100_000
    X, Q, wi, wk = selection_case(n)
    t = pv.Table(O.VECTOR, 4).append(X)
    for impl in (2, 0):
        ids, dist, used = run(pv, t, O.L2_SQUARED, Q, k, impl)
        assert used == launches(O.VECTOR, 4, len(Q), n, k), (k, impl, used)
        assert_same(ids, dist, wi[:, :k], wk[:, :k], f"k={k} impl={impl}")
    if k in (1, 2049):
        for j in (0, 71):
            oi, od = O.exact_topk(O.VECTOR, O.L2_SQUARED, Q[j], X, k)
            assert np.array_equal(oi, wi[j, :k]) and np.array_equal(od, wk[j, :k]), j
    t.free()


@gpu
@pytest.mark.parametrize("n", [1500, 3000])
def test_selection_at_k_around_n(pv, n):
    """k = n - 1 (the radix passes), n (every row: no radix pass) and n + 1 (padding); below and above 2048"""
    X, Q, wi, wk = selection_case(n)
    t = pv.Table(O.VECTOR, 4).append(X)
    for impl in (2, 0):
        for k in (n - 1, n, n + 1):
            ids, dist, used = run(pv, t, O.L2_SQUARED, Q, k, impl)
            assert used == launches(O.VECTOR, 4, len(Q), n, k), (k, impl, used)
            assert_same(ids, dist, wi[:, :k], wk[:, :k], f"n={n} k={k} impl={impl}")
    t.free()


# ------------------------------------------------------------------------------------------- the query image limit

@gpu
def test_rows_past_the_scan_query_image_are_refused(pv):
    """a table or distance batch whose query image is over the 227 KiB the scan can hold is refused before anything
    runs, with the limit in the message; rows at the limit scan like any other"""
    for e, d in IMAGE_LIMIT.items():
        rows = np.zeros((2, raw_bytes(e, d + 1) // (4 if e == O.VECTOR else 2 if e == O.HALFVEC else 1)),
                        np.float32 if e == O.VECTOR else np.uint16 if e == O.HALFVEC else np.uint8)
        with pytest.raises(pv.VecB200Error, match="227 KiB"):
            pv.Table(e, d + 1)
        metric = O.HAMMING if e == O.BIT else O.L2_SQUARED
        with pytest.raises(pv.VecB200Error, match="227 KiB"):
            pv.distance_batch(e, metric, rows[0], rows, dim=d + 1)
    for e, d in IMAGE_LIMIT.items():
        X, Q = grid(e, 40, d, seed=40), grid(e, 2, d, seed=41)
        t = pv.Table(e, d).append(X)
        for metric in ((O.HAMMING, O.JACCARD) if e == O.BIT else (O.L2_SQUARED, O.NEG_IP)):
            kv = keys(e, metric, Q, X, d)
            check_run(pv, t, e, d, metric, Q, kv, 41, 0, f"elem {e} at the limit m={metric}")
            assert np.array_equal(pv.distance_batch(e, metric, Q[0], X, dim=d), O.distance_batch(e, metric, Q[0], X, dim=d))
        t.free()
