"""Device scratch of nested library calls (Scratch, vb_runtime.cu): calls that take ranges of the one scratch arena,
run interleaved in one process at growing sizes so that inner calls overflow the arena while their callers hold
ranges, give exactly what each gives in a process that makes only that call; and a repeated search, once warm,
allocates no device memory."""
import os
import subprocess
import sys
import tempfile

import numpy as np
import pytest

import oracle as O

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SIZES = (1, 3, 8)   # growing: each round's calls need more scratch than the arena holds after the round before


def _dense(seed, n, dim):
    return np.random.default_rng(seed).standard_normal((n, dim)).astype(np.float32)


def _sparse_topk(pv, s):
    S = pv.sparsevec
    rng = np.random.default_rng(100 + s)
    dim, n = 2000, 400 * s
    rows = []
    for _ in range(n):
        nnz = int(rng.integers(1, 60))
        idx = np.sort(rng.choice(dim, nnz, replace=False))
        rows.append(S.SparseVector(dim, idx.tolist(), rng.standard_normal(nnz).astype(np.float32).tolist()))
    queries = rows[: 16 * s]
    t = S.SparseTable(dim)
    t.append(rows)
    filters = [t.filter(np.sort(rng.choice(n, m, replace=False))) for m in (5, n // 3, n - 1)]
    fq = rng.integers(0, len(filters), len(queries)).astype(np.int32)
    ids, dist = t.exact_topk(O.L2, queries, 10, filter=filters, filter_of_query=fq)
    for f in filters:
        f.free()
    return [ids, dist]


def _ivf(pv, s, seed):
    dim, n, lists = 64, 3000 * s, 8 * s
    rows = _dense(seed, n, dim)
    ix = pv.IvfflatIndex("vector_l2_ops", dim, lists)
    built = ix.build(rows, np.arange(n, dtype=np.int64), seed=seed)
    return ix, rows, built


def _ivf_build(pv, s):
    _, _, (lists, order, iters) = _ivf(pv, s, 200 + s)
    return [lists, order, np.array([iters])]


def _ivf_filtered_search(pv, s):
    ix, rows, _ = _ivf(pv, s, 300 + s)
    rng = np.random.default_rng(301 + s)
    with ix.filter(np.sort(rng.choice(len(rows), len(rows) // 2, replace=False))) as f:
        ids, dist = ix.search(rows[: 300 * s] + 0.01, k=10, probes=4, filter=f)
    return [ids, dist]


def _kmeans(pv, s):
    samp = _dense(400 + s, 2000 * s, 32)
    t = pv.Table(pv.VECTOR, 32).append(samp)
    centers, iters = pv.kmeans(t, pv.L2, samp[: 16 * s].copy(), max_iter=10)
    t.free()
    return [np.asarray(centers), np.asarray(iters)]


def _hnsw_build(pv, s):
    x = _dense(500 + s, 1500 * s, 16)
    gi = pv.HnswIndex("vector_l2_ops", 16, m=8).build(x, ef_construction=32, seed=3)
    ids, dist, _ = gi.search(x[: 64 * s], k=10, ef_search=40)
    return [ids, dist]


def _vector_in(pv, s):
    x = _dense(600 + s, 500 * s, 24 * s)
    rows = pv.vector_in(["[" + ",".join(repr(float(v)) for v in r) + "]" for r in x])
    return [np.stack(rows)]


def _order_bounds(pv, s):
    x = np.round(_dense(700 + s, 4000 * s, 8))
    t = pv.Table(pv.VECTOR, 8).append(x)
    o = t.order()
    lo, hi = o.bounds(x[: 200 * s])
    return [lo, hi]


CALLS = {"sparse_topk_filtered": _sparse_topk, "ivf_search_filtered": _ivf_filtered_search, "kmeans": _kmeans,
         "hnsw_build": _hnsw_build, "vector_in": _vector_in, "ivf_build": _ivf_build, "order_bounds": _order_bounds}


def run_alone(name, s, path):
    """what `name` at size s gives in a process that makes only that call (run in a subprocess)"""
    import pgvector_b200 as pv
    pv.init(0)
    np.savez(path, *CALLS[name](pv, s))


@pytest.mark.gpu
def test_interleaved_calls_match_each_call_alone():
    import pgvector_b200 as pv
    pv.init(0)
    got = {}
    for s in SIZES:
        for name, call in CALLS.items():
            got[(name, s)] = call(pv, s)
    with tempfile.TemporaryDirectory() as tmp:
        for (name, s), arrays in got.items():
            path = os.path.join(tmp, f"{name}_{s}.npz")
            code = f"import sys; sys.path.insert(0, {ROOT!r}); from tests.test_gpu_scratch import run_alone; run_alone({name!r}, {s}, {path!r})"
            subprocess.run([sys.executable, "-c", code], check=True, cwd=ROOT)
            with np.load(path) as want:
                assert len(want.files) == len(arrays), name
                for i, a in enumerate(arrays):
                    b = want[f"arr_{i}"]
                    assert a.shape == b.shape and a.tobytes() == b.tobytes(), f"{name} at size {s}: output {i} differs"


class _PoolWatch:
    """high-water mark of the device's current memory pool, which the library's stream-ordered one-off allocations
    (Scratch::own, and take() beyond the arena) come from; the driver resets it to the memory in use on request"""

    USED_MEM_HIGH = 8   # CU_MEMPOOL_ATTR_USED_MEM_HIGH

    def __init__(self):
        import ctypes as C
        self.C, self.cu = C, C.CDLL("libcuda.so.1")
        dev = C.c_int()
        self.pool = C.c_void_p()
        assert self.cu.cuInit(0) == 0 and self.cu.cuDeviceGet(C.byref(dev), 0) == 0
        assert self.cu.cuDeviceGetMemPool(C.byref(self.pool), dev) == 0

    def reset(self):
        assert self.cu.cuMemPoolSetAttribute(self.pool, self.USED_MEM_HIGH, self.C.byref(self.C.c_uint64(0))) == 0

    def high(self):
        v = self.C.c_uint64()
        assert self.cu.cuMemPoolGetAttribute(self.pool, self.USED_MEM_HIGH, self.C.byref(v)) == 0
        return v.value


def _assert_searches_allocate_nothing(ix, queries):
    import torch
    for _ in range(3):
        ix.search(queries, k=10, probes=4)
    torch.cuda.synchronize()
    watch = _PoolWatch()
    watch.reset()
    free_before = torch.cuda.mem_get_info()[0]
    for _ in range(50):
        ix.search(queries, k=10, probes=4)
    torch.cuda.synchronize()
    assert watch.high() == 0, "a warm search made stream-ordered one-off allocations"
    assert torch.cuda.mem_get_info()[0] == free_before, "a warm search grew device memory"


@pytest.mark.gpu
def test_repeated_search_allocates_nothing():
    import pgvector_b200 as pv
    pv.init(0)
    ix, rows, _ = _ivf(pv, 4, 7)
    for name, call in CALLS.items():   # the other calls grow the arena and leave their one-off allocations behind
        call(pv, 2)
    _assert_searches_allocate_nothing(ix, rows[:1000] + 0.01)


@pytest.mark.gpu
def test_a_failed_oversized_call_leaves_later_calls_allocation_free():
    import ctypes as C
    import pgvector_b200 as pv
    pv.init(0)
    ix, rows, _ = _ivf(pv, 4, 9)
    queries = rows[:1000] + 0.01
    _assert_searches_allocate_nothing(ix, queries)
    # an exact top-k whose selection needs 8 B x 64 queries x (2^31 - 1) results (~1.1 TB): refused with VB_ENOMEM when
    # the scratch is taken, before anything is written to the (one-entry) outputs
    t = pv.Table(pv.VECTOR, 64).append(rows[:1])
    q = np.ascontiguousarray(rows[:64])
    ids, dist = np.zeros(1, np.int64), np.zeros(1, np.float64)
    lib = pv._lib.load()
    rc = lib.vb_exact_topk(t.h, O.L2, q.ctypes.data_as(C.c_void_p), 64, 2**31 - 1, ids.ctypes.data_as(C.c_void_p),
                           dist.ctypes.data_as(C.c_void_p))
    assert rc == -4, lib.vb_last_error().decode()   # VB_ENOMEM
    t.free()
    _assert_searches_allocate_nothing(ix, queries)
