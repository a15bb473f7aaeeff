"""The btree order on the device (vb_order): sort + groups of a resident table, and batched bounds.  Workloads:
  - 1M x 1536 fp32 rows, uniform random (rows differ in their first key word);
  - the same shape with every row repeated 8 times, shuffled (the deduplication case: groups of 8 equal rows);
  - 1M x 768 halfvec rows quantised to 16 levels per element (deep shared prefixes);
  - 1M sparsevec rows of dimension 30 522 with 120 stored entries each (SPLADE-like);
  - 100 000 bounds queries against the first table, half of them rows of the table.
For each it reports, in one JSON line, the ms per call (CUDA events around a call that ends in a synchronise, after one
warm-up call; median of --reps), the refinement passes, the groups, and the time one read of the table's bytes would
take at the data-sheet 3.35 TB/s (a derived floor, not a measurement), with the card's name and power limit read in the
same run.  Every timed output is checked against the CPU oracle's comparators (tests/order_oracle.c) on a subsample:
adjacent pairs of the order (sorted, ties by row number, group numbers), and for sampled queries the rows around lo and
hi.  Exit 1 on a mismatch.
Usage: python tools/order_bench.py [--rows N --reps K --pairs P --queries Q]"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

HBM = 3.35e12


def card():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=60)
        return [line.strip() for line in r.stdout.splitlines() if line.strip()] or r.stderr.strip()
    except (OSError, subprocess.SubprocessError) as e:
        return f"nvidia-smi failed: {e}"


def timed(torch, stream, fn, reps):
    fn()   # warm-up: module load, CUB's first launches
    ms = []
    for _ in range(reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(stream)
        r = fn()
        e1.record(stream)
        e1.synchronize()
        ms.append(e0.elapsed_time(e1))
        if r is not None and hasattr(r, "free"):
            r.free()
    return float(np.median(ms))


class DenseRows:
    def __init__(self, x, half):
        self.x, self.half = x, half

    def get(self, idx):
        import torch
        a = self.x[torch.as_tensor(np.asarray(idx), device=self.x.device)].cpu().numpy()
        return a.view(np.uint16) if self.half else a

    def cmp(self, OO, a, b):
        return OO.halfvec_cmp(a, b) if self.half else OO.vector_cmp(a, b)


class SparseRowsDev:
    def __init__(self, off, idx, val, dim):
        self.off, self.idx, self.val, self.dim = off, idx, val, dim

    def get(self, rows):
        import types
        out = []
        for r in np.asarray(rows).tolist():
            b, e = int(self.off[r]), int(self.off[r + 1])
            out.append(types.SimpleNamespace(dim=self.dim, indices=self.idx[b:e].cpu().numpy(), values=self.val[b:e].cpu().numpy()))
        return out

    def cmp(self, OO, a, b):
        return OO.sparsevec_cmp(a, b)


def check_order(OO, src, perm, gor, pairs, rng):
    """adjacent pairs of the order: non-decreasing by the oracle comparator, ties by row number, group numbers step by
    one exactly where the value changes"""
    n = perm.shape[0]
    pos = rng.integers(0, n - 1, pairs)
    a, b = src.get(perm[pos]), src.get(perm[pos + 1])
    bad = 0
    for k in range(pairs):
        c = src.cmp(OO, a[k], b[k])
        ok = c < 0 or (c == 0 and perm[pos[k]] < perm[pos[k] + 1])
        ok = ok and gor[perm[pos[k] + 1]] == gor[perm[pos[k]]] + (1 if c < 0 else 0)
        bad += not ok
    return bad


def check_bounds(OO, src, qsrc, perm, lo, hi, sample, rng):
    """for sampled queries: the row before lo is < q, rows lo and hi - 1 equal q, the row at hi is > q"""
    n = perm.shape[0]
    bad = 0
    for k in rng.integers(0, lo.shape[0], sample).tolist():
        q = qsrc.get([k])[0]
        l, h = int(lo[k]), int(hi[k])
        if l > 0:
            bad += src.cmp(OO, src.get([perm[l - 1]])[0], q) >= 0
        if h > l:
            bad += src.cmp(OO, src.get([perm[l]])[0], q) != 0
            bad += src.cmp(OO, src.get([perm[h - 1]])[0], q) != 0
        if h < n:
            bad += src.cmp(OO, src.get([perm[h]])[0], q) <= 0
    return bad


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=1_000_000)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--pairs", type=int, default=20000)
    ap.add_argument("--queries", type=int, default=100_000)
    args = ap.parse_args()
    import torch
    import pgvector_b200 as pv
    from tests import order_oracle as OO
    pv.init(0)
    dev = torch.device("cuda", 0)
    stream = torch.cuda.ExternalStream(pv.stream_handle())
    g = torch.Generator(device=dev).manual_seed(5)
    rng = np.random.default_rng(5)
    n = args.rows
    out = {"bench": "order", "card": card(), "hbm_peak_tb_s": HBM / 1e12, "rows": n}
    bad_total = 0

    def dense_case(name, x, half):
        nonlocal bad_total
        t = pv.Table(pv.HALFVEC if half else pv.VECTOR, x.shape[1])
        for i in range(0, x.shape[0], 131072):
            t.append(x[i:i + 131072].contiguous())
        pv.synchronize()
        ms = timed(torch, stream, t.order, args.reps)
        o = t.order()
        perm, gor, _ = o.read()
        nbytes = x.shape[0] * x.shape[1] * x.element_size()
        res = {"ms": ms, "passes": o.passes, "groups": o.groups, "table_bytes": nbytes, "full_read_floor_ms_at_3_35_tb_s": nbytes / HBM * 1e3}
        res["oracle_bad_pairs"] = check_order(OO, DenseRows(x, half), perm, gor, args.pairs, rng)
        bad_total += res["oracle_bad_pairs"]
        out[name] = res
        return t, o, perm

    x = torch.rand((n, 1536), generator=g, device=dev)
    t, o, perm = dense_case("vector_1M_x_1536_uniform", x, False)
    # bounds: half the queries are rows of the table, half are new rows
    nq = args.queries
    present = torch.randint(0, n, (nq // 2,), generator=g, device=dev)
    q = torch.cat([x[present], torch.rand((nq - nq // 2, 1536), generator=g, device=dev)]).contiguous()
    ms = timed(torch, stream, lambda: o.bounds(q), args.reps)
    lo, hi = o.bounds(q)
    lo, hi = lo.cpu().numpy(), hi.cpu().numpy()
    bad = check_bounds(OO, DenseRows(x, False), DenseRows(q, False), perm, lo, hi, 300, rng)
    bad_total += bad
    out["bounds_100k_queries_half_present"] = {"ms": ms, "queries": nq, "found": int((hi > lo).sum()), "oracle_bad_checks": bad,
                                               "log2_rows": float(np.log2(n))}
    o.free()
    t.free()
    del q

    u = torch.rand((n // 8, 1536), generator=g, device=dev)
    xr = u.repeat_interleave(8, dim=0)[torch.randperm(n // 8 * 8, generator=g, device=dev)].contiguous()
    del u
    t, o, _ = dense_case("vector_1M_x_1536_each_row_8_times", xr, False)
    o.free()
    t.free()
    del xr, x
    torch.cuda.empty_cache()

    xh = (torch.randint(0, 16, (n, 768), generator=g, device=dev).float() / 15).half()
    t, o, _ = dense_case("halfvec_1M_x_768_16_levels", xh, True)
    o.free()
    t.free()
    del xh
    torch.cuda.empty_cache()

    # sparse: 120 entries per row, one in each run of 254 indices (strictly ascending), values standard normal
    dim, nnz = 30522, 120
    idx = (torch.arange(nnz, device=dev) * 254 + torch.randint(0, 254, (n, nnz), generator=g, device=dev)).to(torch.int32).reshape(-1)
    val = torch.randn(n * nnz, generator=g, device=dev)
    off = torch.arange(0, n * nnz + 1, nnz, device=dev, dtype=torch.int64)
    st = pv.SparseTable(dim)
    st.append((off, idx, val))
    ms = timed(torch, stream, st.order, args.reps)
    so = st.order()
    perm, gor, _ = so.read()
    nbytes = n * nnz * 8 + (n + 1) * 8
    src = SparseRowsDev(off.cpu().numpy(), idx, val, dim)
    res = {"ms": ms, "passes": so.passes, "groups": so.groups, "table_bytes": nbytes, "full_read_floor_ms_at_3_35_tb_s": nbytes / HBM * 1e3,
           "oracle_bad_pairs": check_order(OO, src, perm, gor, min(args.pairs, 5000), rng)}
    bad_total += res["oracle_bad_pairs"]
    out["sparsevec_1M_dim_30522_nnz_120"] = res
    so.free()
    st.free()
    out["oracle_mismatches"] = bad_total
    print(json.dumps(out))
    sys.exit(1 if bad_total else 0)


if __name__ == "__main__":
    main()
