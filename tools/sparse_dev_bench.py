"""sparsevec calls on device buffers against their host variants, on the table of tools/sparse_filter_bench.py (2M
SPLADE-like rows of dimension 30 522, nnz lognormal with a mean near 120; 64 queries of about 30 nnz, k = 10), and the
throughput of the casts between vector / halfvec and sparsevec.  Timing as sparse_filter_bench.py: CUDA events around
back-to-back synchronous calls (the Python mirrors hand back complete results), a window of at least a second after two
warm-up calls.  It reports, for the exact, the 1 % filtered and the 1000-candidate re-rank call and for an append of
200k rows: ms per call of the host and of the _dev variant, and the host <-> device bytes the _dev variant does not move
(queries, candidates and results; the appended rows).  The casts run on 32k rows of the same distribution at dimension
16 000 (the largest a vector or halfvec may have): rows / s and the algorithmic bytes (dense rows read once, CSR written
or read) over the time as a fraction of 3.35 TB/s.
The card's name and power limit are read in the same run.  Checks: every _dev result equals the host variant's (ids,
float of the float8), and the casts invert each other.
Usage: python tools/sparse_dev_bench.py [--rows N] [--dim D] [--nnz MEAN] [--queries Q] [--cast_rows R] [--cast_dim E] [--seed S]"""
import argparse
import json
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from sparse_filter_bench import HBM_BYTES_PER_S, card, make_csr  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=2_000_000)
    ap.add_argument("--dim", type=int, default=30_522)
    ap.add_argument("--nnz", type=float, default=120.0)
    ap.add_argument("--queries", type=int, default=64)
    ap.add_argument("--cands", type=int, default=1000)
    ap.add_argument("--append_rows", type=int, default=200_000)
    ap.add_argument("--cast_rows", type=int, default=32_768)
    ap.add_argument("--cast_dim", type=int, default=16_000)
    ap.add_argument("--window_s", type=float, default=1.0)
    ap.add_argument("--seed", type=int, default=2024)
    args = ap.parse_args()
    import torch
    import pgvector_b200 as pv
    S = pv.sparsevec
    pv.init(0)
    dev = torch.device("cuda", 0)
    rng = np.random.default_rng(args.seed)
    n, k, nq, c = args.rows, 10, args.queries, args.cands
    off, idx, val = make_csr(n, args.dim, args.nnz, 0.6, rng, torch, dev)
    R = S.SparseRows(args.dim, off, idx, val)
    R_dev = tuple(torch.from_numpy(a).to(dev) for a in (off, idx, val))
    table = S.SparseTable(args.dim).append(R)
    qoff, qidx, qval = make_csr(nq, args.dim, 30.0, 0.1, rng, torch, dev)
    Q = S.SparseRows(args.dim, qoff, qidx, qval)
    Q_dev = tuple(torch.from_numpy(a).to(dev) for a in (qoff, qidx, qval))
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]

    def timed(fn):
        for _ in range(2):
            fn()
        ev[0].record()
        fn()
        ev[1].record()
        ev[1].synchronize()
        steps = max(3, int(np.ceil(args.window_s * 1e3 / max(ev[0].elapsed_time(ev[1]), 1e-3))))
        ev[0].record()
        for _ in range(steps):
            fn()
        ev[1].record()
        ev[1].synchronize()
        return ev[0].elapsed_time(ev[1]) / steps, steps

    def same(got, want):
        ids, dist = got[0].cpu().numpy(), got[1].cpu().numpy()
        w = want[1].astype(np.float32)
        return bool(np.array_equal(ids, want[0]) and np.array_equal(np.isnan(dist), np.isnan(w))
                    and np.array_equal(dist[~np.isnan(w)].view(np.int32), w[~np.isnan(w)].view(np.int32)))

    q_bytes = 8 * (nq + 1) + 8 * len(qidx)     # offsets, indices and values of the queries
    res_bytes = nq * k * (8 + 8)               # ids and float8 distances back
    out = {"bench": "sparse_dev", "card": card(),
           "workload": f"sparsevec {n} rows x dim {args.dim}, stored nnz {len(idx) / n:.1f}/row, {nq} queries of ~{len(qidx) / nq:.1f} "
                       f"nnz, k={k}",
           "timing": f"CUDA events around back-to-back synchronous calls, window >= {args.window_s:g} s after 2 warm-up calls"}
    legs, checks = {}, {}
    allowed = np.sort(rng.choice(n, n // 100, replace=False))
    f = table.filter(allowed)
    cand = rng.integers(0, n, size=(nq, c)).astype(np.int64)
    cand_dev = torch.from_numpy(cand).to(dev)
    for name, host_fn, dev_fn, saved in (
            ("exact", lambda: table.exact_topk(S.L2, Q, k), lambda: table.exact_topk(S.L2, Q_dev, k), q_bytes + res_bytes),
            ("filtered_1pct", lambda: table.exact_topk(S.L2, Q, k, filter=f), lambda: table.exact_topk(S.L2, Q_dev, k, filter=f),
             q_bytes + res_bytes),
            ("rerank", lambda: table.rerank(S.L2, Q, cand, k), lambda: table.rerank(S.L2, Q_dev, cand_dev, k),
             q_bytes + 8 * nq * c + res_bytes)):
        h_ms, h_st = timed(host_fn)
        d_ms, d_st = timed(dev_fn)
        legs[name] = {"host_ms": h_ms, "dev_ms": d_ms, "calls_timed": [h_st, d_st], "dev_vs_host": h_ms / d_ms,
                      "host_device_bytes_saved": int(saved)}
        checks[f"{name}_dev_equals_host"] = same(dev_fn(), host_fn())
    f.free()
    # append: a fresh table per call, so every call allocates as the first append of a table does
    m = min(args.append_rows, n)
    Ra = S.SparseRows(args.dim, off[:m + 1], idx[:off[m]], val[:off[m]])
    Ra_dev = (R_dev[0][:m + 1], R_dev[1][:off[m]], R_dev[2][:off[m]])
    h_ms, h_st = timed(lambda: S.SparseTable(args.dim).append(Ra).free())
    d_ms, d_st = timed(lambda: S.SparseTable(args.dim).append(Ra_dev).free())
    legs["append"] = {"rows": m, "host_ms": h_ms, "dev_ms": d_ms, "calls_timed": [h_st, d_st], "dev_vs_host": h_ms / d_ms,
                      "host_device_bytes_saved": int(8 * (m + 1) + 8 * off[m])}
    out["calls"] = legs
    # casts: cast_rows rows of the table's distribution at cast_dim
    cr, cdim = args.cast_rows, args.cast_dim
    coff, cidx, cval = make_csr(cr, cdim, args.nnz, 0.6, rng, torch, dev)
    Rc = tuple(torch.from_numpy(a).to(dev) for a in (coff, cidx, cval))
    tot = int(coff[cr])
    csr_bytes = 8 * (cr + 1) + 8 * tot
    casts = {}
    for elem, to_dense, to_sparse, esize in ((0, S.sparsevec_to_vector, S.vector_to_sparsevec, 4),
                                            (1, S.sparsevec_to_halfvec, S.halfvec_to_sparsevec, 2)):
        name = "vector" if elem == 0 else "halfvec"
        dense = to_dense(Rc, dim=cdim)
        dense_bytes = cr * cdim * esize
        ms, st = timed(lambda: to_dense(Rc, dim=cdim))
        casts[f"sparsevec_to_{name}"] = {"ms": ms, "calls_timed": st, "rows_per_s": cr / (ms / 1e3), "algorithmic_bytes": dense_bytes + csr_bytes,
                                         "fraction_of_3.35_TB/s": (dense_bytes + csr_bytes) / (ms / 1e3) / HBM_BYTES_PER_S}
        ms, st = timed(lambda: to_sparse(dense, cap=tot))
        casts[f"{name}_to_sparsevec"] = {"ms": ms, "calls_timed": st, "rows_per_s": cr / (ms / 1e3), "algorithmic_bytes": dense_bytes + csr_bytes,
                                         "fraction_of_3.35_TB/s": (dense_bytes + csr_bytes) / (ms / 1e3) / HBM_BYTES_PER_S,
                                         "note": "two passes over the dense rows (count, write)"}
        o2, i2, v2 = to_sparse(dense, cap=tot)
        checks[f"{name}_round_trip"] = bool(torch.equal(o2, Rc[0]) and torch.equal(i2, Rc[1])
                                            and (elem == 1 or torch.equal(v2, Rc[2])))
        del dense
    out["casts"] = {"rows": cr, "dim": cdim, "stored_nnz": tot, **casts}
    out["checks"] = checks
    out["checks_pass"] = all(checks.values())
    table.free()
    print(json.dumps(out))
    if not out["checks_pass"]:
        sys.exit(1)


if __name__ == "__main__":
    main()
