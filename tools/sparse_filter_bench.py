"""Filtered and re-ranked sparsevec queries on a SPLADE-like resident table: 2M rows of dimension 30 522, per-row nnz
lognormal with a mean near 120 (indices skewed towards the low term ids, positive weights), from a seed; 64 queries of
about 30 nnz, k = 10.  It times, with CUDA events around back-to-back synchronous calls over a window of at least a
second after two warm-up calls:
  - vb_sparse_exact_topk, unfiltered, for reference;
  - vb_sparse_exact_topk_filtered at 0.1 %, 1 %, 10 % and 100 % selectivity, with one filter for the batch and with 16
    filters assigned by filter_of_query (query q takes filter q % 16);
  - vb_sparse_table_rerank with 1000 random candidates per query.
For each it reports ms per call and the algorithmic bytes -- for every query, the sum over the rows it scores of 8 B per
stored entry (index and value) plus 16 B of offsets -- over the time, as a fraction of the H100's 3.35 TB/s.  The card's
name and power limit are read in the same run.  Checks, at the timed size: the 100 % filter equals the unfiltered call
bit for bit, and the 1 % filters equal the re-rank of their allowed rows in ascending order.
Usage: python tools/sparse_filter_bench.py [--rows N] [--dim D] [--nnz MEAN] [--queries Q] [--seed S]"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

HBM_BYTES_PER_S = 3.35e12


def card():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=60)
        return [line.strip() for line in r.stdout.splitlines() if line.strip()] or r.stderr.strip()
    except (OSError, subprocess.SubprocessError) as e:
        return f"nvidia-smi failed: {e}"


def make_csr(n, dim, mean_nnz, sigma, rng, torch, dev):
    """n rows: nnz ~ lognormal (mean mean_nnz), indices u^2-skewed over [0, dim), sorted and distinct, positive values"""
    mu = np.log(mean_nnz) - sigma * sigma / 2
    nnz = np.clip(np.rint(rng.lognormal(mu, sigma, n)), 1, 16000).astype(np.int64)
    g = torch.Generator(device=dev).manual_seed(int(rng.integers(1 << 62)))
    row = torch.repeat_interleave(torch.arange(n, device=dev), torch.from_numpy(nnz).to(dev))
    u = torch.rand(row.numel(), device=dev, generator=g, dtype=torch.float64)
    idx = torch.clamp((u * u * dim).to(torch.int64), max=dim - 1)
    key, _ = torch.sort(row * dim + idx)
    keep = torch.ones_like(key, dtype=torch.bool)
    keep[1:] = key[1:] != key[:-1]
    key = key[keep]
    row, idx = key // dim, key % dim
    counts = torch.bincount(row, minlength=n)
    off = torch.zeros(n + 1, dtype=torch.int64, device=dev)
    off[1:] = torch.cumsum(counts, 0)
    val = torch.rand(idx.numel(), device=dev, generator=g) * 2 + 0.01
    return off.cpu().numpy(), idx.to(torch.int32).cpu().numpy(), val.cpu().numpy()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=2_000_000)
    ap.add_argument("--dim", type=int, default=30_522)
    ap.add_argument("--nnz", type=float, default=120.0)
    ap.add_argument("--queries", type=int, default=64)
    ap.add_argument("--cands", type=int, default=1000)
    ap.add_argument("--window_s", type=float, default=1.0)
    ap.add_argument("--seed", type=int, default=2024)
    args = ap.parse_args()
    import torch
    import pgvector_b200 as pv
    S = pv.sparsevec
    pv.init(0)
    dev = torch.device("cuda", 0)
    rng = np.random.default_rng(args.seed)
    n, k, nq = args.rows, 10, args.queries
    off, idx, val = make_csr(n, args.dim, args.nnz, 0.6, rng, torch, dev)
    table = S.SparseTable(args.dim).append(S.SparseRows(args.dim, off, idx, val))
    qoff, qidx, qval = make_csr(nq, args.dim, 30.0, 0.1, rng, torch, dev)
    Q = S.SparseRows(args.dim, qoff, qidx, qval)
    row_bytes = 8 * np.diff(off) + 16
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

    def entry(ms, steps, nbytes):
        return {"ms": ms, "calls_timed": steps, "algorithmic_bytes": int(nbytes),
                "fraction_of_3.35_TB/s": nbytes / (ms / 1e3) / HBM_BYTES_PER_S}

    out = {"bench": "sparse_filter", "card": card(),
           "workload": f"sparsevec {n} rows x dim {args.dim}, nnz lognormal mean ~{args.nnz:g} (stored {len(idx) / n:.1f}/row), "
                       f"{nq} queries of ~{len(qidx) / nq:.1f} nnz, k={k}",
           "timing": f"CUDA events around back-to-back synchronous calls, window >= {args.window_s:g} s after 2 warm-up calls"}
    ms, st = timed(lambda: table.exact_topk(S.L2, Q, k))
    out["unfiltered"] = entry(ms, st, nq * row_bytes.sum())
    want = table.exact_topk(S.L2, Q, k)
    results, checks = [], {}
    fq16 = (np.arange(nq) % 16).astype(np.int32)
    for sel in (0.001, 0.01, 0.1, 1.0):
        for nf in (1, 16):
            allowed = [np.arange(n) if sel == 1.0 else np.sort(rng.choice(n, int(n * sel), replace=False)) for _ in range(nf)]
            filters = [table.filter(a) for a in allowed]
            fq = None if nf == 1 else fq16
            farg = filters[0] if nf == 1 else filters
            ms, st = timed(lambda: table.exact_topk(S.L2, Q, k, filter=farg, filter_of_query=fq))
            per_filter = [row_bytes[a].sum() for a in allowed]
            nbytes = sum(per_filter[0 if fq is None else fq[q]] for q in range(nq))
            results.append({"selectivity": sel, "filters": nf, **entry(ms, st, nbytes),
                            "vs_unfiltered": out["unfiltered"]["ms"] / ms})
            got = table.exact_topk(S.L2, Q, k, filter=farg, filter_of_query=fq)
            if sel == 1.0:
                checks[f"full_filter_x{nf}_equals_unfiltered"] = bool(
                    np.array_equal(got[0], want[0]) and np.array_equal(got[1].view(np.int64), want[1].view(np.int64)))
            if sel == 0.01:
                ok = True
                for j in range(nf):
                    sel_q = np.arange(nq) if fq is None else np.flatnonzero(fq == j)
                    sub = S.SparseRows.from_vectors([Q.row(int(q)) for q in sel_q], args.dim)
                    rr = table.rerank(S.L2, sub, np.tile(allowed[j].astype(np.int64), (sel_q.size, 1)), k)
                    ok = ok and np.array_equal(got[0][sel_q], rr[0]) and np.array_equal(got[1][sel_q].view(np.int64), rr[1].view(np.int64))
                checks[f"filter_1pct_x{nf}_equals_rerank"] = bool(ok)
            for f in filters:
                f.free()
    out["filtered"] = results
    cand = rng.integers(0, n, size=(nq, args.cands)).astype(np.int64)
    ms, st = timed(lambda: table.rerank(S.L2, Q, cand, k))
    out["rerank"] = {"candidates_per_query": args.cands, **entry(ms, st, row_bytes[cand].sum())}
    out["checks"] = checks
    out["checks_pass"] = all(checks.values())
    table.free()
    print(json.dumps(out))
    if not out["checks_pass"]:
        sys.exit(1)


if __name__ == "__main__":
    main()
