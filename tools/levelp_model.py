#!/usr/bin/env python3
"""CPU model of a projection lower-bound level (level P) in front of the batched IVFFlat list scan, to be run before any
kernel is written for it.

For any r x dim matrix P with spectral norm ||P||_2 <= sigma, |x - q|^2 >= |P(x - q)|^2 / sigma^2 for every row x and
query q.  The basis only decides how tight the bound is.  This model takes P from the index's own rows: the k-means
sample, subspace iteration for the top dim/8 directions, r = the smallest multiple of 16 that holds at
least 90 % of the sample's energy about the origin (no level P when none does), sigma^2 from a Gershgorin bound on P P^T
in double.  It draws bench.py's config-B data through bench.py's own functions on the CPU (the law and shape match; the
random draw differs from the GPU's), builds the index with bench.py's reference-arm recipe and takes each query's probe
lists from the CPU oracle.  It then evaluates the LIST refine's rule with d~ = LB and zero per-row terms:
    re-score the k smallest LB, T1 = their k-th exact distance; re-score the other listed ones with LB <= T1;
    T = the k-th exact distance of the re-scored set; a query fails when it has more than k' candidates and the k'-th
    smallest LB is <= T,
and reports r, the rows re-scored per query (mean, p90) and the failures per 2048-query batch for k' = 64 and 128.
LB is formed here in float64 from fp32 projections; the kernel's rounded-down fp32 LB is lower by a relative 1e-4 at
most, far below the gap between LB and the distance on these laws.

    python tools/levelp_model.py [--rows N --dim D --lists L --probes P --queries Q --law rank16|mixture]
"""
from __future__ import annotations

import argparse
import json
import os
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def basis(sample, rng, iters=6, frac=0.9):
    """(P fp32 r x dim, sigma^2 upper bound, energy captured by r, eigenvalue profile) or (None, ...) when no r <= dim/8 holds
    frac of the sample's energy about the origin"""
    s = sample.astype(np.float64)
    dim = s.shape[1]
    cap = max(16, (dim // 8) // 16 * 16)
    b = np.linalg.qr(rng.standard_normal((dim, cap)))[0]
    for _ in range(iters):
        b = np.linalg.qr(s.T @ (s @ b))[0]
    sb = s @ b
    lam, v = np.linalg.eigh(sb.T @ sb)
    lam, v = lam[::-1], v[:, ::-1]
    total = float((s * s).sum())
    cum = np.cumsum(lam) / total
    r = next((m for m in range(16, cap + 1, 16) if cum[m - 1] >= frac), None)
    if r is None:
        return None, None, float(cum[cap - 1]), cap
    p = (b @ v[:, :r]).T.astype(np.float32)
    g = p.astype(np.float64) @ p.astype(np.float64).T
    sigma2 = float(np.abs(g).sum(1).max()) * (1 + 2.0 ** -40)
    return p, sigma2, float(cum[r - 1]), r


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=1_000_000)
    ap.add_argument("--dim", type=int, default=1536)
    ap.add_argument("--lists", type=int, default=1000)
    ap.add_argument("--probes", type=int, default=10)
    ap.add_argument("--queries", type=int, default=2048)
    ap.add_argument("--k", type=int, default=10)
    ap.add_argument("--law", default="rank16", choices=["rank16", "mixture"])
    a = ap.parse_args()
    os.environ["VB_BENCH_CACHE"] = tempfile.mkdtemp(prefix="levelp_model_")
    import torch
    import bench
    import oracle as O

    bargs = argparse.Namespace(rows=a.rows, dim=a.dim, lists=a.lists, latent_dim=16, components=1000, queries=a.queries)
    rows_t, q_t = bench.make_dataset(bargs, a.law, torch.device("cpu"))
    centers_t, offsets, grouped_t, order_t, how = bench.build_index_arrays(bargs, a.law, rows_t, None)
    del rows_t
    grouped = grouped_t.numpy()
    centers, queries = centers_t.numpy(), q_t.numpy().astype(np.float32)
    oix = O.Ivf(O.VECTOR, O.L2_SQUARED, centers, offsets, grouped, order_t.numpy())

    rng = np.random.default_rng(42)
    ns = min(a.rows, max(a.lists * 50, 10000))
    sample = grouped[np.sort(rng.choice(a.rows, ns, replace=False))]
    p, sigma2, energy, r = basis(sample, rng)
    out = {"tool": "levelp_model",
           "workload": f"bench.py {a.law} law, {a.rows}x{a.dim}, lists={a.lists}, probes={a.probes}, k={a.k}, "
                       f"{a.queries} queries (CPU draw; {how})"}
    if p is None:
        out.update({"levelp": False, "energy_at_cap": energy, "cap": r})
        print(json.dumps(out))
        return
    y = np.empty((a.rows, r), np.float32)
    for lo in range(0, a.rows, 65536):
        y[lo:lo + 65536] = grouped[lo:lo + 65536] @ p.T
    fails = {64: 0, 128: 0}
    rescored = {64: [], 128: []}
    gap = []
    for qi in range(a.queries):
        q = queries[qi]
        lists, _ = oix.scan_lists(q, a.probes)
        cand = np.concatenate([np.arange(offsets[l], offsets[l + 1]) for l in lists if l >= 0])
        yq = p @ q
        lb = ((y[cand].astype(np.float64) - yq) ** 2).sum(1) / sigma2
        order = np.argsort(lb, kind="stable")
        sl = lb[order]
        top = cand[order[:128]]
        diff = grouped[top] - q                                               # fp32, as the oracle forms it
        exact = (diff.astype(np.float64) ** 2).sum(1)
        assert (sl[:128] <= exact * (1 + 1e-6)).all()
        gap.append(float(np.median(exact[:a.k] - sl[:a.k])))
        kk = min(a.k, len(sl))
        t1 = exact[:kk].max() if kk == a.k else np.inf
        for kp in (64, 128):
            sel = np.concatenate([np.arange(kk), kk + np.flatnonzero(~(sl[kk:kp] > t1))])
            t = np.sort(exact[sel])[a.k - 1] if len(sel) >= a.k else np.inf
            rescored[kp].append(len(sel))
            if len(sl) > kp and not sl[kp - 1] > t:
                fails[kp] += 1
    per_batch = lambda f: f * 2048 / a.queries
    out.update({
        "levelp": True, "r": r, "energy_captured": energy, "sigma2": sigma2,
        "plane_bytes_per_row": 4 * r, "median_exact_minus_lb_top_k": float(np.median(gap)),
        "rescored_rows_per_query_mean": {str(kp): float(np.mean(rescored[kp])) for kp in rescored},
        "rescored_rows_per_query_p90": {str(kp): float(np.percentile(rescored[kp], 90)) for kp in rescored},
        "failures_per_2048_batch": {str(kp): per_batch(fails[kp]) for kp in fails},
    })
    print(json.dumps(out))


if __name__ == "__main__":
    main()
