#!/usr/bin/env python3
"""CPU model of filter level 0 of the batched IVFFlat list scan (vb_list_tc.cu), to be run before touching its bound.

It draws bench.py's config-B data through bench.py's own functions, on the CPU. The law and shape match; the random
draw differs from the GPU's, whose generator is another. It builds the index with bench.py's reference-arm recipe
(torch k-means++ / Lloyd / assign), takes each query's probe lists from the CPU oracle (vb's GetScanLists port), and
quantises rows and queries exactly as the kernels do:
    rows:    s_x = max|x_i| / 127 (fp32), x8 = clip(rint(x / s_x), -127, 127)
    queries: t_q = max|q_i| / 127, q_hi = clip(rint(q / t_q)), q_lo = clip(rint(fl(fma(-t_q, q_hi, q) * 254) / t_q))
It then evaluates l0_query_kernel's bound eps(q) and the certificate of the refine kernels on every query's real
candidates:
    d~ = |x|^2 + |q|^2 - 2 s_x t_q (x8.q_hi + x8.q_lo / 254),  T = (k-th smallest d~) + 2 eps(q),
    a query fails when it has more than k' candidates and the k'-th smallest d~ is <= T,
    the candidates with d~ <= T among the k' are re-scored exactly.
It reports R_max (absolute and relative to |x|), eps(q) against level 1's, the failures per 2048-query batch and the
re-scored rows per query, for k' = 64 and 128.  (d~ is evaluated in float64 here; the kernel's fp32 epilogue differs from
it by far less than the bound's rounding terms.)

It also evaluates the rule the level-0 refine uses, with each row's own bound E(x, q) (R_x and |x| in the place of R_max
and x_max) and an exact threshold:
    re-score the k smallest d~, T1 = their k-th exact distance; re-score the other listed ones with d~ - E(x, q) <= T1;
    T = the k-th exact distance of the re-scored set; a query fails when it has more than k' candidates and the k'-th
    smallest d~ is <= T + eps(q),
and reports its re-scored rows per query and its failures for k' = 32, 64 and 128.

    python tools/level0_model.py [--rows N --dim D --lists L --probes P --queries Q --law rank16|mixture]
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


def quant_rows(x, slab=65536):
    """s_x, x8 (int8), the residual |x - s_x x8| and |x|^2 per row, in slabs of rows"""
    n = x.shape[0]
    sx = np.empty(n, np.float32)
    x8 = np.empty(x.shape, np.int8)
    res = np.empty(n)
    xn = np.empty(n)
    for lo in range(0, n, slab):
        xs = x[lo:lo + slab]
        s = (np.abs(xs).max(axis=1).astype(np.float32) / np.float32(127)).astype(np.float32)
        safe = np.where(s > 0, s, np.float32(1))
        q = np.where(s[:, None] > 0, np.clip(np.rint(xs / safe[:, None]), -127, 127), 0).astype(np.float32)
        sx[lo:lo + slab], x8[lo:lo + slab] = s, q.astype(np.int8)
        res[lo:lo + slab] = np.sqrt(((xs.astype(np.float64) - s[:, None].astype(np.float64) * q) ** 2).sum(1))
        xn[lo:lo + slab] = (xs.astype(np.float64) ** 2).sum(1)
    return sx, x8, res, xn


def quant_query(q):
    tq = np.float32(np.abs(q).max()) / np.float32(127)
    if not (tq > 0):
        return tq, np.zeros_like(q), np.zeros_like(q)
    h = np.clip(np.rint(q / tq), -127, 127).astype(np.float32)
    r = (q.astype(np.float64) - np.float64(tq) * h).astype(np.float32)          # fma(-t_q, h, q): one rounding
    lo = np.clip(np.rint((r * np.float32(254)).astype(np.float32) / tq), -127, 127).astype(np.float32)
    return tq, h, lo


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
    # a private index cache: bench.py's shared one is keyed without the device, and this index is drawn on the CPU
    os.environ["VB_BENCH_CACHE"] = tempfile.mkdtemp(prefix="level0_model_")
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

    sx, x8, res, xn = quant_rows(grouped)
    xnorm = np.sqrt(xn)
    rmax = float(res.max())
    xmax = float(xnorm.max())
    X = xmax * (1 + 1 / 1024) + rmax
    c_sum = max(1 / 65536, 3 * (a.dim / 32 + 8) / 16777216)
    steps = ((a.dim + 63) // 64) * 4
    c_ip1 = max(1 / 256 + 1 / 8192, 1 / 256 + 1 / 65536 + 2 * 2 * steps / 8388608)

    fails = {64: 0, 128: 0}
    rescored = {64: [], 128: []}
    row_fails = {32: 0, 64: 0, 128: 0}
    row_rescored = []
    eps0, eps1 = [], []
    w = 1 + 1 / 1024
    res_up = res * (1 + 1 / 1048576)
    Xrow = xnorm * w + res_up
    for qi in range(a.queries):
        q = queries[qi]
        lists, _ = oix.scan_lists(q, a.probes)
        cand = np.concatenate([np.arange(offsets[l], offsets[l + 1]) for l in lists if l >= 0])
        tq, h, lo = quant_query(q)
        qhat = np.float64(tq) * (h.astype(np.float64) + lo.astype(np.float64) / 254)
        n2 = float((q.astype(np.float64) ** 2).sum())
        rq = float(np.sqrt(((q - qhat) ** 2).sum()))
        qabs = float(tq) * (np.sqrt((h.astype(np.float64) ** 2).sum()) + np.sqrt((lo.astype(np.float64) ** 2).sum()) / 254)
        dot = rmax * np.sqrt(n2) + X * rq + X * qabs / 1048576 + 1e-30
        e0 = (2 * dot + c_sum * (X * X + n2)) * (1 + 1 / 1024)
        e1 = 2 * c_ip1 * np.sqrt(n2) * xmax + c_sum * (xmax * xmax + n2)
        eps0.append(e0)
        eps1.append(e1)
        xi = x8[cand].astype(np.float64)
        approx = xn[cand] + n2 - 2 * sx[cand].astype(np.float64) * float(tq) * (xi @ h.astype(np.float64) + (xi @ lo.astype(np.float64)) / 254)
        # the per-row rule (l0_query_kernel's coefficients, cta_refine_body's two phases)
        order = np.argsort(approx, kind="stable")
        sa = approx[order]
        top = cand[order[:128]]
        exact = ((grouped[top].astype(np.float64) - q) ** 2).sum(1)
        dq = rq + qabs / 1048576
        Xc = Xrow[top]
        lb = sa[:128] - w * (2 * np.sqrt(n2) * res_up[top] + 2 * dq * Xc + c_sum * Xc * Xc + c_sum * n2 + 2e-30)
        kk = min(a.k, len(sa))
        T1 = exact[:kk].max() if kk == a.k else np.inf
        for kp in (32, 64, 128):
            sel = np.concatenate([np.arange(kk), kk + np.flatnonzero(~(lb[kk:kp] > T1))])
            T = np.sort(exact[sel])[a.k - 1] if len(sel) >= a.k else np.inf
            if kp == 128:
                row_rescored.append(len(sel))
            if len(sa) > kp and not sa[kp - 1] > T + e0:
                row_fails[kp] += 1
        approx.sort()
        for kp in (64, 128):
            top = approx[:kp]
            T = top[min(a.k, kp) - 1] + 2 * e0
            rescored[kp].append(int((top <= T).sum()))
            if len(approx) > kp and not approx[kp - 1] > T:
                fails[kp] += 1
    per_batch = lambda f: f * 2048 / a.queries
    print(json.dumps({
        "tool": "level0_model", "workload": f"bench.py {a.law} law, {a.rows}x{a.dim}, lists={a.lists}, probes={a.probes}, k={a.k}, "
                                             f"{a.queries} queries (CPU draw; {how})",
        "rmax": rmax, "rmax_over_row_norm_max": float((res / np.maximum(xnorm, 1e-30)).max()),
        "row_residual_over_norm_median": float(np.median(res / np.maximum(xnorm, 1e-30))),
        "xmax": xmax, "eps_level0_median": float(np.median(eps0)), "eps_level1_median": float(np.median(eps1)),
        "eps_ratio_median": float(np.median(np.array(eps0) / np.array(eps1))),
        "failures_per_2048_batch": {str(kp): per_batch(fails[kp]) for kp in fails},
        "failure_fraction": {str(kp): fails[kp] / a.queries for kp in fails},
        "rescored_rows_per_query_mean": {str(kp): float(np.mean(rescored[kp])) for kp in rescored},
        "per_row_rule": {
            "rescored_rows_per_query_mean": float(np.mean(row_rescored)),
            "rescored_rows_per_query_p90": float(np.percentile(row_rescored, 90)),
            "failures_per_2048_batch": {str(kp): per_batch(row_fails[kp]) for kp in row_fails},
        },
    }))


if __name__ == "__main__":
    main()
