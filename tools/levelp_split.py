#!/usr/bin/env python3
"""Where the time of a level-P search step goes, kernel by kernel: bench.py's config-B data and index (its functions and
build recipe; 1M x 1536 fp32, lists 1000, probes 10, k 10, its first 4 batches of 2048 queries), `tc_levelp` on, S steps
under torch.profiler with CUDA activities after W untimed ones.  Prints one JSON line: device microseconds per step and
launches per step of every kernel, largest first, the sum over the level-P list-scan bracket (query projection, grouping,
scan and bounds), the level-P fallbacks per batch, the last batch's candidate count and the card's name and power limit.
The grouping kernels (lt_group_kernel, lt_scatter_kernel) also serve the probe selection and the level-0 re-run: their
figures count every launch.  Profile in a run of its own: the tracing slows the host, so the step time it implies is
not bench.py's.

    python tools/levelp_split.py [--rows N --dim D --lists L --probes P --steps S --warmup W]
"""
from __future__ import annotations

import argparse
import json
import os
import sys
from collections import defaultdict

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

# the kernels of the level-P list-scan bracket (launch_list_proj), before and after the fused scan
LEVELP_SCAN = ("lp_project_kernel", "lt_group_kernel", "lt_scatter_kernel", "lt_count_kernel", "lt_scan_kernel",
               "list_tile_kernel", "lp_bound_kernel", "lp_scan_kernel")


def short(name):
    """a kernel's name without its namespace, template arguments and parameter list"""
    base = name.split("(")[0]
    base = base.split("<")[0]
    return base.split("::")[-1].strip()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=1_000_000)
    ap.add_argument("--dim", type=int, default=1536)
    ap.add_argument("--lists", type=int, default=1000)
    ap.add_argument("--probes", type=int, default=10)
    ap.add_argument("--steps", type=int, default=40)
    ap.add_argument("--warmup", type=int, default=40)
    args = ap.parse_args()

    import torch
    from torch.profiler import ProfilerActivity, profile

    import bench
    import pgvector_b200 as pv
    from bench_extra import card

    pv.init(0)
    dev = torch.device("cuda", 0)
    bargs = argparse.Namespace(rows=args.rows, dim=args.dim, lists=args.lists, latent_dim=16, components=1000, queries=4 * 2048)
    rows, queries = bench.make_dataset(bargs, "rank16", dev)
    torch.cuda.synchronize()
    centers, offsets, grouped, order, how = bench.build_index_arrays(bargs, "rank16", rows, pv)
    del rows
    torch.cuda.empty_cache()
    ix = pv.IvfflatIndex("vector_l2_ops", args.dim, args.lists).load(centers, offsets, grouped, order)
    k, B = 10, 2048
    batches = [queries[i:i + B].contiguous() for i in range(0, queries.shape[0] - B + 1, B)]
    ids = torch.empty((B, k), dtype=torch.int64, device=dev)
    dist = torch.empty((B, k), dtype=torch.float32, device=dev)
    pv.set_option("scan_impl", 2)
    pv.set_option("tc_levelp", 1)
    for i in range(args.warmup):
        ix.search_into(batches[i % len(batches)], k, args.probes, ids, dist)
    pv.synchronize()
    f0 = ix.tc_levelp_fallbacks()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for i in range(args.steps):
            ix.search_into(batches[i % len(batches)], k, args.probes, ids, dist)
        pv.synchronize()
        torch.cuda.synchronize()
    fails = (ix.tc_levelp_fallbacks() - f0) / args.steps
    cands = ix.last_candidates()
    us, n = defaultdict(float), defaultdict(int)
    for e in prof.events():
        if e.device_type == torch.autograd.DeviceType.CUDA and e.device_time_total > 0:
            nm = short(e.name)
            us[nm] += e.device_time_total
            n[nm] += 1
    kernels = sorted(({"kernel": nm, "us_per_step": us[nm] / args.steps, "launches_per_step": n[nm] / args.steps} for nm in us),
                     key=lambda d: -d["us_per_step"])
    bracket = {nm: us[nm] / args.steps for nm in LEVELP_SCAN if nm in us}
    print(json.dumps({"bench": "levelp_split", "card": card(),
                      "workload": f"IVFFlat vector_l2_ops {args.rows}x{args.dim}, lists={args.lists}, probes={args.probes}, k={k}, "
                                  f"{len(batches)} batches of {B} queries, bench.py's rank16 law and index ({how}), tc_levelp 1, "
                                  f"{args.steps} profiled steps after {args.warmup}",
                      "levelp_scan_us_per_step": sum(bracket.values()), "levelp_scan_split_us": bracket,
                      "levelp_fallback_queries_per_batch": fails, "last_candidates": cands, "kernels": kernels}))


if __name__ == "__main__":
    main()
