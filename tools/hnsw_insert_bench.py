"""INSERT into a resident HNSW image on the device (vb_hnsw_insert), at config C's shape by default: a graph built on
the device over N x 768 halfvec cosine rows of config C's law (Gaussian mixture of 1000 components, sigma 0.3,
l2-normalised, rounded to half), m 16, ef_construction 64.  Reports, in one JSON line:
  - rows/s of inserting --insert rows with the default batching;
  - p50 / p99 latency of --single single-row calls (what one aminsert pays);
  - recall@10 at ef_search 100 of the grown graph and of a full build of the same rows, against the exact top 10;
  - the serial on-disk insert rate on one host thread (the oracle's HNSW, tests/hnsw_ondisk_oracle.c), on a --oracle-rows subset of the same shape;
  - the card's name and power limit, read in the same run.
Usage: python tools/hnsw_insert_bench.py [--rows N] [--insert K] [--single S] [--queries Q] [--oracle-rows R]"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def card():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=60)
        return [line.strip() for line in r.stdout.splitlines() if line.strip()] or r.stderr.strip()
    except (OSError, subprocess.SubprocessError) as e:
        return f"nvidia-smi failed: {e}"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=1_000_000)
    ap.add_argument("--insert", type=int, default=100_000)
    ap.add_argument("--single", type=int, default=1000)
    ap.add_argument("--queries", type=int, default=1000)
    ap.add_argument("--dim", type=int, default=768)
    ap.add_argument("--oracle-rows", type=int, default=20000)
    args = ap.parse_args()
    import torch
    import oracle as O
    import pgvector_b200 as pv
    from tests.hnsw_ondisk_oracle import DiskHnsw
    pv.init(0)
    dev = torch.device("cuda", 0)
    n, k_ins, dim = args.rows, args.insert, args.dim
    total = n + k_ins + args.single
    g = torch.Generator(device=dev).manual_seed(3)
    centres = torch.nn.functional.normalize(torch.randn((1000, dim), generator=g, device=dev), dim=1)

    def law(m):
        which = torch.randint(0, 1000, (m,), generator=g, device=dev)
        x = centres[which] + 0.3 * torch.randn((m, dim), generator=g, device=dev) / dim ** 0.5
        return torch.nn.functional.normalize(x, dim=1).half().contiguous()

    rows = torch.cat([law(min(65536, total - i)) for i in range(0, total, 65536)])
    q = law(args.queries)
    out = {"bench": "hnsw-insert", "card": card(),
           "workload": f"HNSW halfvec_cosine_ops, {n} x {dim} built on the device, m=16, ef_construction=64; insert {k_ins} rows "
                       f"(default batches), then {args.single} single-row calls; config C's law"}
    gi = pv.HnswIndex("halfvec_cosine_ops", dim, m=16)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    gi.build(rows[:n])
    pv.synchronize()
    out["build_s"] = time.perf_counter() - t0
    gi.insert(rows[n:n + 64], seed=0)    # warm-up: modules, workspaces, visited tables
    t0 = time.perf_counter()
    _, recs = gi.insert(rows[n + 64:n + k_ins], seed=1)
    pv.synchronize()
    dt = time.perf_counter() - t0
    out["insert_rows_per_s"] = (k_ins - 64) / dt
    out["insert_s"] = dt
    out["change_records_per_row"] = len(recs) / (k_ins - 64)
    lat = []
    for i in range(args.single):
        r = rows[n + k_ins + i:n + k_ins + i + 1]
        t0 = time.perf_counter()
        gi.insert(r, seed=10 + i)
        lat.append(time.perf_counter() - t0)
    lat = np.array(lat) * 1e3
    out["single_row_ms"] = {"p50": float(np.percentile(lat, 50)), "p99": float(np.percentile(lat, 99)), "calls": args.single}
    # recall@10 at ef_search 100 against the exact top 10 (the device's exact top-k over the same rows)
    table = pv.Table(pv.HALFVEC, dim)
    table.append(rows)
    qh = q.view(torch.int16).cpu().numpy().view(np.uint16)
    truth, _ = table.exact_topk(pv.NEG_IP, qh, 10)
    ids, _, _ = gi.search(qh, k=10, ef_search=100)
    full = pv.HnswIndex("halfvec_cosine_ops", dim, m=16).build(rows)
    fids, _, _ = full.search(qh, k=10, ef_search=100)

    def rec(a):
        return float(np.mean([len(set(a[i].tolist()) & set(truth[i].tolist())) / 10 for i in range(len(a))]))

    out["recall_at_10_ef100"] = {"grown": rec(ids), "full_build": rec(fids)}
    # the oracle's serial on-disk insert on the host cores, same shape, on a subset
    r_host = rows[:args.oracle_rows].view(torch.int16).cpu().numpy().view(np.uint16)
    half = args.oracle_rows // 2
    og = DiskHnsw(O.HALFVEC, O.NEG_IP, r_host[:half], m=16, ef_construction=64, dim=dim)
    t0 = time.perf_counter()
    og.insert_on_disk(r_host[half:])
    out["oracle_serial_insert_rows_per_s"] = (args.oracle_rows - half) / (time.perf_counter() - t0)
    out["oracle_note"] = f"one host thread, {half} rows inserted into a {half}-element oracle graph"
    print(json.dumps(out))


if __name__ == "__main__":
    main()
