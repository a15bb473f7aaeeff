"""VACUUM of a resident HNSW image on the device (vb_hnsw_vacuum), at config C's shape by default: a graph built on the
device over N x 768 halfvec cosine rows of config C's law (Gaussian mixture of 1000 components, sigma 0.3,
l2-normalised, rounded to half), m 16, ef_construction 64.  For each deleted fraction (a random 1 % and 10 % of the
elements, each on a fresh build) it reports, in one JSON line:
  - the vacuum's time, the elements it repaired and repairs/s (default batching);
  - recall@10 at ef_search 100 over the live rows, after the vacuum and for a vb_hnsw_build of the surviving rows (what a
    repack costs today), and that rebuild's time;
and once:
  - the serial vacuum rate on one host thread (the oracle's HNSW, tests/hnsw_vacuum_oracle.c), on an --oracle-rows
    subset of the same shape with 10 % deleted;
  - the card's name and power limit, read in the same run.
Usage: python tools/hnsw_vacuum_bench.py [--rows N] [--queries Q] [--oracle-rows R]"""
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
    ap.add_argument("--queries", type=int, default=1000)
    ap.add_argument("--dim", type=int, default=768)
    ap.add_argument("--fractions", type=float, nargs="+", default=[0.01, 0.10])
    ap.add_argument("--oracle-rows", type=int, default=10000)
    args = ap.parse_args()
    import torch
    import oracle as O
    import pgvector_b200 as pv
    from tests.hnsw_vacuum_oracle import VacuumHnsw
    pv.init(0)
    dev = torch.device("cuda", 0)
    n, dim = args.rows, args.dim
    g = torch.Generator(device=dev).manual_seed(3)
    centres = torch.nn.functional.normalize(torch.randn((1000, dim), generator=g, device=dev), dim=1)

    def law(m):
        which = torch.randint(0, 1000, (m,), generator=g, device=dev)
        x = centres[which] + 0.3 * torch.randn((m, dim), generator=g, device=dev) / dim ** 0.5
        return torch.nn.functional.normalize(x, dim=1).half().contiguous()

    rows = torch.cat([law(min(65536, n - i)) for i in range(0, n, 65536)])
    qh = law(args.queries).view(torch.int16).cpu().numpy().view(np.uint16)
    out = {"bench": "hnsw-vacuum", "card": card(),
           "workload": f"HNSW halfvec_cosine_ops, {n} x {dim} built on the device, m=16, ef_construction=64; a random "
                       f"{', '.join(f'{f:.0%}' for f in args.fractions)} of the elements deleted, default batches; config C's law"}
    rng = np.random.default_rng(7)
    for frac in args.fractions:
        gi = pv.HnswIndex("halfvec_cosine_ops", dim, m=16)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        gi.build(rows)
        pv.synchronize()
        build_s = time.perf_counter() - t0
        counts = np.ones(n, np.int32)
        counts[rng.choice(n, int(n * frac), replace=False)] = 0
        t0 = time.perf_counter()
        recs, nrep = gi.vacuum(counts)
        pv.synchronize()
        vac_s = time.perf_counter() - t0
        live = np.nonzero(counts)[0]
        live_t = torch.from_numpy(live).to(dev)
        table = pv.Table(pv.HALFVEC, dim)
        table.append(rows[live_t])
        truth, _ = table.exact_topk(pv.NEG_IP, qh, 10)
        truth = live[truth]
        ids, _, _ = gi.search(qh, k=10, ef_search=100)
        t0 = time.perf_counter()
        rb = pv.HnswIndex("halfvec_cosine_ops", dim, m=16).build(rows[live_t].contiguous())
        pv.synchronize()
        rebuild_s = time.perf_counter() - t0
        rids, _, _ = rb.search(qh, k=10, ef_search=100)
        rids = np.where(rids >= 0, live[np.maximum(rids, 0)], -1)

        def rec(a):
            return float(np.mean([len(set(a[i].tolist()) & set(truth[i].tolist())) / 10 for i in range(len(a))]))

        assert np.all(counts[ids[ids >= 0]] > 0)
        out[f"deleted_{frac:g}"] = {"vacuum_s": vac_s, "repaired": nrep, "repairs_per_s": nrep / vac_s, "change_records": len(recs),
                                    "recall_at_10_ef100": {"vacuumed": rec(ids), "rebuilt": rec(rids)}, "rebuild_s": rebuild_s,
                                    "build_s": build_s}
        del gi, rb, table
    # the oracle's serial vacuum on one host thread, same shape, on a subset
    r_host = rows[:args.oracle_rows].view(torch.int16).cpu().numpy().view(np.uint16)
    og = VacuumHnsw(O.HALFVEC, O.NEG_IP, r_host, m=16, ef_construction=64, dim=dim)
    counts = np.ones(args.oracle_rows, np.int32)
    counts[rng.choice(args.oracle_rows, args.oracle_rows // 10, replace=False)] = 0
    t0 = time.perf_counter()
    _, onrep = og.vacuum(counts)
    dt = time.perf_counter() - t0
    out["oracle_serial_vacuum"] = {"repairs_per_s": onrep / dt, "repaired": onrep,
                                   "note": f"one host thread, 10 % of a {args.oracle_rows}-element oracle graph deleted"}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
