"""avg / sum over a resident table on the device (vb_table_aggregate_dev), at the shapes of the reference's centroid
queries: 1M x 1536 fp32 rows (6.1 GB) and 2M x 768 halfvec rows, "SELECT avg(v) FROM t" and "... GROUP BY g" with 1000
uniform groups, at run_rows 0 (the serial plan) and the default.  For each case it reports, in one JSON line:
  - ms per call, event-timed on the library stream after warm-up (median of --reps);
  - the bytes read (rows + group ids + the sorted row list) per second, and that as a fraction of the data-sheet 3.35 TB/s;
and once:
  - the oracle's serial plan (tests/aggregate_oracle.c) on one host thread over an --oracle-rows sample of each shape,
    in rows/s, as the baseline;
  - the card's name and power limit, read in the same run.
Usage: python tools/aggregate_bench.py [--reps K] [--oracle-rows R]"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

HBM = 3.35e12


def card():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=60)
        return [line.strip() for line in r.stdout.splitlines() if line.strip()] or r.stderr.strip()
    except (OSError, subprocess.SubprocessError) as e:
        return f"nvidia-smi failed: {e}"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--oracle-rows", type=int, default=20000)
    args = ap.parse_args()
    import torch
    import pgvector_b200 as pv
    from tests import aggregate_oracle as A
    pv.init(0)
    dev = torch.device("cuda", 0)
    stream = torch.cuda.ExternalStream(pv.stream_handle())
    out = {"bench": "aggregate", "card": card(), "default_run_rows": pv.DEFAULT_RUN_ROWS, "hbm_peak_tb_s": HBM / 1e12}
    g = torch.Generator(device=dev).manual_seed(11)
    for name, elem, n, dim in (("vector_1M_x_1536", pv.VECTOR, 1_000_000, 1536), ("halfvec_2M_x_768", pv.HALFVEC, 2_000_000, 768)):
        dt = torch.float32 if elem == pv.VECTOR else torch.float16
        t = pv.Table(elem, dim)
        for i in range(0, n, 131072):
            t.append(torch.randn((min(131072, n - i), dim), generator=g, device=dev).to(dt).contiguous())
        pv.synchronize()
        esize = 4 if elem == pv.VECTOR else 2
        groups = torch.randint(0, 1000, (n,), generator=g, device=dev, dtype=torch.int32)
        res = {}
        for gname, gr, ng in (("no_groups", None, 1), ("1000_groups", groups, 1000)):
            for R in (0, pv.DEFAULT_RUN_ROWS):
                for aname, fn in (("avg", t.avg), ("sum", t.sum)):
                    if gr is None:   # without groups the Python method takes the host variant: time the _dev call directly
                        vals = torch.empty((1, dim), dtype=dt, device=dev)
                        cnt = torch.empty(1, dtype=torch.int64, device=dev)
                        agg = pv.AGG_AVG if aname == "avg" else pv.AGG_SUM

                        def call():
                            pv._lib.check(pv.load().vb_table_aggregate_dev(t.h, agg, None, 1, R, pv._ptr(vals), pv._ptr(cnt), None))
                    else:
                        def call():
                            fn(gr, 1000, run_rows=R)
                    reps = 1 if R == 0 else args.reps
                    call()
                    pv.synchronize()
                    ms = []
                    for _ in range(reps):
                        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                        e0.record(stream)
                        call()
                        e1.record(stream)
                        e1.synchronize()
                        ms.append(e0.elapsed_time(e1))
                    m = float(np.median(ms))
                    nbytes = n * dim * esize + (0 if gr is None else n * 4 * 2)
                    res[f"{aname}_{gname}_R{R}"] = {"ms": m, "bytes_read": nbytes, "tb_s": nbytes / m / 1e9,
                                                    "fraction_of_3_35_tb_s": nbytes / m / 1e9 / (HBM / 1e12), "reps": reps}
        # the oracle's serial plan on one host thread, on a sample of the same shape
        k = args.oracle_rows
        sample = torch.randn((k, dim), generator=g, device=dev).to(dt).cpu().numpy()
        t0 = time.perf_counter()
        A.table_aggregate(elem == pv.HALFVEC, A.AVG, sample, dim, run_rows=0)
        res["oracle_serial_avg_rows_per_s"] = k / (time.perf_counter() - t0)
        res["oracle_sample_rows"] = k
        out[name] = res
        del t
        torch.cuda.empty_cache()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
