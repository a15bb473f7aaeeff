"""Filtered LIMIT queries on a resident IVFFlat image at config B's shape: bench.py's law (rank16), 1M x 1536 rows,
1000 lists, probes 10, batches of 2048 queries, k = 10, built through bench.py's functions.  For filter selectivities of
50 %, 10 %, 2 % and 1 %, with one filter for the batch and with 64 per-query filters, it times three routes, with CUDA
events around synchronised calls (median of the timed calls, after warm-up):
  - vb_ivf_search_filtered_dev (the batched list scan with its runs masked);
  - the filtered iterative scan handle's first page (vb_ivf_scan_begin_filtered with max_probes = probes, page = k, then
    one next; host queries and outputs, as that API has them);
  - unfiltered vb_ivf_search_dev on the same batch, for reference.
Also reported, in the same JSON line: the card's name and power limit, read in the same run; the mask pass's share of
the filtered step (VB_PROF_FILTER_MASK brackets in a separate profiled pass); whether repeated filtered calls return
identical outputs; and whether the filtered search equals the handle's first page on the batch's first 64 queries.
Usage: python tools/ivf_filter_bench.py [--rows N] [--dim D] [--lists L] [--probes P] [--steps S]"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

PROF_FILTER_MASK = 7


def card():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=60)
        return [line.strip() for line in r.stdout.splitlines() if line.strip()] or r.stderr.strip()
    except (OSError, subprocess.SubprocessError) as e:
        return f"nvidia-smi failed: {e}"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=1_000_000)
    ap.add_argument("--dim", type=int, default=1536)
    ap.add_argument("--lists", type=int, default=1000)
    ap.add_argument("--probes", type=int, default=10)
    ap.add_argument("--batch", type=int, default=2048)
    ap.add_argument("--steps", type=int, default=5)
    args = ap.parse_args()
    import torch
    import bench
    import pgvector_b200 as pv
    from pgvector_b200 import _lib
    pv.init(0)
    L = _lib.load()
    dev = torch.device("cuda", 0)
    bargs = argparse.Namespace(rows=args.rows, dim=args.dim, lists=args.lists, latent_dim=16, components=1000, queries=4 * args.batch)
    rows, queries = bench.make_dataset(bargs, "rank16", dev)
    torch.cuda.synchronize()
    centers, offsets, grouped, order, _ = bench.build_index_arrays(bargs, "rank16", rows, pv)
    del rows
    torch.cuda.empty_cache()
    off = np.asarray(offsets.cpu() if torch.is_tensor(offsets) else offsets, dtype=np.int64)
    ids = (order.to(torch.int64) if torch.is_tensor(order) else torch.from_numpy(np.asarray(order, np.int64)).to(dev)).contiguous()
    ix = pv.IvfflatIndex("vector_l2_ops", args.dim, args.lists).load(centers, off, grouped.contiguous(), ids)
    all_ids = ids.cpu().numpy()
    k, B, P = 10, args.batch, args.probes
    qb = queries[:B].contiguous()
    qh = qb.cpu().numpy()
    o_ids = torch.empty((B, k), dtype=torch.int64, device=dev)
    o_dist = torch.empty((B, k), dtype=torch.float32, device=dev)
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]

    def timed(fn, steps):
        for _ in range(2):
            fn()
        pv.synchronize()
        ms = []
        for _ in range(steps):
            ev[0].record()
            fn()
            pv.synchronize()
            ev[1].record()
            ev[1].synchronize()
            ms.append(ev[0].elapsed_time(ev[1]))
        return float(np.median(ms))

    def unfiltered():
        ix.search_into(qb, k, P, o_ids, o_dist)

    def filtered_call(farr, nf, fq):
        def run():
            pv._after_torch(qb)
            _lib.check(L.vb_ivf_search_filtered_dev(ix.h, qb.data_ptr(), B, P, k, farr, nf,
                                                    None if fq is None else fq.ctypes.data_as(C.c_void_p), o_ids.data_ptr(), o_dist.data_ptr()))
        return run

    def handle_call(filters, fq):
        def run():
            with ix.iterative_scan(qh, probes=P, max_probes=P, page=k, filter=filters, filter_of_query=fq) as s:
                return s.next_batch()
        return run

    out = {"bench": "ivf_filter", "card": card(),
           "workload": f"IVFFlat vector_l2_ops {args.rows}x{args.dim}, lists={args.lists}, probes={P}, {B} queries per batch, k={k}",
           "timing": f"CUDA events around synchronised calls, median of {args.steps} after 2 warm-up calls"}
    t_unf = timed(unfiltered, args.steps)
    out["unfiltered_search"] = {"ms": t_unf, "queries_per_s": B / (t_unf / 1e3)}
    rng = np.random.default_rng(7)
    results = []
    for sel in (0.5, 0.1, 0.02, 0.01):
        for nf in (1, 64):
            allowed = [np.sort(rng.choice(all_ids, int(len(all_ids) * sel), replace=False)) for _ in range(nf)]
            filters = [ix.filter(a) for a in allowed]
            farr = (C.c_void_p * nf)(*[f.h.value for f in filters])
            fq = None if nf == 1 else rng.integers(0, nf, B).astype(np.int32)
            run = filtered_call(farr, nf, fq)
            t_f = timed(run, args.steps)
            run()
            pv.synchronize()
            first = (o_ids.cpu().numpy().copy(), o_dist.cpu().numpy().copy())
            same = True
            for _ in range(3):
                run()
                pv.synchronize()
                same = same and np.array_equal(o_ids.cpu().numpy(), first[0]) and np.array_equal(o_dist.cpu().numpy(), first[1])
            # the mask pass's share, from its event brackets in a profiled pass of its own
            pv.prof_enable(True)
            pv.prof_read(PROF_FILTER_MASK)
            ev[0].record()
            for _ in range(args.steps):
                run()
            pv.synchronize()
            ev[1].record()
            ev[1].synchronize()
            step_ms = ev[0].elapsed_time(ev[1]) / args.steps
            mask_ms, mask_n = pv.prof_read(PROF_FILTER_MASK)
            pv.prof_enable(False)
            t_h = timed(handle_call(filters if nf > 1 else filters[0], fq), max(1, args.steps // 2))
            hi, hd, _ = handle_call(filters if nf > 1 else filters[0], fq)()
            agree = float((first[0][:64] == hi[:64]).mean())
            results.append({"selectivity": sel, "filters": nf,
                            "filtered_search": {"ms": t_f, "queries_per_s": B / (t_f / 1e3)},
                            "handle_first_page": {"ms": t_h, "queries_per_s": B / (t_h / 1e3)},
                            "mask_share_of_step": (mask_ms / args.steps) / step_ms if step_ms > 0 else None,
                            "mask_ms_per_step": mask_ms / args.steps, "mask_launches": mask_n,
                            "identical_across_runs": bool(same), "id_agreement_with_handle_first_64": agree})
            for f in filters:
                f.free()
    out["filtered"] = results
    ix.free()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
