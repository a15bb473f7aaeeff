"""CREATE INDEX ... USING ivfflat in one call (vb_ivf_build_dev / vb_ivf_build) at config B's index: 1M x 1536 fp32 rows of
bench.py's mixture law (1000 Gaussians), lists = 1000, 50 000 samples -- beside the hand-written route bench.py takes
(vb_kmeans_pp_init + vb_kmeans + vb_assign, torch argsort / bincount / cumsum, a gather in slabs of 65 536 rows,
vb_ivf_load_dev), in one process, alternating, after a warm-up build of each.  All three routes get the same sample rows
and seed, so they must build the same image.  Prints one JSON line:
  - the card's name and power limit, read in the same run;
  - per route: seconds per build (host clock around the synchronised call; median, min, max) and rows/s;
  - per one-call route the seconds per phase from CUDA events on the library stream (sample, seeding, Lloyd, assign,
    destinations, placement), the placement kernel's bytes (2 x indexed rows x stride, from the shapes) over its event
    time as a share of the data-sheet 3.35 TB/s, and the host route's host-to-device bytes;
  - the hand-written route's phases by host clock;
  - recall@10 at probes = 10 of the built index against the exact scan, and whether the routes' search results (ids and
    distances of 2048 queries) are identical;
  - the same one-call builds of 1M x 768 halfvec and 4M x bit(1024) rows at fewer repetitions (1536- and 128-byte rows).
It needs a GPU.  Usage: python tools/ivf_build_bench.py [--rows N] [--reps R] [--skip-extra]"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

HBM = 3.35e12   # H100 SXM data-sheet bandwidth, bytes/s


def card():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=60)
        return [line.strip() for line in r.stdout.splitlines() if line.strip()] or r.stderr.strip()
    except (OSError, subprocess.SubprocessError) as e:
        return f"nvidia-smi failed: {e}"


def stats(xs):
    return {"median_s": float(np.median(xs)), "min_s": float(min(xs)), "max_s": float(max(xs)), "builds": len(xs)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=1_000_000)
    ap.add_argument("--dim", type=int, default=1536)
    ap.add_argument("--lists", type=int, default=1000)
    ap.add_argument("--samples", type=int, default=50_000)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--skip-extra", action="store_true")
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("ivf_build_bench.py measures on a GPU; none is visible")
    import bench
    import pgvector_b200 as pv
    pv.init(0)
    pv.prof_enable(True)
    dev = torch.device("cuda", 0)
    PHASES = {"sample": pv.PROF_BUILD_SAMPLE, "seeding": pv.PROF_BUILD_SEED, "lloyd": pv.PROF_BUILD_LLOYD, "assign": pv.PROF_BUILD_ASSIGN,
              "destinations": pv.PROF_BUILD_DEST, "placement": pv.PROF_BUILD_PLACE}

    def sync():
        torch.cuda.synchronize()
        pv.synchronize()

    def read_phases():
        pv.prof_read(pv.PROF_ASSIGN)   # (the assign step of the Lloyd iterations and vb_assign: inside other phases)
        return {name: pv.prof_read(slot)[0] / 1e3 for name, slot in PHASES.items()}

    def one_call(opclass, dim, lists, rows, ids, sample_rows, reps, raw, hand=None):
        """alternating builds -- the hand-written route (if given), device rows, pinned host rows -- after one warm-up
        build of each: times, phases, and the last index of each route"""
        n, out, keep = rows.shape[0], {}, {}
        host_rows = rows.cpu().pin_memory()
        host_view = host_rows.numpy() if host_rows.dtype != torch.float16 else host_rows.view(torch.int16).numpy().view(np.uint16)
        runs = {"build_dev": (rows, ids), "build_host_pinned": (host_view, ids.cpu().numpy())}
        times = {r: [] for r in list(runs) + ["hand_written"]}
        phases = {r: [] for r in times}
        iters = 0
        for rep in range(reps + 1):
            if hand is not None:
                if "hand_written" in keep:
                    keep.pop("hand_written").free()
                sync()
                keep["hand_written"], dt, ph = hand()
                if rep:
                    times["hand_written"].append(dt)
                    phases["hand_written"].append(ph)
            for route, (r, i) in runs.items():
                if route in keep:
                    keep.pop(route).free()
                ix = pv.IvfflatIndex(opclass, dim, lists)
                read_phases()
                sync()
                t = time.perf_counter()
                _, _, iters = ix.build(r, i, seed=42, sample_rows=sample_rows)
                sync()
                dt = time.perf_counter() - t
                ph = read_phases()
                if rep:
                    times[route].append(dt)
                    phases[route].append(ph)
                keep[route] = ix
        stride = (raw + 15) // 16 * 16
        for route in runs:
            med = {p: float(np.median([ph[p] for ph in phases[route]])) for p in PHASES}
            placed = 2 * len(keep[route]) * stride
            out[route] = dict(stats(times[route]), rows_per_s=n / float(np.median(times[route])), phases_s=med, lloyd_iterations=iters,
                              placement_bytes=placed, placement_share_of_3_35_TBps=placed / med["placement"] / HBM)
        out["build_host_pinned"]["h2d_bytes"] = 2 * n * raw + sample_rows.shape[0] * raw + 8 * n
        if hand is not None:
            ht = times["hand_written"]
            out["hand_written"] = dict(stats(ht), rows_per_s=n / float(np.median(ht)),
                                       phases_s={p: float(np.median([h[p] for h in phases["hand_written"]])) for p in phases["hand_written"][0]})
        return out, keep

    # ---------------------------------------------------------------- config B's index: vector_l2_ops
    bargs = argparse.Namespace(rows=args.rows, dim=args.dim, lists=args.lists, latent_dim=16, components=1000, queries=4096)
    rows, queries = bench.make_dataset(bargs, "mixture", dev)
    n, L = args.rows, args.lists
    ids = torch.arange(n, device=dev, dtype=torch.int64)
    g = torch.Generator(device=dev).manual_seed(42)
    sample_rows_dev = torch.randperm(n, generator=g, device=dev)[:min(n, args.samples)]
    sample_rows = sample_rows_dev.cpu().numpy()
    torch.cuda.synchronize()

    def hand_written():
        ph, t0 = {}, time.perf_counter()

        def lap(name, t):
            sync()
            ph[name] = time.perf_counter() - t
            return time.perf_counter()

        t = t0
        samp = rows[sample_rows_dev]
        tab = pv.Table(pv.VECTOR, args.dim).append(samp)
        t = lap("sample", t)
        init = pv.kmeans_pp_init(tab, pv.L2, L, seed=42)
        t = lap("seeding", t)
        c_host, iters = pv.kmeans(tab, pv.L2, init, max_iter=500)
        tab.free()
        t = lap("lloyd", t)
        centers = torch.from_numpy(c_host).to(dev)
        tr = pv.Table(pv.VECTOR, args.dim).append(rows)
        assign = pv.assign(tr, pv.L2_SQUARED, centers).to(torch.int64)
        pv.synchronize()
        tr.free()
        t = lap("assign (with the copy of the rows into a table)", t)
        order = torch.argsort(assign, stable=True)
        counts = torch.bincount(assign, minlength=L)
        offsets = torch.zeros(L + 1, dtype=torch.int64)
        offsets[1:] = torch.cumsum(counts.cpu(), 0)
        t = lap("argsort + bincount + cumsum", t)
        grouped = torch.empty_like(rows)
        for lo in range(0, n, 65536):
            grouped[lo:lo + 65536] = rows[order[lo:lo + 65536]]
        t = lap("slab gather", t)
        ix = pv.IvfflatIndex("vector_l2_ops", args.dim, L).load(centers, offsets.numpy(), grouped, order.contiguous())
        pv.synchronize()
        lap("vb_ivf_load_dev", t)
        del grouped
        return ix, time.perf_counter() - t0, ph

    result = {"card": card(), "config": f"{n} x {args.dim} fp32, mixture of 1000 Gaussians, lists = {L}, {sample_rows.shape[0]} samples "
                                        f"(torch.randperm, seed 42, shared by the routes), seed 42, {args.reps} timed builds per route after one warm-up"}
    out, keep = one_call("vector_l2_ops", args.dim, L, rows, ids, sample_rows, args.reps, args.dim * 4, hand=hand_written)
    result.update(out)
    routes = ("build_dev", "build_host_pinned")

    # the same image from the three routes, and its recall
    q = queries[:2048].contiguous()
    got = {name: ix.search(q, 10, probes=10) for name, ix in keep.items()}
    torch.cuda.synchronize()
    result["identical_search_results"] = bool(all(torch.equal(got[r][0], got["hand_written"][0]) and torch.equal(got[r][1], got["hand_written"][1])
                                                   for r in routes))
    exact = pv.Table(pv.VECTOR, args.dim).append(rows)
    ti, _ = exact.exact_topk(pv.L2_SQUARED, q[:1000].contiguous(), 10)
    gi = got["build_dev"][0][:1000]
    result["recall_at_10_probes_10"] = float(np.mean([len(set(a.tolist()) & set(b.tolist())) / 10 for a, b in zip(gi.cpu().numpy(), ti.cpu().numpy())]))
    exact.free()
    for ix in keep.values():
        ix.free()
    del rows, exact, keep
    torch.cuda.empty_cache()

    # ---------------------------------------------------------------- shorter rows: 1536 and 128 bytes
    if not args.skip_extra:
        reps = max(2, args.reps // 2)
        n_h = args.rows
        hb = argparse.Namespace(rows=n_h, dim=768, lists=L, latent_dim=16, components=1000, queries=16)
        half = bench.make_dataset(hb, "mixture", dev)[0].half()
        sr = torch.randperm(n_h, generator=g, device=dev)[:min(n_h, args.samples)].cpu().numpy()
        out, keep = one_call("halfvec_l2_ops", 768, L, half, torch.arange(n_h, device=dev), sr, reps, 768 * 2)
        result[f"halfvec_{n_h}x768"] = out
        for ix in keep.values():
            ix.free()
        del half
        torch.cuda.empty_cache()
        n_b = 4 * args.rows
        bits = torch.empty((n_b, 128), dtype=torch.uint8, device=dev)
        comp = torch.randn((1000, 1024), generator=g, device=dev)
        w = (2 ** torch.arange(7, -1, -1, device=dev)).to(torch.int32)
        for lo in range(0, n_b, 65536):
            hi = min(n_b, lo + 65536)
            x = comp[torch.randint(0, 1000, (hi - lo,), generator=g, device=dev)] + 0.3 * torch.randn((hi - lo, 1024), generator=g, device=dev)
            bits[lo:hi] = ((x > 0).view(hi - lo, 128, 8).to(torch.int32) * w).sum(-1).to(torch.uint8)
        sr = torch.randperm(n_b, generator=g, device=dev)[:min(n_b, args.samples)].cpu().numpy()
        out, keep = one_call("bit_hamming_ops", 1024, L, bits, torch.arange(n_b, device=dev), sr, reps, 128)
        result[f"bit_{n_b}x1024"] = out
        for ix in keep.values():
            ix.free()
    print(json.dumps(result))


if __name__ == "__main__":
    main()
