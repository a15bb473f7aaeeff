#!/usr/bin/env python3
"""Secondary measurements (one JSON line each) for the rows of SURVEY section 8 that bench.py's headline
does not cover: k-means assign on the tensor cores (config D shape, one GPU's share), HNSW search
(configs C / E at reduced row counts: the graph is built by the CPU oracle, which bounds n), exact scan.

    python tools/bench_extra.py assign   [--rows N --dim D --k K]
    python tools/bench_extra.py hnsw     [--elem halfvec|bit --rows N --dim D --ef EF]
    python tools/bench_extra.py exact    [--rows N --dim D]
    python tools/bench_extra.py rerank   [--rows N --dim D]     (bit HNSW candidates re-ranked on the fp32 rows)
    python tools/bench_extra.py ivf-iter [--rows N --dim D --lists L --probes P --max-probes M --page K --queries Q]
                                          (ivfflat.iterative_scan for filtered LIMIT 10 queries vs the per-scan loop)
    python tools/bench_extra.py filter   [--rows N --dim D --lists L --probes P --max-probes M --page K --queries Q]
                                          (row filters on the device: filtered iterative scan and exact top-k vs host filtering)
    python tools/bench_extra.py level0   [--rows N --dim D --lists L --probes P --rounds R --law rank16|mixture --load S]
    python tools/bench_extra.py levelp   [the same]
                                          (the batched list scan with filter level 0 (int8 rows) on and off, alternating)
    python tools/bench_extra.py hnsw-filter [--rows N --dim D --ef EF --queries Q]
                                          (element filters on the device for hnsw.iterative_scan vs host filtering)

All timing with CUDA events on the library stream; inputs resident in HBM.
"""
from __future__ import annotations

import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def peaks():
    p = os.path.join(ROOT, "MEASURED_PEAKS.json")
    if os.path.exists(p):
        d = json.load(open(p))
        return d["hbm_gbs"], d["bf16_tflops"], d.get("bf16_tflops_sustained", d["bf16_tflops"]), "measured"
    return 3350.0, 989.0, 989.0, "fallback (H100 SXM data sheet: HBM3, dense BF16)"


def timed(pv, torch, stream, fn, warmup=2, steps=5):
    for _ in range(warmup):
        fn()
    pv.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(stream)
    for _ in range(steps):
        fn()
    e1.record(stream)
    pv.synchronize()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / steps


def bench_assign(args):
    import torch
    import pgvector_b200 as pv
    pv.init(0)
    dev = torch.device("cuda", 0)
    stream = torch.cuda.ExternalStream(pv.stream_handle(), device=dev)
    g = torch.Generator(device=dev).manual_seed(5)
    comp = torch.randn((args.k, args.dim), generator=g, device=dev)
    which = torch.randint(0, args.k, (args.rows,), generator=g, device=dev)
    rows = comp[which] + 0.3 * torch.randn((args.rows, args.dim), generator=g, device=dev)
    centers = (comp + 0.05 * torch.randn((args.k, args.dim), generator=g, device=dev)).contiguous()
    torch.cuda.synchronize()
    t = pv.Table(pv.VECTOR, args.dim).append(rows)
    out = torch.empty(args.rows, dtype=torch.int32, device=dev)
    res = {}
    for name, tc in (("wgmma_split_bf16", True), ("exact_fp32_cuda_cores", False)):
        pv.set_tensor_cores(tc)
        n_eff = args.rows if tc else min(args.rows, 131072)
        tt = t if tc else pv.Table(pv.VECTOR, args.dim).append(rows[:n_eff].contiguous())
        o = out[:n_eff]
        ms = timed(pv, torch, stream, lambda: pv._lib.check(pv.load().vb_assign_dev(tt.h, pv.L2_SQUARED, pv._ptr(centers), args.k, pv._ptr(o))),
                   warmup=1, steps=3)
        flops = 2.0 * n_eff * args.k * args.dim
        pv.prof_enable(True)
        pv.prof_read(pv.PROF_ASSIGN)
        pv._lib.check(pv.load().vb_assign_dev(tt.h, pv.L2_SQUARED, pv._ptr(centers), args.k, pv._ptr(o)))
        dev_ms, _ = pv.prof_read(pv.PROF_ASSIGN)     # pack + GEMM + re-check on the device, without host-side allocation
        pv.prof_enable(False)
        res[name] = {"ms": ms, "device_ms": dev_ms, "rows": n_eff, "useful_tflops": flops / ms / 1e9,
                     "useful_tflops_device": flops / dev_ms / 1e9, "rechecked_rows": pv.last_assign_rechecked()}
        if tc:
            a_tc = out.clone()
    pv.set_tensor_cores(True)
    # agreement between the two paths on the exact sample
    pv.set_tensor_cores(False)
    n_eff = res["exact_fp32_cuda_cores"]["rows"]
    ex = torch.empty(n_eff, dtype=torch.int32, device=dev)
    tt = pv.Table(pv.VECTOR, args.dim).append(rows[:n_eff].contiguous())
    pv._lib.check(pv.load().vb_assign_dev(tt.h, pv.L2_SQUARED, pv._ptr(centers), args.k, pv._ptr(ex)))
    pv.set_tensor_cores(True)
    agree = float((ex == a_tc[:n_eff]).float().mean().item())
    hbm, bf16_burst, bf16_sus, src = peaks()
    tc_ms = res["wgmma_split_bf16"]["ms"]
    issued = 3 * 2.0 * args.rows * args.k * args.dim / tc_ms / 1e9      # three bf16 MMAs per fp32-accurate product
    print(json.dumps({"bench": "assign", "workload": f"assign {args.rows}x{args.dim} fp32 rows to {args.k} centres (L2)", "results": res,
                      "tc_vs_exact_agreement": agree,
                      "roofline": {"bound": "tensor", "achieved": issued, "peak": bf16_sus, "unit": "TFLOP/s", "frac": issued / bf16_sus,
                                   "peak_source": src + " bf16_tflops_sustained", "note": "issued bf16 MMA flops (3 per useful fp32-accurate MAC pair)"}}))


def bench_hnsw(args):
    import torch
    import oracle as O
    import pgvector_b200 as pv
    from tests.util import f32_to_half_bits, mixture
    pv.init(0)
    dev = torch.device("cuda", 0)
    stream = torch.cuda.ExternalStream(pv.stream_handle(), device=dev)
    # low intrinsic dimension (like bench.py): a graph index on it has a meaningful recall
    rng = np.random.default_rng(6)
    frame = np.linalg.qr(rng.standard_normal((args.dim, 16)))[0].astype(np.float32)
    x = (rng.standard_normal((args.rows, 16)).astype(np.float32) @ frame.T + 0.02 * rng.standard_normal((args.rows, args.dim)).astype(np.float32))
    q = (rng.standard_normal((args.queries, 16)).astype(np.float32) @ frame.T + 0.02 * rng.standard_normal((args.queries, args.dim)).astype(np.float32))
    if args.elem == "halfvec":
        elem, opclass, metric = O.HALFVEC, "halfvec_cosine_ops", O.NEG_IP
        rows = O.l2_normalize(O.HALFVEC, f32_to_half_bits(x))
        queries = O.l2_normalize(O.HALFVEC, f32_to_half_bits(q))
        rb = args.dim * 2
    else:
        elem, opclass, metric = O.BIT, "bit_hamming_ops", O.HAMMING
        rows, queries = O.binary_quantize(O.VECTOR, x), O.binary_quantize(O.VECTOR, q)
        rb = (args.dim + 7) // 8
    t0 = time.perf_counter()
    og = O.Hnsw(elem, metric, rows, m=16, ef_construction=64, seed=1, dim=args.dim)
    build_s = time.perf_counter() - t0
    g = og.export()
    gi = pv.HnswIndex(opclass, args.dim, m=16).load(rows[g["elem_row"]], g["levels"], g["nbr0"], g["upper_off"], g["upper"], g["entry"])
    qd = torch.from_numpy(queries).to(dev)
    k = 10
    ids = torch.empty((args.queries, k), dtype=torch.int64, device=dev)
    dist = torch.empty((args.queries, k), dtype=torch.float32, device=dev)
    nd = torch.empty(args.queries, dtype=torch.int64, device=dev)
    torch.cuda.synchronize()
    ms = timed(pv, torch, stream, lambda: gi.search_into(qd, k, args.ef, ids, dist, nd), warmup=2, steps=5)
    ndist = float(nd.double().mean().item())
    # parity + recall on a sample
    ns = min(256, args.queries)
    wi, wd, wnd = og.search_batch(queries[:ns], args.ef, k, ties=O.TIES_TOTAL, threads=os.cpu_count() or 1)
    same = float(np.all(ids[:ns].cpu().numpy() == wi, axis=1).mean())
    erows = rows[g["elem_row"]]
    truth = [O.exact_topk(elem, metric, qq, erows, k, dim=args.dim)[0] for qq in queries[:64]]
    rec = sum(len(set(a.tolist()) & set(b.tolist())) for a, b in zip(ids[:64].cpu().numpy(), truth)) / (64 * k)
    t0 = time.perf_counter()
    og.search_batch(queries[:ns], args.ef, k, ties=O.TIES_PG, threads=os.cpu_count() or 1)
    cpu_qps = ns / (time.perf_counter() - t0)
    hbm, _, _, src = peaks()
    qps = args.queries / (ms / 1000.0)
    gbs = qps * (ndist * rb + (ndist / 16.0) * 32 * 4) / 1e9
    print(json.dumps({"bench": "hnsw", "workload": f"HNSW {opclass} {args.rows}x{args.dim}, m=16, ef_search={args.ef}, k={k} "
                                                   f"(graph built by the CPU oracle in {build_s:.0f}s)",
                      "queries_per_s": qps, "ms_per_batch": ms, "batch": args.queries, "distance_evals_per_query": ndist,
                      "recall_at_10": rec, "queries_identical_to_oracle": same,
                      "roofline": {"bound": "hbm", "achieved": gbs, "peak": hbm, "unit": "GB/s", "frac": gbs / hbm, "peak_source": src,
                                   "note": "latency-bound random gathers; bytes = n_dist*row + n_expand*lm*4"},
                      "cpu_baseline": {"value": cpu_qps, "unit": "queries/s", "cores": os.cpu_count(), "kind": "port"}}))


def card():
    """name and power limit of the cards, read in the same run as the numbers they qualify (a read-only query)"""
    import subprocess
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=60)
        return [line.strip() for line in r.stdout.splitlines() if line.strip()] or r.stderr.strip()
    except (OSError, subprocess.SubprocessError) as e:
        return f"nvidia-smi failed: {e}"


def bench_rerank(args):
    """pgvector's quantize-then-rerank on config E's law at a reduced row count: a bit(dim) HNSW over binary_quantize(rows)
    fetches ef_search candidates per query, then the fp32 rows re-rank them under cosine (vb_table_rerank_dev)."""
    import torch
    import pgvector_b200 as pv
    pv.init(0)
    dev = torch.device("cuda", 0)
    stream = torch.cuda.ExternalStream(pv.stream_handle(), device=dev)
    n, dim, nq, ef, k = args.rows, args.dim, args.queries, args.ef, 10
    assert dim % 8 == 0, "--dim must be a multiple of 8"
    # low intrinsic dimension (the law of bench_hnsw), generated on the device in slices
    g = torch.Generator(device=dev).manual_seed(6)
    frame = torch.linalg.qr(torch.randn((dim, 16), generator=g, device=dev))[0]
    weights = torch.tensor([128, 64, 32, 16, 8, 4, 2, 1], dtype=torch.uint8, device=dev)

    def law(m):
        return (torch.randn((m, 16), generator=g, device=dev) @ frame.T + 0.02 * torch.randn((m, dim), generator=g, device=dev)).contiguous()

    def quantize(x):   # binary_quantize: a bit per element, set where it is > 0, MSB first
        return ((x > 0).to(torch.uint8).reshape(x.shape[0], -1, 8) * weights).sum(-1).to(torch.uint8).contiguous()

    table = pv.Table(pv.VECTOR, dim)
    bits = []
    for r0 in range(0, n, 1 << 17):
        x = law(min(1 << 17, n - r0))
        table.append(x)
        bits.append(quantize(x))
        if r0 == 0:
            sample = x[:1000].cpu().numpy()
            assert np.array_equal(bits[0][:1000].cpu().numpy(), pv.binary_quantize(sample)), "device quantization != binary_quantize"
        del x
    bits = torch.cat(bits)
    q = law(nq)
    qbits = quantize(q)
    torch.cuda.synchronize()
    ix = pv.HnswIndex("bit_hamming_ops", dim, m=16)
    t0 = time.perf_counter()
    ix.build(bits, ef_construction=64, seed=42)
    pv.synchronize()
    build_s = time.perf_counter() - t0
    folded = int((ix.export()["dup_of"] >= 0).sum())

    cids = torch.empty((nq, ef), dtype=torch.int64, device=dev)
    cdist = torch.empty((nq, ef), dtype=torch.float32, device=dev)
    rids = torch.empty((nq, k), dtype=torch.int64, device=dev)
    rdist = torch.empty((nq, k), dtype=torch.float32, device=dev)

    def search():
        ix.search_into(qbits, ef, ef, cids, cdist)

    def rerank(qq=q, cand=cids, out_i=rids, out_d=rdist):
        pv._lib.check(pv.load().vb_table_rerank_dev(table.h, pv.COSINE, pv._ptr(qq), qq.shape[0], pv._ptr(cand), cand.shape[1], k,
                                                    pv._ptr(out_i), pv._ptr(out_d)))

    def both():
        search()
        rerank()

    ms_search = timed(pv, torch, stream, search, warmup=2, steps=10)
    ms_both = timed(pv, torch, stream, both, warmup=2, steps=10)
    ms_rerank = timed(pv, torch, stream, rerank, warmup=3, steps=20)   # on the candidates of the last search
    single = {}
    for c in (20, 200):
        c1 = cids[:1, :c].contiguous()
        i1, d1 = rids[:1].clone(), rdist[:1].clone()
        single[f"c{c}"] = timed(pv, torch, stream, lambda: rerank(q[:1], c1, i1, d1), warmup=10, steps=200)

    # recall@10 against fp32 cosine truth (vb_exact_topk)
    truth = torch.empty((nq, k), dtype=torch.int64, device=dev)
    tdist = torch.empty((nq, k), dtype=torch.float32, device=dev)
    pv._lib.check(pv.load().vb_exact_topk_dev(table.h, pv.COSINE, pv._ptr(q), nq, k, pv._ptr(truth), pv._ptr(tdist)))
    pv.synchronize()
    tr, ca, rr = truth.cpu().numpy(), cids.cpu().numpy(), rids.cpu().numpy()

    def recall(got):
        return sum(len(set(a.tolist()) & set(b.tolist())) for a, b in zip(got, tr)) / (nq * k)

    valid = int((cids >= 0).sum().item())
    stride = table.device_rows()[1]
    moved = valid * stride + nq * ef * 8 + nq * dim * 4
    hbm, _, _, src = peaks()
    gbs = moved / (ms_rerank / 1000.0) / 1e9
    print(json.dumps({"bench": "rerank", "workload": f"bit({dim}) HNSW (bit_hamming_ops, m=16, ef_construction=64) over binary_quantize of {n}x{dim} fp32 rows, "
                                                     f"{nq} queries, ef_search={ef}, candidates c={ef}, re-ranked by cosine on the fp32 rows, k={k}",
                      "card": card(), "index_build_s": build_s, "rows_folded_as_duplicates": folded,
                      "ms_per_batch": {"bit_search": ms_search, "rerank": ms_rerank, "search_then_rerank": ms_both},
                      "single_query_rerank_ms": single,
                      "recall_at_10": {"bit_top10": recall(ca[:, :k]), "reranked_top10": recall(rr), "candidate_set": recall(ca)},
                      "roofline": {"bound": "hbm", "kernel": "rerank (prepare + gathered scan + select + finish)", "achieved": gbs, "peak": hbm,
                                   "unit": "GB/s", "frac": gbs / hbm, "bytes_per_batch": moved, "valid_candidates": valid, "peak_source": src,
                                   "note": "bytes = valid candidates x row stride + candidate ids + queries"}}))


def build_ivf_index(args, seed=3):
    """the index of bench_ivf: rows of a low intrinsic dimension generated on the device, k-means on 50 * lists samples,
    rows grouped by list, loaded from device buffers (ids = row numbers)"""
    import torch
    import pgvector_b200 as pv
    pv.init(0)
    dev = torch.device("cuda", 0)
    g = torch.Generator(device=dev).manual_seed(seed)
    frame = torch.linalg.qr(torch.randn((args.dim, 16), generator=g, device=dev))[0]
    x = torch.randn((args.rows, 16), generator=g, device=dev) @ frame.T + 0.02 * torch.randn((args.rows, args.dim), generator=g, device=dev)
    q = torch.randn((args.queries, 16), generator=g, device=dev) @ frame.T + 0.02 * torch.randn((args.queries, args.dim), generator=g, device=dev)
    if args.elem == "vector":
        elem, opclass, kmetric, pmetric, rb = pv.VECTOR, "vector_l2_ops", pv.L2, pv.L2_SQUARED, args.dim * 4
        rows_t, q_t = x.contiguous(), q.contiguous()
        host = lambda t: t.cpu().numpy()
    elif args.elem == "halfvec":
        elem, opclass, kmetric, pmetric, rb = pv.HALFVEC, "halfvec_l2_ops", pv.L2, pv.L2_SQUARED, args.dim * 2
        rows_t, q_t = x.half().contiguous(), q.half().contiguous()
        host = lambda t: t.cpu().numpy().view(np.uint16)
    else:
        elem, opclass, kmetric, pmetric, rb = pv.BIT, "bit_hamming_ops", pv.HAMMING, pv.HAMMING, args.dim // 8
        def pack(t):
            b = (t > 0).to(torch.uint8).reshape(t.shape[0], -1, 8)
            w = torch.tensor([128, 64, 32, 16, 8, 4, 2, 1], dtype=torch.uint8, device=dev)
            return (b * w).sum(-1).to(torch.uint8).contiguous()
        rows_t, q_t = pack(x), pack(q)
        host = lambda t: t.cpu().numpy()
    del x
    torch.cuda.synchronize()
    ns = min(args.rows, 50 * args.lists)
    ts = pv.Table(elem, args.dim).append(host(rows_t[:ns]))
    init = pv.kmeans_pp_init(ts, kmetric, args.lists, seed=42)
    centers, iters = pv.kmeans(ts, kmetric, init, max_iter=100)
    ts.free()
    ta = pv.Table(elem, args.dim).append(rows_t)
    assign = pv.assign(ta, pmetric, centers)
    ta.free()
    a = torch.from_numpy(assign).to(dev).long()
    order = torch.argsort(a, stable=True)
    counts = torch.bincount(a, minlength=args.lists).cpu()
    offsets = np.zeros(args.lists + 1, dtype=np.int64)
    offsets[1:] = np.cumsum(counts.numpy())
    grouped = rows_t[order].contiguous()
    del rows_t
    centers_t = torch.from_numpy(centers).to(dev)
    torch.cuda.synchronize()
    ix = pv.IvfflatIndex(opclass, args.dim, args.lists).load(centers_t, offsets, grouped, order.contiguous())
    return dict(pv=pv, torch=torch, dev=dev, ix=ix, q_t=q_t, host=host, opclass=opclass, rb=rb, counts=counts, offsets=offsets,
                iters=iters, keep=(centers_t, grouped, order))


def bench_ivf(args):
    """IVFFlat scan throughput for halfvec / bit rows (bench.py covers vector)."""
    b = build_ivf_index(args)
    pv, torch, dev, ix, q_t, opclass, rb, counts, iters = b["pv"], b["torch"], b["dev"], b["ix"], b["q_t"], b["opclass"], b["rb"], b["counts"], b["iters"]
    stream = torch.cuda.ExternalStream(pv.stream_handle(), device=dev)
    k, B = 10, args.queries
    ids = torch.empty((B, k), dtype=torch.int64, device=dev)
    dist = torch.empty((B, k), dtype=torch.float32, device=dev)
    pv.prof_enable(True)
    pv.prof_read(pv.PROF_SCAN_ITEMS)
    ms = timed(pv, torch, stream, lambda: ix.search_into(q_t, k, args.probes, ids, dist), warmup=3, steps=10)
    scan_ms, scan_n = pv.prof_read(pv.PROF_SCAN_ITEMS)
    pv.prof_enable(False)
    cand = ix.last_candidates()
    hbm, _, _, src = peaks()
    gbs = cand * rb / (scan_ms / scan_n / 1000.0) / 1e9
    print(json.dumps({"bench": "ivf", "workload": f"IVFFlat {opclass} {args.rows}x{args.dim}, lists={args.lists}, probes={args.probes}, k={k}, {B} queries per batch "
                                                  f"(k-means {iters} it; list sizes {int(counts.min())}/{int(counts.float().mean())}/{int(counts.max())})",
                      "queries_per_s": B / (ms / 1000.0), "ms_per_batch": ms, "candidates_per_query": cand / B,
                      "roofline": {"bound": "hbm", "kernel": "list scan", "achieved": gbs, "peak": hbm, "unit": "GB/s", "frac": gbs / hbm,
                                   "bytes_per_launch": cand * rb, "avg_launch_ms": scan_ms / scan_n, "share_of_step": scan_ms / scan_n / ms, "peak_source": src}}))


def bench_level0(args, level="0"):
    """config B (IVFFlat L2, 2048-query batches, k 10) on bench.py's own data and index -- its law, its queries (the first
    four batches of 2048) and its index recipe, through its functions -- with "tc_level0" (level "p": "tc_levelp") 1 and 0
    in alternating rounds in one process: step time, list scan time (the filter pass with its grouping), list_tc_kernel
    time and bytes, refine time and rows it re-scored per query, the level's fallbacks per batch, and whether the two arms
    return identical ids and distances for every batch."""
    import argparse as ap_
    import torch
    import bench
    import pgvector_b200 as pv
    pv.init(0)
    dev = torch.device("cuda", 0)
    bargs = ap_.Namespace(rows=args.rows, dim=args.dim, lists=args.lists, latent_dim=16, components=1000, queries=10_000)
    rows, queries = bench.make_dataset(bargs, args.law, dev)
    torch.cuda.synchronize()
    centers, offsets, grouped, order, how = bench.build_index_arrays(bargs, args.law, rows, pv)
    del rows
    torch.cuda.empty_cache()
    ix = pv.IvfflatIndex("vector_l2_ops", args.dim, args.lists).load(centers, offsets, grouped, order)
    q_t = queries[:4 * 2048]
    stream = torch.cuda.ExternalStream(pv.stream_handle(), device=dev)
    k, B = 10, 2048
    batches = [q_t[i:i + B].contiguous() for i in range(0, q_t.shape[0] - B + 1, B)]
    ids = torch.empty((B, k), dtype=torch.int64, device=dev)
    dist = torch.empty((B, k), dtype=torch.float32, device=dev)
    step = [0]

    def one():
        ix.search_into(batches[step[0] % len(batches)], k, args.probes, ids, dist)
        step[0] += 1

    def outputs():
        got = []
        for qb in batches:
            ix.search_into(qb, k, args.probes, ids, dist)
            got.append((ids.cpu().numpy().copy(), dist.cpu().numpy().copy()))
        return got

    rounds, ref = [], {}
    pv.set_option("scan_impl", 2)
    for r in range(args.rounds):
        for arm in (1, 0):
            pv.set_option("tc_level" + level, arm)
            n = 16 * len(batches)
            fallbacks = ix.tc_levelp_fallbacks if level == "p" else ix.tc_level0_fallbacks
            f0 = fallbacks()
            # bench.py's conditions: the timed steps follow `--load` untimed ones (its clock-sampler load, 600 steps), so
            # a power-limited card is at its sustained clock; the SM clock is sampled over both (bench.ClockSampler)
            sampler = bench.ClockSampler(0)
            sampler.start()
            ms = timed(pv, torch, stream, one, warmup=args.load, steps=n)
            clocks = sampler.stop()
            fails = (fallbacks() - f0) / (n + args.load)
            pv.prof_enable(True)
            for p in (pv.PROF_LIST_TC, pv.PROF_TOPK, pv.PROF_SCAN_ITEMS):
                pv.prof_read(p)
            ms_prof = timed(pv, torch, stream, one, warmup=0, steps=2 * len(batches))   # as bench.py times: kernel brackets on
            tc_ms, tc_n = pv.prof_read(pv.PROF_LIST_TC)
            rf_ms, rf_n = pv.prof_read(pv.PROF_TOPK)
            sc_ms, sc_n = pv.prof_read(pv.PROF_SCAN_ITEMS)
            pv.prof_enable(False)
            pv.tc_traffic(True, read=True)
            pv.tc_level0_rescored()
            one()
            pv.synchronize()
            t = pv.tc_traffic(False, read=True)
            rs = pv.tc_level0_rescored()
            got = outputs()
            if arm not in ref:
                ref[arm] = got
            rounds.append({"round": r, "tc_level" + level: arm, "ms_per_step": ms, "queries_per_s": B / (ms / 1000.0),
                           "ms_per_step_with_kernel_brackets": ms_prof, "sm_mhz": clocks.get("sm_mhz"),
                           "clock_reasons": clocks.get("reasons"),
                           "list_tc_ms": tc_ms / max(tc_n, 1), "list_tc_launches_per_step": tc_n / (2 * len(batches)),
                           "list_tc_bytes_per_launch": int((t[1] + t[2]) / max(t[3], 1)), "refine_ms": rf_ms / max(rf_n, 1),
                           "list_scan_ms": sc_ms / max(sc_n, 1), "listing_refine_rows_rescored_per_query": int(rs[0]) / max(int(rs[2]), 1),
                           "level%s_fallback_queries_per_batch" % level: fails})
    same = all(np.array_equal(a[0], b_[0]) and np.array_equal(a[1], b_[1]) for a, b_ in zip(ref[1], ref[0]))
    ratio = [rounds[i + 1]["ms_per_step"] / rounds[i]["ms_per_step"] for i in range(0, len(rounds), 2)]   # off / on
    print(json.dumps({"bench": "level" + level, "card": card(),
                      "workload": f"IVFFlat vector_l2_ops {args.rows}x{args.dim}, lists={args.lists}, probes={args.probes}, k={k}, "
                                  f"{len(batches)} batches of {B} queries, bench.py's {args.law} law and index ({how})",
                      "rounds": rounds, "speedup_level%s_per_round" % level: ratio, "outputs_identical": bool(same)}))


def bench_ivf_iter(args):
    """ivfflat.iterative_scan for a batch of filtered LIMIT 10 queries (WHERE id % 100 = 0): vb_ivf_scan_next pages until every
    query has 10 matches or is exhausted, against the per-scan loop (vb_ivf_scan_lists + successive vb_ivf_scan_items) on a
    sample of the queries, whose results must be equal."""
    b = build_ivf_index(args)
    pv, ix, q_t, opclass, rb, counts, offsets = b["pv"], b["ix"], b["q_t"], b["opclass"], b["rb"], b["counts"], b["offsets"]
    q = b["host"](q_t)
    nq, p, page, limit = args.queries, min(args.probes, args.lists), args.page, 10
    P = min(max(args.max_probes, args.probes), args.lists)
    keep = lambda ids: ids % 100 == 0
    lens = np.diff(offsets)
    order, _ = ix.scan_lists(q, P)                                   # the probe order the handle uses
    cum = np.concatenate([np.zeros((nq, 1), np.int64), np.cumsum(lens[order], axis=1)], axis=1)

    def run():
        t0 = time.perf_counter()
        scan = ix.iterative_scan(q, probes=p, max_probes=P, page=page)
        begin_s = time.perf_counter() - t0
        found = [[] for _ in range(nq)]
        live = np.ones(nq, dtype=bool)
        call_s, rows_read = [], []
        done = np.zeros(nq, dtype=np.int64)
        while live.any():
            t0 = time.perf_counter()
            ids, dist, cnt = scan.next_batch()
            call_s.append(time.perf_counter() - t0)
            now = scan.lists_done().astype(np.int64)
            rows_read.append(int((cum[np.arange(nq), now] - cum[np.arange(nq), done]).sum()))
            done = now
            for i in np.nonzero(live)[0]:
                c = int(cnt[i])
                m = keep(ids[i, :c])
                found[i].extend(zip(ids[i, :c][m].tolist(), dist[i, :c][m].tolist()))
                if len(found[i]) >= limit or c == 0:
                    found[i] = found[i][:limit]
                    live[i] = False
        scan.close()
        return begin_s, call_s, rows_read, found, done

    run()                                                            # warm-up: modules, workspaces, pinned staging
    begin_s, call_s, rows_read, found, done = run()

    def per_scan(i):                                                 # today's path for one query
        out = []
        for g0 in range(0, P, p):
            ids, dist, n = ix.scan_items(q[i], order[i, g0:g0 + p])
            m = keep(ids)
            out.extend(zip(ids[m].tolist(), dist[m].tolist()))
            if len(out) >= limit:
                break
        return out[:limit]

    sample = list(range(0, nq, max(1, nq // args.sample)))[:args.sample]
    per_scan(0)
    t0 = time.perf_counter()
    base = [per_scan(i) for i in sample]
    base_s = time.perf_counter() - t0
    pv.set_option("scan_impl", 0)                                    # the LDG scan everywhere: the arithmetic the handle uses
    base0 = [per_scan(i) for i in sample]
    pv.set_option("scan_impl", 2)
    assert all(found[i] == w for i, w in zip(sample, base0)), "iterative scan != per-scan loop (scan_impl = 0)"
    hbm, _, _, src = peaks()
    total_s = begin_s + sum(call_s)
    scan_bytes = [r * rb for r in rows_read]
    rate = [by / s / 1e9 for by, s in zip(scan_bytes, call_s)]
    print(json.dumps({"bench": "ivf-iter",
                      "workload": f"IVFFlat {opclass} {args.rows}x{args.dim}, lists={args.lists}, probes={p}, max_probes={P}, page={page}, {nq} queries, "
                                  f"WHERE id % 100 = 0 LIMIT {limit} (list sizes {int(counts.min())}/{int(counts.float().mean())}/{int(counts.max())})",
                      "card": card(),
                      "begin_ms": begin_s * 1e3, "next_calls": len(call_s),
                      "ms_per_next": {"first": call_s[0] * 1e3, "resumed_mean": float(np.mean(call_s[1:]) * 1e3) if len(call_s) > 1 else None,
                                      "resumed_max": float(np.max(call_s[1:]) * 1e3) if len(call_s) > 1 else None},
                      "groups_per_query": float(np.mean(np.ceil(done / p))),
                      "queries_done": {"with_10_matches": int(sum(len(f) >= limit for f in found)), "exhausted_first": int(sum(len(f) < limit for f in found))},
                      "filtered_queries_per_s": nq / total_s,
                      "roofline": {"bound": "hbm", "kernel": "whole vb_ivf_scan_next call (advance + chunks + LDG group scan + page select + finish + copy)",
                                   "bytes_per_call": scan_bytes, "achieved_per_call": rate, "peak": hbm, "unit": "GB/s",
                                   "frac_first_call": rate[0] / hbm, "peak_source": src,
                                   "note": "bytes = rows of the groups scanned in the call x row bytes; later calls scan only queries that moved to a new group"},
                      "per_scan_baseline": {"queries": len(sample), "filtered_queries_per_s": len(sample) / base_s,
                                            "identical_to_handle_scan_impl0": True,
                                            "identical_to_handle_default_options": all(found[i] == w for i, w in zip(sample, base))}}))


def bench_filter(args):
    """Row filters on the device against filtering on the host, on bench_ivf's index (ids = row numbers):
    - the filtered iterative scan (vb_ivf_scan_begin_filtered) of WHERE id % c = 0 LIMIT 10 against the unfiltered
      handle whose pages the host filters (the ivf-iter workload), first 10 matches of every query asserted equal;
    - the filtered exact top-k (vb_exact_topk_filtered_dev) over the same rows as a table against vb_table_rerank_dev
      with the allowed rows expanded into a candidate matrix, results asserted equal;
    - 64 per-query filters (id % 64) in one call against 64 single-filter calls, results asserted equal."""
    b = build_ivf_index(args)
    pv, torch, dev, ix, q_t, opclass, rb, counts, offsets = (b["pv"], b["torch"], b["dev"], b["ix"], b["q_t"], b["opclass"], b["rb"],
                                                             b["counts"], b["offsets"])
    grouped, order = b["keep"][1], b["keep"][2]
    stream = torch.cuda.ExternalStream(pv.stream_handle(), device=dev)
    q = b["host"](q_t)
    nq, p, limit = args.queries, min(args.probes, args.lists), 10
    P = min(max(args.max_probes, args.probes), args.lists)
    img_ids = order.cpu().numpy()                                     # heap id (= row number) of every image row
    list_of_row = np.repeat(np.arange(args.lists), np.diff(offsets))
    probe_order, _ = ix.scan_lists(q, P)
    hbm, _, _, src = peaks()

    def drain(scan, keep):
        """pages until every query has `limit` matches or is exhausted: (seconds per call, lists_done per call, matches)"""
        found = [[] for _ in range(nq)]
        live = np.ones(nq, dtype=bool)
        call_s, done = [], [np.zeros(nq, dtype=np.int64)]
        while live.any():
            t0 = time.perf_counter()
            ids, dist, cnt = scan.next_batch()
            call_s.append(time.perf_counter() - t0)
            done.append(scan.lists_done().astype(np.int64))
            for i in np.nonzero(live)[0]:
                c = int(cnt[i])
                m = keep(ids[i, :c]) if keep else slice(None)
                found[i].extend(zip(ids[i, :c][m].tolist(), dist[i, :c][m].tolist()))
                if len(found[i]) >= limit or c == 0:
                    found[i] = found[i][:limit]
                    live[i] = False
        return call_s, done, found

    def rows_per_call(done, per_list):
        cum = np.concatenate([np.zeros((nq, 1), np.int64), np.cumsum(per_list[probe_order], axis=1)], axis=1)
        return [int((cum[np.arange(nq), b1] - cum[np.arange(nq), b0]).sum()) for b0, b1 in zip(done, done[1:])]

    out = {"bench": "filter", "card": card(), "peak": {"hbm_gbs": hbm, "source": src},
           "workload": f"IVFFlat {opclass} {args.rows}x{args.dim}, lists={args.lists}, probes={p}, max_probes={P}, {nq} queries, "
                       f"WHERE id % c = 0 LIMIT {limit} (list sizes {int(counts.min())}/{int(counts.float().mean())}/{int(counts.max())})"}
    for c in (100, 1000):
        allowed_ids = np.arange(0, args.rows, c, dtype=np.int64)
        allowed_per_list = np.bincount(list_of_row[img_ids % c == 0], minlength=args.lists)
        keep = lambda ids, c=c: ids % c == 0
        res = {}
        for name, make in (("host_filtered", lambda: ix.iterative_scan(q, probes=p, max_probes=P, page=args.page)),
                           ("device_filtered", lambda: ix.iterative_scan(q, probes=p, max_probes=P, page=limit, filter=f))):
            for rep in range(2):                                      # the first run warms modules, workspaces and staging
                t0 = time.perf_counter()
                f = ix.filter(allowed_ids) if name == "device_filtered" else None   # (building the filter is counted)
                scan = make()
                begin_s = time.perf_counter() - t0
                call_s, done, found = drain(scan, keep if name == "host_filtered" else None)
                scan.close()
                if f is not None:
                    f.free()
            per_list = np.diff(offsets) if name == "host_filtered" else allowed_per_list
            rows = rows_per_call(done, per_list)
            rate = [r * rb / s / 1e9 for r, s in zip(rows, call_s)]
            res[name] = {"page": args.page if name == "host_filtered" else limit, "begin_ms": begin_s * 1e3, "next_calls": len(call_s),
                         "ms_per_next": {"first": call_s[0] * 1e3, "mean": float(np.mean(call_s)) * 1e3},
                         "groups_per_query": float(np.mean(np.ceil(done[-1] / p))),
                         "filtered_queries_per_s": nq / (begin_s + sum(call_s)),
                         "gathered_bytes_per_call": [r * rb for r in rows],
                         "frac_of_peak_per_call": [x / hbm for x in rate], "found": found}
        assert res["host_filtered"]["found"] == res["device_filtered"]["found"], f"id % {c}: device filter != host filter"
        for r in res.values():
            r.pop("found")
        res["note"] = ("bytes = rows of the groups a call scanned (host_filtered: every row; device_filtered: the allowed rows) x row "
                       "bytes, over the whole call's time (selection, finish and the copy back included)")
        out[f"ivf_iterative_id_mod_{c}"] = res

    # the same rows as a table, in image order: row r holds heap id img_ids[r]
    table = pv.Table(pv.VECTOR if args.elem == "vector" else pv.HALFVEC if args.elem == "halfvec" else pv.BIT, args.dim).append(grouped)
    metric = pv.L2 if args.elem != "bit" else pv.HAMMING
    k = limit
    ids_a = torch.empty((nq, k), dtype=torch.int64, device=dev)
    dist_a = torch.empty((nq, k), dtype=torch.float32, device=dev)
    ids_b, dist_b = torch.empty_like(ids_a), torch.empty_like(dist_a)
    stride = table.device_rows()[1]
    lib = pv.load()

    def filtered(fs, fq, qq=q_t, oi=ids_a, od=dist_a):
        farr, nf, fqa = pv._filter_args(fs, fq)
        pv._lib.check(lib.vb_exact_topk_filtered_dev(table.h, metric, pv._ptr(qq), qq.shape[0], k, farr, nf, pv._ptr(fqa), pv._ptr(oi),
                                                     pv._ptr(od)))

    for c in (100, 1000):
        rows = np.nonzero(img_ids % c == 0)[0].astype(np.int64)
        with table.filter(rows) as f:
            cand = torch.from_numpy(rows).to(dev).expand(nq, -1).contiguous()

            def rerank():
                pv._lib.check(lib.vb_table_rerank_dev(table.h, metric, pv._ptr(q_t), nq, pv._ptr(cand), cand.shape[1], k, pv._ptr(ids_b),
                                                      pv._ptr(dist_b)))

            ms_f = timed(pv, torch, stream, lambda: filtered(f, None), warmup=2, steps=10)
            ms_r = timed(pv, torch, stream, rerank, warmup=2, steps=10)
            assert torch.equal(ids_a, ids_b) and torch.equal(dist_a, dist_b), f"id % {c}: filtered top-k != rerank"
            by = nq * len(rows) * stride
            out[f"exact_id_mod_{c}"] = {"allowed_rows": len(rows), "ms_per_batch": {"filtered": ms_f, "rerank_expanded": ms_r},
                                        "candidate_bytes_uploaded_by_rerank": int(cand.numel() * 8), "gathered_bytes": by,
                                        "frac_of_peak": {"filtered": by / (ms_f / 1e3) / 1e9 / hbm, "rerank_expanded": by / (ms_r / 1e3) / 1e9 / hbm},
                                        "identical_results": True}
            del cand

    # 64 per-query filters in one call against one call per filter
    nf = 64
    fs = [table.filter(np.nonzero(img_ids % nf == i)[0]) for i in range(nf)]
    fq = (np.arange(nq) % nf).astype(np.int32)
    ms_one = timed(pv, torch, stream, lambda: filtered(fs, fq), warmup=2, steps=5)
    sel = [torch.from_numpy(np.nonzero(fq == i)[0]).to(dev) for i in range(nf)]
    qs = [q_t[s].contiguous() for s in sel]
    outs = [(torch.empty((len(s), k), dtype=torch.int64, device=dev), torch.empty((len(s), k), dtype=torch.float32, device=dev)) for s in sel]

    def per_filter():
        for i in range(nf):
            filtered(fs[i], None, qs[i], *outs[i])

    ms_many = timed(pv, torch, stream, per_filter, warmup=2, steps=5)
    for i in range(nf):
        assert torch.equal(ids_a[sel[i]], outs[i][0]) and torch.equal(dist_a[sel[i]], outs[i][1]), f"filter {i}: one call != per-filter call"
    by = sum(len(s) * len(fs[i]) for i, s in enumerate(sel)) * stride
    out["exact_64_filters_id_mod_64"] = {"ms_per_batch": {"one_call": ms_one, "64_calls": ms_many}, "gathered_bytes": by,
                                         "frac_of_peak": {"one_call": by / (ms_one / 1e3) / 1e9 / hbm, "64_calls": by / (ms_many / 1e3) / 1e9 / hbm},
                                         "identical_results": True}
    for f in fs:
        f.free()
    table.free()
    print(json.dumps(out))


def bench_hnsw_filter(args):
    """Element filters on the device against filtering on the host for hnsw.iterative_scan, at config C's shape: halfvec
    cosine rows of bench_hnsw's low-intrinsic-dimension law, the graph built on the device (m 16), ef_search 100,
    max_scan_tuples 20000, WHERE element % c = 0 LIMIT 10.
    - host_filtered: the unfiltered handle, drained until every query has 10 matches (every call advances every query);
    - device_filtered: the filtered handle with page = 10 (building the filter is counted).
    The first 10 matches of every query are asserted identical."""
    import torch
    import pgvector_b200 as pv
    pv.init(0)
    dev = torch.device("cuda", 0)
    n, dim, nq, ef, mst, limit = args.rows, args.dim, args.queries, args.ef, 20000, 10
    g = torch.Generator(device=dev).manual_seed(6)
    frame = torch.linalg.qr(torch.randn((dim, 16), generator=g, device=dev))[0]

    def law(m):
        x = torch.randn((m, 16), generator=g, device=dev) @ frame.T + 0.02 * torch.randn((m, dim), generator=g, device=dev)
        return torch.nn.functional.normalize(x, dim=1).half()

    rows = torch.cat([law(min(65536, n - i)) for i in range(0, n, 65536)])
    q = law(nq).view(torch.int16).cpu().numpy().view(np.uint16)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    gi = pv.HnswIndex("halfvec_cosine_ops", dim, m=16).build(rows, ef_construction=64)
    pv.synchronize()
    build_s = time.perf_counter() - t0
    del rows
    dup = int((gi.export()["dup_of"] >= 0).sum())
    out = {"bench": "hnsw-filter", "card": card(),
           "workload": f"HNSW halfvec_cosine_ops {n}x{dim}, m=16 (built on the device in {build_s:.0f}s, {dup} folded duplicates), "
                       f"ef_search={ef}, max_scan_tuples={mst}, {nq} queries, WHERE element % c = 0 LIMIT {limit}"}

    def host_arm(c, tuples_each_call=False):
        t0 = time.perf_counter()
        sc = gi.iterative_scan(q, ef_search=ef, max_scan_tuples=mst)
        found = [[] for _ in range(nq)]
        live = np.ones(nq, dtype=bool)
        at_call = np.zeros(nq, np.int64)
        tup = [np.zeros(nq, np.int64)]
        calls = 0
        while live.any():
            ids, dist, cnt = sc.next_batch()
            calls += 1
            if tuples_each_call:
                tup.append(sc.tuples())
            for i in np.nonzero(live)[0]:
                k = int(cnt[i])
                m = ids[i, :k] % c == 0
                found[i].extend(zip(ids[i, :k][m].tolist(), dist[i, :k][m].tolist()))
                if len(found[i]) >= limit or k == 0:
                    found[i] = found[i][:limit]
                    live[i] = False
                    at_call[i] = calls
        tuples = sc.tuples()
        sec = time.perf_counter() - t0
        sc.close()
        return sec, calls, found, tuples, at_call, tup

    def device_arm(c):
        t0 = time.perf_counter()
        f = gi.filter(np.arange(0, n, c, dtype=np.int64))
        sc = gi.iterative_scan(q, ef_search=ef, max_scan_tuples=mst, filter=f, page=limit)
        f.free()
        found = [[] for _ in range(nq)]
        live = np.ones(nq, dtype=bool)
        calls = 0
        while live.any():
            ids, dist, cnt = sc.next_batch()
            calls += 1
            for i in np.nonzero(live)[0]:
                k = int(cnt[i])
                found[i].extend(zip(ids[i, :k].tolist(), dist[i, :k].tolist()))
                if len(found[i]) >= limit or k < limit:
                    live[i] = False
        tuples = sc.tuples()
        sec = time.perf_counter() - t0
        sc.close()
        return sec, calls, found, tuples

    for c in (10, 100, 1000):
        for _ in range(2):                                            # the first run warms modules, workspaces and staging
            h_s, h_calls, h_found, h_tup, _, _ = host_arm(c)
            d_s, d_calls, d_found, d_tup = device_arm(c)
        assert h_found == d_found, f"element % {c}: device filter != host filter"
        # untimed: the unfiltered batch holding each query's 10th match, and whether it came from the drain
        _, _, _, _, at_call, tup = host_arm(c, tuples_each_call=True)
        tup = np.stack(tup)
        drained = tup[at_call - 1, np.arange(nq)] >= mst
        out[f"element_mod_{c}"] = {
            "host_filtered": {"next_calls": h_calls, "ms": h_s * 1e3, "filtered_queries_per_s": nq / h_s,
                              "mean_tuples_per_query": float(h_tup.mean())},
            "device_filtered": {"next_calls": d_calls, "ms": d_s * 1e3, "filtered_queries_per_s": nq / d_s,
                                "mean_tuples_per_query": float(d_tup.mean()),
                                # from the untimed replay of the unfiltered handle, not read from the filtered kernel: the
                                # batch holding each query's 10th match, which is where the filtered handle stops that query
                                "unfiltered_batches_to_10th_match_replayed": {"mean": float(at_call.mean()), "max": int(at_call.max())},
                                "queries_reaching_the_drain_replayed": int(drained.sum())},
            "identical_first_10": True}
    print(json.dumps(out))


def bench_kmeans(args):
    """k-means of config D on one GPU: 50 * lists samples x dim, lists centres (k-means++ seeding + Lloyd iterations)."""
    import torch
    import pgvector_b200 as pv
    pv.init(0)
    dev = torch.device("cuda", 0)
    n = 50 * args.k
    g = torch.Generator(device=dev).manual_seed(5)
    frame = torch.linalg.qr(torch.randn((args.dim, 16), generator=g, device=dev))[0]
    rows = torch.randn((n, 16), generator=g, device=dev) @ frame.T + 0.02 * torch.randn((n, args.dim), generator=g, device=dev)
    torch.cuda.synchronize()
    t = pv.Table(pv.VECTOR, args.dim).append(rows)
    pv.synchronize()
    # one untimed pass of each entry point first: workspace growth, pinned staging and lazy module loading are
    # one-time costs of the process, not of a build
    pv.kmeans(t, pv.L2, pv.kmeans_pp_init(t, pv.L2, min(args.k, 64), seed=1), max_iter=1)
    pv.kmeans(t, pv.L2, rows[:args.k].cpu().numpy(), max_iter=1)
    t0 = time.perf_counter()
    init = pv.kmeans_pp_init(t, pv.L2, args.k, seed=42)
    pp_s = time.perf_counter() - t0
    pv.prof_enable(True)
    pv.prof_read(pv.PROF_ASSIGN)
    t0 = time.perf_counter()
    centers, iters = pv.kmeans(t, pv.L2, init, max_iter=args.iters)
    km_s = time.perf_counter() - t0
    assign_ms, assign_n = pv.prof_read(pv.PROF_ASSIGN)
    pv.prof_enable(False)
    _, _, bf16_sus, src = peaks()
    flops = 2.0 * n * args.k * args.dim
    issued = 3 * flops / (assign_ms / assign_n) / 1e9
    print(json.dumps({"bench": "kmeans", "workload": f"k-means {n}x{args.dim} fp32 samples, {args.k} centres (config D sample phase on one GPU)",
                      "kmeanspp_s": pp_s, "kmeans_s": km_s, "iterations": iters, "s_per_iteration": km_s / max(iters, 1),
                      "assign_ms_per_iteration": assign_ms / assign_n, "rechecked_rows_last": pv.last_assign_rechecked(),
                      "roofline": {"bound": "tensor", "kernel": "assign step (pack + wgmma GEMM + re-check)", "achieved": issued, "peak": bf16_sus,
                                   "unit": "TFLOP/s", "frac": issued / bf16_sus, "peak_source": src + " bf16_tflops_sustained"}}))


def bench_exact(args):
    import torch
    import pgvector_b200 as pv
    pv.init(0)
    dev = torch.device("cuda", 0)
    stream = torch.cuda.ExternalStream(pv.stream_handle(), device=dev)
    g = torch.Generator(device=dev).manual_seed(1)
    rows = torch.randn((args.rows, args.dim), generator=g, device=dev)
    q = torch.randn((args.queries, args.dim), generator=g, device=dev)
    torch.cuda.synchronize()
    t = pv.Table(pv.VECTOR, args.dim).append(rows)
    k = 10
    ids = torch.empty((args.queries, k), dtype=torch.int64, device=dev)
    dist = torch.empty((args.queries, k), dtype=torch.float32, device=dev)
    ms = timed(pv, torch, stream, lambda: pv._lib.check(pv.load().vb_exact_topk_dev(t.h, pv.L2, pv._ptr(q), args.queries, k, pv._ptr(ids), pv._ptr(dist))))
    hbm, _, _, src = peaks()
    gbs = args.queries * args.rows * args.dim * 4 / (ms / 1000.0) / 1e9
    print(json.dumps({"bench": "exact", "workload": f"exact L2 top-{k} over {args.rows}x{args.dim} fp32, {args.queries} queries per batch",
                      "queries_per_s": args.queries / (ms / 1000.0), "ms_per_batch": ms,
                      "roofline": {"bound": "hbm (L2-resident when the table fits in 126 MB)", "achieved": gbs, "peak": hbm, "unit": "GB/s",
                                   "frac": gbs / hbm, "peak_source": src}}))


def bench_sparse(args):
    """sparsevec exact scan: resident CSR table, a batch of sparse queries per call (host buffers for the queries and the
    results); the roofline is the table's CSR bytes read once per query (8 bytes per stored entry)"""
    import torch
    import pgvector_b200 as pv
    import oracle as O
    S = pv.sparsevec
    pv.init(0)
    dev = torch.device("cuda", 0)
    stream = torch.cuda.ExternalStream(pv.stream_handle(), device=dev)
    rng = np.random.default_rng(1)
    n, dim, row_nnz, q_nnz, nq, k = args.rows, args.dim, args.nnz, 2 * args.nnz, args.queries, 10

    def ascending(count, nnz):
        """count rows of nnz strictly ascending indices in [0, dim): cumulative sums of gaps >= 1"""
        gaps = rng.integers(1, max(2, dim // nnz), size=(count, nnz))
        return (np.cumsum(gaps, axis=1) - 1).astype(np.int32)

    off = np.arange(n + 1, dtype=np.int64) * row_nnz
    idx = np.empty(n * row_nnz, dtype=np.int32)
    for r0 in range(0, n, 100_000):
        r1 = min(n, r0 + 100_000)
        idx[off[r0]:off[r1]] = ascending(r1 - r0, row_nnz).ravel()
    val = rng.standard_normal(off[-1]).astype(np.float32)
    table = S.SparseTable(dim).append(S.SparseRows(dim, off, idx, val))
    qidx = ascending(nq, q_nnz)
    qs = [S.SparseVector(dim, qidx[i], rng.standard_normal(q_nnz).astype(np.float32)) for i in range(nq)]
    Q = S.SparseRows.from_vectors(qs, dim)
    out = {}
    for name, metric in (("l2", O.L2), ("ip", O.NEG_IP)):
        ms = timed(pv, torch, stream, lambda: table.exact_topk(metric, Q, k), warmup=2, steps=5)
        out[name] = ms
    ids, dist = table.exact_topk(O.L2, Q, k)
    # parity on a few queries against the oracle
    same = 0
    for qi in range(min(8, nq)):
        d = O.sparse_distance_batch(O.L2, (qs[qi].indices, qs[qi].values), off, idx, val)
        want = np.argsort(d, kind="stable")[:k]
        same += int(np.array_equal(ids[qi], want))
    hbm, _, _, src = peaks()
    csr_bytes = off[-1] * 8 + (n + 1) * 8
    line = {"bench": "sparse", "workload": f"sparsevec exact top-{k}: {n} rows x {row_nnz} stored entries (dim {dim}), {nq} queries of ~{q_nnz} entries per call",
            "queries_per_s": {m: nq / (ms / 1000.0) for m, ms in out.items()}, "ms_per_call": out,
            "parity": {"queries_checked": min(8, nq), "identical_top_k_ids": same},
            "roofline": {"bound": "hbm", "kernel": "sparse_scan_kernel + segment_topk_kernel", "unit": "GB/s", "peak": hbm, "peak_source": src,
                         "traffic_per_query": int(csr_bytes), "achieved": {m: nq * csr_bytes / (ms / 1000.0) / 1e9 for m, ms in out.items()},
                         "frac": {m: nq * csr_bytes / (ms / 1000.0) / 1e9 / hbm for m, ms in out.items()},
                         "note": "the call also uploads the queries, writes and re-reads the nq x rows key matrix for the selection and returns the results"}}
    print(json.dumps(line))


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("what", choices=["assign", "hnsw", "exact", "ivf", "ivf-iter", "filter", "kmeans", "sparse", "rerank", "level0",
                                        "levelp", "hnsw-filter"])
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--lists", type=int, default=1000)
    ap.add_argument("--probes", type=int, default=10)
    ap.add_argument("--rows", type=int, default=None)
    ap.add_argument("--dim", type=int, default=None)
    ap.add_argument("--k", type=int, default=4096)
    ap.add_argument("--elem", default="halfvec")
    ap.add_argument("--ef", type=int, default=None)
    ap.add_argument("--queries", type=int, default=None)
    ap.add_argument("--nnz", type=int, default=100)
    ap.add_argument("--max-probes", type=int, default=100)
    ap.add_argument("--page", type=int, default=100)
    ap.add_argument("--sample", type=int, default=16)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--law", default="rank16", choices=["rank16", "mixture"])
    ap.add_argument("--load", type=int, default=600)
    a = ap.parse_args()
    if a.what == "rerank":      # config E's query batch and ef_search
        a.queries, a.ef = a.queries or 2048, a.ef or 200
    if a.what in ("ivf-iter", "filter", "hnsw-filter"):
        a.queries = a.queries or 2048
    if a.what in ("level0", "levelp"):
        a.queries = a.queries or 4 * 2048
    a.queries, a.ef = a.queries or 4096, a.ef or 100
    if a.what == "sparse":
        a.rows = a.rows or 1_000_000
        a.dim = a.dim or 100_000
        a.queries = min(a.queries, 64)
        bench_sparse(a)
    elif a.what == "assign":
        a.rows = a.rows or 1_250_000          # one GPU's share of config D (10M rows / 8)
        a.dim = a.dim or 1536
        bench_assign(a)
    elif a.what == "hnsw":
        a.rows = a.rows or 100_000
        a.dim = a.dim or (768 if a.elem == "halfvec" else 1024)
        bench_hnsw(a)
    elif a.what == "hnsw-filter":         # config C's shape
        a.rows = a.rows or 1_000_000
        a.dim = a.dim or 768
        bench_hnsw_filter(a)
    elif a.what == "rerank":
        a.rows = a.rows or 1_000_000
        a.dim = a.dim or 1024
        bench_rerank(a)
    elif a.what == "kmeans":
        a.dim = a.dim or 1536
        bench_kmeans(a)
    elif a.what in ("ivf-iter", "filter"):
        a.rows = a.rows or 1_000_000
        a.dim = a.dim or 1536
        a.elem = "vector" if a.elem == "halfvec" and "--elem" not in sys.argv else a.elem
        (bench_ivf_iter if a.what == "ivf-iter" else bench_filter)(a)
    elif a.what in ("level0", "levelp"):
        a.rows = a.rows or 1_000_000
        a.dim = a.dim or 1536
        a.elem = "vector" if "--elem" not in sys.argv else a.elem
        bench_level0(a, a.what[5:])
    elif a.what == "ivf":
        a.rows = a.rows or 1_000_000
        a.dim = a.dim or (1536 if a.elem == "halfvec" else 1024)
        bench_ivf(a)
    else:
        a.rows = a.rows or 10_000
        a.dim = a.dim or 128
        bench_exact(a)
