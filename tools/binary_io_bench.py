#!/usr/bin/env python3
"""Binary type I/O throughput: vector_recv / vector_send and their halfvec and sparsevec twins on the device.

    python tools/binary_io_bench.py [--rows 1000000] [--dim 1536] [--sparse-rows 200000] [--reps 5]

For 1M x 1536 vector, 1M x 1536 halfvec and 200k SPLADE-like sparsevec rows (about 120 entries of 30522 dimensions,
as tools/text_io_bench.py): the _dev receive and send timed with CUDA events after a warm-up, next to a
device-to-device copy of the same payload bytes (the floor a realigning byte swap can reach), and the host variants
next to pinned H2D / D2H copies of the same bytes.  Prints bytes moved (payload read + rows written, or the reverse),
GB/s and the share of 3.35 TB/s, with the card's name and power limit.
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))

HBM = 3.35e12


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30).stdout.strip().split("\n")[0]
        return q
    except Exception as e:  # noqa: BLE001
        return f"unknown ({e})"


def timed(fn, reps, stream):
    import torch
    fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record(stream)
    for _ in range(reps):
        fn()
    b.record(stream)
    torch.cuda.synchronize()
    return a.elapsed_time(b) / reps / 1e3


def host_timed(fn, reps):
    fn()
    t = time.perf_counter()
    for _ in range(reps):
        fn()
    return (time.perf_counter() - t) / reps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=1_000_000)
    ap.add_argument("--dim", type=int, default=1536)
    ap.add_argument("--sparse-rows", type=int, default=200_000)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--host-rows", type=int, default=100_000, help="rows of the host-variant runs")
    args = ap.parse_args()
    import torch
    import pgvector_b200 as pv
    from pgvector_b200._lib import load
    pv.init(0)
    lib = load()
    stream = torch.cuda.ExternalStream(pv.stream_handle())
    res = {"card": card(), "results": []}
    rng = torch.Generator(device="cuda").manual_seed(1)

    def report(name, seconds, nbytes, floor=None):
        r = {"call": name, "ms": round(seconds * 1e3, 3), "bytes": int(nbytes), "GB/s": round(nbytes / seconds / 1e9, 1),
             "share_of_3.35TB/s": round(nbytes / seconds / HBM, 3)}
        if floor is not None:
            r["vs_copy"] = round(seconds / floor, 2)
        res["results"].append(r)
        print(json.dumps(r), flush=True)

    def copy_floor(nbytes):
        src = torch.empty(nbytes, dtype=torch.uint8, device="cuda")
        dst = torch.empty_like(src)
        t = timed(lambda: dst.copy_(src), args.reps, torch.cuda.current_stream())
        report(f"d2d copy {nbytes} B", t, 2 * nbytes)
        del src, dst
        return t

    for elem, dt, name in ((0, torch.float32, "vector"), (1, torch.float16, "halfvec")):
        n, dim = args.rows, args.dim
        x = torch.randn((n, dim), generator=rng, device="cuda").to(dt)
        esz = x.element_size()
        total = n * (4 + dim * esz)
        payload = torch.empty(total, dtype=torch.uint8, device="cuda")
        off = torch.empty(n + 1, dtype=torch.int64, device="cuda")
        torch.cuda.synchronize()
        floor = copy_floor(total)
        send = lambda: lib.vb_rows_to_binary_batch_dev(elem, dim, x.data_ptr(), n, total, off.data_ptr(), payload.data_ptr())  # noqa: E731
        assert send() == 0
        pv.synchronize()
        report(f"{name}_send_dev {n}x{dim}", timed(send, args.reps, stream), 2 * total, floor)
        rows = torch.empty_like(x)
        roff = torch.empty(n + 1, dtype=torch.int64, device="cuda")
        bad = C.c_int64(0)
        recv = lambda: lib.vb_binary_to_rows_batch_dev(elem, dim, n, payload.data_ptr(), off.data_ptr(), n * dim,  # noqa: E731
                                                       roff.data_ptr(), rows.data_ptr(), C.byref(bad))
        assert recv() == 0, lib.vb_last_error()
        assert torch.equal(rows.view(torch.int16 if esz == 2 else torch.int32), x.view(torch.int16 if esz == 2 else torch.int32))
        report(f"{name}_recv_dev {n}x{dim}", timed(recv, args.reps, stream), 2 * total, floor)
        # host variants over a slice, next to pinned copies of the same bytes
        hn = min(args.host_rows, n)
        xh = x[:hn].cpu().numpy()
        hb = hn * (4 + dim * esz)
        ph = np.empty(hb, np.uint8)
        oh = np.empty(hn + 1, np.int64)
        rh = np.empty_like(xh)
        roh = np.empty(hn + 1, np.int64)
        report(f"{name}_send host {hn}x{dim}",
               host_timed(lambda: lib.vb_rows_to_binary_batch(elem, dim, xh.ctypes.data, hn, hb, oh.ctypes.data, ph.ctypes.data), 2), hb)
        report(f"{name}_recv host {hn}x{dim}",
               host_timed(lambda: lib.vb_binary_to_rows_batch(elem, dim, hn, ph.ctypes.data, oh.ctypes.data, hn * dim, roh.ctypes.data,
                                                              rh.ctypes.data, C.byref(bad)), 2), hb)
        pin = torch.empty(hb, dtype=torch.uint8).pin_memory()
        dev = torch.empty(hb, dtype=torch.uint8, device="cuda")
        report(f"pinned h2d {hb} B", host_timed(lambda: (dev.copy_(pin), torch.cuda.synchronize()), 3), hb)
        report(f"pinned d2h {hb} B", host_timed(lambda: (pin.copy_(dev), torch.cuda.synchronize()), 3), hb)
        del x, payload, rows, dev, pin
        torch.cuda.empty_cache()

    # SPLADE-like sparsevec rows
    n, dim = args.sparse_rows, 30522
    g = np.random.default_rng(2)
    nnz = np.clip(g.normal(120, 30, n).astype(np.int64), 1, 400)
    roff = np.zeros(n + 1, np.int64)
    roff[1:] = np.cumsum(nnz)
    idx = np.concatenate([np.sort(g.choice(dim, k, replace=False)) for k in nnz]).astype(np.int32)
    val = (g.random(int(roff[-1])) + 0.1).astype(np.float32)
    droff, didx, dval = (torch.from_numpy(a).cuda() for a in (roff, idx, val))
    total = 12 * n + 8 * int(roff[-1])
    payload = torch.empty(total, dtype=torch.uint8, device="cuda")
    off = torch.empty(n + 1, dtype=torch.int64, device="cuda")
    floor = copy_floor(total)
    send = lambda: lib.vb_sparsevec_to_binary_batch_dev(dim, n, droff.data_ptr(), didx.data_ptr(), dval.data_ptr(), total,  # noqa: E731
                                                        off.data_ptr(), payload.data_ptr())
    report(f"sparsevec_send_dev {n} rows", timed(send, args.reps, stream), 2 * total, floor)
    ro2 = torch.empty(n + 1, dtype=torch.int64, device="cuda")
    i2 = torch.empty_like(didx)
    v2 = torch.empty_like(dval)
    d2 = torch.empty(n, dtype=torch.int32, device="cuda")
    bad = C.c_int64(0)
    recv = lambda: lib.vb_binary_to_sparsevec_batch_dev(-1, n, payload.data_ptr(), off.data_ptr(), int(roff[-1]), d2.data_ptr(),  # noqa: E731
                                                        ro2.data_ptr(), i2.data_ptr(), v2.data_ptr(), C.byref(bad))
    assert recv() == 0, lib.vb_last_error()
    assert torch.equal(i2, didx) and torch.equal(v2, dval)
    report(f"sparsevec_recv_dev {n} rows", timed(recv, args.reps, stream), 2 * total, floor)
    ph = payload.cpu().numpy()
    oh = off.cpu().numpy()
    roh, ih, vh, dh = np.empty(n + 1, np.int64), np.empty_like(idx), np.empty_like(val), np.empty(n, np.int32)
    report(f"sparsevec_recv host {n} rows",
           host_timed(lambda: lib.vb_binary_to_sparsevec_batch(-1, n, ph.ctypes.data, oh.ctypes.data, int(roff[-1]), dh.ctypes.data,
                                                               roh.ctypes.data, ih.ctypes.data, vh.ctypes.data, C.byref(bad)), 2), total)
    report(f"sparsevec_send host {n} rows",
           host_timed(lambda: lib.vb_sparsevec_to_binary_batch(dim, n, roff.ctypes.data, idx.ctypes.data, val.ctypes.data, total,
                                                               oh.ctypes.data, ph.ctypes.data), 2), total)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
