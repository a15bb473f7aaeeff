"""The operators + - * || and the array casts on device rows against their host variants, on 1M x 1536 rows: fp32 +
of two row sets and with one broadcast row (v - $1), fp32 *, halfvec +, || of 768 + 768 columns, and double
precision[] -> vector and -> halfvec.

Timing: CUDA events on the library stream around `--launches` back-to-back calls of the C entry point (into preallocated
outputs) after `--warmup` calls.  vb_arith_batch_dev and vb_array_to_rows_batch_dev read their 8-byte first-offender
key back and synchronise every call, and that wait is inside their time; vb_concat_batch_dev only enqueues.  Bytes are
computed from the shapes: the operands read once (a broadcast row counts once) and the result written once.  GB/s, and
the share of the 3.35 TB/s data-sheet HBM bandwidth.  For contrast, the host variant of each call on the same rows from
pageable host memory, PCIe both ways included.  The card's name and power limit are read in the same run.  Checks: the
_dev output equals the host output bit for bit on the first and last rows (exit 1 otherwise).
Usage: python tools/row_arith_bench.py [--rows N] [--dim D] [--launches L] [--warmup W] [--host_calls H]"""
import argparse
import ctypes as C
import json
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from sparse_filter_bench import HBM_BYTES_PER_S, card  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=1_000_000)
    ap.add_argument("--dim", type=int, default=1536)
    ap.add_argument("--launches", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--host_calls", type=int, default=1)
    ap.add_argument("--seed", type=int, default=7)
    args = ap.parse_args()
    import torch
    import pgvector_b200 as pv
    pv.init(0)
    lib = pv._lib.load()
    dev = torch.device("cuda", 0)
    n, dim = args.rows, args.dim
    half = dim // 2
    g = torch.Generator(device=dev).manual_seed(args.seed)
    x = torch.randn((n, dim), generator=g, device=dev, dtype=torch.float32)
    y = torch.randn((n, dim), generator=g, device=dev, dtype=torch.float32)
    w = torch.randn((1, dim), generator=g, device=dev, dtype=torch.float32)
    lib_stream = torch.cuda.ExternalStream(pv.stream_handle())
    p = pv._ptr
    d = C.c_int(0)
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]

    def timed_dev(call):
        for _ in range(args.warmup):
            assert call() == 0, lib.vb_last_error()
        pv.synchronize()
        ev[0].record(lib_stream)
        for _ in range(args.launches):
            assert call() == 0, lib.vb_last_error()
        ev[1].record(lib_stream)
        ev[1].synchronize()
        return ev[0].elapsed_time(ev[1]) / args.launches

    def timed_host(fn):
        fn()
        torch.cuda.synchronize()
        ev[0].record()
        for _ in range(args.host_calls):
            out = fn()
        ev[1].record()
        ev[1].synchronize()
        return ev[0].elapsed_time(ev[1]) / args.host_calls, out

    def bits(a):
        a = np.ascontiguousarray(a)
        return a.view({8: np.uint64, 4: np.uint32, 2: np.uint16, 1: np.uint8}[a.itemsize])

    def same_ends(dev_out, host_out, m=65_536):
        h = np.asarray(host_out)
        head = dev_out[:m].cpu().numpy()
        tail = dev_out[-1000:].cpu().numpy()
        return bool(np.array_equal(bits(head), bits(h[:m])) and np.array_equal(bits(tail), bits(h[-1000:])))

    legs, checks = {}, {}
    f32 = lambda shape: torch.empty(shape, dtype=torch.float32, device=dev)   # noqa: E731
    f16 = lambda shape: torch.empty(shape, dtype=torch.float16, device=dev)   # noqa: E731

    def run(name, shape, out, call, host_fn, rd, wr):
        ms = timed_dev(lambda: call(out))
        h_ms, h_out = timed_host(host_fn)
        legs[name] = {"shape": shape, "dev_ms": ms, "bytes_read": int(rd), "bytes_written": int(wr),
                      "dev_GB_per_s": (rd + wr) / (ms / 1e3) / 1e9, "fraction_of_3.35_TB/s": (rd + wr) / (ms / 1e3) / HBM_BYTES_PER_S,
                      "host_ms": h_ms, "host_vs_dev": h_ms / ms}
        checks[f"{name}_dev_equals_host"] = same_ends(out, h_out)

    xh_, yh_, wh_ = x.cpu().numpy(), y.cpu().numpy(), w.cpu().numpy()
    out = f32((n, dim))
    run("vector_add", f"{n} x {dim} fp32 + {n} x {dim}", out,
        lambda o: lib.vb_arith_batch_dev(0, 0, dim, p(x), n, dim, p(y), n, p(o)),
        lambda: pv.vector_add(xh_, yh_), 8 * n * dim, 4 * n * dim)
    run("vector_add_broadcast", f"{n} x {dim} fp32 + 1 x {dim}", out,
        lambda o: lib.vb_arith_batch_dev(0, 0, dim, p(x), n, dim, p(w), 1, p(o)),
        lambda: pv.vector_add(xh_, wh_), 4 * n * dim + 4 * dim, 4 * n * dim)
    run("vector_mul", f"{n} x {dim} fp32 * {n} x {dim}", out,
        lambda o: lib.vb_arith_batch_dev(0, 2, dim, p(x), n, dim, p(y), n, p(o)),
        lambda: pv.vector_mul(xh_, yh_), 8 * n * dim, 4 * n * dim)
    del out
    xh, yh = x.half(), y.half()
    xhh, yhh = xh.cpu().numpy().view(np.uint16), yh.cpu().numpy().view(np.uint16)
    run("halfvec_add", f"{n} x {dim} halfvec + {n} x {dim}", f16((n, dim)),
        lambda o: lib.vb_arith_batch_dev(1, 0, dim, p(xh), n, dim, p(yh), n, p(o)),
        lambda: pv.vector_add(xhh, yhh, pv.HALFVEC), 4 * n * dim, 2 * n * dim)
    del xh, yh, xhh, yhh
    a, b = x[:, :half].contiguous(), y[:, :half].contiguous()
    ah, bh = a.cpu().numpy(), b.cpu().numpy()
    run("vector_concat", f"{n} x {half} fp32 || {n} x {half}", f32((n, 2 * half)),
        lambda o: lib.vb_concat_batch_dev(0, half, p(a), n, half, p(b), n, p(o), C.byref(d)),
        lambda: pv.vector_concat(ah, bh), 8 * n * half, 8 * n * half)
    del a, b, ah, bh, yh_, wh_
    x8 = x.double()
    x8h = x8.cpu().numpy()
    del xh_
    run("float8_to_vector", f"{n} x {dim} double precision[]", f32((n, dim)),
        lambda o: lib.vb_array_to_rows_batch_dev(0, 2, dim, -1, p(x8), n, p(o)),
        lambda: pv.array_to_vector(x8h), 8 * n * dim, 4 * n * dim)
    run("float8_to_halfvec", f"{n} x {dim} double precision[]", f16((n, dim)),
        lambda o: lib.vb_array_to_rows_batch_dev(1, 2, dim, -1, p(x8), n, p(o)),
        lambda: pv.array_to_halfvec(x8h), 8 * n * dim, 2 * n * dim)
    result = {"bench": "row_arith", "card": card(),
              "timing": f"CUDA events on vb_stream() over {args.launches} back-to-back C calls after {args.warmup} warm-up calls; "
                        f"host variants: pageable host rows, PCIe both ways, {args.host_calls} calls after one warm-up",
              "bytes": "operands read once (a broadcast row once) + result written once, from the shapes",
              "calls": legs, "checks": checks, "checks_pass": all(checks.values())}
    print(json.dumps(result))
    if not result["checks_pass"]:
        sys.exit(1)


if __name__ == "__main__":
    main()
