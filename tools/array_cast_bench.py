"""array_to_sparsevec on device rows (vb_array_to_sparsevec_batch_dev) against a device-to-device copy of its input,
and the host variant against pinned host-to-device copies of the same bytes.

Workloads: R x D (default 100k x 30522, a SPLADE vocabulary) float32 and float64 rows with about 1 % non-zero
elements, and 4 rows of 50M float32 elements with 0.01 % non-zero (too few rows to fill the device: each row is split
across warps).  The host variant runs on H x D float32 rows from pageable host memory.  numeric[]: N x 768 (default 1M)
numeric_send fields of 6 to 9 significant digits (0.ddddddddd, three base-10000 digits, 14 bytes, plus 8 bytes of
offset) to vector through vb_numeric_array_to_rows_batch_dev: elements/s and GB/s of fields plus offsets; its host
variant on NH x 768 of them.

Timing: CUDA events on the library stream around K calls of the C entry point into outputs sized by a first call,
after one warm-up call.  The _dev call reads its 24-byte check back and synchronises once per call, between its two
passes; that wait is inside its time.  The copy is a device-to-device copy of the input bytes on the same stream.  The
call reads its input twice (count pass, write pass), so its floor is about twice the copy.  Checks: the _dev result
equals the host variant's bit for bit on the host workload (exit 1 otherwise).  The card's name and power limit are
read in the same run.
Usage: python tools/array_cast_bench.py [--rows R] [--dim D] [--density P] [--reps K] [--host-rows H]
                                     [--numeric-rows N] [--numeric-host-rows NH]"""
import argparse
import ctypes as C
import json
import os
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from sparse_filter_bench import HBM_BYTES_PER_S, card  # noqa: E402

SRC = {"float32": 1, "float64": 2}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=100_000)
    ap.add_argument("--dim", type=int, default=30522)
    ap.add_argument("--density", type=float, default=0.01)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--host-rows", type=int, default=10_000)
    ap.add_argument("--numeric-rows", type=int, default=1_000_000)
    ap.add_argument("--numeric-host-rows", type=int, default=20_000)
    ap.add_argument("--seed", type=int, default=7)
    args = ap.parse_args()
    import torch
    import pgvector_b200 as pv
    pv.init(0)
    lib = pv._lib.load()
    dev = torch.device("cuda", 0)
    g = torch.Generator(device=dev).manual_seed(args.seed)
    lib_stream = torch.cuda.ExternalStream(pv.stream_handle())
    tp = lambda t: C.c_void_p(t.data_ptr())   # noqa: E731
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    bad = C.c_int64(-1)

    def rows(n, dim, dtype, block=2000, density=args.density):
        """n x dim rows, about density of them N(0, 1), the rest 0; made in blocks of rows to bound the temporaries"""
        x = torch.empty((n, dim), dtype=dtype, device=dev)
        for r in range(0, n, block):
            m = min(block, n - r)
            keep = torch.rand((m, dim), generator=g, device=dev) < density
            x[r:r + m] = torch.where(keep, torch.randn((m, dim), generator=g, device=dev), 0).to(dtype)
        return x

    def timed(call):
        call()
        pv.synchronize()
        ev[0].record(lib_stream)
        for _ in range(args.reps):
            call()
        ev[1].record(lib_stream)
        ev[1].synchronize()
        return ev[0].elapsed_time(ev[1]) / args.reps

    def run_dev(name, x):
        n, dim = x.shape
        src = SRC[str(x.dtype).split(".")[1]]
        off = torch.empty(n + 1, dtype=torch.int64, device=dev)
        torch.cuda.synchronize()
        lib.vb_array_to_sparsevec_batch_dev(src, dim, -1, tp(x), None, n, 0, tp(off), None, None, C.byref(bad))   # sizes
        total = int(off[-1].item())
        idx = torch.empty(max(total, 1), dtype=torch.int32, device=dev)
        val = torch.empty(max(total, 1), dtype=torch.float32, device=dev)

        def call():
            rc = lib.vb_array_to_sparsevec_batch_dev(src, dim, -1, tp(x), None, n, total, tp(off), tp(idx), tp(val), C.byref(bad))
            assert rc == 0, lib.vb_last_error()
        ms = timed(call)
        dst = torch.empty_like(x)
        with torch.cuda.stream(lib_stream):
            copy_ms = timed(lambda: dst.copy_(x))
        del dst
        in_b = x.numel() * x.element_size()
        out_b = 8 * (n + 1) + 8 * total
        legs[name] = {"shape": f"{n} x {dim} {x.dtype}", "nnz": total, "dev_ms": ms, "copy_ms": copy_ms, "vs_copy": ms / copy_ms,
                      "input_GB_per_s": in_b / (ms / 1e3) / 1e9,
                      "fraction_of_3.35_TB/s_two_reads": (2 * in_b + out_b) / (ms / 1e3) / HBM_BYTES_PER_S}
        return off, idx[:total], val[:total]

    legs, checks = {}, {}
    x = rows(args.rows, args.dim, torch.float32)
    run_dev("float4_dev", x)
    del x
    torch.cuda.empty_cache()
    x = rows(args.rows, args.dim, torch.float64)
    run_dev("float8_dev", x)
    del x
    torch.cuda.empty_cache()
    x = rows(4, 50_000_000, torch.float32, block=1, density=1e-4)   # 5000 per row: under CheckNnz
    run_dev("float4_4x50M_dev", x)
    del x
    torch.cuda.empty_cache()
    # the host variant from pageable host rows, against pinned copies of the same bytes to the device
    x = rows(args.host_rows, args.dim, torch.float32)
    xh = x.cpu().numpy()
    d_off, d_idx, d_val = run_dev("float4_dev_host_shape", x)
    t = {}

    def host_call():
        t["R"] = pv.sparsevec.array_to_sparsevec(xh, cap=int(d_off[-1].item()))
    host_call()   # warm-up: pinned staging and device scratch grow on the first call
    t0 = time.perf_counter()
    host_call()
    h_ms = (time.perf_counter() - t0) * 1e3
    pinned = torch.from_numpy(xh).pin_memory()
    dst = torch.empty_like(x)
    ev[0].record()
    dst.copy_(pinned, non_blocking=True)
    ev[1].record()
    ev[1].synchronize()
    h2d_ms = ev[0].elapsed_time(ev[1])
    R = t["R"]
    legs["float4_host"] = {"shape": f"{args.host_rows} x {args.dim} float32, pageable host", "host_ms": h_ms,
                           "pinned_h2d_copy_ms": h2d_ms, "vs_h2d_copy": h_ms / h2d_ms,
                           "input_GB_per_s": xh.nbytes / (h_ms / 1e3) / 1e9}
    checks["dev_equals_host"] = bool(np.array_equal(d_off.cpu().numpy(), R.row_off) and np.array_equal(d_idx.cpu().numpy(), R.idx)
                                     and np.array_equal(d_val.cpu().numpy().view(np.int32), R.val.view(np.int32)))
    del x, xh, pinned, dst, d_off, d_idx, d_val
    torch.cuda.empty_cache()

    # numeric[] -> vector: fields 0.ddddddddd with 6 to 9 significant digits, made on the device
    def numeric_fields(m):
        k = torch.randint(6, 10, (m,), generator=g, device=dev)
        lo = 10 ** (k - 1)
        v = lo + (torch.rand(m, generator=g, device=dev, dtype=torch.float64) * (9 * lo)).long()   # k digits
        v = v * 10 ** (12 - k)                                                                        # 12 digits
        f = torch.zeros((m, 14), dtype=torch.uint8, device=dev)
        f[:, 1] = 3                                     # ndigits 3
        f[:, 2] = 0xFF
        f[:, 3] = 0xFF                                  # weight -1
        f[:, 4] = torch.where(torch.rand(m, generator=g, device=dev) < 0.5, 0x40, 0).to(torch.uint8)
        f[:, 7] = k.to(torch.uint8)                     # dscale k
        for j, grp in enumerate((v // 10**8, v // 10**4 % 10**4, v % 10**4)):
            f[:, 8 + 2 * j] = (grp >> 8).to(torch.uint8)
            f[:, 9 + 2 * j] = (grp & 0xFF).to(torch.uint8)
        return f.reshape(-1), torch.arange(m + 1, dtype=torch.int64, device=dev) * 14

    nd = 768
    m = args.numeric_rows * nd
    data, offs = numeric_fields(m)
    out = torch.empty((args.numeric_rows, nd), dtype=torch.float32, device=dev)
    torch.cuda.synchronize()

    def num_call():
        rc = lib.vb_numeric_array_to_rows_batch_dev(0, nd, -1, tp(data), tp(offs), args.numeric_rows, tp(out), C.byref(bad))
        assert rc == 0, lib.vb_last_error()
    ms = timed(num_call)
    payload = data.numel() + 8 * offs.numel()
    legs["numeric_to_vector_dev"] = {"shape": f"{args.numeric_rows} x {nd} numeric, 6-9 digits, 14-byte fields", "dev_ms": ms,
                                     "elements_per_s": m / (ms / 1e3), "payload_GB_per_s": payload / (ms / 1e3) / 1e9,
                                     "payload_bytes": payload}
    nh = args.numeric_host_rows
    hd, ho = data[: nh * nd * 14].cpu().numpy(), offs[: nh * nd + 1].cpu().numpy()
    want = out[:nh].cpu().numpy()
    del data, offs, out
    torch.cuda.empty_cache()
    x = pv.numeric.NumericArrays(hd, ho, nd)
    pv.array_to_vector(x)    # warm-up
    t0 = time.perf_counter()
    got = pv.array_to_vector(x)
    h_ms = (time.perf_counter() - t0) * 1e3
    legs["numeric_to_vector_host"] = {"shape": f"{nh} x {nd} numeric, pageable host", "host_ms": h_ms,
                                      "elements_per_s": nh * nd / (h_ms / 1e3),
                                      "payload_GB_per_s": (hd.nbytes + ho.nbytes) / (h_ms / 1e3) / 1e9}
    checks["numeric_dev_equals_host"] = bool(np.array_equal(got.view(np.uint32), want.view(np.uint32)))
    result = {"bench": "array_cast", "card": card(),
              "timing": f"CUDA events on vb_stream() over {args.reps} C calls after one warm-up call; copy: device-to-device "
                        f"copy of the input bytes; host: one call from pageable host rows after a warm-up call (wall clock) against one pinned H2D copy",
              "calls": legs, "checks": checks, "checks_pass": all(checks.values())}
    print(json.dumps(result))
    if not result["checks_pass"]:
        sys.exit(1)


if __name__ == "__main__":
    main()
