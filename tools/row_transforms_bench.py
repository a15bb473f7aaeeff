"""The dense row transforms on device rows against their host variants: vb_norm_batch_dev, vb_l2_normalize_batch_dev,
vb_binary_quantize_batch_dev and vb_vector_to_halfvec_batch_dev on 1M x 1536 fp32 rows, the halfvec-input calls
(vb_halfvec_to_vector_batch_dev, and norm / l2_normalize / binary_quantize of halfvec rows) on 1M x 768 halfvec rows, and
vb_subvector_batch_dev taking 1536 -> 256 (subvector(embedding, 1, 256)).

Timing: CUDA events on the library stream around `--launches` back-to-back calls of the C entry point (into preallocated
outputs) after `--warmup` calls.  The read-free calls only enqueue; l2_normalize and vector_to_halfvec read their flag
back and synchronise every call, and that wait is inside their time.  Bytes are computed from the shapes: the rows read
once (subvector: the 256 columns it copies) and the output written once.  GB/s, and the share of the 3.35 TB/s data-sheet
HBM bandwidth.  For contrast, the host variant of each call on the same rows from pageable host memory, PCIe both ways
included (event time over `--host_calls` calls).  The card's name and power limit are read in the same run.  Checks: the
_dev output equals the host output bit for bit on the first and last rows (exit 1 otherwise).
Usage: python tools/row_transforms_bench.py [--rows N] [--dim D] [--half_dim E] [--sub S] [--launches L] [--warmup W] [--host_calls H]"""
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
    ap.add_argument("--half_dim", type=int, default=768)
    ap.add_argument("--sub", type=int, default=256)
    ap.add_argument("--launches", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--host_calls", type=int, default=3)
    ap.add_argument("--seed", type=int, default=7)
    args = ap.parse_args()
    import torch
    import pgvector_b200 as pv
    pv.init(0)
    lib = pv._lib.load()
    dev = torch.device("cuda", 0)
    n, dim, hdim, sub = args.rows, args.dim, args.half_dim, args.sub
    g = torch.Generator(device=dev).manual_seed(args.seed)
    x = torch.randn((n, dim), generator=g, device=dev, dtype=torch.float32)
    xh = torch.randn((n, hdim), generator=g, device=dev, dtype=torch.float32).half()
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

    x_host = x.cpu().numpy()
    xh_host = xh.cpu().numpy().view(np.uint16)
    legs, checks = {}, {}
    nb, hnb = (dim + 7) // 8, (hdim + 7) // 8
    cases = [
        # name, shape, device call factory -> (call, out), host fn, bytes read, bytes written
        ("vector_norm", f"{n} x {dim} fp32",
         lambda: torch.empty(n, dtype=torch.float64, device=dev), lambda o: lib.vb_norm_batch_dev(0, dim, p(x), n, p(o)),
         lambda: pv.vector_norm(x_host), 4 * n * dim, 8 * n),
        ("l2_normalize", f"{n} x {dim} fp32",
         lambda: torch.empty((n, dim), dtype=torch.float32, device=dev), lambda o: lib.vb_l2_normalize_batch_dev(0, dim, p(x), n, p(o)),
         lambda: pv.l2_normalize(x_host), 4 * n * dim, 4 * n * dim),
        ("binary_quantize", f"{n} x {dim} fp32",
         lambda: torch.empty((n, nb), dtype=torch.uint8, device=dev), lambda o: lib.vb_binary_quantize_batch_dev(0, dim, p(x), n, p(o)),
         lambda: pv.binary_quantize(x_host), 4 * n * dim, n * nb),
        ("vector_to_halfvec", f"{n} x {dim} fp32",
         lambda: torch.empty((n, dim), dtype=torch.float16, device=dev), lambda o: lib.vb_vector_to_halfvec_batch_dev(dim, p(x), n, p(o)),
         lambda: pv.vector_to_halfvec(x_host), 4 * n * dim, 2 * n * dim),
        ("subvector", f"{n} x {dim} fp32 -> {sub}",
         lambda: torch.empty((n, sub), dtype=torch.float32, device=dev),
         lambda o: lib.vb_subvector_batch_dev(0, dim, p(x), n, 1, sub, p(o), C.byref(d)),
         lambda: pv.subvector(x_host, 1, sub), 4 * n * sub, 4 * n * sub),
        ("halfvec_to_vector", f"{n} x {hdim} halfvec",
         lambda: torch.empty((n, hdim), dtype=torch.float32, device=dev), lambda o: lib.vb_halfvec_to_vector_batch_dev(hdim, p(xh), n, p(o)),
         lambda: pv.halfvec_to_vector(xh_host), 2 * n * hdim, 4 * n * hdim),
        ("halfvec_norm", f"{n} x {hdim} halfvec",
         lambda: torch.empty(n, dtype=torch.float64, device=dev), lambda o: lib.vb_norm_batch_dev(1, hdim, p(xh), n, p(o)),
         lambda: pv.vector_norm(xh_host, pv.HALFVEC), 2 * n * hdim, 8 * n),
        ("halfvec_l2_normalize", f"{n} x {hdim} halfvec",
         lambda: torch.empty((n, hdim), dtype=torch.float16, device=dev), lambda o: lib.vb_l2_normalize_batch_dev(1, hdim, p(xh), n, p(o)),
         lambda: pv.l2_normalize(xh_host, pv.HALFVEC), 2 * n * hdim, 2 * n * hdim),
        ("halfvec_binary_quantize", f"{n} x {hdim} halfvec",
         lambda: torch.empty((n, hnb), dtype=torch.uint8, device=dev), lambda o: lib.vb_binary_quantize_batch_dev(1, hdim, p(xh), n, p(o)),
         lambda: pv.binary_quantize(xh_host, pv.HALFVEC), 2 * n * hdim, n * hnb),
    ]
    for name, shape, alloc, call, host_fn, rd, wr in cases:
        out = alloc()
        ms = timed_dev(lambda: call(out))
        h_ms, h_out = timed_host(host_fn)
        legs[name] = {"shape": shape, "dev_ms": ms, "bytes_read": int(rd), "bytes_written": int(wr),
                      "dev_GB_per_s": (rd + wr) / (ms / 1e3) / 1e9, "fraction_of_3.35_TB/s": (rd + wr) / (ms / 1e3) / HBM_BYTES_PER_S,
                      "host_ms": h_ms, "host_vs_dev": h_ms / ms}
        checks[f"{name}_dev_equals_host"] = same_ends(out, h_out)
        del out, h_out
    out = {"bench": "row_transforms", "card": card(),
           "timing": f"CUDA events on vb_stream() over {args.launches} back-to-back C calls after {args.warmup} warm-up calls; "
                     f"host variants: pageable host rows, PCIe both ways, {args.host_calls} calls after one warm-up",
           "bytes": "rows read once (subvector: the copied columns) + output written once, from the shapes",
           "calls": legs, "checks": checks, "checks_pass": all(checks.values())}
    print(json.dumps(out))
    if not out["checks_pass"]:
        sys.exit(1)


if __name__ == "__main__":
    main()
