"""Exhaustive round trip of the device float formatter and parser: every finite float32 bit pattern (NaN and +-inf
are refused by vector_in) is printed with vb_rows_to_text_batch_dev as a one-element vector literal and read back with
vb_text_to_rows_batch_dev; every pattern must return its own bits.  Prints the count of mismatches (0 expected; exit 1
otherwise), the patterns covered, and the time.
Usage: python tools/text_io_check.py [--chunk_log2 K] [--stride S]   (S > 1 checks every S-th pattern only)"""
import argparse
import ctypes as C
import json
import os
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--chunk_log2", type=int, default=26)
    ap.add_argument("--stride", type=int, default=1)
    args = ap.parse_args()
    import torch
    import pgvector_b200 as pv
    pv.init(0)
    lib = pv._lib.load()
    dev = torch.device("cuda", 0)
    chunk = 1 << args.chunk_log2
    vp = lambda t: C.c_void_p(t.data_ptr())  # noqa: E731
    bad = C.c_int64(-1)
    mismatches, covered, first = 0, 0, []
    t0 = time.time()
    cap_text = chunk * 18
    text = torch.empty(cap_text, dtype=torch.uint8, device=dev)
    toff = torch.empty(chunk + 1, dtype=torch.int64, device=dev)
    roff = torch.empty(chunk + 1, dtype=torch.int64, device=dev)
    back = torch.empty(chunk, dtype=torch.float32, device=dev)
    for base in range(0, 1 << 32, chunk * args.stride):
        u = torch.arange(base, min(base + chunk * args.stride, 1 << 32), args.stride, dtype=torch.int64, device=dev)
        u = u[((u >> 23) & 0xFF) != 0xFF].to(torch.int32)        # finite patterns only
        x = u.view(torch.float32).contiguous()
        n = x.numel()
        torch.cuda.synchronize()
        pv._lib.check(lib.vb_rows_to_text_batch_dev(0, 1, vp(x), n, cap_text, vp(toff), vp(text)))
        rc = lib.vb_text_to_rows_batch_dev(0, 1, n, vp(text), vp(toff), n, vp(roff), vp(back), C.byref(bad))
        if rc != 0:
            print(json.dumps({"error": lib.vb_last_error().decode()[:200], "row": bad.value, "base": base}))
            sys.exit(1)
        diff = back[:n].view(torch.int32) != u
        k = int(diff.sum())
        if k and len(first) < 10:
            first += [hex(int(v) & 0xFFFFFFFF) for v in u[diff][:10].tolist()]
        mismatches += k
        covered += n
    print(json.dumps({"patterns": covered, "mismatches": mismatches, "first_mismatches": first[:10],
                      "seconds": round(time.time() - t0, 1)}))
    sys.exit(1 if mismatches else 0)


if __name__ == "__main__":
    main()
