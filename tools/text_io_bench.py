"""The type I/O on the device and from the host: vector text of N x D rows (default 1M x 1536), halfvec text of
N x E rows (default 1M x 768) and sparsevec text of sparse_filter_bench.py's SPLADE-like shape (default 200k rows of
dimension 30 522, ~120 stored entries).

Rows are random normal values (sparsevec: sparse_filter_bench's table); their text is what vb_rows_to_text_batch_dev
prints.  Timing: CUDA events around L back-to-back synchronised calls after a warm-up call: the _dev format (length pass,
scan, write pass; the output is formatted twice) and the _dev parse (count pass, parse, status read back).  Reported:
ms, GB/s of text, elements/s, and the bytes each call moves (text once, rows once, offsets) against the data-sheet
3.35 TB/s.  The host variants end to end (host clock) on H rows from pinned and from pageable text, and COPY-style
loading (host text copied to the device -> vb_text_to_rows_batch_dev with typmod = D -> vb_table_append_dev).  The CPU restatement's rate on one host thread
(tests/text_io_oracle, glibc strtof) on a sample.  Checks (exit 1 otherwise): the parse returns the rows bit for bit,
the host variants equal the _dev ones, a sample of the text equals the oracle's formatting.  The card's name and power
limit are read in the same run.
Usage: python tools/text_io_bench.py [--rows N --dim D --half_rows M --half_dim E --sparse_rows S --launches L
                                      --host_rows H --oracle_rows R]"""
import argparse
import ctypes as C
import json
import os
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from sparse_filter_bench import HBM_BYTES_PER_S, card, make_csr  # noqa: E402


def vp(t):
    return C.c_void_p(t.data_ptr()) if t is not None else None


def timed(torch, fn, launches):
    fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(launches):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / launches


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=1_000_000)
    ap.add_argument("--dim", type=int, default=1536)
    ap.add_argument("--half_rows", type=int, default=1_000_000)
    ap.add_argument("--half_dim", type=int, default=768)
    ap.add_argument("--sparse_rows", type=int, default=200_000)
    ap.add_argument("--sparse_dim", type=int, default=30522)
    ap.add_argument("--launches", type=int, default=3)
    ap.add_argument("--host_rows", type=int, default=50_000)
    ap.add_argument("--oracle_rows", type=int, default=200)
    args = ap.parse_args()
    import torch
    import pgvector_b200 as pv
    from pgvector_b200._lib import load, check
    from tests import text_io_oracle as T
    pv.init(0)
    lib = load()
    dev = torch.device("cuda", 0)
    res = {"card": card(), "format_passes": "two (length pass, CUB scan, write pass)", "shapes": {}}
    ok = True
    bad = C.c_int64(-1)
    g = torch.Generator(device=dev).manual_seed(7)

    def dense(name, elem, n, dim):
        nonlocal ok
        x = torch.randn((n, dim), generator=g, device=dev, dtype=torch.float32)
        if elem == pv.HALFVEC:
            x = x.half()
        esz = x.element_size()
        off = torch.empty(n + 1, dtype=torch.int64, device=dev)
        check(lib.vb_rows_to_text_batch_dev(elem, dim, vp(x), n, 0, vp(off), None))
        tb = int(off[-1])
        text = torch.empty(tb, dtype=torch.uint8, device=dev)
        fmt = lambda: check(lib.vb_rows_to_text_batch_dev(elem, dim, vp(x), n, tb, vp(off), vp(text)))  # noqa: E731
        ms_f = timed(torch, fmt, args.launches)
        roff = torch.empty(n + 1, dtype=torch.int64, device=dev)
        back = torch.empty_like(x)
        par = lambda: check(lib.vb_text_to_rows_batch_dev(elem, -1, n, vp(text), vp(off), n * dim, vp(roff), vp(back), C.byref(bad)))  # noqa: E731
        ms_p = timed(torch, par, args.launches)
        same = bool(torch.equal(back.view(torch.int16 if esz == 2 else torch.int32), x.view(torch.int16 if esz == 2 else torch.int32)))
        ok &= same
        # a sample against the oracle's formatting
        k = min(200, n)
        blob = text[: int(off[k])].cpu().numpy().tobytes()
        o = off[: k + 1].cpu().numpy()
        xs = x[:k].cpu().numpy()
        hs = xs.view(np.uint16) if esz == 2 else xs
        want = [T.vector_out(r, esz == 2) for r in hs]
        sample_ok = [blob[o[i]:o[i + 1]].decode() for i in range(k)] == want
        ok &= sample_ok
        moved_f = n * dim * esz + tb + 8 * (n + 1) * 2     # rows read, text written, lengths and offsets
        moved_p = tb * 2 + n * dim * esz + 8 * (n + 1) * 3  # text read by the count and parse passes, rows written
        r = {"rows": n, "dim": dim, "text_bytes": tb,
             "format_dev_ms": round(ms_f, 2), "format_GBps_text": round(tb / ms_f / 1e6, 1),
             "format_elements_per_s": round(n * dim / ms_f * 1e3), "format_share_hbm": round(moved_f / (ms_f / 1e3) / HBM_BYTES_PER_S, 4),
             "parse_dev_ms": round(ms_p, 2), "parse_GBps_text": round(tb / ms_p / 1e6, 1),
             "parse_elements_per_s": round(n * dim / ms_p * 1e3), "parse_share_hbm": round(moved_p / (ms_p / 1e3) / HBM_BYTES_PER_S, 4),
             "round_trip_exact": same, "sample_equals_oracle": sample_ok}
        # host variants on the first host_rows rows: pinned and pageable text, and COPY-style loading
        h = min(args.host_rows, n)
        htext = text[: int(off[h])].cpu().numpy()
        hoff = off[: h + 1].cpu().numpy()
        pinned = torch.empty(htext.size, dtype=torch.uint8, pin_memory=True)
        pinned.numpy()[:] = htext
        hrow = np.empty(h + 1, np.int64)
        hout = np.empty(h * dim, np.float32 if esz == 4 else np.uint16)
        for label, src in (("pageable", htext.ctypes.data), ("pinned", pinned.data_ptr())):
            t0 = time.perf_counter()
            check(lib.vb_text_to_rows_batch(elem, -1, h, C.c_void_p(src), hoff.ctypes.data, h * dim, hrow.ctypes.data,
                                            hout.ctypes.data, C.byref(bad)))
            dt = time.perf_counter() - t0
            r[f"host_parse_{label}_s"] = round(dt, 3)
            r[f"host_parse_{label}_GBps_text"] = round(htext.size / dt / 1e9, 2)
        same_h = np.array_equal(hout.view(np.uint16 if esz == 2 else np.uint32),
                                x[:h].cpu().numpy().reshape(-1).view(np.uint16 if esz == 2 else np.uint32))
        ok &= same_h
        r["host_equals_dev"] = same_h
        # COPY-style loading: host text -> device -> vb_text_to_rows_batch_dev (typmod = dim) -> vb_table_append_dev
        tab = pv.Table(elem, dim)
        drow = torch.empty(h + 1, dtype=torch.int64, device=dev)
        dout = torch.empty((h, dim), dtype=x.dtype, device=dev)
        t0 = time.perf_counter()
        dtext = pinned.to(dev, non_blocking=True)
        doff = torch.from_numpy(hoff).to(dev)
        torch.cuda.synchronize()
        check(lib.vb_text_to_rows_batch_dev(elem, dim, h, vp(dtext), vp(doff), h * dim, vp(drow), vp(dout), C.byref(bad)))
        check(lib.vb_table_append_dev(tab.h, vp(dout), h))
        check(lib.vb_synchronize())
        r["copy_load_rows_per_s"] = round(h / (time.perf_counter() - t0))
        # the oracle on one host thread
        R = min(args.oracle_rows, n)
        lits = [blob[o[i]:o[i + 1]].decode() for i in range(min(R, k))]
        t0 = time.perf_counter()
        for lit in lits:
            T.dense_in(esz == 2, lit)
        r["oracle_one_thread_elements_per_s"] = round(len(lits) * dim / (time.perf_counter() - t0))
        res["shapes"][name] = r
        del x, back, text

    dense("vector", pv.VECTOR, args.rows, args.dim)
    torch.cuda.empty_cache()
    dense("halfvec", pv.HALFVEC, args.half_rows, args.half_dim)
    torch.cuda.empty_cache()
    # sparsevec
    rng = np.random.default_rng(3)
    roff, idx, val = (torch.from_numpy(a).to(dev) for a in make_csr(args.sparse_rows, args.sparse_dim, 120, 0.5, rng, torch, dev))
    n = args.sparse_rows
    toff = torch.empty(n + 1, dtype=torch.int64, device=dev)
    check(lib.vb_sparsevec_to_text_batch_dev(args.sparse_dim, n, vp(roff), vp(idx), vp(val), 0, vp(toff), None))
    tb = int(toff[-1])
    text = torch.empty(tb, dtype=torch.uint8, device=dev)
    fmt = lambda: check(lib.vb_sparsevec_to_text_batch_dev(args.sparse_dim, n, vp(roff), vp(idx), vp(val), tb, vp(toff), vp(text)))  # noqa: E731
    ms_f = timed(torch, fmt, args.launches)
    nnz = int(roff[-1])
    dims = torch.empty(n, dtype=torch.int32, device=dev)
    r2 = torch.empty(n + 1, dtype=torch.int64, device=dev)
    bound = nnz + n
    i2 = torch.empty(bound, dtype=torch.int32, device=dev)
    v2 = torch.empty(bound, dtype=torch.float32, device=dev)
    par = lambda: check(lib.vb_text_to_sparsevec_batch_dev(-1, n, vp(text), vp(toff), bound, vp(dims), vp(r2), vp(i2), vp(v2), C.byref(bad)))  # noqa: E731
    ms_p = timed(torch, par, args.launches)
    same = bool(torch.equal(r2, roff)) and bool(torch.equal(i2[:nnz], idx)) and bool(torch.equal(v2[:nnz].view(torch.int32), val.view(torch.int32)))
    ok &= same
    moved_f = nnz * 8 + 8 * (n + 1) * 3 + tb
    moved_p = tb * 2 + nnz * 16 + 8 * (n + 1) * 4
    res["shapes"]["sparsevec"] = {"rows": n, "dim": args.sparse_dim, "nnz": nnz, "text_bytes": tb,
                                  "format_dev_ms": round(ms_f, 2), "format_GBps_text": round(tb / ms_f / 1e6, 1),
                                  "format_share_hbm": round(moved_f / (ms_f / 1e3) / HBM_BYTES_PER_S, 4),
                                  "parse_dev_ms": round(ms_p, 2), "parse_GBps_text": round(tb / ms_p / 1e6, 1),
                                  "parse_share_hbm": round(moved_p / (ms_p / 1e3) / HBM_BYTES_PER_S, 4),
                                  "round_trip_exact": same}
    res["checks_pass"] = bool(ok)
    print(json.dumps(res, indent=1))
    sys.exit(0 if ok else 1)


if __name__ == "__main__":
    main()
