"""INSERT and VACUUM on a resident IVFFlat image (vb_ivf_insert / vb_ivf_delete) at config B's shape: bench.py's law
(rank16), its 1M x 1536 rows and its 1000-list index, built through bench.py's functions (as `bench_extra.py level0`
does), loaded with heap ids, with the bf16 planes and the int8 plane resident (four 2048-query batches searched first).
Reports, in one JSON line:
  - the card's name and power limit, read in the same run;
  - the first insert after the load (one row), which grows the table by half;
  - the insert that first outgrows the plane buffers (sized to the loaded rows), which re-allocates them and re-packs
    them whole;
  - per m = 1 / 64 / 1024 / 16384 inserted rows, three calls each (none grows the table or the planes): the call's
    time (host clock around the synchronised call), the bytes it moved and re-packed (computed from the shifted
    suffix), that over the time as a share of 3.35 TB/s, and free device memory before the call;
  - the vb_ivf_replace_list loop that inserts the same rows one touched list at a time (m = 1 / 64 / 1024; list contents
    staged on the host before the clock starts), and the first batched search after it;
  - the first batched search step after each insert against a steady step;
  - deletes of 1000 ids and of 1 % of the rows;
  - whether the final image's search outputs equal those of a fresh load of the same arrays, bit for bit.
Usage: python tools/ivf_insert_bench.py [--rows N] [--lists L] [--probes P]"""
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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=1_000_000)
    ap.add_argument("--dim", type=int, default=1536)
    ap.add_argument("--lists", type=int, default=1000)
    ap.add_argument("--probes", type=int, default=10)
    args = ap.parse_args()
    import torch
    import bench
    import pgvector_b200 as pv
    pv.init(0)
    dev = torch.device("cuda", 0)
    bargs = argparse.Namespace(rows=args.rows, dim=args.dim, lists=args.lists, latent_dim=16, components=1000, queries=80_000)
    rows, queries = bench.make_dataset(bargs, "rank16", dev)
    torch.cuda.synchronize()
    centers, offsets, grouped, order, _ = bench.build_index_arrays(bargs, "rank16", rows, pv)
    del rows
    torch.cuda.empty_cache()
    L = args.lists
    off = np.asarray(offsets.cpu() if torch.is_tensor(offsets) else offsets, dtype=np.int64)
    grouped = grouped.contiguous()
    ids = (order.to(torch.int64) if torch.is_tensor(order) else torch.from_numpy(np.asarray(order, np.int64)).to(dev)).contiguous()
    ix = pv.IvfflatIndex("vector_l2_ops", args.dim, L).load(centers, off, grouped, ids)
    stride = args.dim * 4
    k, B = 10, 2048
    batches = [queries[i:i + B].contiguous() for i in range(0, 4 * B, B)]
    new = queries[10_000:].contiguous()
    o_ids = torch.empty((B, k), dtype=torch.int64, device=dev)
    o_dist = torch.empty((B, k), dtype=torch.float32, device=dev)
    state = {"grouped": grouped, "ids": ids, "off": off, "next": 0, "nid": 10 ** 12}

    def step(qb):
        t = time.perf_counter()
        ix.search_into(qb, k, args.probes, o_ids, o_dist)
        pv.synchronize()
        return (time.perf_counter() - t) * 1e3

    def steady():
        return float(np.median([step(batches[i % 4]) for i in range(12)]))

    def model_insert(x, nid, lists):
        lab = torch.from_numpy(np.concatenate([np.repeat(np.arange(L), np.diff(state["off"])), lists])).to(dev)
        perm = torch.sort(lab, stable=True).indices
        state["grouped"] = torch.cat([state["grouped"], x])[perm].contiguous()
        state["ids"] = torch.cat([state["ids"], nid])[perm].contiguous()
        state["off"] = np.concatenate([[0], np.cumsum(np.bincount(lab.cpu().numpy(), minlength=L))]).astype(np.int64)

    def take(m):
        x = new[state["next"]:state["next"] + m].contiguous()
        state["next"] += m
        nid = torch.arange(state["nid"], state["nid"] + m, device=dev, dtype=torch.int64)
        state["nid"] += m
        return x, nid

    def moved_bytes(lists, off_before, whole=False):
        n_old = int(off_before[-1])
        first = int(off_before[int(lists.min()) + 1])
        suffix, m = n_old - first, len(lists)
        moved = 4 * suffix * (stride + 8) + 2 * m * (stride + 8)           # staged out and back: two reads, two writes
        t0 = 0 if whole else first // 128 * 128
        rep = n_old + m - t0
        kp = (args.dim + 63) // 64 * 64
        k8 = (args.dim + 127) // 128 * 128
        repacked = rep * (3 * stride + 4 * kp + 4 + k8 + 8)                  # rows read three times; planes, |x|^2, int8, s_x, R_x
        return moved, repacked

    for qb in batches:
        step(qb)
    out = {"bench": "ivf_insert", "card": card(), "workload": f"IVFFlat vector_l2_ops {args.rows}x{args.dim}, lists={L}, bf16 and int8 planes resident",
           "steady_step_ms": steady()}
    # the first insert after the load: the table has no headroom and grows by half
    x, nid = take(1)
    t = time.perf_counter()
    lists = ix.insert(x, nid)
    out["first_insert_growth_ms"] = (time.perf_counter() - t) * 1e3
    model_insert(x, nid, lists)
    out["first_step_after_growth_ms"] = step(batches[0])
    # the plane buffers were sized to the loaded rows' tiles: the insert that first needs one more tile allocates them
    # again with half again as many tiles and re-packs them whole (bf16 and int8)
    tiles = lambda n: (n + 127) // 128
    plane_cap = tiles(args.rows)
    m = plane_cap * 128 - int(state["off"][-1]) + 1
    x, nid = take(m)
    off_before = state["off"].copy()
    t = time.perf_counter()
    lists = ix.insert(x, nid)
    ms = (time.perf_counter() - t) * 1e3
    model_insert(x, nid, lists)
    mv, rp = moved_bytes(lists, off_before, whole=True)
    out["plane_growth_insert"] = {"m": m, "ms": ms, "bytes_moved": mv, "bytes_repacked": rp, "share_of_3.35TB_s": (mv + rp) / (ms / 1e3) / HBM,
                                  "first_step_after_ms": step(batches[0])}
    plane_cap = max(tiles(int(state["off"][-1])), plane_cap + plane_cap // 2)
    # per m: three calls, none of which grows the table or the plane buffers (checked)
    rows_out = []
    for m in (1, 64, 1024, 16384):
        samples = []
        for _ in range(3):
            x, nid = take(m)
            off_before = state["off"].copy()
            assert tiles(int(off_before[-1]) + m) <= plane_cap
            free_b = torch.cuda.mem_get_info()[0]
            t = time.perf_counter()
            lists = ix.insert(x, nid)
            ms = (time.perf_counter() - t) * 1e3
            model_insert(x, nid, lists)
            first = step(batches[1])
            mv, rp = moved_bytes(lists, off_before)
            samples.append({"ms": ms, "lists_touched": int(len(np.unique(lists))), "bytes_moved": mv, "bytes_repacked": rp,
                            "share_of_3.35TB_s": (mv + rp) / (ms / 1e3) / HBM, "free_gb_before": free_b / 1e9, "first_step_after_ms": first})
        rows_out.append({"m": m, "ms_median": float(np.median([r["ms"] for r in samples])), "samples": samples})
    out["insert"] = rows_out
    out["steady_step_after_inserts_ms"] = steady()
    # the same kind of rows through vb_ivf_replace_list, one touched list at a time
    rep = []
    for m in (1, 64, 1024):
        x, nid = take(m)
        lists, _ = ix.scan_lists(x.cpu().numpy(), 1)
        lists = lists[:, 0]
        g_host = {}
        for l in np.unique(lists):
            lo, hi = state["off"][l], state["off"][l + 1]
            sel = np.flatnonzero(lists == l)
            g_host[int(l)] = (np.concatenate([state["grouped"][lo:hi].cpu().numpy(), x[sel].cpu().numpy()]),
                              np.concatenate([state["ids"][lo:hi].cpu().numpy(), nid[sel].cpu().numpy()]))
        pv.synchronize()
        t = time.perf_counter()
        for l, (r, i) in g_host.items():
            ix.replace_list(l, r, i)
        ms = (time.perf_counter() - t) * 1e3
        model_insert(x, nid, lists)
        rep.append({"m": m, "calls": len(g_host), "ms": ms, "first_step_after_ms": step(batches[2])})
    out["replace_list_loop"] = rep
    for qb in batches:
        step(qb)
    # deletes
    dl = []
    rng = np.random.default_rng(5)
    for cnt in (1000, args.rows // 100):
        all_ids = state["ids"].cpu().numpy()
        victims = rng.choice(all_ids, cnt, replace=False)
        t = time.perf_counter()
        removed = ix.delete(victims)
        ms = (time.perf_counter() - t) * 1e3
        keep = torch.from_numpy(~np.isin(all_ids, victims)).to(dev)
        lab = np.repeat(np.arange(L), np.diff(state["off"]))[keep.cpu().numpy()]
        state["grouped"] = state["grouped"][keep].contiguous()
        state["ids"] = state["ids"][keep].contiguous()
        state["off"] = np.concatenate([[0], np.cumsum(np.bincount(lab, minlength=L))]).astype(np.int64)
        dl.append({"ids": cnt, "removed": removed, "ms": ms, "first_step_after_ms": step(batches[3])})
    out["delete"] = dl
    # bit identity with a fresh load of the same arrays
    def outputs(index):
        got = []
        for qb in batches:
            index.search_into(qb, k, args.probes, o_ids, o_dist)
            pv.synchronize()
            got.append((o_ids.cpu().numpy().copy(), o_dist.cpu().numpy().copy()))
        return got
    a = outputs(ix)
    same_off = bool(np.array_equal(ix.list_offsets(), state["off"]))
    ix.free()
    torch.cuda.empty_cache()
    e = pv.IvfflatIndex("vector_l2_ops", args.dim, L).load(centers, state["off"], state["grouped"], state["ids"])
    b = outputs(e)
    out["identical_to_fresh_load"] = same_off and all(np.array_equal(x[0], y[0]) and np.array_equal(x[1], y[1]) for x, y in zip(a, b))
    e.free()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
