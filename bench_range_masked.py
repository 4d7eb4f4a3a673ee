"""Subset range search by gathered copy (b2_index_range_search with ids) against masked range search
(b2_index_range_search_masked) on the same rows and the same strictly ascending random subsets, on one GPU, alternated in one
process so that clock and power drift hit both alike.

    python bench_range_masked.py [--steps 3] [--warmup 1] [--n 1000000] [--d 768] [--nq 100000] [--sample 64] [--no-host]

Store: n x d bf16 rows (bench.gen_rows_torch, corpus seed 0), inner product; nq bf16 queries (seed 1). The radius is the one
bench_range.py picks: the median 32nd-best score (knn K = 32) of a seeded sample of 1024 queries over the whole index, so a
query averages about 32 hits over all rows and about 32 p over a subset of a share p. Legs: "device" (a device-resident index)
and "host" (a host-resident index with a 384 MB ring, where the gathered path gathers a subset larger than the ring on the
host). Selectivities 0.9 / 0.5 / 0.25 / 0.1 / 0.01, plus "all rows": the unmasked range search against an all-ones mask, the
cost of the mask itself. Each path gets a fresh index handle per point, so the drop in free device memory over its calls is
the memory that path needed beyond the index (a handle keeps its workspaces until it is closed). Times are host-clock times
of the synchronous host-buffer calls, the calls B200VS makes, query upload and result download included. Per leg, selectivity
and path the script reports queries/s, b2_last_filter_ms, the candidate peak and hits (b2_debug_range_stats), whether both
paths returned identical lims / ids / score bits, and the parity of a head-and-tail sample of --sample queries against the
canonical oracle over x[ids] (lims, ids, score bits). Prints one JSON line with the card's name and power limit. Needs an
H100: there is no CPU path. Writes nothing."""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import bench  # noqa: E402
import oracle  # noqa: E402
from bench_range import card  # noqa: E402
from lotus_b200 import _native as nv  # noqa: E402
from range_oracle import range_search as oracle_range  # noqa: E402

SELECTIVITIES = [0.9, 0.5, 0.25, 0.1, 0.01]


def identical(a, b):
    return bool(np.array_equal(a[0], b[0]) and np.array_equal(a[2], b[2]) and np.array_equal(a[1].view(np.uint32), b[1].view(np.uint32)))


def head_tail(res, h):
    """(lims re-based, D, I) of the first h and the last h queries of a range search result."""
    lims, D, I = res
    nq = len(lims) - 1
    lo, hi = slice(int(lims[0]), int(lims[h])), slice(int(lims[nq - h]), int(lims[nq]))
    counts = np.r_[np.diff(lims[:h + 1]), np.diff(lims[nq - h:])]
    out = np.zeros(2 * h + 1, np.int64)
    np.cumsum(counts, out=out[1:])
    return out, np.r_[D[lo], D[hi]].astype(np.float32), np.r_[I[lo], I[hi]].astype(np.int64)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--n", type=int, default=1_000_000)
    ap.add_argument("--d", type=int, default=768)
    ap.add_argument("--nq", type=int, default=100_000)
    ap.add_argument("--sample", type=int, default=64)
    ap.add_argument("--no-host", action="store_true")
    args = ap.parse_args()
    import torch
    nv.require_device()
    dev = torch.device("cuda", 0)
    n, d, nq = args.n, args.d, args.nq
    x = bench.gen_rows_torch(torch, 0, n, d, 0, dev, torch.bfloat16)
    xh = x.cpu().view(torch.int16).numpy().view(np.uint16)
    qh = bench.gen_rows_torch(torch, 0, nq, d, 1, dev, torch.bfloat16).cpu().view(torch.int16).numpy().view(np.uint16)
    del x
    torch.cuda.empty_cache()

    def free():
        torch.cuda.synchronize()
        return int(torch.cuda.mem_get_info(dev)[0])

    # the oracle's answer for the head-and-tail sample, per selectivity (the same for both legs)
    h = args.sample // 2
    xv = nv.bf16_bits_to_f32(xh) if h else None
    qv = nv.bf16_bits_to_f32(np.r_[qh[:h], qh[nq - h:]]) if h else None
    if h:
        oracle.use_all_cores()
    want = {}

    def parity(res, key, ids):
        if not h:
            return "not measured"
        if key not in want:
            lims, D, pos = oracle_range(xv if ids is None else xv[ids], qv, radius, oracle.IP)
            want[key] = (lims, D, pos if ids is None else ids[pos])
        return identical(head_tail(res, h), want[key])

    pick = np.sort(np.random.default_rng(0).choice(nq, min(1024, nq), replace=False))
    idx0 = nv.Index(xh, nv.BF16, nv.METRIC_IP, 0)
    D32, _ = idx0.search(np.ascontiguousarray(qh[pick]), 32, nv.BF16)
    idx0.close()
    radius = float(np.median(D32[:, 31]))

    def leg(residency):
        kw = {"residency": "host", "ring_bytes": 384 << 20} if residency == "host" else {}
        out = {"residency": residency, "ring_bytes": kw.get("ring_bytes", 0), "selectivity": {}}
        rng = np.random.default_rng(2)
        points = [(p, rng.random(n) < p) for p in SELECTIVITIES] + [("all rows", np.ones(n, bool))]
        for p, mask in points:
            ids = np.flatnonzero(mask)
            words = nv.pack_mask(mask, n)
            # fresh handles per point: the drop in free device memory over a path's calls is what that path needed beyond the
            # index (a handle keeps its workspaces until it is closed)
            idx = {"gathered": nv.Index(xh, nv.BF16, nv.METRIC_IP, 0, **kw), "masked": nv.Index(xh, nv.BF16, nv.METRIC_IP, 0, **kw)}
            if p == "all rows":  # the unmasked range search against an all-ones mask
                call = {"gathered": lambda ix: ix.range_search(qh, radius, nv.BF16),
                        "masked": lambda ix: ix.range_search_masked(qh, radius, nv.BF16, words)}
            else:
                call = {"gathered": lambda ix: ix.range_search(qh, radius, nv.BF16, ids=ids),
                        "masked": lambda ix: ix.range_search_masked(qh, radius, nv.BF16, words)}
            runs = {name: [] for name in idx}
            drop = {name: 0 for name in idx}
            last = {}
            for step in range(args.warmup + args.steps):
                for name, ix in idx.items():
                    before = free()
                    t0 = time.perf_counter()
                    last[name] = call[name](ix)
                    ms = (time.perf_counter() - t0) * 1e3
                    st = ix.range_stats()
                    drop[name] += max(0, before - free())  # only this path's handle allocated in between
                    if step >= args.warmup:
                        runs[name].append({"ms": ms, "filter_ms": ix.last_filter_ms(), **st})
            for ix in idx.values():
                ix.close()
            o = {"rows": int(len(ids)), "hits": int(last["masked"][0][-1]), "identical": identical(last["gathered"], last["masked"]),
                 "oracle_sample": 2 * h, "oracle_parity": parity(last["masked"], str(p), None if p == "all rows" else ids)}
            for name, rs in runs.items():
                ms = float(np.median([r["ms"] for r in rs]))
                o["unmasked" if (p == "all rows" and name == "gathered") else name] = {
                    "queries_per_s": round(nq / (ms * 1e-3)), "search_ms": round(ms, 1),
                    "filter_ms": round(float(np.median([r["filter_ms"] for r in rs])), 1),
                    "candidates_peak": rs[-1]["candidates_peak"], "hits": rs[-1]["hits"], "dense_queries": rs[-1]["dense_queries"],
                    "device_bytes_drop": drop[name], "ms_per_step": [round(r["ms"], 1) for r in rs]}
            out["selectivity"][str(p)] = o
        return out

    res = {"card": card(), "torch_device": torch.cuda.get_device_name(dev), "n": n, "d": d, "nq": nq, "metric": "ip",
           "store": "bf16", "radius": radius, "steps": args.steps, "device": leg("device"),
           "host": "not measured" if args.no_host else leg("host")}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
