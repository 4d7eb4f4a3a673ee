"""Range search against knn K = 32 on the same store, on one GPU, timed alternately in one process so that clock and power
drift hit both alike.

    python bench_range.py [--steps 3] [--warmup 1] [--n 1000000] [--d 768] [--nq 100000] [--host-chunks 0]

Store: n x d bf16 rows (bench.gen_rows_torch, corpus seed 0), inner product; nq bf16 queries (seed 1). The radius is chosen
deterministically so that queries average about 32 hits: the median 32nd-best score (knn K = 32) of a seeded sample of 1024
queries. Both calls take host queries and return host results (b2_index_range_search / b2_index_search), so both include the
query upload and the result download. Per call the script reports queries/s and wall ms; for the range search also the filter
time and its TFLOP/s (2 nq n d / filter time), candidates against hits, the peak candidate-buffer size, and the time not spent
in the filter (thresholds, verification, assembly and the copies). 256 head and 256 tail queries are checked against the
canonical oracle: lims, ids and score bits. --host-chunks C > 0 adds a host-resident index whose ring cuts the corpus into at
least C chunks; its result must equal the device-resident one. Prints one JSON line with the card's name and power limit.
Needs an H100: there is no CPU path. Writes nothing."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import bench  # noqa: E402
import oracle  # noqa: E402
from lotus_b200 import _native as nv  # noqa: E402
from range_oracle import range_search as oracle_range  # noqa: E402


def card():
    try:
        return subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception:
        return None


def timed(fn):
    t0 = time.perf_counter()
    out = fn()
    return out, (time.perf_counter() - t0) * 1e3


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--n", type=int, default=1_000_000)
    ap.add_argument("--d", type=int, default=768)
    ap.add_argument("--nq", type=int, default=100_000)
    ap.add_argument("--host-chunks", type=int, default=0)
    args = ap.parse_args()
    import torch
    nv.require_device()
    dev = torch.device("cuda", 0)
    n, d, nq = args.n, args.d, args.nq
    x = bench.gen_rows_torch(torch, 0, n, d, 0, dev, torch.bfloat16)
    xh = x.cpu().view(torch.int16).numpy().view(np.uint16)
    q = bench.gen_rows_torch(torch, 0, nq, d, 1, dev, torch.bfloat16).cpu().view(torch.int16).numpy().view(np.uint16)
    idx = nv.Index(None, nv.BF16, nv.METRIC_IP, 0, on_device_ptr=x.data_ptr(), n=n, d=d)
    torch.cuda.synchronize()
    del x
    torch.cuda.empty_cache()

    sample = np.sort(np.random.default_rng(0).choice(nq, min(1024, nq), replace=False))
    D32, _ = idx.search(np.ascontiguousarray(q[sample]), 32, nv.BF16)
    radius = float(np.median(D32[:, 31]))

    rs, ks = [], []
    for step in range(args.warmup + args.steps):
        (res, ms) = timed(lambda: idx.range_search(q, radius, nv.BF16))
        st = idx.range_stats()
        rec = {"ms": ms, "filter_ms": idx.last_filter_ms(), **st}
        _, kms = timed(lambda: idx.search(q, 32, nv.BF16))
        if step >= args.warmup:
            rs.append(rec)
            ks.append(kms)
    lims, D, I = res
    med = lambda key: float(np.median([r[key] for r in rs]))  # noqa: E731
    range_ms, filter_ms, knn_ms = med("ms"), med("filter_ms"), float(np.median(ks))
    out = {"card": card(), "torch_device": torch.cuda.get_device_name(dev), "n": n, "d": d, "nq": nq, "metric": "ip",
           "store": "bf16", "radius": radius, "mean_hits": round(float(lims[-1]) / nq, 2),
           "range": {"queries_per_s": round(nq / (range_ms * 1e-3)), "ms": round(range_ms, 1), "filter_ms": round(filter_ms, 2),
                     "filter_tflops": round(2.0 * nq * n * d / (filter_ms * 1e-3) / 1e12, 1),
                     "not_filter_ms": round(range_ms - filter_ms, 1), "candidates": rs[-1]["candidates_peak"],
                     "hits": rs[-1]["hits"], "peak_candidate_buffer": rs[-1]["candidates_peak"],
                     "dense_queries": rs[-1]["dense_queries"], "ms_per_step": [round(r["ms"], 1) for r in rs]},
           "knn32": {"queries_per_s": round(nq / (knn_ms * 1e-3)), "ms": round(knn_ms, 1), "ms_per_step": [round(v, 1) for v in ks]},
           "range_over_knn_time": round(range_ms / knn_ms, 3)}

    # parity: head and tail of the batch against the canonical oracle (lims, ids, score bits)
    oracle.use_all_cores()
    xv = nv.bf16_bits_to_f32(xh)
    parity = True
    for lo, hi in [(0, min(256, nq)), (max(0, nq - 256), nq)]:
        qv = nv.bf16_bits_to_f32(q[lo:hi])
        for a in range(lo, hi, 64):
            b = min(hi, a + 64)
            wl, wd, wi = oracle_range(xv, qv[a - lo:b - lo], radius, oracle.IP)
            gl = lims[a:b + 1] - lims[a]
            gd, gi = D[lims[a]:lims[b]], I[lims[a]:lims[b]]
            parity &= np.array_equal(gl, wl) and np.array_equal(gi, wi) and np.array_equal(gd.view(np.uint32), wd.view(np.uint32))
    out["parity_512_queries"] = bool(parity)

    host = {"measured": False}
    if args.host_chunks > 0:
        rows = max(256, (-(-n // args.host_chunks)) // 256 * 256)
        ring = 2 * rows * (-(-d * 2 // 16) * 16)
        plan = nv.stream_plan(n, d, nv.BF16, ring)
        hidx = nv.Index(xh, nv.BF16, nv.METRIC_IP, 0, residency="host", ring_bytes=ring)
        hidx.range_search(q, radius, nv.BF16)
        (hres, hms) = timed(lambda: hidx.range_search(q, radius, nv.BF16))
        same = all(np.array_equal(a.view(np.uint32) if a.dtype == np.float32 else a, b.view(np.uint32) if b.dtype == np.float32 else b)
                   for a, b in zip(hres, res))
        host = {"measured": True, "stream_plan": plan, "queries_per_s": round(nq / (hms * 1e-3)), "ms": round(hms, 1),
                "filter_ms": round(hidx.last_filter_ms(), 2), "identical_to_device": bool(same)}
        hidx.close()
    out["host_resident"] = host
    idx.close()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
