"""Host-resident against device-resident indexes on the same rows, on one GPU, timed alternately in one process with CUDA
events so that clock and power drift hit both alike.

    python bench_host_resident.py [--steps 3] [--warmup 1] [--n 1000000] [--d 768] [--chunks 8] [--big-n 0]

Legs (inner product, bench.gen_rows_torch rows, corpus seed 0, queries seed 1):
  bf16: 1M x 768 bf16 rows, 100k bf16 queries, K = 32;
  f32:  1M x 768 fp32 rows, 10k fp32 queries, K = 10 (two levels: bf16 first level streamed from the host copy, tf32 second).
The host-resident index gets a ring that cuts the corpus into at least --chunks chunks. Per leg and residency the script
reports queries/s, the summed filter time, and for the host-resident index the copy time (events on its copy stream), the span
of the streamed pipeline on the search stream, the part of that span not spent in the filter (copies the filter did not hide,
plus the folds), finalize time and the bytes streamed. It asserts that both indexes return identical indices and score bits.
--big-n N adds a host-resident-only bf16 leg over N rows (e.g. 40M: 61 GB pinned) when N rows do not fit in free device memory;
it is skipped, and reported as not measured, when the host lacks the memory. Prints one JSON line with the card's name and
power limit. Needs an H100: there is no CPU path. Writes nothing."""
import argparse
import json
import os
import subprocess

import numpy as np

import bench
from lotus_b200 import _native as nv


def card():
    try:
        return subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception:
        return None


def ring_for(n, d, code, chunks):
    esz = {nv.F32: 4, nv.BF16: 2}[code]
    rows = max(256, (-(-n // chunks)) // 256 * 256)
    ring = 2 * rows * (-(-d * esz // 16) * 16)
    assert nv.stream_plan(n, d, code, ring)["n_chunks"] >= chunks
    return ring


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--n", type=int, default=1_000_000)
    ap.add_argument("--d", type=int, default=768)
    ap.add_argument("--chunks", type=int, default=8)
    ap.add_argument("--big-n", type=int, default=0)
    args = ap.parse_args()
    import torch
    nv.require_device()
    dev = torch.device("cuda", 0)
    n, d = args.n, args.d

    def run(idx, q, code, k):
        out_s = torch.empty((len(q), k), dtype=torch.float32, device=dev)
        out_i = torch.empty((len(q), k), dtype=torch.int64, device=dev)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        nv.stats_reset()
        e0.record()
        idx.search_dev(q.data_ptr(), len(q), k, code, out_s.data_ptr(), out_i.data_ptr(), stream=torch.cuda.current_stream().cuda_stream)
        e1.record()
        torch.cuda.synchronize()
        r = {"ms": e0.elapsed_time(e1), "filter_ms": idx.last_filter_ms(), "stats": nv.stats()}
        if idx.resident == "host":
            r.update(idx.stream_times())
        return r, out_s, out_i

    def leg(code, tdt, nq, k):
        x = bench.gen_rows_torch(torch, 0, n, d, 0, dev, tdt)
        xh = x.cpu().view(torch.int16).numpy().view(np.uint16) if code == nv.BF16 else x.cpu().numpy()
        q = bench.gen_rows_torch(torch, 0, nq, d, 1, dev, tdt)
        ring = ring_for(n, d, code, args.chunks)
        idx = {"device": nv.Index(None, code, nv.METRIC_IP, 0, on_device_ptr=x.data_ptr(), n=n, d=d),
               "host": nv.Index(xh, code, nv.METRIC_IP, 0, residency="host", ring_bytes=ring)}
        torch.cuda.synchronize()
        del x
        torch.cuda.empty_cache()
        runs = {name: [] for name in idx}
        last = {}
        for step in range(args.warmup + args.steps):
            for name, ix in idx.items():
                r, s, i = run(ix, q, code, k)
                if step >= args.warmup:
                    runs[name].append(r)
                last[name] = (s.cpu().numpy(), i.cpu().numpy())
        assert np.array_equal(last["host"][1], last["device"][1]), "host-resident indices differ from the device-resident index"
        assert np.array_equal(last["host"][0].view(np.uint32), last["device"][0].view(np.uint32)), "score bits differ"
        out = {"nq": nq, "k": k, "ring_bytes": ring, "stream_plan": nv.stream_plan(n, d, code, ring), "identical": True}
        for name, rs in runs.items():
            med = lambda key: round(float(np.median([r[key] for r in rs])), 2)  # noqa: E731
            o = {"queries_per_s": round(nq / (med("ms") * 1e-3)), "search_ms": med("ms"), "filter_ms": med("filter_ms"),
                 "fallback_queries": rs[-1]["stats"]["fallback_queries"], "second_level_queries": rs[-1]["stats"]["second_level_queries"],
                 "ms_per_step": [round(r["ms"], 1) for r in rs]}
            if name == "host":
                o.update({"copy_ms": med("copy_ms"), "span_ms": med("span_ms"), "not_filter_in_span_ms": round(med("span_ms") - med("filter_ms"), 2),
                          "finalize_ms": med("finalize_ms"), "streamed_bytes": rs[-1]["stats"]["streamed_bytes"],
                          "streamed_chunks": rs[-1]["stats"]["streamed_chunks"],
                          "copy_gb_per_s": round(rs[-1]["stats"]["streamed_bytes"] / (med("copy_ms") * 1e-3) / 1e9, 1)})
            out[name] = o
        for ix in idx.values():
            ix.close()
        return out

    res = {"card": card(), "torch_device": torch.cuda.get_device_name(dev), "n": n, "d": d, "metric": "ip",
           "bf16": leg(nv.BF16, torch.bfloat16, 100_000, 32),
           "f32": leg(nv.F32, torch.float32, 10_000, 10)}
    big = {"n": args.big_n, "measured": False}
    if args.big_n:
        need = args.big_n * d * 2
        avail = os.sysconf("SC_AVPHYS_PAGES") * os.sysconf("SC_PAGE_SIZE")
        free_dev = torch.cuda.mem_get_info(dev)[0]
        big.update({"host_bytes_needed": need, "host_bytes_available": avail, "device_bytes_free": free_dev})
        if need * 2.2 < avail and need > free_dev:  # the caller's array plus the pinned copy
            xh = np.empty((args.big_n, d), dtype=np.uint16)
            for lo in range(0, args.big_n, 1 << 20):
                hi = min(args.big_n, lo + (1 << 20))
                xh[lo:hi] = bench.gen_rows_torch(torch, lo, hi, d, 0, dev, torch.bfloat16).cpu().view(torch.int16).numpy().view(np.uint16)
            ix = nv.Index(xh, nv.BF16, nv.METRIC_IP, 0, residency="host")
            del xh
            q = bench.gen_rows_torch(torch, 0, 100_000, d, 1, dev, torch.bfloat16)
            run(ix, q, nv.BF16, 32)
            r, _, _ = run(ix, q, nv.BF16, 32)
            big.update({"measured": True, "queries_per_s": round(100_000 / (r["ms"] * 1e-3)), "search_ms": round(r["ms"], 1),
                        "filter_ms": round(r["filter_ms"], 1), "copy_ms": round(r["copy_ms"], 1), "span_ms": round(r["span_ms"], 1),
                        "finalize_ms": round(r["finalize_ms"], 1), "streamed_bytes": r["stats"]["streamed_bytes"]})
            ix.close()
    res["big"] = big
    print(json.dumps(res))


if __name__ == "__main__":
    main()
