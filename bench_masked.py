"""Subset search by gathered copy (b2_index_search with ids) against masked search (b2_index_search_masked) on the same rows
and the same strictly ascending random subsets, on one GPU, alternated in one process so that clock and power drift hit both
alike.

    python bench_masked.py [--steps 3] [--warmup 1] [--n 1000000] [--d 768] [--sample 256] [--no-host]

Legs (inner product, bench.gen_rows_torch rows, corpus seed 0, queries seed 1):
  bf16: n x d bf16 rows, 100k bf16 queries, K = 32;
  f32:  n x d fp32 rows, 10k fp32 queries, K = 10 (two levels);
  host: the bf16 leg on a host-resident index with a 384 MB ring, where the gathered path gathers on the host.
Selectivities 0.9 / 0.5 / 0.25 / 0.1 / 0.01. Each path has an index handle of its own, so the drop in free device memory over
its calls is the memory that path needed beyond the index (its workspaces are kept by the handle until it is closed). Times are
host-clock times of the synchronous host-buffer calls, the calls B200VS makes. Per leg, selectivity and path the script reports
queries/s, b2_last_filter_ms, that memory, whether both paths returned identical indices and score bits, and the parity of a
head-and-tail sample of --sample queries against the oracle over x[ids]. Prints one JSON line with the card's name and power
limit. Needs an H100: there is no CPU path. Writes nothing."""
import argparse
import json
import time

import numpy as np

import bench
import oracle
from bench_host_resident import card
from lotus_b200 import _native as nv

SELECTIVITIES = [0.9, 0.5, 0.25, 0.1, 0.01]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--n", type=int, default=1_000_000)
    ap.add_argument("--d", type=int, default=768)
    ap.add_argument("--sample", type=int, default=256)
    ap.add_argument("--no-host", action="store_true")
    args = ap.parse_args()
    import torch
    nv.require_device()
    dev = torch.device("cuda", 0)
    n, d = args.n, args.d

    def free():
        torch.cuda.synchronize()
        return int(torch.cuda.mem_get_info(dev)[0])

    def leg(code, tdt, nq, k, residency):
        x = bench.gen_rows_torch(torch, 0, n, d, 0, dev, tdt)
        q = bench.gen_rows_torch(torch, 0, nq, d, 1, dev, tdt)
        if code == nv.BF16:
            xh = x.cpu().view(torch.int16).numpy().view(np.uint16)
            qh = q.cpu().view(torch.int16).numpy().view(np.uint16)
        else:
            xh, qh = x.cpu().numpy(), q.cpu().numpy()
        del x, q
        torch.cuda.empty_cache()
        kw = {"residency": "host", "ring_bytes": 384 << 20} if residency == "host" else {}
        idx = {"gathered": nv.Index(xh, code, nv.METRIC_IP, 0, **kw), "masked": nv.Index(xh, code, nv.METRIC_IP, 0, **kw)}
        xf = nv.stored_to_f32(xh, code) if args.sample else None
        qf = nv.stored_to_f32(qh, code)
        base = free()
        low = {name: base for name in idx}
        out = {"nq": nq, "k": k, "residency": residency, "selectivity": {}}
        rng = np.random.default_rng(2)
        for p in SELECTIVITIES:
            mask = rng.random(n) < p
            ids = np.flatnonzero(mask)
            words = nv.pack_mask(mask, n)
            call = {"gathered": lambda ix: ix.search(qh, k, code, ids=ids), "masked": lambda ix: ix.search_masked(qh, k, code, words)}
            runs = {name: [] for name in idx}
            last = {}
            for step in range(args.warmup + args.steps):
                for name, ix in idx.items():
                    before = free()
                    t0 = time.perf_counter()
                    last[name] = call[name](ix)
                    ms = (time.perf_counter() - t0) * 1e3
                    after = free()
                    low[name] -= max(0, before - after)  # only this path's handle allocated in between
                    if step >= args.warmup:
                        runs[name].append({"ms": ms, "filter_ms": ix.last_filter_ms()})
            same = bool(np.array_equal(last["gathered"][1], last["masked"][1])
                        and np.array_equal(last["gathered"][0].view(np.uint32), last["masked"][0].view(np.uint32)))
            o = {"rows": int(len(ids)), "identical": same}
            if args.sample:
                h = args.sample // 2
                sel = np.r_[0:h, nq - h:nq]
                Do, Io = oracle.knn_subset(xf, qf[sel], k, ids, oracle.IP)
                o["oracle_sample"] = len(sel)
                o["oracle_parity"] = bool(np.array_equal(last["masked"][1][sel], Io)
                                          and np.array_equal(last["masked"][0][sel].view(np.uint32), Do.view(np.uint32)))
            else:
                o["oracle_parity"] = "not measured"
            for name, rs in runs.items():
                ms = float(np.median([r["ms"] for r in rs]))
                o[name] = {"queries_per_s": round(nq / (ms * 1e-3)), "search_ms": round(ms, 1),
                           "filter_ms": round(float(np.median([r["filter_ms"] for r in rs])), 1),
                           "ms_per_step": [round(r["ms"], 1) for r in rs]}
            out["selectivity"][str(p)] = o
        out["extra_device_bytes"] = {name: base - low[name] for name in idx}
        for ix in idx.values():
            ix.close()
        return out

    res = {"card": card(), "torch_device": torch.cuda.get_device_name(dev), "n": n, "d": d, "metric": "ip", "steps": args.steps,
           "bf16": leg(nv.BF16, torch.bfloat16, 100_000, 32, "device"),
           "f32": leg(nv.F32, torch.float32, 10_000, 10, "device"),
           "host": "not measured" if args.no_host else leg(nv.BF16, torch.bfloat16, 100_000, 32, "host")}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
