"""int8 indexes against bf16 and fp16 on the same integers, on one GPU, timed alternately in one process with CUDA events so
that clock and power drift hit every store alike.

    python bench_i8.py [--steps 5] [--warmup 2] [--n 1000000] [--nq 100000] [--d 768]

Inputs: bench.gen_rows_torch rows (corpus seed 0, queries seed 1), quantized to int8 with one scale per matrix (127 / max|.|,
rounded, clamped), the way quantized embeddings are usually made. The same integers are stored as i8, bf16 and fp16 indexes
(both hold them exactly), and each store is searched with queries of its own type holding the same integers.

Headline leg: 100k queries x 1M x 768, K = 32, inner product. The script asserts that the three stores return identical
indices and score bits, checks a 256-query head-and-tail sample against the oracle, and reports per store queries/s, the
filter kernel's time and rate (2 n d operations per query; int8 against the 1,979 TOPS dense int8 data-sheet rate, the 2-byte
types against 989, both quoted for 700 W), fallbacks, the store's layout bytes and the measured drop in free device memory,
and the card's name and power limit. Second leg: 10k float32 queries (not integral), K = 10, on the i8 store (filtered
against its fp16 copy of the rows) and on the bf16 store. Prints one JSON line. Needs an H100: there is no CPU path. Writes
nothing."""
import argparse
import json
import subprocess
import time

import numpy as np

import bench
from lotus_b200 import _native as nv

PEAK = {"i8": 1979.0, "bf16": 989.0, "f16": 989.0}  # dense data-sheet rates at 700 W (TOPS / TFLOP/s), not measured


def card():
    try:
        return subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception:
        return None


def quant(torch, t):
    return torch.clamp(torch.round(t * (127.0 / t.abs().max())), -128, 127).to(torch.int8)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--n", type=int, default=1_000_000)
    ap.add_argument("--nq", type=int, default=100_000)
    ap.add_argument("--d", type=int, default=768)
    ap.add_argument("--parity-queries", type=int, default=256)
    args = ap.parse_args()
    import torch
    nv.require_device()
    dev = torch.device("cuda", 0)
    n, d = args.n, args.d
    codes = {"i8": (nv.I8, torch.int8, 1), "bf16": (nv.BF16, torch.bfloat16, 2), "f16": (nv.F16, torch.float16, 2)}
    x8 = quant(torch, bench.gen_rows_torch(torch, 0, n, d, 0, dev, torch.float32))
    q8 = quant(torch, bench.gen_rows_torch(torch, 0, args.nq, d, 1, dev, torch.float32))
    idx, mem, layout = {}, {}, {}
    for name, (code, tdt, es) in codes.items():
        src = x8.to(tdt).contiguous()
        torch.cuda.synchronize()
        free0 = torch.cuda.mem_get_info(dev)[0]
        idx[name] = nv.Index(None, code, nv.METRIC_IP, 0, on_device_ptr=src.data_ptr(), n=n, d=d)
        torch.cuda.synchronize()
        mem[name] = int(free0 - torch.cuda.mem_get_info(dev)[0])
        layout[name] = n * d * es  # the copied rows (the filter operand aliases them at d % 16 == 0)
        del src
    torch.cuda.empty_cache()

    def run(name, q, code, k):
        out_s = torch.empty((len(q), k), dtype=torch.float32, device=dev)
        out_i = torch.empty((len(q), k), dtype=torch.int64, device=dev)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        nv.stats_reset()
        e0.record()
        idx[name].search_dev(q.data_ptr(), len(q), k, code, out_s.data_ptr(), out_i.data_ptr(),
                             stream=torch.cuda.current_stream().cuda_stream)
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1), idx[name].last_filter_ms(), nv.stats(), out_s, out_i

    import oracle
    oracle.build()
    oracle.use_all_cores()
    xs = x8.cpu().numpy().astype(np.float32)

    def leg(stores, queries, k, qvals):
        """stores: names; queries[name] = (device tensor, code). Returns per-store results and the last outputs."""
        nq = len(qvals)
        times = {name: [] for name in stores}
        last = {}
        for step in range(args.warmup + args.steps):
            for name in stores:  # alternated: every store sees the same drift
                q, code = queries[name]
                ms, fms, st, s, i = run(name, q, code, k)
                if step >= args.warmup:
                    times[name].append((ms, fms, st))
                last[name] = (s.cpu().numpy(), i.cpu().numpy())
        npar = min(args.parity_queries, nq)
        rows = np.concatenate([np.arange(npar - npar // 2), np.arange(nq - npar // 2, nq)])
        t0 = time.perf_counter()
        Do, Io = oracle.knn(xs, qvals[rows], k, oracle.IP)
        osec = round(time.perf_counter() - t0, 1)
        res = {}
        for name in stores:
            ms = float(np.median([t[0] for t in times[name]]))
            fms = float(np.median([t[1] for t in times[name]]))
            st = times[name][-1][2]
            Dg, Ig = last[name][0][rows], last[name][1][rows]
            ops = 2.0 * nq * n * d / (fms * 1e-3) / 1e12 if fms > 0 else None
            filt = "i8" if name == "i8" and queries[name][1] == nv.I8 else ("f16" if name == "i8" else name)
            res[name] = {"queries_per_s": round(nq / (ms * 1e-3)), "search_ms": round(ms, 2), "filter_ms": round(fms, 2),
                         "filter_tops": round(ops, 1) if ops else None, "filter_operand": filt,
                         "datasheet_peak_700w": PEAK[filt], "filter_share_of_datasheet_peak": round(ops / PEAK[filt], 3) if ops else None,
                         "fallback_queries": st["fallback_queries"],
                         "store_layout_bytes": layout[name], "store_device_bytes_measured": mem[name],
                         "parity": {"queries": int(len(rows)), "idx_bit_exact": bool(np.array_equal(Ig, Io)),
                                    "score_bit_exact": bool(np.array_equal(Dg.view(np.uint32), Do.view(np.uint32))),
                                    "oracle_seconds": osec},
                         "ms_per_step": [round(t[0], 2) for t in times[name]]}
        return res, last

    k = 32
    head, last = leg(["i8", "bf16", "f16"], {name: (q8.to(codes[name][1]).contiguous(), codes[name][0]) for name in codes}, k,
                     q8.cpu().numpy().astype(np.float32))
    ref_s, ref_i = last["i8"]
    for name in ("bf16", "f16"):
        assert np.array_equal(last[name][1], ref_i), f"{name} store: indices differ from the i8 store's"
        assert np.array_equal(last[name][0].view(np.uint32), ref_s.view(np.uint32)), f"{name} store: score bits differ"
    for name, r in head.items():
        assert r["parity"]["idx_bit_exact"] and r["parity"]["score_bit_exact"], f"{name} store: oracle sample differs"
    nq2 = min(10_000, args.nq)
    qf = bench.gen_rows_torch(torch, 0, nq2, d, 2, dev, torch.float32)  # float queries, not integral
    float_leg, _ = leg(["i8", "bf16"], {"i8": (qf, nv.F32), "bf16": (qf, nv.F32)}, 10, qf.cpu().numpy())
    for name, r in float_leg.items():
        assert r["parity"]["idx_bit_exact"] and r["parity"]["score_bit_exact"], f"{name} store, float queries: oracle sample differs"
    out = {"card": card(), "torch_device": torch.cuda.get_device_name(dev), "n": n, "d": d, "metric": "ip",
           "data": "bench.gen_rows_torch rows quantized to int8 (one scale per matrix), stored exactly as i8 / bf16 / f16",
           "headline": {"nq": args.nq, "k": k, "cross_store_identical": True, "stores": head},
           "float_queries": {"nq": nq2, "k": 10, "stores": float_leg},
           "i8_store_f16_copy_bytes": n * (-(-d // 8) * 8) * 2}
    for ix in idx.values():
        ix.close()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
