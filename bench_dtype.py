"""Store element types side by side on one GPU: fp16 (B2_F16), bf16 and fp32 indexes over the same corpus, timed alternately in
one process with CUDA events, so clock and power drift hit every store alike.

    python bench_dtype.py [--steps 5] [--warmup 2] [--n 1000000] [--nq 100000]

Headline shape: 100k queries x 1M x 768 rows (bench.gen_rows_torch: N(0,1), L2-normalised), K = 32, inner product, every
store searched with queries of its own type. C2-like shape: 10k queries, K = 10, fp16 against fp32 (fp32 queries on the fp32
store, which searches two-level: a bf16 first level, then tf32 for what it cannot certify). Per store it reports queries/s,
the filter kernel's time and TFLOP/s (2 n d per query), the fallback and second-level counts, the device bytes of the store
(layout, and the measured change of free device memory when it was built), a 256-query head-and-tail parity check against
the oracle on the store's exact values, and the card's name and power limit. Prints one JSON line. Needs an H100: there is
no CPU path. Writes nothing."""
import argparse
import json
import subprocess
import time

import numpy as np

import bench
from lotus_b200 import _native as nv


def card():
    try:
        return subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception:
        return None


def host_values(t, code):
    """float32 host copy of the exact values of a device tensor stored as element type `code`."""
    import torch
    a = t.cpu()
    return nv.stored_to_f32(a.view(torch.int16).numpy().view(np.uint16) if code == nv.BF16 else a.numpy(), code)


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
    codes = {"f16": (nv.F16, torch.float16), "bf16": (nv.BF16, torch.bfloat16), "f32": (nv.F32, torch.float32)}
    corpus32 = bench.gen_rows_torch(torch, 0, n, d, 0, dev, torch.float32)
    q32 = bench.gen_rows_torch(torch, 0, args.nq, d, 1, dev, torch.float32)
    idx, mem, layout = {}, {}, {}
    for name, (code, tdt) in codes.items():
        src = corpus32.to(tdt).contiguous()
        torch.cuda.synchronize()
        free0 = torch.cuda.mem_get_info(dev)[0]
        idx[name] = nv.Index(None, code, nv.METRIC_IP, 0, on_device_ptr=src.data_ptr(), n=n, d=d)
        torch.cuda.synchronize()
        mem[name] = int(free0 - torch.cuda.mem_get_info(dev)[0])
        # the copied rows, plus the bf16 first-level copy an fp32 store keeps (filter copies alias the rows at d % 8 == 0)
        layout[name] = n * d * (4 if code == nv.F32 else 2) + (n * (-(-d // 8) * 8) * 2 if code == nv.F32 else 0)
        del src
    torch.cuda.empty_cache()

    def run(name, q, k):
        code = codes[name][0]
        out_s = torch.empty((len(q), k), dtype=torch.float32, device=dev)
        out_i = torch.empty((len(q), k), dtype=torch.int64, device=dev)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        nv.stats_reset()
        e0.record()
        idx[name].search_dev(q.data_ptr(), len(q), k, code, out_s.data_ptr(), out_i.data_ptr(),
                             stream=torch.cuda.current_stream().cuda_stream)
        e1.record()
        torch.cuda.synchronize()
        st = nv.stats()
        return e0.elapsed_time(e1), idx[name].last_filter_ms(), st, out_s, out_i

    def shape(stores, nq, k):
        qs = {name: q32[:nq].to(codes[name][1]).contiguous() for name in stores}
        times = {name: [] for name in stores}
        last = {}
        for step in range(args.warmup + args.steps):
            for name in stores:  # alternated: every store sees the same drift
                ms, fms, st, s, i = run(name, qs[name], k)
                if step >= args.warmup:
                    times[name].append((ms, fms, st))
                last[name] = (s, i)
        res = {}
        import oracle
        oracle.build()
        oracle.use_all_cores()
        npar = min(args.parity_queries, nq)
        rows = np.concatenate([np.arange(npar - npar // 2), np.arange(nq - npar // 2, nq)])
        for name in stores:
            ms = float(np.median([t[0] for t in times[name]]))
            fms = float(np.median([t[1] for t in times[name]]))
            st = times[name][-1][2]
            code, tdt = codes[name]
            xs = host_values(corpus32.to(tdt), code)
            qv = host_values(qs[name][torch.from_numpy(rows).to(dev)], code)
            t0 = time.perf_counter()
            Do, Io = oracle.knn(xs, qv, k, oracle.IP)
            s, i = last[name]
            Dg, Ig = s[torch.from_numpy(rows).to(dev)].cpu().numpy(), i[torch.from_numpy(rows).to(dev)].cpu().numpy()
            res[name] = {"queries_per_s": round(nq / (ms * 1e-3)), "search_ms": round(ms, 2), "filter_ms": round(fms, 2),
                         "filter_tflops": round(2.0 * nq * n * d / (fms * 1e-3) / 1e12, 1) if fms > 0 else None,
                         "fallback_queries": st["fallback_queries"], "second_level_queries": st["second_level_queries"],
                         "store_layout_bytes": layout[name], "store_device_bytes_measured": mem[name],
                         "parity": {"queries": int(len(rows)), "idx_bit_exact": bool(np.array_equal(Ig, Io)),
                                    "score_bit_exact": bool(np.array_equal(Dg.view(np.uint32), Do.view(np.uint32))),
                                    "oracle_seconds": round(time.perf_counter() - t0, 1)},
                         "ms_per_step": [round(t[0], 2) for t in times[name]]}
            del xs
        return res

    out = {"card": card(), "torch_device": torch.cuda.get_device_name(dev), "n": n, "d": d, "metric": "ip",
           "queries": "bench.gen_rows_torch seed 1, each store searched with queries of its own type (device buffers, search_dev)",
           "headline": {"nq": args.nq, "k": 32, "stores": shape(["f16", "bf16", "f32"], args.nq, 32)},
           "c2_like": {"nq": min(10_000, args.nq), "k": 10, "stores": shape(["f16", "f32"], min(10_000, args.nq), 10)}}
    for ix in idx.values():
        ix.close()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
