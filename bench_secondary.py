"""The secondary BASELINE.json configurations behind `bench.py --config c2|c4|c5` — same launch contract as the headline
(`python bench.py --config cX --gpus N --steps K --warmup W`, torchrun for N > 1, one JSON line from rank 0 with metric / value /
unit / roofline / cpu_baseline / parity / e2e / clocks):

  c2  sem_search over a 1M x 768 fp32 index, 10k queries, top-10 (TF32 wgmma filter + exact fp32 re-score); index row-sharded at N > 1
  c4  sem_dedup relation, 10M rows x 384-d bf16, cosine > 0.95, 1 % planted near-duplicates; corpus replicated, the upper-triangular
      tile grid dealt over max(N, --dedup-parts) parts (at N = 1 the default times ONE rank's share of the 8-GPU split)
  c5  sem_cluster_by k-means, 5M x 768 bf16, k = 1024, 20 Lloyd iterations + final assignment; points row-sharded at N > 1
"""
from __future__ import annotations

import argparse
import json
import os
import sys
import time

import numpy as np

import bench


def _peaks():
    # H100 SXM data sheet at 700 W (not measured): dense bf16 TFLOP/s and HBM3 GB/s
    return {"bf16_tflops": 989.0, "hbm_gbs": 3350.0}


class Ctx:
    def __init__(self, args):
        import torch
        import torch.distributed as dist
        self.torch, self.dist = torch, dist
        self.world, self.rank, self.local = bench.env_int("WORLD_SIZE", 1), bench.env_int("RANK", 0), bench.env_int("LOCAL_RANK", 0)
        torch.cuda.set_device(self.local)
        self.dev = torch.device("cuda", self.local)
        if self.world > 1:
            os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
            if os.environ.get("NCCL_DEBUG", "").upper() in ("", "VERSION"):
                os.environ["NCCL_DEBUG"] = "WARN"
            dist.init_process_group("nccl", device_id=self.dev)
        self.args = args

    def barrier(self):
        if self.world > 1:
            self.dist.barrier()
        self.torch.cuda.synchronize()

    def max_over_ranks(self, v: float) -> float:
        if self.world == 1:
            return v
        t = self.torch.tensor([v], device=self.dev, dtype=self.torch.float64)
        self.dist.all_reduce(t, op=self.dist.ReduceOp.MAX)
        return float(t.item())

    def timed_wall(self, fn, steps: int) -> float:
        """ms per step of a SYNCHRONOUS host-API call (the library returns when the result is complete), max over ranks."""
        self.barrier()
        t0 = time.perf_counter()
        for _ in range(steps):
            fn()
        self.torch.cuda.synchronize()
        ms = (time.perf_counter() - t0) / steps * 1e3
        return self.max_over_ranks(ms)

    def finish(self, line: dict | None):
        if self.rank == 0 and line is not None:
            print(json.dumps(line), flush=True)
        if self.world > 1:
            self.dist.barrier()
            self.dist.destroy_process_group()


def _base(ctx: Ctx, metric: str, value: float, unit: str, ms: float, hib: bool, dtype: str, workload: dict, scaling: str) -> dict:
    a = ctx.args
    return {"metric": metric, "value": value, "unit": unit, "n_gpus": ctx.world, "steps": a.steps, "warmup": a.warmup, "ms_per_step": ms,
            "higher_is_better": hib, "scaling": scaling, "vs_baseline": None, "dtype": dtype, "data": "synthetic", "config": workload}


# ---- C2 ---------------------------------------------------------------------------------------------------------------------------
def c2(ctx: Ctx, extra):
    import oracle
    from lotus_b200 import _native as nv
    from lotus_b200.distributed import ShardedIndex, shard_bounds
    torch, dev = ctx.torch, ctx.dev
    ap = argparse.ArgumentParser()
    ap.add_argument("--c2-n", type=int, default=1_000_000)
    ap.add_argument("--c2-nq", type=int, default=10_000)
    o, _ = ap.parse_known_args(extra)
    n, d, nq, k = o.c2_n, 768, o.c2_nq, 10
    lo, hi = shard_bounds(n, ctx.world, ctx.rank)
    x = bench.gen_rows_torch(torch, lo, hi, d, 0, dev, torch.float32)
    q = bench.gen_rows_torch(torch, 0, nq, d, 1, dev, torch.float32)
    index = ShardedIndex(x, lo, nv.METRIC_IP)
    fms = []

    def step():
        index.search(q, k)
        fms.append(index.last_filter_ms())

    for _ in range(ctx.args.warmup):
        step()
    fms.clear()
    nv.stats_reset()
    sampler = bench.ClockSampler(ctx.local) if ctx.rank == 0 else None
    if sampler:
        sampler.start()
    ctx.barrier()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(ctx.args.steps):
        step()
    e1.record()
    torch.cuda.synchronize()
    ms = ctx.max_over_ranks(e0.elapsed_time(e1) / ctx.args.steps)
    clocks = sampler.stop() if sampler else None
    st = nv.stats()
    kms = float(np.mean(fms))
    # e2e: pinned host queries in, host result out
    q_host = q.cpu().pin_memory()
    os_h, oi_h = torch.empty((nq, k), dtype=torch.float32).pin_memory(), torch.empty((nq, k), dtype=torch.int64).pin_memory()
    if ctx.world == 1:
        qn = q_host.numpy()
        index.index.search(qn, k, nv.F32)
        ms_e2e = ctx.timed_wall(lambda: index.index.search(qn, k, nv.F32), ctx.args.steps)
        api = "b2_index_search (host buffers)"
    else:
        index.search_host(q_host, k, os_h if ctx.rank == 0 else None, oi_h if ctx.rank == 0 else None)
        ms_e2e = ctx.timed_wall(lambda: index.search_host(q_host, k, os_h if ctx.rank == 0 else None, oi_h if ctx.rank == 0 else None), ctx.args.steps)
        api = "ShardedIndex.search_host"
    npar = min(256, nq)
    s_par, i_par = index.search(q[:npar].contiguous(), k)
    line = None
    if ctx.rank == 0:
        oracle.build()
        oracle.use_all_cores()
        xs = (x if ctx.world == 1 else bench.gen_rows_torch(torch, 0, n, d, 0, dev, torch.float32)).cpu().numpy()
        Do, Io = oracle.knn(xs, q[:npar].cpu().numpy(), k, oracle.IP)
        Ig, Dg = i_par.cpu().numpy(), s_par.cpu().numpy()
        parity = {"queries": npar, "oracle": bench.faiss_probe()["oracle"], "idx_bit_exact_vs_oracle": bool(np.array_equal(Ig, Io)),
                  "score_bit_exact_vs_oracle": bool(np.array_equal(Dg.view(np.uint32), Do.view(np.uint32)))}
        cpu = None
        if ctx.world == 1 and not ctx.args.no_cpu_baseline:
            cpu = bench.cpu_arms(xs, q[:min(8192, nq)].cpu().numpy(), k, ctx.args.cpu_sample, 10.0)
            for key in ("_sample", "_I", "_D"):
                cpu.pop(key, None)
        pk = _peaks()
        peak = pk["bf16_tflops"] / 2.0
        fl = 2.0 * nq * (hi - lo) * d
        line = _base(ctx, "sem_search queries/sec (1M x 768 fp32, top-10)", nq / ms * 1e3, "queries/s", ms, True, "f32 (tf32 filter, exact fp32 re-score)",
                     {"workload": f"sem_search {nq} queries x {n} index, {d}-d fp32, K={k} (BASELINE.json configs[1])", "nq": nq, "n": n, "d": d, "k": k,
                      "parallelism": f"index row-sharded x{ctx.world}", "l2_policy": "inputs exceed L2 (corpus shard %.0f MB)" % ((hi - lo) * d * 4 / 1e6)},
                     "strong")
        line.update({"e2e": {"value": nq / ms_e2e * 1e3, "unit": "queries/s", "ms_per_step": ms_e2e, "h2d_bytes_per_step": nq * d * 4 // ctx.world,
                             "d2h_bytes_per_step": nq * k * 12, "api": api},
                     "gpu_launches": int(st["launches"]), "fallback_queries": int(st["fallback_queries"]),
                     "roofline": {"bound": "tensor", "achieved": fl / kms / 1e9, "peak": peak, "unit": "TFLOP/s", "frac": fl / kms / 1e9 / peak, "traffic": None,
                                  "kernel": "knn_filter_kernel<KP=32,IP,tf32,CTA pair>", "kernel_ms": kms,
                                  "peak_source": "H100 SXM data-sheet dense tf32 rate (half the bf16 rate; not measured)"},
                     "cpu_baseline": cpu, "parity": parity, "clocks": clocks})
    index.close()
    ctx.finish(line)


# ---- C4 ---------------------------------------------------------------------------------------------------------------------------
def c4(ctx: Ctx, extra):
    import oracle
    from lotus_b200 import _native as nv
    from lotus_b200.distributed import sharded_threshold_pairs
    torch, dev = ctx.torch, ctx.dev
    ap = argparse.ArgumentParser()
    ap.add_argument("--c4-n", type=int, default=10_000_000)
    ap.add_argument("--dedup-parts", type=int, default=8, help="at N = 1: time one rank's share of this many parts (8 = the 8-GPU split)")
    o, _ = ap.parse_known_args(extra)
    n, d, tau = o.c4_n, 384, 0.95
    x = bench.gen_rows_torch(torch, 0, n, d, 2, dev, torch.float32)
    g = torch.Generator(device=dev)
    g.manual_seed(22)
    m = n // 100
    src = torch.randint(0, n, (m,), generator=g, device=dev)
    dst = torch.randperm(n, generator=g, device=dev)[:m]
    x[dst] = x[src] + torch.randn((m, d), generator=g, device=dev) * (0.1 / d ** 0.5)
    x = (x / x.norm(dim=1, keepdim=True)).to(torch.bfloat16).contiguous()
    idx = nv.Index(None, nv.BF16, nv.METRIC_IP, ctx.local, on_device_ptr=x.data_ptr(), n=n, d=d)
    if ctx.world > 1:
        part, nparts = ctx.rank, ctx.world
        run = lambda: sharded_threshold_pairs(idx, tau)  # noqa: E731
    else:
        part, nparts = 0, max(1, o.dedup_parts)
        run = lambda: idx.threshold_pairs(tau, part=part, nparts=nparts)  # noqa: E731
    for _ in range(ctx.args.warmup if n <= 2_000_000 else 1):  # a 10M-row pass takes seconds: one warm-up pass
        run()
    nv.stats_reset()
    sampler = bench.ClockSampler(ctx.local) if ctx.rank == 0 else None
    if sampler:
        sampler.start()
    ms = ctx.timed_wall(run, ctx.args.steps)
    clocks = sampler.stop() if sampler else None
    st = nv.stats()
    pi, pj = run()
    line = None
    if ctx.rank == 0:
        oracle.build()
        lab = nv.connected_components(n, pi, pj, ctx.local) if ctx.world > 1 or nparts == 1 else None
        # parity: (a) the relation restricted to the first 3000 rows equals the oracle's (canonical scores, strict >) on the tiles this
        # result covers; (b) size-independent properties at full size: i < j, sorted unique, every returned pair above tau when
        # recomputed in fp64, every planted pair above tau present
        sub = 3000
        oi, oj, _ = oracle.threshold_pairs(x[:sub].float().cpu().numpy(), tau)
        if ctx.world == 1 and nparts > 1:
            mine = nv.pair_owner(oi, nparts) == part
            oi, oj = oi[mine], oj[mine]
        keep = (pi < sub) & (pj < sub)
        slice_ok = bool(np.array_equal(pi[keep], oi) and np.array_equal(pj[keep], oj))
        key = pi.astype(np.uint64) << np.uint64(32) | pj.astype(np.uint64)
        shape_ok = bool((pi < pj).all() and (np.diff(key.astype(np.int64)) > 0).all())
        tpi, tpj = torch.from_numpy(pi).to(dev), torch.from_numpy(pj).to(dev)
        sc = torch.empty(len(pi), dtype=torch.float64, device=dev)
        for s in range(0, len(pi), 1 << 18):
            e = min(len(pi), s + (1 << 18))
            sc[s:e] = (x[tpi[s:e]].double() * x[tpj[s:e]].double()).sum(1)
        all_above = bool((sc.float() > tau).all()) if len(pi) else True
        lo_, hi_ = torch.minimum(src, dst), torch.maximum(src, dst)
        spl = torch.empty(m, dtype=torch.float64, device=dev)
        for s in range(0, m, 1 << 18):
            e = min(m, s + (1 << 18))
            spl[s:e] = (x[lo_[s:e]].double() * x[hi_[s:e]].double()).sum(1)
        want = (spl.float() > tau) & (lo_ != hi_)
        if ctx.world == 1 and nparts > 1:
            want &= torch.from_numpy(nv.pair_owner(lo_.cpu().numpy(), nparts)).to(dev) == part
        wkey = (lo_[want].cpu().numpy().astype(np.uint64) << np.uint64(32)) | hi_[want].cpu().numpy().astype(np.uint64)
        parity = {"slice_relation_exact_vs_oracle_first_3000_rows": slice_ok, "pairs_sorted_unique_upper_triangle": shape_ok,
                  "all_returned_pairs_above_tau_fp64": all_above, "planted_pairs_expected": int(want.sum()),
                  "planted_pairs_all_found": bool(np.isin(wkey, key).all()), "pairs": int(len(pi)),
                  "rows_removed_by_dedup": int((lab != np.arange(n)).sum()) if lab is not None else None}
        # CPU arm: the oracle's canonical all-pairs scan on a bounded sample of rows, extrapolated quadratically (an ESTIMATE)
        cpu = None
        if not ctx.args.no_cpu_baseline:
            oracle.use_all_cores()
            ns = 20_000
            xs = x[:ns].float().cpu().numpy()
            t0 = time.perf_counter()
            oracle.knn_tiled(xs, xs, 2, oracle.IP)  # all-pairs scores of the sample through the timed fp32 port (top-2 heap = negligible)
            dt = time.perf_counter() - t0
            share = (1.0 / nparts) if ctx.world == 1 else 1.0
            est = dt * (float(n) / ns) ** 2 / 2 * share  # symmetric half
            cpu = {"value": est, "unit": "s", "cores": oracle.num_threads(), "kind": "port",
                   "sample": f"{ns} x {ns} x {d} all-pairs scores in {dt:.2f} s (orc_knn_tiled, -march=native), scaled by (n/ns)^2/2"
                             f"{' x this share' if share < 1 else ''}: an ESTIMATE — the reference materialises an N^2-row DataFrame (sem_dedup.py:45) and cannot run at this size"}
        pk = _peaks()
        peak = pk["bf16_tflops"]
        fl = float(n) * (n - 1) / 2 * 2 * d / (nparts if ctx.world == 1 else ctx.world)
        share_txt = f"one rank's share (part 0 of {nparts})" if ctx.world == 1 and nparts > 1 else f"tile grid dealt over {ctx.world} ranks"
        line = _base(ctx, "sem_dedup seconds (10M x 384, cosine > 0.95)", ms / 1e3, "s", ms, False, "bf16",
                     {"workload": f"sem_dedup relation, {n} rows x {d}-d bf16, tau={tau}, 1 % planted near-duplicates (BASELINE.json configs[3]); {share_txt}",
                      "n": n, "d": d, "tau": tau, "parallelism": share_txt, "l2_policy": "corpus %.0f MB exceeds L2" % (n * d * 2 / 1e6)},
                     "strong")
        line.update({"e2e": {"value": ms / 1e3, "unit": "s", "ms_per_step": ms, "h2d_bytes_per_step": 0, "d2h_bytes_per_step": int(len(pi)) * 16,
                             "api": "b2_threshold_pairs (corpus resident in the index handle; sorted verified pair list returned in HOST buffers"
                                    + ("; + all-gather of the per-rank lists)" if ctx.world > 1 else ")")},
                     "gpu_launches": int(st["launches"]),
                     "roofline": {"bound": "tensor", "achieved": fl / ms / 1e9, "peak": peak, "unit": "TFLOP/s", "frac": fl / ms / 1e9 / peak, "traffic": None,
                                  "kernel": "pair_filter_kernel<bf16,CTA pair>", "kernel_ms": ms,
                                  "note": "whole call timed (filter + verify + sort + D2H): the filter kernel is > 95 % of it; symmetric FLOP count N(N-1)/2*2d"},
                     "cpu_baseline": cpu, "parity": parity, "clocks": clocks})
    idx.close()
    ctx.finish(line)


# ---- C5 ---------------------------------------------------------------------------------------------------------------------------
def c5(ctx: Ctx, extra):
    import oracle
    from lotus_b200 import _native as nv
    from lotus_b200.distributed import shard_bounds, sharded_kmeans
    torch, dev = ctx.torch, ctx.dev
    ap = argparse.ArgumentParser()
    ap.add_argument("--c5-n", type=int, default=5_000_000)
    ap.add_argument("--c5-k", type=int, default=1024)
    ap.add_argument("--c5-niter", type=int, default=20)
    ap.add_argument("--c5-mode", default="full", choices=["full", "parity"], help="full Lloyd over all points, or faiss's 256*k subsample (N = 1 only)")
    o, _ = ap.parse_known_args(extra)
    n, d, k, niter = o.c5_n, 768, o.c5_k, o.c5_niter
    lo, hi = shard_bounds(n, ctx.world, ctx.rank)
    g = torch.Generator(device=dev)
    g.manual_seed(3)
    centers = torch.randn((k, d), generator=g, device=dev)
    x = torch.empty((hi - lo, d), dtype=torch.bfloat16, device=dev)
    for b in range(lo // bench.BLOCK_ROWS, (hi - 1) // bench.BLOCK_ROWS + 1):  # same matrix for every world size
        gb = torch.Generator(device=dev)
        gb.manual_seed(3_000_003 + b)
        lab = torch.randint(0, k, (bench.BLOCK_ROWS,), generator=gb, device=dev)
        blk = (centers[lab] + 0.5 * torch.randn((bench.BLOCK_ROWS, d), generator=gb, device=dev)).to(torch.bfloat16)
        s, e = max(lo, b * bench.BLOCK_ROWS), min(hi, (b + 1) * bench.BLOCK_ROWS)
        x[s - lo:e - lo] = blk[s - b * bench.BLOCK_ROWS:e - b * bench.BLOCK_ROWS]
    idx = nv.Index(None, nv.BF16, nv.METRIC_L2, ctx.local, on_device_ptr=x.data_ptr(), n=hi - lo, d=d)
    full = o.c5_mode == "full" or ctx.world > 1
    res = {}

    def run():
        if ctx.world > 1:
            res["a"], res["c"], res["obj"] = sharded_kmeans(idx, n, lo, k, niter=niter, want_obj=True)
        else:
            res["a"], res["c"], res["obj"] = idx.kmeans(k, niter=niter, full_lloyd=full)

    for _ in range(min(ctx.args.warmup, 3)):
        run()
    nv.stats_reset()
    sampler = bench.ClockSampler(ctx.local) if ctx.rank == 0 else None
    if sampler:
        sampler.start()
    ms = ctx.timed_wall(run, ctx.args.steps)
    clocks = sampler.stop() if sampler else None
    st = nv.stats()
    a, c, obj = res["a"], res["c"], res["obj"]
    # size-independent properties at full size: the returned assignment is a fixed point of the assignment against the returned
    # centroids (kmeans.index.search(x, 1), utils.py:65) and equals the fp64 argmin on a sample with a clear winner
    a2, _ = idx.kmeans_assign(c)
    idem = bool(np.array_equal(a, a2))
    smp = torch.arange(0, hi - lo, max(1, (hi - lo) // 4096), device=dev)[:4096]
    dd = torch.cdist(x[smp].double(), torch.from_numpy(c).to(dev).double())
    srt = dd.topk(2, dim=1, largest=False)
    clear = ((srt.values[:, 1] - srt.values[:, 0]) > 1e-6 * srt.values[:, 1]).cpu().numpy()
    amin_ok = bool((srt.indices[:, 0].cpu().numpy()[clear] == a[smp.cpu().numpy()][clear]).all())
    flags = torch.tensor([int(idem), int(amin_ok)], device=dev)
    if ctx.world > 1:
        ctx.dist.all_reduce(flags, op=ctx.dist.ReduceOp.MIN)
    line = None
    if ctx.rank == 0:
        oracle.build()
        oracle.use_all_cores()
        # bit-exact parity with the faiss restatement at a size the oracle finishes in seconds (single-process engine)
        ns, ks = 20_000, 128
        xs = x[:ns].contiguous()
        sub = nv.Index(None, nv.BF16, nv.METRIC_L2, ctx.local, on_device_ptr=xs.data_ptr(), n=ns, d=d)
        ag, cg, og = sub.kmeans(ks, niter=5, full_lloyd=True)
        t0 = time.perf_counter()
        ao, co, oo = oracle.kmeans(xs.float().cpu().numpy(), ks, niter=5, full_lloyd=True)
        t_or = time.perf_counter() - t0
        sub.close()
        parity = {"assignment_is_fixed_point_all_ranks": bool(flags[0].item()), "assignment_equals_fp64_argmin_4096_sample_all_ranks": bool(flags[1].item()),
                  "small_problem": f"{ns} x {d} bf16, k={ks}, 5 iterations, full Lloyd", "assign_bit_exact_vs_oracle": bool(np.array_equal(ag, ao)),
                  "centroids_bit_exact_vs_oracle": bool(np.array_equal(cg.view(np.uint32), co.view(np.uint32))),
                  "objective_rel_err_vs_oracle": float(np.max(np.abs(og - oo) / np.maximum(np.abs(oo), 1e-30))),
                  "objective_first_last": [float(obj[0]), float(obj[-1])] if len(obj) else None, "clusters_used": int(len(np.unique(a)))}
        cpu = None
        if not ctx.args.no_cpu_baseline:
            per_it = t_or / 6  # 5 iterations + final assignment
            scale = (n / ns) * (k / ks)
            cpu = {"value": per_it * scale, "unit": "s/iteration", "cores": oracle.num_threads(), "kind": "port",
                   "sample": f"oracle.kmeans (canonical fp64 scorer, OpenMP) on {ns} points x {ks} centroids: {per_it:.3f} s/iteration, scaled by n*k to "
                             f"{n} x {k}: an ESTIMATE (faiss's sgemm path would be faster than this scalar port)"}
        pk = _peaks()
        peak = pk["bf16_tflops"]
        npts = (n if full else min(n, 256 * k))
        passes_fl = 2.0 * k * d * (npts * niter + n) / ctx.world
        s_per_it = ms / 1e3 / (niter + 1)
        line = _base(ctx, "sem_cluster_by seconds per k-means pass (5M x 768 bf16, k=1024)", s_per_it, "s/iteration", ms, False, "bf16",
                     {"workload": f"k-means {n} x {d} bf16, k={k}, {niter} Lloyd iterations + final assignment, "
                                  f"{'full Lloyd' if full else 'faiss parity (256*k subsample)'} (BASELINE.json configs[4])",
                      "n": n, "d": d, "k": k, "niter": niter, "parallelism": f"points row-sharded x{ctx.world}",
                      "l2_policy": "points %.0f MB per rank exceed L2" % ((hi - lo) * d * 2 / 1e6)}, "strong")
        line.update({"e2e": {"value": s_per_it, "unit": "s/iteration", "ms_per_step": ms, "h2d_bytes_per_step": 0, "d2h_bytes_per_step": (hi - lo) * 8 + k * d * 4,
                             "api": "b2_kmeans (points resident in the index handle; assignment + centroids + objective returned in HOST buffers)"
                             if ctx.world == 1 else "sharded_kmeans (b2_kmeans_assign_dev + b2_kmeans_accumulate_dev + NCCL all-reduce per iteration)"},
                     "gpu_launches": int(st["launches"]), "second_level_points": int(st["fallback_queries"]),
                     "roofline": {"bound": "tensor", "achieved": passes_fl / ms / 1e9, "peak": peak, "unit": "TFLOP/s", "frac": passes_fl / ms / 1e9 / peak,
                                  "traffic": None, "kernel": "knn_filter_kernel<16,L2,bf16,CTA pair,TOP1> (+ update pass)", "kernel_ms": ms,
                                  "note": "whole run timed: 2*n*k*d FLOP per assignment pass; the centroid update adds one HBM pass over the points per iteration "
                                          "(n*d*2 bytes = %.2f ms at the data-sheet %.0f GB/s)" % ((hi - lo) * d * 2 / pk["hbm_gbs"] / 1e6, pk["hbm_gbs"])},
                     "cpu_baseline": cpu, "parity": parity, "clocks": clocks})
    idx.close()
    ctx.finish(line)


def main(args, extra):
    if args.impl == "reference":
        if bench.env_int("RANK", 0) == 0:
            print(json.dumps({"impl": "reference", "config": args.config,
                              "unavailable": "the reference arm is implemented for the headline configuration; the secondary configurations carry their CPU arm in cpu_baseline"}), flush=True)
        return
    ctx = Ctx(args)
    {"c2": c2, "c4": c4, "c5": c5}[args.config](ctx, extra)
