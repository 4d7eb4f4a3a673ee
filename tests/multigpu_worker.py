"""Worker of tests/test_gpu_multi.py (run under torchrun on N >= 2 GPUs of one machine): multi-GPU parity of the sharded paths:
   row-sharded search (+ ids subset), sharded dedup relation, sharded Lloyd k-means — each against the oracle."""
import os
import sys

import numpy as np
import torch
import torch.distributed as dist

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import oracle  # noqa: E402
from lotus_b200 import _native as nv  # noqa: E402
from lotus_b200.distributed import ShardedIndex, shard_bounds, sharded_kmeans, sharded_threshold_pairs  # noqa: E402


def gauss(n, d, seed):
    rng = np.random.default_rng(seed)
    x = rng.standard_normal((n, d), dtype=np.float32)
    return x / np.linalg.norm(x, axis=1, keepdims=True)


def main():
    rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    os.environ.setdefault("NCCL_DEBUG", "WARN")
    dist.init_process_group("nccl", device_id=dev)
    ok = True

    # 1. row-sharded search, with and without an ids subset
    x, q = gauss(20_011, 96, 0), gauss(333, 96, 1)
    lo, hi = shard_bounds(len(x), world, rank)
    for metric in (nv.METRIC_IP, nv.METRIC_L2):
        sh = ShardedIndex(torch.from_numpy(x[lo:hi]).to(dev).contiguous(), lo, metric)
        s, i = sh.search(torch.from_numpy(q).to(dev), 10)
        Do, Io = oracle.knn(x, q, 10, metric)
        good = np.array_equal(i.cpu().numpy(), Io) and np.array_equal(s.cpu().numpy().view(np.uint32), Do.view(np.uint32))
        ids = np.arange(7, len(x), 5)
        s, i = sh.search(torch.from_numpy(q).to(dev), 10, ids=ids)
        Ds, Is = oracle.knn_subset(x, q, 10, ids, metric)
        good &= np.array_equal(i.cpu().numpy(), Is) and np.array_equal(s.cpu().numpy().view(np.uint32), Ds.view(np.uint32))
        # the end-to-end form: every rank copies 1/world of the pinned host queries, slices all-gathered over NVLink
        qh = torch.from_numpy(q).pin_memory()
        s2, i2 = sh.search_host(qh, 10)
        good &= np.array_equal(i2.cpu().numpy(), Io) and np.array_equal(s2.cpu().numpy().view(np.uint32), Do.view(np.uint32))
        # a large k through the packed exchange (8 ranks x 128 = the merge kernel's 1024-candidate limit)
        s3, i3 = sh.search(torch.from_numpy(q[:50]).to(dev), 100)
        D3, I3 = oracle.knn(x, q[:50], 100, metric)
        good &= np.array_equal(i3.cpu().numpy(), I3) and np.array_equal(s3.cpu().numpy().view(np.uint32), D3.view(np.uint32))
        print(f"[rank {rank}] sharded search metric={metric} (device, host-buffer and k=100 forms): {'OK' if good else 'MISMATCH'}", flush=True)
        ok &= good
        sh.close()

    # 2. dedup relation: corpus replicated, tile triangle dealt over the ranks
    xd = gauss(4000, 64, 2)
    rng = np.random.default_rng(3)
    src, dst = rng.choice(4000, 200, replace=False), rng.choice(4000, 200, replace=False)
    xd[dst] = xd[src] + 0.02 * gauss(200, 64, 4)
    xd /= np.linalg.norm(xd, axis=1, keepdims=True)
    idx = nv.Index(xd, nv.F32, nv.METRIC_IP, local)
    pi, pj = sharded_threshold_pairs(idx, 0.9)
    oi, oj, cnt = oracle.threshold_pairs(xd, 0.9)
    good = np.array_equal(pi, oi) and np.array_equal(pj, oj) and cnt > 50
    print(f"[rank {rank}] sharded dedup pairs ({len(pi)}): {'OK' if good else 'MISMATCH'}", flush=True)
    ok &= good
    idx.close()

    # 3. k-means: points sharded, sums all-reduced
    centers = gauss(6, 48, 5) * 4
    xk = (centers[np.random.default_rng(6).integers(0, 6, 6000)] + gauss(6000, 48, 7) * 6.9).astype(np.float32)
    lo, hi = shard_bounds(len(xk), world, rank)
    idx = nv.Index(xk[lo:hi].copy(), nv.F32, nv.METRIC_L2, local)
    a, c, obj = sharded_kmeans(idx, len(xk), lo, 6, niter=5)
    ao, co, oo = oracle.kmeans(xk, 6, niter=5, full_lloyd=True)
    good = np.allclose(c, co, rtol=1e-5, atol=1e-6) and np.allclose(obj, oo, rtol=1e-5) and np.array_equal(a, ao[lo:hi])
    print(f"[rank {rank}] sharded k-means: {'OK' if good else 'MISMATCH'} (max |dc| {np.abs(c - co).max():.2e})", flush=True)
    ok &= good
    idx.close()

    flag = torch.tensor([1 if ok else 0], device=dev)
    dist.all_reduce(flag, op=dist.ReduceOp.MIN)
    if rank == 0:
        print("MULTIGPU CHECK", "OK" if int(flag.item()) == 1 else "FAILED", flush=True)
    dist.destroy_process_group()
    sys.exit(0 if int(flag.item()) == 1 else 1)


if __name__ == "__main__":
    main()
