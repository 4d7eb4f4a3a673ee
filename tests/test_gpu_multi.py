"""Multi-GPU parity against the oracle: the torchrun-sharded search, dedup and k-means paths (tests/multigpu_worker.py) and the
single-process store over several devices, B200VS(devices=[...]). Both need two GPUs or more and skip on a one-GPU machine."""
import os
import subprocess
import sys
import tempfile

import numpy as np
import pytest

import oracle

HERE = os.path.dirname(os.path.abspath(__file__))


def gauss(n, d, seed):
    rng = np.random.default_rng(seed)
    x = rng.standard_normal((n, d), dtype=np.float32)
    return x / np.linalg.norm(x, axis=1, keepdims=True)


def _need_two(nv) -> int:
    g = nv.device_count()
    if g < 2:
        pytest.skip(f"needs two GPUs or more ({g} visible)")
    return g


@pytest.mark.gpu
def test_sharded_paths_match_the_oracle_under_torchrun(gpu):
    g = min(_need_two(gpu), 8)
    r = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--standalone", f"--nproc-per-node={g}",
                        os.path.join(HERE, "multigpu_worker.py")], capture_output=True, text=True, timeout=900)
    assert r.returncode == 0 and "MULTIGPU CHECK OK" in r.stdout, (r.stdout[-3000:], r.stderr[-3000:])


@pytest.mark.gpu
def test_single_process_store_over_several_devices(gpu):
    import lotus_b200 as lotus
    nv = gpu
    g = _need_two(nv)
    x, q = gauss(50_021, 96, 0), gauss(500, 96, 1)
    # two independent handles, one per device, used alternately from this process (the kernels' shared-memory attribute is
    # per device)
    a, b = nv.Index(x[:30_000].copy(), nv.F32, nv.METRIC_IP, 0), nv.Index(x[30_000:].copy(), nv.F32, nv.METRIC_IP, 1)
    for _ in range(2):
        for idx, xs in ((a, x[:30_000]), (b, x[30_000:])):
            D, I = idx.search(q, 10)
            Do, Io = oracle.knn(xs, q, 10, oracle.IP)
            assert np.array_equal(I, Io) and np.array_equal(D.view(np.uint32), Do.view(np.uint32))
    a.close()
    b.close()
    with tempfile.TemporaryDirectory() as tmp:
        for metric, om in ((lotus.METRIC_INNER_PRODUCT, oracle.IP), (lotus.METRIC_L2, oracle.L2)):
            for dtype in ("f32", "bf16"):
                vs = lotus.B200VS(metric=metric, dtype=dtype, devices=list(range(g)))
                vs.index(None, x, os.path.join(tmp, f"i{metric}{dtype}"))
                xf = x if dtype == "f32" else nv.bf16_bits_to_f32(nv.f32_to_bf16_bits(x))
                r = vs(q, 10)
                Do, Io = oracle.knn(xf, q, 10, om)
                assert np.array_equal(r.indices, Io) and np.array_equal(np.asarray(r.distances).view(np.uint32), Do.view(np.uint32))
                ids = np.arange(5, len(x), 3)
                r = vs(q, 10, ids=ids)
                Ds, Is = oracle.knn_subset(xf, q, 10, ids, om)
                assert np.array_equal(r.indices, Is) and np.array_equal(np.asarray(r.distances).view(np.uint32), Ds.view(np.uint32))
                got = vs.get_vectors_from_index(os.path.join(tmp, f"i{metric}{dtype}"), [50_020, 0, 25_000])
                assert np.array_equal(np.asarray(got), xf[[50_020, 0, 25_000]])
                vs.close()
