"""bench.py contract (CPU-checkable part): the reference arm runs without a GPU, prints ONE JSON line with the keys the
driver reads, and never touches lotus_b200's CUDA library."""
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_reference_arm_prints_one_json_line():
    r = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--impl", "reference", "--n", "30000", "--nq", "500",
                        "--cpu-sample", "8", "--steps", "1", "--warmup", "3"], capture_output=True, text=True, timeout=600,
                       env=dict(os.environ, RANK="0", WORLD_SIZE="1"))
    assert r.returncode == 0, r.stderr[-2000:]
    lines = [ln for ln in r.stdout.splitlines() if ln.strip()]
    assert len(lines) == 1
    d = json.loads(lines[0])
    assert d["impl"] == "reference" and d["unit"] == "queries/s" and d["higher_is_better"] is True and d["value"] > 0
    for key in ("metric", "n_gpus", "steps", "warmup", "ms_per_step", "scaling", "vs_baseline", "dtype", "data", "config",
                "cpu_baseline", "e2e"):
        assert key in d
    assert d["cpu_baseline"]["kind"] == "port" and d["cpu_baseline"]["cores"] >= 1
    assert d["e2e"]["h2d_bytes_per_step"] == 0 and d["e2e"]["d2h_bytes_per_step"] == 0 and "workload" in d["config"]


def test_reference_arm_other_ranks_exit_quietly():
    r = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--impl", "reference", "--gpus", "2"], capture_output=True,
                       text=True, timeout=120, env=dict(os.environ, RANK="1", WORLD_SIZE="2"))
    assert r.returncode == 0 and r.stdout.strip() == ""


def test_reference_arm_sizes_its_own_sample():
    # --cpu-sample 0 (the default): the step is calibrated to ~10 s of the host cores, clamped to [128, 8192] and to nq
    r = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--impl", "reference", "--n", "20000", "--nq", "300",
                        "--steps", "1", "--warmup", "3"], capture_output=True, text=True, timeout=600,
                       env=dict(os.environ, RANK="0", WORLD_SIZE="1"))
    assert r.returncode == 0, r.stderr[-2000:]
    d = json.loads(r.stdout.strip().splitlines()[-1])
    assert 128 <= d["reference_run"]["sample_queries_per_step"] <= 300 and d["value"] > 0
    assert set(d["config"]) == {"workload", "nq", "n", "d", "k", "parallelism", "l2_policy"}  # the GPU arm's config keys


def test_reference_arm_uses_every_core_even_under_torchrun_env():
    # torchrun exports OMP_NUM_THREADS=1 to its workers; rank 0 of the reference arm must still use the host's cores
    r = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--impl", "reference", "--n", "20000", "--nq", "300",
                        "--cpu-sample", "64", "--steps", "1", "--warmup", "3"], capture_output=True, text=True, timeout=600,
                       env=dict(os.environ, RANK="0", WORLD_SIZE="2", OMP_NUM_THREADS="1"))
    assert r.returncode == 0, r.stderr[-2000:]
    d = json.loads(r.stdout.strip().splitlines()[-1])
    import oracle
    assert d["cpu_baseline"]["cores"] == oracle.cpu_budget()["threads"] >= 1
