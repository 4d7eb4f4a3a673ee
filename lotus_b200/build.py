"""Build libb2lotus.so (sm_90a only) in-tree with nvcc. No torch, no CPU fallback.

    python -m lotus_b200.build [--force]

The shared library is a plain C-ABI library (include/lotus_b200.h); it links the CUDA runtime statically and
resolves cuTensorMapEncodeTiled through cudaGetDriverEntryPoint, so it has no link-time dependency on libcuda.
"""
from __future__ import annotations

import concurrent.futures as cf
import glob
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
OBJ = os.path.join(HERE, "csrc", "_obj")
LIB = os.path.join(HERE, "libb2lotus.so")
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-std=c++17", "-O3", "-lineinfo",
         "-Xcompiler", "-fPIC", "-Xcompiler", "-fvisibility=hidden", "--expt-relaxed-constexpr",
         "-diag-suppress", "177"]


def sources() -> list[str]:
    return sorted(glob.glob(os.path.join(CSRC, "*.cu")))


def _deps_mtime() -> float:
    files = sources() + glob.glob(os.path.join(CSRC, "*.cuh")) + [os.path.join(HERE, "..", "include", "lotus_b200.h")]
    return max(os.path.getmtime(f) for f in files)


def _compile(src: str) -> str:
    obj = os.path.join(OBJ, os.path.basename(src)[:-3] + ".o")
    if os.path.exists(obj) and os.path.getmtime(obj) >= _deps_mtime():
        return obj
    cmd = [NVCC, *FLAGS, "-c", src, "-o", obj]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        sys.stderr.write(r.stdout + r.stderr)
        raise RuntimeError(f"nvcc failed for {src}")
    return obj


def build(force: bool = False) -> str:
    os.makedirs(OBJ, exist_ok=True)
    objs_now = [os.path.join(OBJ, os.path.basename(s)[:-3] + ".o") for s in sources()]
    fresh = all(os.path.exists(o) and os.path.getmtime(o) >= _deps_mtime() for o in objs_now)  # a library newer than the sources is not
    if not force and fresh and os.path.exists(LIB) and os.path.getmtime(LIB) >= max(os.path.getmtime(o) for o in objs_now):  # enough: it may have
        return LIB                                                                                    # been linked from stale objects
    if force:
        for f in glob.glob(os.path.join(OBJ, "*.o")):
            os.remove(f)
    with cf.ThreadPoolExecutor(max_workers=min(8, os.cpu_count() or 1)) as ex:
        objs = list(ex.map(_compile, sources()))
    cmd = [NVCC, "-shared", "-gencode", "arch=compute_90a,code=sm_90a", "-o", LIB, *objs]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        sys.stderr.write(r.stdout + r.stderr)
        raise RuntimeError("link failed")
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv))
