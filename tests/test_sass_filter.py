"""SASS guard for the filter kernels' mainloop: releasing an operand stage must not fence the whole GPU.

A cluster-scope release on the remote mbarrier arrive is lowered to MEMBAR.ALL.GPU, which every consumer warp would then
wait out once per K-block, between its wgmma groups. Reads the built library with cuobjdump; no GPU needed."""
import re
import shutil
import subprocess

import pytest


def sass_functions(lib_path):
    sass = subprocess.run(["cuobjdump", "-sass", lib_path], capture_output=True, text=True).stdout
    parts = re.split(r"^\s*Function : (\S+)\s*$", sass, flags=re.M)
    return dict(zip(parts[1::2], parts[2::2]))


def test_filter_mainloop_has_no_gpu_scope_fence(nv):
    if shutil.which("cuobjdump") is None:
        pytest.skip("cuobjdump not on PATH")
    funcs = {name: body for name, body in sass_functions(nv.LIB_PATH).items()
             if "knn_filter_kernel" in name or "pair_filter_kernel" in name}
    assert len(funcs) >= 40, f"expected every filter instantiation in the SASS, found {len(funcs)}"
    for name, body in funcs.items():
        lines = body.splitlines()
        hgmma = [i for i, line in enumerate(lines) if "HGMMA" in line]
        depbar = [i for i, line in enumerate(lines) if "WARPGROUP.DEPBAR" in line]
        assert hgmma and depbar, f"{name}: no wgmma mainloop"
        fenced = [lines[i].strip() for i in range(hgmma[0], depbar[-1]) if "MEMBAR.ALL.GPU" in lines[i]]
        assert not fenced, f"{name}: GPU-scope fence inside the wgmma mainloop: {fenced}"
