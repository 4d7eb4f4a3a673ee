"""SASS guard for the range filter kernels (range_filter_kernel, range_i8_filter_kernel): no local memory, pipelined wgmmas and
no GPU-scope fence in the mainloop, as the knn and pair filters are held to. Reads the built library; no GPU needed."""
import re
import shutil

import pytest

from test_sass_filter import sass_functions

LOCAL = re.compile(r"\b(LDL|STL)(\.\S+)?\s")


@pytest.fixture(scope="module")
def range_kernels(nv):
    if shutil.which("cuobjdump") is None:
        pytest.skip("cuobjdump not on PATH")
    funcs = {name: body for name, body in sass_functions(nv.LIB_PATH).items() if "range_filter_kernel" in name or "range_i8_filter_kernel" in name}
    # {tf32, bf16, fp16} x {IP, L2} x clusters of {1, 2, 4}, and the int8 entry {IP, L2} x {1, 2, 4}
    assert len(funcs) == 24, f"expected 24 range filter instantiations, found {len(funcs)}"
    return funcs


def test_range_filter_uses_no_local_memory(range_kernels):
    for name, body in range_kernels.items():
        spills = [line.strip() for line in body.splitlines() if LOCAL.search(line)]
        assert not spills, f"{name}: local memory (register spills): {spills[:4]}"


def test_range_filter_wgmmas_are_pipelined(range_kernels):
    for name, body in range_kernels.items():
        lines = body.splitlines()
        assert ("IGMMA" in body) == ("range_i8" in name) and ("HGMMA" in body) != ("range_i8" in name), name
        wait0 = sum("WARPGROUP.DEPBAR.LE gsb0, 0x0" in line for line in lines)
        wait1 = sum("WARPGROUP.DEPBAR.LE gsb0, 0x1" in line for line in lines)
        assert wait0 == 1 and wait1 >= 1, f"{name}: wgmma serialized ({wait0} full waits, {wait1} pipelined waits)"


def test_range_filter_mainloop_has_no_gpu_scope_fence(range_kernels):
    for name, body in range_kernels.items():
        lines = body.splitlines()
        mma = [i for i, line in enumerate(lines) if "GMMA" in line]
        depbar = [i for i, line in enumerate(lines) if "WARPGROUP.DEPBAR" in line]
        assert mma and depbar, f"{name}: no wgmma mainloop"
        fenced = [lines[i].strip() for i in range(mma[0], depbar[-1]) if "MEMBAR.ALL.GPU" in lines[i]]
        assert not fenced, f"{name}: GPU-scope fence inside the wgmma mainloop: {fenced}"
