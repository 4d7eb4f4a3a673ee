"""SASS guard for the masked range filter (range_masked_filter_kernel, range_masked_i8_filter_kernel): the row bitmap must cost
the mainloop nothing. Every instantiation stays out of local memory, keeps its wgmmas pipelined, has no GPU-scope fence in the
mainloop, and runs IGMMA exactly in the int8 entries. Reads the built library with cuobjdump; no GPU needed."""
import re
import shutil

import pytest

from test_sass_filter import sass_functions

LOCAL = re.compile(r"\b(LDL|STL)(\.\S+)?\s")


@pytest.fixture(scope="module")
def masked_range_kernels(nv):
    if shutil.which("cuobjdump") is None:
        pytest.skip("cuobjdump not on PATH")
    funcs = {name: body for name, body in sass_functions(nv.LIB_PATH).items()
             if "range_masked_filter_kernel" in name or "range_masked_i8_filter_kernel" in name}
    # {tf32, bf16, fp16} x {IP, L2} x clusters of {1, 2, 4}, and the int8 entry {IP, L2} x {1, 2, 4}
    assert len(funcs) == 24, f"expected 24 masked range filter instantiations, found {len(funcs)}"
    return funcs


def test_masked_range_filter_uses_no_local_memory(masked_range_kernels):
    for name, body in masked_range_kernels.items():
        spills = [line.strip() for line in body.splitlines() if LOCAL.search(line)]
        assert not spills, f"{name}: local memory (register spills): {spills[:4]}"


def test_masked_range_filter_wgmmas_are_pipelined(masked_range_kernels):
    for name, body in masked_range_kernels.items():
        lines = body.splitlines()
        i8 = "range_masked_i8" in name
        assert ("IGMMA" in body) == i8 and ("HGMMA" in body) != i8, name
        wait0 = sum("WARPGROUP.DEPBAR.LE gsb0, 0x0" in line for line in lines)
        wait1 = sum("WARPGROUP.DEPBAR.LE gsb0, 0x1" in line for line in lines)
        assert wait0 == 1 and wait1 >= 1, f"{name}: wgmma serialized ({wait0} full waits, {wait1} pipelined waits)"


def test_masked_range_filter_mainloop_has_no_gpu_scope_fence(masked_range_kernels):
    for name, body in masked_range_kernels.items():
        lines = body.splitlines()
        gmma = [i for i, line in enumerate(lines) if "GMMA" in line]
        depbar = [i for i, line in enumerate(lines) if "WARPGROUP.DEPBAR" in line]
        assert gmma and depbar, f"{name}: no wgmma mainloop"
        fenced = [lines[i].strip() for i in range(gmma[0], depbar[-1]) if "MEMBAR.ALL.GPU" in lines[i]]
        assert not fenced, f"{name}: GPU-scope fence inside the wgmma mainloop: {fenced}"
