"""SASS guard for the int8 knn filter (knn_i8_filter_kernel, IGMMA): the same mainloop properties the floating-point filter
kernels are held to — register-A wgmmas for the resident K-blocks on registers of their own, shared-memory wgmmas past them, no
local memory, pipelined wgmmas and no GPU-scope fence in the mainloop. Reads the built library with cuobjdump; no GPU needed."""
import re
import shutil

import pytest

from test_sass_filter import sass_functions

RS_IGMMA = re.compile(r"IGMMA\.\S+\s+R\d+,\s*(R\d+),\s*gdesc")
LOCAL = re.compile(r"\b(LDL|STL)(\.\S+)?\s")


@pytest.fixture(scope="module")
def i8_kernels(nv):
    if shutil.which("cuobjdump") is None:
        pytest.skip("cuobjdump not on PATH")
    funcs = {name: body for name, body in sass_functions(nv.LIB_PATH).items() if "knn_i8_filter_kernel" in name}
    # every KP (16, 32, 64, 72) x {IP, L2} x clusters of {1, 2, 4}
    assert len(funcs) == 24, f"expected 24 knn_i8_filter_kernel instantiations, found {len(funcs)}"
    return funcs


def test_int8_filter_issues_register_a_and_shared_memory_igmma(i8_kernels):
    counts = set()
    for name, body in i8_kernels.items():
        assert "HGMMA" not in body, f"{name}: floating-point wgmma in the int8 kernel"
        regs = RS_IGMMA.findall(body)
        assert regs, f"{name}: no register-A IGMMA"
        assert len(set(regs)) == len(regs), f"{name}: register-A IGMMAs share fragment registers: {regs}"
        assert any("IGMMA" in line and not RS_IGMMA.search(line) for line in body.splitlines()), \
            f"{name}: no shared-memory IGMMA for the K-blocks past the resident ones"
        counts.add(len(regs))
    assert counts == {12}, f"expected 6 resident K-blocks x 2 k32 steps of register-A IGMMA, found {sorted(counts)}"


def test_int8_filter_uses_no_local_memory(i8_kernels):
    for name, body in i8_kernels.items():
        spills = [line.strip() for line in body.splitlines() if LOCAL.search(line)]
        assert not spills, f"{name}: local memory (register spills): {spills[:4]}"


def test_int8_filter_wgmmas_are_pipelined(i8_kernels):
    for name, body in i8_kernels.items():
        lines = body.splitlines()
        wait0 = sum("WARPGROUP.DEPBAR.LE gsb0, 0x0" in line for line in lines)
        wait1 = sum("WARPGROUP.DEPBAR.LE gsb0, 0x1" in line for line in lines)
        assert wait0 == 1 and wait1 >= 1, f"{name}: wgmma serialized ({wait0} full waits, {wait1} pipelined waits)"


def test_int8_filter_mainloop_has_no_gpu_scope_fence(i8_kernels):
    for name, body in i8_kernels.items():
        lines = body.splitlines()
        igmma = [i for i, line in enumerate(lines) if "IGMMA" in line]
        depbar = [i for i, line in enumerate(lines) if "WARPGROUP.DEPBAR" in line]
        assert igmma and depbar, f"{name}: no wgmma mainloop"
        fenced = [lines[i].strip() for i in range(igmma[0], depbar[-1]) if "MEMBAR.ALL.GPU" in lines[i]]
        assert not fenced, f"{name}: GPU-scope fence inside the wgmma mainloop: {fenced}"
