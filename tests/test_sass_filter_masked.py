"""SASS guard for the masked knn filter (knn_masked_filter_kernel, knn_masked_i8_filter_kernel): the row bitmap must cost the
mainloop nothing. Every instantiation keeps the register-resident query K-blocks (register-A wgmmas on registers of their own,
shared-memory wgmmas past them), stays out of local memory, keeps its wgmmas pipelined and has no GPU-scope fence in the
mainloop. Reads the built library with cuobjdump; no GPU needed."""
import re
import shutil

import pytest

from test_sass_filter import sass_functions

RS_GMMA = re.compile(r"[HI]GMMA\.\S+\s+R\d+,\s*(R\d+),\s*gdesc")
LOCAL = re.compile(r"\b(LDL|STL)(\.\S+)?\s")


@pytest.fixture(scope="module")
def masked_kernels(nv):
    if shutil.which("cuobjdump") is None:
        pytest.skip("cuobjdump not on PATH")
    funcs = {name: body for name, body in sass_functions(nv.LIB_PATH).items()
             if "knn_masked_filter_kernel" in name or "knn_masked_i8_filter_kernel" in name}
    # every KP (16, 32, 64, 72) x {IP, L2} x clusters of {1, 2, 4} x {tf32, bf16, fp16, int8}
    assert len(funcs) == 96, f"expected 96 masked knn filter instantiations, found {len(funcs)}"
    return funcs


def test_masked_filter_keeps_the_resident_query_blocks(masked_kernels):
    counts = set()
    for name, body in masked_kernels.items():
        regs = RS_GMMA.findall(body)
        assert regs, f"{name}: no register-A wgmma"
        assert len(set(regs)) == len(regs), f"{name}: register-A wgmmas share fragment registers: {regs}"
        assert any("GMMA" in line and not RS_GMMA.search(line) for line in body.splitlines()), \
            f"{name}: no shared-memory wgmma for the K-blocks past the resident ones"
        counts.add(len(regs))
    assert counts == {10}, f"expected 5 resident K-blocks x 2 K steps of register-A wgmma, found {sorted(counts)}"


def test_masked_filter_uses_no_local_memory(masked_kernels):
    for name, body in masked_kernels.items():
        spills = [line.strip() for line in body.splitlines() if LOCAL.search(line)]
        assert not spills, f"{name}: local memory (register spills): {spills[:4]}"


def test_masked_filter_wgmmas_are_pipelined_and_unfenced(masked_kernels):
    for name, body in masked_kernels.items():
        lines = body.splitlines()
        wait0 = sum("WARPGROUP.DEPBAR.LE gsb0, 0x0" in line for line in lines)
        wait1 = sum("WARPGROUP.DEPBAR.LE gsb0, 0x1" in line for line in lines)
        assert wait0 == 1 and wait1 >= 1, f"{name}: wgmma serialized ({wait0} full waits, {wait1} pipelined waits)"
        gmma = [i for i, line in enumerate(lines) if "GMMA" in line]
        depbar = [i for i, line in enumerate(lines) if "WARPGROUP.DEPBAR" in line]
        fenced = [lines[i].strip() for i in range(gmma[0], depbar[-1]) if "MEMBAR.ALL.GPU" in lines[i]]
        assert not fenced, f"{name}: GPU-scope fence inside the wgmma mainloop: {fenced}"
