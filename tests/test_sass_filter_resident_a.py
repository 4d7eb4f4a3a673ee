"""SASS guard for the knn filter's register-resident query K-blocks (knn_filter_sm90.cu, mma_tile): every knn_filter_kernel
instantiation must issue register-A wgmmas, keep each resident fragment in registers of its own, stay out of local memory and
keep its wgmmas pipelined. Reads the built library with cuobjdump; no GPU needed."""
import re
import shutil

import pytest

from test_sass_filter import sass_functions

# register-A form: HGMMA.64x256x16.F32 R24, R152, gdesc[UR8], ... (the shared-memory form has gdesc where R152 is)
RS_HGMMA = re.compile(r"HGMMA\.\S+\s+R\d+,\s*(R\d+),\s*gdesc")
LOCAL = re.compile(r"\b(LDL|STL)(\.\S+)?\s")


@pytest.fixture(scope="module")
def knn_kernels(nv):
    if shutil.which("cuobjdump") is None:
        pytest.skip("cuobjdump not on PATH")
    funcs = {name: body for name, body in sass_functions(nv.LIB_PATH).items() if "knn_filter_kernel" in name}
    assert len(funcs) >= 80, f"expected every knn_filter_kernel instantiation in the SASS, found {len(funcs)}"
    return funcs


def test_every_knn_filter_instantiation_issues_register_a_wgmma(knn_kernels):
    counts = set()
    for name, body in knn_kernels.items():
        regs = RS_HGMMA.findall(body)
        assert regs, f"{name}: no register-A HGMMA"
        # one 4-register fragment per K step of each resident K-block, none shared: a fragment register reused by a later
        # K-block would mean that the fragments are not held across the tiles of an item
        assert len(set(regs)) == len(regs), f"{name}: register-A HGMMAs share fragment registers: {regs}"
        assert any("HGMMA" in line and not RS_HGMMA.search(line) for line in body.splitlines()), \
            f"{name}: no shared-memory HGMMA for the K-blocks past the resident ones"
        counts.add(len(regs))
    assert len(counts) == 1, f"instantiations disagree on the resident K-blocks: {sorted(counts)} register-A HGMMAs"


def test_knn_filter_uses_no_local_memory(knn_kernels):
    for name, body in knn_kernels.items():
        spills = [line.strip() for line in body.splitlines() if LOCAL.search(line)]
        assert not spills, f"{name}: local memory (register spills): {spills[:4]}"


def test_knn_filter_wgmmas_are_not_serialized(knn_kernels):
    # When ptxas serializes wgmma (notices C7510 / C7512), every HGMMA waits for its own completion:
    # each one is followed by WARPGROUP.DEPBAR.LE gsb0, 0x0. The pipelined mainloop keeps one group in flight (0x1), and
    # waits for 0 once per tile.
    for name, body in knn_kernels.items():
        lines = body.splitlines()
        wait0 = sum("WARPGROUP.DEPBAR.LE gsb0, 0x0" in line for line in lines)
        wait1 = sum("WARPGROUP.DEPBAR.LE gsb0, 0x1" in line for line in lines)
        assert wait0 == 1 and wait1 >= 1, f"{name}: wgmma serialized ({wait0} full waits, {wait1} pipelined waits)"
