"""The C-ABI library loads, exports every symbol include/lotus_b200.h declares, and refuses to compute without a GPU
(no CPU fallback). No compute calls here."""
import ctypes
import os
import re

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def declared_symbols():
    hdr = open(os.path.join(ROOT, "include", "lotus_b200.h")).read()
    return sorted(set(re.findall(r"B2_API[^;]*?\b(b2_\w+)\s*\(", hdr, flags=re.S)))


def test_header_and_binding_agree(nv):
    assert declared_symbols() == sorted(nv.SYMBOLS)


def test_library_exports_every_declared_symbol(nv):
    lib = ctypes.CDLL(nv.LIB_PATH)
    for name in declared_symbols():
        assert hasattr(lib, name), f"libb2lotus.so does not export {name}"
    assert lib.b2_abi_version() == 1


def test_no_torch_types_in_signatures():
    hdr = open(os.path.join(ROOT, "include", "lotus_b200.h")).read()
    protos = re.findall(r"^B2_API [^;]*;", hdr, flags=re.S | re.M)
    assert len(protos) == len(declared_symbols())
    for p in protos:
        for banned in ("torch", "at::", "Tensor", "cudaStream_t", "CUstream", "std::"):
            assert banned not in p, f"{banned} in the C-ABI: {p}"


def test_library_is_sm90a_native(nv):
    import shutil
    import subprocess
    if shutil.which("cuobjdump") is None:
        pytest.skip("cuobjdump not on PATH")
    out = subprocess.run(["cuobjdump", "-lelf", nv.LIB_PATH], capture_output=True, text=True).stdout
    assert "sm_90a" in out and "sm_100" not in out and "sm_80" not in out
    sass = subprocess.run(["cuobjdump", "-sass", nv.LIB_PATH], capture_output=True, text=True).stdout
    for mnemonic in ("HGMMA", "UTMALDG", "SYNCS"):  # wgmma, TMA load, mbarrier
        assert mnemonic in sass, f"{mnemonic} missing from the SASS"


@pytest.mark.skipif(os.environ.get("B2_EXPECT_GPU") == "1", reason="GPU machine")
def test_refuses_to_compute_without_a_gpu(nv):
    if nv.device_count() > 0:
        pytest.skip("an H100 is visible")
    with pytest.raises(nv.NativeError) as e:
        nv.Index(np.zeros((4, 8), np.float32), nv.F32)
    assert e.value.code == nv.ENODEV and "no CPU fallback" in e.value.msg
    with pytest.raises(RuntimeError):
        nv.require_device()
    from lotus_b200 import B200VS
    vs = B200VS()
    with pytest.raises(ValueError, match="Index not loaded"):
        vs(np.zeros((1, 8), np.float32), 1)
    with pytest.raises(RuntimeError):
        vs.index(None, np.zeros((4, 8), np.float32), "/tmp/_b2_never_written")


def test_product_does_not_import_the_oracle():
    """Only tests/, __graft_entry__.smoke() and bench.py may touch oracle/."""
    pkg = os.path.join(ROOT, "lotus_b200")
    for dirpath, _, files in os.walk(pkg):
        for f in files:
            if f.endswith((".py", ".cu", ".cuh", ".h")):
                src = open(os.path.join(dirpath, f)).read()
                assert not re.search(r"^\s*(import|from)\s+oracle\b", src, flags=re.M), f"{f} imports the oracle"
                assert "liborc" not in src and "faiss_flat.c" not in src.replace("oracle/faiss_flat.c", ""), f
