"""int8 indexes (B2_I8) on CPU: the C-ABI's validation and error model, the int8 storage helpers, and the int8 paths of B200VS
and the index directory (GPU runs of the same surface are in tests/test_gpu_i8.py)."""
import ctypes
import os
import re

import numpy as np
import pytest

from lotus_b200 import _native as nv
from lotus_b200 import faiss_io
from lotus_b200.vs import B200VS, _as_int8, _to_host_matrix

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_header_keeps_int8_apart_from_the_float_codes(nv):
    hdr = open(os.path.join(ROOT, "include", "lotus_b200.h")).read()
    assert re.search(r"enum\s*\{\s*B2_I8\s*=\s*8\s*\}", hdr)
    assert nv.I8 == 8 and nv.I8 not in nv.DTYPES and nv.DTYPES == (0, 1, 2)
    assert nv.lib().b2_abi_version() == 1


def _create(nv, dtype, d=8):
    x = np.zeros((4, d), np.int8)
    h = ctypes.c_void_p()
    rc = nv.lib().b2_index_create(ctypes.c_void_p(x.ctypes.data), 4, d, dtype, 0, 0, 0, ctypes.byref(h))
    if rc == 0:
        nv.lib().b2_index_free(h)
    return rc


def test_index_create_validates_int8(nv):
    assert _create(nv, 3) == nv.EINVAL and "B2_I8" in nv.lib().b2_last_error().decode()
    # the s32 accumulators bound the dimension of an int8 index, checked before any device is needed
    assert _create(nv, nv.I8, d=1 << 17) == nv.EINVAL and "2^17" in nv.lib().b2_last_error().decode()
    assert _create(nv, nv.I8, d=(1 << 17) - 1) == (nv.ENODEV if nv.device_count() == 0 else nv.OK)
    assert _create(nv, nv.I8) == (nv.ENODEV if nv.device_count() == 0 else nv.OK)


def _ulp_eq(a, b):
    return abs(a - float(b)) <= 2.0 ** -23 * abs(float(b))


def test_int8_error_model(nv):
    """rel_eps / abs_eps of every combination involving int8 (DESIGN.md §2): int8 values are exact in every filter type, and
    the int8 filter accumulates exactly, so its one error is the rounding of the s32 sum to fp32 (2^-24)."""
    F32, BF16, F16, I8 = nv.F32, nv.BF16, nv.F16, nv.I8
    for d in (8, 30, 768, 2048, (1 << 17) - 1):
        acc = (d + 64) * 2.0 ** -23 + 1e-6
        rel, ab = nv.filter_eps(I8, I8, I8, d)
        assert _ulp_eq(rel, np.float32(2.0 ** -24 + 1e-6)) and ab == 0.0
        # floating-point queries on the fp16 copy of an int8 store: only the query is rounded
        for q, eq, rounded in [(F16, 0.0, 0), (F32, 2.0 ** -11, 1), (BF16, 2.0 ** -11, 1)]:
            rel, ab = nv.filter_eps(I8, F16, q, d)
            assert _ulp_eq(rel, np.float32(acc + eq)), (q, d)
            assert _ulp_eq(ab, np.float32(rounded * 2.0 ** -25 * np.sqrt(d) * (1 + 1e-6))), (q, d)
        # int8 queries carry no operand error on any filter
        for store, filt, ex in [(F32, F32, 2.0 ** -10), (BF16, BF16, 0.0), (F16, F16, 0.0), (F32, BF16, 2.0 ** -8)]:
            rel, ab = nv.filter_eps(store, filt, I8, d)
            assert _ulp_eq(rel, np.float32(acc + ex)) and ab == 0.0, (store, filt, d)
    with pytest.raises(nv.NativeError):
        nv.filter_eps(3, I8, I8, 8)


def test_int8_storage_helpers(nv):
    x = np.array([[-128, -1, 0, 1, 127]], np.int8)
    assert nv.storage_dtype(nv.I8) == np.int8
    up = nv.stored_to_f32(x, nv.I8)
    assert up.dtype == np.float32 and np.array_equal(up, x.astype(np.float32))


def test_int8_store_input_validation():
    rng = np.random.default_rng(0)
    ints = rng.integers(-128, 128, size=(50, 12))
    for a in (ints.astype(np.int8), ints.astype(np.int16), ints.astype(np.int64), ints.astype(np.float32), ints.astype(np.float64)):
        x = _as_int8(a)
        assert x.dtype == np.int8 and np.array_equal(x, ints)
    for bad in (ints.astype(np.float32) + 0.5, np.full((2, 3), 128), np.full((2, 3), -129.0), np.full((2, 3), np.nan),
                np.array([["a", "b"]])):
        with pytest.raises(ValueError):
            _as_int8(bad)
    with pytest.raises(ValueError):
        _as_int8(ints[0])  # 1-D
    host, code, f32 = _to_host_matrix(ints.astype(np.float32), False, want_i8=True)
    assert code == nv.I8 and host.dtype == np.int8 and np.array_equal(f32, ints.astype(np.float32))
    with pytest.raises(ValueError):
        B200VS(dtype="i4")
    assert B200VS(dtype="i8").dtype == "i8"


def test_query_codes_shipped():
    """int8 queries travel as 1-byte I8 operands; every other type keeps its existing code."""
    q = np.arange(-6, 6, dtype=np.int8).reshape(2, 6)
    host, code, f32 = _to_host_matrix(q, False, pass_f16=True, pass_i8=True)
    assert code == nv.I8 and host.dtype == np.int8 and np.array_equal(f32, q.astype(np.float32))
    assert _to_host_matrix(q.astype(np.float32), False, pass_f16=True, pass_i8=True)[1] == nv.F32
    assert _to_host_matrix(q.astype(np.float16), False, pass_f16=True, pass_i8=True)[1] == nv.F16
    assert _to_host_matrix(q, False)[1] == nv.F32  # without pass_i8 (dtype='auto' stores): float32, as before
    torch = pytest.importorskip("torch")
    host, code, _ = _to_host_matrix(torch.from_numpy(q), False, pass_f16=True, pass_i8=True)
    assert code == nv.I8 and host.dtype == np.int8


def test_int8_index_directory_round_trip(tmp_path):
    """The reference format: the vecs pickle keeps the int8 array, the index file its float32 upcast; a directory without the
    pickle loads the float32 values, which dtype='i8' accepts since they are integral."""
    x = np.random.default_rng(1).integers(-128, 128, size=(40, 16)).astype(np.int8)
    d = str(tmp_path / "ix")
    faiss_io.write_index_dir(d, x, x.astype(np.float32), 0)
    vecs, xf, metric = faiss_io.read_index_dir(d)
    assert vecs.dtype == np.int8 and np.array_equal(vecs, x) and xf.dtype == np.float32 and metric == 0
    assert np.array_equal(_to_host_matrix(vecs, False, want_i8=True)[0], x)
    os.remove(os.path.join(d, "vecs"))
    vecs, xf, _ = faiss_io.read_index_dir(d)
    assert vecs.dtype == np.float32 and np.array_equal(_to_host_matrix(vecs, False, want_i8=True)[0], x)


def test_sharded_index_takes_int8_tensors():
    torch = pytest.importorskip("torch")
    from lotus_b200.distributed import torch_dtype_code
    assert torch_dtype_code(torch.zeros((2, 4), dtype=torch.int8)) == nv.I8
    with pytest.raises(TypeError):
        torch_dtype_code(torch.zeros((2, 4), dtype=torch.int16))


def test_int8_l2_index_dimension_limit(nv):
    x = np.zeros((4, 1 << 15), np.int8)
    h = ctypes.c_void_p()
    rc = nv.lib().b2_index_create(ctypes.c_void_p(x.ctypes.data), 4, 1 << 15, nv.I8, nv.METRIC_L2, 0, 0, ctypes.byref(h))
    assert rc == nv.EINVAL and "2^15" in nv.lib().b2_last_error().decode()


# ---- the operators over int8 embeddings, with the native index replaced by an oracle-backed fake ----------------------------
class Int8RM:
    """HashRM embeddings quantized to int8 with a fixed scale, as an int8-quantizing encoder returns them."""

    def __new__(cls, dim):
        import lotus_b200 as lotus

        class _RM(lotus.HashRM):
            def _embed(self, docs):
                return np.clip(np.rint(np.asarray(super()._embed(docs), dtype=np.float64) * 100), -128, 127).astype(np.int8)
        return _RM(dim=dim)


def test_operators_over_int8_embeddings_equal_the_oracle_frames(monkeypatch, tmp_path):
    import pandas as pd

    import lotus_b200 as lotus
    from helpers import NumpyVS
    from test_f16_host import FakeF16Index, _frames
    FakeF16Index.live = 0
    monkeypatch.setattr(nv, "Index", FakeF16Index)
    monkeypatch.setattr(nv, "require_device", lambda: None)
    rm = Int8RM(32)
    try:
        lotus.settings.configure(rm=rm, vs=NumpyVS(), enable_cache=False)  # the oracle on the float32 upcast
        want = _frames(tmp_path / "w", monkeypatch)
        vs = B200VS(dtype="i8")
        lotus.settings.configure(rm=rm, vs=vs, enable_cache=False)
        got = _frames(tmp_path / "g", monkeypatch)
        assert vs.b2_index.dtype == nv.I8
        # sem_sim_join fetched the right frame's vectors (int8, get_vectors_from_index) and searched with them as I8 operands
        assert any(c == (np.dtype(np.int8), nv.I8) for c in vs.b2_index.calls)
    finally:
        lotus.settings.configure(rm=None, vs=None)
    for key in want:
        pd.testing.assert_frame_equal(got[key], want[key], check_exact=True, obj=key)
