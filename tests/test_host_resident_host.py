"""Host-resident indexes on CPU: the new C-ABI symbols, the chunking of the streamed search (b2_debug_stream_plan), and the
residency arguments of B200VS (GPU runs of the same surface are in tests/test_gpu_host_resident.py)."""
import ctypes

import numpy as np
import pytest

from lotus_b200 import vs as vsmod
from lotus_b200.vs import B200VS

NEW = ["b2_index_create_host", "b2_index_resident", "b2_debug_stream_plan", "b2_debug_stream_times"]


def test_new_symbols_are_exported(nv):
    L = nv.lib()
    for name in NEW:
        assert name in nv.SYMBOLS and hasattr(L, name), name
    assert L.b2_abi_version() == 1
    assert L.b2_index_resident(None) == -1


def _create_host(nv, n=4, d=8, dtype=0, ring=0):
    x = np.zeros((n, d), np.float32)  # large enough for every element type
    h = ctypes.c_void_p()
    rc = nv.lib().b2_index_create_host(ctypes.c_void_p(x.ctypes.data), n, d, dtype, 0, 0, ring, ctypes.byref(h))
    if rc == 0:
        nv.lib().b2_index_free(h)
    return rc


def test_create_host_validates_then_needs_a_device(nv):
    want = nv.ENODEV if nv.device_count() == 0 else nv.OK
    for dtype in (nv.F32, nv.BF16, nv.F16, nv.I8):
        assert _create_host(nv, dtype=dtype) == want
    assert _create_host(nv, dtype=3) == nv.EINVAL
    assert _create_host(nv, ring=-1) == nv.EINVAL
    assert _create_host(nv, ring=1000) == nv.EINVAL and "256 rows" in nv.lib().b2_last_error().decode()
    # ids are int32: 2^31 rows are refused before any memory is touched
    h = ctypes.c_void_p()
    x = np.zeros((1, 8), np.float32)
    rc = nv.lib().b2_index_create_host(ctypes.c_void_p(x.ctypes.data), 1 << 31, 8, nv.F32, 0, 0, 0, ctypes.byref(h))
    assert rc == nv.EINVAL and "2^31" in nv.lib().b2_last_error().decode()


def _ring_row_bytes(nv, d, dtype):
    esz = {nv.F32: 4, nv.BF16: 2, nv.F16: 2, nv.I8: 1}[dtype]
    align = 16 // esz
    b = -(-d // align) * align * esz
    if dtype == nv.I8:
        b += -(-d // 8) * 8 * 2
    return b


@pytest.mark.parametrize("dtype", [0, 1, 2, 8])
def test_stream_plan_covers_every_row_once_within_the_ring(nv, dtype):
    rng = np.random.default_rng(dtype)
    for _ in range(300):
        d = int(rng.choice([8, 30, 100, 768, 1000]))
        n = int(rng.integers(0, 3_000_000))
        ring = int(rng.integers(1 << 16, 1 << 31))
        row = _ring_row_bytes(nv, d, dtype)
        if ring // (2 * row) < 256:
            with pytest.raises(nv.NativeError):
                nv.stream_plan(n, d, dtype, ring)
            continue
        p = nv.stream_plan(n, d, dtype, ring)
        R, nc = p["chunk_rows"], p["n_chunks"]
        assert p["slots"] >= 2
        assert p["slots"] * R * row <= ring, (n, d, ring, p)
        if n == 0:
            assert nc == 0
            continue
        assert nc >= 1 and (nc == 1 or R % 256 == 0), p
        if nc == 1:
            assert R == n
        # chunk c owns [c R, min(n, (c + 1) R)): together they cover every row exactly once
        owned = np.zeros(n, np.int32)
        for c in range(nc):
            lo, hi = c * R, min(n, (c + 1) * R)
            assert lo < hi
            owned[lo:hi] += 1
            base = min(c * R, n - R)  # the streamed window holds the owned rows
            assert 0 <= base <= lo and hi <= base + R
        assert (owned == 1).all()
        # balanced: the last chunk re-streams fewer than 256 rows per chunk
        assert nc * R - n < 256 * nc


def test_stream_plan_default_ring_and_validation(nv):
    p = nv.stream_plan(1_000_000, 768, nv.BF16)
    assert p["n_chunks"] == 3 and p["chunk_rows"] * 768 * 2 * p["slots"] <= 1 << 30
    with pytest.raises(nv.NativeError):
        nv.stream_plan(10, 0, nv.BF16)
    with pytest.raises(nv.NativeError):
        nv.stream_plan(10, 8, 3)


def test_b200vs_residency_arguments():
    assert B200VS().residency == "device" and B200VS().ring_bytes is None
    with pytest.raises(ValueError, match="residency"):
        B200VS(residency="gpu")
    with pytest.raises(ValueError, match="devices"):
        B200VS(residency="host", devices=[0, 1])
    with pytest.raises(ValueError, match="ring_bytes"):
        B200VS(residency="host", ring_bytes=-5)
    B200VS(residency="auto", devices=[0, 1])  # auto never picks host for several devices: they take the sharded path


def test_device_footprint(nv):
    assert vsmod.device_footprint(1000, 768, nv.BF16) == 1000 * 768 * 2 + 1000 * 4
    # fp32: the rows, the bf16 first-level copy from 4096 rows on, the norms
    assert vsmod.device_footprint(4096, 768, nv.F32) == 4096 * 768 * 4 + 4096 * 768 * 2 + 4096 * 4
    assert vsmod.device_footprint(4095, 768, nv.F32) == 4095 * 768 * 4 + 4095 * 4
    # a row that is not a multiple of 16 bytes adds its padded copy
    assert vsmod.device_footprint(10, 100, nv.BF16) == 10 * 100 * 2 + 10 * 104 * 2 + 10 * 4
    assert vsmod.device_footprint(10, 100, nv.I8) == 10 * 100 + 10 * 112 + 10 * 8


def test_auto_residency_follows_free_memory(monkeypatch, nv):
    s = B200VS(residency="auto")
    need = vsmod.device_footprint(1_000_000, 768, nv.BF16) + vsmod.AUTO_MARGIN
    monkeypatch.setattr(vsmod, "_free_device_bytes", lambda device: need)
    assert s._choose_residency(1_000_000, 768, nv.BF16) == "device"
    monkeypatch.setattr(vsmod, "_free_device_bytes", lambda device: need - 1)
    assert s._choose_residency(1_000_000, 768, nv.BF16) == "host"
    # explicit choices never ask for the free memory
    monkeypatch.setattr(vsmod, "_free_device_bytes", lambda device: 1 / 0)
    assert B200VS(residency="host")._choose_residency(10, 8, nv.F32) == "host"
    assert B200VS()._choose_residency(10, 8, nv.F32) == "device"
