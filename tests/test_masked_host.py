"""Masked search, the parts that need no GPU: the bitmap's packing and per-shard slicing, the test for ids a bitmap can stand
for, the header's declarations, and B2_ENODEV from the entry points on a machine without an H100."""
import ctypes
import os
import re

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NEW = ["b2_index_search_masked", "b2_index_search_masked_dev", "b2_debug_filter_lists_masked"]


@pytest.mark.parametrize("n", [0, 1, 31, 32, 33, 255, 256, 70_001])
def test_pack_mask_is_little_endian_words_padded_with_zeros(nv, n):
    rng = np.random.default_rng(n)
    m = rng.random(n) < 0.4
    w = nv.pack_mask(m, n)
    assert w.dtype == np.uint32 and len(w) == (n + 31) // 32 == nv.mask_nwords(n)
    for j in list(range(min(n, 70))) + ([n - 1] if n else []):
        assert bool((int(w[j >> 5]) >> (j & 31)) & 1) == bool(m[j])
    if n % 32:
        assert int(w[-1]) >> (n % 32) == 0  # bits at or past n are zero (the library ignores them either way)
    assert np.array_equal(nv.unpack_mask(w, n), m)
    assert nv.pack_mask(w, n) is w or np.array_equal(nv.pack_mask(w, n), w)  # packed words pass through


def test_pack_mask_rejects_other_shapes_and_types(nv):
    with pytest.raises(ValueError):
        nv.pack_mask(np.ones(9, bool), 10)
    with pytest.raises(ValueError):
        nv.pack_mask(np.ones(10, np.int64), 10)
    with pytest.raises(ValueError):
        nv.pack_mask(np.zeros(2, np.uint32), 10)


def test_slice_mask_rebases_unaligned_shard_bounds(nv):
    from lotus_b200.distributed import shard_bounds
    n = 50_021
    m = np.random.default_rng(1).random(n) < 0.3
    w = nv.pack_mask(m, n)
    seen = 0
    for g in range(3):
        lo, hi = shard_bounds(n, 3, g)
        part = nv.slice_mask(w, n, lo, hi)
        assert len(part) == (hi - lo + 31) // 32 and np.array_equal(nv.unpack_mask(part, hi - lo), m[lo:hi])
        seen += hi - lo
    assert seen == n and any(shard_bounds(n, 3, g)[0] % 32 for g in range(3))


def test_ids_a_bitmap_can_stand_for(nv):
    assert nv.strictly_ascending(np.array([], np.int64)) and nv.strictly_ascending(np.array([7]))
    assert nv.strictly_ascending(np.array([0, 3, 4, 900]))
    assert not nv.strictly_ascending(np.array([0, 3, 3, 4]))  # a repeat is two rows of the temporary index
    assert not nv.strictly_ascending(np.array([0, 4, 3]))     # a permutation changes the tie order
    ids = np.array([0, 31, 32, 69])
    assert np.array_equal(np.flatnonzero(nv.unpack_mask(nv.ids_to_mask(ids, 70), 70)), ids)
    with pytest.raises(nv.NativeError) as e:
        nv.ids_to_mask(np.array([1, 70]), 70)
    assert e.value.code == nv.ERANGE


def test_subset_switch_is_validated_and_defaults_to_gather():
    import lotus_b200 as lotus
    assert lotus.B200VS().subset == "gather"
    for mode in ("mask", "auto"):
        assert lotus.B200VS(subset=mode).subset == mode
    with pytest.raises(ValueError, match="subset"):
        lotus.B200VS(subset="bitmap")


def test_auto_masks_only_where_the_gathered_copy_hurts(nv, monkeypatch):
    """subset="auto": a host-resident subset larger than the ring, or a device-resident one whose gathered copy does not fit in
    free device memory; never a permuted or repeating ids."""
    from types import SimpleNamespace
    import lotus_b200 as lotus
    from lotus_b200 import vs as vsmod
    free = {"bytes": 80 << 30}
    monkeypatch.setattr(vsmod, "_free_device_bytes", lambda device: free["bytes"])
    n, d = 1_000_000, 768
    ids = np.arange(0, n, 2)
    for mode, want_dev, want_tight, want_host in (("gather", False, False, False), ("mask", True, True, True), ("auto", False, True, True)):
        store = lotus.B200VS(subset=mode)
        store.b2_index = SimpleNamespace(n=n, d=d, dtype=nv.BF16, device=0, resident="device", ring_bytes=0)
        free["bytes"] = 80 << 30
        assert store._subset_by_mask(ids) == want_dev, mode
        free["bytes"] = (1 << 30) + 100 * d * 2  # room for a copy of 100 rows beyond the margin
        assert store._subset_by_mask(ids) == want_tight and store._subset_by_mask(ids[:50]) == (mode == "mask"), mode
        store.b2_index = SimpleNamespace(n=n, d=d, dtype=nv.BF16, device=0, resident="host", ring_bytes=384 << 20)
        assert store._subset_by_mask(ids) == want_host, mode  # 500k rows x 1536 B = 768 MB: twice the ring
        assert store._subset_by_mask(ids[:100_000]) == (mode == "mask"), mode
        assert not store._subset_by_mask(ids[::-1]) and not store._subset_by_mask(np.repeat(ids[:10], 2)), mode
        store.b2_index = None


def test_header_declares_the_masked_entry_points_and_the_library_exports_them(nv):
    header = open(os.path.join(ROOT, "include", "lotus_b200.h")).read()
    assert "#define B2_ABI_VERSION 1" in header
    L = nv.lib()
    for name in NEW:
        assert re.search(r"B2_API int %s\(" % name, header), name
        assert name in nv.SYMBOLS and hasattr(L, name)


def test_masked_entry_points_return_enodev_without_a_device(nv):
    if nv.device_count() != 0:
        pytest.skip("an H100 is visible")
    L = nv.lib()
    q = np.zeros((1, 8), np.float32)
    w = np.zeros(1, np.uint32)
    D, I = np.zeros((1, 1), np.float32), np.zeros((1, 1), np.int64)
    p = lambda a: ctypes.c_void_p(a.ctypes.data)  # noqa: E731
    assert L.b2_index_search_masked(None, p(q), 1, nv.F32, 1, p(w), p(D), p(I)) == nv.ENODEV
    assert "no CPU fallback" in L.b2_last_error().decode()
    assert L.b2_index_search_masked_dev(None, p(q), 1, nv.F32, 1, p(w), 0, p(D), p(I), None) == nv.ENODEV
