"""Masked range search without a GPU: the header's declaration and the binding, B2_ENODEV from the entry point on a machine
without an H100, the definition a masked range search must match (the oracle over the selected rows, reported by row id), and
the host-side logic of the Python layers against fakes: which call `B200VS.range_search` makes under each `subset` mode, and
the shard combination of `MultiDeviceIndex.range_search_masked` over shard bounds that are not word-aligned."""
import ctypes
import os
import re

import numpy as np
import pytest

import oracle
from helpers import grid
from range_oracle import range_search as oracle_range

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def masked_oracle(x, q, radius, metric, mask):
    """The masked range search's definition: the oracle over x[flatnonzero(mask)], each hit's position mapped to its row."""
    rows = np.flatnonzero(mask)
    lims, D, pos = oracle_range(np.asarray(x)[rows].reshape(len(rows), np.asarray(x).shape[1]), q, radius, metric)
    return lims, D, rows[pos]


def equal(a, b):
    return all(np.array_equal(u, v) for u, v in zip(a, b)) and np.array_equal(a[1].view(np.uint32), b[1].view(np.uint32))


def test_header_declares_the_entry_point_and_the_library_exports_it(nv):
    header = open(os.path.join(ROOT, "include", "lotus_b200.h")).read()
    assert "#define B2_ABI_VERSION 1" in header
    m = re.search(r"B2_API int b2_index_range_search_masked\(([^)]*)\)", header)
    assert m, "b2_index_range_search_masked is not declared"
    params = [p.strip() for p in m.group(1).replace("\n", " ").split(",")]
    assert params == ["b2_index* idx", "const void* q", "int64_t nq", "int32_t q_dtype", "float radius", "const uint32_t* mask",
                      "int64_t* lims", "float* out_d", "int64_t* out_i", "int64_t cap", "int64_t* n_results"], params
    L = nv.lib()
    assert "b2_index_range_search_masked" in nv.SYMBOLS and hasattr(L, "b2_index_range_search_masked")
    assert len(L.b2_index_range_search_masked.argtypes) == len(params)


def test_entry_point_returns_enodev_without_a_device(nv):
    if nv.device_count() != 0:
        pytest.skip("an H100 is visible")
    L = nv.lib()
    q = np.zeros((1, 8), np.float32)
    w = np.zeros(1, np.uint32)
    lims = np.zeros(2, np.int64)
    D, I = np.zeros(4, np.float32), np.zeros(4, np.int64)
    total = ctypes.c_int64(0)
    p = lambda a: ctypes.c_void_p(a.ctypes.data)  # noqa: E731
    rc = L.b2_index_range_search_masked(None, p(q), 1, nv.F32, 0.5, p(w), p(lims), p(D), p(I), 4, ctypes.byref(total))
    assert rc == nv.ENODEV
    assert "no CPU fallback" in L.b2_last_error().decode()


@pytest.mark.parametrize("metric", [oracle.IP, oracle.L2])
def test_masked_oracle_is_the_oracle_over_the_selected_rows(nv, metric):
    x, q = grid(333, 16, 1), grid(9, 16, 2)
    r = 0.02 if metric == oracle.IP else 0.3
    rng = np.random.default_rng(3)
    full = oracle_range(x, q, r, metric)
    for mask in (rng.random(333) < 0.4, np.ones(333, bool), np.zeros(333, bool), np.arange(333) == 332):
        got = masked_oracle(x, q, r, metric, mask)
        assert equal(got, oracle_range(x, q, r, metric, ids=np.flatnonzero(mask)))  # = the gathered search, ids ascending
        keep = mask[full[2]]  # = the full search with the cleared rows' hits dropped, row order kept
        qs = np.repeat(np.arange(len(q)), np.diff(full[0]))
        lims = np.zeros(len(q) + 1, np.int64)
        np.cumsum(np.bincount(qs[keep], minlength=len(q)), out=lims[1:])
        assert equal(got, (lims, full[1][keep], full[2][keep]))
    assert masked_oracle(x, q, r, metric, np.zeros(333, bool))[0].tolist() == [0] * 10


class RecordingIndex:
    """A fake native index that records which range search it was asked for and answers it through the oracle."""

    def __init__(self, nv, x, metric, resident="device", ring_bytes=0):
        self.nv, self.x, self.metric = nv, x, metric
        self.n, self.d, self.dtype, self.device = x.shape[0], x.shape[1], nv.F32, 0
        self.resident, self.ring_bytes = resident, ring_bytes
        self.calls = []

    def range_search(self, q, radius, q_dtype=0, ids=None):
        self.calls.append("ids" if ids is not None else "whole")
        return oracle_range(self.x, q, radius, self.metric, ids=ids)

    def range_search_masked(self, q, radius, q_dtype, mask):
        self.calls.append("mask")
        return masked_oracle(self.x, q, radius, self.metric, self.nv.unpack_mask(self.nv.pack_mask(mask, self.n), self.n))


def test_b200vs_range_search_follows_the_subset_switch(nv, monkeypatch):
    from lotus_b200 import vs as vsmod
    x, q = grid(400, 8, 4), grid(5, 8, 5)
    r = 0.0
    monkeypatch.setattr(vsmod, "_free_device_bytes", lambda device: 80 << 30)
    asc = np.arange(0, 400, 3)
    perm, rep = asc[::-1].copy(), np.repeat(asc[:20], 2)
    for mode, want_asc in (("gather", "ids"), ("mask", "mask"), ("auto", "ids")):
        store = vsmod.B200VS(subset=mode)
        store.b2_index, store.index_dir = RecordingIndex(nv, x, oracle.IP), "/nonexistent"
        assert equal(store.range_search(q, r, ids=asc), oracle_range(x, q, r, oracle.IP, ids=asc)), mode
        assert equal(store.range_search(q, r, ids=list(perm)), oracle_range(x, q, r, oracle.IP, ids=perm)), mode
        assert equal(store.range_search(q, r, ids=rep), oracle_range(x, q, r, oracle.IP, ids=rep)), mode
        assert equal(store.range_search(q, r), oracle_range(x, q, r, oracle.IP)), mode
        assert store.b2_index.calls == [want_asc, "ids", "ids", "whole"], (mode, store.b2_index.calls)
    # "auto" takes the bitmap for a host-resident subset larger than the ring (400 rows x 32 B > 1 KB)
    store = vsmod.B200VS(subset="auto")
    store.b2_index, store.index_dir = RecordingIndex(nv, x, oracle.IP, resident="host", ring_bytes=1024), "/nonexistent"
    assert equal(store.range_search(q, r, ids=asc), oracle_range(x, q, r, oracle.IP, ids=asc))
    store.range_search(q, r, ids=asc[:10])
    assert store.b2_index.calls == ["mask", "ids"]


def test_b200vs_range_search_masked_always_takes_the_bitmap(nv):
    from lotus_b200.vs import B200VS
    x, q = grid(300, 8, 6), grid(4, 8, 7)
    store = B200VS()
    with pytest.raises(ValueError, match="Index not loaded"):
        store.range_search_masked(q, 0.0, np.ones(300, bool))
    store.b2_index, store.index_dir = RecordingIndex(nv, x, oracle.L2), "/nonexistent"
    mask = np.random.default_rng(8).random(300) < 0.3
    assert equal(store.range_search_masked(q, 0.2, mask), masked_oracle(x, q, 0.2, oracle.L2, mask))
    assert equal(store.range_search_masked(q, 0.2, list(mask.astype(int))), masked_oracle(x, q, 0.2, oracle.L2, mask))
    assert store.b2_index.calls == ["mask", "mask"]
    with pytest.raises(ValueError, match="mask"):
        store.range_search_masked(q, 0.2, mask[:-1])
    with pytest.raises(ValueError, match="dimension"):
        store.range_search_masked(q[:, :4], 0.2, mask)
    s2 = B200VS(subset="mask")
    s2.b2_index, s2.index_dir = RecordingIndex(nv, x, oracle.L2), "/nonexistent"
    with pytest.raises(ValueError, match="outside"):  # an id past the index, on its way into the bitmap
        s2.range_search(q, 0.2, ids=np.array([1, 300]))
    assert s2.b2_index.calls == []


class FakeShard:
    def __init__(self, nv, x, metric):
        self.nv, self.x, self.metric = nv, x, metric

    def range_search_masked(self, q, radius, q_dtype, mask):
        n = self.x.shape[0]
        assert np.asarray(mask).dtype == np.uint32 and len(mask) == (n + 31) // 32  # the shard's own, re-based words
        return masked_oracle(self.x, q, radius, self.metric, self.nv.unpack_mask(mask, n))


@pytest.mark.parametrize("metric", [oracle.IP, oracle.L2])
def test_multi_device_combination_over_unaligned_shard_bounds(nv, metric):
    from concurrent.futures import ThreadPoolExecutor
    from lotus_b200.distributed import shard_bounds
    from lotus_b200.vs import MultiDeviceIndex
    n = 1001
    x, q = grid(n, 12, 9), grid(6, 12, 10)
    r = 0.02 if metric == oracle.IP else 0.3
    md = object.__new__(MultiDeviceIndex)
    md.n, md.d, md.metric = n, x.shape[1], metric
    md.bounds = [shard_bounds(n, 3, g) for g in range(3)]
    assert any(lo % 32 for lo, _ in md.bounds)
    md.shards = [FakeShard(nv, x[lo:hi], metric) for lo, hi in md.bounds]
    md.pool = ThreadPoolExecutor(3)
    rng = np.random.default_rng(11)
    for mask in (rng.random(n) < 0.5, rng.random(n) < 0.02, np.ones(n, bool), np.zeros(n, bool)):
        want = masked_oracle(x, q, r, metric, mask)
        assert equal(md.range_search_masked(q, r, 0, mask), want)
        assert equal(md.range_search_masked(q, r, 0, nv.pack_mask(mask, n)), want)
    md.pool.shutdown()
