"""ctypes binding of libb2lotus.so (include/lotus_b200.h). No CPU fallback: if the library is not built or no
H100 is visible, calls raise — they never degrade to a host implementation."""
from __future__ import annotations

import ctypes
import os
from typing import Optional

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libb2lotus.so")

F32, BF16, F16 = 0, 1, 2
DTYPES = (F32, BF16, F16)  # the floating-point types
I8 = 8  # signed 8-bit integers (B2_I8), kept apart from the floating-point codes
METRIC_IP, METRIC_L2 = 0, 1
OK, EINVAL, ENODEV, ECUDA, ENOMEM, ERANGE = 0, -1, -2, -3, -4, -5

# every symbol include/lotus_b200.h declares (tests check the library exports all of them)
SYMBOLS = [
    "b2_abi_version", "b2_last_error", "b2_device_count", "b2_max_k", "b2_index_create", "b2_index_free",
    "b2_index_ntotal", "b2_index_dim", "b2_index_dtype", "b2_index_metric", "b2_index_device", "b2_index_data_dev",
    "b2_index_search", "b2_index_search_dev", "b2_merge_topk_dev", "b2_index_search_packed_dev", "b2_merge_topk_packed_dev", "b2_index_search_stage1_dev", "b2_index_search_stage2_packed_dev", "b2_index_gather", "b2_threshold_pairs",
    "b2_connected_components", "b2_kmeans", "b2_kmeans_assign", "b2_kmeans_accumulate", "b2_kmeans_assign_dev", "b2_kmeans_accumulate_dev", "b2_stats", "b2_stats_reset", "b2_last_filter_ms", "b2_host_f32_to_bf16", "b2_host_bf16_to_f32", "b2_debug_filter_plan",
    "b2_debug_filter_lists", "b2_debug_filter_eps", "b2_index_create_host", "b2_index_resident", "b2_debug_stream_plan",
    "b2_debug_stream_times", "b2_index_range_search", "b2_debug_range_stats",
    "b2_index_search_masked", "b2_index_search_masked_dev", "b2_debug_filter_lists_masked", "b2_index_range_search_masked",
]


class NativeError(RuntimeError):
    def __init__(self, code: int, msg: str):
        super().__init__(f"libb2lotus error {code}: {msg}")
        self.code = code
        self.msg = msg


_lib = None


def lib() -> ctypes.CDLL:
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise RuntimeError(
            f"{LIB_PATH} is missing: build it with `python -m lotus_b200.build` "
            "(lotus_b200 has no CPU fallback and refuses to run without its CUDA library)")
    L = ctypes.CDLL(LIB_PATH)
    c = ctypes
    vp, i32, i64, f32 = c.c_void_p, c.c_int32, c.c_int64, c.c_float
    L.b2_abi_version.restype = c.c_int
    L.b2_last_error.restype = c.c_char_p
    L.b2_device_count.restype = c.c_int
    L.b2_max_k.restype = c.c_int
    L.b2_index_create.restype = c.c_int
    L.b2_index_create.argtypes = [vp, i64, i32, i32, i32, i32, i32, c.POINTER(vp)]
    L.b2_index_create_host.restype = c.c_int
    L.b2_index_create_host.argtypes = [vp, i64, i32, i32, i32, i32, i64, c.POINTER(vp)]
    L.b2_index_resident.restype = i32
    L.b2_index_resident.argtypes = [vp]
    L.b2_debug_stream_plan.restype = c.c_int
    L.b2_debug_stream_plan.argtypes = [i64, i32, i32, i64, c.POINTER(i64), c.POINTER(i64), c.POINTER(i32)]
    L.b2_debug_stream_times.restype = c.c_int
    L.b2_debug_stream_times.argtypes = [vp, c.POINTER(f32)]
    L.b2_index_free.restype = None
    L.b2_index_free.argtypes = [vp]
    for name, rt in [("b2_index_ntotal", i64), ("b2_index_dim", i32), ("b2_index_dtype", i32),
                     ("b2_index_metric", i32), ("b2_index_device", i32), ("b2_index_data_dev", vp),
                     ("b2_last_filter_ms", f32)]:
        getattr(L, name).restype = rt
        getattr(L, name).argtypes = [vp]
    L.b2_index_search.restype = c.c_int
    L.b2_index_search.argtypes = [vp, vp, i64, i32, i32, vp, i64, vp, vp]
    L.b2_index_search_dev.restype = c.c_int
    L.b2_index_search_dev.argtypes = [vp, vp, i64, i32, i32, vp, i64, i64, vp, vp, vp]
    L.b2_index_search_masked.restype = c.c_int
    L.b2_index_search_masked.argtypes = [vp, vp, i64, i32, i32, vp, vp, vp]
    L.b2_index_search_masked_dev.restype = c.c_int
    L.b2_index_search_masked_dev.argtypes = [vp, vp, i64, i32, i32, vp, i64, vp, vp, vp]
    L.b2_debug_filter_lists_masked.restype = c.c_int
    L.b2_debug_filter_lists_masked.argtypes = [vp, vp, i64, i32, i32, i32, vp, c.POINTER(i32), c.POINTER(f32), vp, vp, vp]
    L.b2_merge_topk_dev.restype = c.c_int
    L.b2_merge_topk_dev.argtypes = [vp, vp, i32, i64, i32, i32, i32, vp, vp, vp]
    L.b2_index_search_packed_dev.restype = c.c_int
    L.b2_index_search_packed_dev.argtypes = [vp, vp, i64, i32, i32, vp, vp]
    L.b2_merge_topk_packed_dev.restype = c.c_int
    L.b2_merge_topk_packed_dev.argtypes = [vp, vp, i32, i64, i32, i32, i32, vp, vp, vp]
    L.b2_index_search_stage1_dev.restype = c.c_int
    L.b2_index_search_stage1_dev.argtypes = [vp, vp, i64, i32, i32, i32, vp, vp]
    L.b2_index_search_stage2_packed_dev.restype = c.c_int
    L.b2_index_search_stage2_packed_dev.argtypes = [vp, vp, vp, vp]
    L.b2_index_range_search.restype = c.c_int
    L.b2_index_range_search.argtypes = [vp, vp, i64, i32, f32, vp, i64, vp, vp, vp, i64, c.POINTER(i64)]
    L.b2_index_range_search_masked.restype = c.c_int
    L.b2_index_range_search_masked.argtypes = [vp, vp, i64, i32, f32, vp, vp, vp, vp, i64, c.POINTER(i64)]
    L.b2_debug_range_stats.restype = c.c_int
    L.b2_debug_range_stats.argtypes = [vp, c.POINTER(i64)]
    L.b2_index_gather.restype = c.c_int
    L.b2_index_gather.argtypes = [vp, vp, i64, vp, i32]
    L.b2_threshold_pairs.restype = c.c_int
    L.b2_threshold_pairs.argtypes = [vp, f32, i32, i32, vp, vp, i64, c.POINTER(i64)]
    L.b2_connected_components.restype = c.c_int
    L.b2_connected_components.argtypes = [i64, vp, vp, i64, i32, vp]
    L.b2_kmeans.restype = c.c_int
    L.b2_kmeans.argtypes = [vp, vp, i64, i32, i32, i64, i32, vp, vp, vp]
    L.b2_kmeans_assign.restype = c.c_int
    L.b2_kmeans_assign.argtypes = [vp, vp, i64, vp, i32, vp, vp]
    L.b2_kmeans_accumulate.restype = c.c_int
    L.b2_kmeans_accumulate.argtypes = [vp, vp, i64, vp, i32, vp, vp]
    L.b2_kmeans_assign_dev.restype = c.c_int
    L.b2_kmeans_assign_dev.argtypes = [vp, vp, i64, vp, i32, vp, vp, vp]
    L.b2_kmeans_accumulate_dev.restype = c.c_int
    L.b2_kmeans_accumulate_dev.argtypes = [vp, vp, i64, vp, i32, vp, vp, vp, vp, vp]
    L.b2_host_f32_to_bf16.restype = c.c_int
    L.b2_host_f32_to_bf16.argtypes = [vp, i64, vp, c.POINTER(i32)]
    L.b2_host_bf16_to_f32.restype = c.c_int
    L.b2_host_bf16_to_f32.argtypes = [vp, i64, vp]
    L.b2_debug_filter_plan.restype = c.c_int
    L.b2_debug_filter_plan.argtypes = [i64, i64, i32, i32, c.POINTER(i32), c.POINTER(i32), c.POINTER(i32), c.POINTER(i32)]
    L.b2_debug_filter_lists.restype = c.c_int
    L.b2_debug_filter_lists.argtypes = [vp, vp, i64, i32, i32, i32, i32, c.POINTER(i32), c.POINTER(f32), vp, vp, vp]
    L.b2_debug_filter_eps.restype = c.c_int
    L.b2_debug_filter_eps.argtypes = [i32, i32, i32, i32, c.POINTER(f32), c.POINTER(f32)]
    L.b2_stats.restype = c.c_int
    L.b2_stats.argtypes = [c.POINTER(i64), i32]
    L.b2_stats_reset.restype = None
    if L.b2_abi_version() != 1:
        raise RuntimeError("libb2lotus.so ABI version mismatch; rebuild with `python -m lotus_b200.build --force`")
    _lib = L
    return L


def check(rc: int) -> None:
    if rc != 0:
        raise NativeError(rc, lib().b2_last_error().decode("utf-8", "replace"))


def device_count() -> int:
    return int(lib().b2_device_count())


def require_device() -> None:
    if device_count() == 0:
        raise RuntimeError("lotus_b200 needs an H100 (sm_90) GPU; none is visible and there is no CPU fallback")


def filter_plan(nq: int, n: int, k: int, num_sms: int = 132) -> dict:
    """The filter kernel's schedule for a shape (host logic only, no device needed). two_cta: cluster mode, in which a query
    unit is two query tiles and a worker a CTA pair (num_sms / 2 of them); cluster: CTAs per cluster (a cluster of four runs
    two workers in lockstep)."""
    kp, ns, uw, cl = ctypes.c_int32(), ctypes.c_int32(), ctypes.c_int32(), ctypes.c_int32()
    check(lib().b2_debug_filter_plan(nq, n, k, num_sms, ctypes.byref(kp), ctypes.byref(ns), ctypes.byref(uw), ctypes.byref(cl)))
    return {"kp": kp.value, "n_splits": ns.value, "units_whole": uw.value, "two_cta": cl.value > 1, "cluster": cl.value}


def filter_eps(store_dtype: int, filt_dtype: int, q_dtype: int, d: int) -> tuple[float, float]:
    """(rel_eps, abs_eps) of the filter's error model for an operand combination (host logic only, no device needed)."""
    rel, ab = ctypes.c_float(), ctypes.c_float()
    check(lib().b2_debug_filter_eps(store_dtype, filt_dtype, q_dtype, d, ctypes.byref(rel), ctypes.byref(ab)))
    return float(rel.value), float(ab.value)


def stats() -> dict:
    buf = (ctypes.c_int64 * 8)()
    lib().b2_stats(buf, 8)
    return {"launches": buf[0], "queries": buf[1], "fallback_queries": buf[2], "filter_launches": buf[3],
            "rescored_rows": buf[4], "second_level_queries": buf[5], "streamed_bytes": buf[6], "streamed_chunks": buf[7]}


def stream_plan(n: int, d: int, dtype: int, ring_bytes: int = 0) -> dict:
    """Chunking of a host-resident index (host logic only, no device needed): chunk_rows, n_chunks, slots. Chunk c owns the
    rows [c * chunk_rows, min(n, (c + 1) * chunk_rows)) and streams chunk_rows rows from min(c * chunk_rows, n - chunk_rows)."""
    rows, nc, slots = ctypes.c_int64(), ctypes.c_int64(), ctypes.c_int32()
    check(lib().b2_debug_stream_plan(n, d, dtype, ring_bytes, ctypes.byref(rows), ctypes.byref(nc), ctypes.byref(slots)))
    return {"chunk_rows": rows.value, "n_chunks": nc.value, "slots": slots.value}


def stats_reset() -> None:
    lib().b2_stats_reset()


# ---- bf16 helpers (numpy has no bfloat16: bit patterns travel as uint16) ------------------------------------------
def f32_to_bf16_checked(a: np.ndarray, out: "np.ndarray | None" = None) -> tuple[np.ndarray, bool]:
    """Round-to-nearest-even float32 -> bfloat16 bit patterns (uint16; NaN stays a quiet NaN) plus whether every value
    was already bfloat16-representable. Host marshalling done by the library's threaded helper (no device work). `out`: a
    C-contiguous uint16 array of the same shape to write into (callers that convert a batch per call keep one: a fresh 150 MB
    array costs more in page faults than the conversion itself)."""
    a = np.ascontiguousarray(a, dtype=np.float32)
    if out is None or out.shape != a.shape or out.dtype != np.uint16 or not out.flags.c_contiguous:
        out = np.empty(a.shape, dtype=np.uint16)
    exact = ctypes.c_int32(0)
    check(lib().b2_host_f32_to_bf16(_ptr(a), a.size, _ptr(out), ctypes.byref(exact)))
    return out, bool(exact.value)


def f32_to_bf16_bits(a: np.ndarray) -> np.ndarray:
    """Round-to-nearest-even float32 -> bfloat16 bit patterns (uint16)."""
    return f32_to_bf16_checked(a)[0]


def bf16_bits_to_f32(b: np.ndarray) -> np.ndarray:
    b = np.ascontiguousarray(b, dtype=np.uint16)
    if b.size < (1 << 18):
        return (b.astype(np.uint32) << 16).view(np.float32).reshape(b.shape)
    out = np.empty(b.shape, dtype=np.float32)
    check(lib().b2_host_bf16_to_f32(_ptr(b), b.size, _ptr(out)))
    return out


def storage_dtype(code: int) -> np.dtype:
    """numpy dtype of a matrix's elements as the C-ABI holds them: float32, bfloat16 bit patterns (uint16; numpy has no
    bfloat16), float16 or int8."""
    if code == F32:
        return np.dtype(np.float32)
    if code == I8:
        return np.dtype(np.int8)
    if code == BF16:
        return np.dtype(np.uint16)
    if code == F16:
        return np.dtype(np.float16)
    raise ValueError(f"unknown element type code {code}")


def stored_to_f32(a: np.ndarray, code: int) -> np.ndarray:
    """float32 values of a matrix stored as element type `code` (exact for every type): the one place that knows how each
    type's storage turns into numbers."""
    if code == F32:
        return np.ascontiguousarray(a, dtype=np.float32)
    if code == BF16:
        return bf16_bits_to_f32(a)
    if code == F16:
        a = np.ascontiguousarray(a)
        return (a.view(np.float16) if a.dtype == np.uint16 else a.astype(np.float16, copy=False)).astype(np.float32)
    if code == I8:
        return np.ascontiguousarray(a, dtype=np.int8).astype(np.float32)
    raise ValueError(f"unknown element type code {code}")


# ---- row bitmaps of a masked search (host logic only) -------------------------------------------------------------------
def mask_nwords(n: int) -> int:
    return (int(n) + 31) // 32


def pack_mask(mask, n: int) -> np.ndarray:
    """The bitmap of a masked search over n rows as the C-ABI takes it: ceil(n / 32) uint32 words, bit j & 31 of word j >> 5
    set = row j takes part. `mask` is a bool array of length n, or such words already (returned as they are)."""
    a = np.asarray(mask)
    if a.dtype == np.uint32:
        if a.ndim != 1 or len(a) != mask_nwords(n):
            raise ValueError(f"a packed mask over {n} rows has {mask_nwords(n)} uint32 words, got shape {a.shape}")
        return np.ascontiguousarray(a)
    if a.dtype != np.bool_ or a.ndim != 1 or len(a) != n:
        raise ValueError(f"mask must be a bool array of length {n} or packed uint32 words, got {a.dtype} of shape {a.shape}")
    by = np.zeros(4 * mask_nwords(n), dtype=np.uint8)
    packed = np.packbits(a, bitorder="little")
    by[:len(packed)] = packed
    return by.view("<u4").astype(np.uint32, copy=False)


def unpack_mask(words: np.ndarray, n: int) -> np.ndarray:
    """bool[n] of packed mask words (the inverse of pack_mask)."""
    by = np.ascontiguousarray(words, dtype="<u4").view(np.uint8)
    return np.unpackbits(by, bitorder="little")[:n].astype(np.bool_)


def strictly_ascending(ids: np.ndarray) -> bool:
    """Whether ids has no repeats and is in ascending order: the order of such a subset is the row order, so a masked search
    over its bitmap has the tie semantics of the temporary index over x[ids]."""
    ids = np.asarray(ids)
    return len(ids) < 2 or bool((ids[1:] > ids[:-1]).all())


def ids_to_mask(ids: np.ndarray, n: int) -> np.ndarray:
    """Packed bitmap over n rows with the bits of `ids` set; ids outside [0, n) raise NativeError(ERANGE) like a search."""
    ids = np.asarray(ids, dtype=np.int64)
    if len(ids) and (ids.min() < 0 or ids.max() >= n):
        raise NativeError(ERANGE, f"ids contains a position outside [0, {n})")
    b = np.zeros(n, dtype=np.bool_)
    b[ids] = True
    return pack_mask(b, n)


def slice_mask(words: np.ndarray, n: int, lo: int, hi: int) -> np.ndarray:
    """The packed bitmap of the rows [lo, hi) of a bitmap over n rows, re-based so that row lo is bit 0 (shard bounds need not
    fall on word boundaries)."""
    return pack_mask(unpack_mask(words, n)[lo:hi], hi - lo)


def _ptr(a: Optional[np.ndarray]):
    return None if a is None else ctypes.c_void_p(a.ctypes.data)


class Index:
    """Owning wrapper of a b2_index handle."""

    def __init__(self, x, dtype: int, metric: int = METRIC_IP, device: int = 0, on_device_ptr: Optional[int] = None,
                 n: Optional[int] = None, d: Optional[int] = None, residency: str = "device", ring_bytes: int = 0):
        """residency="host": the rows stay in pinned host memory and searches stream them through a device ring of ring_bytes
        (0 = the library default); x must then be a host array."""
        L = lib()
        self._h = ctypes.c_void_p()
        if residency not in ("device", "host"):
            raise ValueError("residency must be 'device' or 'host'")
        if residency == "host" and on_device_ptr is not None:
            raise ValueError("a host-resident index is built from a host array")
        if on_device_ptr is not None:
            assert n is not None and d is not None
            check(L.b2_index_create(ctypes.c_void_p(on_device_ptr), n, d, dtype, metric, device, 1, ctypes.byref(self._h)))
        else:
            x = np.ascontiguousarray(x)
            want = storage_dtype(dtype)
            if dtype == F16 and x.dtype == np.uint16:  # fp16 bit patterns are accepted as well
                x = x.view(np.float16)
            if x.dtype != want:
                raise TypeError(f"matrix must be {want} for dtype {dtype}, got {x.dtype}")
            if x.ndim != 2:
                raise ValueError("matrix must be 2-D")
            n, d = x.shape
            if residency == "host":
                check(L.b2_index_create_host(_ptr(x) if n else None, n, d, dtype, metric, device, int(ring_bytes), ctypes.byref(self._h)))
            else:
                check(L.b2_index_create(_ptr(x) if n else None, n, d, dtype, metric, device, 0, ctypes.byref(self._h)))
        self.n, self.d, self.dtype, self.metric, self.device = int(n), int(d), dtype, metric, device
        self.ring_bytes = (int(ring_bytes) or (1 << 30)) if residency == "host" else 0  # 0 = the library default, 1 GiB

    def close(self) -> None:
        if getattr(self, "_h", None) is not None and self._h.value:
            lib().b2_index_free(self._h)
            self._h = ctypes.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    @property
    def handle(self):
        return self._h

    @property
    def resident(self) -> str:
        """Where the rows live: "device" or "host"."""
        return "host" if lib().b2_index_resident(self._h) == 1 else "device"

    def stream_times(self) -> dict:
        """CUDA-event times (ms) of the last search of a host-resident index (b2_debug_stream_times)."""
        t = (ctypes.c_float * 4)()
        check(lib().b2_debug_stream_times(self._h, t))
        return {"copy_ms": t[0], "span_ms": t[1], "filter_ms": t[2], "finalize_ms": t[3]}

    @property
    def data_ptr(self) -> int:
        return int(lib().b2_index_data_dev(self._h) or 0)

    def search(self, q: np.ndarray, k: int, q_dtype: int = F32, ids: Optional[np.ndarray] = None):
        """Host buffers in, host buffers out: (scores[nq,k] float32, idx[nq,k] int64)."""
        q = np.ascontiguousarray(q)
        nq = q.shape[0]
        if nq and q.shape[1] != self.d:
            raise ValueError(f"query dimension {q.shape[1]} != index dimension {self.d}")
        D = np.empty((nq, k), dtype=np.float32)
        I = np.empty((nq, k), dtype=np.int64)
        ids_a = None if ids is None else np.ascontiguousarray(ids, dtype=np.int64)
        check(lib().b2_index_search(self._h, _ptr(q) if nq else None, nq, q_dtype, k, _ptr(ids_a),
                                    0 if ids_a is None else len(ids_a), _ptr(D), _ptr(I)))
        return D, I

    def search_masked(self, q: np.ndarray, k: int, q_dtype: int, mask):
        """search(q, k, q_dtype, ids=np.flatnonzero(mask)), bit for bit, without a gathered copy of the subset: the filter sweeps
        the whole index and leaves the cleared rows out. mask: bool[n], or packed uint32 words (pack_mask)."""
        q = np.ascontiguousarray(q)
        nq = q.shape[0]
        if nq and q.shape[1] != self.d:
            raise ValueError(f"query dimension {q.shape[1]} != index dimension {self.d}")
        words = pack_mask(mask, self.n)
        D = np.empty((nq, k), dtype=np.float32)
        I = np.empty((nq, k), dtype=np.int64)
        check(lib().b2_index_search_masked(self._h, _ptr(q) if nq else None, nq, q_dtype, k, _ptr(words) if self.n else None,
                                           _ptr(D), _ptr(I)))
        return D, I

    def search_masked_dev(self, q_ptr: int, nq: int, k: int, q_dtype: int, mask_ptr: int, out_scores_ptr: int, out_idx_ptr: int,
                          id_offset: int = 0, stream: int = 0) -> None:
        check(lib().b2_index_search_masked_dev(self._h, ctypes.c_void_p(q_ptr), nq, q_dtype, k, ctypes.c_void_p(mask_ptr), id_offset,
                                               ctypes.c_void_p(out_scores_ptr), ctypes.c_void_p(out_idx_ptr),
                                               ctypes.c_void_p(stream) if stream else None))

    def range_search(self, q: np.ndarray, radius: float, q_dtype: int = F32, ids: Optional[np.ndarray] = None,
                     cap: Optional[int] = None):
        """faiss IndexFlat.range_search: (lims[nq+1] int64, D[lims[nq]] float32, I[lims[nq]] int64), query i's hits at
        [lims[i], lims[i+1]) in ascending row id (with ids: in the order of `ids`, reported as the original ids). IP keeps the
        rows scoring strictly above `radius`, L2 those strictly closer than it (squared distance). Host buffers; when the
        result outgrows `cap` the call is repeated once with the exact size."""
        q = np.ascontiguousarray(q)
        nq = q.shape[0]
        if nq and q.shape[1] != self.d:
            raise ValueError(f"query dimension {q.shape[1]} != index dimension {self.d}")
        ids_a = None if ids is None else np.ascontiguousarray(ids, dtype=np.int64)
        return self._range_call(nq, cap, lambda lims, D, I, cap, total: lib().b2_index_range_search(
            self._h, _ptr(q) if nq else None, nq, q_dtype, float(radius), _ptr(ids_a), 0 if ids_a is None else len(ids_a),
            _ptr(lims), _ptr(D), _ptr(I), cap, total))

    def range_search_masked(self, q: np.ndarray, radius: float, q_dtype: int, mask, cap: Optional[int] = None):
        """range_search(q, radius, q_dtype, ids=np.flatnonzero(mask)), bit for bit, without a gathered copy of the subset: the
        range filter sweeps the whole index and only the selected rows become candidates. mask: bool[n], or packed uint32
        words (pack_mask). Hits are reported by row id."""
        q = np.ascontiguousarray(q)
        nq = q.shape[0]
        if nq and q.shape[1] != self.d:
            raise ValueError(f"query dimension {q.shape[1]} != index dimension {self.d}")
        words = pack_mask(mask, self.n)
        return self._range_call(nq, cap, lambda lims, D, I, cap, total: lib().b2_index_range_search_masked(
            self._h, _ptr(q) if nq else None, nq, q_dtype, float(radius), _ptr(words) if self.n else None,
            _ptr(lims), _ptr(D), _ptr(I), cap, total))

    @staticmethod
    def _range_call(nq: int, cap: Optional[int], call):
        """Runs call(lims, D, I, cap, byref(total)) of a range search entry point into host buffers, once more with the exact
        size when the result outgrows `cap`, and returns (lims, D, I)."""
        lims = np.zeros(nq + 1, dtype=np.int64)
        cap = int(cap) if cap is not None else max(1 << 16, 64 * nq)
        for attempt in range(2):
            D = np.empty(cap, dtype=np.float32)
            I = np.empty(cap, dtype=np.int64)
            total = ctypes.c_int64(0)
            rc = call(lims, D, I, cap, ctypes.byref(total))
            if rc == ERANGE and attempt == 0 and total.value > cap:
                cap = int(total.value)
                continue
            check(rc)
            break
        m = int(total.value)
        return lims, D[:m].copy(), I[:m].copy()

    def range_stats(self) -> dict:
        """Counts of the last range_search or range_search_masked (b2_debug_range_stats)."""
        out = (ctypes.c_int64 * 4)()
        check(lib().b2_debug_range_stats(self._h, out))
        return {"candidates_peak": out[0], "hits": out[1], "dense_queries": out[2], "filtered": bool(out[3])}

    def search_dev(self, q_ptr: int, nq: int, k: int, q_dtype: int, out_scores_ptr: int, out_idx_ptr: int,
                   id_offset: int = 0, ids_ptr: Optional[int] = None, n_ids: int = 0, stream: int = 0) -> None:
        check(lib().b2_index_search_dev(self._h, ctypes.c_void_p(q_ptr), nq, q_dtype, k,
                                        ctypes.c_void_p(ids_ptr) if ids_ptr else None, n_ids, id_offset,
                                        ctypes.c_void_p(out_scores_ptr), ctypes.c_void_p(out_idx_ptr),
                                        ctypes.c_void_p(stream) if stream else None))

    def search_packed_dev(self, q_ptr: int, nq: int, k: int, q_dtype: int, out_packed_ptr: int, stream: int = 0) -> None:
        """Whole-index search, result as one uint64 per entry (float32 score bits << 32 | local row id, 0xffffffff = none)."""
        check(lib().b2_index_search_packed_dev(self._h, ctypes.c_void_p(q_ptr), nq, q_dtype, k, ctypes.c_void_p(out_packed_ptr),
                                               ctypes.c_void_p(stream) if stream else None))

    def search_stage1_dev(self, q_ptr: int, nq: int, k: int, q_dtype: int, j: int, lower_ptr: int, stream: int = 0) -> None:
        check(lib().b2_index_search_stage1_dev(self._h, ctypes.c_void_p(q_ptr), nq, q_dtype, k, j, ctypes.c_void_p(lower_ptr),
                                               ctypes.c_void_p(stream) if stream else None))

    def search_stage2_packed_dev(self, hint_ptr: int, out_packed_ptr: int, stream: int = 0) -> None:
        check(lib().b2_index_search_stage2_packed_dev(self._h, ctypes.c_void_p(hint_ptr), ctypes.c_void_p(out_packed_ptr),
                                                      ctypes.c_void_p(stream) if stream else None))

    def gather(self, ids) -> np.ndarray:
        ids = np.ascontiguousarray(ids, dtype=np.int64)
        out = np.empty((len(ids), self.d), dtype=storage_dtype(self.dtype))
        check(lib().b2_index_gather(self._h, _ptr(ids), len(ids), _ptr(out), 0))
        return out

    def filter_lists(self, q: np.ndarray, k: int, q_dtype: int = F32, top1: bool = False, level: int = 0,
                     plan_only: bool = False, mask=None) -> dict:
        """The filter kernel's raw candidate lists for host queries, run as a search (or, with top1, the k-means assignment)
        runs it: the plan (use_filter, kp, n_splits, units_whole, two_cta, cluster, two_level, filt_dtype, rel_eps) plus, unless
        plan_only or the plan declines the filter, score/id [nq, n_splits, 2, kp/2] and thr [nq, n_splits, 2]. mask: the
        lists of a masked search (search_masked) instead."""
        q = np.ascontiguousarray(q)
        nq = q.shape[0]
        if q.ndim != 2 or q.shape[1] != self.d:
            raise ValueError(f"queries must be [nq, {self.d}]")
        plan = (ctypes.c_int32 * 8)()
        eps = ctypes.c_float()
        L = lib()
        if mask is not None:
            if top1:
                raise ValueError("the k-means assignment takes no mask")
            words = pack_mask(mask, self.n)

            def run(*bufs):
                return L.b2_debug_filter_lists_masked(self._h, _ptr(q), nq, q_dtype, k, level, _ptr(words), plan, ctypes.byref(eps), *bufs)
        else:
            def run(*bufs):
                return L.b2_debug_filter_lists(self._h, _ptr(q), nq, q_dtype, k, int(top1), level, plan, ctypes.byref(eps), *bufs)
        check(run(None, None, None))
        out = {"use_filter": bool(plan[0]), "kp": plan[1], "n_splits": plan[2], "units_whole": plan[3], "two_cta": plan[4] > 1,
               "cluster": plan[4],
               "two_level": bool(plan[5]), "filt_dtype": plan[6], "rel_eps": float(eps.value)}
        if plan_only or not out["use_filter"]:
            return out
        ns, kph = out["n_splits"], out["kp"] // 2
        sc = np.empty((nq, ns, 2, kph), dtype=np.float32)
        ids = np.empty((nq, ns, 2, kph), dtype=np.int32)
        thr = np.empty((nq, ns, 2), dtype=np.float32)
        check(run(_ptr(sc), _ptr(ids), _ptr(thr)))
        out.update(score=sc, id=ids, thr=thr)
        return out

    def last_filter_ms(self) -> float:
        return float(lib().b2_last_filter_ms(self._h))

    def threshold_pairs(self, thr: float, cap: int = 1 << 24, part: int = 0, nparts: int = 1):
        oi = np.empty(cap, dtype=np.int64)
        oj = np.empty(cap, dtype=np.int64)
        cnt = ctypes.c_int64(0)
        rc = lib().b2_threshold_pairs(self._h, float(thr), part, nparts, _ptr(oi), _ptr(oj), cap, ctypes.byref(cnt))
        if rc == ERANGE and cnt.value > cap:
            return self.threshold_pairs(thr, cap=int(cnt.value), part=part, nparts=nparts)
        check(rc)
        m = int(cnt.value)
        return oi[:m].copy(), oj[:m].copy()

    def kmeans(self, k: int, niter: int = 20, seed: int = 1234, ids=None, full_lloyd: bool = False):
        ids_a = None if ids is None else np.ascontiguousarray(ids, dtype=np.int64)
        m = self.n if ids_a is None else len(ids_a)
        assign = np.empty(m, dtype=np.int64)
        cent = np.empty((k, self.d), dtype=np.float32)
        obj = np.zeros(max(niter, 1), dtype=np.float32)
        check(lib().b2_kmeans(self._h, _ptr(ids_a), m, k, niter, seed, int(full_lloyd), _ptr(assign), _ptr(cent), _ptr(obj)))
        return assign, cent, obj[:niter]

    def kmeans_assign(self, centroids: np.ndarray, ids=None):
        c = np.ascontiguousarray(centroids, dtype=np.float32)
        ids_a = None if ids is None else np.ascontiguousarray(ids, dtype=np.int64)
        m = self.n if ids_a is None else len(ids_a)
        assign = np.empty(m, dtype=np.int64)
        dist = np.empty(m, dtype=np.float32)
        check(lib().b2_kmeans_assign(self._h, _ptr(ids_a), m, _ptr(c), c.shape[0], _ptr(assign), _ptr(dist)))
        return assign, dist


def merge_topk_packed_dev(packed_ptr: int, shard_offsets, g: int, nq: int, k: int, metric: int, device: int,
                          out_scores_ptr: int, out_idx_ptr: int, stream: int = 0) -> None:
    offs = np.ascontiguousarray(shard_offsets, dtype=np.int64)
    assert len(offs) == g
    check(lib().b2_merge_topk_packed_dev(ctypes.c_void_p(packed_ptr), _ptr(offs), g, nq, k, metric, device,
                                         ctypes.c_void_p(out_scores_ptr), ctypes.c_void_p(out_idx_ptr),
                                         ctypes.c_void_p(stream) if stream else None))


def _index_kmeans_assign_dev(self, centroids_ptr: int, k: int, assign_ptr: int, dist_ptr: int = 0, ids_ptr: int = 0, m: int = 0,
                             stream: int = 0) -> None:
    """DEVICE buffers: assign[m] int64 (and dist[m] float32 when dist_ptr) against centroids[k,d] float32."""
    check(lib().b2_kmeans_assign_dev(self._h, ctypes.c_void_p(ids_ptr) if ids_ptr else None, m, ctypes.c_void_p(centroids_ptr), k,
                                     ctypes.c_void_p(assign_ptr), ctypes.c_void_p(dist_ptr) if dist_ptr else None,
                                     ctypes.c_void_p(stream) if stream else None))


def _index_kmeans_accumulate_dev(self, assign_ptr: int, k: int, sums_ptr: int, counts_ptr: int, centroids_ptr: int = 0, obj_ptr: int = 0,
                                 ids_ptr: int = 0, m: int = 0, stream: int = 0) -> None:
    """DEVICE buffers: per-shard point-order sums[k,d] + counts[k] (float32); *obj += sum of squared distances (float64)."""
    check(lib().b2_kmeans_accumulate_dev(self._h, ctypes.c_void_p(ids_ptr) if ids_ptr else None, m, ctypes.c_void_p(assign_ptr), k,
                                         ctypes.c_void_p(centroids_ptr) if centroids_ptr else None, ctypes.c_void_p(sums_ptr),
                                         ctypes.c_void_p(counts_ptr), ctypes.c_void_p(obj_ptr) if obj_ptr else None,
                                         ctypes.c_void_p(stream) if stream else None))


def pair_owner(i, nparts: int):
    """Rank that owns the pairs (i, j > i) in `threshold_pairs(part=, nparts=)`: 128-row query tiles are dealt to the ranks in
    groups of one tile per SM (132 on H100; B2_PAIR_GROUP overrides) — mirrors launch_pair_filter in knn_filter_sm90.cu."""
    group = int(os.environ.get("B2_PAIR_GROUP", "0")) or 132
    tile = np.asarray(i, dtype=np.int64) // 128
    if int(os.environ.get("B2_PAIR_2CTA", "1")):  # CTA pairs (default): the unit is two consecutive query tiles, one unit per pair of SMs
        return ((tile // 2) // max(1, group // 2)) % nparts
    return (tile // group) % nparts


def _index_kmeans_accumulate(self, assign, k: int, ids=None):
    """Per-shard centroid sums [k,d] (point order, fp32, not normalised) and counts [k] for multi-GPU Lloyd."""
    a = np.ascontiguousarray(assign, dtype=np.int64)
    ids_a = None if ids is None else np.ascontiguousarray(ids, dtype=np.int64)
    sums = np.empty((k, self.d), dtype=np.float32)
    counts = np.empty(k, dtype=np.float32)
    check(lib().b2_kmeans_accumulate(self._h, _ptr(ids_a), len(a), _ptr(a), k, _ptr(sums), _ptr(counts)))
    return sums, counts


Index.kmeans_accumulate = _index_kmeans_accumulate
Index.kmeans_assign_dev = _index_kmeans_assign_dev
Index.kmeans_accumulate_dev = _index_kmeans_accumulate_dev


def connected_components(n: int, pi: np.ndarray, pj: np.ndarray, device: int = 0) -> np.ndarray:
    pi = np.ascontiguousarray(pi, dtype=np.int64)
    pj = np.ascontiguousarray(pj, dtype=np.int64)
    labels = np.empty(n, dtype=np.int64)
    check(lib().b2_connected_components(n, _ptr(pi), _ptr(pj), len(pi), device, _ptr(labels)))
    return labels


def merge_topk_dev(scores_ptr: int, idx_ptr: int, g: int, nq: int, k: int, metric: int, device: int,
                   out_scores_ptr: int, out_idx_ptr: int, stream: int = 0) -> None:
    check(lib().b2_merge_topk_dev(ctypes.c_void_p(scores_ptr), ctypes.c_void_p(idx_ptr), g, nq, k, metric, device,
                                  ctypes.c_void_p(out_scores_ptr), ctypes.c_void_p(out_idx_ptr),
                                  ctypes.c_void_p(stream) if stream else None))
