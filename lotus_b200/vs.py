"""Vector-store boundary: the `VS` ABC of the reference (lotus/vector_store/vs.py:10-58) and `B200VS`, the
drop-in replacement of `FaissVS` (lotus/vector_store/faiss_vs.py:13-77) backed by libb2lotus.so.

    lotus.settings.configure(rm=rm, vs=B200VS())          # where the reference says vs=FaissVS()

There is no CPU path: without the CUDA library / an H100 every method that computes raises.
"""
from __future__ import annotations

import os
from abc import ABC, abstractmethod
from collections import OrderedDict
from typing import Any

import numpy as np

from . import _native as nv
from . import faiss_io
from .types import RMOutput

try:  # when the real package is importable, plug into ITS class hierarchy so isinstance checks pass
    from lotus.vector_store.vs import VS as _RefVS  # type: ignore
    from lotus.types import RMOutput as _RefRMOutput  # type: ignore
    RMOutput = _RefRMOutput  # noqa: F811
except Exception:  # lotus (litellm, faiss, ...) is not importable in this image: mirror the ABC
    _RefVS = None

METRIC_INNER_PRODUCT = faiss_io.METRIC_INNER_PRODUCT  # == faiss.METRIC_INNER_PRODUCT
METRIC_L2 = faiss_io.METRIC_L2  # == faiss.METRIC_L2

if _RefVS is not None:
    VS = _RefVS
else:

    class VS(ABC):  # type: ignore[no-redef]
        """Abstract class for vector stores (lotus/vector_store/vs.py:10-58)."""

        def __init__(self) -> None:
            self.index_dir: str | None = None

        @abstractmethod
        def index(self, docs: Any, embeddings: Any, index_dir: str, **kwargs: Any):
            ...

        @abstractmethod
        def load_index(self, index_dir: str):
            ...

        @abstractmethod
        def __call__(self, query_vectors: Any, K: int, ids: list[int] | None = None, **kwargs: Any) -> RMOutput:
            ...

        @abstractmethod
        def get_vectors_from_index(self, index_dir: str, ids: list[int]) -> Any:
            ...


def _cuda_tensor(a: Any):
    """The tensor itself when `a` is a torch CUDA tensor (device hand-off, SURVEY §8f-2), else None."""
    try:
        import torch
        if isinstance(a, torch.Tensor) and a.is_cuda:
            return a
    except ImportError:  # pragma: no cover
        pass
    return None


class BF16Backed(np.ndarray):
    """float32 matrix handed out by `B200VS.get_vectors_from_index` for bf16 indexes. It is a plain float32 array to every
    caller; the name only records where it came from. (Round 1 carried the bf16 bit patterns along as an attribute; an
    in-place edit such as `q /= norm` left them stale. `B200VS.__call__` now re-derives the 2-byte form from the VALUES —
    see `_to_host_matrix(exact_bf16_ok=True)` — so nothing can go stale.)"""

    @staticmethod
    def wrap(f32: np.ndarray, bits: "np.ndarray | None" = None) -> "BF16Backed":
        return np.ascontiguousarray(f32, dtype=np.float32).view(BF16Backed)


def f32_to_f16_checked(f: np.ndarray) -> np.ndarray:
    """float32 -> float16, round to nearest even. A finite value that would overflow to inf raises ValueError (|v| >= 65520):
    an fp16 store must hold the user's numbers, not infinities."""
    with np.errstate(over="ignore"):
        h = f.astype(np.float16)
    bad = np.isinf(h) & np.isfinite(f)
    if bad.any():
        v = f[bad].flat[0]
        raise ValueError(f"value {v!r} is outside the float16 range (|v| < 65520); use dtype='f32' or 'bf16' for these embeddings")
    return h


def _as_int8(a: Any) -> np.ndarray:
    """The int8 matrix holding exactly the values of `a` (numpy or torch, any numeric type): every value must be an integer in
    [-128, 127], otherwise ValueError. The store never picks a quantization scale."""
    try:
        import torch
        if isinstance(a, torch.Tensor):
            a = a.detach().cpu().numpy() if a.dtype != torch.bfloat16 else a.detach().to(torch.float32).cpu().numpy()
    except ImportError:  # pragma: no cover
        pass
    arr = np.asarray(a)
    if arr.ndim != 2:
        raise ValueError(f"embeddings must be 2-D, got shape {arr.shape}")
    if arr.dtype == np.int8:
        return np.ascontiguousarray(arr)
    if arr.dtype.kind not in "iuf" or arr.dtype.kind == "f" and not np.isfinite(arr).all():
        raise ValueError(f"dtype='i8' needs integer values in [-128, 127]; got {arr.dtype} data")
    if arr.size and (arr.min() < -128 or arr.max() > 127 or (arr.dtype.kind == "f" and not (arr == np.round(arr)).all())):
        raise ValueError("dtype='i8' needs integer values in [-128, 127] (quantize the embeddings first; the store never "
                         "picks a scale)")
    return np.ascontiguousarray(arr, dtype=np.int8)


def _to_host_matrix(a: Any, want_bf16: bool, exact_bf16_ok: bool = False, scratch: "dict | None" = None,
                    want_f16: bool = False, pass_f16: bool = False, want_i8: bool = False, pass_i8: bool = False):
    """-> (array for the C-ABI, native dtype code, float32 view of the stored values).
    exact_bf16_ok: when every float32 value is bfloat16-representable (e.g. vectors fetched from a bf16 index,
    sem_sim_join.py:112-118 -> :130-134) ship the exact 2-byte patterns instead: half the H2D bytes and the exact-operand
    error bound in the certificate. Decided from the values themselves on every call (one threaded host pass).
    want_f16: store as float16 (float16 input as it is, anything else rounded once; overflow raises ValueError).
    pass_f16: float16 input (numpy or torch) is shipped as it is, as 2-byte F16 operands (queries: exact in fp32).
    want_i8: store as int8 (integer values in [-128, 127] only, see _as_int8).
    pass_i8: int8 input (numpy or torch) is shipped as it is, as 1-byte I8 operands (queries: exact on every store)."""
    if want_i8:
        x = _as_int8(a)
        return x, nv.I8, x.astype(np.float32)
    try:
        import torch
        if isinstance(a, torch.Tensor):
            t = a.detach()
            if t.dtype == torch.int8 and pass_i8:
                x = np.ascontiguousarray(t.cpu().numpy())
                return x, nv.I8, x.astype(np.float32)
            if t.dtype == torch.float16 and (want_f16 or pass_f16) and not want_bf16:
                a = t.contiguous().cpu().numpy()  # float16 ndarray: handled below
            elif t.dtype == torch.bfloat16 or want_bf16:
                bits = t.to(torch.bfloat16).contiguous().cpu().view(torch.int16).numpy().view(np.uint16)
                return bits, nv.BF16, nv.bf16_bits_to_f32(bits)
            else:
                a = t.to(torch.float32).contiguous().cpu().numpy()
    except ImportError:  # pragma: no cover
        pass
    arr = np.asarray(a)
    if arr.dtype == np.int8 and pass_i8:
        if arr.ndim != 2:
            raise ValueError(f"embeddings must be 2-D, got shape {arr.shape}")
        x = np.ascontiguousarray(arr)
        return x, nv.I8, x.astype(np.float32)
    if arr.dtype == np.float16 and (want_f16 or pass_f16) and not want_bf16:
        if arr.ndim != 2:
            raise ValueError(f"embeddings must be 2-D, got shape {arr.shape}")
        h = np.ascontiguousarray(arr)
        return h, nv.F16, h.astype(np.float32)
    f = np.ascontiguousarray(arr, dtype=np.float32)  # faiss casts whatever it is given to float32
    if f.ndim != 2:
        raise ValueError(f"embeddings must be 2-D, got shape {f.shape}")
    if want_f16:
        h = f32_to_f16_checked(f)
        return h, nv.F16, h.astype(np.float32)
    if want_bf16:
        bits = nv.f32_to_bf16_bits(f)
        return bits, nv.BF16, nv.bf16_bits_to_f32(bits)
    if exact_bf16_ok and f.size:
        buf = None
        if scratch is not None:  # one reusable staging array per store (the C call copies it to the device before returning)
            buf = scratch.get("q16")
            if buf is None or buf.size < f.size:
                buf = scratch["q16"] = np.empty(f.size, dtype=np.uint16)
            buf = buf[:f.size].reshape(f.shape)
        bits, exact = nv.f32_to_bf16_checked(f, out=buf)
        if exact:
            return bits, nv.BF16, f
    return f, nv.F32, f


class MultiDeviceIndex:
    """Row-sharded flat index over several H100s driven from ONE process (for users who do not run under torchrun; under
    torchrun use lotus_b200.distributed.ShardedIndex, whose exchange runs over NCCL/NVLink). Shard g holds the contiguous rows
    `shard_bounds(n, G, g)` on devices[g]; a search runs the G per-device C-ABI calls concurrently (ctypes releases the GIL),
    then merges the G sorted lists on the host with the same (score, shard order) rule as the k-way merge kernel.
    Same surface as `_native.Index` as far as B200VS uses it."""

    def __init__(self, host_matrix: np.ndarray, code: int, metric: int, devices: list[int]):
        from concurrent.futures import ThreadPoolExecutor
        from .distributed import shard_bounds
        self.devices = list(devices)
        self.n, self.d = host_matrix.shape
        self.dtype, self.metric, self.device = code, metric, self.devices[0]
        self.bounds = [shard_bounds(self.n, len(self.devices), g) for g in range(len(self.devices))]
        self.pool = ThreadPoolExecutor(max_workers=len(self.devices))
        self.shards = list(self.pool.map(lambda gb: nv.Index(np.ascontiguousarray(host_matrix[gb[1][0]:gb[1][1]]), code, metric, gb[0]),
                                         zip(self.devices, self.bounds)))
        self._host = host_matrix  # kept for the operators that need the whole matrix on one device (dedup, k-means)
        self._replica: nv.Index | None = None

    def search(self, q: np.ndarray, k: int, q_dtype: int = nv.F32, ids: np.ndarray | None = None):
        def one(g):
            lo, hi = self.bounds[g]
            if ids is None:
                D, I = self.shards[g].search(q, k, q_dtype)
            else:
                mine = ids[(ids >= lo) & (ids < hi)] - lo
                if len(mine) == 0:
                    pad = np.finfo(np.float32).max if self.metric == nv.METRIC_L2 else -np.finfo(np.float32).max
                    return np.full((len(q), k), pad, np.float32), np.full((len(q), k), -1, np.int64)
                D, I = self.shards[g].search(q, k, q_dtype, ids=np.ascontiguousarray(mine))
            return D, np.where(I >= 0, I + lo, -1)
        if ids is not None and len(ids) and (ids.min() < 0 or ids.max() >= self.n):
            raise nv.NativeError(nv.ERANGE, f"ids contains a position outside [0, {self.n})")
        parts = list(self.pool.map(one, range(len(self.shards))))
        return merge_shard_lists([p[0] for p in parts], [p[1] for p in parts], self.metric)

    def search_masked(self, q: np.ndarray, k: int, q_dtype: int, mask):
        """As `_native.Index.search_masked`: every shard searches its rows under its slice of the bitmap (built on the host:
        shard bounds need not fall on word boundaries)."""
        words = nv.pack_mask(mask, self.n)

        def one(g):
            lo, hi = self.bounds[g]
            D, I = self.shards[g].search_masked(q, k, q_dtype, nv.slice_mask(words, self.n, lo, hi))
            return D, np.where(I >= 0, I + lo, -1)
        parts = list(self.pool.map(one, range(len(self.shards))))
        return merge_shard_lists([p[0] for p in parts], [p[1] for p in parts], self.metric)

    def range_search(self, q: np.ndarray, radius: float, q_dtype: int = nv.F32, ids: np.ndarray | None = None):
        """(lims, D, I) as `_native.Index.range_search`. Each shard answers for its rows (an ids subset: the distinct ids it
        holds); the hits are then ordered per query by row id, or with ids by position in `ids`, where a repeated id
        contributes one hit per occurrence."""
        nq = len(q)
        ids_a = None if ids is None else np.asarray(ids, dtype=np.int64)
        if ids_a is not None and len(ids_a) and (ids_a.min() < 0 or ids_a.max() >= self.n):
            raise nv.NativeError(nv.ERANGE, f"ids contains a position outside [0, {self.n})")
        uniq = None if ids_a is None else np.unique(ids_a)

        def one(g):
            lo, hi = self.bounds[g]
            if uniq is None:
                lims, D, I = self.shards[g].range_search(q, radius, q_dtype)
            else:
                mine = uniq[(uniq >= lo) & (uniq < hi)] - lo
                if len(mine) == 0:
                    return np.empty(0, np.int64), np.empty(0, np.float32), np.empty(0, np.int64)
                lims, D, I = self.shards[g].range_search(q, radius, q_dtype, ids=mine)
            return np.repeat(np.arange(nq, dtype=np.int64), np.diff(lims)), D, I + lo

        parts = list(self.pool.map(one, range(len(self.shards))))
        return combine_range_hits(nq, [p[0] for p in parts], [p[1] for p in parts], [p[2] for p in parts], ids_a)

    def range_search_masked(self, q: np.ndarray, radius: float, q_dtype: int, mask):
        """As `_native.Index.range_search_masked`: every shard searches its rows under its slice of the bitmap (built on the
        host: shard bounds need not fall on word boundaries); the hits are then ordered per query by row id."""
        words = nv.pack_mask(mask, self.n)
        nq = len(q)

        def one(g):
            lo, hi = self.bounds[g]
            lims, D, I = self.shards[g].range_search_masked(q, radius, q_dtype, nv.slice_mask(words, self.n, lo, hi))
            return np.repeat(np.arange(nq, dtype=np.int64), np.diff(lims)), D, I + lo

        parts = list(self.pool.map(one, range(len(self.shards))))
        return combine_range_hits(nq, [p[0] for p in parts], [p[1] for p in parts], [p[2] for p in parts])

    def gather(self, ids) -> np.ndarray:
        ids = np.asarray(ids, dtype=np.int64)
        if len(ids) and (ids.min() < 0 or ids.max() >= self.n):
            raise nv.NativeError(nv.ERANGE, f"ids contains a position outside [0, {self.n})")
        out = np.empty((len(ids), self.d), dtype=nv.storage_dtype(self.dtype))
        for g, (lo, hi) in enumerate(self.bounds):
            m = (ids >= lo) & (ids < hi)
            if m.any():
                out[m] = self.shards[g].gather(ids[m] - lo)
        return out

    def _whole(self) -> "nv.Index":
        if self._replica is None:  # all-pairs dedup and k-means want the whole matrix on one device
            self._replica = nv.Index(np.ascontiguousarray(self._host), self.dtype, self.metric, self.devices[0])
        return self._replica

    def threshold_pairs(self, thr: float, **kw):
        return self._whole().threshold_pairs(thr, **kw)

    def kmeans(self, k: int, **kw):
        return self._whole().kmeans(k, **kw)

    def close(self) -> None:
        for s in self.shards:
            s.close()
        if self._replica is not None:
            self._replica.close()
        self.pool.shutdown(wait=False)


def merge_shard_lists(D_parts: list, I_parts: list, metric: int):
    """Host k-way merge of per-shard (score, global id) lists [nq, k] -> [nq, k]: best first; equal scores keep each shard's
    (already faiss-ordered) list order, lower shards first for L2, higher shards first for IP — the rule of merge_topk_kernel."""
    g = len(D_parts)
    order = range(g) if metric == nv.METRIC_L2 else range(g - 1, -1, -1)
    D = np.concatenate([D_parts[i] for i in order], axis=1)
    I = np.concatenate([I_parts[i] for i in order], axis=1)
    k = D_parts[0].shape[1]
    key = np.where(I >= 0, D if metric == nv.METRIC_L2 else -D, np.inf)
    sel = np.argsort(key, axis=1, kind="stable")[:, :k]
    return np.take_along_axis(D, sel, axis=1), np.take_along_axis(I, sel, axis=1)


def combine_range_hits(nq: int, q_parts: list, d_parts: list, row_parts: list, ids: "np.ndarray | None" = None):
    """Per-shard range hits (query, score, global row) -> (lims[nq+1], D, I) ordered per query by row id; with `ids`, each
    hit row is expanded to every position of `ids` holding it, ordered per query by position and reported as ids[position]."""
    qs = np.concatenate(q_parts).astype(np.int64, copy=False) if q_parts else np.empty(0, np.int64)
    D = np.concatenate(d_parts).astype(np.float32, copy=False) if d_parts else np.empty(0, np.float32)
    rows = np.concatenate(row_parts).astype(np.int64, copy=False) if row_parts else np.empty(0, np.int64)
    if ids is None:
        key, I = rows, rows
    else:
        order = np.argsort(ids, kind="stable")
        sid = ids[order]
        left = np.searchsorted(sid, rows, "left")
        cnt = np.searchsorted(sid, rows, "right") - left
        rep = np.repeat(np.arange(len(rows)), cnt)
        within = np.arange(len(rep)) - np.repeat(np.cumsum(cnt) - cnt, cnt)
        key = order[left[rep] + within]  # positions in ids
        qs, D, I = qs[rep], D[rep], ids[key]
    o = np.lexsort((key, qs))
    lims = np.zeros(nq + 1, dtype=np.int64)
    np.cumsum(np.bincount(qs, minlength=nq), out=lims[1:])
    return lims, D[o], I[o]


def _free_device_bytes(device: int) -> int:
    """Free memory of a device in bytes (cudaMemGetInfo)."""
    import torch
    return int(torch.cuda.mem_get_info(device)[0])


def device_footprint(n: int, d: int, code: int) -> int:
    """Device bytes of a device-resident index of n x d rows of element type `code`: the rows, their padded copy when a row is
    not a multiple of 16 bytes, the bf16 copy of an fp32 store of at least 4096 rows, and the norms."""
    esz = {nv.F32: 4, nv.BF16: 2, nv.F16: 2, nv.I8: 1}[code]
    align = 16 // esz
    total = n * d * esz
    if d % align:
        total += n * (-(-d // align) * align) * esz
    if code == nv.F32 and n >= 4096:
        total += n * (-(-d // 8) * 8) * 2
    return total + n * (8 if code == nv.I8 else 4)


def ring_row_bytes(d: int, code: int) -> int:
    """Device bytes one streamed row of a host-resident index takes in its ring (the filter-ready row, plus its fp16 form for
    an int8 store): mirrors ring_row_bytes in api.cu."""
    esz = {nv.F32: 4, nv.BF16: 2, nv.F16: 2, nv.I8: 1}[code]
    align = 16 // esz
    b = -(-d // align) * align * esz
    return b + (-(-d // 8) * 8 * 2 if code == nv.I8 else 0)


AUTO_MARGIN = 1 << 30  # residency="auto": device memory left free beyond the footprint, for search workspaces


class B200VS(VS):
    """Flat (brute-force, exact) vector store on one H100 (or, with devices=[...], row-sharded over several from one process).

    Args mirror FaissVS(factory_string="Flat", metric=faiss.METRIC_INNER_PRODUCT) (faiss_vs.py:14).
    dtype: "f32" (store what faiss would: float32), "bf16" (round the corpus to bfloat16 once; exact search
    over those values), "f16" (store float16: float16 embeddings as they are, anything else rounded once, and a value
    outside float16's range raises ValueError; searched at the bf16 rate with results equal to faiss on the float32
    upcast of the stored values), "i8" (store int8: embeddings whose values are all integers in [-128, 127], such as
    quantized embeddings, of any numeric type; anything else raises ValueError, as the store never picks a scale. int8 queries
    are searched on the int8 tensor cores, floating-point queries against an fp16 copy of the rows made on their first
    search; results equal faiss on the float32 upcast; dedup runs the int8 pair filter, with its threshold in units of int8
    inner products, and k-means an fp16 copy of the rows), or "auto" (bf16 only when handed a bf16 tensor, float32 otherwise;
    int8 input still gives a float32 store).
    residency: "device" (default: the rows live in device memory), "host" (the rows stay in pinned host memory and every
    search streams them through a device ring of ring_bytes, None = the library default: corpora larger than free device
    memory, same results bit for bit; threshold_pairs / kmeans, hence sem_dedup / sem_cluster_by, raise ValueError) or
    "auto" (device when the store's device footprint plus a 1 GiB margin fits in free device memory, host otherwise;
    `resident(index_dir)` reports the choice). CUDA tensors given to a host-resident store are copied to the host.
    subset: how `__call__(..., ids=...)` and `range_search(..., ids=...)` search a subset of the rows. "gather" (default): a
    temporary index over a gathered copy of vecs[ids], as the reference does. "mask": when ids is strictly ascending (what a
    pandas filter leaves) the whole index is swept under a row bitmap instead, with the same result bit for bit, no copy of
    the subset in device memory and, on a host-resident index, no gather on the host; any other ids (permuted or repeating:
    different tie order) take the gathered path. "auto": the bitmap, for a strictly ascending ids, where the gathered copy is
    what hurts: on a host-resident index when the subset does not fit its ring (it would be gathered on the host), on a
    device-resident one when the copy's footprint plus a 1 GiB margin does not fit in free device memory (the gathered
    search would fail with an allocation error). Everywhere else the gathered search was the faster one in bench_masked.py (H100 80GB HBM3 at a
    700 W power limit, 1M x 768, subsets of 90 % down to 1 % of the rows: a masked search sweeps every row whatever the
    subset's size), so "auto" keeps it there; on the host-resident index the bitmap won for the subsets of 90 % and 50 %,
    the ones larger than its 384 MB ring. Range search follows the same rule: bench_range_masked.py on the same card and
    shapes found the same split (the bitmap slower at every share on the device-resident index, faster for the 90 % and
    50 % subsets on the host-resident one).
    """

    accepts_id_arrays = True  # `ids=` may be a numpy int64 array (the operators then skip building a Python list)

    def __init__(self, factory_string: str = "Flat", metric: int = METRIC_INNER_PRODUCT, dtype: str = "auto",
                 device: int = 0, cache_size: int = 4, devices: "list[int] | None" = None, residency: str = "device",
                 ring_bytes: "int | None" = None, subset: str = "gather"):
        super().__init__()
        if subset not in ("gather", "mask", "auto"):
            raise ValueError("subset must be 'gather', 'mask' or 'auto'")
        self.subset = subset
        if residency not in ("device", "host", "auto"):
            raise ValueError("residency must be 'device', 'host' or 'auto'")
        if ring_bytes is not None and (not isinstance(ring_bytes, int) or ring_bytes < 0):
            raise ValueError("ring_bytes must be a non-negative int or None")
        if devices and len(devices) > 1 and residency == "host":
            raise ValueError("residency='host' serves one device; it cannot be combined with devices=[...]")
        if factory_string != "Flat":
            raise ValueError(f"B200VS implements the flat (exact) index only; factory_string={factory_string!r}")
        if metric not in (METRIC_INNER_PRODUCT, METRIC_L2):
            raise ValueError("metric must be METRIC_INNER_PRODUCT (0) or METRIC_L2 (1)")
        if dtype not in ("auto", "f32", "bf16", "f16", "i8"):
            raise ValueError("dtype must be 'auto', 'f32', 'bf16', 'f16' or 'i8'")
        self.factory_string = factory_string
        self.metric = metric
        self.dtype = dtype
        self.devices = list(devices) if devices else None
        self.device = self.devices[0] if self.devices else device
        self.index_dir: str | None = None
        self.b2_index: nv.Index | None = None
        self.vecs: Any = None
        self._cache: "OrderedDict[str, tuple[float, nv.Index, Any]]" = OrderedDict()
        self._cache_size = max(2, cache_size)
        self._scratch: dict = {}
        self.residency = residency
        self.ring_bytes = ring_bytes

    def _choose_residency(self, n: int, d: int, code: int) -> str:
        if self.residency != "auto":
            return self.residency
        return "device" if device_footprint(n, d, code) + AUTO_MARGIN <= _free_device_bytes(self.device) else "host"

    def resident(self, index_dir: "str | None" = None) -> str:
        """Where the rows of the loaded index (or of the cached index of `index_dir`) live: "device" or "host"."""
        idx = self.b2_index if index_dir is None else self._cache[os.path.abspath(index_dir)][1]
        if idx is None:
            raise ValueError("Index not loaded")
        return getattr(idx, "resident", "device")

    # -- index lifetime ---------------------------------------------------------------------------------------------
    def _build(self, embeddings: Any) -> nv.Index:
        nv.require_device()
        t = _cuda_tensor(embeddings)
        if self.devices and len(self.devices) > 1:
            want16 = self.dtype == "bf16"
            if t is not None:
                import torch
                want16 = want16 or (self.dtype == "auto" and t.dtype == torch.bfloat16)
            host, code, _ = _to_host_matrix(embeddings, want16, want_f16=self.dtype == "f16", want_i8=self.dtype == "i8")
            return MultiDeviceIndex(host, code, self.metric, self.devices)  # type: ignore[return-value]
        if self.residency != "device":
            want16 = self.dtype == "bf16" or (self.dtype == "auto" and t is not None and str(t.dtype) == "torch.bfloat16")
            host, code, _ = _to_host_matrix(embeddings, want16, want_f16=self.dtype == "f16", want_i8=self.dtype == "i8")
            where = self._choose_residency(host.shape[0], host.shape[1], code)
            return nv.Index(host, code, self.metric, self.device, residency=where, ring_bytes=self.ring_bytes or 0)
        if t is not None and t.dim() == 2 and t.device.index == self.device:
            # device hand-off: the encoder's output never visits the host on its way into the index (a tensor that
            # already has the store's type is read in place)
            import torch
            if self.dtype == "i8":
                src = t.detach()
                if src.dtype != torch.int8:
                    fl = src.to(torch.float32)
                    if not bool(((fl == fl.round()) & (fl >= -128) & (fl <= 127)).all()):
                        raise ValueError("dtype='i8' needs integer values in [-128, 127] (quantize the embeddings first; the "
                                         "store never picks a scale)")
                t = src.to(torch.int8).contiguous()
                return nv.Index(None, nv.I8, self.metric, self.device, on_device_ptr=t.data_ptr(), n=t.shape[0], d=t.shape[1])
            if self.dtype == "f16":
                want = torch.float16
            else:
                want = torch.bfloat16 if (self.dtype == "bf16" or (self.dtype == "auto" and t.dtype == torch.bfloat16)) else torch.float32
            src = t.detach()
            t = src.to(want).contiguous()
            if want == torch.float16 and src.dtype != torch.float16 and bool((torch.isinf(t) & torch.isfinite(src)).any()):
                raise ValueError("embeddings hold values outside the float16 range (|v| < 65520); use dtype='f32' or 'bf16'")
            code = {torch.float32: nv.F32, torch.bfloat16: nv.BF16, torch.float16: nv.F16}[want]
            return nv.Index(None, code, self.metric, self.device, on_device_ptr=t.data_ptr(), n=t.shape[0], d=t.shape[1])
        host, code, _ = _to_host_matrix(embeddings, self.dtype == "bf16", want_f16=self.dtype == "f16",
                                        want_i8=self.dtype == "i8")
        return nv.Index(host, code, self.metric, self.device)

    def _remember(self, index_dir: str, idx: nv.Index, vecs: Any) -> None:
        key = os.path.abspath(index_dir)
        try:
            stamp = os.path.getmtime(f"{index_dir}/index")
        except OSError:
            stamp = 0.0
        old = self._cache.pop(key, None)
        if old is not None and old[1] is not idx:
            old[1].close()
        self._cache[key] = (stamp, idx, vecs)
        while len(self._cache) > self._cache_size:
            _, (_, victim, _) = self._cache.popitem(last=False)
            if victim is not self.b2_index:
                victim.close()

    def index(self, docs: Any, embeddings: Any, index_dir: str, **kwargs: Any) -> None:
        """faiss_vs.py:22-30: build the flat index, persist `vecs` (pickle) and `index` (faiss IndexFlat file)."""
        idx = self._build(embeddings)
        _, _, f32 = _to_host_matrix(embeddings, False)
        faiss_io.write_index_dir(index_dir, embeddings, f32, self.metric)
        self.b2_index = idx
        self.vecs = embeddings
        self.index_dir = index_dir
        self._remember(index_dir, idx, embeddings)

    def load_index(self, index_dir: str) -> None:
        """faiss_vs.py:32-36. Directories written by FaissVS load unchanged; a device-resident copy is cached per
        directory so operators that alternate between two indexes (sem_sim_join.py:111-127) do not rebuild."""
        key = os.path.abspath(index_dir)
        hit = self._cache.get(key)
        if hit is not None:
            try:
                fresh = os.path.getmtime(f"{index_dir}/index") == hit[0]
            except OSError:
                fresh = False
            if fresh:
                self._cache.move_to_end(key)
                self.index_dir, self.b2_index, self.vecs = index_dir, hit[1], hit[2]
                return
        vecs, x, metric = faiss_io.read_index_dir(index_dir)
        if metric != self.metric:
            raise ValueError(f"index at {index_dir} was built with metric {metric}, this store uses {self.metric}")
        idx = self._build(vecs if self.dtype != "f32" else x)
        self.index_dir, self.b2_index, self.vecs = index_dir, idx, vecs
        self._remember(index_dir, idx, vecs)

    # -- queries ----------------------------------------------------------------------------------------------------
    def _entry_for(self, index_dir: str) -> nv.Index:
        """Device index of `index_dir` WITHOUT making it the loaded one (faiss_vs.py:38-41 only reads the `vecs` pickle and
        leaves `self.faiss_index` / `self.index_dir` alone)."""
        key = os.path.abspath(index_dir)
        if self.index_dir is not None and self.b2_index is not None and os.path.abspath(self.index_dir) == key:
            return self.b2_index
        keep = (self.index_dir, self.b2_index, self.vecs)
        if self.index_dir is not None and os.path.abspath(self.index_dir) in self._cache:
            self._cache.move_to_end(os.path.abspath(self.index_dir))  # the loaded index must not be the eviction victim
        try:
            self.load_index(index_dir)  # per-directory cache hit, or build + cache the device copy ...
            return self.b2_index  # type: ignore[return-value]
        finally:
            self.index_dir, self.b2_index, self.vecs = keep  # ... but the loaded index stays what it was

    def get_vectors_from_index(self, index_dir: str, ids: Any) -> np.ndarray:
        """faiss_vs.py:38-41 (`pickle.load(vecs)[ids]`), served by the device row-gather kernel. Like the reference it does
        not change which index is loaded."""
        idx = self._entry_for(index_dir)
        ids_a = np.asarray(list(ids) if not isinstance(ids, np.ndarray) else ids, dtype=np.int64)
        out = idx.gather(ids_a)
        if idx.dtype == nv.BF16:
            return BF16Backed.wrap(nv.bf16_bits_to_f32(out))
        return out  # float32, or the float16 / int8 values of an fp16 / int8 index (like pickle.load(vecs)[ids])

    def __call__(self, query_vectors: Any, K: int, ids: list[int] | None = None, **kwargs: Any) -> RMOutput:
        """faiss_vs.py:43-77. Returns float32 distances [Q,K] and int64 indices [Q,K] (global ids; -1 = no result).
        The reference's wrap-around of -1 to the last id when K > len(ids) (faiss_vs.py:71-72) is NOT reproduced."""
        if self.b2_index is None or self.index_dir is None:
            raise ValueError("Index not loaded")
        ids_a = None if ids is None else np.asarray(list(ids) if not isinstance(ids, np.ndarray) else ids, dtype=np.int64)
        t = _cuda_tensor(query_vectors)
        if t is not None and ids_a is None and t.dim() == 2 and t.device.index == self.device and not isinstance(self.b2_index, MultiDeviceIndex):
            return self._call_device(t, int(K))
        q, code, _ = _to_host_matrix(query_vectors, False, exact_bf16_ok=self.b2_index.dtype == nv.BF16, scratch=self._scratch,
                                     pass_f16=True, pass_i8=True)
        if q.shape[1] != self.b2_index.d:
            raise ValueError(f"query dimension {q.shape[1]} does not match the index dimension {self.b2_index.d}")
        try:
            if ids_a is not None and self._subset_by_mask(ids_a):
                distances, indices = self.b2_index.search_masked(q, int(K), code, nv.ids_to_mask(ids_a, self.b2_index.n))
            else:
                distances, indices = self.b2_index.search(q, int(K), code, ids=ids_a)
        except nv.NativeError as e:
            if e.code in (nv.EINVAL, nv.ERANGE):
                raise ValueError(e.msg) from e
            raise
        return RMOutput(distances=distances, indices=indices)

    def _subset_by_mask(self, ids: np.ndarray) -> bool:
        """Whether `subset` sends this ids subset through the masked search (see the class docstring)."""
        idx = self.b2_index
        if self.subset == "gather" or len(ids) == 0 or not nv.strictly_ascending(ids):
            return False
        if self.subset == "mask":
            return True
        if getattr(idx, "resident", "device") == "host":
            return len(ids) * ring_row_bytes(idx.d, idx.dtype) > idx.ring_bytes
        return device_footprint(len(ids), idx.d, idx.dtype) + AUTO_MARGIN > _free_device_bytes(idx.device)

    def search_masked(self, query_vectors: Any, K: int, mask: Any) -> RMOutput:
        """__call__(query_vectors, K, ids=np.flatnonzero(mask)) for callers that hold a boolean column rather than ids: the
        rows whose entry of `mask` (bool, one per row of the index) is set, always searched under the bitmap."""
        if self.b2_index is None or self.index_dir is None:
            raise ValueError("Index not loaded")
        q, code, _ = _to_host_matrix(query_vectors, False, exact_bf16_ok=self.b2_index.dtype == nv.BF16, scratch=self._scratch,
                                     pass_f16=True, pass_i8=True)
        if q.shape[1] != self.b2_index.d:
            raise ValueError(f"query dimension {q.shape[1]} does not match the index dimension {self.b2_index.d}")
        try:
            distances, indices = self.b2_index.search_masked(q, int(K), code, np.asarray(mask, dtype=np.bool_))
        except nv.NativeError as e:
            if e.code in (nv.EINVAL, nv.ERANGE):
                raise ValueError(e.msg) from e
            raise
        return RMOutput(distances=distances, indices=indices)

    def _call_device(self, t: Any, K: int) -> RMOutput:
        """Queries already on the GPU (e.g. straight out of the encoder): search in place, only the [Q,K] result travels."""
        import torch
        assert self.b2_index is not None
        if t.shape[1] != self.b2_index.d:
            raise ValueError(f"query dimension {t.shape[1]} does not match the index dimension {self.b2_index.d}")
        q = t.detach()
        q = q.contiguous() if q.dtype in (torch.float32, torch.bfloat16, torch.float16, torch.int8) else q.to(torch.float32).contiguous()
        code = {torch.float32: nv.F32, torch.bfloat16: nv.BF16, torch.float16: nv.F16, torch.int8: nv.I8}[q.dtype]
        out_s = torch.empty((q.shape[0], K), dtype=torch.float32, device=q.device)
        out_i = torch.empty((q.shape[0], K), dtype=torch.int64, device=q.device)
        try:
            self.b2_index.search_dev(q.data_ptr(), q.shape[0], K, code, out_s.data_ptr(), out_i.data_ptr(),
                                     stream=torch.cuda.current_stream().cuda_stream)
        except nv.NativeError as e:
            if e.code in (nv.EINVAL, nv.ERANGE):
                raise ValueError(e.msg) from e
            raise
        return RMOutput(distances=out_s.cpu().numpy(), indices=out_i.cpu().numpy())

    def range_search(self, query_vectors: Any, radius: float, ids: Any = None):
        """faiss IndexFlat.range_search(x, radius) over the loaded index: (lims[Q+1] int64, D float32, I int64), query i's
        hits at [lims[i], lims[i+1]) in ascending id. IP keeps rows whose score is strictly greater than `radius`; L2 those
        whose squared distance is strictly less. D holds the values __call__ reports. ids: only those rows, as a temporary
        index over vecs[ids] (faiss_vs.py:57-72): hits follow the order of `ids`, a repeated id once per occurrence; `subset`
        decides, as for __call__, whether a strictly ascending ids is searched under a row bitmap instead (same result).
        Queries as __call__ accepts them."""
        ids_a = None if ids is None else np.asarray(list(ids) if not isinstance(ids, np.ndarray) else ids, dtype=np.int64)
        return self._range(query_vectors, radius, ids=ids_a)

    def range_search_masked(self, query_vectors: Any, radius: float, mask: Any):
        """range_search(query_vectors, radius, ids=np.flatnonzero(mask)) for callers that hold a boolean column rather than
        ids: the rows whose entry of `mask` (bool, one per row of the index) is set, always searched under the bitmap."""
        return self._range(query_vectors, radius, mask=np.asarray(mask, dtype=np.bool_))

    def _range(self, query_vectors: Any, radius: float, ids: "np.ndarray | None" = None, mask: Any = None):
        if self.b2_index is None or self.index_dir is None:
            raise ValueError("Index not loaded")
        q, code, _ = _to_host_matrix(query_vectors, False, exact_bf16_ok=self.b2_index.dtype == nv.BF16, scratch=self._scratch,
                                     pass_f16=True, pass_i8=True)
        if q.shape[1] != self.b2_index.d:
            raise ValueError(f"query dimension {q.shape[1]} does not match the index dimension {self.b2_index.d}")
        try:
            if ids is not None and self._subset_by_mask(ids):
                mask = nv.ids_to_mask(ids, self.b2_index.n)
            if mask is None:
                return self.b2_index.range_search(q, float(radius), code, ids=ids)
            return self.b2_index.range_search_masked(q, float(radius), code, mask)
        except nv.NativeError as e:
            if e.code in (nv.EINVAL, nv.ERANGE):
                raise ValueError(e.msg) from e
            raise

    # -- extensions used by the re-registered operators --------------------------------------------------------------
    def _refuse_host(self, what: str) -> None:
        if getattr(self.b2_index, "resident", "device") == "host":
            raise ValueError(f"{what} is not available on a host-resident index (B200VS(residency='host')): build the store "
                             "with residency='device'")

    def threshold_pairs(self, threshold: float):
        if self.b2_index is None:
            raise ValueError("Index not loaded")
        self._refuse_host("threshold_pairs (sem_dedup)")
        return self.b2_index.threshold_pairs(threshold)

    def kmeans(self, ids: Any, ncentroids: int, niter: int = 20, seed: int = 1234, full_lloyd: bool = False):
        if self.b2_index is None:
            raise ValueError("Index not loaded")
        self._refuse_host("kmeans (sem_cluster_by)")
        return self.b2_index.kmeans(ncentroids, niter=niter, seed=seed, ids=np.asarray(ids, dtype=np.int64), full_lloyd=full_lloyd)

    def close(self) -> None:
        for _, idx, _ in self._cache.values():
            idx.close()
        self._cache.clear()
        self.b2_index = None
