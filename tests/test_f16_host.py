"""fp16 indexes (B2_F16) on CPU: the C-ABI's validation and error model, the float16 paths of B200VS and the index directory,
and the operators over float16 embeddings with the native index replaced by an oracle-backed fake (GPU runs of the same
surface are in tests/test_gpu_f16.py)."""
import ctypes
import os
import pickle
import re

import numpy as np
import pandas as pd
import pytest

import lotus_b200 as lotus
import oracle
from filter_lists import rel_eps_formula
from helpers import NumpyVS, gauss
from lotus_b200 import _native as nv
from lotus_b200 import faiss_io
from lotus_b200.vs import B200VS

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


# ---- C-ABI ------------------------------------------------------------------------------------------------------------------
def test_header_and_binding_agree_on_the_element_types(nv):
    hdr = open(os.path.join(ROOT, "include", "lotus_b200.h")).read()
    enum = re.search(r"enum\s*\{\s*(B2_F32[^}]*)\}", hdr).group(1)
    codes = {name: int(v) for name, v in re.findall(r"(B2_\w+)\s*=\s*(\d+)", enum)}
    assert codes == {"B2_F32": nv.F32, "B2_BF16": nv.BF16, "B2_F16": nv.F16} == {"B2_F32": 0, "B2_BF16": 1, "B2_F16": 2}
    assert nv.DTYPES == (0, 1, 2)
    assert nv.lib().b2_abi_version() == 1


def _create(nv, dtype):
    x = np.zeros((4, 8), np.float32)
    h = ctypes.c_void_p()
    rc = nv.lib().b2_index_create(ctypes.c_void_p(x.ctypes.data), 4, 8, dtype, 0, 0, 0, ctypes.byref(h))
    if rc == 0:
        nv.lib().b2_index_free(h)
    return rc


def test_index_create_validates_the_element_type(nv):
    assert _create(nv, 3) == nv.EINVAL and "B2_F16" in nv.lib().b2_last_error().decode()
    assert _create(nv, -1) == nv.EINVAL
    if nv.device_count() == 0:  # B2_F16 passes validation and only then meets the missing device
        assert _create(nv, nv.F16) == nv.ENODEV
    else:
        assert _create(nv, nv.F16) == nv.OK


def _ulp_eq(a, b):
    # the library writes 2^-23 as the decimal 1.1920929e-7: the two can round to float32 values one ulp apart
    return abs(a - float(b)) <= 2.0 ** -23 * abs(float(b))


def test_filter_error_model(nv):
    """rel_eps and abs_eps of every operand combination (DESIGN.md §2). The bf16 / tf32 combinations are unchanged."""
    F32, BF16, F16 = nv.F32, nv.BF16, nv.F16
    for d in (8, 30, 768, 1000):
        for store, filt, q in [(BF16, BF16, BF16), (BF16, BF16, F32), (F32, F32, F32), (F32, BF16, F32), (F32, F32, BF16)]:
            rel, ab = nv.filter_eps(store, filt, q, d)
            assert _ulp_eq(rel, rel_eps_formula(d, store, filt, q)) and ab == 0.0
        acc = (d + 64) * 2.0 ** -23 + 1e-6
        u = 2.0 ** -11
        for store, q, ex, eq, rounded in [(F16, F16, 0, 0, 0), (F16, F32, 0, u, 1), (F16, BF16, 0, u, 1), (F32, F16, u, 0, 1)]:
            rel, ab = nv.filter_eps(store, F16, q, d)
            assert _ulp_eq(rel, np.float32(acc + ex + eq + ex * eq)), (store, q, d)
            assert _ulp_eq(ab, np.float32(rounded * 2.0 ** -25 * np.sqrt(d) * (1 + 1e-6))), (store, q, d)
        # fp16 queries: exact in tf32, rounded (2^-8) on a bf16 filter, no absolute term either way
        for store, filt, want in [(F32, F32, acc + 2.0 ** -10), (BF16, BF16, acc + 2.0 ** -8), (F32, BF16, acc + 2 * 2.0 ** -8 + 2.0 ** -16)]:
            rel, ab = nv.filter_eps(store, filt, F16, d)
            assert _ulp_eq(rel, np.float32(want)) and ab == 0.0, (store, filt, d)
    with pytest.raises(nv.NativeError):
        nv.filter_eps(3, F16, F16, 8)


def test_stored_to_f32_on_every_dtype_code(nv):
    x = (gauss(5, 6, 1) * 3).astype(np.float32)
    assert np.array_equal(nv.stored_to_f32(x, nv.F32), x)
    b = nv.f32_to_bf16_bits(x)
    assert np.array_equal(nv.stored_to_f32(b, nv.BF16), nv.bf16_bits_to_f32(b))
    h = x.astype(np.float16)
    up = nv.stored_to_f32(h, nv.F16)
    assert up.dtype == np.float32 and np.array_equal(up, h.astype(np.float32))
    assert np.array_equal(nv.stored_to_f32(h.view(np.uint16), nv.F16), up)  # bit patterns as well
    assert nv.storage_dtype(nv.F16) == np.float16 and nv.storage_dtype(nv.BF16) == np.uint16
    with pytest.raises(ValueError):
        nv.stored_to_f32(x, 3)


# ---- B200VS over a fake fp16-aware native index ----------------------------------------------------------------------------
class FakeF16Index:
    """Stands in for _native.Index for every element type, computed by the oracle on the stored values' fp32 upcast."""
    live = 0

    def __init__(self, x, dtype, metric=0, device=0, on_device_ptr=None, n=None, d=None):
        assert on_device_ptr is None
        x = np.ascontiguousarray(x)
        assert x.dtype == nv.storage_dtype(dtype) and x.ndim == 2, (x.dtype, dtype)
        self.raw, self.dtype, self.metric, self.device = x, dtype, metric, device
        self.vals = nv.stored_to_f32(x, dtype)
        self.n, self.d = x.shape
        self.calls = []
        FakeF16Index.live += 1

    def close(self):
        FakeF16Index.live -= 1

    def search(self, q, k, q_dtype=0, ids=None):
        assert q.dtype == nv.storage_dtype(q_dtype)
        self.calls.append((q.dtype, q_dtype))
        qv = nv.stored_to_f32(q, q_dtype)
        if ids is None:
            return oracle.knn(self.vals, qv, k, self.metric)
        return oracle.knn_subset(self.vals, qv, k, ids, self.metric)

    def gather(self, ids):
        return self.raw[np.asarray(ids, dtype=np.int64)]

    def threshold_pairs(self, thr, cap=1 << 24, part=0, nparts=1):
        pi, pj, _ = oracle.threshold_pairs(self.vals, float(thr))
        return pi, pj

    def kmeans(self, k, niter=20, seed=1234, ids=None, full_lloyd=False):
        x = self.vals if ids is None else self.vals[np.asarray(ids, dtype=np.int64)]
        return oracle.kmeans(np.ascontiguousarray(x), k, niter=niter, full_lloyd=full_lloyd)


@pytest.fixture
def fake_native(monkeypatch):
    FakeF16Index.live = 0
    monkeypatch.setattr(nv, "Index", FakeF16Index)
    monkeypatch.setattr(nv, "require_device", lambda: None)
    yield


def test_f16_store_validation_and_rounding(fake_native, tmp_path):
    assert B200VS(dtype="f16").dtype == "f16"
    with pytest.raises(ValueError, match="dtype"):
        B200VS(dtype="fp16")
    x = gauss(40, 16, 2)
    vs = B200VS(dtype="f16")
    vs.index(None, x, str(tmp_path / "r"))                       # float32 input: rounded once, to nearest even
    assert vs.b2_index.dtype == nv.F16 and np.array_equal(vs.b2_index.raw.view(np.uint16), x.astype(np.float16).view(np.uint16))
    big = x.copy()
    big[3, 5] = 70000.0                                          # would round to inf
    with pytest.raises(ValueError, match="float16 range"):
        B200VS(dtype="f16").index(None, big, str(tmp_path / "o"))
    ok = x.copy()
    ok[3, 5] = 65519.0                                           # still rounds to 65504
    B200VS(dtype="f16").index(None, ok, str(tmp_path / "ok"))
    # dtype="auto" keeps its meaning: float16 input becomes an fp32 store
    vs = B200VS()
    vs.index(None, x.astype(np.float16), str(tmp_path / "a"))
    assert vs.b2_index.dtype == nv.F32


def test_index_directory_from_float16_embeddings(fake_native, tmp_path):
    xh = gauss(30, 8, 3).astype(np.float16)
    d = str(tmp_path / "h")
    vs = B200VS(dtype="f16")
    vs.index(None, xh, d)
    with open(f"{d}/vecs", "rb") as fp:
        vecs = pickle.load(fp)
    assert vecs.dtype == np.float16 and np.array_equal(vecs.view(np.uint16), xh.view(np.uint16))     # kept as given
    xr, metric = faiss_io.read_flat_index(f"{d}/index")
    assert xr.dtype == np.float32 and np.array_equal(xr, xh.astype(np.float32))                      # the exact upcast
    fresh = B200VS(dtype="f16")
    fresh.load_index(d)
    assert fresh.b2_index.dtype == nv.F16 and np.array_equal(fresh.b2_index.raw.view(np.uint16), xh.view(np.uint16))
    # a directory written the way FaissVS writes it (float16 vecs pickle, faiss's float32 cast in the index) loads unrounded
    d2 = str(tmp_path / "faiss_made")
    faiss_io.write_index_dir(d2, xh, xh.astype(np.float32), faiss_io.METRIC_INNER_PRODUCT)
    vs2 = B200VS(dtype="f16")
    vs2.load_index(d2)
    assert np.array_equal(vs2.b2_index.raw.view(np.uint16), xh.view(np.uint16))
    got = vs2.get_vectors_from_index(d2, [4, 0])
    assert got.dtype == np.float16 and np.array_equal(got, xh[[4, 0]])                               # pickle.load(vecs)[ids]
    out = vs2(got, 3)                                                                                # float16 queries: F16 operands
    assert vs2.b2_index.calls[-1] == (np.dtype(np.float16), nv.F16)
    D, I = oracle.knn(xh.astype(np.float32), xh[[4, 0]].astype(np.float32), 3, oracle.IP)
    assert np.array_equal(out.indices, I) and np.array_equal(out.distances, D)


def test_float16_queries_ship_as_f16_on_every_store(fake_native, tmp_path):
    x, q = gauss(25, 8, 4), gauss(3, 8, 5).astype(np.float16)
    for dt, code in (("f32", nv.F32), ("bf16", nv.BF16), ("f16", nv.F16)):
        vs = B200VS(dtype=dt)
        vs.index(None, x, str(tmp_path / dt))
        out = vs(q, 4)
        assert vs.b2_index.dtype == code and vs.b2_index.calls[-1] == (np.dtype(np.float16), nv.F16)
        D, I = oracle.knn(vs.b2_index.vals, q.astype(np.float32), 4, oracle.IP)
        assert np.array_equal(out.indices, I) and np.array_equal(out.distances, D)


# ---- the operators over float16 embeddings -----------------------------------------------------------------------------------
class HalfRM(lotus.HashRM):
    """HashRM in half precision, as a sentence-transformers model loaded in fp16 produces it."""

    def _embed(self, docs):
        return super()._embed(docs).astype(np.float16)


def _frames(tmp, monkeypatch):
    import lotus_b200.sem_ops.sem_dedup as sd
    monkeypatch.setattr(sd.nv, "connected_components", lambda n, pi, pj, device=0: oracle.connected_components(n, pi, pj))
    left = pd.DataFrame({"a": [f"doc {i % 23}" for i in range(60)]})
    right = pd.DataFrame({"b": [f"skill {i}" for i in range(40)]})
    out = {}
    out["index"] = left.sem_index("a", str(tmp / "l"))
    right = right.sem_index("b", str(tmp / "r"))
    out["search"] = out["index"].sem_search("a", "doc 7", K=5, return_scores=True)
    out["join"] = out["index"].sem_sim_join(right, "a", "b", K=3, lsuffix="_l", rsuffix="_r")
    out["join_sub"] = out["index"].sem_sim_join(right[right.index % 3 == 0], "a", "b", K=2)
    out["dedup"] = out["index"].sem_dedup("a", threshold=0.9)
    out["cluster"] = out["index"].sem_cluster_by("a", 4, niter=3)
    return out


def test_operators_over_float16_embeddings_equal_the_oracle_frames(fake_native, monkeypatch, tmp_path):
    rm = HalfRM(dim=32)
    try:
        lotus.settings.configure(rm=rm, vs=NumpyVS(), enable_cache=False)   # the oracle on the float32 upcast
        want = _frames(tmp_path / "w", monkeypatch)
        vs = B200VS(dtype="f16")
        lotus.settings.configure(rm=rm, vs=vs, enable_cache=False)
        got = _frames(tmp_path / "g", monkeypatch)
        assert vs.b2_index.dtype == nv.F16
        # sem_sim_join fetched the right frame's vectors (float16, get_vectors_from_index) and searched with them as F16
        assert any(c == (np.dtype(np.float16), nv.F16) for c in vs.b2_index.calls)
    finally:
        lotus.settings.configure(rm=None, vs=None)
    for key in want:
        pd.testing.assert_frame_equal(got[key], want[key], check_exact=True, obj=key)
