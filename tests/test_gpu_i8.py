"""int8 indexes (B2_I8) on the GPU: every search entry point against the oracle on the float32 upcast of the stored int8 values.

int8 x int8 is filtered on the int8 tensor cores with exact s32 accumulation; the only filter error is the rounding of the sum
to fp32, and none while |s| < 2^24. Floating-point queries on an int8 store are filtered against its fp16 copy (exact), and
int8 queries on the other stores are widened exactly. Answers must be bit-identical to the oracle in every case."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest

import oracle
from filter_lists import check_lists
from helpers import bits, gauss

pytestmark = pytest.mark.gpu


def quant(a):
    """int8 with one scale per matrix: 127 / max|a|, rounded, clamped (how quantized embeddings are usually made)."""
    a = np.asarray(a, dtype=np.float64)
    return np.clip(np.rint(a * (127.0 / np.abs(a).max())), -128, 127).astype(np.int8)


def data(kind, n, d, seed):
    rng = np.random.default_rng(seed)
    if kind == "gauss":
        return quant(gauss(n, d, seed))
    if kind == "ties":  # tie-heavy: values in {-2..2}
        return rng.integers(-2, 3, size=(n, d)).astype(np.int8)
    if kind == "extreme":  # +-127 and -128 only: at d = 2048 the scores pass 2^24, so the fp32 conversion rounds
        return rng.choice(np.array([-128, -127, 127], np.int8), size=(n, d))
    raise ValueError(kind)


def assert_same(D, I, Do, Io, tag=""):
    assert np.array_equal(I, Io), f"{tag}: {(I != Io).any(axis=1).sum()} rows differ"
    assert np.array_equal(bits(D), bits(Do)), f"{tag}: score bits differ"


# d = 8, 30, 100, 1000 are not multiples of 16 bytes (padded filter copy); 2048 with extreme rows passes 2^24
@pytest.mark.parametrize("metric", [oracle.IP, oracle.L2])
@pytest.mark.parametrize("d", [8, 16, 30, 100, 768, 1000, 2048])
def test_i8_store_search_parity(gpu, metric, d):
    n = 6000
    for kind in ("gauss", "ties", "extreme"):
        if kind == "extreme" and d not in (30, 2048):
            continue
        x, q = data(kind, n, d, d), data(kind, 300, d, d + 1)
        x[n // 2: n // 2 + 20] = x[:20]  # duplicate rows
        xf, qf = x.astype(np.float32), q.astype(np.float32)
        idx = gpu.Index(x, gpu.I8, metric)
        assert idx.dtype == gpu.I8
        for k in (1, 5, 32, 64, 100, 1000):
            gpu.stats_reset()
            D, I = idx.search(q, k, gpu.I8)
            st = gpu.stats()
            Do, Io = oracle.knn(xf, qf, k, metric)
            assert_same(D, I, Do, Io, f"{kind} d={d} k={k}")
            if kind == "gauss" and d >= 16 and k <= 100:
                assert st["filter_launches"] >= 1, st
        ids = np.arange(7, n, 3)
        D, I = idx.search(q, 10, gpu.I8, ids=ids)
        Do, Io = oracle.knn_subset(xf, qf, 10, ids, metric)
        assert_same(D, I, Do, Io, f"{kind} d={d} ids=")
        assert np.array_equal(idx.gather(np.array([0, n - 1, 5])), x[[0, n - 1, 5]])
        idx.close()


def test_i8_fallback_bound(gpu):
    """duplicate-free quantized Gaussian data: the int8 filter certifies (nearly) every query"""
    x, q = data("gauss", 50_000, 768, 11), data("gauss", 2000, 768, 12)
    for metric in (oracle.IP, oracle.L2):
        idx = gpu.Index(x, gpu.I8, metric)
        for k in (10, 32, 100):
            gpu.stats_reset()
            D, I = idx.search(q, k, gpu.I8)
            st = gpu.stats()
            assert st["filter_launches"] >= 1 and st["fallback_queries"] <= 4, (metric, k, st)
            Do, Io = oracle.knn(x.astype(np.float32), q.astype(np.float32), k, metric)
            assert_same(D, I, Do, Io, f"metric={metric} k={k}")
        idx.close()


@pytest.mark.parametrize("metric", [oracle.IP, oracle.L2])
def test_query_types_and_cross_store_identity(gpu, metric):
    """The same integers in i8 / bf16 / f16 / f32 stores give identical results, for i8 / f32 / bf16 / f16 queries holding the
    same integers; float queries that are not integers on an i8 store go through its fp16 copy and still match the oracle."""
    n, d = 20_000, 100
    x, q = data("gauss", n, d, 5), data("gauss", 400, d, 6)
    xf, qf = x.astype(np.float32), q.astype(np.float32)
    stores = {
        "i8": gpu.Index(x, gpu.I8, metric),
        "bf16": gpu.Index(gpu.f32_to_bf16_bits(xf), gpu.BF16, metric),
        "f16": gpu.Index(xf.astype(np.float16), gpu.F16, metric),
        "f32": gpu.Index(xf, gpu.F32, metric),
    }
    qs = {"i8": (q, gpu.I8), "f32": (qf, gpu.F32), "bf16": (gpu.f32_to_bf16_bits(qf), gpu.BF16), "f16": (qf.astype(np.float16), gpu.F16)}
    for k in (1, 10, 64):
        Do, Io = oracle.knn(xf, qf, k, metric)
        for sname, idx in stores.items():
            for qname, (qa, code) in qs.items():
                D, I = idx.search(qa, k, code)
                assert_same(D, I, Do, Io, f"store={sname} q={qname} k={k}")
    qr = gauss(300, d, 7)  # non-integral queries on the int8 store
    for k in (1, 10, 100):
        gpu.stats_reset()
        D, I = stores["i8"].search(qr, k, gpu.F32)
        assert gpu.stats()["fallback_queries"] <= 3
        Do, Io = oracle.knn(xf, qr, k, metric)
        assert_same(D, I, Do, Io, f"f32 queries k={k}")
    for idx in stores.values():
        idx.close()


def test_search_dev_sharded_paths_and_gather(gpu):
    torch = pytest.importorskip("torch")
    n, d, k = 30_000, 256, 10
    x, q = data("gauss", n, d, 21), data("gauss", 500, d, 22)
    xf, qf = x.astype(np.float32), q.astype(np.float32)
    Do, Io = oracle.knn(xf, qf, k, oracle.IP)
    idx = gpu.Index(x, gpu.I8, oracle.IP)
    qt = torch.from_numpy(q).cuda()
    out_s = torch.empty((len(q), k), dtype=torch.float32, device="cuda")
    out_i = torch.empty((len(q), k), dtype=torch.int64, device="cuda")
    idx.search_dev(qt.data_ptr(), len(q), k, gpu.I8, out_s.data_ptr(), out_i.data_ptr())
    assert_same(out_s.cpu().numpy(), out_i.cpu().numpy(), Do, Io, "search_dev")
    # packed path and the two-stage sharded path, emulated with two shards in one process
    half = n // 2
    shards = [gpu.Index(x[:half], gpu.I8, oracle.IP), gpu.Index(x[half:], gpu.I8, oracle.IP)]
    lowers, packed = [], []
    for s in shards:
        lo = torch.empty(len(q), dtype=torch.float32, device="cuda")
        s.search_stage1_dev(qt.data_ptr(), len(q), k, gpu.I8, (k + 1) // 2, lo.data_ptr())
        lowers.append(lo)
    hint = torch.minimum(lowers[0], lowers[1])
    for s in shards:
        pk = torch.empty((len(q), k), dtype=torch.int64, device="cuda")
        s.search_stage2_packed_dev(hint.data_ptr(), pk.data_ptr())
        torch.cuda.synchronize()
        packed.append(pk.cpu().numpy().view(np.uint64))
    D_parts, I_parts = [], []
    for g, pk in enumerate(packed):
        sc = (pk >> np.uint64(32)).astype(np.uint32).view(np.float32)
        loc = (pk & np.uint64(0xffffffff)).astype(np.int64)
        I_parts.append(np.where(loc == 0xffffffff, -1, loc + g * half))
        D_parts.append(sc)
    from lotus_b200.vs import merge_shard_lists
    D, I = merge_shard_lists(D_parts, I_parts, oracle.IP)
    assert_same(D, I, Do, Io, "staged sharded")
    D_parts, I_parts = [], []
    for g, s in enumerate(shards):
        pk = torch.empty((len(q), k), dtype=torch.int64, device="cuda")
        s.search_packed_dev(qt.data_ptr(), len(q), k, gpu.I8, pk.data_ptr())
        torch.cuda.synchronize()
        w = pk.cpu().numpy().view(np.uint64)
        loc = (w & np.uint64(0xffffffff)).astype(np.int64)
        D_parts.append((w >> np.uint64(32)).astype(np.uint32).view(np.float32))
        I_parts.append(np.where(loc == 0xffffffff, -1, loc + g * half))
    D, I = merge_shard_lists(D_parts, I_parts, oracle.IP)
    assert_same(D, I, Do, Io, "packed sharded")
    g = idx.gather(np.array([3, 0, n - 1]))
    assert g.dtype == np.int8 and np.array_equal(g, x[[3, 0, n - 1]])
    idx.close()
    for s in shards:
        s.close()


LISTS_SCRIPT = r"""
import json, sys
import numpy as np
sys.path[:0] = [sys.argv[1], sys.argv[2]]
from lotus_b200 import _native as nv
from filter_lists import check_lists
from test_gpu_i8 import data
clusters = []
for n in (40_000, 6_000):  # a long corpus runs clusters of four, a short one CTA pairs (single CTAs with B2_FILTER_2CTA=0)
    x, q = data("gauss", n, 192, 31), data("gauss", 600, 192, 32)
    for metric in (0, 1):
        for k in (5, 32, 100):
            idx = nv.Index(x, nv.I8, metric)
            res = idx.filter_lists(q, k, nv.I8)
            assert res["use_filter"] and res["filt_dtype"] == nv.I8, res
            # |2 <q, x> - |x|^2| < 2^24 here: every list score is the exact integer, the discard bound exact
            check_lists(res, q.astype(np.float64), x.astype(np.float64), metric, exact=True, tag=f"n={n} metric={metric} k={k}")
            clusters.append(res["cluster"])
            idx.close()
print(json.dumps({"clusters": sorted(set(clusters))}))
"""


@pytest.mark.parametrize("two_cta", ["1", "0"])
def test_raw_filter_lists_against_fp64(gpu, two_cta):
    """Raw int8 x int8 lists against fp64 in both CTA modes and in clusters of four: scores bit-equal to the exact values."""
    here = os.path.dirname(os.path.abspath(__file__))
    r = subprocess.run([sys.executable, "-c", LISTS_SCRIPT, os.path.dirname(here), here], capture_output=True, text=True,
                       timeout=900, env=dict(os.environ, B2_FILTER_2CTA=two_cta))
    assert r.returncode == 0, r.stderr[-3000:]
    clusters = json.loads(r.stdout.strip().splitlines()[-1])["clusters"]
    assert clusters == ([2, 4] if two_cta == "1" else [1]), clusters


def test_threshold_pairs(gpu):
    """b2_threshold_pairs on the int8 pair filter (both CTA modes through the group size); the threshold is in units of int8
    inner products"""
    rng = np.random.default_rng(12)
    x = data("gauss", 3000, 64, 12)
    x[1500:1600] = np.clip(x[:100].astype(np.int16) + rng.integers(-1, 2, size=(100, 64)), -128, 127).astype(np.int8)
    x[2000:2010] = x[:10]  # exact duplicates: scores equal to |x|^2
    xf = x.astype(np.float32)
    idx = gpu.Index(x, gpu.I8, 0)
    norms = np.einsum("ij,ij->i", xf, xf)
    for thr in (float(np.median(norms)) * 0.9, float(np.median(norms)) * 0.5, float(norms[0]), float(norms[0]) - 0.5):
        pi, pj = idx.threshold_pairs(thr)
        oi, oj, _ = oracle.threshold_pairs(xf, thr)
        assert np.array_equal(pi, oi) and np.array_equal(pj, oj), thr
    assert len(oi) >= 10  # the last threshold keeps the exact duplicates
    idx.close()


@pytest.mark.parametrize("n,d,k,full", [(30_000, 48, 640, False), (6_000, 30, 17, True), (5_000, 768, 300, True)])
def test_kmeans_bit_identical(gpu, n, d, k, full):
    rng = np.random.default_rng(300 + d)
    centers = rng.integers(-100, 101, size=(min(k, 50), d))
    x = np.clip(centers[rng.integers(0, len(centers), n)] + rng.integers(-20, 21, size=(n, d)), -128, 127).astype(np.int8)
    xf = x.astype(np.float32)
    idx = gpu.Index(x, gpu.I8, 1)
    a, c, obj = idx.kmeans(k, niter=5, full_lloyd=full)
    ao, co, oo = oracle.kmeans(xf, k, niter=5, full_lloyd=full)
    assert np.array_equal(a, ao), f"{(a != ao).sum()} of {n} assignments differ"
    assert np.array_equal(bits(c), bits(co))
    assert np.allclose(obj, oo, rtol=1e-5)
    a2, dist = idx.kmeans_assign(co)
    Dk, Ik = oracle.knn(co, xf, 1, oracle.L2)
    assert np.array_equal(a2, Ik[:, 0]) and np.array_equal(bits(dist), bits(Dk[:, 0]))
    D, I = idx.search(x[:100], 5, gpu.I8)  # the int8 search of the same handle is unaffected by its fp16 k-means copy
    Do, Io = oracle.knn(xf, xf[:100], 5, oracle.L2)
    assert_same(D, I, Do, Io, "search after k-means")
    idx.close()


def test_kmeans_empty_clusters(gpu):
    rng = np.random.default_rng(21)
    x = rng.integers(-60, 61, size=(1500, 16)).astype(np.int8)
    x[rng.random(1500) < 0.7] = x[0]  # duplicates: clusters empty out and split_clusters runs
    xf = x.astype(np.float32)
    idx = gpu.Index(x, gpu.I8, 1)
    a, c, obj = idx.kmeans(24, niter=6, full_lloyd=True)
    ao, co, oo = oracle.kmeans(xf, 24, niter=6, full_lloyd=True)
    assert np.array_equal(a, ao) and np.array_equal(bits(c), bits(co))
    idx.close()


def test_b200vs_int8_store(gpu, tmp_path):
    torch = pytest.importorskip("torch")
    from lotus_b200.vs import B200VS
    x, q = data("gauss", 8000, 64, 41), data("gauss", 50, 64, 42)
    xf, qf = x.astype(np.float32), q.astype(np.float32)
    Do, Io = oracle.knn(xf, qf, 10, oracle.IP)
    vs = B200VS(dtype="i8")
    vs.index(None, x, str(tmp_path / "a"))
    assert vs.b2_index.dtype == gpu.I8
    out = vs(q, 10)
    assert_same(out.distances, out.indices, Do, Io, "host int8 queries")
    out = vs(qf, 10)
    assert_same(out.distances, out.indices, Do, Io, "host float queries")
    out = vs(torch.from_numpy(q).cuda(), 10)
    assert_same(out.distances, out.indices, Do, Io, "device int8 queries")
    got = vs.get_vectors_from_index(str(tmp_path / "a"), [5, 1, 7999])
    assert got.dtype == np.int8 and np.array_equal(got, x[[5, 1, 7999]])
    vs2 = B200VS(dtype="i8")
    vs2.index(None, torch.from_numpy(x).cuda(), str(tmp_path / "b"))  # device hand-off
    out = vs2(q, 10)
    assert_same(out.distances, out.indices, Do, Io, "device hand-off")
    with pytest.raises(ValueError):
        B200VS(dtype="i8").index(None, torch.from_numpy(xf + 0.5).cuda(), str(tmp_path / "c"))
    vs.close()
    vs2.close()
