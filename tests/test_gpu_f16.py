"""fp16 indexes (B2_F16) on the GPU: every entry point against the oracle on the fp32 upcast of the stored fp16 values.

fp16 values and their pairwise products are exact in fp32, so an fp16 store adds no operand error to the filter; fp32 / bf16
queries on it are rounded to fp16 for the filter only, which the certificate covers with a relative term 2^-11 and an absolute
term 2^-25 sqrt(d) for the subnormal range (DESIGN.md §2). Answers must be bit-identical to the oracle either way."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest

import oracle
from helpers import bits, gauss, grid

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def f16(a):
    return np.ascontiguousarray(np.asarray(a, dtype=np.float32).astype(np.float16))


def queries(gpu, q, qdt):
    """(array to ship, dtype code, exact fp32 values) of the fp32 queries q in query dtype qdt."""
    if qdt == "f16":
        h = f16(q)
        return h, gpu.F16, h.astype(np.float32)
    if qdt == "bf16":
        b = gpu.f32_to_bf16_bits(q)
        return b, gpu.BF16, gpu.bf16_bits_to_f32(b)
    return q, gpu.F32, q


def assert_same(D, I, Do, Io, tag=""):
    assert np.array_equal(I, Io), f"{tag}: {(I != Io).any(axis=1).sum()} rows differ"
    assert np.array_equal(bits(D), bits(Do)), f"{tag}: score bits differ"


# d % 8 != 0 (30, 100) takes the padded filter copy; k spans every candidate capacity and the multi-split k > 40 path
@pytest.mark.parametrize("metric", [oracle.IP, oracle.L2])
@pytest.mark.parametrize("d", [30, 96, 100, 384, 768])
def test_f16_store_search_parity(gpu, metric, d):
    n = 6000
    for data in ("grid", "gauss"):
        x = grid(n, d, d) if data == "grid" else gauss(n, d, d)
        q = grid(300, d, d + 1) if data == "grid" else gauss(300, d, d + 1)
        xh = f16(x)
        xf = xh.astype(np.float32)
        idx = gpu.Index(xh, gpu.F16, metric)
        assert idx.dtype == gpu.F16
        for k in (1, 10, 32, 64, 100, 400):
            qdt = ("f16", "f32", "bf16")[k % 3]
            qa, code, qf = queries(gpu, q, qdt)
            gpu.stats_reset()
            D, I = idx.search(qa, k, code)
            st = gpu.stats()
            Do, Io = oracle.knn(xf, qf, k, metric)
            assert_same(D, I, Do, Io, f"{data} d={d} k={k} q={qdt}")
            if data == "gauss" and k <= 100:  # the filter ran and certified (nearly) every query
                assert st["filter_launches"] >= 1 and st["fallback_queries"] <= 3, (data, d, k, qdt, st)
        ids = np.arange(7, n, 3)
        qa, code, qf = queries(gpu, q, "f16")
        D, I = idx.search(qa, 10, code, ids=ids)
        Do, Io = oracle.knn_subset(xf, qf, 10, ids, metric)
        assert_same(D, I, Do, Io, f"{data} d={d} ids=")
        idx.close()


@pytest.mark.parametrize("store", ["bf16", "f32"])
def test_f16_queries_on_bf16_and_fp32_stores(gpu, store):
    x, q = gauss(20_000, 128, 3), gauss(500, 128, 4)
    if store == "bf16":
        xb = gpu.f32_to_bf16_bits(x)
        idx, xf = gpu.Index(xb, gpu.BF16, 0), gpu.bf16_bits_to_f32(xb)
    else:
        idx, xf = gpu.Index(x, gpu.F32, 0), x
    qh = f16(q)
    for k in (1, 10, 32, 100):
        gpu.stats_reset()
        D, I = idx.search(qh, k, gpu.F16)
        Do, Io = oracle.knn(xf, qh.astype(np.float32), k, oracle.IP)
        assert_same(D, I, Do, Io, f"{store} k={k}")
        assert gpu.stats()["fallback_queries"] <= 3
    idx.close()


def test_range_edges_subnormal_and_overflowing_queries(gpu):
    """fp32 queries on an fp16 store with components in fp16's subnormal range (~1e-6) and above 65504: still bit-exact, and
    the queries that would overflow in fp16 go to the dense path."""
    d = 96
    x = gauss(8000, d, 5)
    xh = f16(x)
    xf = xh.astype(np.float32)
    q = gauss(256, d, 6) * np.float32(1e-6) * np.sqrt(d)   # components around 1e-6: below fp16's smallest normal 6.1e-5
    big = gauss(4, d, 7)
    big[:, 0] = 70000.0                                     # rounds to inf in fp16
    big[1, 0] = 65519.0                                     # largest value that still rounds to 65504: finite
    qq = np.concatenate([q, big]).astype(np.float32)
    for metric in (oracle.IP, oracle.L2):
        idx = gpu.Index(xh, gpu.F16, metric)
        gpu.stats_reset()
        D, I = idx.search(qq, 10, gpu.F32)
        st = gpu.stats()
        Do, Io = oracle.knn(xf, qq, 10, metric)
        assert_same(D, I, Do, Io, f"metric {metric}")
        assert st["fallback_queries"] >= 3, st   # the three queries with a component >= 65520 at least
        idx.close()


def test_device_entry_points_and_gather(gpu):
    import torch
    dev = torch.device("cuda", 0)
    x, q = gauss(24_000, 96, 10), gauss(6000, 96, 11)
    xh, qh = f16(x), f16(q)
    xf, qf = xh.astype(np.float32), qh.astype(np.float32)
    k = 32
    st = torch.cuda.current_stream().cuda_stream
    q_dev = torch.from_numpy(qh).to(dev)
    for metric in (oracle.IP, oracle.L2):
        Do, Io = oracle.knn(xf, qf, k, metric)
        idx = gpu.Index(xh, gpu.F16, metric)
        out_s = torch.empty((len(q), k), dtype=torch.float32, device=dev)
        out_i = torch.empty((len(q), k), dtype=torch.int64, device=dev)
        idx.search_dev(q_dev.data_ptr(), len(q), k, gpu.F16, out_s.data_ptr(), out_i.data_ptr(), stream=st)
        assert_same(out_s.cpu().numpy(), out_i.cpu().numpy(), Do, Io, "search_dev")
        # gather hands back the stored fp16 values, on the host and on the device
        ids = np.array([5, 0, 23_999, 77])
        g = idx.gather(ids)
        assert g.dtype == np.float16 and np.array_equal(g.view(np.uint16), xh[ids].view(np.uint16))
        idx.close()
        # row-sharded: packed single-stage and two-stage searches over G = 3 shards in one process
        G = 3
        shards = [gpu.Index(np.ascontiguousarray(xh[g * 8000:(g + 1) * 8000]), gpu.F16, metric) for g in range(G)]
        packed = torch.empty((G, len(q), k), dtype=torch.int64, device=dev)
        for g, s in enumerate(shards):
            s.search_packed_dev(q_dev.data_ptr(), len(q), k, gpu.F16, packed[g].data_ptr(), stream=st)
        gpu.merge_topk_packed_dev(packed.data_ptr(), np.arange(G) * 8000, G, len(q), k, metric, 0, out_s.data_ptr(),
                                  out_i.data_ptr(), stream=st)
        assert_same(out_s.cpu().numpy(), out_i.cpu().numpy(), Do, Io, "packed")
        for qname, qsrc, code in (("f16", q_dev, gpu.F16), ("f32", torch.from_numpy(q).to(dev), gpu.F32)):
            lowers = [torch.empty(len(q), dtype=torch.float32, device=dev) for _ in range(G)]
            j = -(-k // G)
            for s, lo in zip(shards, lowers):
                s.search_stage1_dev(qsrc.data_ptr(), len(q), k, code, j, lo.data_ptr(), stream=st)
            hint = torch.stack(lowers).min(dim=0).values.contiguous()
            assert bool(torch.isfinite(hint).any().item()), "the staged path was not taken"
            for g, s in enumerate(shards):
                s.search_stage2_packed_dev(hint.data_ptr(), packed[g].data_ptr(), stream=st)
            gpu.merge_topk_packed_dev(packed.data_ptr(), np.arange(G) * 8000, G, len(q), k, metric, 0, out_s.data_ptr(),
                                      out_i.data_ptr(), stream=st)
            Dq, Iq = (Do, Io) if qname == "f16" else oracle.knn(xf, q, k, metric)
            assert_same(out_s.cpu().numpy(), out_i.cpu().numpy(), Dq, Iq, f"staged {qname}")
        for s in shards:
            s.close()


def test_threshold_pairs(gpu):
    rng = np.random.default_rng(12)
    x = gauss(3000, 64, 12)
    x[1500:1600] = x[:100] + 1e-3 * rng.standard_normal((100, 64)).astype(np.float32)
    xh = f16(x)
    xf = xh.astype(np.float32)
    idx = gpu.Index(xh, gpu.F16, 0)
    for thr in (0.9, 0.5):
        pi, pj = idx.threshold_pairs(thr)
        oi, oj, _ = oracle.threshold_pairs(xf, thr)
        assert np.array_equal(pi, oi) and np.array_equal(pj, oj), thr
    idx.close()


def _mixture(n, d, k_true, seed):
    rng = np.random.default_rng(seed)
    centers = gauss(k_true, d, seed + 1) * 4
    return (centers[rng.integers(0, k_true, n)] + gauss(n, d, seed + 2, normalize=False)).astype(np.float32)


@pytest.mark.parametrize("n,d,k,full", [(30_000, 48, 640, False), (6_000, 30, 17, True), (5_000, 768, 300, True)])
def test_kmeans_bit_identical(gpu, n, d, k, full):
    xh = f16(_mixture(n, d, min(k, 50), 300 + d))
    xf = xh.astype(np.float32)
    idx = gpu.Index(xh, gpu.F16, 1)
    a, c, obj = idx.kmeans(k, niter=5, full_lloyd=full)
    ao, co, oo = oracle.kmeans(xf, k, niter=5, full_lloyd=full)
    assert np.array_equal(a, ao), f"{(a != ao).sum()} of {n} assignments differ"
    assert np.array_equal(bits(c), bits(co))
    assert np.allclose(obj, oo, rtol=1e-5)
    a2, dist = idx.kmeans_assign(co)
    Dk, Ik = oracle.knn(co, xf, 1, oracle.L2)
    assert np.array_equal(a2, Ik[:, 0]) and np.array_equal(bits(dist), bits(Dk[:, 0]))
    idx.close()


def test_kmeans_empty_clusters_and_out_of_range_centroids(gpu):
    rng = np.random.default_rng(21)
    x = gauss(1500, 16, 22, normalize=False)
    x[rng.random(1500) < 0.7] = x[0]                        # duplicates: split_clusters runs
    xh = f16(x)
    xf = xh.astype(np.float32)
    idx = gpu.Index(xh, gpu.F16, 1)
    a, c, obj = idx.kmeans(24, niter=6, full_lloyd=True)
    ao, co, oo = oracle.kmeans(xf, 24, niter=6, full_lloyd=True)
    assert np.array_equal(a, ao) and np.array_equal(bits(c), bits(co))
    # explicit centroids beyond fp16's range: the assignment filters them in tf32 instead, still exact
    cent = co.copy()
    cent[3] = 1e5
    a2, dist = idx.kmeans_assign(cent)
    Dk, Ik = oracle.knn(cent, xf, 1, oracle.L2)
    assert np.array_equal(a2, Ik[:, 0]) and np.array_equal(bits(dist), bits(Dk[:, 0]))
    idx.close()


def test_b200vs_f16_store_and_device_hand_off(gpu, tmp_path):
    import torch
    from lotus_b200 import B200VS
    x, q = gauss(5000, 64, 30), gauss(50, 64, 31)
    xh = f16(x)
    xf = xh.astype(np.float32)
    vs = B200VS(dtype="f16")
    d = str(tmp_path / "h")
    vs.index(None, xh, d)
    assert vs.b2_index.dtype == gpu.F16
    out = vs(q, 10)
    Do, Io = oracle.knn(xf, q, 10, oracle.IP)
    assert_same(out.distances, out.indices, Do, Io, "fp32 queries")
    got = vs.get_vectors_from_index(d, [3, 1, 4])
    assert got.dtype == np.float16 and np.array_equal(got, xh[[3, 1, 4]])
    out = vs(got, 5)                                         # float16 queries ship as 2-byte operands
    Do, Io = oracle.knn(xf, xf[[3, 1, 4]], 5, oracle.IP)
    assert_same(out.distances, out.indices, Do, Io, "round trip")
    a, c, _ = vs.kmeans(np.arange(5000), 20, niter=3)
    ao, co, _ = oracle.kmeans(xf, 20, niter=3)
    assert np.array_equal(a, ao) and np.array_equal(bits(c), bits(co))
    vs.close()
    # device hand-off: a torch.float16 CUDA tensor is read in place, and CUDA float16 queries are searched in place
    t = torch.from_numpy(xh).to("cuda:0")
    vs = B200VS(dtype="f16")
    vs.index(None, t, str(tmp_path / "t"))
    assert vs.b2_index.dtype == gpu.F16
    out = vs(torch.from_numpy(f16(q)).to("cuda:0"), 10)
    Do, Io = oracle.knn(xf, f16(q).astype(np.float32), 10, oracle.IP)
    assert_same(out.distances, out.indices, Do, Io, "device hand-off")
    vs.close()


# ---- filter lists: every entry against fp64, the fp16 error model pinned --------------------------------------------------
F32, BF16, F16 = 0, 1, 2
LIST_SCRIPT = r"""
import json, sys
sys.path.insert(0, %r); sys.path.insert(0, %r + "/tests")
import test_gpu_f16
from lotus_b200 import _native as nv
print(json.dumps(test_gpu_f16.run_f16_lists(nv)))
""" % (ROOT, ROOT)


def rel_eps_f16(d, store, q):
    """DESIGN.md §2 for an fp16 filter: accumulation (d + 64) 2^-23, 2^-11 for each side rounded to fp16, their product, 1e-6."""
    ex = 0.0 if store == F16 else 2.0 ** -11
    eq = 0.0 if q == F16 else 2.0 ** -11
    return float(np.float32((d + 64) * 2.0 ** -23 + ex + eq + ex * eq + 1e-6))


def abs_eps_f16(d, store, q):
    """2^-25 sqrt(d) for each side rounded to fp16 (half the subnormal spacing, summed over a row)."""
    return float(np.float32(((store != F16) + (q != F16)) * 2.0 ** -25 * np.sqrt(d) * (1 + 1e-6)))


def check_abs_margin(res, Q, X, metric, abs_eps, tag):
    """The list entries against |err| <= rel_eps |q| |x| + abs_eps (|q| + |x|) (per row; twice that plus the epilogue rounding
    for L2), where check_lists' relative-only margin does not apply. -> largest |err| / margin."""
    ids = res["id"].reshape(len(Q), -1)
    sc = res["score"].reshape(len(Q), -1).astype(np.float64)
    r, c = np.nonzero(ids >= 0)
    rows = ids[r, c]
    S = np.einsum("ij,ij->i", Q[r], X[rows])
    xn2 = np.einsum("ij,ij->i", X, X)
    if metric == 1:
        S = 2.0 * S - xn2[rows]
    qn = np.sqrt(np.einsum("ij,ij->i", Q, Q))[r]
    xn = np.sqrt(xn2)[rows]
    m = res["rel_eps"] * qn * xn + abs_eps * (qn + xn)
    if metric == 1:
        m = 2.0 * m + 2.4e-7 * (xn * xn + 2.0 * qn * xn)
    ratio = np.abs(sc[r, c] - S) / np.maximum(m, 1e-300)
    bad = ratio > 1.0
    assert not bad.any(), f"{tag}: entry {int(np.argmax(bad))}: |filter - exact| beyond rel_eps |q||x| + abs_eps (|q| + |x|)"
    return float(ratio.max()) if len(ratio) else 0.0


def f16_list_cases():
    """(store, q dtype, top1, metric, n, d, nq, k, data)."""
    out = []
    for i, (qdt, metric, d, k, data) in enumerate([
            (F16, 0, 64, 10, "gauss"), (F16, 1, 100, 32, "grid"), (F16, 0, 768, 5, "unnorm"),
            (F32, 0, 96, 10, "gauss"), (F32, 1, 30, 41, "gauss"), (F32, 0, 384, 16, "tiny"),
            (BF16, 0, 200, 10, "gauss"), (BF16, 1, 8, 5, "unnorm")]):
        out.append((F16, qdt, False, metric, 2048 + 9 * i, d, 129 + 64 * i, k, data))
    # the k-means TOP1 variant of the fp16 filter, one side rounded to fp16 as the fp32 centroids are in the assignment
    out.append((F16, F32, True, 1, 769, 48, 383, 1, "gauss"))
    out.append((F16, F16, True, 1, 300, 8, 257, 1, "grid"))
    return out


def run_f16_lists(nv):
    import filter_lists as fl
    failures, ratios = [], {}
    for ci, (store, qdt, top1, metric, n, d, nq, k, data) in enumerate(f16_list_cases()):
        if data == "tiny":  # fp32 queries with most components in fp16's subnormal range: the absolute term matters
            x, q = gauss(n, d, 900 + ci), (gauss(nq, d, 901 + ci) * np.float32(3e-5)).astype(np.float32)
        else:
            x, q = fl.make_data(data, n, nq, d, 900 + ci)
        xs = f16(x)
        X = xs.astype(np.float64)
        if qdt == F16:
            qa = f16(q)
            Q = qa.astype(np.float64)
        elif qdt == BF16:
            qa = nv.f32_to_bf16_bits(q)
            Q = nv.bf16_bits_to_f32(qa).astype(np.float64)
        else:
            qa, Q = q, q.astype(np.float64)
        tag = f"f16 case {ci} [store {store} q {qdt}{' top1' if top1 else ''} metric {metric} n={n} d={d} nq={nq} k={k} {data}]"
        try:
            idx = nv.Index(xs, F16, metric)
            try:
                res = idx.filter_lists(qa, k, qdt, top1=top1)
            finally:
                idx.close()
            store_e, q_e = F16, qdt
            assert res["use_filter"], f"{tag}: the plan does not use the filter"
            assert res["filt_dtype"] == F16, f"{tag}: filter operand {res['filt_dtype']}"
            want = rel_eps_f16(d, store_e, q_e)
            assert abs(res["rel_eps"] - want) <= 2.0 ** -23 * want, f"{tag}: rel_eps {res['rel_eps']!r} != formula {want!r}"
            lib_rel, lib_abs = nv.filter_eps(store_e, F16, q_e, d)
            assert lib_rel == res["rel_eps"], tag
            ab = abs_eps_f16(d, store_e, q_e)
            assert abs(lib_abs - ab) <= 2.0 ** -23 * max(ab, 1e-30), f"{tag}: abs_eps {lib_abs!r} != formula {ab!r}"
            if lib_abs == 0.0:
                r = fl.check_lists(res, Q, X, metric, exact=data == "grid", top1=top1, tag=tag)
            else:
                # structure and discard bound through check_lists with the absolute term folded into a relative one for these
                # norms, then every entry against the exact margin
                qn, xn = np.sqrt((Q * Q).sum(1)), np.sqrt((X * X).sum(1))
                fold = lib_abs * float(((qn.max() + xn.max()) / (qn.min() * xn.min())))
                fl.check_lists(dict(res, rel_eps=res["rel_eps"] + fold), Q, X, metric, top1=top1, tag=tag)
                r = check_abs_margin(res, Q, X, metric, lib_abs, tag)
            names = {F32: "fp32", BF16: "bf16", F16: "fp16"}
            key = f"fp16 filter, {names[q_e]} q{' top1' if top1 else ''} d={d} {data}"
            ratios[key] = r
        except AssertionError as e:
            failures.append(str(e))
    return {"failures": failures, "ratios": ratios}


@pytest.mark.parametrize("two_cta", ["1", "0"])
def test_f16_filter_lists_hold_the_certificate_premises(gpu, two_cta):
    r = subprocess.run([sys.executable, "-c", LIST_SCRIPT], capture_output=True, text=True, timeout=900,
                       env=dict(os.environ, B2_FILTER_2CTA=two_cta))
    assert r.returncode == 0, r.stderr[-3000:]
    res = json.loads(r.stdout.strip().splitlines()[-1])
    print(f"\nB2_FILTER_2CTA={two_cta}: largest |err| / margin per fp16 case:")
    for key, v in sorted(res["ratios"].items()):
        print(f"  {key:60s} {v:.4f}")
    assert not res["failures"], "\n".join(res["failures"])
