"""Host-resident indexes (b2_index_create_host) on the H100: every search streams the rows through a small device ring in
several chunks, and must return the indices and score bits of a device-resident index over the same rows, and of the oracle.
The folded candidate lists are checked against fp64 in both CTA modes, since an end-to-end test would only see a broken fold
as a query sent to the dense path."""
import ctypes
import json
import os
import subprocess
import sys

import numpy as np
import pytest

import oracle
from helpers import gauss, grid

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
KS = [1, 5, 32, 64, 100, 1000]


def ring_row_bytes(nv, d, code):
    esz = {nv.F32: 4, nv.BF16: 2, nv.F16: 2, nv.I8: 1}[code]
    align = 16 // esz
    b = -(-d // align) * align * esz
    return b + (-(-d // 8) * 8 * 2 if code == nv.I8 else 0)


def ring_for(nv, n, d, code, chunks=6):
    """A ring whose slots hold about n / chunks rows: at least five chunks, the last one not dividing n."""
    rows = max(256, (n // chunks) // 256 * 256)
    ring = 2 * rows * ring_row_bytes(nv, d, code)
    p = nv.stream_plan(n, d, code, ring)
    assert p["n_chunks"] >= 5 and n % p["chunk_rows"] != 0, p
    return ring


def store(nv, x, code):
    """(array the C-ABI takes, its fp32 values) of fp32 data x stored as `code`."""
    if code == nv.F32:
        a = np.ascontiguousarray(x, np.float32)
    elif code == nv.BF16:
        a = nv.f32_to_bf16_bits(x)
    elif code == nv.F16:
        a = x.astype(np.float16)
    else:
        a = np.clip(np.round(x * 64), -128, 127).astype(np.int8)
    return a, nv.stored_to_f32(a, code)


def same(a, b, tag):
    (Da, Ia), (Db, Ib) = a, b
    assert np.array_equal(Ia, Ib), f"{tag}: indices differ ({int((Ia != Ib).any(axis=1).sum())} queries)"
    assert np.array_equal(Da.view(np.uint32), Db.view(np.uint32)), f"{tag}: score bits differ"


QDTYPES = {0: (0, 8), 1: (1, 0), 2: (2, 8), 8: (8, 0)}  # store -> query types (i8 queries, fp32 on the fp32 two-level path)


@pytest.mark.gpu
@pytest.mark.parametrize("d,n", [(8, 300_001), (100, 200_003), (768, 60_001)])
@pytest.mark.parametrize("code", [0, 1, 2, 8])
def test_streamed_search_equals_device_index_and_oracle(gpu, d, n, code):
    nv = gpu
    x, xv = store(nv, gauss(n, d, 10 + d), code)
    nq = 520  # five query tiles: the filter runs clusters of CTAs
    qf = gauss(nq, d, 20 + d)
    for metric in (nv.METRIC_IP, nv.METRIC_L2):
        if code == nv.I8 and metric == nv.METRIC_L2 and d > 32767:
            continue
        dev = nv.Index(x, code, metric)
        host = nv.Index(x, code, metric, residency="host", ring_bytes=ring_for(nv, n, d, code))
        assert host.resident == "host" and dev.resident == "device" and host.data_ptr == 0
        try:
            for qd in QDTYPES[code]:
                q, qv = store(nv, qf, qd)
                for k in KS:
                    if k == 1000 and (d != 100 or qd != QDTYPES[code][0]):
                        continue  # the dense path over every row: once per store
                    tag = f"d={d} n={n} store={code} q={qd} metric={metric} k={k}"
                    nv.stats_reset()
                    got = host.search(q, k, qd)
                    st = nv.stats()
                    assert st["streamed_chunks"] >= 5 or k == 1000, (tag, st)
                    same(got, dev.search(q, k, qd), tag + " vs device")
                    if k in (5, 100):
                        Do, Io = oracle.knn(xv, qv[:16], k, metric)
                        same((got[0][:16], got[1][:16]), (Do, Io), tag + " vs oracle")
        finally:
            host.close()
            dev.close()


@pytest.mark.gpu
@pytest.mark.parametrize("metric", [0, 1])
def test_ties_across_chunk_boundaries(gpu, metric):
    """Grid data (exact scores, many ties) with duplicated rows on both sides of every chunk boundary and of the overlap of
    the last chunk: the tie rule must pick the same rows as on the device."""
    nv = gpu
    n, d = 250_007, 64
    x = grid(n, d, 3)
    ring = ring_for(nv, n, d, nv.BF16)
    p = nv.stream_plan(n, d, nv.BF16, ring)
    R = p["chunk_rows"]
    q = grid(600, d, 4)
    for c in range(1, p["n_chunks"]):
        for b in (c * R, n - R):
            x[b - 4:b + 4] = x[c]  # the same row on both sides of the boundary
            x[b - 2] = q[c % len(q)]  # and one that scores high for a query
    xb, xv = store(nv, x, nv.BF16)
    qb, qv = store(nv, q, nv.BF16)
    dev = nv.Index(xb, nv.BF16, metric)
    host = nv.Index(xb, nv.BF16, metric, residency="host", ring_bytes=ring)
    try:
        for k in (1, 5, 32, 100):
            got = host.search(qb, k, nv.BF16)
            same(got, dev.search(qb, k, nv.BF16), f"grid k={k}")
            Do, Io = oracle.knn(xv, qv[:32], k, metric)
            same((got[0][:32], got[1][:32]), (Do, Io), f"grid k={k} vs oracle")
    finally:
        host.close()
        dev.close()


@pytest.mark.gpu
def test_dense_path_shapes(gpu):
    """Shapes the filter does not take: k beyond its lists, and a corpus too short to tile."""
    nv = gpu
    for n, k in [(300, 10), (5000, 2000)]:
        x, xv = store(nv, gauss(n, 40, n), nv.F32)
        q = gauss(50, 40, 1)
        dev = nv.Index(x, nv.F32, nv.METRIC_L2)
        host = nv.Index(x, nv.F32, nv.METRIC_L2, residency="host", ring_bytes=2 * 256 * 160)
        try:
            nv.stats_reset()
            got = host.search(q, k)
            assert nv.stats()["fallback_queries"] == 50
            same(got, dev.search(q, k), f"dense n={n} k={k}")
            same(got, oracle.knn(xv, q, k, nv.METRIC_L2), f"dense n={n} k={k} vs oracle")
        finally:
            host.close()
            dev.close()


@pytest.mark.gpu
@pytest.mark.parametrize("code", [0, 1, 8])
def test_ids_subsets(gpu, code):
    nv = gpu
    n, d = 120_011, 96
    x, xv = store(nv, gauss(n, d, 5), code)
    qf = gauss(300, d, 6)
    q, qv = store(nv, qf, nv.F32)
    ring = ring_for(nv, n, d, code)
    rng = np.random.default_rng(7)
    small = rng.choice(n, 2000, replace=False)
    large = rng.permutation(n)[: n * 4 // 5]  # more rows than the ring holds: gathered on the host and streamed
    assert len(large) * ring_row_bytes(nv, d, code) > ring
    for metric in (0, 1):
        dev = nv.Index(x, code, metric)
        host = nv.Index(x, code, metric, residency="host", ring_bytes=ring)
        try:
            for name, ids in [("identity", np.arange(n)), ("small", small), ("large", large)]:
                for k in (5, 64):
                    tag = f"ids={name} store={code} metric={metric} k={k}"
                    nv.stats_reset()
                    got = host.search(q, k, nv.F32, ids=ids)
                    if name != "small":
                        assert nv.stats()["streamed_chunks"] >= 5, tag
                    same(got, dev.search(q, k, nv.F32, ids=ids), tag)
                    if k == 5:
                        Do, Io = oracle.knn_subset(xv, qv[:8], k, ids, metric)
                        same((got[0][:8], got[1][:8]), (Do, Io), tag + " vs oracle")
        finally:
            host.close()
            dev.close()


@pytest.mark.gpu
def test_search_dev_and_gather(gpu):
    import torch
    nv = gpu
    n, d = 90_001, 128
    x, xv = store(nv, gauss(n, d, 8), nv.BF16)
    ring = ring_for(nv, n, d, nv.BF16)
    dev = nv.Index(x, nv.BF16, 0)
    host = nv.Index(x, nv.BF16, 0, residency="host", ring_bytes=ring)
    try:
        q = torch.from_numpy(gauss(700, d, 9)).cuda().to(torch.bfloat16)
        ids = torch.from_numpy(np.random.default_rng(1).permutation(n)[: n // 2]).cuda()
        for use_ids in (False, True):
            outs = []
            for idx in (host, dev):
                s = torch.empty((700, 32), dtype=torch.float32, device="cuda")
                i = torch.empty((700, 32), dtype=torch.int64, device="cuda")
                idx.search_dev(q.data_ptr(), 700, 32, nv.BF16, s.data_ptr(), i.data_ptr(), id_offset=0 if use_ids else 7,
                               ids_ptr=ids.data_ptr() if use_ids else None, n_ids=len(ids) if use_ids else 0,
                               stream=torch.cuda.current_stream().cuda_stream)
                torch.cuda.synchronize()
                outs.append((s.cpu().numpy(), i.cpu().numpy()))
            same(outs[0], outs[1], f"search_dev ids={use_ids}")
        assert host.last_filter_ms() > 0
        t = host.stream_times()
        assert t["copy_ms"] > 0 and t["filter_ms"] > 0 and t["span_ms"] >= t["filter_ms"] * 0.99 and t["finalize_ms"] > 0
        g = np.array([0, n - 1, 5, 77_000, 5])
        assert np.array_equal(host.gather(g), x[g])
        gd = torch.from_numpy(g).cuda()
        out = torch.empty((len(g), d), dtype=torch.int16, device="cuda")
        nv.check(nv.lib().b2_index_gather(host.handle, ctypes.c_void_p(gd.data_ptr()), len(g), ctypes.c_void_p(out.data_ptr()), 1))
        torch.cuda.synchronize()
        assert np.array_equal(out.cpu().numpy().view(np.uint16), x[g])
        with pytest.raises(nv.NativeError) as e:
            host.gather([n])
        assert e.value.code == nv.ERANGE
    finally:
        host.close()
        dev.close()


@pytest.mark.gpu
def test_stats_count_chunks_and_bytes(gpu):
    nv = gpu
    n, d = 150_001, 200
    x, _ = store(nv, gauss(n, d, 11), nv.BF16)
    ring = ring_for(nv, n, d, nv.BF16)
    p = nv.stream_plan(n, d, nv.BF16, ring)
    host = nv.Index(x, nv.BF16, 0, residency="host", ring_bytes=ring)
    try:
        q, _ = store(nv, gauss(1000, d, 12), nv.BF16)
        nv.stats_reset()
        host.search(q, 10, nv.BF16)
        st = nv.stats()
        assert st["streamed_chunks"] == p["n_chunks"]
        assert st["streamed_bytes"] == p["n_chunks"] * p["chunk_rows"] * d * 2
        assert st["queries"] == 1000 and st["filter_launches"] >= p["n_chunks"]
    finally:
        host.close()


LISTS_SCRIPT = r"""
import json, sys
sys.path.insert(0, %r); sys.path.insert(0, %r + "/tests")
import numpy as np
import filter_lists as fl
from helpers import gauss, grid
from lotus_b200 import _native as nv

def check_folded(res, Q, X, metric, exact, tag):
    # the certificate's premises for the folded lists: (a) every score within eps of exact, (b) every row the lists do not
    # hold scores at most thr + eps; plus no row twice and only real rows
    nq, n = len(Q), len(X)
    ids = res["id"].reshape(nq, -1).astype(np.int64)
    V = res["score"].reshape(nq, -1).astype(np.float64)
    T = res["thr"].reshape(nq, -1)[:, 0].astype(np.float64)
    assert (res["thr"].reshape(nq, -1)[:, 1] == res["thr"].reshape(nq, -1)[:, 0]).all(), tag
    S = fl.scores(Q, X, metric)
    qn = np.sqrt(np.einsum("ij,ij->i", Q, Q))
    xn = np.sqrt(np.einsum("ij,ij->i", X, X))
    eps = np.zeros(nq) if exact else fl._margins(metric, res["rel_eps"], qn, xn.max())[0]
    valid = ids >= 0
    assert ((ids >= -1) & (ids < n)).all() and (V[~valid] == -np.inf).all(), tag + ": bad empty entries"
    for r in range(nq):
        L = ids[r][valid[r]]
        assert len(np.unique(L)) == len(L), f"{tag}: query {r} holds a row twice"
        err = np.abs(V[r][valid[r]] - S[r, L])
        assert (err <= eps[r]).all(), f"{tag}: accuracy: query {r} |err| {err.max()} > eps {eps[r]}"
        held = np.zeros(n, bool)
        held[L] = True
        top = np.max(np.where(held, -np.inf, S[r]))
        assert top <= T[r] + eps[r], f"{tag}: discard bound: query {r} drops a row of score {top} > thr {T[r]} + {eps[r]}"
    return True

out = []
for code, qd, level, metric, data, k in [(1, 1, 0, 0, "gauss", 10), (1, 0, 0, 1, "grid", 32), (0, 0, 0, 0, "gauss", 4),
                                          (0, 0, 1, 1, "gauss", 100), (2, 2, 0, 1, "gauss", 64), (8, 8, 0, 0, "grid", 5)]:
    n, d, nq = 40_009, 72, 520
    x, q = (grid(n, d, 1), grid(nq, d, 2)) if data == "grid" else (gauss(n, d, 1), gauss(nq, d, 2))
    if code == 8:
        xs, qs = (x * 64).astype(np.int8), (q * 64).astype(np.int8)
    elif code == 1:
        xs = nv.f32_to_bf16_bits(x); qs = nv.f32_to_bf16_bits(q) if qd == 1 else q
    elif code == 2:
        xs, qs = x.astype(np.float16), q.astype(np.float16)
    else:
        xs, qs = x, q
    X = nv.stored_to_f32(xs, code).astype(np.float64)
    Q = nv.stored_to_f32(qs, qd).astype(np.float64)
    esz = {0: 4, 1: 2, 2: 2, 8: 1}[code]
    ring = 2 * 6656 * (-(-d * esz // 16) * 16 + (-(-d // 8) * 16 if code == 8 else 0))
    idx = nv.Index(xs, code, metric, residency="host", ring_bytes=ring)
    res = idx.filter_lists(qs, k, qd, level=level)
    idx.close()
    tag = f"store={code} q={qd} level={level} metric={metric} {data} k={k}"
    assert res["use_filter"] and res["n_splits"] == 1, tag
    assert res["two_level"] == (code == 0 and level == 0 and k <= 24), tag
    check_folded(res, Q, X, metric, data == "grid" and not res["two_level"] and code != 0, tag)
    out.append({"tag": tag, "cluster": res["cluster"]})
print(json.dumps(out))
""" % (ROOT, ROOT)


@pytest.mark.gpu
@pytest.mark.parametrize("two_cta", ["1", "0"])
def test_folded_lists_hold_the_certificate_premises(gpu, two_cta):
    r = subprocess.run([sys.executable, "-c", LISTS_SCRIPT], capture_output=True, text=True, timeout=900,
                       env=dict(os.environ, B2_FILTER_2CTA=two_cta))
    assert r.returncode == 0, r.stderr[-3000:]
    res = json.loads(r.stdout.strip().splitlines()[-1])
    assert len(res) == 6
    assert any(c["cluster"] > 1 for c in res) == (two_cta == "1")


@pytest.mark.gpu
def test_unsupported_operations_fail_loudly(gpu):
    nv = gpu
    x, _ = store(nv, gauss(5000, 32, 1), nv.BF16)
    host = nv.Index(x, nv.BF16, 0, residency="host")
    try:
        for call in (lambda: host.threshold_pairs(0.9), lambda: host.kmeans(4, niter=2),
                     lambda: host.kmeans_assign(np.zeros((4, 32), np.float32))):
            with pytest.raises(nv.NativeError) as e:
                call()
            assert e.value.code == nv.EINVAL and "host-resident" in e.value.msg
        import torch
        q = torch.zeros((4, 32), dtype=torch.bfloat16, device="cuda")
        out = torch.empty((4, 2), dtype=torch.int64, device="cuda")
        with pytest.raises(nv.NativeError) as e:
            host.search_packed_dev(q.data_ptr(), 4, 2, nv.BF16, out.data_ptr())
        assert e.value.code == nv.EINVAL and "host-resident" in e.value.msg
        lower = torch.empty(4, dtype=torch.float32, device="cuda")
        with pytest.raises(nv.NativeError) as e:
            host.search_stage1_dev(q.data_ptr(), 4, 2, nv.BF16, 1, lower.data_ptr())
        assert e.value.code == nv.EINVAL
    finally:
        host.close()


@pytest.mark.gpu
def test_b200vs_host_residency_gives_the_same_frames(gpu, tmp_path):
    import pandas as pd
    import lotus_b200 as lotus
    from lotus_b200.vs import B200VS
    rm = lotus.HashRM(dim=32)
    frames = {}
    for where in ("device", "host"):
        vs = B200VS(residency=where, ring_bytes=2 * 512 * 128 if where == "host" else None)
        lotus.settings.configure(rm=rm, vs=vs, enable_cache=False)
        try:
            left = pd.DataFrame({"a": [f"left {i}" for i in range(700)]})
            right = pd.DataFrame({"b": [f"doc {i % 2900} x{i}" for i in range(3000)]}).sem_index("b", str(tmp_path / where / "r"))
            assert vs.resident(str(tmp_path / where / "r")) == where
            j = left.sem_sim_join(right, "a", "b", K=7)
            s = right.sem_search("b", "doc 17", K=20, return_scores=True)
            frames[where] = (j, s)
            if where == "host":
                with pytest.raises(ValueError, match="host-resident"):
                    vs.threshold_pairs(0.5)
                with pytest.raises(ValueError, match="host-resident"):
                    vs.kmeans(np.arange(10), 2)
        finally:
            lotus.settings.configure(rm=None, vs=None)
            vs.close()
    for a, b in zip(frames["device"], frames["host"]):
        pd.testing.assert_frame_equal(a, b)
