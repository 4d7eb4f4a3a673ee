"""Range search (b2_index_range_search) on the H100: lims, ids and score bits must equal range_oracle.range_search, the
canonical restatement of faiss IndexFlat.range_search, for every store and query type, both metrics, clusters and single CTAs,
the dense fallback, ids subsets, host-resident stores and the B200VS surface."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest

import oracle
from helpers import gauss, grid
from range_oracle import range_search as oracle_range

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CODES = (0, 1, 2, 8)  # F32, BF16, F16, I8


def store(nv, x, code):
    """(array the C-ABI takes, its fp32 values) of fp32 data x stored as `code` (int8: x * 64 rounded and clipped)."""
    if code == nv.F32:
        a = np.ascontiguousarray(x, np.float32)
    elif code == nv.BF16:
        a = nv.f32_to_bf16_bits(x)
    elif code == nv.F16:
        a = x.astype(np.float16)
    else:
        a = np.clip(np.round(x * 64), -128, 127).astype(np.int8)
    return a, nv.stored_to_f32(a, code)


def same(got, want, tag):
    (lg, dg, ig), (lw, dw, iw) = got, want
    assert np.array_equal(lg, lw), f"{tag}: lims differ ({int((np.diff(lg) != np.diff(lw)).sum())} queries)"
    assert np.array_equal(ig, iw), f"{tag}: ids differ"
    assert np.array_equal(dg.view(np.uint32), dw.view(np.uint32)), f"{tag}: score bits differ"


def radius_for(S, metric, frac):
    """A radius that about `frac` of the scores in S pass."""
    return float(np.quantile(S, 1 - frac) if metric == oracle.IP else np.quantile(S, frac))


def core_cases(nv):
    """Every store with every query type, IP and L2, d in {8, 100, 768, 1000}, odd n and nq. Returns the cluster sizes seen."""
    out = []
    for d, n, nq in [(8, 20_011, 521), (100, 9_001, 261), (768, 3_001, 131), (1000, 3_001, 67)]:
        xf, qf = gauss(n, d, 10 + d), gauss(nq, d, 20 + d)
        for code in CODES:
            x, xv = store(nv, xf, code)
            for metric in (nv.METRIC_IP, nv.METRIC_L2):
                idx = nv.Index(x, code, metric)
                for qd in CODES:
                    q, qv = store(nv, qf, qd)
                    S = oracle.scores(xv, qv, metric)
                    r = radius_for(S, metric, 0.004)
                    tag = f"d={d} n={n} store={code} q={qd} metric={metric}"
                    got = idx.range_search(q, r, qd)
                    same(got, oracle_range(xv, qv, r, metric), tag)
                    st = idx.range_stats()
                    assert st["filtered"] and st["dense_queries"] == 0, tag
                    assert st["candidates_peak"] >= st["hits"] == got[0][-1], tag
                idx.close()
        out.append(d)
    return out


CORE_SCRIPT = """
import json, sys
sys.path.insert(0, %r); sys.path.insert(0, %r)
from lotus_b200 import _native as nv
import test_gpu_range_search as t
print(json.dumps(t.core_cases(nv)))
""" % (ROOT, os.path.join(ROOT, "tests"))


@pytest.mark.gpu
@pytest.mark.parametrize("two_cta", ["1", "0"])
def test_every_type_and_shape_matches_the_oracle(gpu, two_cta):
    r = subprocess.run([sys.executable, "-c", CORE_SCRIPT], capture_output=True, text=True, timeout=1800,
                       env=dict(os.environ, B2_FILTER_2CTA=two_cta))
    assert r.returncode == 0, r.stderr[-3000:]
    assert json.loads(r.stdout.strip().splitlines()[-1]) == [8, 100, 768, 1000]


@pytest.mark.gpu
@pytest.mark.parametrize("metric", [0, 1])
@pytest.mark.parametrize("code", [0, 1, 8])
def test_radius_exactly_at_a_score(gpu, metric, code):
    """Grid data: scores are exact and tie often. Rows scoring exactly the radius are excluded; one ulp further in, included."""
    nv = gpu
    n, d, nq = 12_003, 64, 200
    xf, qf = grid(n, d, 1), grid(nq, d, 2)
    x, xv = store(nv, xf, code)
    q, qv = store(nv, qf, code)
    idx = nv.Index(x, code, metric)
    S = oracle.scores(xv, qv, metric)
    r0 = float(np.sort(S[0])[::-1][50] if metric == nv.METRIC_IP else np.sort(S[0])[50])
    assert (S == np.float32(r0)).sum() > 1
    inward = np.nextafter(np.float32(r0), np.float32(-np.inf if metric == nv.METRIC_IP else np.inf))
    for r in (r0, float(inward)):
        got = idx.range_search(q, r, code)
        want = oracle_range(xv, qv, r, metric)
        same(got, want, f"store={code} metric={metric} r={r!r}")
    at = idx.range_search(q, r0, code)
    past = idx.range_search(q, float(inward), code)
    assert past[0][-1] - at[0][-1] == int((S == np.float32(r0)).sum())
    idx.close()


@pytest.mark.gpu
def test_zero_hits_and_almost_everything(gpu):
    """A radius nothing passes, and one every row passes for half the queries: the candidate buffer overflows and is rerun at
    the exact size, and the host buffers grow through the ERANGE retry."""
    nv = gpu
    n, d, nq = 20_011, 48, 300
    x, xv = store(nv, gauss(n, d, 3), nv.BF16)
    qf = gauss(nq, d, 4)
    qf[::2] *= 0  # zero queries: every row scores 0 (IP) or |x|^2 (L2)
    for metric, r_none, r_most in [(nv.METRIC_IP, 10.0, -0.5), (nv.METRIC_L2, 0.0, 1.5)]:
        idx = nv.Index(x, nv.BF16, metric)
        none = idx.range_search(qf, r_none)
        assert none[0][-1] == 0 and len(none[1]) == 0
        same(none, oracle_range(xv, qf, r_none, metric), f"metric={metric} none")
        most = idx.range_search(qf, r_most, cap=1000)
        assert most[0][-1] > n * nq // 2
        same(most, oracle_range(xv, qf, r_most, metric), f"metric={metric} most")
        idx.close()


@pytest.mark.gpu
def test_two_phase_sized_batch(gpu):
    """20k queries against 100k rows; head and tail of the batch checked against the oracle."""
    nv = gpu
    n, d, nq = 100_003, 64, 20_000
    x, xv = store(nv, gauss(n, d, 7), nv.BF16)
    q, qv = store(nv, gauss(nq, d, 8), nv.BF16)
    idx = nv.Index(x, nv.BF16, nv.METRIC_IP)
    r = radius_for(oracle.scores(xv, qv[:64], nv.METRIC_IP), nv.METRIC_IP, 2e-4)
    lims, D, I = idx.range_search(q, r, nv.BF16)
    for lo, hi in [(0, 256), (nq - 256, nq)]:
        want = oracle_range(xv, qv[lo:hi], r, nv.METRIC_IP)
        got = (lims[lo:hi + 1] - lims[lo], D[lims[lo]:lims[hi]], I[lims[lo]:lims[hi]])
        same(got, want, f"queries [{lo}, {hi})")
    idx.close()


@pytest.mark.gpu
@pytest.mark.parametrize("metric", [0, 1])
def test_dense_fallback_for_queries_past_fp16_range(gpu, metric):
    """fp32 queries whose fp16 rounding overflows have no finite filter margin: the dense path answers them exactly."""
    nv = gpu
    n, d, nq = 8_191, 40, 100
    x, xv = store(nv, gauss(n, d, 5), nv.F16)
    q = gauss(nq, d, 6)
    q[:7] *= 1e5
    idx = nv.Index(x, nv.F16, metric)
    S = oracle.scores(xv, q, metric)
    r = radius_for(S[7:], metric, 0.01)
    same(idx.range_search(q, r, nv.F32), oracle_range(xv, q, r, metric), f"metric={metric}")
    st = idx.range_stats()
    assert st["dense_queries"] == 7 and st["filtered"]
    idx.close()


@pytest.mark.gpu
@pytest.mark.parametrize("metric", [0, 1])
def test_ids_subsets(gpu, metric):
    nv = gpu
    n, d, nq = 30_011, 96, 150
    x, xv = store(nv, gauss(n, d, 9), nv.BF16)
    q, qv = store(nv, gauss(nq, d, 10), nv.BF16)
    idx = nv.Index(x, nv.BF16, metric)
    rng = np.random.default_rng(0)
    r = radius_for(oracle.scores(xv, qv, metric), metric, 0.01)
    subsets = {"sorted": np.sort(rng.choice(n, 9_000, replace=False)), "unsorted": rng.choice(n, 9_000, replace=False),
               "duplicated": rng.integers(0, n, 12_000), "small": rng.choice(n, 100, replace=False),
               "empty": np.empty(0, np.int64)}
    for name, ids in subsets.items():
        got = idx.range_search(q, r, nv.BF16, ids=ids)
        same(got, oracle_range(xv, qv, r, metric, ids=ids), f"metric={metric} ids={name}")
    idx.close()


def ring_for(nv, n, d, code, chunks=6):
    """A ring whose slots hold about n / chunks rows: at least five chunks, the last one not dividing n."""
    esz = {nv.F32: 4, nv.BF16: 2, nv.F16: 2, nv.I8: 1}[code]
    row = -(-d * esz // 16) * 16 + (-(-d // 8) * 16 if code == nv.I8 else 0)
    ring = 2 * max(256, (n // chunks) // 256 * 256) * row
    p = nv.stream_plan(n, d, code, ring)
    assert p["n_chunks"] >= 5 and n % p["chunk_rows"] != 0, p
    return ring


@pytest.mark.gpu
@pytest.mark.parametrize("code", CODES)
def test_host_resident_equals_device_and_oracle(gpu, code):
    nv = gpu
    n, d, nq = 60_001, 72, 261
    xf = gauss(n, d, 12)
    xf[20_000:20_500] = xf[0]  # repeated rows across chunk boundaries: hits on both sides of a cut
    x, xv = store(nv, xf, code)
    for metric in (nv.METRIC_IP, nv.METRIC_L2):
        dev = nv.Index(x, code, metric)
        host = nv.Index(x, code, metric, residency="host", ring_bytes=ring_for(nv, n, d, code))
        for qd in sorted({code, nv.F32}):
            q, _ = store(nv, gauss(nq, d, 13), qd)
            if qd == code:
                q[0] = x[0]  # a query equal to a row repeated across chunk boundaries
            qv = nv.stored_to_f32(q, qd)
            r = radius_for(oracle.scores(xv, qv, metric), metric, 0.003)
            tag = f"store={code} q={qd} metric={metric}"
            want = oracle_range(xv, qv, r, metric)
            got_h = host.range_search(q, r, qd)
            same(got_h, want, tag + " host")
            same(dev.range_search(q, r, qd), want, tag + " device")
            lims, _, I = got_h
            for i in range(nq):
                assert len(np.unique(I[lims[i]:lims[i + 1]])) == lims[i + 1] - lims[i], f"{tag}: query {i} holds a row twice"
            for ids in (np.random.default_rng(1).integers(0, n, 50_000), np.arange(0, n, 97)[::-1].copy()):
                same(host.range_search(q, r, qd, ids=ids), oracle_range(xv, qv, r, metric, ids=ids), tag + f" ids={len(ids)}")
        dev.close()
        host.close()


@pytest.mark.gpu
def test_b200vs_range_search_over_an_index_directory(gpu, tmp_path):
    from lotus_b200 import faiss_io
    from lotus_b200.vs import B200VS
    nv = gpu
    n, d = 10_007, 128
    x = gauss(n, d, 14)
    q = gauss(33, d, 15)
    faiss_io.write_index_dir(str(tmp_path / "ix"), x, x, 0)
    vs = B200VS()
    with pytest.raises(ValueError, match="Index not loaded"):
        vs.range_search(q, 0.5)
    vs.load_index(str(tmp_path / "ix"))
    r = radius_for(oracle.scores(x, q, 0), 0, 0.01)
    same(vs.range_search(q, r), oracle_range(x, q, r, 0), "B200VS")
    ids = np.random.default_rng(2).integers(0, n, 3000)
    same(vs.range_search(q, r, ids=list(ids)), oracle_range(x, q, r, 0, ids=ids), "B200VS ids")
    with pytest.raises(ValueError, match="dimension"):
        vs.range_search(q[:, :64], r)
    vs.close()


@pytest.mark.gpu
def test_b200vs_two_devices(gpu, tmp_path):
    if gpu.device_count() < 2:
        pytest.skip("needs two H100s")
    from lotus_b200.vs import B200VS
    n, d = 20_011, 64
    x, q = gauss(n, d, 16), gauss(50, d, 17)
    vs = B200VS(devices=[0, 1])
    vs.index(None, x, str(tmp_path / "ix"))
    r = radius_for(oracle.scores(x, q, 0), 0, 0.01)
    same(vs.range_search(q, r), oracle_range(x, q, r, 0), "two devices")
    ids = np.random.default_rng(3).integers(0, n, 5000)
    same(vs.range_search(q, r, ids=ids), oracle_range(x, q, r, 0, ids=ids), "two devices ids")
    vs.close()
