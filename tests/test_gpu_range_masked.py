"""Masked range search (b2_index_range_search_masked) on the H100: the rows a bitmap selects are searched in place, and every
result must equal, in lims, ids and score bits, both the gathered range search over ids = flatnonzero(mask) and the oracle over
x[mask] with the positions mapped back to rows. Every store and query type, IP and L2, both CTA modes, the dense path, a
host-resident ring and the B200VS surface; one test shows that the mask acts in the filter, not after it."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest

import oracle
from helpers import gauss, grid
from test_gpu_range_search import radius_for, ring_for, same, store
from test_range_masked_host import masked_oracle

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CODES = (0, 1, 2, 8)  # F32, BF16, F16, I8


def masks(nv, n, seed):
    """name -> (mask as the call takes it, bool[n] it stands for). n is not a multiple of 32, so the last word has bits past n."""
    assert n % 32
    rng = np.random.default_rng(seed)
    one = np.zeros(n, bool)
    one[rng.integers(n)] = True
    half = rng.random(n) < 0.5
    tail = nv.pack_mask(half, n).copy()
    tail[-1] |= np.uint32((0xFFFFFFFF << (n % 32)) & 0xFFFFFFFF)  # set bits at or past n: ignored
    return {"zeros": (np.zeros(n, bool), np.zeros(n, bool)), "one row": (one, one), "ones": (np.ones(n, bool), np.ones(n, bool)),
            "random 0.1": (rng.random(n) < 0.1,) * 2, "random 0.5": (half, half), "bits past n": (tail, half)}


def check(idx, xv, q, qv, qd, r, metric, mask, sel, tag, n_oracle=None):
    """The masked search against the gathered search and the oracle (on the first n_oracle queries). Returns its result and
    its range_stats."""
    got = idx.range_search_masked(q, r, qd, mask)
    st = idx.range_stats()
    ids = np.flatnonzero(sel)
    if len(ids) == 0:
        assert got[0].tolist() == [0] * (len(q) + 1) and len(got[2]) == 0, f"{tag}: an empty mask reports rows"
    same(got, idx.range_search(q, r, qd, ids=ids), tag + " vs gathered")
    m = len(q) if n_oracle is None else n_oracle
    lims, D, I = got
    head = (lims[:m + 1], D[:lims[m]], I[:lims[m]])
    same(head, masked_oracle(xv, qv[:m], r, metric, sel), tag + " vs oracle")
    return got, st


def core_cases(nv):
    """Every store with every query type, IP and L2, d in {8, 100, 768}, every mask shape. Returns the d values done."""
    out = []
    for d, n, nq in [(8, 20_011, 521), (100, 9_001, 261), (768, 3_001, 131)]:
        xf, qf = gauss(n, d, 30 + d), gauss(nq, d, 40 + d)
        for code in CODES:
            x, xv = store(nv, xf, code)
            for metric in (nv.METRIC_IP, nv.METRIC_L2):
                idx = nv.Index(x, code, metric)
                for qd in CODES:
                    q, qv = store(nv, qf, qd)
                    r = radius_for(oracle.scores(xv, qv[:64], metric), metric, 0.01)
                    for name, (mask, sel) in masks(nv, n, d + code + qd).items():
                        tag = f"d={d} n={n} store={code} q={qd} metric={metric} mask={name}"
                        got, st = check(idx, xv, q, qv, qd, r, metric, mask, sel, tag)
                        assert st["filtered"] and st["dense_queries"] == 0, tag
                        assert st["candidates_peak"] >= st["hits"] == got[0][-1], tag
                idx.close()
        out.append(d)
    return out


CORE_SCRIPT = """
import json, sys
sys.path.insert(0, %r); sys.path.insert(0, %r)
from lotus_b200 import _native as nv
import test_gpu_range_masked as t
print(json.dumps(t.core_cases(nv)))
""" % (ROOT, os.path.join(ROOT, "tests"))


@pytest.mark.gpu
@pytest.mark.parametrize("two_cta", ["1", "0"])
def test_every_type_and_mask_matches_the_gathered_search_and_the_oracle(gpu, two_cta):
    r = subprocess.run([sys.executable, "-c", CORE_SCRIPT], capture_output=True, text=True, timeout=1800,
                       env=dict(os.environ, B2_FILTER_2CTA=two_cta))
    assert r.returncode == 0, r.stderr[-3000:]
    assert json.loads(r.stdout.strip().splitlines()[-1]) == [8, 100, 768]


@pytest.mark.gpu
@pytest.mark.parametrize("metric", [0, 1])
@pytest.mark.parametrize("code", [0, 1, 8])
def test_radius_exactly_at_a_score(gpu, metric, code):
    """Grid data: scores are exact and tie often. A selected row scoring exactly the radius is excluded; one ulp further in,
    included."""
    nv = gpu
    n, d, nq = 12_003, 64, 200
    x, xv = store(nv, grid(n, d, 21), code)
    q, qv = store(nv, grid(nq, d, 22), code)
    idx = nv.Index(x, code, metric)
    sel = np.random.default_rng(23).random(n) < 0.5
    S = oracle.scores(xv[sel], qv, metric)
    r0 = float(np.sort(S[0])[::-1][30] if metric == nv.METRIC_IP else np.sort(S[0])[30])
    assert (S == np.float32(r0)).sum() > 1
    inward = float(np.nextafter(np.float32(r0), np.float32(-np.inf if metric == nv.METRIC_IP else np.inf)))
    at, _ = check(idx, xv, q, qv, code, r0, metric, sel, sel, f"store={code} metric={metric} at")
    past, _ = check(idx, xv, q, qv, code, inward, metric, sel, sel, f"store={code} metric={metric} inward")
    assert past[0][-1] - at[0][-1] == int((S == np.float32(r0)).sum())
    idx.close()


@pytest.mark.gpu
@pytest.mark.parametrize("metric", [0, 1])
def test_dense_path_skips_the_cleared_rows(gpu, metric):
    """Fewer than 512 rows (every query verified densely), and fp32 queries past the fp16 range on an fp16 store (those
    queries verified densely): the dense verification must leave the cleared rows out."""
    nv = gpu
    n, d, nq = 333, 24, 70
    x, xv = store(nv, gauss(n, d, 24), nv.BF16)
    q, qv = store(nv, gauss(nq, d, 25), nv.BF16)
    idx = nv.Index(x, nv.BF16, metric)
    r = radius_for(oracle.scores(xv, qv, metric), metric, 0.2)
    for name, (mask, sel) in masks(nv, n, 26).items():
        _, st = check(idx, xv, q, qv, nv.BF16, r, metric, mask, sel, f"n={n} metric={metric} mask={name}")
        assert not st["filtered"] and st["dense_queries"] == nq
    idx.close()
    n, d, nq = 8_191, 40, 100
    x, xv = store(nv, gauss(n, d, 27), nv.F16)
    q = gauss(nq, d, 28)
    q[:7] *= 1e5
    idx = nv.Index(x, nv.F16, metric)
    r = radius_for(oracle.scores(xv, q[7:], metric), metric, 0.01)
    for name, (mask, sel) in masks(nv, n, 29).items():
        _, st = check(idx, xv, q, q, nv.F32, r, metric, mask, sel, f"fp16 store, large queries, metric={metric} mask={name}")
        assert st["filtered"] and st["dense_queries"] == 7
    idx.close()


@pytest.mark.gpu
def test_the_mask_acts_in_the_filter(gpu):
    """64 queries with thousands of hits over the whole index: under a one-row mask the filter emits at most one candidate per
    query, and under an all-zero mask none."""
    nv = gpu
    n, d, nq = 100_003, 64, 64
    x, xv = store(nv, gauss(n, d, 31), nv.BF16)
    q, qv = store(nv, gauss(nq, d, 32), nv.BF16)
    idx = nv.Index(x, nv.BF16, nv.METRIC_IP)
    r = radius_for(oracle.scores(xv, qv, nv.METRIC_IP), nv.METRIC_IP, 0.001)
    full = idx.range_search(q, r, nv.BF16)
    assert full[0][-1] >= 2000 and idx.range_stats()["candidates_peak"] >= full[0][-1]
    one = np.zeros(n, bool)
    one[full[2][0]] = True  # a row that is a hit of query 0
    got, st = check(idx, xv, q, qv, nv.BF16, r, nv.METRIC_IP, one, one, "one row")
    assert st["filtered"] and st["dense_queries"] == 0 and 1 <= got[0][-1] <= st["candidates_peak"] <= nq, st
    _, st = check(idx, xv, q, qv, nv.BF16, r, nv.METRIC_IP, np.zeros(n, bool), np.zeros(n, bool), "zeros")
    assert st["filtered"] and st["candidates_peak"] == 0 and st["hits"] == 0, st
    idx.close()


@pytest.mark.gpu
@pytest.mark.parametrize("code", CODES)
def test_host_resident_equals_device_and_oracle(gpu, code):
    """A small ring: several chunks, the last one re-streaming its predecessor's tail from a row that is not on a word
    boundary; the masked search of the host-resident index equals the device-resident one and the oracle."""
    nv = gpu
    n, d, nq = 60_001, 72, 261
    x, xv = store(nv, gauss(n, d, 33), code)
    ring = ring_for(nv, n, d, code)
    plan = nv.stream_plan(n, d, code, ring)
    assert (n - plan["chunk_rows"]) % 32 != 0, plan
    for metric in (nv.METRIC_IP, nv.METRIC_L2):
        dev = nv.Index(x, code, metric)
        host = nv.Index(x, code, metric, residency="host", ring_bytes=ring)
        for qd in sorted({code, nv.F32}):
            q, qv = store(nv, gauss(nq, d, 34), qd)
            r = radius_for(oracle.scores(xv, qv[:64], metric), metric, 0.005)
            for name, (mask, sel) in masks(nv, n, 35 + code).items():
                tag = f"host store={code} q={qd} metric={metric} mask={name}"
                nv.stats_reset()
                got, _ = check(host, xv, q, qv, qd, r, metric, mask, sel, tag, n_oracle=64)
                assert nv.stats()["streamed_chunks"] >= plan["n_chunks"], tag
                same(got, dev.range_search_masked(q, r, qd, mask), tag + " vs device")
        dev.close()
        host.close()


@pytest.mark.gpu
def test_b200vs_subset_mask_equals_gather(gpu, tmp_path):
    from lotus_b200 import faiss_io
    from lotus_b200.vs import B200VS
    n, d = 10_007, 128
    x, q = gauss(n, d, 36), gauss(33, d, 37)
    faiss_io.write_index_dir(str(tmp_path / "ix"), x, x, 0)
    r = radius_for(oracle.scores(x, q, 0), 0, 0.01)
    rng = np.random.default_rng(38)
    stores = {mode: B200VS(subset=mode) for mode in ("gather", "mask")}
    for vs in stores.values():
        vs.load_index(str(tmp_path / "ix"))
    for ids in (np.sort(rng.choice(n, 3000, replace=False)), np.arange(n), np.array([n - 1])):
        want = masked_oracle(x, q, r, 0, np.isin(np.arange(n), ids))
        got = {mode: vs.range_search(q, r, ids=list(ids)) for mode, vs in stores.items()}
        same(got["mask"], got["gather"], f"mask vs gather, {len(ids)} ids")
        same(got["mask"], want, f"mask vs oracle, {len(ids)} ids")
        same(stores["gather"].range_search_masked(q, r, np.isin(np.arange(n), ids)), want, f"range_search_masked, {len(ids)} ids")
    for vs in stores.values():
        vs.close()


@pytest.mark.gpu
def test_b200vs_two_devices(gpu, tmp_path):
    if gpu.device_count() < 2:
        pytest.skip("needs two H100s")
    from lotus_b200.vs import B200VS
    n, d = 20_011, 64
    x, q = gauss(n, d, 39), gauss(50, d, 40)
    vs = B200VS(devices=[0, 1], subset="mask")
    vs.index(None, x, str(tmp_path / "ix"))
    r = radius_for(oracle.scores(x, q, 0), 0, 0.01)
    sel = np.random.default_rng(41).random(n) < 0.3
    same(vs.range_search_masked(q, r, sel), masked_oracle(x, q, r, 0, sel), "two devices, mask")
    same(vs.range_search(q, r, ids=np.flatnonzero(sel)), masked_oracle(x, q, r, 0, sel), "two devices, subset='mask'")
    vs.close()
