"""Masked search (b2_index_search_masked) on the H100: the rows a bitmap selects are searched in place, and every result must
equal, in indices and score bits, both the gathered search over ids = flatnonzero(mask) and the oracle over x[mask] with the
ids mapped back. The raw lists of a masked filter run are checked against fp64 as well: an end-to-end test alone would see a
broken masked epilogue only as queries sent to the dense path."""
import json
import os
import subprocess
import sys

import numpy as np
import pandas as pd
import pytest

import filter_lists as fl
import oracle
from helpers import bits, gauss, grid
from test_gpu_host_resident import ring_row_bytes, store

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
KS = [1, 5, 32, 100, 1000]
N = 70_001  # a ragged last tile (256 rows) and last mask word (32 rows)
NQ = 520    # five query tiles: clusters of four CTAs


def masks(n, seed):
    """name -> bool[n]: the mask shapes the kernel treats differently."""
    rng = np.random.default_rng(seed)
    out = {f"random {p}": rng.random(n) < p for p in (0.9, 0.5, 0.05, 0.001)}
    block = np.zeros(n, bool)
    block[n // 3 + 5: n // 3 + 5 + n // 4] = True
    out["block"] = block
    tiles = rng.random(n) < 0.6
    for t in rng.choice(n // 256, size=n // 512, replace=False):  # whole corpus tiles without a selected row
        tiles[256 * t: 256 * (t + 1)] = False
    out["tiles cleared"] = tiles
    last = np.zeros(n, bool)
    last[-1] = True
    out["last row"] = last
    out["ones"] = np.ones(n, bool)
    out["zeros"] = np.zeros(n, bool)
    few = np.zeros(n, bool)
    few[rng.choice(n, size=3, replace=False)] = True
    out["three rows"] = few
    return out


def same(a, b, tag):
    (Da, Ia), (Db, Ib) = a, b
    assert np.array_equal(Ia, Ib), f"{tag}: indices differ ({int((Ia != Ib).any(axis=1).sum())} queries)"
    assert np.array_equal(bits(Da), bits(Db)), f"{tag}: score bits differ"


def check_masked(nv, idx, xv, q, qv, qd, k, mask, metric, tag, n_oracle=8):
    got = idx.search_masked(q, k, qd, mask)
    ids = np.flatnonzero(mask)
    m = len(ids)
    pad = np.float32(np.finfo(np.float32).max if metric == nv.METRIC_L2 else -np.finfo(np.float32).max)
    assert int((got[1] == -1).sum()) == len(q) * max(0, k - m), f"{tag}: padding count"
    assert (got[0][got[1] == -1] == pad).all(), f"{tag}: padding scores"
    if m == 0:
        assert (got[1] == -1).all(), f"{tag}: an empty mask reports rows"
        return got
    same(got, idx.search(q, k, qd, ids=ids), tag + " vs gathered")
    if k <= 2048:  # (beyond it the library truncates the sorted row, which keeps other ties at the cut than faiss's heap)
        Do, Io = oracle.knn_subset(xv, qv[:n_oracle], k, ids, metric)
        same((got[0][:n_oracle], got[1][:n_oracle]), (Do, Io), tag + " vs oracle")
    return got


@pytest.mark.gpu
@pytest.mark.parametrize("d", [32, 100, 768])
@pytest.mark.parametrize("code", [0, 1, 2, 8])
def test_masked_search_equals_gathered_search_and_oracle(gpu, code, d):
    nv = gpu
    x, xv = store(nv, gauss(N, d, 30 + d), code)
    qf = gauss(NQ, d, 40 + d)
    qdtypes = {0: (0,), 1: (1,), 2: (2,), 8: (8, 0)}[code]  # an int8 store: int8 queries and float queries (its fp16 copy)
    for metric in (nv.METRIC_IP, nv.METRIC_L2):
        idx = nv.Index(x, code, metric)
        try:
            for qd in qdtypes:
                q, qv = store(nv, qf, qd)
                for mi, (name, mask) in enumerate(masks(N, d + code).items()):
                    for k in (KS[(mi + metric) % 5], KS[(mi + metric + 2) % 5]):
                        if k == 1000 and (d == 768 or name == "random 0.001"):
                            k = 100  # (the oracle over k = 1000 at d = 768 takes minutes; 0.001 selects ~70 rows)
                        tag = f"store={code} q={qd} d={d} metric={metric} k={k} mask={name}"
                        nv.stats_reset()
                        got = check_masked(nv, idx, xv, q, qv, qd, k, mask, metric, tag)
                        if name == "ones":
                            same(got, idx.search(q, k, qd), tag + " vs unmasked")
        finally:
            idx.close()


@pytest.mark.gpu
@pytest.mark.parametrize("metric", [0, 1])
def test_fp32_two_level_keeps_the_mask_for_deferred_queries(gpu, metric):
    """Near-duplicate rows: the bf16 first level of an fp32 store cannot separate them, so queries are deferred to the tf32
    level (and some on to the dense path), which must search under the same mask."""
    nv = gpu
    x, q = fl.make_data("neardup", N, NQ, 100, 7)
    idx = nv.Index(x, nv.F32, metric)
    try:
        for name, mask in list(masks(N, 5).items())[:6]:
            for k in (5, 12):
                nv.stats_reset()
                check_masked(nv, idx, x, q, q, nv.F32, k, mask, metric, f"two-level metric={metric} k={k} mask={name}")
                st = nv.stats()
                if name != "random 0.001":
                    assert st["second_level_queries"] > 0, (name, k, st)
    finally:
        idx.close()


@pytest.mark.gpu
@pytest.mark.parametrize("code", [0, 1])
def test_tie_windows_across_cleared_rows(gpu, code):
    """Grid data: scores are exact under any summation order and ties are abundant, so the tie window at rank k spans cleared
    rows; the dense path (k = 1000 on few selected rows) and the filter must both skip them."""
    nv = gpu
    n, d = 20_003, 32
    x, xv = store(nv, grid(n, d, 11), code)
    q, qv = store(nv, grid(300, d, 12), code)
    for metric in (nv.METRIC_IP, nv.METRIC_L2):
        idx = nv.Index(x, code, metric)
        try:
            for name, mask in masks(n, 9).items():
                for k in (1, 32, 100, 1000, 3000):  # 3000: the full-sort dense path
                    check_masked(nv, idx, xv, q, qv, code, k, mask, metric, f"grid store={code} metric={metric} k={k} mask={name}",
                                 n_oracle=4)
        finally:
            idx.close()


def masked_scores(mask):
    """filter_lists.scores with the cleared rows at -inf: check_lists then demands the discard bound of the selected rows only,
    and a cleared row on a list fails its accuracy check."""
    plain = fl.scores

    def f(Q, X, metric):
        S = plain(Q, X, metric)
        S[:, ~mask] = -np.inf
        return S
    return f


LISTS_SCRIPT = r"""
import json, sys
sys.path.insert(0, %r); sys.path.insert(0, %r + "/tests")
import numpy as np
import filter_lists as fl
import test_gpu_masked_search as t
from lotus_b200 import _native as nv
failures, plans = [], []
CASES = [  # (store, metric, n, d, nq, k, data, mask density): 4 to 7 query tiles over 32 corpus tiles or more, two-phase shapes
    (1, fl.IP, 8193, 96, 512, 10, "gauss", 0.5), (1, fl.L2, 8200, 96, 640, 10, "unnorm", 0.9), (1, fl.IP, 8449, 96, 700, 32, "cancel", 0.05),
    (1, fl.L2, 8192, 96, 801, 5, "grid", 0.5), (0, fl.IP, 8500, 64, 600, 10, "gauss", 0.5), (0, fl.L2, 8500, 40, 520, 32, "grid", 0.25),
    (1, fl.IP, 200_000, 32, 20_000, 10, "gauss", 0.5), (1, fl.L2, 9000, 48, 19_200, 32, "grid", 0.1),
]
for ci, (code, metric, n, d, nq, k, data, p) in enumerate(CASES):
    x, q = fl.make_data(data, n, nq, d, 3000 + ci)
    rng = np.random.default_rng(ci)
    mask = rng.random(n) < p
    mask[256 * 3: 256 * 5] = False  # two whole tiles cleared
    xs, xv = t.store(nv, x, code)
    qs, qv = t.store(nv, q, code)
    idx = nv.Index(xs, code, metric)
    tag = f"masked lists case {ci} [store={code} nq={nq} n={n} d={d} k={k} {data} p={p}]"
    try:
        for level in ((0, 1) if code == 0 else (0,)):
            res = idx.filter_lists(qs, k, code, level=level, mask=mask, plan_only=n * nq > 10 ** 9)  # (fp64 scores of 20k x 200k: the search only)
            plans.append({key: res[key] for key in ("n_splits", "units_whole", "cluster")})
            assert res["use_filter"], tag
            if "id" not in res:
                continue
            on = res["id"][res["id"] >= 0]
            assert mask[on].all(), f"{tag}: cleared rows on the lists"
            orig = fl.scores
            fl.scores = t.masked_scores(mask)
            try:
                with np.errstate(invalid="ignore"):
                    fl.check_lists(res, qv.astype("float64"), xv.astype("float64"), metric,
                                   exact=data == "grid" and not (code == 0 and level == 0), tag=tag + f" level {level}")
            finally:
                fl.scores = orig
        got = idx.search_masked(qs, k, code, mask)
        t.same(got, idx.search(qs, k, code, ids=np.flatnonzero(mask)), tag + " vs gathered")
        head = np.r_[0:128, nq - 128:nq]
        Do, Io = __import__("oracle").knn_subset(xv, qv[head], k, np.flatnonzero(mask), metric)
        t.same((got[0][head], got[1][head]), (Do, Io), tag + " vs oracle")
    except AssertionError as e:
        failures.append(str(e))
    finally:
        idx.close()
print(json.dumps({"failures": failures, "plans": plans}))
""" % (ROOT, ROOT)


@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["1", "0"])
def test_masked_lists_hold_the_certificate_premises_in_both_cta_modes(gpu, mode):
    """(a) every list entry within the margin of its exact score, (b) every SELECTED row off a list at most thr + eps,
    (c) no cleared row on any list; then the search itself against the gathered path and the oracle."""
    r = subprocess.run([sys.executable, "-c", LISTS_SCRIPT], capture_output=True, text=True, timeout=1500,
                       env=dict(os.environ, B2_FILTER_2CTA=mode))
    assert r.returncode == 0, r.stderr[-3000:]
    res = json.loads(r.stdout.strip().splitlines()[-1])
    assert not res["failures"], "\n".join(res["failures"])
    assert all(p["cluster"] == (4 if mode == "1" else 1) for p in res["plans"]), res["plans"]
    assert any(p["units_whole"] > 0 and p["n_splits"] > 1 for p in res["plans"]), "no two-phase shape ran"


@pytest.mark.gpu
@pytest.mark.parametrize("code", [0, 1, 2, 8])
def test_host_resident_masked_search_streams_the_corpus_once(gpu, code):
    """A small ring: several chunks, the last one re-streaming its predecessor's tail from a row that is not on a word
    boundary, and a subset larger than the ring. The result is the device-resident one; the rows cross the bus once."""
    nv = gpu
    n, d = 150_013, 64
    x, xv = store(nv, gauss(n, d, 50), code)
    rows = 20_224  # 79 tiles per slot
    ring = 2 * rows * ring_row_bytes(nv, d, code)
    plan = nv.stream_plan(n, d, code, ring)
    assert plan["n_chunks"] >= 5 and (n - plan["chunk_rows"]) % 32 != 0, plan
    qf = gauss(NQ, d, 51)
    for metric in (nv.METRIC_IP, nv.METRIC_L2):
        dev = nv.Index(x, code, metric)
        host = nv.Index(x, code, metric, residency="host", ring_bytes=ring)
        try:
            for qd in ((8, 0) if code == 8 else (code,)):
                q, qv = store(nv, qf, qd)
                for mi, (name, mask) in enumerate(masks(n, 60 + code).items()):
                    k = (5, 32, 100)[mi % 3]
                    if code == 0:
                        k = (5, 12, 100)[mi % 3]  # 5 and 12: the two-level search of an fp32 store
                    tag = f"host store={code} q={qd} metric={metric} k={k} mask={name}"
                    nv.stats_reset()
                    got = host.search_masked(q, k, qd, mask)
                    st = nv.stats()
                    assert host.last_filter_ms() > 0 and host.stream_times()["filter_ms"] > 0, tag
                    same(got, dev.search_masked(q, k, qd, mask), tag + " vs device")
                    levels = 1 + (st["second_level_queries"] > 0)
                    assert st["streamed_chunks"] == levels * plan["n_chunks"], (tag, st, plan)
                    per_level = [plan["n_chunks"] * plan["chunk_rows"] * d * e for e in ((2, 4) if code == 0 and k <= 24 else
                                                                                     (nv.storage_dtype(code).itemsize,))]
                    assert st["streamed_bytes"] == sum(per_level[:levels]), (tag, st, per_level)
                    if name in ("random 0.5", "three rows"):
                        assert mask.sum() * ring_row_bytes(nv, d, code) > ring or name == "three rows"
                        check_masked(nv, host, xv, q, qv, qd, k, mask, metric, tag)
        finally:
            host.close()
            dev.close()


@pytest.fixture
def stores(gpu, tmp_path):
    import lotus_b200 as lotus
    made = []

    def make(**kw):
        vs = lotus.B200VS(**kw)
        made.append(vs)
        lotus.settings.configure(rm=lotus.HashRM(dim=64), vs=vs, enable_cache=False)
        return vs
    yield make, tmp_path
    for vs in made:
        vs.close()
    lotus.settings.configure(rm=None, vs=None)


@pytest.mark.gpu
def test_operators_give_the_same_frames_under_every_subset_mode(stores, monkeypatch):
    import lotus_b200 as lotus
    from lotus_b200 import _native as nv
    make, tmp = stores
    frames = {}
    calls = {"masked": 0}
    orig = nv.Index.search_masked

    def counting(self, *a, **kw):
        calls["masked"] += 1
        return orig(self, *a, **kw)
    monkeypatch.setattr(nv.Index, "search_masked", counting)
    for mode in ("gather", "mask", "auto"):
        make(subset=mode)
        calls["masked"] = 0
        df = pd.DataFrame({"t": [f"doc {i}" for i in range(3000)]}).sem_index("t", str(tmp / f"s{mode}"))
        sub = df[df.index % 3 != 1]  # 2/3 of the rows, ascending
        small = df[df.index % 50 == 7]  # 2 %
        left = pd.DataFrame({"a": [f"left {i}" for i in range(200)]})
        frames[mode] = (sub.sem_search("t", "doc 1234", K=7, return_scores=True),
                        small.sem_search("t", ["doc 57", "doc 1007"], K=4, return_scores=True),
                        left.sem_sim_join(sub, "a", "t", K=5))
        # "auto" on a device-resident store with memory to spare gathers: there the gathered search is the faster one
        assert calls["masked"] == {"gather": 0, "mask": 3, "auto": 0}[mode], (mode, calls)
    for mode in ("mask", "auto"):
        for got, want in zip(frames[mode], frames["gather"]):
            for g, w in zip(*(f if isinstance(f, list) else [f] for f in (got, want))):  # (a list of queries: a list of frames)
                pd.testing.assert_frame_equal(g, w)
    # a shuffled (or repeating) ids takes the gathered path: its tie order is not the row order
    vs = make(subset="mask")
    x = grid(5000, 64, 3)
    vs.index(None, x, str(tmp / "g"))
    q = grid(20, 64, 4)
    ids = np.random.default_rng(0).permutation(5000)[:2500]
    calls["masked"] = 0
    r = vs(q, 10, ids=ids)
    assert calls["masked"] == 0
    Do, Io = oracle.knn_subset(x, q, 10, ids, oracle.IP)
    assert np.array_equal(np.asarray(r.indices), Io) and np.array_equal(bits(r.distances), bits(Do))
    r = vs(q, 10, ids=np.sort(ids))
    assert calls["masked"] == 1
    Do, Io = oracle.knn_subset(x, q, 10, np.sort(ids), oracle.IP)
    assert np.array_equal(np.asarray(r.indices), Io) and np.array_equal(bits(r.distances), bits(Do))
    m = np.zeros(5000, bool)
    m[ids] = True
    r2 = vs.search_masked(q, 10, m)
    assert np.array_equal(np.asarray(r2.indices), Io) and np.array_equal(bits(r2.distances), bits(Do))


@pytest.mark.gpu
def test_auto_masks_a_host_resident_subset_that_does_not_fit_the_ring(stores):
    make, tmp = stores
    x = gauss(40_000, 64, 8)
    ring = 2 * 2048 * 64 * 4
    vs = make(subset="auto", residency="host", ring_bytes=ring, dtype="f32")
    vs.index(None, x, str(tmp / "h"))
    ids = np.arange(0, 40_000, 5)  # a fifth of the rows: twice the ring
    assert vs._subset_by_mask(ids) and not vs._subset_by_mask(ids[:100])
    q = gauss(50, 64, 9)
    r = vs(q, 10, ids=ids)
    Do, Io = oracle.knn_subset(x, q, 10, ids, oracle.IP)
    assert np.array_equal(np.asarray(r.indices), Io) and np.array_equal(bits(r.distances), bits(Do))


@pytest.mark.gpu
def test_masked_search_over_several_devices(gpu, tmp_path):
    import lotus_b200 as lotus
    nv = gpu
    g = nv.device_count()
    if g < 2:
        pytest.skip(f"needs two GPUs or more ({g} visible)")
    x, q = gauss(50_021, 96, 0), gauss(300, 96, 1)
    for metric, om in ((lotus.METRIC_INNER_PRODUCT, oracle.IP), (lotus.METRIC_L2, oracle.L2)):
        vs = lotus.B200VS(metric=metric, dtype="f32", devices=list(range(g)), subset="mask")
        vs.index(None, x, str(tmp_path / f"m{metric}"))
        for name, mask in masks(len(x), 3).items():
            ids = np.flatnonzero(mask)
            if len(ids) == 0:
                continue
            r = vs(q, 10, ids=ids)
            Do, Io = oracle.knn_subset(x, q, 10, ids, om)
            assert np.array_equal(np.asarray(r.indices), Io) and np.array_equal(bits(r.distances), bits(Do)), name
        vs.close()
