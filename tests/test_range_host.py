"""Range search without a GPU: the oracle's definition against an fp64 numpy restatement, and the host-side logic of the
Python layers (the ERANGE retry of `_native.Index.range_search`, the shard combination of `MultiDeviceIndex.range_search`,
the errors of `B200VS.range_search`) against fake native layers."""
import ctypes

import numpy as np
import pytest

import oracle
from helpers import grid
from range_oracle import range_search as oracle_range


def numpy_range(x, q, radius, metric, ids=None):
    """fp64 restatement on grid data (every product and partial sum is exact, so fp64 = canonical)."""
    x64 = np.asarray(x, np.float64) if ids is None else np.asarray(x, np.float64)[np.asarray(ids, np.int64)]
    q64 = np.asarray(q, np.float64)
    S = q64 @ x64.T if metric == oracle.IP else ((q64[:, None, :] - x64[None, :, :]) ** 2).sum(-1)
    lims, D, I = [0], [], []
    for i in range(len(q64)):
        pos = [j for j in range(x64.shape[0]) if (S[i, j] > radius if metric == oracle.IP else S[i, j] < radius)]
        lims.append(lims[-1] + len(pos))
        D += [S[i, j] for j in pos]
        I += [j if ids is None else int(ids[j]) for j in pos]
    return np.array(lims, np.int64), np.array(D, np.float32), np.array(I, np.int64)


def equal(a, b):
    return all(np.array_equal(u, v) for u, v in zip(a, b))


@pytest.mark.parametrize("metric", [oracle.IP, oracle.L2])
def test_oracle_matches_fp64_and_is_strict(metric):
    x, q = grid(300, 16, 1), grid(7, 16, 2)
    S = q.astype(np.float64) @ x.T.astype(np.float64) if metric == oracle.IP else \
        ((q[:, None, :].astype(np.float64) - x[None]) ** 2).sum(-1)
    r = float(np.sort(S[0])[::-1][20] if metric == oracle.IP else np.sort(S[0])[20])
    at, past = oracle_range(x, q, r, metric), oracle_range(x, q, float(np.nextafter(np.float32(r), np.float32(
        -np.inf if metric == oracle.IP else np.inf))), metric)
    assert equal(at, numpy_range(x, q, r, metric))
    assert past[0][-1] - at[0][-1] == int((S == r).sum()) > 0  # rows exactly at the radius are excluded
    for i in range(7):
        assert (np.diff(at[2][at[0][i]:at[0][i + 1]]) > 0).all()  # ascending row id


def test_oracle_empty_results_and_ids_order():
    x, q = grid(200, 8, 3), grid(5, 8, 4)
    none = oracle_range(x, q, 1e9, oracle.IP)
    assert np.array_equal(none[0], np.zeros(6, np.int64)) and len(none[1]) == len(none[2]) == 0
    empty_q = oracle_range(x, q[:0], 0.0, oracle.IP)
    assert np.array_equal(empty_q[0], [0]) and len(empty_q[2]) == 0
    ids = np.array([150, 3, 77, 3, 199, 0, 150], np.int64)
    for metric, r in [(oracle.IP, 0.0), (oracle.L2, 0.05)]:
        got = oracle_range(x, q, r, metric, ids=ids)
        assert equal(got, numpy_range(x, q, r, metric, ids=ids))
        for i in range(5):  # order of positions in ids; a duplicated id appears once per occurrence
            row = got[2][got[0][i]:got[0][i + 1]]
            pos = [p for p in range(len(ids)) if ids[p] in set(row.tolist())]
            assert row.tolist() == ids[pos].tolist()
    assert oracle_range(x, q, 0.0, oracle.IP, ids=np.empty(0, np.int64))[0].tolist() == [0] * 6


class FakeLib:
    """b2_index_range_search over the oracle, honouring the cap / ERANGE convention of the C-ABI."""

    def __init__(self, nv, x, metric):
        self.nv, self.x, self.metric, self.calls = nv, x, metric, []

    def b2_last_error(self):
        return b"fake error"

    def b2_index_range_search(self, h, q, nq, q_dtype, radius, ids, n_ids, lims, out_d, out_i, cap, n_results):
        def arr(p, ct, count):
            return np.ctypeslib.as_array(ctypes.cast(p, ctypes.POINTER(ct)), (count,)) if count else np.empty(0)
        qa = arr(q, ctypes.c_float, nq * self.x.shape[1]).reshape(nq, -1)
        ida = None if ids is None else arr(ids, ctypes.c_int64, n_ids)
        L, D, I = oracle_range(self.x, qa, radius, self.metric, ids=ida)
        self.calls.append(cap)
        arr(lims, ctypes.c_int64, nq + 1)[:] = L
        n_results._obj.value = int(L[-1])
        if L[-1] > cap:
            return self.nv.ERANGE
        arr(out_d, ctypes.c_float, L[-1])[:] = D
        arr(out_i, ctypes.c_int64, L[-1])[:] = I
        return self.nv.OK


def fake_index(nv, x, metric, monkeypatch):
    fake = FakeLib(nv, x, metric)
    monkeypatch.setattr(nv, "lib", lambda: fake)
    idx = object.__new__(nv.Index)
    idx._h = ctypes.c_void_p()
    idx.n, idx.d, idx.dtype, idx.metric, idx.device = x.shape[0], x.shape[1], nv.F32, metric, 0
    return idx, fake


def test_index_range_search_retries_once_with_the_exact_size(nv, monkeypatch):
    x, q = grid(500, 16, 5), grid(9, 16, 6)
    idx, fake = fake_index(nv, x, oracle.IP, monkeypatch)
    want = oracle_range(x, q, -0.05, oracle.IP)
    got = idx.range_search(q, -0.05, cap=10)
    assert equal(got, want) and fake.calls == [10, int(want[0][-1])]
    fake.calls.clear()
    assert equal(idx.range_search(q, -0.05), want) and len(fake.calls) == 1
    ids = np.array([5, 4, 4, 499, 0], np.int64)
    assert equal(idx.range_search(q, 0.0, ids=ids), oracle_range(x, q, 0.0, oracle.IP, ids=ids))
    with pytest.raises(ValueError, match="dimension"):
        idx.range_search(q[:, :8], 0.0)


class FakeShard:
    def __init__(self, x, metric):
        self.x, self.metric = x, metric

    def range_search(self, q, radius, q_dtype=0, ids=None):
        return oracle_range(self.x, q, radius, self.metric, ids=ids)


@pytest.mark.parametrize("metric", [oracle.IP, oracle.L2])
def test_multi_device_combination(nv, metric):
    from lotus_b200.distributed import shard_bounds
    from lotus_b200.vs import MultiDeviceIndex
    from concurrent.futures import ThreadPoolExecutor
    x, q = grid(1000, 12, 7), grid(6, 12, 8)
    r = 0.02 if metric == oracle.IP else 0.3
    md = object.__new__(MultiDeviceIndex)
    md.n, md.d, md.metric = x.shape[0], x.shape[1], metric
    md.bounds = [shard_bounds(md.n, 3, g) for g in range(3)]
    md.shards = [FakeShard(x[lo:hi], metric) for lo, hi in md.bounds]
    md.pool = ThreadPoolExecutor(3)
    rng = np.random.default_rng(0)
    assert equal(md.range_search(q, r), oracle_range(x, q, r, metric))
    for ids in (np.sort(rng.choice(1000, 300, replace=False)), rng.choice(1000, 300, replace=False),
                rng.integers(0, 1000, 400), np.empty(0, np.int64)):
        assert equal(md.range_search(q, r, ids=ids), oracle_range(x, q, r, metric, ids=ids))
    with pytest.raises(nv.NativeError):
        md.range_search(q, r, ids=np.array([1000]))
    md.pool.shutdown()


def test_b200vs_range_search_errors(nv):
    from lotus_b200.vs import B200VS
    vs = B200VS()
    with pytest.raises(ValueError, match="Index not loaded"):
        vs.range_search(np.zeros((1, 8), np.float32), 0.5)

    class Refusing:
        d, dtype = 8, nv.F32

        def range_search(self, *a, **k):
            raise nv.NativeError(nv.ERANGE, "ids contains a position outside [0, 4)")
    vs.b2_index, vs.index_dir = Refusing(), "/nonexistent"
    with pytest.raises(ValueError, match="outside"):
        vs.range_search(np.zeros((2, 8), np.float32), 0.5, ids=[9])
    with pytest.raises(ValueError, match="dimension"):
        vs.range_search(np.zeros((2, 4), np.float32), 0.5)
