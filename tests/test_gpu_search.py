"""Parity tests proper: the CUDA path, called through the C-ABI (ctypes -> libb2lotus.so), against the oracle on the
same seeded inputs — bit-exact top-k indices AND bit-exact fp32 scores (integer/index work: exact; floating point: the
canonical score is defined bit-for-bit, which is stricter than north_star's 1e-5 fp32 / 1e-2 bf16 tolerance)."""
import os

import numpy as np
import pytest

import oracle
from helpers import bits, gauss, grid

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(__file__), "golden")
FMAX = np.finfo(np.float32).max


def build(nv, x, dtype, metric):
    if dtype == "bf16":
        xb = nv.f32_to_bf16_bits(x)
        return nv.Index(xb, nv.BF16, metric), nv.bf16_bits_to_f32(xb)
    return nv.Index(x, nv.F32, metric), x


def qarg(nv, q, dtype):
    if dtype == "bf16":
        qb = nv.f32_to_bf16_bits(q)
        return qb, nv.BF16, nv.bf16_bits_to_f32(qb)
    return q, nv.F32, q


def check(nv, x, q, k, metric, dtype, ids=None, expect_filter=None):
    idx, xf = build(nv, x, dtype, metric)
    qa, qdt, qf = qarg(nv, q, dtype)
    nv.stats_reset()
    D, I = idx.search(qa, k, qdt, ids=ids)
    st = nv.stats()
    if ids is None:
        Do, Io = oracle.knn(xf, qf, k, metric)
    else:
        Do, Io = oracle.knn_subset(xf, qf, k, ids, metric)
    idx.close()
    assert np.array_equal(I, Io), f"top-k indices differ in {(I != Io).any(axis=1).sum()} of {len(I)} rows"
    assert np.array_equal(bits(D), bits(Do)), "scores are not bit-identical to the canonical oracle score"
    if expect_filter is True:
        assert st["filter_launches"] >= 1, "the wgmma filter did not run"
    if expect_filter is False:
        assert st["filter_launches"] == 0
    return st


@pytest.mark.parametrize("metric", [0, 1])
@pytest.mark.parametrize("k", [1, 2, 5, 17, 64, 400])
def test_dense_path_tie_rules_on_grid(gpu, metric, k):
    check(gpu, grid(300, 16, 0), grid(40, 16, 1), k, metric, "f32", expect_filter=False)


@pytest.mark.parametrize("dtype", ["bf16", "f32"])
@pytest.mark.parametrize("metric", [0, 1])
@pytest.mark.parametrize("k", [1, 10, 32, 64])
def test_filter_path_gaussian(gpu, dtype, metric, k):
    st = check(gpu, gauss(6000, 96, 2), gauss(300, 96, 3), k, metric, dtype, expect_filter=True)
    assert st["fallback_queries"] <= 3  # the certificate should cover continuous data


@pytest.mark.parametrize("dtype,d", [("bf16", 768), ("f32", 768), ("bf16", 100), ("f32", 30), ("bf16", 384)])
def test_filter_path_dims(gpu, dtype, d):
    st = check(gpu, gauss(9001, d, 4), gauss(257, d, 5), 10, 0, dtype, expect_filter=True)
    assert st["fallback_queries"] <= 3, st  # measured 0 of 257 for every (dtype, d) (H100 80GB HBM3, 400 W)


@pytest.mark.parametrize("metric", [0, 1])
def test_filter_path_tie_heavy_takes_certified_fallback(gpu, metric):
    """Thousands of rows share each score level (coordinates in {-1/2, 0, 1/2}, d = 4: nine possible values), so the
    K-th and the KP-th best scores coincide: the certificate cannot hold, the dense exact path must take over and
    reproduce faiss's heap rule (which rows of the tied level survive, and in which order)."""
    rng = np.random.default_rng(6)
    x = (rng.integers(-1, 2, size=(5000, 4)) / 2).astype(np.float32)
    q = (rng.integers(-1, 2, size=(64, 4)) / 2).astype(np.float32)
    st = check(gpu, x, q, 10, metric, "f32", expect_filter=True)
    assert st["fallback_queries"] > 0
    check(gpu, grid(5000, 8, 6), grid(64, 8, 7), 10, metric, "bf16", expect_filter=True)


def test_unnormalised_and_duplicate_rows(gpu):
    x = gauss(4000, 64, 8, normalize=False) * 3
    x[100] = x[7]
    x[2500] = x[7]
    x[3999] = x[0]
    q = np.concatenate([x[[7, 0]], gauss(30, 64, 9, normalize=False)])
    for metric in (0, 1):
        for dtype in ("f32", "bf16"):
            st = check(gpu, x, q, 5, metric, dtype, expect_filter=True)
            assert st["fallback_queries"] <= 2, st  # measured 0 of 32 in all four runs (H100 80GB HBM3, 400 W)


def test_ids_subset_semantics(gpu):
    x, q = gauss(6000, 64, 10), gauss(120, 64, 11)
    rng = np.random.default_rng(5)
    check(gpu, x, q, 8, 0, "bf16", ids=rng.permutation(6000)[:2500])       # permuted subset through the filter
    check(gpu, x, q, 8, 0, "f32", ids=np.arange(6000))                      # identity: same as no ids
    check(gpu, x, q, 8, 1, "f32", ids=np.array([5, 7, 7, 100, 2999]))       # duplicates, K > len(ids): -1 padding
    idx, _ = build(gpu, x, "f32", 0)
    D, I = idx.search(q, 3, gpu.F32, ids=np.zeros(0, np.int64))
    assert (I == -1).all() and (D == -FMAX).all()
    with pytest.raises(gpu.NativeError) as e:
        idx.search(q, 3, gpu.F32, ids=np.array([1, 6000]))
    assert e.value.code == gpu.ERANGE
    idx.close()


def test_edge_shapes(gpu):
    x, q = gauss(700, 32, 12), gauss(3, 32, 13)
    idx, xf = build(gpu, x, "f32", 0)
    D, I = idx.search(np.zeros((0, 32), np.float32), 4)
    assert D.shape == (0, 4)
    D, I = idx.search(q, 900)  # K > N: padded with -1 / -FLT_MAX like faiss
    Do, Io = oracle.knn(x, q, 900)
    assert np.array_equal(I, Io) and np.array_equal(bits(D), bits(Do))
    with pytest.raises(gpu.NativeError):
        idx.search(q, 0)
    with pytest.raises(gpu.NativeError):
        idx.search(q[:1], gpu.lib().b2_max_k() + 1)
    idx.close()
    empty = gpu.Index(np.zeros((0, 32), np.float32), gpu.F32, 1)
    D, I = empty.search(q, 2)
    assert (I == -1).all() and (D == FMAX).all()
    empty.close()


def test_golden_vectors_through_the_cuda_path(gpu):
    g = np.load(os.path.join(GOLD, "knn_golden.npz"))
    for name in ("grid", "gauss"):
        x, q = g[f"{name}_x"], g[f"{name}_q"]
        for mname, metric in (("ip", 0), ("l2", 1)):
            idx = gpu.Index(x, gpu.F32, metric)
            for k in (1, 5, 32):
                D, I = idx.search(q, k)
                assert np.array_equal(I, g[f"{name}_{mname}_k{k}_I"])
                assert np.array_equal(bits(D), bits(g[f"{name}_{mname}_k{k}_D"]))
            idx.close()


def test_gather_rows(gpu):
    x = gauss(1000, 40, 14)
    for dtype in ("f32", "bf16"):
        idx, xf = build(gpu, x, dtype, 0)
        ids = np.array([999, 0, 5, 5, 123])
        out = idx.gather(ids)
        got = gpu.bf16_bits_to_f32(out) if dtype == "bf16" else out
        assert np.array_equal(got, xf[ids])
        with pytest.raises(gpu.NativeError):
            idx.gather(np.array([1000]))
        idx.close()


def test_large_scale_properties(gpu):
    """BASELINE-scale shapes are too slow for the CPU oracle; check size-independent properties instead:
    rows sorted best-first, ids valid and unique, scores equal the canonical score of the reported id, a planted
    duplicate of each query is its own top-1, and a sample of rows equals the oracle exactly."""
    n, d, nq, k = 300_000, 768, 8192, 32
    x = gauss(n, d, 15)
    xb = gpu.f32_to_bf16_bits(x)
    xf = gpu.bf16_bits_to_f32(xb)
    q_ids = np.random.default_rng(16).choice(n, nq, replace=False)
    qb = xb[q_ids]
    idx = gpu.Index(xb, gpu.BF16, 0)
    gpu.stats_reset()
    D, I = idx.search(qb, k, gpu.BF16)
    st = gpu.stats()
    idx.close()
    assert st["filter_launches"] == 1 and st["fallback_queries"] <= 8
    assert (np.diff(D, axis=1) <= 0).all() and (I >= 0).all() and (I < n).all()
    assert all(len(set(r)) == k for r in I[:512].tolist())
    assert np.array_equal(I[:, 0], q_ids)  # <x,x> is the largest product with x for normalised rows
    rows = np.random.default_rng(17).choice(nq, 24, replace=False)
    Do, Io = oracle.knn(xf, xf[q_ids[rows]], k, 0)
    assert np.array_equal(I[rows], Io) and np.array_equal(bits(D[rows]), bits(Do))


def test_filter_error_stays_inside_the_certified_margin(gpu):
    """The certificate assumes |tensor-core score - exact score| <= rel_eps * |q| * |x|; measure the real gap through
    a K=1 vs exact comparison on hard (near-tie) data: if the margin were too small, uncertified wrong answers would
    show up here as index mismatches without a fallback."""
    base = gauss(1, 256, 18)
    x = base + 1e-3 * gauss(4096, 256, 19, normalize=False)  # all rows nearly identical: scores differ by ~1e-6
    q = base + 1e-3 * gauss(64, 256, 20, normalize=False)
    for dtype in ("f32", "bf16"):
        check(gpu, x.astype(np.float32), q.astype(np.float32), 4, 0, dtype, expect_filter=True)
        check(gpu, x.astype(np.float32), q.astype(np.float32), 4, 1, dtype, expect_filter=True)


@pytest.mark.parametrize("metric", [0, 1])
def test_large_k_full_sort_path(gpu, metric):
    """k beyond the radix-select limit (the cascade callers' K = len(df)): whole-row sort in faiss heap order."""
    x, q = gauss(5000, 48, 30), gauss(6, 48, 31)
    x[17] = x[4000]  # an exact duplicate pair: tie order must follow the heap convention
    idx = gpu.Index(x, gpu.F32, metric)
    S = oracle.scores(x, q, metric)
    for k in (3000, 5000, 6000):
        D, I = idx.search(q, k)
        for r in range(len(q)):
            ids = np.arange(5000)
            order = np.lexsort((-ids, -S[r].astype(np.float64))) if metric == 0 else np.lexsort((ids, S[r].astype(np.float64)))
            m = min(k, 5000)
            assert np.array_equal(I[r, :m], order[:m])
            assert np.array_equal(bits(D[r, :m]), bits(S[r][order[:m]]))
            assert (I[r, m:] == -1).all() and (D[r, m:] == (-FMAX if metric == 0 else FMAX)).all()
    idx.close()


# ---- k > 64: several corpus splits share the candidate lists; K = len(df): full sort (SURVEY §8f-3 cascade callers) ---------
@pytest.mark.parametrize("dtype", ["bf16", "f32"])
@pytest.mark.parametrize("metric", [0, 1])
@pytest.mark.parametrize("k", [65, 128, 1000])
def test_large_k_goes_through_the_filter(gpu, dtype, metric, k):
    st = check(gpu, gauss(30_000, 64, 60 + k), gauss(200, 64, 61 + k), k, metric, dtype, expect_filter=True)
    # the certificate should cover continuous data while k + 32 survivors leave room (k = 1000 keeps 1024: with the tf32 operand
    # error many rows straddle the last 24 ranks of a 30k-row corpus and those queries take the dense path — still exact)
    if k <= 128:
        assert st["fallback_queries"] <= 20, st


def test_large_k_on_a_corpus_sorted_by_topic(gpu):
    """Rows of one topic are contiguous, so a query's best k all sit in ONE corpus split and overflow its candidate lists:
    the certificate must notice (bound >= k-th exact score) and the dense path must answer — still exact."""
    rng = np.random.default_rng(70)
    centers = gauss(20, 48, 71)
    lab = np.sort(rng.integers(0, 20, 20_000))
    x = centers[lab] + 0.05 * gauss(20_000, 48, 72, normalize=False)
    x = (x / np.linalg.norm(x, axis=1, keepdims=True)).astype(np.float32)
    q = (centers[rng.integers(0, 20, 50)] + 0.05 * gauss(50, 48, 73, normalize=False)).astype(np.float32)
    st = check(gpu, x, q, 200, 0, "bf16", expect_filter=True)
    assert st["fallback_queries"] > 0


@pytest.mark.parametrize("metric", [0, 1])
def test_k_equal_to_the_index_size_returns_every_row_sorted(gpu, metric):
    # sem_filter / sem_join cascade: vs(query, K=len(df)) -> all rows best first (lotus/sem_ops/sem_filter.py:486-497)
    x, q = gauss(5000, 32, 80), gauss(3, 32, 81)
    check(gpu, x, q, 5000, metric, "f32", expect_filter=False)
    check(gpu, x, q[:1], 7000, metric, "bf16", expect_filter=False)      # K > n: padded with -1
    check(gpu, grid(3000, 6, 82), grid(9, 6, 83), 3000, metric, "f32", expect_filter=False)   # ties: (score, id) heap order


@pytest.mark.parametrize("metric", [0, 1])
@pytest.mark.parametrize("dtype", ["bf16", "f32"])
def test_staged_sharded_search_emulated_in_one_process(gpu, metric, dtype):
    """The two-stage row-sharded search (stage 1: filter + lower bound of the ceil(k/G) best local candidates; all-reduce MIN;
    stage 2: finalize with that hint, packed lists; k-way merge) with G = 3 shards held by ONE process on one device: the merged
    result must equal the single-index oracle, and the hint must actually prune (fewer exact re-scores than the plain search)."""
    import torch
    dev = torch.device("cuda", 0)
    x, q = gauss(24_000, 96, 200 + metric), gauss(6000, 96, 201)   # enough queries that the filter needs few corpus splits
    k, G = 32, 3
    if dtype == "bf16":
        xb, qb = gpu.f32_to_bf16_bits(x), gpu.f32_to_bf16_bits(q)
        xf, qf, code = gpu.bf16_bits_to_f32(xb), gpu.bf16_bits_to_f32(qb), gpu.BF16
        q_dev = torch.from_numpy(qb.view(np.int16)).to(dev)
        parts = [xb[g * 8000:(g + 1) * 8000] for g in range(G)]
    else:
        xf, qf, code = x, q, gpu.F32
        q_dev = torch.from_numpy(q).to(dev)
        parts = [x[g * 8000:(g + 1) * 8000] for g in range(G)]
    shards = [gpu.Index(np.ascontiguousarray(p), code, metric) for p in parts]
    st = torch.cuda.current_stream().cuda_stream
    lowers = [torch.empty(len(q), dtype=torch.float32, device=dev) for _ in range(G)]
    j = -(-k // G)
    for s, lo in zip(shards, lowers):
        s.search_stage1_dev(q_dev.data_ptr(), len(q), k, code, j, lo.data_ptr(), stream=st)
    hint = torch.stack(lowers).min(dim=0).values.contiguous()          # what all-reduce(MIN) delivers on every rank
    packed = torch.empty((G, len(q), k), dtype=torch.int64, device=dev)
    gpu.stats_reset()
    for g, s in enumerate(shards):
        s.search_stage2_packed_dev(hint.data_ptr(), packed[g].data_ptr(), stream=st)
    out_s = torch.empty((len(q), k), dtype=torch.float32, device=dev)
    out_i = torch.empty((len(q), k), dtype=torch.int64, device=dev)
    gpu.merge_topk_packed_dev(packed.data_ptr(), np.arange(G) * 8000, G, len(q), k, metric, 0, out_s.data_ptr(), out_i.data_ptr(), stream=st)
    Do, Io = oracle.knn(xf, qf, k, metric)
    assert np.array_equal(out_i.cpu().numpy(), Io), f"{(out_i.cpu().numpy() != Io).any(axis=1).sum()} rows differ"
    assert np.array_equal(bits(out_s.cpu().numpy()), bits(Do))
    # every shard reported only rows that can matter: far fewer than k valid entries per query on average
    # (fp32 shards of this size take the two-level bf16-first search, which the staged path leaves to the plain search: -inf bounds)
    staged = bool(torch.isfinite(hint).any().item())
    assert staged or dtype == "f32"
    valid = (packed.cpu().numpy().astype(np.uint64) & np.uint64(0xffffffff)) != np.uint64(0xffffffff)
    if staged:
        assert valid.sum(axis=2).mean() < 0.75 * k, valid.sum(axis=2).mean()
    # hint = -inf (unknown) must give the plain per-shard top-k back
    for s, lo in zip(shards, lowers):
        s.search_stage1_dev(q_dev.data_ptr(), len(q), k, code, j, lo.data_ptr(), stream=st)
    none = torch.full((len(q),), float("-inf"), dtype=torch.float32, device=dev)
    shards[0].search_stage2_packed_dev(none.data_ptr(), packed[0].data_ptr(), stream=st)
    D0, I0 = oracle.knn(xf[:8000], qf, k, metric)
    got = packed[0].cpu().numpy().astype(np.uint64)
    assert np.array_equal((got & np.uint64(0xffffffff)).astype(np.int64), I0)
    for s in shards:
        s.close()


@pytest.mark.parametrize("metric,dtype,k", [(0, "bf16", 10), (1, "bf16", 32), (0, "f32", 5)])
def test_two_phase_schedule_whole_waves_and_split_remainder(gpu, metric, dtype, k):
    """Batches of at least one query unit per worker (>= 74 CTA pairs x 256 queries) take the two-phase schedule: whole waves of
    (one unit per worker x the whole corpus) and a remainder cut into corpus splits whose extra candidate lists are empty for the
    whole-wave units. 40,000 queries = 157 units = 2 whole waves + 9 leftover units: EVERY query is checked against the oracle,
    so both phases (and the unit that is half empty at the end of the batch) are covered."""
    x, q = gauss(20_000, 64, 300 + k), gauss(40_000, 64, 301 + k)
    st = check(gpu, x, q, k, metric, dtype, expect_filter=True)
    assert st["fallback_queries"] <= 40, st
