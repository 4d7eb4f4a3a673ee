"""The pandas operators end to end on the H100 (B200VS through the C-ABI) against oracle-derived expectations, plus
the dedup / k-means / merge entry points."""
import os

import numpy as np
import pandas as pd
import pytest

import lotus_b200 as lotus
import oracle
from helpers import bits, gauss

pytestmark = pytest.mark.gpu


@pytest.fixture
def env(gpu, tmp_path):
    rm = lotus.HashRM(dim=64)
    vs = lotus.B200VS()
    lotus.settings.configure(rm=rm, vs=vs, enable_cache=False)
    yield rm, vs, tmp_path
    vs.close()
    lotus.settings.configure(rm=None, vs=None)


def test_vs_roundtrip_and_faiss_dir_compat(env):
    rm, vs, tmp = env
    x = gauss(2000, 64, 0)
    vs.index(pd.Series(["d"] * 2000), x, str(tmp / "i"))
    out = vs(x[:5], 3)
    Do, Io = oracle.knn(x, x[:5], 3)
    assert np.array_equal(np.asarray(out.indices), Io) and np.array_equal(bits(out.distances), bits(Do))
    assert np.array_equal(vs.get_vectors_from_index(str(tmp / "i"), [3, 1]), x[[3, 1]])
    vs2 = lotus.B200VS()           # a fresh store loads the directory (as FaissVS.load_index would)
    vs2.load_index(str(tmp / "i"))
    out2 = vs2(x[:5], 3, ids=list(range(0, 2000, 2)))
    Ds, Is = oracle.knn_subset(x, x[:5], 3, np.arange(0, 2000, 2))
    assert np.array_equal(np.asarray(out2.indices), Is) and np.array_equal(bits(out2.distances), bits(Ds))
    vs2.close()
    with pytest.raises(ValueError, match="Index not loaded"):
        lotus.B200VS()(x[:1], 1)
    with pytest.raises(ValueError):
        lotus.B200VS(factory_string="IVF64,Flat")


def test_sem_sim_join_on_gpu_matches_oracle_join(env):
    rm, vs, tmp = env
    left = pd.DataFrame({"a": [f"left {i}" for i in range(300)]})
    right = pd.DataFrame({"b": [f"right {i}" for i in range(1500)]}).sem_index("b", str(tmp / "r"))
    got = left.sem_sim_join(right, "a", "b", K=5)
    D, I = oracle.knn(rm(right["b"].tolist()), rm(left["a"].tolist()), 5)
    assert len(got) == 1500 and list(got.columns) == ["a", "_scores", "b"]
    assert got["b"].tolist() == [f"right {i}" for i in I.reshape(-1)]
    assert np.array_equal(bits(got["_scores"].to_numpy(np.float32)), bits(D.reshape(-1)))
    assert list(got.index) == np.repeat(np.arange(300), 5).tolist()
    # indexed left column: query vectors come from the left index (sem_sim_join.py:109-119)
    left.sem_index("a", str(tmp / "l"))
    got2 = left.sem_sim_join(right, "a", "b", K=5)
    pd.testing.assert_frame_equal(got, got2)


def test_sem_search_on_gpu(env):
    rm, vs, tmp = env
    df = pd.DataFrame({"t": [f"doc {i}" for i in range(3000)]}).sem_index("t", str(tmp / "s"))
    out = df.sem_search("t", "doc 1234", K=7, return_scores=True)
    D, I = oracle.knn(rm(df["t"].tolist()), rm(["doc 1234"]), 7)
    assert list(out.index) == I[0].tolist() and out.index[0] == 1234
    assert np.array_equal(bits(out["vec_scores_sim_score"].to_numpy(np.float32)), bits(D[0]))
    sub = df[df.index % 7 == 3]
    out = sub.sem_search("t", "doc 1234", K=4)
    Ds, Is = oracle.knn_subset(rm(df["t"].tolist()), rm(["doc 1234"]), 4, np.asarray(sub.index))
    assert list(out.index) == Is[0].tolist()


def test_baseline_config0_sem_sim_join_two_1k_frames_384d_fp32_k5(env):
    """BASELINE.json configs[0] at its stated shape: sem_sim_join on two 1k-row DataFrames, precomputed 384-d fp32 embeddings,
    K=5 — the GPU operator against the oracle-backed join (indices exact, scores bit-exact), both frames indexed."""
    _, vs, tmp = env
    table = {}
    xl, xr = gauss(1000, 384, 90), gauss(1000, 384, 91)
    for i in range(1000):
        table[f"left {i}"], table[f"right {i}"] = xl[i], xr[i]
    lotus.settings.configure(rm=lotus.TableRM(table))
    left = pd.DataFrame({"a": [f"left {i}" for i in range(1000)]}).sem_index("a", str(tmp / "c0l"))
    right = pd.DataFrame({"b": [f"right {i}" for i in range(1000)]}).sem_index("b", str(tmp / "c0r"))
    got = left.sem_sim_join(right, "a", "b", K=5)
    D, I = oracle.knn(xr, xl, 5)
    assert len(got) == 5000 and list(got.columns) == ["a", "_scores", "b"]
    assert got["b"].tolist() == [f"right {i}" for i in I.reshape(-1)]
    assert np.array_equal(bits(got["_scores"].to_numpy(np.float32)), bits(D.reshape(-1)))
    assert list(got.index) == np.repeat(np.arange(1000), 5).tolist()
    many = right.sem_search("b", ["left 3", "left 4"], K=5, return_scores=True)   # multi-query search, one device call
    assert [list(f.index) for f in many] == [I[3].tolist(), I[4].tolist()]


def planted(n, d, seed, frac=0.05):
    x = gauss(n, d, seed)
    rng = np.random.default_rng(seed + 1)
    src = rng.choice(n, int(n * frac), replace=False)
    dst = rng.choice(n, int(n * frac), replace=False)
    x[dst] = x[src] + 0.05 * gauss(len(src), d, seed + 2, normalize=False) / np.sqrt(d) * 3
    x /= np.linalg.norm(x, axis=1, keepdims=True)
    return x


@pytest.mark.parametrize("dtype", ["f32", "bf16"])
def test_threshold_pairs_equal_the_exact_relation(gpu, dtype):
    x = planted(3000, 96, 30)
    if dtype == "bf16":
        xb = gpu.f32_to_bf16_bits(x)
        idx, xf = gpu.Index(xb, gpu.BF16, 0), gpu.bf16_bits_to_f32(xb)
    else:
        idx, xf = gpu.Index(x, gpu.F32, 0), x
    pi, pj = idx.threshold_pairs(0.9)
    oi, oj, cnt = oracle.threshold_pairs(xf, 0.9)
    assert cnt > 20 and np.array_equal(pi, oi) and np.array_equal(pj, oj)
    # sharded over 3 "ranks": the union of the parts is the same relation
    # (query tiles are dealt in groups; B2_PAIR_GROUP=4 makes the 24 tiles of this matrix span 6 groups, default: 1 group)
    for group in ("4", "5", None):
        if group is None:
            os.environ.pop("B2_PAIR_GROUP", None)
        else:
            os.environ["B2_PAIR_GROUP"] = group
        try:
            parts = [idx.threshold_pairs(0.9, part=p, nparts=3) for p in range(3)]
            for p, (a, _) in enumerate(parts):
                assert (gpu.pair_owner(a, 3) == p).all()
            if group is not None:
                assert all(len(a) for a, _ in parts)
        finally:
            os.environ.pop("B2_PAIR_GROUP", None)
        allp = sorted(zip(np.concatenate([p[0] for p in parts]).tolist(), np.concatenate([p[1] for p in parts]).tolist()))
        assert allp == list(zip(oi.tolist(), oj.tolist()))
    lab = gpu.connected_components(len(x), pi, pj)
    assert np.array_equal(lab, oracle.connected_components(len(x), oi, oj))
    idx.close()


def test_sem_dedup_partition_parity(env):
    # mirrors .github/tests/rm_tests.py:131-149 (test_dedup) with table embeddings standing in for e5-small
    rm, vs, tmp = env
    texts = ["Probability and Random Processes", "Probability and Markov Chains", "Harry Potter", "Harry James Potter"]
    e = gauss(2, 64, 40)
    emb = {texts[0]: e[0], texts[1]: e[0] * 0.97 + e[1] * 0.03, texts[2]: e[1], texts[3]: e[1] * 0.98 + e[0] * 0.02}
    emb = {k: (v / np.linalg.norm(v)).astype(np.float32) for k, v in emb.items()}
    lotus.settings.configure(rm=lotus.TableRM(emb))
    df = pd.DataFrame({"Text": texts}).sem_index("Text", str(tmp / "d")).sem_dedup("Text", threshold=0.85)
    kept = sorted(df["Text"].tolist())
    assert len(kept) == 2 and "Harry" in kept[0] and "Probability" in kept[1]
    # value semantics (sem_dedup.py:47,87-91): rows with IDENTICAL text are never paired with each other and survive or
    # fall together; the representative is the value that appears first
    lotus.settings.configure(rm=lotus.HashRM(dim=64))
    vals = [f"v{i % 40}" for i in range(100)]
    df = pd.DataFrame({"Text": vals}).sem_index("Text", str(tmp / "e"))
    out = df.sem_dedup("Text", threshold=0.5)
    x = lotus.HashRM(dim=64)(vals)
    oi, oj, _ = oracle.threshold_pairs(x, 0.5)
    codes, uniq = pd.factorize(pd.Series(vals))
    keep_edges = codes[oi] != codes[oj]
    lab = oracle.connected_components(len(uniq), codes[oi][keep_edges], codes[oj][keep_edges])
    removed = set(uniq[np.nonzero(lab != np.arange(len(uniq)))[0]])
    assert out["Text"].tolist() == [v for v in vals if v not in removed]


@pytest.mark.parametrize("dtype", ["f32", "bf16"])
def test_kmeans_matches_the_faiss_restatement(gpu, dtype):
    rng = np.random.default_rng(50)
    centers = gauss(8, 48, 51) * 4
    x = (centers[rng.integers(0, 8, 3000)] + gauss(3000, 48, 52, normalize=False)).astype(np.float32)
    if dtype == "bf16":
        xb = gpu.f32_to_bf16_bits(x)
        idx, xf = gpu.Index(xb, gpu.BF16, 1), gpu.bf16_bits_to_f32(xb)
    else:
        idx, xf = gpu.Index(x, gpu.F32, 1), x
    a, c, obj = idx.kmeans(8, niter=6)
    ao, co, oo = oracle.kmeans(xf, 8, niter=6)          # 3000 > 8*256: exercises the faiss subsampling
    assert np.array_equal(a, ao), f"{(a != ao).sum()} assignments differ"
    assert np.array_equal(bits(c), bits(co)), "centroids are not bit-identical (point-order fp32 sums)"
    assert np.allclose(obj, oo, rtol=1e-5)
    a2, dist = idx.kmeans_assign(co)
    assert np.array_equal(a2, ao)
    Dk, Ik = oracle.knn(co, xf, 1, oracle.L2)
    assert np.array_equal(bits(dist), bits(Dk[:, 0]))
    ids = np.arange(0, 3000, 3)
    a3, c3, _ = idx.kmeans(4, niter=3, ids=ids, full_lloyd=True)
    a3o, c3o, _ = oracle.kmeans(xf[ids], 4, niter=3, full_lloyd=True)
    assert np.array_equal(a3, a3o) and np.array_equal(bits(c3), bits(c3o))
    with pytest.raises(gpu.NativeError):
        idx.kmeans(5000)
    idx.close()


def test_sem_cluster_by_reference_test_case(env):
    # .github/tests/rm_tests.py:52-79 (test_cluster_by) with table embeddings
    rm, vs, tmp = env
    names = ["Probability and Random Processes", "Cooking", "Food Sciences", "Optimization Methods in Engineering"]
    e = gauss(2, 32, 60)
    emb = {names[0]: e[0], names[1]: e[1], names[2]: e[1] * 0.95 + e[0] * 0.05, names[3]: e[0] * 0.95 + e[1] * 0.05}
    lotus.settings.configure(rm=lotus.TableRM({k: (v / np.linalg.norm(v)).astype(np.float32) for k, v in emb.items()}))
    df = pd.DataFrame({"Course Name": names})
    df = df.sem_index("Course Name", str(tmp / "c"))
    out = df.sem_cluster_by("Course Name", 2)
    assert out is df and "cluster_id" in df.columns
    groups = df.groupby("cluster_id")["Course Name"].apply(set).to_dict()
    assert len(groups) == 2
    assert {"Cooking", "Food Sciences"} in groups.values()
    assert {"Probability and Random Processes", "Optimization Methods in Engineering"} in groups.values()
    part = df.sem_partition_by(lotus.utils.cluster("Course Name", 2))
    assert part["_lotus_partition_id"].tolist() == df["cluster_id"].tolist()


def test_merge_topk_kernel_equals_host_rule(gpu):
    import torch
    from lotus_b200.distributed import merge_host_lists
    rng = np.random.default_rng(70)
    for metric in (0, 1):
        for g, k in ((2, 5), (8, 32), (3, 64)):
            nq = 77
            sc = rng.integers(0, 6, size=(g, nq, k)).astype(np.float32) / 4  # many exact ties
            sc = -np.sort(-sc, axis=2) if metric == 0 else np.sort(sc, axis=2)
            ids = np.stack([np.sort(rng.choice(1000, size=(nq, k), replace=True) + 1000 * gi, axis=1) for gi in range(g)])
            if metric == 0:
                ids = ids[:, :, ::-1].copy()  # IP lists carry equal scores in descending id
            ids[:, :, k - 1] = np.where(rng.random((g, nq)) < 0.2, -1, ids[:, :, k - 1])
            ts, ti = torch.from_numpy(sc).cuda(), torch.from_numpy(ids.astype(np.int64)).cuda()
            os_, oi = torch.empty((nq, k), dtype=torch.float32, device="cuda"), torch.empty((nq, k), dtype=torch.int64, device="cuda")
            gpu.merge_topk_dev(ts.data_ptr(), ti.data_ptr(), g, nq, k, metric, 0, os_.data_ptr(), oi.data_ptr(),
                               stream=torch.cuda.current_stream().cuda_stream)
            hs, hi = merge_host_lists(sc, ids.astype(np.int64), metric)
            assert np.array_equal(oi.cpu().numpy(), hi) and np.array_equal(bits(os_.cpu().numpy()), bits(hs))


def test_kmeans_accumulate_and_sharded_driver_single_rank(gpu):
    """The multi-GPU Lloyd driver on one rank (world 1): per-shard sums are faiss's point-order fp32 sums, and the driver's
    full-Lloyd result equals the oracle's full-Lloyd restatement bit for bit."""
    from lotus_b200.distributed import sharded_kmeans
    rng = np.random.default_rng(80)
    centers = gauss(5, 32, 81) * 4
    x = (centers[rng.integers(0, 5, 1500)] + gauss(1500, 32, 82, normalize=False)).astype(np.float32)
    idx = gpu.Index(x, gpu.F32, 1)
    ao, co, oo = oracle.kmeans(x, 5, niter=4, full_lloyd=True)
    sums, counts = idx.kmeans_accumulate(ao, 5)
    cref, href = oracle.compute_centroids(x, ao, 5)
    assert np.array_equal(counts, href)
    assert np.array_equal(bits(sums * (np.float32(1) / counts)[:, None]), bits(cref))
    a, c, obj = sharded_kmeans(idx, len(x), 0, 5, niter=4)
    assert np.array_equal(a, ao) and np.array_equal(bits(c), bits(co)) and np.allclose(obj, oo, rtol=1e-5)
    idx.close()


def test_device_hand_off_and_sharded_ids_single_rank(env):
    """torch CUDA tensors go into the index and the search without a host round trip (SURVEY §8f-2); the sharded index
    honours an ids subset."""
    import torch
    from lotus_b200.distributed import ShardedIndex
    rm, vs, tmp = env
    x = gauss(3000, 64, 90)
    xt = torch.from_numpy(x).cuda()
    vs.index(pd.Series(["d"] * 3000), xt, str(tmp / "dev"))
    out = vs(xt[:7], 4)
    Do, Io = oracle.knn(x, x[:7], 4)
    assert np.array_equal(np.asarray(out.indices), Io) and np.array_equal(bits(out.distances), bits(Do))
    xb = xt.to(torch.bfloat16)
    vs_b = lotus.B200VS()
    vs_b.index(None, xb, str(tmp / "devb"))
    xbf = xb.float().cpu().numpy()
    out = vs_b(xb[:7], 4)
    Do, Io = oracle.knn(xbf, xbf[:7], 4)
    assert np.array_equal(np.asarray(out.indices), Io) and np.array_equal(bits(out.distances), bits(Do))
    vs_b.close()
    sh = ShardedIndex(xt.contiguous(), 0)
    ids = np.arange(5, 3000, 3)
    s, i = sh.search(xt[:9].contiguous(), 6, ids=ids)
    Ds, Is = oracle.knn_subset(x, x[:9], 6, ids)
    assert np.array_equal(i.cpu().numpy(), Is) and np.array_equal(bits(s.cpu().numpy()), bits(Ds))
    sh.close()


def test_reference_operator_frames_on_gpu(env):
    """The frames the REFERENCE's operator code produced (tests/golden/reference_ops.json) are reproduced with B200VS."""
    import test_reference_golden as trg
    rm, vs, tmp = env
    lotus.settings.configure(rm=lotus.HashRM(dim=trg.GOLD["sim_join"]["dim"]))
    trg.replay_sim_join(tmp)
    trg.replay_search(tmp)
    trg.replay_dedup(tmp)
    trg.replay_cluster(tmp)
