"""Host-side mirror of the reference's plugin/operator surface, exercised on CPU with a test-double vector store
(tests/helpers.NumpyVS, backed by the oracle). The assertions restate what the reference's own operator code does
(file:line cited per test) and, where the reference has a test for it, mirror that test (.github/tests/rm_tests.py)."""
import os
import struct

import numpy as np
import pandas as pd
import pytest

import lotus_b200 as lotus
import oracle
from helpers import NumpyVS, gauss, schedule_items
from lotus_b200 import faiss_io


@pytest.fixture
def env(tmp_path):
    rm = lotus.HashRM(dim=32)
    vs = NumpyVS()
    lotus.settings.configure(rm=rm, vs=vs, enable_cache=False)
    yield rm, vs, tmp_path
    lotus.settings.configure(rm=None, vs=None)


def test_settings_configure_and_context():
    # lotus/settings.py:41-70
    with pytest.raises(ValueError, match="Invalid setting"):
        lotus.settings.configure(nope=1)
    lotus.settings.configure(enable_cache=False)
    with lotus.settings.context(enable_cache=True):
        assert lotus.settings.enable_cache is True
        with lotus.settings.context(parallel_groupby_max_threads=2):
            assert lotus.settings.enable_cache is True and lotus.settings.parallel_groupby_max_threads == 2
    assert lotus.settings.enable_cache is False
    with pytest.raises(ValueError):
        with lotus.settings.context(bogus=1):
            pass


def test_rm_passes_ndarrays_through():
    # lotus/models/rm.py:73-85
    rm = lotus.HashRM(dim=8)
    q = np.ones((2, 8), np.float32)
    assert rm.convert_query_to_query_vector(q) is q
    assert rm.convert_query_to_query_vector("a").shape == (1, 8)
    assert rm.convert_query_to_query_vector(pd.Series(["a", "b"])).shape == (2, 8)
    assert np.array_equal(rm(["x"]), rm(["x"]))


def test_faiss_index_file_layout_roundtrip(tmp_path):
    x = gauss(5, 4, 0)
    p = str(tmp_path / "index")
    faiss_io.write_flat_index(p, x, faiss_io.METRIC_INNER_PRODUCT)
    raw = open(p, "rb").read()
    # faiss/impl/index_write.cpp: fourcc, d, ntotal, dummy, dummy, is_trained, metric_type, then WRITEXBVECTOR(codes)
    assert raw[:4] == b"IxFI"
    d, n, d1, d2, trained, metric = struct.unpack("<iqqqBi", raw[4:4 + 33])
    assert (d, n, d1, d2, trained, metric) == (4, 5, 1 << 20, 1 << 20, 1, 0)
    assert struct.unpack("<Q", raw[37:45])[0] == 20 and len(raw) == 45 + 80
    y, m = faiss_io.read_flat_index(p)
    assert m == 0 and np.array_equal(x, y)
    faiss_io.write_flat_index(p, x, faiss_io.METRIC_L2)
    assert open(p, "rb").read(4) == b"IxF2" and faiss_io.read_flat_index(p)[1] == 1
    open(p, "wb").write(b"IwFl" + raw[4:])
    with pytest.raises(ValueError, match="IndexFlat"):
        faiss_io.read_flat_index(p)


def test_index_dir_keeps_the_callers_vecs_like_the_reference(tmp_path):
    # faiss_vs.py:27-30: vecs is a pickle of the array as given (float64 for LiteLLMRM), the index holds float32
    x64 = gauss(6, 8, 1).astype(np.float64)
    faiss_io.write_index_dir(str(tmp_path / "d"), x64, x64.astype(np.float32), 0)
    vecs, x, metric = faiss_io.read_index_dir(str(tmp_path / "d"))
    assert vecs.dtype == np.float64 and x.dtype == np.float32 and np.array_equal(vecs.astype(np.float32), x)
    with pytest.raises(ValueError, match="not found"):
        faiss_io.read_index_dir(str(tmp_path / "missing"))


def test_sem_index_sets_attrs_and_load_sem_index(env):
    rm, vs, tmp = env
    df = pd.DataFrame({"t": ["a", "b", "c"]})
    out = df.sem_index("t", str(tmp / "i1"))
    assert out is df and df.attrs["index_dirs"]["t"] == str(tmp / "i1") and vs.index_dir == str(tmp / "i1")
    df["u"] = ["x", "y", "z"]
    df.sem_index("u", str(tmp / "i2"))
    assert set(df.attrs["index_dirs"]) == {"t", "u"}  # pandas>=3 accessor re-creation must not wipe earlier entries
    df2 = pd.DataFrame({"t": ["a", "b", "c"]}).load_sem_index("t", str(tmp / "i1"))
    assert df2.attrs["index_dirs"] == {"t": str(tmp / "i1")}
    with pytest.raises(AttributeError):
        pd.Series([1]).to_frame().T.sem_index  # accessor only validates DataFrames; a frame is fine
        lotus.sem_ops.SemIndexDataframe([1, 2])


def reference_sim_join(left, right, vs, rm, left_on, right_on, K, lsuffix="", rsuffix="", score_suffix="", keep_index=False):
    """lotus/sem_ops/sem_sim_join.py:130-166 restated literally (Python double loop + the two joins)."""
    queries = left[left_on]
    qv = rm.convert_query_to_query_vector(queries)
    out = vs(qv, K, ids=list(right.index))
    other_index_set = set(right.index)
    join_results = []
    for q_idx, res_ids in enumerate(out.indices):
        for i, res_id in enumerate(res_ids):
            if res_id != -1 and res_id in other_index_set:
                join_results.append((left.index[q_idx], res_id, out.distances[q_idx][i]))
    df1, df2 = left.copy(), right.copy()
    df1["_left_id"] = df1.index
    df2["_right_id"] = df2.index
    temp_df = pd.DataFrame(join_results, columns=["_left_id", "_right_id", "_scores" + score_suffix])
    joined = df1.join(temp_df.set_index("_left_id"), how="right", on="_left_id").join(
        df2.set_index("_right_id"), how="left", on="_right_id", lsuffix=lsuffix, rsuffix=rsuffix)
    if not keep_index:
        joined.drop(columns=["_left_id", "_right_id"], inplace=True)
    return joined


@pytest.mark.parametrize("keep_index", [False, True])
def test_sem_sim_join_equals_the_reference_control_flow(env, keep_index):
    rm, vs, tmp = env
    left = pd.DataFrame({"a": [f"l{i}" for i in range(7)], "v": range(7)})
    right = pd.DataFrame({"b": [f"r{i}" for i in range(11)], "v": range(11)}).sem_index("b", str(tmp / "r"))
    got = left.sem_sim_join(right, "a", "b", K=3, lsuffix="_l", rsuffix="_r", keep_index=keep_index)
    want = reference_sim_join(left, right, vs, rm, "a", "b", 3, "_l", "_r", keep_index=keep_index)
    assert list(got.columns) == list(want.columns) and len(got) == 21
    pd.testing.assert_frame_equal(got.reset_index(drop=True), want.reset_index(drop=True), check_dtype=False)
    assert list(got.index) == list(want.index)
    # filtered right frame: only its rows may come back (ids=list(other.index), sem_sim_join.py:132-134)
    sub = right[right["v"] % 2 == 0]
    got = left.sem_sim_join(sub, "a", "b", K=4, lsuffix="_l", rsuffix="_r")
    assert set(got["b"]) <= set(sub["b"]) and len(got) == 28
    # K larger than the right frame: every right row once per left row, -1 padding dropped
    got = left.sem_sim_join(sub, "a", "b", K=50, lsuffix="_l", rsuffix="_r")
    assert len(got) == 7 * len(sub)


def test_sem_sim_join_errors_like_the_reference(env):
    rm, vs, tmp = env
    left = pd.DataFrame({"a": ["x"]})
    right = pd.DataFrame({"b": ["y"]})
    with pytest.raises(ValueError, match="Index directory for column b not found"):
        left.sem_sim_join(right, "a", "b", K=1)
    with pytest.raises(ValueError, match="must have a name"):
        left.sem_sim_join(pd.Series(["y"]), "a", "b", K=1)
    lotus.settings.configure(vs=None)
    with pytest.raises(ValueError, match="retrieval model"):
        left.sem_sim_join(right, "a", "b", K=1)


def test_sem_sim_join_reference_test_case(env):
    # .github/tests/rm_tests.py:103-123 (test_sim_join) with table embeddings standing in for the live model
    rm, vs, tmp = env
    e = {"History of the Atlantic World": [1, 0.1, 0], "Riemannian Geometry": [0, 0.2, 1], "Math": [0, 0, 1], "History": [1, 0, 0]}
    lotus.settings.configure(rm=lotus.TableRM({k: np.asarray(v, np.float32) for k, v in e.items()}))
    df1 = pd.DataFrame({"Course Name": ["History of the Atlantic World", "Riemannian Geometry"]})
    df2 = pd.DataFrame({"Skill": ["Math", "History"]}).sem_index("Skill", str(tmp / "s"))
    joined = df1.sem_sim_join(df2, left_on="Course Name", right_on="Skill", K=1)
    assert set(zip(joined["Course Name"], joined["Skill"])) == {("History of the Atlantic World", "History"), ("Riemannian Geometry", "Math")}


def test_sem_search_topk_scores_and_filtered_frames(env):
    rm, vs, tmp = env
    df = pd.DataFrame({"t": [f"doc{i}" for i in range(20)]}).sem_index("t", str(tmp / "s"))
    q = "doc7"
    out = df.sem_search("t", q, K=4, return_scores=True)
    D, I = oracle.knn(rm(df["t"].tolist()), rm([q]), 4)
    assert list(out.index) == I[0].tolist() and np.allclose(out["vec_scores_sim_score"], D[0])
    assert out.attrs["index_dirs"] == df.attrs["index_dirs"] and out["t"].iloc[0] == "doc7"
    # filtered frame (sem_search.py:116-138 K-doubling loop in the reference): same rows, one search
    sub = df[df.index % 3 == 0]
    out = sub.sem_search("t", q, K=5, return_scores=True)
    ids = np.asarray(sub.index)
    Ds, Is = oracle.knn_subset(rm(df["t"].tolist()), rm([q]), 5, ids)
    assert list(out.index) == Is[0].tolist() and np.allclose(out["vec_scores_sim_score"], Ds[0])
    assert len(df.sem_search("t", q, K=100)) == 20  # K = min(K, len(df)) (sem_search.py:118)
    assert len(df.iloc[0:0].sem_search("t", q, K=3)) == 0
    with pytest.raises(AssertionError):
        df.sem_search("t", q)
    with pytest.raises(ValueError, match="Reranker not found"):
        df.sem_search("t", q, K=2, n_rerank=1)


def test_sem_search_multi_query_equals_the_single_query_calls(env):
    # SURVEY §8f-4: one batched vs() call for a list of queries; every frame equals its single-query counterpart
    rm, vs, tmp = env
    df = pd.DataFrame({"t": [f"doc{i}" for i in range(40)]}).sem_index("t", str(tmp / "m"))
    qs = ["doc3", "doc17", "something else"]
    calls = []
    orig = type(vs).__call__

    def counting(self, *a, **kw):
        calls.append(1)
        return orig(self, *a, **kw)

    type(vs).__call__ = counting
    try:
        many = df.sem_search("t", qs, K=5, return_scores=True)
        assert len(calls) == 1 and isinstance(many, list) and len(many) == 3
        sub = df[df.index % 2 == 1]
        many_sub = sub.sem_search.batch("t", qs, K=4, return_scores=True)
    finally:
        type(vs).__call__ = orig
    for q, got in zip(qs, many):
        pd.testing.assert_frame_equal(got, df.sem_search("t", q, K=5, return_scores=True))
    for q, got in zip(qs, many_sub):
        pd.testing.assert_frame_equal(got, sub.sem_search("t", q, K=4, return_scores=True))
    vecs = rm(qs)                                            # precomputed query vectors [Q, d]
    for a, b in zip(df.sem_search("t", vecs, K=5), many):
        assert list(a.index) == list(b.index)
    assert [len(f) for f in df.iloc[0:0].sem_search("t", qs, K=3)] == [0, 0, 0]


def test_cluster_fn_validation(env):
    # lotus/utils.py:35-39,49-52
    from lotus_b200.utils import cluster
    df = pd.DataFrame({"t": ["a", "b"]})
    with pytest.raises(ValueError, match="Column zz not found"):
        cluster("zz", 1)(df)
    with pytest.raises(ValueError, match="Number of centroids must be less than number of documents. 5 > 2"):
        cluster("t", 5)(df)
    with pytest.raises(ValueError, match="Index directory for column t not found"):
        cluster("t", 1)(df)


def test_partition_by_stores_ids(env):
    df = pd.DataFrame({"t": ["a", "b", "c"]})
    out = df.sem_partition_by(lambda d: [2, 0, 2])
    assert out is df and df["_lotus_partition_id"].tolist() == [2, 0, 2]


def test_operator_cache_passthrough_and_reference_failure_mode(env):
    rm, vs, tmp = env
    df = pd.DataFrame({"t": ["a", "b"]})
    with lotus.settings.context(enable_cache=True):  # lotus/cache.py:38-41: dereferences settings.lm.cache
        with pytest.raises(AttributeError):
            df.sem_index("t", str(tmp / "c"))


# ---- sem_sim_join frame assembly: positional-take fast path == the reference's two pandas joins ------------------------
def _random_frame(n, kind, cols, seed):
    r = np.random.default_rng(seed)
    data = {}
    for c in cols:
        t = int(r.integers(0, 5))
        if t == 0:
            data[c] = [f"s{r.integers(0, 100)}" for _ in range(n)]
        elif t == 1:
            data[c] = r.integers(0, 100, n)
        elif t == 2:
            data[c] = r.random(n)
        elif t == 3:
            data[c] = r.random(n) > 0.5
        else:
            data[c] = pd.Categorical(r.choice(["x", "y", "z"], n))
    df = pd.DataFrame(data)
    if kind == "perm":
        df.index = r.permutation(n) * 3 + 1
    elif kind == "str":
        df.index = [f"k{i}" for i in r.permutation(n)]
    elif kind == "named":
        df.index = pd.Index(r.permutation(n), name="rid")
    elif kind == "float":
        df.index = r.permutation(n).astype(np.float64)
    elif kind == "dup":
        df.index = r.integers(0, max(1, n // 2), n)
    return df


def test_sim_join_take_assembly_equals_the_reference_joins():
    from lotus_b200.sem_ops.sem_sim_join import assemble_join, assemble_take
    rng = np.random.default_rng(7)
    fast = 0
    for trial in range(400):
        nl, nr, K = int(rng.integers(1, 30)), int(rng.integers(1, 30)), int(rng.integers(1, 6))
        lk = rng.choice(["range", "perm", "str", "named", "float", "dup"])
        rk = rng.choice(["range", "perm", "named", "float"])
        lc = list(rng.choice(["a", "b", "c", "d"], int(rng.integers(1, 4)), replace=False))
        rc = list(rng.choice(["a", "e", "f", "g"], int(rng.integers(1, 4)), replace=False))
        L, R = _random_frame(nl, lk, lc, trial * 2), _random_frame(nr, rk, rc, trial * 2 + 1)
        if trial % 3 == 0:
            L.attrs["index_dirs"] = {"a": "x"}
        if trial % 5 == 0:
            L[lc[0]] = pd.array(rng.integers(0, 9, nl), dtype="Int64")
            L.iloc[0, L.columns.get_loc(lc[0])] = pd.NA
        if trial % 7 == 0:
            R[rc[0]] = pd.to_datetime("2020-01-01") + pd.to_timedelta(rng.integers(0, 99, nr), unit="D")
        ls, rs = [("", ""), ("_l", "_r"), ("", "_r"), ("_l", "")][int(rng.integers(0, 4))]
        keep_index, score_col = bool(rng.integers(0, 2)), "_scores" + ["", "_x"][int(rng.integers(0, 2))]
        m = int(rng.integers(0, nl * K + 1))
        left_pos = np.sort(rng.integers(0, nl, m)).astype(np.int64)
        right_labels = np.asarray(R.index)[rng.integers(0, nr, m)]
        scores = rng.random(m).astype(np.float32)
        got = assemble_take(L, R, left_pos, right_labels, scores, score_col, ls, rs, keep_index)
        if got is None:
            continue
        fast += 1
        temp = pd.DataFrame({"_left_id": np.asarray(L.index)[left_pos] if m else np.asarray([], dtype=object),
                             "_right_id": right_labels, score_col: scores})
        want = assemble_join(L, R, temp, ls, rs, keep_index)
        pd.testing.assert_frame_equal(got, want, check_exact=True, check_index_type=True, check_column_type=True)
        assert list(got.columns) == list(want.columns) and got.attrs == want.attrs
    assert fast > 200  # the plain case is the common one; duplicates / clashes fall back to the joins


def test_sim_join_hands_label_arrays_to_stores_that_take_them(env):
    rm, vs, tmp = env
    seen = []

    class ArrayVS(NumpyVS):
        accepts_id_arrays = True  # what B200VS declares

        def __call__(self, query_vectors, K, ids=None, **kw):
            seen.append(type(ids))
            return super().__call__(query_vectors, K, ids=ids, **kw)

    left = pd.DataFrame({"a": [f"l{i}" for i in range(5)]})
    right = pd.DataFrame({"b": [f"r{i}" for i in range(9)]}).sem_index("b", str(tmp / "r"))
    want = left.sem_sim_join(right[right.index % 2 == 1], "a", "b", K=3)
    avs = ArrayVS()
    avs.dirs, avs.x, avs.index_dir = vs.dirs, vs.x, vs.index_dir
    lotus.settings.configure(vs=avs)
    got = left.sem_sim_join(right[right.index % 2 == 1], "a", "b", K=3)
    assert seen == [np.ndarray]
    pd.testing.assert_frame_equal(got, want)


def test_bf16_exact_queries_ship_two_byte_patterns_decided_from_the_values():
    """ADVICE r1 (vs.py:76): the bf16 form of a query batch is derived from its VALUES on every call, never from a tag
    that an in-place edit could leave stale."""
    from lotus_b200 import _native as nv
    from lotus_b200.vs import BF16Backed, _to_host_matrix
    bits = nv.f32_to_bf16_bits(gauss(6, 16, 3))
    m = BF16Backed.wrap(nv.bf16_bits_to_f32(bits))
    assert isinstance(m, np.ndarray) and m.dtype == np.float32
    # handed back untouched (what sem_sim_join does via rm.convert_query_to_query_vector): 2-byte patterns, bf16 dtype code
    out, code, f32 = _to_host_matrix(lotus.HashRM(dim=16).convert_query_to_query_vector(m), False, exact_bf16_ok=True)
    assert code == nv.BF16 and out.dtype == np.uint16 and np.array_equal(out, bits) and np.array_equal(f32, np.asarray(m))
    # in-place edits that stay bf16-representable ship the NEW values; anything else goes as float32
    m *= 2.0
    out, code, _ = _to_host_matrix(m, False, exact_bf16_ok=True)
    assert code == nv.BF16 and np.array_equal(nv.bf16_bits_to_f32(out), np.asarray(m))
    m[0, 0] = np.float32(1.0) + np.float32(2.0 ** -20)
    out, code, _ = _to_host_matrix(m, False, exact_bf16_ok=True)
    assert code == nv.F32 and out.dtype == np.float32 and np.array_equal(out, np.asarray(m))
    # without the store asking for it (fp32 index) nothing is converted
    out, code, _ = _to_host_matrix(m * 0 + 1, False)
    assert code == nv.F32


def test_f32_to_bf16_rounding_matches_the_reference_formula_and_keeps_nan():
    from lotus_b200 import _native as nv
    rng = np.random.default_rng(5)
    a = rng.standard_normal(100_000).astype(np.float32) * np.float32(10.0) ** rng.integers(-20, 20, 100_000).astype(np.float32)
    a[:8] = [0.0, -0.0, np.inf, -np.inf, 1.0, np.float32(1.0) + np.float32(2.0 ** -8), np.float32(1.0) + np.float32(3 * 2.0 ** -9), 65504.0]
    u = a.view(np.uint32).astype(np.uint64)
    want = ((u + 0x7FFF + ((u >> 16) & 1)) >> 16).astype(np.uint16)
    got, exact = nv.f32_to_bf16_checked(a)
    assert np.array_equal(got, want) and not exact
    assert np.array_equal(oracle.f32_to_bf16_bits(a), got)
    # NaN payloads must stay NaN (ADVICE r1, _native.py:118: 0x7fffffff used to become -0.0)
    nan = np.array([0x7fffffff, 0xffffffff, 0x7fc00000, 0x7f800001], dtype=np.uint32).view(np.float32)
    nb = nv.f32_to_bf16_bits(nan)
    assert np.isnan(nv.bf16_bits_to_f32(nb)).all()
    assert nv.f32_to_bf16_checked(nv.bf16_bits_to_f32(got))[1] is True


def test_quickstart_example_runs_against_the_test_double(monkeypatch, capsys):
    # examples/quickstart.py needs an H100; its control flow (all five operators) is exercised here with the oracle-backed VS
    import lotus_b200.sem_ops.sem_dedup as sd
    monkeypatch.setattr(sd.nv, "connected_components", lambda n, pi, pj, device=0: oracle.connected_components(n, pi, pj))
    path = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "examples", "quickstart.py")
    src = open(path).read()
    assert "vs=lotus.B200VS()" in src
    try:
        exec(compile(src.replace("vs=lotus.B200VS()", "vs=NumpyVS()"), path, "exec"), {"NumpyVS": NumpyVS, "__name__": "__main__"})
    finally:
        lotus.settings.configure(rm=None, vs=None)
    out = capsys.readouterr().out
    assert "bread baking" in out and "vec_scores_sim_score" in out and "cluster_id" in out


def test_operator_cache_is_pass_through_unless_enabled_and_then_keys_on_frame_and_arguments(env):
    rm, vs, tmp = env
    df = pd.DataFrame({"t": [f"doc{i}" for i in range(6)]}).sem_index("t", str(tmp / "c"))
    first = df.sem_search("t", "doc3", K=2)

    class DictCache:
        def __init__(self):
            self.d, self.gets, self.inserts = {}, 0, 0

        def get(self, key):
            self.gets += 1
            return self.d.get(key)

        def insert(self, key, value):
            self.inserts += 1
            self.d[key] = value

    class FakeLM:
        cache = DictCache()

    # enabled without an LM: the reference dereferences settings.lm.cache (lotus/cache.py:38-41) -> AttributeError
    lotus.settings.configure(enable_cache=True, lm=None)
    try:
        with pytest.raises(AttributeError):
            df.sem_search("t", "doc3", K=2)
        lotus.settings.configure(lm=FakeLM())
        a = df.sem_search("t", "doc3", K=2)
        b = df.sem_search("t", "doc3", K=2)          # same frame + arguments: served from the cache
        c = df.sem_search("t", "doc3", K=3)          # different argument: computed
        assert FakeLM.cache.inserts == 2 and b is a and len(c) == 3
        pd.testing.assert_frame_equal(a, first)
    finally:
        lotus.settings.configure(enable_cache=False, lm=None)


def test_sem_search_k_doubling_branch_equals_the_ids_branch_and_rerank_reorders(env):
    rm, vs, tmp = env
    df = pd.DataFrame({"t": [f"doc{i}" for i in range(40)]}).sem_index("t", str(tmp / "s"))
    sub = df[df.index % 5 == 0]                       # a filtered frame: the reference needs its K-doubling loop here
    want = sub.sem_search("t", "doc7", K=3, return_scores=True)

    class NoIdsVS(NumpyVS):
        supports_ids_search = False                   # a store like the reference's Qdrant/Weaviate ones: no ids= argument

        def __call__(self, query_vectors, K, ids=None, **kw):
            assert ids is None
            return super().__call__(query_vectors, K, **kw)

    nvs = NoIdsVS()
    nvs.dirs, nvs.x, nvs.index_dir = vs.dirs, vs.x, vs.index_dir
    lotus.settings.configure(vs=nvs)
    got = sub.sem_search("t", "doc7", K=3, return_scores=True)
    pd.testing.assert_frame_equal(got, want)

    class FlipReranker:                               # sem_search.py:146-154: reranker(query, docs, n) -> .indices into docs
        def __call__(self, query, docs, n):
            from types import SimpleNamespace
            return SimpleNamespace(indices=list(range(len(docs)))[::-1][:n])

    with pytest.raises(ValueError, match="Reranker not found"):
        sub.sem_search("t", "doc7", K=3, n_rerank=2)
    lotus.settings.configure(reranker=FlipReranker())
    try:
        rr = sub.sem_search("t", "doc7", K=3, n_rerank=2)
        assert rr["t"].tolist() == want["t"].tolist()[::-1][:2]
        only = sub.sem_search("t", "doc7", n_rerank=2)   # K=None: rerank the whole frame
        assert only["t"].tolist() == sub["t"].tolist()[::-1][:2]
    finally:
        lotus.settings.configure(reranker=None)


@pytest.mark.parametrize("nq,n", [(100_000, 1_000_000), (100_000, 500_000), (100_000, 250_000), (100_000, 125_000), (40_000, 20_000),
                                  (18_944, 3_000), (19_200, 70_000), (9_472, 500_000), (300, 6_000), (1_000_000, 4_096)])
@pytest.mark.parametrize("k", [10, 32, 64])
def test_filter_schedule_covers_every_unit_tile_pair_once(nq, n, k):
    """The two-phase schedule (whole-corpus waves + split remainder) for the multi-GPU shard shapes and the edge shapes the GPU
    tests do not reach: every (query unit, corpus tile) pair is scored by exactly one item, every split is non-empty, whole units
    only ever write list 0, and the plan is never worse than the uniform split plan under the kernel's own cost model."""
    from lotus_b200 import _native as nv
    plan = nv.filter_plan(nq, n, k)
    assert plan["kp"] > 0 and plan["n_splits"] >= 1
    workers = 66 if plan["two_cta"] else 132
    per_worker, n_units, n_ntiles = schedule_items(plan, nq, n, workers)
    assert plan["units_whole"] % workers == 0 and 0 <= plan["units_whole"] <= n_units
    cover = np.zeros((n_units, n_ntiles), dtype=np.int32)
    lists = set()
    for items in per_worker:
        for unit, split, t0, t1 in items:
            assert t1 > t0, "empty split"
            assert 0 <= split < plan["n_splits"]
            cover[unit, t0:t1] += 1
            assert (unit, split) not in lists
            lists.add((unit, split))
            if unit < plan["units_whole"]:
                assert split == 0 and (t0, t1) == (0, n_ntiles)
    assert (cover == 1).all()
    # load balance: the busiest worker carries at most one item's worth of tiles more than the mean
    loads = [sum(t1 - t0 for _, _, t0, t1 in items) for items in per_worker]
    biggest_item = max(t1 - t0 for items in per_worker for _, _, t0, t1 in items)
    assert max(loads) <= np.mean(loads) + biggest_item


def test_sharded_hint_pruning_never_drops_a_global_topk_member():
    """Host model of the two-stage row-sharded search (DESIGN §6): shard r reports lower_r = (its ceil(k/G)-th best FILTER score)
    - eps; hint = min_r lower_r; a local row is re-scored only if filter + eps >= hint. With |filter - exact| <= eps the rows that
    are pruned can never belong to (or tie with the k-th of) the merged exact top k — checked on random data with adversarial
    filter noise at the full +-eps, including shards that hold none of the top k."""
    rng = np.random.default_rng(0)
    for trial in range(200):
        G, k = int(rng.integers(2, 9)), int(rng.integers(1, 40))
        sizes = rng.integers(max(1, k // G), 400, size=G)
        eps = float(rng.choice([1e-4, 1e-2, 0.3]))
        exact = [np.sort(rng.standard_normal(m))[::-1] * (1.0 if trial % 3 else 0.05) for m in sizes]
        filt = [e + rng.choice([-eps, eps, 0.0], size=len(e)) * rng.random(len(e)) ** 0.2 for e in exact]
        j = -(-k // G)
        lowers = []
        for f in filt:
            top = np.sort(f)[::-1]
            lowers.append(top[j - 1] - eps if len(top) >= j else -np.inf)
        hint = min(lowers)
        all_exact = np.concatenate(exact)
        kth = np.sort(all_exact)[::-1][min(k, len(all_exact)) - 1]
        for e, f in zip(exact, filt):
            pruned = f + eps < hint
            assert not (e[pruned] >= kth).any(), (trial, G, k, eps)


class _PlainVS(NumpyVS):
    """A store WITHOUT the streaming extensions (what the reference's FaissVS looks like to the accessors)."""
    threshold_pairs = property(lambda self: (_ for _ in ()).throw(AttributeError("no threshold_pairs")))
    kmeans = property(lambda self: (_ for _ in ()).throw(AttributeError("no kmeans")))


def test_accessors_fall_back_to_the_reference_flow_for_stores_without_extensions(env, monkeypatch):
    """ADVICE r1 (sem_dedup.py:55): with a VS that has neither threshold_pairs nor kmeans the accessors must follow the reference's
    own control flow — sem_dedup through vs(q, K=n, ids=rows) (sem_dedup.py:45 via sem_sim_join.py:132-134), cluster through
    faiss.Kmeans (utils.py:59-70) — instead of raising; and missing text values never join a component."""
    import sys
    import types
    import lotus_b200.sem_ops.sem_dedup as sd
    rm, vs, tmp = env
    monkeypatch.setattr(sd.nv, "connected_components", lambda n, pi, pj, device=0: oracle.connected_components(n, pi, pj))
    vals = [f"v{i % 12}" for i in range(40)] + [None, None]
    df = pd.DataFrame({"Text": vals}).sem_index("Text", str(tmp / "dd"))
    want = df.sem_dedup("Text", threshold=0.3)               # streaming path of the oracle-backed test double
    plain = _PlainVS()
    plain.dirs, plain.index_dir, plain.x = vs.dirs, vs.index_dir, vs.x
    assert not hasattr(plain, "threshold_pairs") and not hasattr(plain, "kmeans")
    lotus.settings.configure(vs=plain)
    got = df.sem_dedup("Text", threshold=0.3)                # reference flow: vs(q, K=n, ids=rows) + `_scores > threshold`
    assert got["Text"].tolist() == want["Text"].tolist()
    assert got["Text"].isna().sum() == 2                      # None never equals anything: both rows survive
    # cluster: faiss.Kmeans stand-in (what the reference calls, utils.py:61-65)
    calls = {}
    fake = types.ModuleType("faiss")

    class Kmeans:
        def __init__(self, d, k, niter=25, verbose=False):
            calls["args"] = (d, k, niter, verbose)

        def train(self, x):
            self.x = np.asarray(x, dtype=np.float32)
            _, self.cent, _ = oracle.kmeans(self.x, calls["args"][1], niter=calls["args"][2])
            outer = self

            class Ix:
                def search(self, q, kk):
                    return oracle.knn(outer.cent, np.asarray(q, dtype=np.float32), kk, oracle.L2)
            self.index = Ix()

    fake.Kmeans = Kmeans
    monkeypatch.setitem(sys.modules, "faiss", fake)
    cdf = pd.DataFrame({"t": [f"doc{i}" for i in range(30)]}).sem_index("t", str(tmp / "cc"))
    plain.dirs = vs.dirs
    out = cdf.sem_cluster_by("t", 3, niter=4)
    a, _, _ = oracle.kmeans(rm(cdf["t"].tolist()), 3, niter=4)
    assert calls["args"][1:3] == (3, 4) and out["cluster_id"].tolist() == a.tolist()
