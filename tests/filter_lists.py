"""The filter kernel's contract (knn_filter_sm90.cu), checked list by list against fp64 scores of the exact operand values.

For every query the kernel leaves, per corpus split and per set (bit 3 of the row id), a list of kp/2 candidates and `thr`.
finalize's certificate is sound only if
  (a) every list score is within eps of the exact score of its row, and
  (b) every row of the list's range and set that the list does not hold scores at most thr + eps,
with eps = rel_eps * |q| * max|x| (IP), or 2 rel_eps |q| mx + 2.4e-7 (mx^2 + 2 |q| mx) for L2 in the filter's own space
s = 2 q.x - |x|^2 (knn_exact.cu finalize_kernel). `check_lists` checks these and the list structure around them, and names the
broken property in its error. `run_matrix` runs the case matrix of tests/test_gpu_filter_lists.py through the library.
"""
import numpy as np

from helpers import gauss, grid, schedule_items

F32, BF16 = 0, 1
IP, L2 = 0, 1


def rel_eps_formula(d, store_dtype, filt_dtype, q_dtype):
    """DESIGN.md §2, restated: accumulation (d + 64) * 2^-23, plus the representation error of each operand the filter rounds
    (tf32 keeps 10 explicit mantissa bits of fp32: 2^-10; fp32 rounded to bf16: 2^-8; bf16 values are exact in both), plus
    the product of the two operand errors and 1e-6."""
    unit = 2.0 ** -10 if filt_dtype == F32 else 2.0 ** -8
    ex = unit if store_dtype == F32 else 0.0
    eq = unit if q_dtype == F32 else 0.0
    return float(np.float32((d + 64) * 2.0 ** -23 + ex + eq + ex * eq + 1e-6))


def list_ranges(plan, nq, n):
    """Corpus rows [lo, hi) of every (query, split) list, -1 where no work item writes the list (the splits beyond 0 of a query
    unit that swept the whole corpus in the first phase of the two-phase schedule)."""
    items, n_units, _ = schedule_items(plan, nq, n, 1)
    lo = np.full((n_units, plan["n_splits"]), -1, dtype=np.int64)
    hi = np.full((n_units, plan["n_splits"]), -1, dtype=np.int64)
    for unit, split, t0, t1 in items[0]:
        lo[unit, split], hi[unit, split] = t0 * 256, min(t1 * 256, n)
    unit_of_query = np.arange(nq) // 128 // (2 if plan["two_cta"] else 1)
    return lo[unit_of_query], hi[unit_of_query]


def scores(Q, X, metric):
    """Exact fp64 filter-space scores [nq, n] of the exact operand values."""
    S = Q @ X.T
    return S if metric == IP else 2.0 * S - np.einsum("ij,ij->i", X, X)[None, :]


def _margins(metric, rel_eps, qn, xn):
    """eps of finalize for query norms qn against row norms xn (broadcast), and the part of |err| rel_eps has to cover."""
    if metric == IP:
        return rel_eps * qn * xn, qn * xn
    return 2.0 * rel_eps * qn * xn + 2.4e-7 * (xn * xn + 2.0 * qn * xn), 2.0 * qn * xn


def check_lists(res, Q, X, metric, exact=False, top1=False, tag="", chunk=2048):
    """Raise AssertionError naming the first broken property of the lists in `res` (Index.filter_lists output) for exact fp64
    operands Q [nq, d] and X [n, d]. exact=True (grid data: every product and partial sum is exact) demands bit-equal scores and
    a discard bound with eps = 0. Returns the largest |err| / (|q| |x| rel_eps) over the entries (the L2 rounding of |x|^2 and
    of the epilogue fma taken out)."""
    nq, n = len(Q), len(X)
    rel = res["rel_eps"]
    kph = res["kp"] // 2
    lo, hi = list_ranges(res, nq, n)
    xn = np.sqrt(np.einsum("ij,ij->i", X, X))
    mx = xn.max()
    cols = np.arange(n)
    worst = 0.0
    for a in range(0, nq, chunk):
        b = min(nq, a + chunk)
        S = scores(Q[a:b], X, metric)
        qn = np.sqrt(np.einsum("ij,ij->i", Q[a:b], Q[a:b]))
        eps_max = np.zeros(b - a) if exact else _margins(metric, rel, qn, mx)[0]
        ids_all = res["id"][a:b].reshape(b - a, -1)
        srt = np.sort(np.where(ids_all >= 0, ids_all, -1 - np.arange(ids_all.shape[1])[None, :]), axis=1)
        dup = (np.diff(srt, axis=1) == 0).any(axis=1)
        if dup.any():
            r = int(np.argmax(dup))
            raise AssertionError(f"{tag}: partition: query {a + r} holds a row id twice across its lists")
        for s in range(res["n_splits"]):
            for e in range(2):
                where = f"{tag}: split {s} set {e}"
                L = res["id"][a:b, s, e].astype(np.int64)
                V = res["score"][a:b, s, e].astype(np.float64)
                T = res["thr"][a:b, s, e].astype(np.float64)
                l0, h0 = lo[a:b, s], hi[a:b, s]
                idle = l0 < 0
                bad = idle & ((L != -1).any(axis=1) | (T != -np.inf))
                if bad.any():
                    r = int(np.argmax(bad))
                    raise AssertionError(f"{where}: first phase: query {a + r} swept the whole corpus as one item, yet its list at "
                                         f"split {s} is not empty (ids {L[r][L[r] >= 0][:4].tolist()}, thr {T[r]})")
                act = ~idle
                valid = L >= 0
                bad = act[:, None] & ((~valid & ((L != -1) | (V != -np.inf)))
                                      | (valid & ((L < l0[:, None]) | (L >= h0[:, None]))))
                if bad.any():
                    r, c = np.argwhere(bad)[0]
                    raise AssertionError(f"{where}: partition: query {a + r} entry {c} = (id {L[r, c]}, score {V[r, c]}) is neither "
                                         f"(-1, -inf) nor a row of the split's range [{l0[r]}, {h0[r]})")
                bad = act[:, None] & valid & (((L >> 3) & 1) != e)
                if bad.any():
                    r, c = np.argwhere(bad)[0]
                    raise AssertionError(f"{where}: partition: query {a + r} holds row {L[r, c]} of set {1 - e}")
                rows, cc = np.nonzero(act[:, None] & valid)
                ex = S[rows, L[rows, cc]]
                err = V[rows, cc] - ex
                if exact:
                    bad = err != 0
                    if bad.any():
                        i = int(np.argmax(bad))
                        raise AssertionError(f"{where}: grid exactness: query {a + rows[i]} row {L[rows[i], cc[i]]} has filter score "
                                             f"{V[rows[i], cc[i]]!r}, exact {ex[i]!r}")
                else:
                    bad = np.abs(err) > eps_max[rows]
                    if bad.any():
                        i = int(np.argmax(bad))
                        raise AssertionError(f"{where}: accuracy: query {a + rows[i]} row {L[rows[i], cc[i]]}: |filter - exact| = "
                                             f"{abs(err[i]):.3e} > eps {eps_max[rows[i]]:.3e}")
                    eps_row, scale = _margins(metric, rel, qn[rows], xn[L[rows, cc]])
                    bad = np.abs(err) > eps_row
                    if bad.any():
                        i = int(np.argmax(bad))
                        raise AssertionError(f"{where}: per-row accuracy: query {a + rows[i]} row {L[rows[i], cc[i]]}: |filter - exact| "
                                             f"= {abs(err[i]):.3e} > rel_eps |q| |x| form {eps_row[i]:.3e}")
                    rounding = 0.0 if metric == IP else 2.4e-7 * (xn[L[rows, cc]] ** 2 + 2.0 * qn[rows] * xn[L[rows, cc]])
                    if len(err):
                        worst = max(worst, float(np.max(np.maximum(np.abs(err) - rounding, 0.0) / np.maximum(scale, 1e-300))) / rel)
                # every row of the range and set that the list does not hold scores at most thr + eps
                inr = act[:, None] & (cols[None, :] >= l0[:, None]) & (cols[None, :] < h0[:, None]) & (((cols >> 3) & 1) == e)[None, :]
                held = np.zeros_like(inr)
                held[rows, L[rows, cc]] = True
                out = np.where(inr & ~held, S, -np.inf)
                top = out.max(axis=1)
                bad = top > T + eps_max
                if bad.any():
                    r = int(np.argmax(bad))
                    prop = "completeness" if T[r] == -np.inf else "discard bound"
                    raise AssertionError(f"{where}: {prop}: query {a + r} drops row {int(np.argmax(out[r]))} with exact score "
                                         f"{top[r]!r} > thr {T[r]!r} + eps {eps_max[r]:.3e}")
                if top1:
                    b1, b2 = V[:, 0], V[:, 1]
                    bad = act & ~((b1 >= b2) & (b2 >= T) & (L[:, 2:] == -1).all(axis=1) & (V[:, 2:] == -np.inf).all(axis=1))
                    if bad.any():
                        r = int(np.argmax(bad))
                        raise AssertionError(f"{where}: top1: query {a + r} list is not (b1 >= b2 >= b3 = thr, then (-inf, -1)): "
                                             f"{V[r, :3].tolist()} ids {L[r, :3].tolist()} thr {T[r]}")
                    if exact:
                        best = -np.sort(-np.where(inr, S, -np.inf), axis=1)[:, :2]
                        bad = act & ((b1 != best[:, 0]) | (b2 != best[:, 1]))
                        if bad.any():
                            r = int(np.argmax(bad))
                            raise AssertionError(f"{where}: top1: query {a + r} keeps {V[r, :2].tolist()}, the two best exact scores "
                                                 f"are {best[r].tolist()}")
                else:
                    full = act & (T > -np.inf)
                    bad = full & (~valid.all(axis=1) | (V.min(axis=1) != T))
                    if bad.any():
                        r = int(np.argmax(bad))
                        raise AssertionError(f"{where}: list minimum: query {a + r} has thr {T[r]!r} but its list is "
                                             f"{'not full' if not valid[r].all() else f'at least {V[r].min()!r}'}")
    return worst


# ---- case matrix --------------------------------------------------------------------------------------------------------------
DIMS = [8, 30, 33, 100, 200, 768, 1000]
KS = [1, 5, 10, 32, 41, 100, 200]
NQS = [1, 127, 128, 129, 257, 383]
NS = [512, 769, 1032, 1289, 1791, 2048, 1545]  # 256 t + {0, 1, 8, 9, 255}
DATA = ["gauss", "unnorm", "neardup", "cancel", "grid"]


def make_data(kind, n, nq, d, seed):
    """Corpus [n, d] and queries [nq, d] (fp32) of one data kind."""
    rng = np.random.default_rng(seed)
    if kind == "grid":
        return grid(n, d, seed), grid(nq, d, seed + 1)
    if kind == "gauss":
        return gauss(n, d, seed), gauss(nq, d, seed + 1)
    if kind == "unnorm":  # row norms spread over 1e-2 .. 1e2
        return [(gauss(m, d, seed + i) * 10.0 ** rng.uniform(-2, 2, (m, 1))).astype(np.float32) for i, m in ((0, n), (1, nq))]
    if kind == "neardup":  # every row base + 1e-3 noise: scores crowd within a few ulps
        base = gauss(1, d, seed)
        return [(base + 1e-3 * gauss(m, d, seed + 1 + i, normalize=False)).astype(np.float32) for i, m in ((0, n), (1, nq))]
    # cancel: components of +-10 with alternating signs against constant ones, so the large products cancel in the sum
    alt = np.where(np.arange(d) % 2 == 0, 10.0, -10.0)
    x = alt[None, :] * rng.choice([-1.0, 1.0], (n, 1)) + gauss(n, d, seed, normalize=False)
    q = 10.0 * rng.choice([-1.0, 1.0], (nq, 1)) + gauss(nq, d, seed + 1, normalize=False)
    return x.astype(np.float32), q.astype(np.float32)


def _filterable(n, k):
    ms = 1 if k <= 40 else -(-k // 36)
    return n >= 512 and -(-n // 256) >= ms and n >= 4 * k


def cases():
    """(name, store, q_dtype, level, top1, metric, n, d, nq, k, data) of the matrix."""
    out = []
    for ci, (store, qdt) in enumerate([(BF16, BF16), (BF16, F32), (F32, F32)]):
        for metric in (IP, L2):
            for i in range(7):
                d, k = DIMS[i], KS[(i + 2 * ci + metric) % 7]
                n = NS[(i + ci + 3 * metric) % 7]
                while not _filterable(n, k):
                    n += 256
                nq = NQS[(i + ci + metric) % 6]
                data = DATA[(i + ci + 2 * metric) % 5]
                out.append((store, qdt, 1 if store == F32 else 0, False, metric, n, d, nq, k, data))
    # fp32 store, first level: the bf16 copy of the rows with the longer list (kp 32 / 64 / 72 for k <= 4 / 12 / 24)
    for k, n, d, nq, data in [(4, 4096, 100, 129, "gauss"), (12, 4353, 33, 383, "cancel"), (24, 4863, 768, 128, "grid")]:
        for metric in (IP, L2):
            out.append((F32, F32, 0, False, metric, n, d, nq, k, data))
    # k-means assignment: register top-2 epilogue, any number of centroids
    for store in (BF16, F32):
        for metric, (n, d, nq, data) in zip((IP, L2), [(100, 30, 257, "grid"), (1289, 200, 129, "unnorm")]):
            out.append((store, store, 0, True, metric, n, d, nq, 1, data))
        out.append((store, store, 0, True, L2, 769, 8, 383, 1, "grid" if store == F32 else "neardup"))
    # two-phase schedule: whole-corpus waves plus a split remainder, every query checked
    out.append((BF16, BF16, 0, False, IP, 2056, 64, 20_000, 10, "gauss"))
    out.append((F32, F32, 1, False, L2, 1033, 32, 20_000, 5, "grid"))
    return out


def run_matrix(nv):
    """Every case through Index.filter_lists and check_lists. -> {"failures": [...], "ratios": {config: max ratio}, "cases": N,
    "plans": [...]}; a case whose plan does not use the filter, or an operand configuration other than the one the case
    names, is a failure."""
    failures, ratios, plans = [], {}, []
    matrix = cases()
    for ci, (store, qdt, level, top1, metric, n, d, nq, k, data) in enumerate(matrix):
        x, q = make_data(data, n, nq, d, 1000 + ci)
        if store == BF16:
            xs = nv.f32_to_bf16_bits(x)
            X = nv.bf16_bits_to_f32(xs).astype(np.float64)
        else:
            xs, X = x, x.astype(np.float64)
        if qdt == BF16:
            qa = nv.f32_to_bf16_bits(q)
            Q = nv.bf16_bits_to_f32(qa).astype(np.float64)
        else:
            qa, Q = q, q.astype(np.float64)
        two_level = store == F32 and level == 0 and not top1
        filt = BF16 if store == BF16 or two_level else F32
        cfg = {(BF16, BF16): "bf16", (BF16, F32): "bf16 (fp32 q)", (F32, F32): "tf32"}[(store, qdt)]
        if two_level:
            cfg = "bf16 of fp32 store + fp32 q"
        tag = (f"case {ci} [{cfg}{' top1' if top1 else ''} {'L2' if metric else 'IP'} level {level} n={n} d={d} nq={nq} "
               f"k={k} {data}]")
        idx = nv.Index(xs, store, metric)
        try:
            res = idx.filter_lists(qa, k, qdt, top1=top1, level=level)
        finally:
            idx.close()
        plans.append({"case": ci, **{key: res[key] for key in ("kp", "n_splits", "units_whole", "two_cta", "two_level")}})
        try:
            assert res["use_filter"], f"{tag}: the plan does not use the filter"
            assert res["two_level"] == two_level and res["filt_dtype"] == filt, f"{tag}: plan {plans[-1]}, filt_dtype {res['filt_dtype']}"
            # the library writes 2^-23 as the decimal 1.1920929e-7: the two can round to float32 values one ulp apart
            want = rel_eps_formula(d, store, filt, qdt)
            assert abs(res["rel_eps"] - want) <= 2.0 ** -23 * want, f"{tag}: library rel_eps {res['rel_eps']!r} != DESIGN §2 formula {want!r}"
            if nq >= 20_000:
                assert res["units_whole"] > 0 and res["n_splits"] > 1, f"{tag}: not a two-phase schedule: {plans[-1]}"
            r = check_lists(res, Q, X, metric, exact=data == "grid", top1=top1, tag=tag)
            if data != "grid":
                key = f"{cfg} d={d}"
                ratios[key] = max(ratios.get(key, 0.0), r)
        except AssertionError as e:
            failures.append(str(e))
    return {"cases": len(matrix), "failures": failures, "ratios": ratios, "plans": plans}
