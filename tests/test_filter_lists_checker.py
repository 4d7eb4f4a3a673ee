"""The checker of tests/test_gpu_filter_lists.py must fail when the filter is wrong: it accepts lists built by a numpy model of
the epilogue and rejects each single defect, naming the property it breaks. No GPU."""
import numpy as np
import pytest

import filter_lists as fl
from helpers import grid

# a two-phase plan: query units 0 and 1 sweep the whole corpus as one item each, units 2 and 3 are cut into two splits
PLAN = {"kp": 16, "n_splits": 2, "units_whole": 2, "two_cta": False, "rel_eps": fl.rel_eps_formula(64, fl.BF16, fl.BF16, fl.BF16)}
NQ, N, D = 512, 1000, 64


def model_lists(Q, X, metric, plan=PLAN):
    """What the epilogue leaves: per (query, split, set) the exact top kp/2 of the range, thr = the list minimum once the list
    is full (-inf before), empty slots (-inf, -1); lists no item writes hold id -1 and thr -inf (their scores are not written)."""
    S = fl.scores(Q, X, metric)
    nq, n = S.shape
    kph = plan["kp"] // 2
    lo, hi = fl.list_ranges(plan, nq, n)
    sc = np.full((nq, plan["n_splits"], 2, kph), -np.inf, dtype=np.float32)
    ids = np.full(sc.shape, -1, dtype=np.int32)
    thr = np.full((nq, plan["n_splits"], 2), -np.inf, dtype=np.float32)
    sc[lo < 0] = np.nan  # unwritten lists: whatever the workspace held
    for q in range(nq):
        for s in range(plan["n_splits"]):
            if lo[q, s] < 0:
                continue
            for e in range(2):
                rows = np.arange(lo[q, s], hi[q, s])
                rows = rows[((rows >> 3) & 1) == e]
                best = rows[np.argsort(-S[q, rows], kind="stable")[:kph]]
                sc[q, s, e, :len(best)] = S[q, best]
                ids[q, s, e, :len(best)] = best
                if len(rows) >= kph:
                    thr[q, s, e] = S[q, best].min()
    return {**plan, "score": sc, "id": ids, "thr": thr}


@pytest.fixture(scope="module")
def case():
    X = grid(N, D, 1).astype(np.float64)
    Q = grid(NQ, D, 2).astype(np.float64)
    return Q, X, model_lists(Q, X, fl.IP)


def copy(res):
    return {k: (v.copy() if isinstance(v, np.ndarray) else v) for k, v in res.items()}


def test_model_lists_pass_both_ways(case):
    Q, X, res = case
    fl.check_lists(res, Q, X, fl.IP)
    fl.check_lists(res, Q, X, fl.IP, exact=True)
    Xg = X * np.linspace(0.5, 2.0, N)[:, None]  # unequal row norms: the per-row margins differ from the max-norm one
    fl.check_lists(model_lists(Q[:256], Xg, fl.L2), Q[:256], Xg, fl.L2)


def full_list(res, query):
    """(split, set) of a full list of `query` (thr > -inf)."""
    s, e = np.argwhere(res["thr"][query] > -np.inf)[0]
    return int(s), int(e)


def eps_of(Q, X, q):
    return PLAN["rel_eps"] * np.linalg.norm(Q[q]) * np.linalg.norm(X, axis=1).max()


def mutate_drop(res, Q, X):
    s, e = full_list(res, 300)
    res["id"][300, s, e, 0], res["score"][300, s, e, 0] = -1, -np.inf  # the best entry is gone


def mutate_lower_thr(res, Q, X):
    s, e = full_list(res, 300)
    res["thr"][300, s, e] -= 1.0  # grid scores are multiples of 1/4096 apart; discarded rows now sit above thr + eps


def mutate_other_set(res, Q, X):
    s, e = full_list(res, 300)
    res["id"][300, s, e, 3] ^= 8


def mutate_other_split(res, Q, X):
    res["id"][300, 0, 0, 3] += 512  # split 0 covers tiles [0, 2) of units 2 and 3, split 1 the rest


def mutate_duplicate(res, Q, X):
    s, e = full_list(res, 300)
    res["id"][300, s, e, 1], res["score"][300, s, e, 1] = res["id"][300, s, e, 0], res["score"][300, s, e, 0]


def mutate_score(res, Q, X):
    s, e = full_list(res, 300)
    res["score"][300, s, e, 2] += np.float32(2 * eps_of(Q, X, 300))


def mutate_first_phase(res, Q, X):
    res["id"][5, 1, 0, 0], res["score"][5, 1, 0, 0], res["thr"][5, 1, 0] = 8 * 2, 0.0, -np.inf  # unit 0 writes split 1


def mutate_ulp(res, Q, X):
    s, e = full_list(res, 300)
    res["score"][300, s, e, 4] = np.nextafter(res["score"][300, s, e, 4], np.float32(np.inf))


@pytest.mark.parametrize("mutate,exact,prop", [
    (mutate_drop, False, "discard bound"),
    (mutate_lower_thr, False, "discard bound"),
    (mutate_other_set, False, "partition"),
    (mutate_other_split, False, "partition"),
    (mutate_duplicate, False, "partition: query 300 holds a row id twice"),
    (mutate_score, False, "accuracy"),
    (mutate_first_phase, False, "first phase"),
    (mutate_ulp, True, "grid exactness"),
])
def test_checker_rejects_a_single_defect(case, mutate, exact, prop):
    Q, X, res = case
    bad = copy(res)
    mutate(bad, Q, X)
    with pytest.raises(AssertionError) as e:
        fl.check_lists(bad, Q, X, fl.IP, exact=exact, tag="model")
    assert prop in str(e.value), str(e.value)


def test_checker_rejects_top1_lists_out_of_order(case):
    Q, X, _ = case
    plan = {**PLAN, "units_whole": 0, "n_splits": 1}
    res = model_lists(Q[:128], X, fl.IP, plan)
    res["score"][:, :, :, 2:], res["id"][:, :, :, 2:] = -np.inf, -1  # top-2 layout: two entries, thr = third best
    S = fl.scores(Q[:128], X, fl.IP)
    for e in range(2):
        rows = np.arange(N)[((np.arange(N) >> 3) & 1) == e]
        res["thr"][:, 0, e] = -np.sort(-S[:, rows], axis=1)[:, 2]
    fl.check_lists(res, Q[:128], X, fl.IP, exact=True, top1=True)
    bad = copy(res)
    bad["score"][7, 0, 1, [0, 1]] = bad["score"][7, 0, 1, [1, 0]]
    bad["id"][7, 0, 1, [0, 1]] = bad["id"][7, 0, 1, [1, 0]]
    with pytest.raises(AssertionError, match="top1"):
        fl.check_lists(bad, Q[:128], X, fl.IP, exact=True, top1=True)
