"""The definition a range search must match bit for bit: faiss IndexFlat.range_search restated over the oracle's canonical
scorer. IP keeps row j when its canonical fp32 score is strictly greater than the radius, L2 when its canonical fp32 squared
distance is strictly less (faiss's RangeSearchBlockResultHandler, as read from upstream). Output in the layout of faiss's
Python range_search: lims[nq+1], D[lims[nq]], I[lims[nq]], each query's hits in ascending row id; with ids, a temporary
index over x[ids] (faiss_vs.py:57-72): hits in the order of positions in ids, reported as ids[position]."""
import numpy as np

import oracle


def range_search(x, q, radius, metric=oracle.IP, ids=None):
    x = np.ascontiguousarray(x, dtype=np.float32)
    q = np.ascontiguousarray(q, dtype=np.float32)
    ids = None if ids is None else np.asarray(ids, dtype=np.int64)
    sub = x if ids is None else np.ascontiguousarray(x[ids]).reshape(len(ids), x.shape[1])
    nq = q.shape[0]
    if nq == 0 or sub.shape[0] == 0:
        return np.zeros(nq + 1, np.int64), np.empty(0, np.float32), np.empty(0, np.int64)
    S = oracle.scores(sub, q, metric, scorer=oracle.CANONICAL)
    r = np.float32(radius)
    hit = S > r if metric == oracle.IP else S < r
    qi, pos = np.nonzero(hit)  # row-major: by query, then ascending position
    lims = np.zeros(nq + 1, np.int64)
    np.cumsum(hit.sum(axis=1), out=lims[1:])
    return lims, S[qi, pos].astype(np.float32), (pos if ids is None else ids[pos]).astype(np.int64)
