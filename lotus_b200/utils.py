"""`cluster(col_name, ncentroids)` — lotus/utils.py:14-72: returns the function that k-means-clusters a frame's
indexed column and yields one cluster id per row. The reference calls faiss.Kmeans(d, k, niter, verbose).train(x)
then kmeans.index.search(x, 1) (:61-65); here both run on the GPU through `vs.kmeans`."""
from __future__ import annotations

from typing import Callable

import pandas as pd

from .sem_ops._common import resolve_rm_vs


def cluster(col_name: str, ncentroids: int) -> Callable[..., list[int]]:
    def ret(df: pd.DataFrame, niter: int = 20, verbose: bool = False, method: str = "kmeans") -> list[int]:
        if col_name not in df.columns:
            raise ValueError(f"Column {col_name} not found in DataFrame")
        if ncentroids > len(df):
            raise ValueError(f"Number of centroids must be less than number of documents. {ncentroids} > {len(df)}")
        rm, vs = resolve_rm_vs()
        try:
            col_index_dir = df.attrs["index_dirs"][col_name]
        except KeyError:
            raise ValueError(f"Index directory for column {col_name} not found in DataFrame")
        if vs.index_dir != col_index_dir:
            vs.load_index(col_index_dir)
        assert vs.index_dir == col_index_dir
        ids = df.index.tolist()  # assumes df index hasn't been reset and corresponds to index positions (utils.py:58)
        if not hasattr(vs, "kmeans"):
            # some other VS (e.g. the reference's FaissVS): the reference's own code path, faiss included (utils.py:32,59-70)
            import faiss  # type: ignore
            vec_set = vs.get_vectors_from_index(col_index_dir, ids)
            km = faiss.Kmeans(vec_set.shape[1], ncentroids, niter=niter, verbose=verbose)
            km.train(vec_set)
            _scores, indices = km.index.search(vec_set, 1)
            return indices.flatten()
        assign, _centroids, obj = vs.kmeans(ids, ncentroids, niter=niter)
        if verbose:
            for it, o in enumerate(obj):
                print(f"  Iteration {it} objective={float(o):g}")
        return assign  # ndarray int64, like `indices.flatten()` (utils.py:70)

    return ret
