"""lotus_b200 — H100-native (sm_90a) backend for the embedding-similarity hot path of lotus-data/lotus:
`lotus.vector_store.FaissVS` + `sem_index / sem_search / sem_sim_join / sem_dedup / sem_cluster_by`.

    import lotus_b200 as lotus                      # same names as the reference for this path
    lotus.settings.configure(rm=rm, vs=lotus.B200VS())
    df.sem_index("text", "idx_dir").sem_sim_join(other, "a", "b", K=32)

With the real `lotus` package importable, call `lotus_b200.install()` instead: it imports lotus (whose import registers
the reference's accessors), plugs `B200VS` into `lotus.settings`, replaces `lotus.utils.cluster` and THEN re-registers this
package's accessors, so that `sem_dedup` / `sem_search` / `sem_cluster_by` reach the streaming kernels (every accessor here
falls back to the reference's control flow when the configured store is not a B200VS).
The compute lives in libb2lotus.so (include/lotus_b200.h); there is no CPU fallback.
"""
from . import utils
from .rm import RM, BagOfWordsRM, HashRM, TableRM
from .settings import settings
from .types import RMOutput
from .vs import METRIC_INNER_PRODUCT, METRIC_L2, VS, B200VS
from . import sem_ops  # noqa: F401  (registers the accessors)

__version__ = "0.1.0"


def install(vs: "B200VS | None" = None, **vs_kwargs):
    """Make B200VS the vector store of whichever settings object the operators read (the real lotus.settings when
    lotus is importable, ours otherwise) and route lotus.utils.cluster to the device k-means."""
    store = vs if vs is not None else B200VS(**vs_kwargs)
    try:
        import lotus as _ref  # type: ignore  (registers the reference's accessors: must come BEFORE register_all)
        import lotus.utils as _ref_utils  # type: ignore
    except Exception:
        _ref = None
    if _ref is not None:
        _ref.settings.configure(vs=store)
        _ref_utils.cluster = utils.cluster  # sem_cluster_by.py:74 resolves lotus.utils.cluster at call time
        _ref.utils = _ref_utils
    else:
        settings.configure(vs=store)
    sem_ops.register_all()
    return store


__all__ = ["RM", "BagOfWordsRM", "HashRM", "TableRM", "VS", "B200VS", "RMOutput", "settings", "utils", "install",
           "METRIC_INNER_PRODUCT", "METRIC_L2"]
