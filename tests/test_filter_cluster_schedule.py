"""The filter's schedule in clusters of four CTAs (knn_filter_sm90.cu make_sched / item_range), as the kernel deals it: workers
are CTA pairs taking query units of two tiles, and a cluster of four runs workers 2c and 2c + 1 in lockstep, so those two must
sweep the same corpus tiles item for item (their CTAs share every corpus tile by multicast). The host rounds the units cut into
splits up to an even number; the surplus unit lies past the last query tile. No GPU needed."""
import numpy as np
import pytest


def kernel_items(plan, nq, n, workers):
    """Per worker the (unit, split, t0, t1) of its items, dealt as the kernel deals them in clusters of four."""
    n_mtiles = -(-nq // 128)
    n_units = -(-n_mtiles // 2)
    s, uw = plan["n_splits"], plan["units_whole"]
    n_units += (n_units - uw) & 1  # launch_knn_filter: an even number of units cut into splits
    n_ntiles = -(-n // 256)
    tps = -(-n_ntiles // s)
    total = uw + (n_units - uw) * s
    out = [[] for _ in range(workers)]
    for item in range(total):
        if item < uw:
            unit, split, t0, t1 = item, 0, 0, n_ntiles
        else:
            j, rem = item - uw, n_units - uw
            unit, split = uw + j % rem, j // rem
            t0, t1 = split * tps, min(split * tps + tps, n_ntiles)
        out[item % workers].append((unit, split, t0, t1))
    return out, n_mtiles, n_ntiles


@pytest.mark.parametrize("num_sms", [132, 120])
@pytest.mark.parametrize("nq,n", [(100_000, 1_000_000), (20_000, 1_000_000), (40_000, 1_000_000), (40_000, 20_000),
                                  (20_352, 250_000), (700, 9_000), (520, 8_192), (801, 8_300), (512, 12_000)])
@pytest.mark.parametrize("k", [10, 32, 64])
def test_clusters_of_four_sweep_in_lockstep_and_cover_every_tile_once(nq, n, k, num_sms):
    from lotus_b200 import _native as nv
    plan = nv.filter_plan(nq, n, k, num_sms)
    assert plan["cluster"] == 4 and plan["two_cta"]
    workers = num_sms // 2
    assert workers % 2 == 0 and plan["units_whole"] % workers == 0
    per_worker, n_mtiles, n_ntiles = kernel_items(plan, nq, n, workers)
    for c in range(workers // 2):
        a, b = per_worker[2 * c], per_worker[2 * c + 1]
        assert len(a) == len(b), f"cluster {c}: {len(a)} and {len(b)} items"
        assert [(t0, t1) for _, _, t0, t1 in a] == [(t0, t1) for _, _, t0, t1 in b], f"cluster {c} sweeps different corpus tiles"
    # every real query tile meets every corpus tile exactly once; the surplus unit writes no list
    cover = np.zeros((n_mtiles, n_ntiles), dtype=np.int32)
    for items in per_worker:
        for unit, split, t0, t1 in items:
            assert t1 > t0 and 0 <= split < plan["n_splits"]
            for m in (2 * unit, 2 * unit + 1):
                if m < n_mtiles:
                    cover[m, t0:t1] += 1
    assert (cover == 1).all()


@pytest.mark.parametrize("nq,n,k", [(100_000, 1_024, 1), (100_000, 7_936, 10), (5_000, 4_096, 32)])
def test_short_corpora_keep_cta_pairs(nq, n, k):
    """Over fewer than 32 corpus tiles (the k-means second level searches the centroids) clusters of four were slower than
    pairs (DESIGN §5)."""
    from lotus_b200 import _native as nv
    plan = nv.filter_plan(nq, n, k)
    assert plan["cluster"] == 2 and plan["two_cta"]
