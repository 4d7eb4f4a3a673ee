"""The knn filter keeps the first K-blocks of each query tile in registers for a whole item and loads only the corpus operand
for them after the item's first tile (knn_filter_sm90.cu, FILTER_RES_KB = 6). Checked list by list against fp64 scores of the
exact operands (tests/filter_lists.py) where that protocol has edges: d with fewer, exactly as many and one more K-block than
are resident (bf16 / fp16: 32 elements per K-block, tf32: 16), items of a single corpus tile, items that start past the first
tile of the corpus (later splits, the second phase of a two-phase schedule), and the k-means TOP1 variant. bf16, fp16 and
tf32 operands, IP and L2, CTA pairs and clusters of four (corpora of 32 tiles or more), and single CTAs; each CTA mode in a
subprocess (the switch is read once)."""
import json
import os
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

SCRIPT = r"""
import json, sys
import numpy as np
sys.path.insert(0, %r); sys.path.insert(0, %r + "/tests")
import filter_lists as fl
from lotus_b200 import _native as nv
F16 = nv.F16
CASES = [  # (store, level, top1, metric, n, d, nq, k, data); kb = K-blocks per tile
    (fl.BF16, 0, False, fl.IP, 512, 8, 300, 41, "gauss"),       # kb 1; two splits of one tile each
    (fl.BF16, 0, False, fl.L2, 769, 30, 129, 100, "grid"),      # kb 1; four splits of one tile each
    (fl.BF16, 0, False, fl.IP, 9000, 192, 700, 50, "gauss"),    # kb 6 = resident; clusters of four, two splits
    (fl.BF16, 0, False, fl.L2, 8449, 200, 520, 10, "grid"),     # kb 7; clusters of four, a last tile of one row
    (fl.BF16, 0, False, fl.IP, 8456, 64, 20_000, 10, "unnorm"), # kb 2; two-phase schedule
    (fl.F32, 1, False, fl.IP, 8300, 96, 600, 45, "gauss"),      # tf32 kb 6 = resident; clusters of four
    (fl.F32, 1, False, fl.L2, 1289, 8, 257, 5, "grid"),         # tf32 kb 1
    (fl.F32, 1, False, fl.IP, 2048, 100, 383, 41, "unnorm"),    # tf32 kb 7; two splits
    (F16, 0, False, fl.IP, 8456, 160, 20_000, 10, "gauss"),     # fp16 kb 5; two-phase schedule
    (F16, 0, False, fl.L2, 700, 192, 129, 64, "grid"),          # fp16 kb 6; two splits
    (F16, 0, False, fl.L2, 2056, 224, 383, 32, "cancel"),       # fp16 kb 7
    (fl.BF16, 0, True, fl.L2, 1024, 30, 383, 1, "neardup"),     # TOP1, kb 1
    (fl.F32, 0, True, fl.IP, 1289, 96, 257, 1, "grid"),         # TOP1 tf32, kb 6
    (F16, 0, True, fl.L2, 300, 200, 129, 1, "gauss"),           # TOP1 fp16, kb 7; two corpus tiles
]
failures, plans = [], []
for ci, (store, level, top1, metric, n, d, nq, k, data) in enumerate(CASES):
    x, q = fl.make_data(data, n, nq, d, 3000 + ci)
    if store == fl.BF16:
        xs, qs = nv.f32_to_bf16_bits(x), nv.f32_to_bf16_bits(q)
        X, Q = nv.bf16_bits_to_f32(xs), nv.bf16_bits_to_f32(qs)
    elif store == F16:
        xs, qs = x.astype(np.float16), q.astype(np.float16)
        X, Q = xs.astype(np.float32), qs.astype(np.float32)
    else:
        xs, qs, X, Q = x, q, x, q
    tag = f"case {ci} [store {store} level {level}{' top1' if top1 else ''} {'L2' if metric else 'IP'} n={n} d={d} nq={nq} k={k} {data}]"
    idx = nv.Index(xs, store, metric)
    try:
        res = idx.filter_lists(qs, k, store, top1=top1, level=level)
    finally:
        idx.close()
    plans.append({"case": ci, **{key: res[key] for key in ("n_splits", "units_whole", "cluster", "filt_dtype", "two_level")}})
    try:
        assert res["use_filter"], f"{tag}: the plan does not use the filter"
        assert res["filt_dtype"] == store and not res["two_level"], f"{tag}: plan {plans[-1]}"
        fl.check_lists(res, Q.astype(np.float64), X.astype(np.float64), metric, exact=data == "grid", top1=top1, tag=tag)
    except AssertionError as e:
        failures.append(str(e))
print(json.dumps({"failures": failures, "plans": plans}))
""" % (ROOT, ROOT)


@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["1", "0"])
def test_resident_query_kblocks_hold_the_certificate_premises(gpu, mode):
    r = subprocess.run([sys.executable, "-c", SCRIPT], capture_output=True, text=True, timeout=900,
                       env=dict(os.environ, B2_FILTER_2CTA=mode))
    assert r.returncode == 0, r.stderr[-3000:]
    res = json.loads(r.stdout.strip().splitlines()[-1])
    print(f"\nB2_FILTER_2CTA={mode}: plans {res['plans']}")
    assert not res["failures"], "\n".join(res["failures"])
    clusters = {p["cluster"] for p in res["plans"]}
    assert clusters == ({2, 4} if mode == "1" else {1}), f"CTA modes reached: {clusters}"
    assert any(p["n_splits"] > 1 for p in res["plans"]) and any(p["units_whole"] > 0 for p in res["plans"])
