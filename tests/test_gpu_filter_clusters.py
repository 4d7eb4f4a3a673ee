"""The filter kernel's candidate lists in clusters of four CTAs (corpora of 32 tiles or more), against fp64 scores of the exact
operands (tests/filter_lists.py), at the shapes where the cluster schedule has edges: 4 to 7 query tiles (the last unit or the last
cluster holds tiles past the batch, which load zeros and write no list) and multi-cluster two-phase shapes whose units cut into
splits are odd in number (the host adds a surplus unit). Both CTA modes, each in a subprocess (the switch is read once)."""
import json
import os
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

SCRIPT = r"""
import json, sys
sys.path.insert(0, %r); sys.path.insert(0, %r + "/tests")
import filter_lists as fl
from lotus_b200 import _native as nv
CASES = [  # (metric, n, d, nq, k, data)
    (fl.IP, 8193, 96, 512, 10, "gauss"), (fl.L2, 8200, 96, 520, 10, "unnorm"), (fl.IP, 8449, 96, 700, 10, "cancel"),
    (fl.L2, 8192, 96, 801, 10, "grid"), (fl.IP, 8456, 64, 20_000, 10, "gauss"), (fl.IP, 9000, 48, 19_200, 32, "grid"),
    (fl.L2, 8289, 40, 20_352, 5, "gauss"),
]
failures, plans = [], []
for ci, (metric, n, d, nq, k, data) in enumerate(CASES):
    x, q = fl.make_data(data, n, nq, d, 2000 + ci)
    xs, qs = nv.f32_to_bf16_bits(x), nv.f32_to_bf16_bits(q)
    X, Q = nv.bf16_bits_to_f32(xs).astype("float64"), nv.bf16_bits_to_f32(qs).astype("float64")
    idx = nv.Index(xs, fl.BF16, metric)
    try:
        res = idx.filter_lists(qs, k, fl.BF16)
    finally:
        idx.close()
    plans.append({key: res[key] for key in ("n_splits", "units_whole", "cluster")})
    try:
        assert res["use_filter"], f"case {ci}: the plan does not use the filter"
        fl.check_lists(res, Q, X, metric, exact=data == "grid", tag=f"cluster case {ci} [nq={nq} n={n} d={d} k={k} {data}]")
    except AssertionError as e:
        failures.append(str(e))
print(json.dumps({"failures": failures, "plans": plans}))
""" % (ROOT, ROOT)


@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["1", "0"])
def test_cluster_edge_shapes_hold_the_certificate_premises(gpu, mode):
    r = subprocess.run([sys.executable, "-c", SCRIPT], capture_output=True, text=True, timeout=900,
                       env=dict(os.environ, B2_FILTER_2CTA=mode))
    assert r.returncode == 0, r.stderr[-3000:]
    res = json.loads(r.stdout.strip().splitlines()[-1])
    print(f"\nB2_FILTER_2CTA={mode}: plans {res['plans']}")
    assert not res["failures"], "\n".join(res["failures"])
    assert all(p["cluster"] == (4 if mode == "1" else 1) for p in res["plans"])
    if mode == "1":  # the two-phase shapes include one whose units cut into splits are odd in number
        assert any(p["units_whole"] > 0 and p["n_splits"] > 1 for p in res["plans"])
