"""sem_dedup's all-pairs kernel in both CTA modes — CTA pairs sharing each corpus tile through TMA multicast (the default)
and single CTAs (B2_PAIR_2CTA=0). The switch is read once per process -> subprocess, bounded by a timeout because
a barrier-protocol mistake would hang. Identical pair lists to the oracle, whole and sharded."""
import json
import os
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

SCRIPT = r"""
import json, os, sys
import numpy as np
sys.path.insert(0, %r); sys.path.insert(0, %r + "/tests")
import oracle
from helpers import gauss
from lotus_b200 import _native as nv
out = {}
for n, d, dtype in ((3000, 96, "bf16"), (3000, 96, "f32"), (257, 64, "bf16"), (1500, 200, "bf16")):
    x = gauss(n, d, 30 + n)
    rng = np.random.default_rng(n)
    src, dst = rng.choice(n, n // 20, replace=False), rng.choice(n, n // 20, replace=False)
    x[dst] = x[src] + 0.15 * gauss(len(src), d, 31 + n, normalize=False) / np.sqrt(d)
    x /= np.linalg.norm(x, axis=1, keepdims=True)
    if dtype == "bf16":
        xb = nv.f32_to_bf16_bits(x); idx, xf = nv.Index(xb, nv.BF16, 0), nv.bf16_bits_to_f32(xb)
    else:
        idx, xf = nv.Index(x, nv.F32, 0), x
    oi, oj, cnt = oracle.threshold_pairs(xf, 0.9)
    pi, pj = idx.threshold_pairs(0.9)
    res = {"pairs": int(cnt), "whole": bool(np.array_equal(pi, oi) and np.array_equal(pj, oj))}
    for group in ("4", "6", ""):
        if group: os.environ["B2_PAIR_GROUP"] = group
        else: os.environ.pop("B2_PAIR_GROUP", None)
        parts = [idx.threshold_pairs(0.9, part=p, nparts=3) for p in range(3)]
        owned = all((nv.pair_owner(a, 3) == p).all() for p, (a, _) in enumerate(parts))
        allp = sorted(zip(np.concatenate([p[0] for p in parts]).tolist(), np.concatenate([p[1] for p in parts]).tolist()))
        res["parts_" + (group or "default")] = bool(owned and allp == list(zip(oi.tolist(), oj.tolist())))
    os.environ.pop("B2_PAIR_GROUP", None)
    out[f"{n}x{d}_{dtype}"] = res
    idx.close()
print(json.dumps(out))
""" % (ROOT, ROOT)


@pytest.mark.gpu
@pytest.mark.parametrize("two_cta", ["1", "0"])
def test_pair_kernel_is_exact_in_both_cta_modes(two_cta):
    r = subprocess.run([sys.executable, "-c", SCRIPT], capture_output=True, text=True, timeout=300,
                       env=dict(os.environ, B2_PAIR_2CTA=two_cta))
    assert r.returncode == 0, r.stderr[-3000:]
    res = json.loads(r.stdout.strip().splitlines()[-1])
    for name, v in res.items():
        assert v["pairs"] > 5 and all(v[k] for k in v if k != "pairs"), (name, v)
