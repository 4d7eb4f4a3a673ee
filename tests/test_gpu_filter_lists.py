"""The filter kernel's candidate lists against fp64 scores of the exact operands, list by list (tests/filter_lists.py), in both
CTA modes: CTA pairs (the default) and single CTAs (B2_FILTER_2CTA=0). The search's certificate and dense fallback hide most
filter defects from the end-to-end tests (a wrong operand or a skipped tile only costs speed); these checks do not.

The mode switch is read once per process, so each mode runs the whole case matrix in a subprocess, bounded by a timeout. The
largest measured |err| / (|q| |x| rel_eps) per (filter operand, input rounding, d) is printed (pytest -s shows it)."""
import json
import os
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

SCRIPT = r"""
import json, sys
sys.path.insert(0, %r); sys.path.insert(0, %r + "/tests")
import filter_lists
from lotus_b200 import _native as nv
print(json.dumps(filter_lists.run_matrix(nv)))
""" % (ROOT, ROOT)


@pytest.mark.gpu
@pytest.mark.parametrize("two_cta", ["1", "0"])
def test_filter_lists_hold_the_certificate_premises(gpu, two_cta):
    r = subprocess.run([sys.executable, "-c", SCRIPT], capture_output=True, text=True, timeout=900,
                       env=dict(os.environ, B2_FILTER_2CTA=two_cta))
    assert r.returncode == 0, r.stderr[-3000:]
    res = json.loads(r.stdout.strip().splitlines()[-1])
    print(f"\nB2_FILTER_2CTA={two_cta}: {res['cases']} cases; largest |err| / (|q| |x| rel_eps):")
    for key, v in sorted(res["ratios"].items()):
        print(f"  {key:40s} {v:.4f}")
    assert not res["failures"], "\n".join(res["failures"])
    assert len(res["plans"]) == res["cases"]
    # the switch reached the kernel: CTA pairs wherever there are two query tiles, or never
    assert any(p["two_cta"] for p in res["plans"]) == (two_cta == "1")
