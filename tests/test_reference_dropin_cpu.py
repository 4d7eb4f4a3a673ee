"""CPU dry run of the drop-in worker (tests/ref_dropin_worker.py): the REAL reference package (oracle/_ref, made by
build()) + lotus_b200.install() + the reference's unmodified operator classes over B200VS, with the native index
replaced by the oracle-backed fake. Checks the plumbing the GPU test relies on; the numbers come from the oracle here."""
import json
import os
import subprocess
import sys

import pytest

import refpkg

HERE = os.path.dirname(os.path.abspath(__file__))


def test_reference_operators_over_b200vs_plumbing():
    if refpkg.reference_dir() is None:
        pytest.skip("reference package not present (build() puts it under oracle/_ref)")
    r = subprocess.run([sys.executable, os.path.join(HERE, "ref_dropin_worker.py")], capture_output=True, text=True, timeout=600,
                       env=dict(os.environ, B2_TEST_FAKE_NATIVE="1"))
    assert r.returncode == 0, r.stderr[-3000:]
    res = json.loads(r.stdout.strip().splitlines()[-1])
    for name, v in res.items():
        if isinstance(v, bool):
            assert v, (name, res)
