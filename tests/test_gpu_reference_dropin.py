"""The drop-in claim itself: the reference's own, unmodified `sem_index` / `sem_sim_join` / `sem_search` /
`sem_dedup` / `sem_cluster_by` classes (lotus/sem_ops/*.py from oracle/_ref) run with `lotus.settings.configure(vs=B200VS())`
and reproduce the frames the same code produced over its own FaissVS (tests/golden/reference_ops.json). Own process: importing
the real `lotus` changes what lotus_b200 binds to (it then subclasses lotus.vector_store.VS)."""
import json
import os
import subprocess
import sys

import pytest

HERE = os.path.dirname(os.path.abspath(__file__))


@pytest.mark.gpu
def test_reference_operators_run_unmodified_over_b200vs(gpu):
    r = subprocess.run([sys.executable, os.path.join(HERE, "ref_dropin_worker.py")], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-3000:]
    res = json.loads(r.stdout.strip().splitlines()[-1])
    assert "unavailable" not in res, res  # build() makes oracle/_ref; a missing package is a packaging error, not a skip
    for name, v in res.items():
        if isinstance(v, bool):
            assert v, (name, res)
