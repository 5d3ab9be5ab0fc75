"""ApplyStateIncremental while nodes move in BuildState's list: driver pods re-created under new names, DaemonSet blocks
that swap places, full shuffles (tests/host/reorder_spec.hpp). Identical to ApplyState after every reconcile, one full
upload per scenario."""
import os
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _exe():
    sys.path.insert(0, ROOT)
    import __graft_entry__
    __graft_entry__.build()
    return os.path.join(ROOT, "tests", "host", "_build", "reorder_test")


def _run(args):
    p = subprocess.run([_exe()] + args, capture_output=True, text=True, timeout=600)
    out = p.stdout + p.stderr
    assert p.returncode == 0, out
    assert "not ok" not in out, out
    for tag in ("(a)", "(b)", "(c)", "(d)"):
        assert "ok " + tag in out, out
    return out


def test_reorders_host_halves_cpu():
    """The oracle behind the cache; the splice or reorder handed to the device is checked and replayed on the previous
    reconcile's arrays."""
    out = _run([])
    assert "ok the oracle-backed evaluation saw the reorders and splices it checked" in out, out


@pytest.mark.gpu
def test_reorders_on_gpu():
    """The same scenarios through ust_apply_state_delta_reorder / _splice on the H100."""
    _run(["--gpu"])
