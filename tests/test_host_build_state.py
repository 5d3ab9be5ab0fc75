"""The incremental reconcile loop: BuildStateIncremental + ApplyStateIncremental on one manager against BuildState +
ApplyState on a fresh one, over 300 reconciles of a cluster whose pods change phase and get scheduled, whose nodes join and
leave, whose driver pods come back under new names and whose DaemonSet is re-created (tests/host/build_state_spec.hpp).
Identical after every reconcile; one full upload of the driver-pod list and one of ApplyState's snapshot in the whole run."""
import os
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _exe():
    sys.path.insert(0, ROOT)
    import __graft_entry__
    __graft_entry__.build()
    return os.path.join(ROOT, "tests", "host", "_build", "build_state_test")


def _run(args):
    p = subprocess.run([_exe()] + args, capture_output=True, text=True, timeout=1200)
    out = p.stdout + p.stderr
    assert p.returncode == 0, out
    assert "not ok" not in out, out
    assert "ok BuildStateIncremental + ApplyStateIncremental == BuildState + ApplyState" in out, out
    return out


def test_build_state_loop_host_halves_cpu():
    """The oracle behind BuildState's device call and both caches; the runs and overwrites handed to the device are checked
    and replayed on the previous reconcile's arrays."""
    out = _run([])
    assert "ok the oracle-backed evaluation saw the reorders and sparse patches it checked" in out, out


@pytest.mark.gpu
def test_build_state_loop_on_gpu():
    """The same loop through ust_build_state_uids / ust_build_state_delta and the ApplyState entry points on the H100."""
    _run(["--gpu"])
