"""StateOptions::ValidateOnDevice: ValidationManager.Validate answered on the device (tests/host/validation_spec.hpp).
CPU: what Encode and ApplyStateIncremental hand to the device (validation pods in List order, start times and bits, replaced
lists, runs, nothing for a time-only reconcile) and Replay's pass-10 call orders and errors. GPU: the reference's Validate
cases and validation ApplyState specs, and a reconcile loop against the restated ValidationManagerImpl, in-place and
requestor mode."""
import os
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _exe():
    sys.path.insert(0, ROOT)
    import __graft_entry__
    __graft_entry__.build()
    return os.path.join(ROOT, "tests", "host", "_build", "validation_test")


def _run(args):
    p = subprocess.run([_exe()] + args, capture_output=True, text=True, timeout=1200)
    out = p.stdout + p.stderr
    assert p.returncode == 0, out
    assert "not ok" not in out, out
    assert "0 failed" in out, out
    return out


def test_validation_host_halves_cpu():
    out = _run([])
    assert "ok ApplyStateIncremental hands down only what changed" in out, out
    assert "ok Replay, pass 10: a provider error returns at its call" in out, out


@pytest.mark.gpu
def test_validation_on_gpu():
    out = _run(["--gpu"])
    assert "ok ApplyStateIncremental with ValidateOnDevice == ApplyState with ValidationManagerImpl over a reconcile loop (in-place mode)" in out, out
    assert "ok ApplyStateIncremental with ValidateOnDevice == ApplyState with ValidationManagerImpl over a reconcile loop (requestor mode)" in out, out
    assert "ok a reconcile in which only time passed sends nothing" in out, out
