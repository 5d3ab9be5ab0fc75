"""ClusterUpgradeStateManagerImpl::NextTimeout (tests/host/deadline_test.cpp). CPU: the value EvaluateCachedPods supplies is
carried out of ApplyStateIncremental with the on-device options, and nowhere else. GPU: a reconcile loop that sleeps until
NextTimeout() whenever a reconcile changed no object, with a twin manager one second before each deadline, in-place and
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
    return os.path.join(ROOT, "tests", "host", "_build", "deadline_test")


def _run(args):
    p = subprocess.run([_exe()] + args, capture_output=True, text=True, timeout=1800)
    out = p.stdout + p.stderr
    assert p.returncode == 0, out
    assert "not ok" not in out, out
    assert "0 failed" in out, out
    return out


def test_next_timeout_host_halves_cpu():
    out = _run([])
    assert "ok NextTimeout carries EvaluateCachedPods' deadline out of ApplyStateIncremental, and only from a clocked call" in out, out
    assert "ok NextTimeout is nullopt without WaitForCompletionOnDevice and ValidateOnDevice" in out, out


@pytest.mark.gpu
def test_next_timeout_on_gpu():
    out = _run(["--gpu"])
    for mode in ("in-place", "requestor"):
        for validate in ("off", "on"):
            assert ("ok a reconcile loop that sleeps until NextTimeout() makes the reference's calls, and a twin one second before "
                    f"each deadline changes nothing ({mode} mode, ValidateOnDevice {validate})") in out, out
