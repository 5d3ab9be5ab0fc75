"""StateOptions::WaitForCompletionOnDevice: PodManager.ScheduleCheckOnPodCompletion answered on the device
(tests/host/wait_spec.hpp). CPU: what Encode and ApplyStateIncremental hand to the device (wait pods with their phases, after
the validation pods; start times and bits; replaced lists; nothing for a time-only reconcile) and Replay's pass-4 call
orders, swallowed errors and List error. GPU: the reference's wait-for-completion specs, the host's running bit against the
device's outcome, a time-only reconcile, and a reconcile loop against the restated PodManagerImpl, in-place and requestor
mode, with ValidateOnDevice off and on."""
import os
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _exe():
    sys.path.insert(0, ROOT)
    import __graft_entry__
    __graft_entry__.build()
    return os.path.join(ROOT, "tests", "host", "_build", "wait_test")


def _run(args):
    p = subprocess.run([_exe()] + args, capture_output=True, text=True, timeout=1800)
    out = p.stdout + p.stderr
    assert p.returncode == 0, out
    assert "not ok" not in out, out
    assert "0 failed" in out, out
    return out


def test_wait_host_halves_cpu():
    out = _run([])
    assert "ok Encode: one wait List, every node's wait pods with their phases, the start column and the WAIT_START bits" in out, out
    assert "ok Encode with ValidateOnDevice too: two Lists, validation pods first, a pod both selectors match in the list twice" in out, out
    assert "ok ApplyStateIncremental hands down only the changed lists and nodes, and nothing on a time-only reconcile" in out, out
    assert "ok Replay, pass 4: finished = delete, then state; timed out = state, then delete; no start time = set it to now" in out, out
    assert "ok Replay, pass 4: the calls get a copy of the node, and the snapshot's node object is left alone" in out, out
    assert "ok Replay, pass 4: provider errors are swallowed; a failed delete suppresses the state change on the finished path only" in out, out
    assert "ok Replay: a failed List returns at the wait-for-jobs pass (index 4) when it has nodes, and is no error otherwise" in out, out


@pytest.mark.gpu
def test_wait_on_gpu():
    out = _run(["--gpu"])
    assert "ok 200 wait-for-jobs-required nodes: one List, not 200" in out, out
    assert "ok the host's running bit agrees with the device's outcome on every wait-for-jobs-required node" in out, out
    assert "ok a reconcile in which only time passed sends nothing and returns exactly the nodes whose wait deadline passed" in out, out
    for mode in ("in-place", "requestor"):
        for validate in ("off", "on"):
            assert ("ok ApplyStateIncremental with WaitForCompletionOnDevice == ApplyState with PodManagerImpl over a reconcile loop "
                    f"({mode} mode, ValidateOnDevice {validate})") in out, out
