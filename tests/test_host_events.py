"""The events of the managers the three on-device options replace (tests/host/events_spec.hpp). CPU: GetEventReason, the
drain's aggregate error, and Replay of hand-made outputs for every row of the events table, with the event's type, reason,
message and place among the node's calls; a null recorder leaves the calls as they were; with the options off the mirror
records nothing. GPU: the reference's eviction, drain, wait and validation cases with a recorder against the restated
managers, and reconcile loops with injected failures, in-place and requestor mode, each option alone and all three."""
import os
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _exe():
    sys.path.insert(0, ROOT)
    import __graft_entry__
    __graft_entry__.build()
    return os.path.join(ROOT, "tests", "host", "_build", "events_test")


def _run(args):
    p = subprocess.run([_exe()] + args, capture_output=True, text=True, timeout=1800)
    out = p.stdout + p.stderr
    assert p.returncode == 0, out
    assert "not ok" not in out, out
    assert "0 failed" in out, out
    return out


def test_events_host_halves_cpu():
    out = _run([])
    assert "ok GetEventReason is the upper-cased driver name + DriverUpgrade" in out, out
    assert "ok the drain's aggregate error: one message, several messages in first-pod order, a missing DaemonSet" in out, out
    assert "ok Replay: every row of the events table, its type, reason, message and place among the node's calls" in out, out
    assert "ok a null recorder leaves every call as it was; with the options off the mirror records nothing" in out, out


@pytest.mark.gpu
def test_events_on_gpu():
    out = _run(["--gpu"])
    assert "ok events: DrainManager should drain nodes (drain_manager_test.go:33)" in out, out
    assert "ok events: wait checks: start set, timed out, done, unparsable, failing writes" in out, out
    assert "ok events: validation: the start time does not parse" in out, out
    for opts in ("all three options", "ValidateOnDevice alone", "WaitForCompletionOnDevice alone", "EvictionOnDevice alone"):
        for mode in ("in-place", "requestor"):
            assert (f"ok ApplyStateIncremental with {opts} records the events ApplyState with the restated managers records "
                    f"({mode} mode)") in out, out
    assert "ok every row of the events table fired in the loops" in out, out
