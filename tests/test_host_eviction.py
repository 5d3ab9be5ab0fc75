"""StateOptions::EvictionOnDevice: PodManager.SchedulePodEviction and DrainManager.ScheduleNodesDrain decided on the device
(tests/host/eviction_spec.hpp). CPU: what Encode and ApplyStateIncremental hand to the device (every pod of a
pod-deletion-required or drain-required node with its filter-chain bits, after the validation and wait pods; changed parts
only), Replay's calls for every outcome of passes 5 and 6 on a copy of the node with errors dropped, the dedupe sets and
the Lists' errors. GPU: the reference's pod-eviction and drain specs, the host's "nothing to delete" against the device's
outcome, and a reconcile loop against the restated PodManagerImpl and DrainManagerImpl, in-place and requestor mode, with
the other two on-device options off and on."""
import os
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _exe():
    sys.path.insert(0, ROOT)
    import __graft_entry__
    __graft_entry__.build()
    return os.path.join(ROOT, "tests", "host", "_build", "eviction_test")


def _run(args):
    p = subprocess.run([_exe()] + args, capture_output=True, text=True, timeout=1800)
    out = p.stdout + p.stderr
    assert p.returncode == 0, out
    assert "not ok" not in out, out
    assert "0 failed" in out, out
    return out


def test_eviction_host_halves_cpu():
    out = _run([])
    assert "ok Encode: workload entries for pod-deletion-required and drain-required nodes only, each bit from its source" in out, out
    assert ("ok Encode with ValidateOnDevice and WaitForCompletionOnDevice too: validation pods, then wait pods, then workload "
            "pods") in out, out
    assert ("ok ApplyStateIncremental hands down only changed workload parts, nothing for an unchanged node, and drops them on "
            "leaving") in out, out
    assert ("ok Replay, pass 5: nothing to delete, a mismatch with drain on and off, evict OK and evict failure; on a copy, "
            "errors dropped") in out, out
    assert ("ok Replay, pass 6: cordon, then evict, then the state; cordon failure, drain error status and evict failure give "
            "upgrade-failed") in out, out
    assert "ok Dedupe: a node whose eviction or drain is still running gets no second call and no state change" in out, out
    assert "ok Replay: a failed pod or DaemonSet List returns at the pass it serves, only when that pass has nodes" in out, out


@pytest.mark.gpu
def test_eviction_on_gpu():
    out = _run(["--gpu"])
    assert "ok standalone gpu pods with force are deleted: pod-restart-required (pod_manager_test.go:236)" in out, out
    assert "ok DrainManager should drain nodes (drain_manager_test.go:33)" in out, out
    assert "ok on a C4-like snapshot the host's 'nothing to delete' agrees with the device on every pod-deletion-required node" in out, out
    for mode in ("in-place", "requestor"):
        for others in ("off", "on"):
            assert ("ok ApplyStateIncremental with EvictionOnDevice == ApplyState with PodManagerImpl and DrainManagerImpl over a "
                    f"reconcile loop ({mode} mode, the other two options {others})") in out, out
