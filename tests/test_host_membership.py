"""ApplyStateIncremental while nodes leave, join anywhere in BuildState's list and rejoin under old names
(tests/host/membership_spec.hpp): identical to ApplyState after every reconcile, one full upload in the whole run."""
import os
import re
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _exe():
    sys.path.insert(0, ROOT)
    import __graft_entry__
    __graft_entry__.build()
    return os.path.join(ROOT, "tests", "host", "_build", "membership_test")


def _run(args):
    p = subprocess.run([_exe()] + args, capture_output=True, text=True, timeout=600)
    out = p.stdout + p.stderr
    assert p.returncode == 0, out
    assert "not ok" not in out, out
    assert "ok ApplyStateIncremental == ApplyState while nodes leave" in out, out
    assert "1 full uploads" in out, out
    return out


def test_membership_changes_host_halves_cpu():
    """The oracle behind the cache; the splice handed to the device is replayed on the previous reconcile's arrays."""
    out = _run([])
    assert "ok the oracle-backed evaluation saw the splices it checked" in out, out


@pytest.mark.gpu
def test_membership_changes_on_gpu():
    """The same scenarios through ust_apply_state_delta_splice on the H100."""
    out = _run(["--gpu"])
    # the node pool overflowed the sparse outputs, and the aborting reconcile fetched the full outputs
    m = re.search(r"node pool: 1 full uploads, (\d+) inserted, (\d+) outputs received", out)
    assert m and int(m.group(2)) >= int(m.group(1)), out
