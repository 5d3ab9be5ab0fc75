"""The clocked pod-list calls' derivation of the two timeout bits (include/ust.h, ust_clock), restated in clock_model and
pinned here without a device: at the boundaries of `now > start + timeout` with int64 wrap-around, against the
reference's own known answers (the "now-N" wait-start rule of pod_manager_test.go that the golden-vector encoder applies,
and the validation vectors' timed-out cases), and the ust_clock struct layout."""
import ctypes as C
import json
import os
import subprocess
import tempfile

import numpy as np
import pytest

import clock_model as cm
import helpers
from helpers import abi

I64_MAX, I64_MIN = np.iinfo(np.int64).max, np.iinfo(np.int64).min


def one(now, start, timeout):
    return bool(cm.timed_out(now, start, timeout)[0])


@pytest.mark.parametrize("timeout", [0, 1, 30, 600, 86_400])
@pytest.mark.parametrize("start", [0, 1_700_000_000, -5, -1_000_000_000_000])
def test_boundary(start, timeout):
    """now == start + timeout does not time out, one second later does; negative starts and timeout 0 included."""
    assert not one(start + timeout, start, timeout)
    assert one(start + timeout + 1, start, timeout)
    assert not one(start + timeout - 1, start, timeout)
    assert not one(start, start, timeout)


def test_timeout_zero():
    """TimeoutSecond == 0: any now after the start times out (the policy does not look at the bit then)."""
    assert one(11, 10, 0) and not one(10, 10, 0) and not one(9, 10, 0)


def test_extreme_starts_wrap():
    """Go int64: start + timeout wraps, so a start near INT64_MAX counts as timed out, and INT64_MIN is long ago."""
    assert one(0, I64_MAX, 1)                       # INT64_MAX + 1 wraps to INT64_MIN
    assert one(I64_MIN + 1, I64_MAX, 1)
    assert not one(I64_MIN, I64_MAX, 1)             # INT64_MIN > INT64_MIN is false
    assert not one(I64_MAX, I64_MAX, 0)
    assert one(0, I64_MAX, 600)
    assert one(0, I64_MIN, 600)                     # INT64_MIN + 600 is long ago
    assert not one(I64_MIN + 600, I64_MIN, 600)
    assert one(I64_MIN + 601, I64_MIN, 600)
    assert not one(I64_MIN, I64_MIN, 0)
    # a timeout that does not fit: TimeoutSecond is int64 too
    assert one(0, 1, I64_MAX)                       # 1 + INT64_MAX wraps to INT64_MIN
    assert not one(0, 0, I64_MAX)


def test_vectorised_equals_python_ints():
    """The numpy restatement against exact arithmetic reduced to int64, on random and extreme values."""
    rng = np.random.default_rng(7)
    ext = np.array([I64_MIN, I64_MIN + 1, -1, 0, 1, I64_MAX - 1, I64_MAX], np.int64)
    start = np.concatenate([rng.integers(I64_MIN, I64_MAX, 2000, dtype=np.int64), ext])
    for now in (I64_MIN, -7, 0, 1_700_000_000, I64_MAX):
        for timeout in (0, 30, 600, I64_MAX):
            got = cm.timed_out(now, start, timeout)
            wrap = [((int(s) + timeout + 2 ** 63) % 2 ** 64) - 2 ** 63 for s in start]
            assert np.array_equal(got, np.array([now > w for w in wrap])), (now, timeout)


def test_derive_reads_only_the_nodes_state_and_valid_annotations():
    rng = np.random.default_rng(3)
    n = 20_000
    soa, _ = helpers.random_soa(rng, n)
    start = rng.integers(-2000, 2000, n).astype(np.int64)
    now, T = 100, 30
    got = cm.derive(soa["state"], soa["flags"], start, now, T)
    code = soa["state"] & 15
    f = soa["flags"]
    other = (code != 3) & (code != 9)
    assert np.array_equal(got[other], f[other]), "other states keep their bits"
    assert np.array_equal(got & ~np.uint32(cm.TIMED_OUT), f & ~np.uint32(cm.TIMED_OUT)), "only bits 18 and 27 move"
    w = code == 3
    valid = w & ((f & cm.WAIT_BITS) == abi.UST_F_WAIT_START_ANNO)
    assert np.array_equal((got[w] & abi.UST_F_WAIT_TIMED_OUT) != 0, (valid & (now > start + T))[w])
    assert not np.any(got[w] & abi.UST_F_VALIDATION_TIMED_OUT)
    v = code == 9
    valid = v & ((f & cm.VAL_BITS) == abi.UST_F_VALIDATION_START_ANNO)
    assert np.array_equal((got[v] & abi.UST_F_VALIDATION_TIMED_OUT) != 0, (valid & (now > start + 600))[v])
    assert not np.any(got[v] & abi.UST_F_WAIT_TIMED_OUT)
    assert 0 < np.count_nonzero(got[w] & abi.UST_F_WAIT_TIMED_OUT) < np.count_nonzero(w)


@pytest.mark.parametrize("timeout", [0, 10, 100, 3600])
def test_wait_start_now_minus_n_rule(timeout):
    """The golden-vector encoder's "wait-start": "now-N" rule (tests/helpers.py, from pod_manager_test.go:183-229): timed
    out iff N > timeout. The model with start = now - N must set exactly the bit the encoder sets, at any now."""
    G = helpers.load_golden()
    pdict = {"waitForCompletion": {"timeoutSeconds": timeout}}
    ns = sorted({0, 1, timeout - 1, timeout, timeout + 1, 2 * timeout + 5, 10 ** 6} - {-1})
    nodes = [{"state": "wait-for-jobs-required", "ds": True, "anno": {"wait-start": f"now-{k}"},
              "pod": {"hash": G["daemonset_hash"], "phase": "Running", "containers": [[True, 0]]}} for k in ns]
    soa, _ = helpers.encode_nodes(nodes, G["daemonset_hash"], pdict)
    for now in (0, 1_700_000_000, -50):
        start = np.array([now - k for k in ns], np.int64)
        got = cm.derive(soa["state"], soa["flags"] & ~np.uint32(cm.TIMED_OUT), start, now, timeout)
        assert np.array_equal(got, soa["flags"]), (timeout, now, ns)


def test_validation_vectors_timed_out_cases():
    """validation_vectors.json encodes VALIDATION_TIMED_OUT the way validation_manager_test.go:125-136 makes it: a start of
    now - 605. With that start the model sets the bit exactly on the vectors' nodes that carry it; a start of now (set
    by the previous reconcile) never does; 600 seconds is the boundary."""
    with open(os.path.join(helpers.ROOT, "tests", "golden", "validation_vectors.json")) as f:
        vectors = json.load(f)["vectors"]
    seen = 0
    now = 1_700_000_000
    for v in vectors:
        for nd in v["nodes"]:
            if nd["state"] != "validation-required":
                continue
            bits = 0
            for b in nd["flags"]:
                bits |= abi.K["UST_F_" + b]
            timed = bool(bits & abi.UST_F_VALIDATION_TIMED_OUT)
            start = now - 605 if timed else now
            got = int(cm.derive(np.array([abi.UST_STATE_VALIDATION_REQUIRED], np.uint8),
                                np.array([bits & ~abi.UST_F_VALIDATION_TIMED_OUT], np.uint32), np.array([start]), now, 0)[0])
            assert bool(got & abi.UST_F_VALIDATION_TIMED_OUT) == (timed and not bits & abi.UST_F_VALIDATION_START_INVALID), v["name"]
            seen += timed
            edge = cm.derive(np.array([9, 9], np.uint8), np.array([abi.UST_F_VALIDATION_START_ANNO] * 2, np.uint32),
                             np.array([now - 600, now - 601]), now, 0)
            assert list(edge & abi.UST_F_VALIDATION_TIMED_OUT) == [0, abi.UST_F_VALIDATION_TIMED_OUT]
    assert seen >= 3


def test_clock_struct_layout():
    assert abi.UST_VALIDATION_TIMEOUT_SECONDS == 600
    src = ('#include <stdio.h>\n#include <stddef.h>\n#include "ust.h"\nint main(){printf("%zu %zu %zu %zu %zu\\n", sizeof(ust_clock),'
           ' offsetof(ust_clock, now), offsetof(ust_clock, wait_timeout_seconds), offsetof(ust_clock, start),'
           ' offsetof(ust_clock, insert_start));return 0;}')
    with tempfile.TemporaryDirectory() as d:
        c = os.path.join(d, "t.c")
        open(c, "w").write(src)
        exe = os.path.join(d, "t")
        subprocess.check_call(["gcc", "-I", os.path.dirname(abi.HEADER), c, "-o", exe])
        got = [int(x) for x in subprocess.check_output([exe]).split()]
    assert got == [C.sizeof(abi.Clock)] + [getattr(abi.Clock, f).offset for f, _ in abi.Clock._fields_]
    assert got == [32, 0, 8, 16, 24]
