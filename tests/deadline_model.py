"""The next deadline of a clocked pod-list call (include/ust.h, ust_next_deadline), found without the device: the smallest
t > now at which a time-only reconcile returns something, or INT64_MIN (abi.NO_DEADLINE).

`brute_force` follows the definition literally: it collects the times d + 1 at which some node's timed-out bit turns on
(d = start + timeout with Go's int64 wrap, clock_model), runs the unclocked ApplyState with bits 18 and 27 derived for each
such time in order, and returns the first time whose outputs differ from those at `now`.

`apply(policy, soa, pods)` is the unclocked ApplyState that serves as the reference: by default the CPU oracle, with
validation_model's restatement of the validation pass when the policy asks for UST_EVAL_VALIDATION (`reference_apply`).

`flip_model` uses that each of the two bits depends on its own node only: it runs ApplyState twice - at `now`, and with the
bit of every candidate node set at once - and takes the smallest d + 1 over the candidates whose outputs differ. Two calls
instead of one per candidate time, so it also serves snapshots of millions of nodes (with the unclocked device call as
`apply`); the CPU tests check it against the brute force."""
import numpy as np

import clock_model as cm
import helpers
import validation_model as vm
from helpers import abi

I64 = np.iinfo(np.int64)
NONE = abi.NO_DEADLINE


def reference_apply(pol, soa, pods):
    """The CPU reference of an unclocked ApplyState with pod lists (rc, next_state, actions, outcome, counters)."""
    if pol.evaluate_actuators & abi.UST_EVAL_VALIDATION:
        return vm.apply(pol, soa, pods)
    return helpers.oracle_apply(pol, soa, pods)


def candidates(state, flags, start, now, wait_timeout):
    """(mask, d): the nodes whose bit is clear at `now` and turns on at d + 1 > now - wait-for-jobs-required or
    validation-required with the state's start annotation present and parsable, now <= d < INT64_MAX - and every node's d."""
    code = np.asarray(state, np.uint8) & np.uint8(abi.UST_HOT_STATE_MASK)
    flags = np.asarray(flags, np.uint32)
    start = np.asarray(start, np.int64)
    wait = code == abi.UST_STATE_WAIT_FOR_JOBS_REQUIRED
    val = code == abi.UST_STATE_VALIDATION_REQUIRED
    ok = (wait & ((flags & np.uint32(cm.WAIT_BITS)) == abi.UST_F_WAIT_START_ANNO)) | \
        (val & ((flags & np.uint32(cm.VAL_BITS)) == abi.UST_F_VALIDATION_START_ANNO))
    timeout = np.where(wait, np.uint64(int(wait_timeout) & 0xFFFFFFFFFFFFFFFF), np.uint64(abi.UST_VALIDATION_TIMEOUT_SECONDS))
    d = (start.view(np.uint64) + timeout).view(np.int64)
    return ok & (d >= np.int64(now)) & (d != I64.max), d


def _outputs(apply, pol, soa, pods, start, t, wait_timeout):
    r = apply(pol, cm.derived_soa(soa, start, t, wait_timeout), pods)
    return r[1], r[2], r[3]


def _differ(a, b):
    return (a[0] != b[0]) | (a[1] != b[1]) | (a[2] != b[2])


def brute_force(pol, soa, pods, start, now, wait_timeout, apply=reference_apply):
    """The definition: the first candidate time whose outputs differ from the outputs at `now`."""
    m, d = candidates(soa["state"], soa["flags"], start, now, wait_timeout)
    ref = _outputs(apply, pol, soa, pods, start, now, wait_timeout)
    for t in sorted({int(x) + 1 for x in d[m]}):
        if _differ(ref, _outputs(apply, pol, soa, pods, start, t, wait_timeout)).any():
            return t
    return NONE


def flip_model(pol, soa, pods, start, now, wait_timeout, apply=reference_apply):
    """(next deadline, d + 1 per node, mask of the nodes whose outputs change when their bit turns on). The nodes that fire
    at the next deadline T are those of the mask with d + 1 == T."""
    m, d = candidates(soa["state"], soa["flags"], start, now, wait_timeout)
    at = np.full(d.shape, I64.max, np.int64)
    at[m] = d[m] + 1
    if not m.any():
        return NONE, at, m
    s0 = cm.derived_soa(soa, start, now, wait_timeout)
    a = apply(pol, s0, pods)
    s1 = dict(s0)
    wait = (soa["state"] & 15) == abi.UST_STATE_WAIT_FOR_JOBS_REQUIRED
    bit = np.where(wait, np.uint32(abi.UST_F_WAIT_TIMED_OUT), np.uint32(abi.UST_F_VALIDATION_TIMED_OUT))
    s1["flags"] = np.where(m, s0["flags"] | bit, s0["flags"]).astype(np.uint32)
    b = apply(pol, s1, pods)
    fire = m & _differ((a[1], a[2], a[3]), (b[1], b[2], b[3]))
    return (int(at[fire].min()) if fire.any() else NONE), at, fire
