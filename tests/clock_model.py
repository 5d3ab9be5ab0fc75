"""Restatement of the clocked pod-list calls' derivation (include/ust.h, ust_clock) in numpy: bits 18 (UST_F_WAIT_TIMED_OUT)
and 27 (UST_F_VALIDATION_TIMED_OUT) from the wall clock and each node's start time, with Go's int64 semantics (the sum
start + timeout wraps in two's complement). Setting the bits this way on the host and calling the unclocked entry point
is what a clocked call must return."""
import numpy as np

from helpers import abi

WAIT_BITS = abi.UST_F_WAIT_START_ANNO | abi.UST_F_WAIT_START_INVALID
VAL_BITS = abi.UST_F_VALIDATION_START_ANNO | abi.UST_F_VALIDATION_START_INVALID
TIMED_OUT = abi.UST_F_WAIT_TIMED_OUT | abi.UST_F_VALIDATION_TIMED_OUT


def timed_out(now, start, timeout):
    """now > start + timeout on int64, the sum wrapping (pod_manager.go:354, validation_manager.go:161)."""
    start = np.atleast_1d(np.asarray(start, np.int64))
    t = np.uint64(int(timeout) & 0xFFFFFFFFFFFFFFFF)
    deadline = (start.view(np.uint64) + t).view(np.int64)
    return np.int64(now) > deadline


def derive(state, flags, start, now, wait_timeout):
    """flags with bits 18 and 27 of the wait-for-jobs-required and validation-required nodes derived from `now`: a node's
    start counts only with its state's annotation present and parsable. Other nodes keep both bits as given."""
    code = np.asarray(state, np.uint8) & np.uint8(abi.UST_HOT_STATE_MASK)
    flags = np.asarray(flags, np.uint32)
    start = np.asarray(start, np.int64)
    wait = code == abi.UST_STATE_WAIT_FOR_JOBS_REQUIRED
    val = code == abi.UST_STATE_VALIDATION_REQUIRED
    w_out = wait & ((flags & np.uint32(WAIT_BITS)) == abi.UST_F_WAIT_START_ANNO) & timed_out(now, start, wait_timeout)
    v_out = val & ((flags & np.uint32(VAL_BITS)) == abi.UST_F_VALIDATION_START_ANNO) & \
        timed_out(now, start, abi.UST_VALIDATION_TIMEOUT_SECONDS)
    out = np.where(wait | val, flags & np.uint32(~TIMED_OUT & 0xFFFFFFFF), flags).astype(np.uint32)
    out |= np.where(w_out, np.uint32(abi.UST_F_WAIT_TIMED_OUT), np.uint32(0))
    out |= np.where(v_out, np.uint32(abi.UST_F_VALIDATION_TIMED_OUT), np.uint32(0))
    return out


def derived_soa(soa, start, now, wait_timeout):
    """A copy of the snapshot whose flags carry the derived bits: the input of the unclocked call that is the oracle."""
    s = dict(soa)
    s["flags"] = derive(soa["state"], soa["flags"], start, now, wait_timeout)
    return s
