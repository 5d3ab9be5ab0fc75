"""The next deadline of a clocked call (include/ust.h, ust_next_deadline) on the CPU oracle: deadline_model's two-call flip
model against the brute force over every candidate time, on small random snapshots with every abort code, TimeoutSecond 0,
starts at the int64 extremes and wrapping deadlines, validation lists with a ready pod before a not-ready one and wait lists
whose pods have all finished; and two hand-worked cases, on the reference's wait-timeout timeline and its 600 s
validation timeout."""
import numpy as np
import pytest

import clock_model as cm
import deadline_model as dm
import helpers
from helpers import abi

I64 = np.iinfo(np.int64)
NOW = 1_700_000_000
T = 30
POL_KW = dict(max_parallel_upgrades=0, pod_deletion_enabled=True, pod_deletion={"force": False, "deleteEmptyDir": False},
              drain={"enable": True, "force": False, "deleteEmptyDir": False}, validation_enabled=True,
              wait_for_completion={"podSelector": "app=batch", "timeoutSeconds": T}, evaluate_actuators=True,
              evaluate_validation=True)
RUN_JOB = abi.UST_PHASE_RUNNING | abi.UST_POD_HAS_CONTROLLER | abi.UST_POD_MATCH_WAIT_SELECTOR
DONE_JOB = abi.UST_PHASE_SUCCEEDED | abi.UST_POD_HAS_CONTROLLER | abi.UST_POD_MATCH_WAIT_SELECTOR
VAL_READY = abi.UST_PHASE_RUNNING | abi.UST_POD_MATCH_VALIDATION_SELECTOR | abi.UST_POD_READY
VAL_WAIT = abi.UST_PHASE_RUNNING | abi.UST_POD_MATCH_VALIDATION_SELECTOR


def random_case(seed, n=400):
    """A small snapshot most of whose nodes are in the two clocked states, with random bits, lists and starts; the extremes
    of the start column and deadlines that land close to `now` on both sides."""
    rng = np.random.default_rng(seed)
    soa, pods = helpers.random_soa(rng, n, p_err=0.01 if seed % 4 == 0 else 0.0, with_pods=True)
    code = rng.choice([abi.UST_STATE_WAIT_FOR_JOBS_REQUIRED, abi.UST_STATE_VALIDATION_REQUIRED, 0, 1, 4, 8, 12], n,
                      p=[0.35, 0.35, 0.05, 0.1, 0.05, 0.05, 0.05]).astype(np.uint8)
    soa["state"] = ((soa["state"] & np.uint8(0xF0)) | code).astype(np.uint8)
    if seed % 4 != 0:   # mostly parsable starts, so that not every validation-mode call aborts early
        soa["flags"] &= np.where(rng.random(n) < 0.99, np.uint32(~(abi.UST_F_VALIDATION_START_INVALID | abi.UST_F_WAIT_START_INVALID)
                                                                  & 0xFFFFFFFF), np.uint32(0xFFFFFFFF))
    pol = helpers.random_policy(rng)
    pol.evaluate_actuators = 3 if seed % 2 == 0 else 1
    timeout = int(rng.choice([1, 30, 600])) if pol.wait_timeout_nonzero else 0
    now = int(rng.choice([0, NOW, -1000]))
    start = now + rng.integers(-700, 100, n)
    u = rng.random(n)
    start = np.where(u < 0.03, I64.max, start)
    start = np.where((u >= 0.03) & (u < 0.06), I64.min, start)
    start = np.where((u >= 0.06) & (u < 0.08), I64.max - rng.integers(0, 700, n), start)   # start + timeout wraps
    return pol, soa, pods, start.astype(np.int64), now, timeout


@pytest.mark.parametrize("seed", range(48))
def test_flip_model_equals_brute_force(seed):
    pol, soa, pods, start, now, timeout = random_case(seed)
    assert dm.flip_model(pol, soa, pods, start, now, timeout)[0] == dm.brute_force(pol, soa, pods, start, now, timeout)


def test_random_cases_cover_the_ground():
    """The random cases above reach every abort code, both answers, and deadlines that are not simply the first candidate."""
    rcs, found, none, skipped = set(), 0, 0, 0
    for seed in range(48):
        pol, soa, pods, start, now, timeout = random_case(seed)
        rcs.add(dm.reference_apply(pol, cm.derived_soa(soa, start, now, timeout), pods)[0])
        t, at, fire = dm.flip_model(pol, soa, pods, start, now, timeout)
        m, _ = dm.candidates(soa["state"], soa["flags"], start, now, timeout)
        if t == dm.NONE:
            none += 1
        else:
            found += 1
            skipped += int(at[m].min() < t)
    assert {0, abi.UST_ERR_REVISION_HASH, abi.UST_ERR_MAX_UNAVAILABLE, abi.UST_ERR_POD_DELETION_SPEC} <= rcs, rcs
    assert found >= 10 and none >= 1 and skipped >= 8, (found, none, skipped)


def one_node(state, flags, pod_flags, start, now, timeout=T, **kw):
    pol = abi.make_policy(**dict(POL_KW, wait_for_completion={"podSelector": "app=batch", "timeoutSeconds": timeout}, **kw))
    soa = {"state": np.array([state], np.uint8), "flags": np.array([flags], np.uint32), "pod_rev": np.array([1], np.int32),
           "ds_idx": np.array([0], np.int32), "ds_rev": np.array([1], np.int32)}
    pods = {"pod_off": np.array([0, len(pod_flags)], np.int32), "pod_flags": np.array(pod_flags, np.uint16)}
    st = np.array([start], np.int64)
    t = dm.brute_force(pol, soa, pods, st, now, timeout)
    assert dm.flip_model(pol, soa, pods, st, now, timeout)[0] == t
    return t


W, V = abi.UST_STATE_WAIT_FOR_JOBS_REQUIRED, abi.UST_STATE_VALIDATION_REQUIRED
WA, VA = abi.UST_F_WAIT_START_ANNO, abi.UST_F_VALIDATION_START_ANNO


def test_wait_deadline_boundaries():
    assert one_node(W, WA, [RUN_JOB], NOW - 10, NOW) == NOW - 10 + T + 1
    assert one_node(W, WA, [RUN_JOB], NOW - T, NOW) == NOW + 1            # d == now: the bit turns on one second later
    assert one_node(W, WA, [RUN_JOB], NOW - T - 1, NOW) == dm.NONE        # already timed out
    assert one_node(W, WA, [DONE_JOB, DONE_JOB], NOW - 10, NOW) == dm.NONE   # every wait pod finished: nothing to time out
    assert one_node(W, 0, [RUN_JOB], NOW - 10, NOW) == dm.NONE            # no annotation: the call sets it (an object change)
    assert one_node(W, WA | abi.UST_F_WAIT_START_INVALID, [RUN_JOB], NOW - 10, NOW) == dm.NONE


def test_wait_timeout_zero():
    """TimeoutSecond 0: the policy never looks at the bit, so no deadline is pending whatever the start."""
    for start in (NOW - 5, NOW, NOW + 5, I64.max, I64.min):
        assert one_node(W, WA, [RUN_JOB], start, NOW, timeout=0) == dm.NONE


def test_extreme_starts():
    # a deadline of exactly INT64_MAX - 1 fires at INT64_MAX
    assert one_node(W, WA, [RUN_JOB], I64.max - 1 - T, 0) == I64.max
    assert one_node(V, VA, [VAL_WAIT], I64.max - 1 - 600, 0) == I64.max
    # d == INT64_MAX never fires; a start whose sum wraps is long timed out; INT64_MIN is long ago
    assert one_node(W, WA, [RUN_JOB], I64.max - T, 0) == dm.NONE
    assert one_node(W, WA, [RUN_JOB], I64.max, 0) == dm.NONE
    assert one_node(W, WA, [RUN_JOB], I64.min, 0) == dm.NONE
    assert one_node(W, WA, [RUN_JOB], I64.min, I64.min) == I64.min + T + 1


def test_validation_lists():
    assert one_node(V, VA, [VAL_WAIT, VAL_READY], NOW - 10, NOW) == NOW - 10 + 601
    assert one_node(V, VA, [VAL_READY, VAL_WAIT], NOW - 10, NOW) == dm.NONE   # Validate deletes the annotation: no timeout
    assert one_node(V, VA, [VAL_READY, VAL_READY], NOW - 10, NOW) == dm.NONE  # done
    assert one_node(V, VA, [], NOW - 10, NOW) == dm.NONE                      # no matching pod: Validate waits, no timeout
    assert one_node(V, VA, [VAL_WAIT], NOW - 10, NOW, validation_enabled=False) == dm.NONE   # empty selector: done at once


def test_aborts_hide_deadlines():
    """Past the call's abort nothing is evaluated, so nothing can fire there; before it, deadlines count."""
    pol = abi.make_policy(**POL_KW)
    n = 3
    soa = {"state": np.array([W, V, W], np.uint8), "pod_rev": np.ones(n, np.int32), "ds_idx": np.zeros(n, np.int32),
           "ds_rev": np.array([1], np.int32),
           "flags": np.array([WA, VA | abi.UST_F_VALIDATION_START_INVALID, WA], np.uint32)}
    pods = {"pod_off": np.array([0, 1, 2, 3], np.int32), "pod_flags": np.array([RUN_JOB, VAL_WAIT, RUN_JOB], np.uint16)}
    start = np.array([NOW - 20, NOW, NOW - 5], np.int64)
    assert dm.reference_apply(pol, cm.derived_soa(soa, start, NOW, T), pods)[0] == abi.UST_ERR_VALIDATION
    # the validation pass (10) comes after the wait pass (4): both wait nodes are evaluated, the earlier deadline wins
    assert dm.brute_force(pol, soa, pods, start, NOW, T) == NOW - 20 + T + 1 == dm.flip_model(pol, soa, pods, start, NOW, T)[0]
    # a revision-hash abort in the unknown / done pass (0) comes before every wait node: nothing fires
    soa2 = {k: (np.concatenate([[0x80 | abi.UST_STATE_DONE], v]).astype(v.dtype) if k != "ds_rev" else v) for k, v in soa.items()}
    soa2["flags"][2] = VA
    pods2 = {"pod_off": np.array([0, 0, 1, 2, 3], np.int32), "pod_flags": pods["pod_flags"]}
    start2 = np.concatenate([[0], start]).astype(np.int64)
    assert dm.reference_apply(pol, cm.derived_soa(soa2, start2, NOW, T), pods2)[0] == abi.UST_ERR_REVISION_HASH
    assert dm.brute_force(pol, soa2, pods2, start2, NOW, T) == dm.NONE == dm.flip_model(pol, soa2, pods2, start2, NOW, T)[0]


def test_reference_wait_timeline():
    """pod_manager_test.go's wait-timeout timeline (helpers.wait_timeout_timeline, TimeoutSecond 100, a reconcile every
    30 s): the reconcile at 0 sets the start annotation to 0 (pod_manager.go:336-345), so from the reconcile at 30 on the
    next deadline is 0 + 100 + 1 = 101; the reconcile at 120 is the first to see the timeout."""
    G = helpers.load_golden()
    pol, soa, _, _ = helpers.wait_timeout_timeline(G["daemonset_hash"], 100, 30, 8)
    n = soa["state"].shape[0]
    soa = dict(soa, flags=(soa["flags"] | np.uint32(WA)).astype(np.uint32))
    pods = {"pod_off": np.arange(n + 1, dtype=np.int32), "pod_flags": np.full(n, RUN_JOB, np.uint16)}
    start = np.zeros(n, np.int64)
    for now in (30, 60, 90, 100):
        assert dm.brute_force(pol, soa, pods, start, now, 100) == 101
    assert dm.brute_force(pol, soa, pods, start, 101, 100) == dm.NONE
    r = dm.reference_apply(pol, cm.derived_soa(soa, start, 101, 100), pods)
    assert all(o == abi.UST_STATE_POD_DELETION_REQUIRED for o in r[3])


def test_reference_validation_timeout():
    """validation_manager.go's 600 s (:32, :161): a validation pod that is not ready, the start annotation set at S. The
    node fails at S + 601, not at S + 600."""
    S = NOW
    assert one_node(V, VA, [VAL_WAIT], S, S + 10) == S + 601
    assert one_node(V, VA, [VAL_WAIT], S, S + 600) == S + 601
    assert one_node(V, VA, [VAL_WAIT], S, S + 601) == dm.NONE
