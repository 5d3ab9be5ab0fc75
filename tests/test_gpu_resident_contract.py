"""The resident-snapshot contract across entry points: after each kind of call, what ust_apply_state_delta,
ust_apply_state_delta_sparse and ust_fetch_outputs find resident, and how many kernels each call launches.

A call keeps its snapshot and outputs resident when it produced counters (a reference-level abort and UST_ERR_TRUNCATED
included) and had no pod lists. A call rejected by its argument checks leaves the previous snapshot as it was. A rollout
simulation keeps the simulated snapshot without outputs. BuildState and calls with pod lists leave nothing resident."""
import ctypes as C

import numpy as np
import pytest

import helpers
from helpers import abi
from ust import lib as ustlib, synth

pytestmark = pytest.mark.gpu

COLS = ("state", "flags", "pod_rev", "ds_idx")
INVALID = abi.K["UST_ERR_INVALID_ARGUMENT"]
TRUNCATED = abi.K["UST_ERR_TRUNCATED"]
REVISION_HASH = abi.K["UST_ERR_REVISION_HASH"]
SMALL, LARGE = 5000, 600_000   # LARGE >= 2^19: ust_apply_state and _packed upload through the pipelined path
# the pipelined path cuts LARGE (196 tiles of 3072 nodes) into the default six segments (UST_SEGMENTS): one streaming
# launch per segment, one widen launch per segment for the packed format
SEGMENTS = 6
# streaming + verification; pod lists add the pod-summary kernel; a sparse call adds the three diff kernels
CALL, PODS, DIFF = 2, 1, 3
POL = abi.make_policy(max_parallel_upgrades=0, max_unavailable="30%", evaluate_actuators=True)


@pytest.fixture(scope="module")
def handle():
    h = ustlib.Handle(0)
    yield h
    h.close()


def snapshot(seed, n, p_err=0.0):
    return helpers.random_soa(np.random.default_rng(seed), n, wild=True, p_err=p_err, with_pods=True)


def oracle(soa, pods=None):
    return helpers.oracle_apply(POL, soa, pods, variant=1)


def make_resident(handle, seed):
    """A small resident snapshot with outputs, so that a later call's effect on residency shows."""
    soa, _ = snapshot(seed, SMALL)
    helpers.assert_same(handle.apply_state(POL, soa), oracle(soa), "setup")
    return soa


def counted(handle, call):
    before = handle.launch_count()
    result = call()
    return result, handle.launch_count() - before


# Each previous call returns (launches it made, launches expected, snapshot the caller believes resident or None,
# whether that snapshot's outputs are resident).

def apply_state(handle, n, pods=False, abort=False):
    make_resident(handle, 1)
    soa, pl = snapshot(100 + n, n, p_err=0.02 if abort else 0.0)
    pl = pl if pods else None
    got, launched = counted(handle, lambda: handle.apply_state(POL, soa, pl))
    ref = oracle(soa, pl)
    assert (ref[0] == REVISION_HASH) == abort, ref[0]
    helpers.assert_same(got, ref, f"apply_state n={n} pods={pods}")
    if pods:
        return launched, PODS + CALL, None, False
    return launched, (SEGMENTS + 1 if n >= LARGE else CALL), soa, True


def packed(handle, n):
    make_resident(handle, 2)
    soa, _ = snapshot(200 + n, n)
    got, launched = counted(handle, lambda: handle.apply_state_packed(POL, soa))
    helpers.assert_same(got, oracle(soa), f"packed n={n}")
    return launched, (2 * SEGMENTS + 1 if n >= LARGE else 1 + CALL), soa, True


def packed_rejected(handle):
    soa = make_resident(handle, 3)
    other, _ = snapshot(300, SMALL + 7)
    other["ds_rev"] = np.zeros(128, np.int32)   # the packed format holds at most 127 DaemonSets
    got, launched = counted(handle, lambda: handle.apply_state_packed(POL, other))
    assert got[0] == INVALID and "127" in handle.last_error()
    return launched, 0, soa, True


def negative_n_rejected(handle):
    soa = make_resident(handle, 4)
    rc, launched = counted(handle, lambda: ustlib.load().ust_apply_state(handle._h, C.addressof(POL), -1, None, None, None, None, 0,
                                                                         None, None, None, None, None, None))
    assert rc == abi.UST_ERR_NIL_STATE
    return launched, 0, soa, True


def delta(handle):
    soa = make_resident(handle, 5)
    rng = np.random.default_rng(5)
    idx = np.sort(rng.choice(SMALL, size=50, replace=False)).astype(np.int64)
    fresh, _ = helpers.random_soa(rng, idx.shape[0], wild=True)
    for k in COLS:
        soa[k][idx] = fresh[k]
    got, launched = counted(handle, lambda: handle.apply_state_delta(POL, SMALL, idx, fresh, soa["ds_rev"]))
    helpers.assert_same(got, oracle(soa), "delta")
    return launched, 1 + CALL, soa, True


def sparse_truncated(handle):
    soa = make_resident(handle, 6)
    rng = np.random.default_rng(6)
    idx = np.sort(rng.choice(SMALL, size=SMALL // 10, replace=False)).astype(np.int64)
    fresh, _ = helpers.random_soa(rng, idx.shape[0], wild=True)
    for k in COLS:
        soa[k][idx] = fresh[k]
    got, launched = counted(handle, lambda: handle.apply_state_delta_sparse(POL, idx, fresh, soa["ds_rev"], 2))
    ref = oracle(soa)
    assert ref[0] == 0 and got[0] == TRUNCATED and got[1] > 2, (got[0], got[1])
    assert got[5] == ref[4]
    return launched, 1 + CALL + DIFF, soa, True


def simulation(handle):
    soa = synth.make_nodes(SMALL, 7)   # a cluster the simulation can roll forward (the oracle restates its feedback)
    helpers.assert_same(handle.apply_state(POL, soa), oracle(soa), "setup")
    steps = 2
    (rc, done, _, fin), launched = counted(handle, lambda: handle.simulate_rollout(POL, SMALL, steps))
    orc, odone, _, ofin = helpers.oracle_simulate(POL, soa, steps, variant=1)
    assert rc == orc and done == odone and all(np.array_equal(fin[k], ofin[k]) for k in ofin)
    after = dict(soa)
    after.update(ofin)
    return launched, steps * (CALL + 1), after, False   # each step: ApplyState + the feedback kernel


def build_state(handle):
    soa = make_resident(handle, 8)
    (rc, _), launched = counted(handle, lambda: handle.build_state(soa["state"][:10], np.zeros(10, np.int32), np.array([10], np.int32)))
    assert rc not in (abi.K["UST_ERR_CUDA"], INVALID), handle.last_error()
    return launched, 2, None, False


def build_state_uids(handle):
    make_resident(handle, 9)
    rng = np.random.default_rng(9)
    ds_uid = rng.integers(1, 2 ** 63, size=(3, 2), dtype=np.uint64)
    owner = ds_uid[rng.integers(0, 3, 1000)]
    state = rng.integers(0, 13, owner.shape[0]).astype(np.uint8)
    desired = np.array([int(np.sum((owner == ds_uid[d]).all(axis=1))) for d in range(3)], np.int32)
    (rc, ds_idx, cnt), launched = counted(handle, lambda: handle.build_state_uids(state, owner, ds_uid, desired))
    orc, ods, ocnt = helpers.oracle_build_state_uids(state, owner, ds_uid, desired)
    assert rc == orc and np.array_equal(ds_idx, ods) and cnt == ocnt
    return launched, 2, None, False


PREVIOUS = {
    "apply_state": lambda h: apply_state(h, SMALL),
    "apply_state_pipelined": lambda h: apply_state(h, LARGE),
    "apply_state_pods": lambda h: apply_state(h, SMALL, pods=True),
    "apply_state_pods_large": lambda h: apply_state(h, LARGE, pods=True),   # pod lists never take the pipelined path
    "apply_state_abort": lambda h: apply_state(h, SMALL, abort=True),
    "apply_state_pipelined_abort": lambda h: apply_state(h, LARGE, abort=True),
    "packed": lambda h: packed(h, SMALL),
    "packed_pipelined": lambda h: packed(h, LARGE),
    "packed_rejected_n_ds_128": packed_rejected,
    "apply_state_rejected_negative_n": negative_n_rejected,
    "delta": delta,
    "delta_sparse_truncated": sparse_truncated,
    "simulate_rollout": simulation,
    "build_state": build_state,
    "build_state_uids": build_state_uids,
}


@pytest.mark.parametrize("previous", list(PREVIOUS))
def test_what_a_call_leaves_resident(handle, previous):
    launched, expected, snap, outputs = PREVIOUS[previous](handle)
    assert launched == expected, (previous, "launches", launched, expected)
    empty_idx = np.zeros(0, np.int64)
    empty = {k: np.zeros(0) for k in COLS}
    ds_rev = snap["ds_rev"] if snap is not None else np.ones(3, np.int32)
    n = int(snap["state"].shape[0]) if snap is not None else 0
    ref = oracle(snap) if snap is not None else None

    # 1. ust_fetch_outputs: the outputs of the last call on the resident snapshot (arrays large enough for any snapshot)
    (rc, nxt, act), launched = counted(handle, lambda: handle.fetch_outputs(LARGE))
    assert launched == 0
    if snap is None or not outputs:
        assert rc == INVALID, (previous, "fetch", rc)
    else:
        assert rc == 0, (previous, "fetch", handle.last_error())
        assert np.array_equal(nxt[:n], ref[1]) and np.array_equal(act[:n], ref[2]), (previous, "fetched outputs")

    # 2. ust_apply_state_delta_sparse with no changes: same policy, same snapshot, so no output changes
    got, launched = counted(handle, lambda: handle.apply_state_delta_sparse(POL, empty_idx, empty, ds_rev, n + 1))
    if snap is None or not outputs:
        assert got[0] == INVALID and launched == 0, (previous, "sparse", got[0], launched)
    else:
        assert got[0] == ref[0] and got[1] == 0 and got[5] == ref[4], (previous, "sparse", got[0], got[1])
        assert launched == CALL + DIFF, (previous, "sparse launches", launched)

    # 3. ust_apply_state_delta with no changes: evaluates the resident snapshot again
    got, launched = counted(handle, lambda: handle.apply_state_delta(POL, n, empty_idx, empty, ds_rev))
    if snap is None:
        assert got[0] == INVALID and launched == 0, (previous, "delta", got[0], launched)
    else:
        helpers.assert_same(got, ref, f"{previous}: delta on the resident snapshot")
        assert launched == CALL, (previous, "delta launches", launched)
