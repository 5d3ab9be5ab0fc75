"""ust_build_state_delta / ust_fetch_build_state: the resident driver-pod list of BuildState. Every call is checked against
a numpy model (the list in its new order, the previous owner indices, INT32_MIN for joined pods) and the oracle's
ust_build_state_uids on the updated arrays: return code, counters, sparse outputs, and the full owner indices. Contract
violations are rejected before any launch with the list unchanged, and the list and ApplyState's snapshots leave each
other alone."""
import ctypes as C

import numpy as np
import pytest

import helpers
import reorder_model
import test_gpu_resident_contract as resident
from helpers import abi
from ust import lib as ustlib

pytestmark = pytest.mark.gpu

INVALID = abi.K["UST_ERR_INVALID_ARGUMENT"]
TRUNCATED = abi.K["UST_ERR_TRUNCATED"]
UNSCHEDULED = abi.K["UST_ERR_DS_UNSCHEDULED"]
NONE = np.int32(np.iinfo(np.int32).min)
# launches: join + finish, then the scan of the tile counts and the ordered write (no write for an empty list); a reorder
# adds the gather, overwrites add the patch
JOIN, SCAN_WRITE = 2, 2


@pytest.fixture(scope="module")
def handle():
    h = ustlib.Handle(0)
    yield h
    h.close()


def ds_table(rng, n_ds):
    return rng.integers(1, 2 ** 63, size=(n_ds, 2), dtype=np.uint64)


def new_pods(rng, m, ds_uid):
    """m driver pods: owned by a driver DaemonSet, orphaned ((0, 0)) or owned by something else; some excluded."""
    state = rng.integers(0, 16, m).astype(np.uint8) | (rng.integers(0, 16, m).astype(np.uint8) << 4)
    owner = rng.integers(2 ** 63, 2 ** 64 - 1, size=(m, 2), dtype=np.uint64)   # foreign
    kind = rng.random(m)
    if ds_uid.shape[0]:
        own = kind < 0.85
        owner[own] = ds_uid[rng.integers(0, ds_uid.shape[0], int(own.sum()))]
    owner[(kind >= 0.85) & (kind < 0.95)] = 0
    return state, owner


class Model:
    """The resident list as the caller sees it, and the owner indices the device returned last."""

    def __init__(self, handle):
        self.h = handle
        self.state = np.zeros(0, np.uint8)
        self.owner = np.zeros((0, 2), np.uint64)
        self.prev = np.zeros(0, np.int32)

    def call(self, order, ins, idx, chg, ds_uid, desired, max_out, launches=None, what=""):
        """One ust_build_state_delta: `order` (None = no reorder) as in reorder_model.runs_of, `ins` the joined pods,
        `idx` / `chg` the overwrites, `desired` DesiredNumberScheduled (None: what the updated list owns; "wrong": one
        more for DaemonSet 0); checked in full against the oracle."""
        ro = None
        if order is not None:
            src, ln = reorder_model.runs_of(order)
            ro = dict(run_src=src, run_len=ln, state=ins[0], owner_uid=ins[1])
            self.state = reorder_model.reorder(self.state, src, ln, ins[0])
            self.owner = np.stack([reorder_model.reorder(self.owner[:, j].copy(), src, ln, ins[1][:, j]) for j in (0, 1)], 1) \
                if self.state.size else np.zeros((0, 2), np.uint64)
            self.prev = reorder_model.reorder(self.prev, src, ln, np.full(ins[0].shape[0], NONE, np.int32))
        self.state[idx] = chg[0]
        self.owner[idx] = chg[1]
        if desired is None or isinstance(desired, str):
            wrong = desired is not None
            desired = desired_of(self.owner, ds_uid)
            desired[:1] += 1 if wrong else 0
        before = self.h.launch_count()
        rc, n_out, oi, od, cnt = self.h.build_state_delta(ro, idx, chg[0], chg[1], ds_uid, desired, max_out)
        launched = self.h.launch_count() - before
        orc, ods, ocnt = helpers.oracle_build_state_uids(self.state, self.owner, ds_uid, desired)
        changed = np.nonzero(ods != self.prev)[0]
        want = orc if orc != 0 or changed.size <= max_out else TRUNCATED
        assert rc == want, (what, rc, want, self.h.last_error())
        assert cnt == ocnt, (what, "counters")
        assert n_out == changed.size, (what, n_out, changed.size)
        if n_out <= max_out:
            assert np.array_equal(oi[:n_out], changed) and np.array_equal(od[:n_out], ods[changed]), (what, "sparse outputs")
        frc, full = self.h.fetch_build_state(self.state.size)
        assert frc == 0 and np.array_equal(full, ods), (what, "fetch")
        if launches is not None:
            assert launched == launches, (what, "launches", launched, launches)
        self.prev = ods
        return rc, n_out


def nothing(m=0):
    return np.zeros(m, np.uint8), np.zeros((m, 2), np.uint64)


def overwrites(rng, n, f, ds_uid):
    idx = np.sort(rng.choice(n, size=int(n * f), replace=False)).astype(np.int64) if n else np.zeros(0, np.int64)
    return idx, new_pods(rng, idx.size, ds_uid)


def desired_of(owner, ds_uid):
    """DesiredNumberScheduled that matches: the pods each DaemonSet owns."""
    ds_idx = helpers.oracle_build_state_uids(np.zeros(owner.shape[0], np.uint8), owner, ds_uid, np.zeros(ds_uid.shape[0], np.int32))[1]
    return np.bincount(ds_idx[ds_idx >= 0], minlength=ds_uid.shape[0]).astype(np.int32)


@pytest.mark.parametrize("n", [5000, 600_000])
@pytest.mark.parametrize("n_ds", [0, 8, 9, 600])
def test_call_sequence(handle, n, n_ds):
    """Empty list -> everything inserted; re-derived pods; leaves and joins; moves; a DaemonSet table in another order (every
    index shifts); max_out == 0; truncation; UST_ERR_DS_UNSCHEDULED together with truncation; everything removed."""
    rng = np.random.default_rng(n + n_ds)
    ds_uid = ds_table(rng, n_ds)
    none = np.zeros(0, np.int64)
    m = _emptied(handle, ds_uid)
    m.call(np.full(n, -1, np.int64), new_pods(rng, n, ds_uid), none, nothing(), ds_uid, None, n + 1,
           launches=1 + JOIN + SCAN_WRITE, what="insert all")
    idx, chg = overwrites(rng, m.state.size, 0.01, ds_uid)
    m.call(None, nothing(), idx, chg, ds_uid, None, m.state.size, launches=1 + JOIN + SCAN_WRITE, what="1 % re-derived")
    order = reorder_model.random_order(rng, m.state.size, "identity", f_remove=0.001, f_insert=0.001)
    m.call(order, new_pods(rng, int(np.sum(order < 0)), ds_uid), none, nothing(), ds_uid, None, m.state.size,
           launches=1 + JOIN + SCAN_WRITE, what="leaves and joins")
    order = reorder_model.random_order(rng, m.state.size, "moves", k=max(1, m.state.size // 1000))
    idx, chg = overwrites(rng, m.state.size, 0.001, ds_uid)
    m.call(order, nothing(), idx, chg, ds_uid, None, m.state.size, launches=2 + JOIN + SCAN_WRITE, what="moves")
    if n_ds > 1:   # the DaemonSet table in another order: every owned pod's index shifts
        ds_uid = ds_uid[rng.permutation(n_ds)]
        rc, n_out = m.call(None, nothing(), none, nothing(), ds_uid, None, 0, launches=JOIN + SCAN_WRITE, what="table order, max_out 0")
        assert rc == TRUNCATED and n_out > 0
    rc, n_out = m.call(None, nothing(), none, nothing(), ds_uid, None, 0, launches=JOIN + SCAN_WRITE, what="no change, max_out 0")
    assert rc == 0 and n_out == 0
    order = reorder_model.random_order(rng, m.state.size, "shuffle")
    idx, chg = overwrites(rng, m.state.size, 0.01, ds_uid)
    m.call(order, nothing(), idx, chg, ds_uid, None, 3, what="shuffle, truncated")
    if n_ds:
        idx, chg = overwrites(rng, m.state.size, 0.05, ds_uid)
        rc, n_out = m.call(None, nothing(), idx, chg, ds_uid, "wrong", 3, what="unscheduled + truncated")
        assert rc == UNSCHEDULED and n_out > 3
        m.call(None, nothing(), none, nothing(), ds_uid, None, m.state.size + 1, what="recovery")
    m.call(np.zeros(0, np.int64), nothing(), none, nothing(), ds_uid, None, 16, launches=1 + JOIN + 1, what="remove all")
    m.call(np.full(1, -1, np.int64), new_pods(rng, 1, ds_uid), none, nothing(), ds_uid, None, 16, what="one joins")


def _emptied(handle, ds_uid):
    """The resident list emptied (a reorder without runs), and a model of it."""
    rc = handle.build_state_delta(dict(run_src=[], run_len=[]), np.zeros(0, np.int64), *nothing(), ds_uid,
                                  np.zeros(ds_uid.shape[0], np.int32), 0)[0]
    assert rc == 0, handle.last_error()
    return Model(handle)


def _list(handle, rng, n=5000, n_ds=3):
    """A fresh resident list of n pods; returns its model and DaemonSet table."""
    ds_uid = ds_table(rng, n_ds)
    m = _emptied(handle, ds_uid)
    m.call(np.full(n, -1, np.int64), new_pods(rng, n, ds_uid), np.zeros(0, np.int64), nothing(), ds_uid, None, n + 1, what="setup")
    return m, ds_uid


def test_contract_violations(handle):
    rng = np.random.default_rng(11)
    m, ds_uid = _list(handle, rng)
    n = m.state.size
    desired = desired_of(m.owner, ds_uid)
    none = np.zeros(0, np.int64)
    one = new_pods(rng, 1, ds_uid)
    two = new_pods(rng, 2, ds_uid)
    bad = [
        ("run length 0", dict(run_src=[0, 5], run_len=[5, 0]), none, nothing(), ds_uid),
        ("run source -2", dict(run_src=[-2], run_len=[1]), none, nothing(), ds_uid),
        ("old run leaves the list", dict(run_src=[n - 3], run_len=[4]), none, nothing(), ds_uid),
        ("two runs name one pod", dict(run_src=[0, 4], run_len=[5, 3]), none, nothing(), ds_uid),
        ("inserted runs take more", dict(run_src=[-1], run_len=[3], state=two[0], owner_uid=two[1]), none, nothing(), ds_uid),
        ("inserted runs take fewer", dict(run_src=[-1, 0], run_len=[1, n], state=two[0], owner_uid=two[1]), none, nothing(), ds_uid),
        ("idx duplicated", None, np.array([3, 3], np.int64), two, ds_uid),
        ("idx outside the new list", dict(run_src=[0], run_len=[n - 1]), np.array([n - 1], np.int64), one, ds_uid),
        ("idx negative", None, np.array([-1], np.int64), one, ds_uid),
        ("empty DaemonSet UID", None, none, nothing(), np.concatenate([ds_uid, np.zeros((1, 2), np.uint64)])),
        ("duplicated DaemonSet UID", None, none, nothing(), np.concatenate([ds_uid, ds_uid[:1]])),
    ]
    for what, ro, idx, chg, du in bad:
        before = handle.launch_count()
        des = np.resize(desired, du.shape[0])
        rc = handle.build_state_delta(ro, idx, chg[0], chg[1], du, des, 64)[0]
        assert rc == INVALID, (what, rc, handle.last_error())
        assert handle.launch_count() == before, what
    # the raw ABI: negative counts and NULL arrays
    lib = ustlib.load()
    oi, od, n_out, cnt = np.zeros(8, np.int64), np.zeros(8, np.int32), C.c_int64(0), abi.Counters()
    src, ln = np.array([-1], np.int64), np.array([1], np.int64)
    null_ins = abi.DriverPodReorder(1, src.ctypes.data, ln.ctypes.data, 1, None, None)
    null_runs = abi.DriverPodReorder(1, None, None, 0, None, None)
    du, des = ds_uid, desired
    raw = [
        ("NULL joined-pod arrays", C.addressof(null_ins), 0, None, du.ctypes.data, du.shape[0], des.ctypes.data, 8, oi.ctypes.data, C.addressof(n_out)),
        ("NULL run arrays", C.addressof(null_runs), 0, None, du.ctypes.data, du.shape[0], des.ctypes.data, 8, oi.ctypes.data, C.addressof(n_out)),
        ("NULL idx", None, 2, None, du.ctypes.data, du.shape[0], des.ctypes.data, 8, oi.ctypes.data, C.addressof(n_out)),
        ("n_ds < 0", None, 0, None, du.ctypes.data, -1, des.ctypes.data, 8, oi.ctypes.data, C.addressof(n_out)),
        ("NULL DaemonSet table", None, 0, None, None, du.shape[0], None, 8, oi.ctypes.data, C.addressof(n_out)),
        ("max_out < 0", None, 0, None, du.ctypes.data, du.shape[0], des.ctypes.data, -1, oi.ctypes.data, C.addressof(n_out)),
        ("NULL outputs", None, 0, None, du.ctypes.data, du.shape[0], des.ctypes.data, 8, None, C.addressof(n_out)),
        ("NULL n_out", None, 0, None, du.ctypes.data, du.shape[0], des.ctypes.data, 8, oi.ctypes.data, None),
    ]
    for what, ro, m_chg, idx, ds_p, n_ds, des_p, max_out, out_p, n_out_p in raw:
        before = handle.launch_count()
        rc = lib.ust_build_state_delta(handle._h, ro, m_chg, idx, None, None, n_ds, ds_p, des_p, C.c_int64(max_out), out_p,
                                       od.ctypes.data if out_p else None, n_out_p, C.addressof(cnt))
        assert rc == INVALID, (what, rc)
        assert handle.launch_count() == before, what
    assert handle.fetch_build_state(n + 1)[0] == INVALID
    # the list is as it was: a no-change call reports nothing, the fetch returns the previous indices
    rc, n_out = m.call(None, nothing(), none, nothing(), ds_uid, desired, 16, launches=JOIN + SCAN_WRITE, what="after the rejected calls")
    assert rc == 0 and n_out == 0


# ApplyState's calls that resident.PREVIOUS does not make: the delta entry points with a new node order and with pod lists
def _splice(handle):
    soa = resident.make_resident(handle, 12)
    sp = dict(remove_idx=np.array([3, 9], np.int64), insert_before=np.zeros(0, np.int64))
    assert handle.apply_state_delta_splice(resident.POL, sp, np.zeros(0, np.int64), {k: np.zeros(0) for k in resident.COLS}, soa["ds_rev"], 16)[0] in (0, TRUNCATED), handle.last_error()


def _reorder(handle):
    soa = resident.make_resident(handle, 13)
    n = soa["state"].shape[0]
    rc = handle.apply_state_delta_reorder(resident.POL, dict(run_src=[n // 2, 0], run_len=[n - n // 2, n // 2]), np.zeros(0, np.int64),
                                          {k: np.zeros(0) for k in resident.COLS}, soa["ds_rev"], 16)[0]
    assert rc in (0, TRUNCATED), handle.last_error()


def _pods_delta(handle, reorder):
    soa, pl = resident.snapshot(14, resident.SMALL)
    handle.apply_state(resident.POL, soa, pl)
    n = soa["state"].shape[0]
    empty = {k: np.zeros(0) for k in resident.COLS}
    if reorder:
        rc = handle.apply_state_delta_pods_reorder(resident.POL, dict(run_src=[1, 0], run_len=[n - 1, 1]), None, np.zeros(0, np.int64),
                                                   empty, soa["ds_rev"], 16)[0]
    else:
        rc = handle.apply_state_delta_pods(resident.POL, None, np.zeros(0, np.int64), empty, soa["ds_rev"], 16)[0]
    assert rc in (0, TRUNCATED), handle.last_error()


OTHER_CALLS = dict({k: v for k, v in resident.PREVIOUS.items()},
                   splice=_splice, reorder=_reorder, pods_delta=lambda h: _pods_delta(h, False),
                   pods_reorder=lambda h: _pods_delta(h, True))


@pytest.mark.parametrize("previous", list(OTHER_CALLS))
def test_no_other_call_touches_the_list(handle, previous):
    rng = np.random.default_rng(21)
    m, ds_uid = _list(handle, rng)
    OTHER_CALLS[previous](handle)
    rc, n_out = m.call(None, nothing(), np.zeros(0, np.int64), nothing(), ds_uid, desired_of(m.owner, ds_uid), 16,
                       launches=JOIN + SCAN_WRITE, what=previous)
    assert rc == 0 and n_out == 0


def test_the_list_leaves_applystate_alone(handle):
    rng = np.random.default_rng(31)
    empty_idx = np.zeros(0, np.int64)
    empty = {k: np.zeros(0) for k in resident.COLS}
    # the node snapshot and its outputs
    soa = resident.make_resident(handle, 32)
    ref = resident.oracle(soa)
    m, ds_uid = _list(handle, rng)
    order = reorder_model.random_order(rng, m.state.size, "moves")
    m.call(order, nothing(), empty_idx, nothing(), ds_uid, desired_of(m.owner[order], ds_uid), 16, what="a reorder")
    rc, nxt, act = handle.fetch_outputs(soa["state"].shape[0])
    assert rc == 0 and np.array_equal(nxt, ref[1]) and np.array_equal(act, ref[2])
    got = handle.apply_state_delta_sparse(resident.POL, empty_idx, empty, soa["ds_rev"], 16)
    assert got[0] == ref[0] and got[1] == 0 and got[5] == ref[4], (got[0], got[1])
    # the pod-list snapshot and its outputs
    soa, pl = resident.snapshot(33, resident.SMALL)
    handle.apply_state(resident.POL, soa, pl)
    ref = resident.oracle(soa, pl)
    m.call(None, nothing(), empty_idx, nothing(), ds_uid, desired_of(m.owner, ds_uid), 16, what="no change")
    got = handle.apply_state_delta_pods(resident.POL, None, empty_idx, empty, soa["ds_rev"], 16)
    assert got[0] == ref[0] and got[1] == 0 and got[6] == ref[4], (got[0], got[1])
    rc, nxt, act, oc = handle.fetch_outputs_pods(soa["state"].shape[0])
    assert rc == 0 and np.array_equal(nxt, ref[1]) and np.array_equal(act, ref[2]) and np.array_equal(oc, ref[3])
