"""ust_apply_state_delta_pods on the H100: reconcile chains that replace pod lists (same lengths: the in-place scatter;
changed lengths: the relayout) and overwrite nodes, against the oracle on the numpy-updated arrays. After every call the
reported nodes are exactly those whose next_state, actions or actuator_outcome changed, patching the caller's full arrays
with them gives the oracle's outputs, the counters match, and the truncated path hands out the same outputs through
ust_fetch_outputs_pods. Plus the residency contract of the pod-list snapshot."""
import ctypes as C

import numpy as np
import pytest

import helpers
import pods_delta_model as model
from helpers import abi
from ust import lib as ustlib, synth

pytestmark = pytest.mark.gpu

COLS = ("state", "flags", "pod_rev", "ds_idx")
INVALID = abi.K["UST_ERR_INVALID_ARGUMENT"]
TRUNCATED = abi.K["UST_ERR_TRUNCATED"]
REVISION_HASH = abi.K["UST_ERR_REVISION_HASH"]
# streaming + verification, the three diff kernels; the pod-summary kernel when the policy evaluates actuators; the patch
# with overwrites; one scatter launch for lists that keep their lengths, two (run table, relayout) otherwise
CALL, DIFF, PATCH, SCATTER, RELAYOUT = 2, 3, 1, 1, 2
POD_BLOCK = 4096  # nodes per block of the pod-summary kernel
POL_KW = dict(max_parallel_upgrades=0, max_unavailable="30%", pod_deletion_enabled=True,
              pod_deletion={"force": False, "deleteEmptyDir": False}, drain={"enable": True, "force": False, "deleteEmptyDir": False},
              wait_for_completion={"podSelector": "app=batch", "timeoutSeconds": 0}, evaluate_actuators=True)
POL = abi.make_policy(**POL_KW)


@pytest.fixture(scope="module")
def handle():
    h = ustlib.Handle(0)
    yield h
    h.close()


def new_nodes(rng, m):
    fresh, _ = helpers.random_soa(rng, m, wild=True)
    return {k: fresh[k] for k in COLS}


def overwrites(rng, n, frac, idx=None):
    if idx is None:
        m = min(n, int(np.ceil(n * frac))) if frac > 0 else 0
        idx = np.sort(rng.choice(n, size=m, replace=False)).astype(np.int64) if m else np.zeros(0, np.int64)
    return np.asarray(idx, np.int64), new_nodes(rng, len(idx))


def pod_launches(pol):
    return 1 if pol.auto_upgrade and pol.evaluate_actuators else 0


class PodResident:
    """What the caller holds: the snapshot (nodes and pod lists) the device has resident and the outputs of the last call."""

    def __init__(self, handle, pol, soa, pods):
        self.h, self.soa, self.pods = handle, soa, pods
        got = handle.apply_state(pol, soa, pods)
        ref = helpers.oracle_apply(pol, soa, pods, variant=1)
        helpers.assert_same(got, ref, "full call")
        self.nxt, self.act, self.oc = got[1], got[2], got[3]
        self.paths = set()

    @property
    def n(self):
        return int(self.soa["state"].shape[0])

    def step(self, pol, lists, idx, fresh, cap, what=""):
        soa = {k: v.copy() for k, v in self.soa.items()}
        for k in COLS:
            soa[k][idx] = fresh[k]
        pods = self.pods
        path = 0
        if lists is not None and len(lists["node_idx"]):
            off, pf = model.replace(pods["pod_off"], pods["pod_flags"], lists["node_idx"], lists["pod_off"], lists["pod_flags"])
            same = np.array_equal(np.diff(lists["pod_off"]), np.diff(pods["pod_off"])[lists["node_idx"]])
            path = SCATTER if same else RELAYOUT
            self.paths.add("scatter" if same else "relayout")
            pods = {"pod_off": off, "pod_flags": pf}
        before = self.h.launch_count()
        rc, n_out, oi, on, oa, oo, cnt = self.h.apply_state_delta_pods(pol, lists, idx, fresh, soa["ds_rev"], cap)
        launched = self.h.launch_count() - before
        ref = helpers.oracle_apply(pol, soa, pods, variant=1)
        expect = (ref[1] != self.nxt) | (ref[2] != self.act) | (ref[3] != self.oc)
        assert n_out == int(expect.sum()), (what, n_out, int(expect.sum()))
        if n_out > cap:
            assert rc == (TRUNCATED if ref[0] == 0 else ref[0]), (what, rc, ref[0])
            frc, nxt, act, oc = self.h.fetch_outputs_pods(self.n)
            assert frc == 0, (what, self.h.last_error())
        else:
            assert rc == ref[0], (what, rc, ref[0], self.h.last_error())
            assert np.array_equal(oi[:n_out], np.nonzero(expect)[0]), what   # node order, exactly those nodes
            nxt, act, oc = self.nxt.copy(), self.act.copy(), self.oc.copy()
            nxt[oi[:n_out]] = on[:n_out]
            act[oi[:n_out]] = oa[:n_out]
            oc[oi[:n_out]] = oo[:n_out]
        helpers.assert_same((rc, nxt, act, oc, cnt), (rc, ref[1], ref[2], ref[3], ref[4]), what)
        expected_launches = pod_launches(pol) + CALL + DIFF + (PATCH if len(idx) else 0) + path
        assert launched == expected_launches, (what, "launches", launched, expected_launches)
        self.soa, self.pods, self.nxt, self.act, self.oc = soa, pods, nxt, act, oc
        return rc, n_out

    def empty(self, pol, what=""):
        idx, fresh = overwrites(np.random.default_rng(0), self.n, 0.0, idx=[])
        return self.step(pol, None, idx, fresh, self.n + 16, what)


def wide_snapshot(rng, n):
    """random_soa with pod lists, and with the last node in a state whose actuator reads its list (pod deletion), so that
    the pod-summary kernel walks the last list of the array."""
    soa, pods = helpers.random_soa(rng, n, wild=True, with_pods=True)
    if n:
        soa["state"][-1] = abi.UST_STATE_POD_DELETION_REQUIRED
    return soa, pods


def tail_lists(rng, res):
    """A new list for the last node whose end falls inside the final 16 bytes of pod_flags with a total that is no multiple
    of 8 pods: the pod-summary kernel's path for lists that end there."""
    before = int(res.pods["pod_off"][-2])   # pods ahead of the last list
    ln = (5 - before) % 8                    # the new total is 5 mod 8 ...
    ln += 8 if ln < 3 else 0                 # ... and the list at least 3 pods long
    li = {"node_idx": np.array([res.n - 1], np.int64), "pod_off": np.array([0, ln], np.int32), "pod_flags": model.random_flags(rng, ln)}
    last = new_nodes(rng, 1)                 # a state whose actuator reads the list
    last["state"][:] = abi.UST_STATE_POD_DELETION_REQUIRED
    return li, np.array([res.n - 1], np.int64), last


@pytest.mark.parametrize("n", [1, 127, POD_BLOCK - 1, POD_BLOCK, POD_BLOCK + 1, 65_537, 700_001])
def test_pods_delta_chains(handle, n):
    """Every kind of list change at every fraction, with and without node overwrites (also of the replaced nodes); both
    list-replacement paths with their launch counts."""
    rng = np.random.default_rng(7000 + n)
    soa, pods = wide_snapshot(rng, n)
    res = PodResident(handle, POL, soa, pods)
    step = 0
    for frac in (0.0, 0.001, 0.01, 0.3, 1.0):
        for kind in model.KINDS:
            if frac == 0.0 and kind != "same":
                continue
            li = model.random_lists(rng, res.pods["pod_off"], frac, kind)
            # overwrites on their own (frac 0), of other nodes, or of the very nodes whose lists change
            if step % 3 == 0:
                idx, fresh = overwrites(rng, n, 0.01)
            elif step % 3 == 1:
                idx, fresh = overwrites(rng, n, 0.0, idx=li["node_idx"][::2])
            else:
                idx, fresh = overwrites(rng, n, 0.0, idx=[])
            cap = n + 16 if step % 5 != 4 else 2
            res.step(POL, li, idx, fresh, cap, f"n={n} frac={frac} {kind}")
            if kind == "zero":  # and back from empty, on the same nodes
                li = model.random_lists(rng, res.pods["pod_off"], kind="from_zero", node_idx=li["node_idx"])
                res.step(POL, li, *overwrites(rng, n, 0.0, idx=[]), cap=n + 16, what=f"n={n} frac={frac} from_zero")
            step += 1
    res.step(POL, *tail_lists(rng, res), cap=n + 16, what=f"n={n} tail list")
    assert int(res.pods["pod_off"][-1]) % 8 == 5
    res.empty(POL, f"n={n} empty call")
    assert res.paths == {"scatter", "relayout"}, res.paths


def test_policy_changes_without_data_change(handle):
    """Toggling drain_force, pod_deletion_delete_emptydir and evaluate_actuators reports exactly the nodes whose outputs
    (the outcome included) differ in the oracle."""
    rng = np.random.default_rng(21)
    soa, pods = wide_snapshot(rng, 20_000)
    res = PodResident(handle, POL, soa, pods)
    reported = []
    for key, change in (("drain", {"enable": True, "force": True, "deleteEmptyDir": False}),
                        ("pod_deletion", {"force": False, "deleteEmptyDir": True}),
                        ("evaluate_actuators", False), ("evaluate_actuators", True),
                        ("pod_deletion", {"force": False, "deleteEmptyDir": False}),
                        ("drain", {"enable": True, "force": False, "deleteEmptyDir": False})):
        kw = dict(POL_KW)
        kw[key] = change
        reported.append(res.empty(abi.make_policy(**kw), f"{key} -> {change}")[1])
    assert reported[2] > 0 and sum(reported) > reported[2], reported   # actuator evaluation off changes every outcome


def revision_hash_node(rng):
    bad = new_nodes(rng, 1)
    bad["state"][:] = abi.UST_STATE_DONE | abi.UST_HOT_REVISION_HASH_ERROR
    bad["flags"][:] &= ~np.uint32(abi.UST_F_POD_ORPHANED)
    bad["ds_idx"][:] = 0
    return bad


def test_aborts_and_truncation(handle):
    """A revision-hash abort with and without truncation, then UST_ERR_TRUNCATED followed by ust_fetch_outputs_pods."""
    rng = np.random.default_rng(22)
    soa, pods = wide_snapshot(rng, 30_000)
    res = PodResident(handle, POL, soa, pods)
    n = res.n
    li = model.random_lists(rng, res.pods["pod_off"], 0.01, "mixed")
    rc, n_out = res.step(POL, li, np.array([n // 3], np.int64), revision_hash_node(rng), n + 16, "abort")
    assert rc == REVISION_HASH
    li = model.random_lists(rng, res.pods["pod_off"], 0.05, "odd")
    # the passes stop at the aborting node, so few outputs change: truncated at max_out = 0
    rc, n_out = res.step(POL, li, np.array([n // 2], np.int64), revision_hash_node(rng), 0, "abort, truncated")
    assert rc == REVISION_HASH and n_out > 0
    # the snapshot (with its aborting nodes) stays resident; repair them, change lists and truncate
    idx = np.array([n // 3, n // 2], np.int64)
    fresh = new_nodes(rng, 2)
    fresh["state"] &= np.uint8(abi.UST_HOT_STATE_MASK)
    li = model.random_lists(rng, res.pods["pod_off"], 0.3, "mixed")
    rc, n_out = res.step(POL, li, idx, fresh, 3, "truncated")
    assert rc == TRUNCATED and n_out > 3
    li = model.random_lists(rng, res.pods["pod_off"], 0.01, "same")
    res.step(POL, li, *overwrites(rng, n, 0.01), cap=n, what="after the truncated call")


def test_c4_full_size(handle):
    """C4: 10 M nodes and ~300 M pods, 1 % of the lists replaced at the same lengths and at changed lengths."""
    cfg = synth.CONFIGS["C4"]
    soa = synth.make_nodes(cfg["n"], cfg["seed"])
    pods = synth.make_pods_blocked(cfg["n"], cfg["seed"])
    pol = synth.config_policy("C4")
    res = PodResident(handle, pol, soa, pods)
    rng = np.random.default_rng(4)
    for kind in ("same", "mixed"):
        li = model.random_lists(rng, res.pods["pod_off"], 0.01, kind)
        res.step(pol, li, *overwrites(rng, res.n, 0.0, idx=[]), cap=res.n // 8, what=f"C4 {kind}")
    assert res.paths == {"scatter", "relayout"}


def raw_call(handle, pol, lists, n_changed=0, idx=None, cols=None, max_out=16, outcome=True):
    """ust_apply_state_delta_pods with raw pointers (NULL arrays, pod counts that no array backs)."""
    ds_rev = np.ones(3, np.int32)
    oi, on, oa, oo = np.zeros(17, np.int64), np.zeros(17, np.uint8), np.zeros(17, np.uint16), np.zeros(17, np.uint8)
    cols = cols or {}
    n_out = C.c_int64(0)
    cnt = abi.Counters()
    return handle._lib.ust_apply_state_delta_pods(
        handle._h, C.addressof(pol), C.addressof(lists) if lists is not None else None, n_changed, idx,
        cols.get("state"), cols.get("flags"), cols.get("pod_rev"), cols.get("ds_idx"), 3, ds_rev.ctypes.data, C.c_int64(max_out),
        oi.ctypes.data, on.ctypes.data, oa.ctypes.data, oo.ctypes.data if outcome else None, C.addressof(n_out), C.addressof(cnt))


def test_contract_errors_leave_the_snapshot(handle):
    rng = np.random.default_rng(31)
    soa, pods = wide_snapshot(rng, 5000)
    res = PodResident(handle, POL, soa, pods)
    n = res.n
    none = np.zeros(0, np.int64)
    one = np.array([0, 2], np.int32)
    f2 = model.random_flags(rng, 2)
    keep = []

    def pl(node_idx, pod_off, pod_flags, n_pods=None, n_lists=None):
        arrs = [None if a is None else np.ascontiguousarray(a) for a in (node_idx, pod_off, pod_flags)]
        keep.extend(arrs)
        ptr = [None if a is None else a.ctypes.data for a in arrs]
        nl = n_lists if n_lists is not None else (0 if arrs[0] is None else arrs[0].shape[0])
        npods = n_pods if n_pods is not None else (0 if arrs[2] is None else arrs[2].shape[0])
        return abi.PodLists(nl, ptr[0], ptr[1], ptr[2], npods)

    fresh1 = new_nodes(rng, 1)
    idx_far = np.array([n], np.int64)
    big = np.array([0, (1 << 31) - 1], np.int32)
    bad = [
        ("node_idx unsorted", pl(np.array([5, 3], np.int64), np.array([0, 1, 2], np.int32), f2)),
        ("node_idx duplicated", pl(np.array([4, 4], np.int64), np.array([0, 1, 2], np.int32), f2)),
        ("node_idx past the end", pl(np.array([n], np.int64), one, f2)),
        ("node_idx negative", pl(np.array([-1], np.int64), one, f2)),
        ("pod_off[0] != 0", pl(np.array([3], np.int64), np.array([1, 2], np.int32), f2)),
        ("pod_off decreasing", pl(np.array([3, 9], np.int64), np.array([0, 2, 1], np.int32), f2)),
        ("pod_off[n_lists] != n_pods", pl(np.array([3], np.int64), np.array([0, 1], np.int32), f2)),
        ("a pod total of 2^31", pl(np.array([0], np.int64), big, f2, n_pods=(1 << 31) - 1)),
        ("NULL node_idx", pl(None, one, f2, n_lists=1)),
        ("NULL pod_off", pl(np.array([3], np.int64), None, f2)),
        ("NULL pod_flags", pl(np.array([3], np.int64), one, None, n_pods=2)),
        ("negative n_lists", pl(np.array([3], np.int64), one, f2, n_lists=-1)),
    ]
    ok_lists = pl(np.array([3], np.int64), np.array([0, 2], np.int32), f2)
    calls = [(what, lambda li=li: raw_call(handle, POL, li)) for what, li in bad]
    cols = {k: fresh1[k].ctypes.data for k in COLS}
    calls += [
        ("idx outside the snapshot", lambda: raw_call(handle, POL, ok_lists, 1, idx_far.ctypes.data, cols)),
        ("NULL idx", lambda: raw_call(handle, POL, ok_lists, 1, None, cols)),
        ("NULL overwrite columns", lambda: raw_call(handle, POL, ok_lists, 1, idx_far.ctypes.data, {})),
        ("NULL out_outcome", lambda: raw_call(handle, POL, ok_lists, outcome=False)),
    ]
    ref = helpers.oracle_apply(POL, res.soa, res.pods, variant=1)
    for what, call in calls:
        before = handle.launch_count()
        rc = call()
        assert rc == INVALID, (what, rc, handle.last_error())
        assert handle.launch_count() == before, what
        # the pod-list snapshot and its outputs are what they were: an empty call reports nothing, with the same counters
        rc, n_out, *_, cnt = handle.apply_state_delta_pods(POL, None, none, new_nodes(rng, 0), res.soa["ds_rev"], 16)
        assert rc == ref[0] and n_out == 0 and cnt == ref[4], (what, rc, n_out)
    frc, nxt, act, oc = handle.fetch_outputs_pods(n)
    assert frc == 0 and np.array_equal(nxt, ref[1]) and np.array_equal(act, ref[2]) and np.array_equal(oc, ref[3])


def test_pod_list_snapshot_residency(handle):
    """Which calls leave, keep and drop the pod-list snapshot; the node entry points never see it."""
    rng = np.random.default_rng(41)
    soa, pods = wide_snapshot(rng, 6000)
    none = np.zeros(0, np.int64)
    empty = new_nodes(rng, 0)

    def pods_resident():
        rc = handle.apply_state_delta_pods(POL, None, none, empty, soa["ds_rev"], 6016)[0]
        frc = handle.fetch_outputs_pods(6000)[0]
        assert (rc == INVALID) == (frc == INVALID), (rc, frc)
        if rc == INVALID:
            assert "no resident pod-list snapshot" in handle.last_error() or "no resident pod-list outputs" in handle.last_error()
        return rc != INVALID

    def node_calls_find_nothing():
        assert handle.apply_state_delta(POL, 6000, none, empty, soa["ds_rev"])[0] == INVALID
        assert handle.apply_state_delta_sparse(POL, none, empty, soa["ds_rev"], 16)[0] == INVALID
        assert handle.apply_state_delta_splice(POL, None, none, empty, soa["ds_rev"], 16)[0] == INVALID
        assert handle.apply_state_delta_reorder(POL, None, none, empty, soa["ds_rev"], 16)[0] == INVALID
        assert handle.fetch_outputs(6000)[0] == INVALID
        assert handle.simulate_rollout(POL, 6000, 1, want_final=False)[0] == INVALID

    def leave():
        PodResident(handle, POL, soa, pods)
        assert pods_resident()

    leave()
    node_calls_find_nothing()
    assert pods_resident()   # the rejected node calls left it as it was
    res = PodResident(handle, POL, soa, pods)
    res.step(POL, model.random_lists(rng, pods["pod_off"], 0.01, "mixed"), none, empty, 6016, "delta")
    node_calls_find_nothing()
    assert pods_resident()
    # a call with pod lists but without actuator_outcome, the node-only calls, BuildState and a simulation drop it
    droppers = [
        ("pods without outcome", lambda: handle.apply_state(POL, soa, pods, want_outcome=False)),
        ("without pods", lambda: handle.apply_state(POL, soa)),
        ("packed", lambda: handle.apply_state_packed(POL, soa)),
        ("build_state", lambda: handle.build_state(soa["state"][:10], np.zeros(10, np.int32), np.array([10], np.int32))),
    ]
    for what, call in droppers:
        leave()
        call()
        assert not pods_resident(), what
    # a node delta and a simulation run on the node snapshot, which a pod-list call never leaves: each follows a call
    # without pods, which has dropped the pod-list snapshot already
    for what, call in (("node delta", lambda: handle.apply_state_delta(POL, 6000, none, empty, soa["ds_rev"])),
                       ("simulation", lambda: handle.simulate_rollout(POL, 6000, 1, want_final=False))):
        leave()
        handle.apply_state(POL, soa)
        rc = call()[0]
        assert rc != INVALID, (what, handle.last_error())
        assert not pods_resident(), what
    # ust_apply_state_device leaves it alone
    import torch
    leave()
    d = {k: torch.from_numpy(np.ascontiguousarray(soa[k])).cuda() for k in ("state", "flags", "pod_rev", "ds_idx", "ds_rev")}
    nxt = torch.zeros(6000, dtype=torch.uint8, device="cuda")
    act = torch.zeros(6000, dtype=torch.int16, device="cuda")
    handle.apply_state_device(POL, 6000, d["state"].data_ptr(), d["flags"].data_ptr(), d["pod_rev"].data_ptr(), d["ds_idx"].data_ptr(),
                              3, d["ds_rev"].data_ptr(), nxt.data_ptr(), act.data_ptr())
    handle.sync()
    assert pods_resident()
    # a pod-list ust_apply_state rejected by its offset check keeps it
    bad = {"pod_off": pods["pod_off"].copy(), "pod_flags": pods["pod_flags"]}
    bad["pod_off"][0] = 1
    assert handle.apply_state(POL, soa, bad)[0] == INVALID
    assert pods_resident()
