"""ust_apply_state_delta_pods_reorder on the H100: reconcile chains in which nodes of the resident pod-list snapshot join,
leave and move with their pod lists, lists are replaced (on nodes that stay and on every inserted node) and nodes are
overwritten, against the oracle on the numpy-reordered arrays. After every call the reported nodes are exactly the
inserted ones plus those whose next_state, actions or actuator_outcome changed wherever they moved, patching the
reordered previous outputs gives the oracle's outputs, the counters match, and the truncated path hands out the same
outputs through ust_fetch_outputs_pods. Plain ust_apply_state_delta_pods calls in between show that the host's list
lengths followed the reorder."""
import numpy as np
import pytest

import helpers
import pods_delta_model
import pods_reorder_model as model
import reorder_model
from helpers import abi
from ust import lib as ustlib, synth

pytestmark = pytest.mark.gpu

COLS = ("state", "flags", "pod_rev", "ds_idx")
INVALID = abi.K["UST_ERR_INVALID_ARGUMENT"]
TRUNCATED = abi.K["UST_ERR_TRUNCATED"]
REVISION_HASH = abi.K["UST_ERR_REVISION_HASH"]
# streaming + verification, the three diff kernels; the pod-summary kernel when the policy evaluates actuators; the patch
# with overwrites; one scatter launch for lists that keep their lengths, two (run table, relayout) otherwise; a reorder:
# the node gather, the pod run table and the pod gather
CALL, DIFF, PATCH, SCATTER, RELAYOUT, REORDER = 2, 3, 1, 1, 2, 3
POD_BLOCK = 4096  # nodes per block of the pod-summary kernel
POL_KW = dict(max_parallel_upgrades=0, max_unavailable="30%", pod_deletion_enabled=True,
              pod_deletion={"force": False, "deleteEmptyDir": False}, drain={"enable": True, "force": False, "deleteEmptyDir": False},
              wait_for_completion={"podSelector": "app=batch", "timeoutSeconds": 0}, evaluate_actuators=True)
POL = abi.make_policy(**POL_KW)
ORDERS = ("identity", "moves", "swap", "reverse", "shuffle", "none", "insert_only", "mixed")


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


def base_launches(pol, n):
    """ust_apply_state_delta_pods without lists or overwrites on a snapshot of n > 0 nodes."""
    return (1 if pol.auto_upgrade and pol.evaluate_actuators else 0) + CALL + DIFF


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

    def _check(self, pol, call, soa, pods, prev, cap, inserted, what):
        before = self.h.launch_count()
        rc, n_out, oi, on, oa, oo, cnt = call()
        launched = self.h.launch_count() - before
        ref = helpers.oracle_apply(pol, soa, pods, variant=1)
        nxt, act, oc = prev
        expect = (ref[1] != nxt) | (ref[2] != act) | (ref[3] != oc)
        assert np.all(expect[inserted]), what   # every inserted node is reported
        assert n_out == int(expect.sum()), (what, n_out, int(expect.sum()))
        if n_out > cap:
            assert rc == (TRUNCATED if ref[0] == 0 else ref[0]), (what, rc, ref[0])
            frc, nxt, act, oc = self.h.fetch_outputs_pods(soa["state"].shape[0])
            assert frc == 0, (what, self.h.last_error())
        else:
            assert rc == ref[0], (what, rc, ref[0], self.h.last_error())
            assert np.array_equal(oi[:n_out], np.nonzero(expect)[0]), what   # new-index order, exactly those nodes
            nxt, act, oc = nxt.copy(), act.copy(), oc.copy()
            nxt[oi[:n_out]] = on[:n_out]
            act[oi[:n_out]] = oa[:n_out]
            oc[oi[:n_out]] = oo[:n_out]
        helpers.assert_same((rc, nxt, act, oc, cnt), (rc, ref[1], ref[2], ref[3], ref[4]), what)
        self.soa, self.pods, self.nxt, self.act, self.oc = soa, pods, nxt, act, oc
        return rc, n_out, launched

    def reorder(self, pol, order, ins, lists, idx, fresh, cap, what=""):
        """`order`: the target order (reorder_model.runs_of); `ins`: the inserted nodes' columns; `lists`: index the new
        snapshot and name every inserted node."""
        order = np.asarray(order, np.int64)
        src, ln = reorder_model.runs_of(order)
        n_ins = int(np.sum(order < 0))
        soa = {k: reorder_model.reorder(self.soa[k], src, ln, ins[k]) for k in COLS}
        for k in COLS:
            soa[k][idx] = fresh[k]
        soa["ds_rev"] = self.soa["ds_rev"]
        li = lists if lists is not None else {"node_idx": np.zeros(0, np.int64), "pod_off": np.zeros(1, np.int32),
                                             "pod_flags": np.zeros(0, np.uint16)}
        pods = dict(zip(("pod_off", "pod_flags"),
                        model.reorder(self.pods["pod_off"], self.pods["pod_flags"], src, ln, li["node_idx"], li["pod_off"], li["pod_flags"])))
        prev = (reorder_model.reorder(self.nxt, src, ln, np.full(n_ins, 0xFF, np.uint8)),
                reorder_model.reorder(self.act, src, ln, np.zeros(n_ins, np.uint16)),
                reorder_model.reorder(self.oc, src, ln, np.full(n_ins, 0xFF, np.uint8)))
        ro = dict(run_src=src, run_len=ln, **{k: ins[k] for k in COLS})
        return self._check(pol, lambda: self.h.apply_state_delta_pods_reorder(pol, ro, lists, idx, fresh, soa["ds_rev"], cap),
                           soa, pods, prev, cap, order < 0, what)

    def pods_delta(self, pol, lists, idx, fresh, cap, what=""):
        """A plain ust_apply_state_delta_pods call; returns (rc, n_out, launches, path launches)."""
        soa = {k: v.copy() for k, v in self.soa.items()}
        for k in COLS:
            soa[k][idx] = fresh[k]
        pods, path = self.pods, 0
        if lists is not None and len(lists["node_idx"]):
            off, pf = pods_delta_model.replace(pods["pod_off"], pods["pod_flags"], lists["node_idx"], lists["pod_off"], lists["pod_flags"])
            same = np.array_equal(np.diff(lists["pod_off"]), np.diff(pods["pod_off"])[lists["node_idx"]])
            path = SCATTER if same else RELAYOUT
            self.paths.add("scatter" if same else "relayout")
            pods = {"pod_off": off, "pod_flags": pf}
        none = np.zeros(self.n, bool)
        rc, n_out, launched = self._check(pol, lambda: self.h.apply_state_delta_pods(pol, lists, idx, fresh, soa["ds_rev"], cap),
                                          soa, pods, (self.nxt, self.act, self.oc), cap, none, what)
        return rc, n_out, launched, path

    def empty(self, pol, what=""):
        idx, fresh = overwrites(np.random.default_rng(0), self.n, 0.0, idx=[])
        return self.pods_delta(pol, None, idx, fresh, self.n + 16, what)


def wide_snapshot(rng, n):
    """random_soa with pod lists, and with the last node in a state whose actuator reads its list (pod deletion)."""
    soa, pods = helpers.random_soa(rng, n, wild=True, with_pods=True)
    if n:
        soa["state"][-1] = abi.UST_STATE_POD_DELETION_REQUIRED
    return soa, pods


def tail_reorder(rng, res):
    """A reorder (nodes moved) with a new list for the last new node whose end falls inside the final 16 bytes of
    pod_flags, with a total that is no multiple of 8 pods, and that node in a state whose actuator reads the list."""
    order = reorder_model.random_order(rng, res.n, "moves", k=5)
    src, ln = reorder_model.runs_of(order)
    off, _ = model.moved(res.pods["pod_off"], res.pods["pod_flags"], src, ln)
    before = int(off[-2])                    # pods ahead of the last list
    tl = (5 - before) % 8                    # the new total is 5 mod 8 ...
    tl += 8 if tl < 3 else 0                 # ... and the list at least 3 pods long
    li = {"node_idx": np.array([order.size - 1], np.int64), "pod_off": np.array([0, tl], np.int32),
          "pod_flags": pods_delta_model.random_flags(rng, tl)}
    last = new_nodes(rng, 1)
    last["state"][:] = abi.UST_STATE_POD_DELETION_REQUIRED
    return order, li, np.array([order.size - 1], np.int64), last


def random_step(rng, res, kind, f=0.0):
    k = int(rng.integers(1, 12))
    order = reorder_model.random_order(rng, res.n, kind, k=k, f_remove=f, f_insert=f)
    return order, new_nodes(rng, int(np.sum(order < 0)))


@pytest.mark.parametrize("n", [1, 127, POD_BLOCK - 1, POD_BLOCK, POD_BLOCK + 1, 65_537, 700_001])
def test_pods_reorder_chains(handle, n):
    """Every order kind (and mixed with 0.1 % and 1 % of the nodes leaving and joining), each with list replacements of
    every kind and overwrites with and without overlap; a plain pod-list delta on the scatter or the relayout path after
    each; the launch count pinned against the plain delta's."""
    rng = np.random.default_rng(9000 + n)
    soa, pods = wide_snapshot(rng, n)
    res = PodResident(handle, POL, soa, pods)
    steps = [(kind, 0.0) for kind in ORDERS] + [("mixed", 0.001), ("mixed", 0.01), ("shuffle", 0.0)]
    for step, (kind, f) in enumerate(steps):
        if res.n == 0 and kind not in ("insert_only", "none", "identity", "mixed"):
            kind = "insert_only"
        order, ins = random_step(rng, res, kind, f)
        lkind = pods_delta_model.KINDS[step % len(pods_delta_model.KINDS)]
        li = model.random_lists(rng, order, res.pods["pod_off"], (0.0, 0.001, 0.01, 0.3)[step % 4], lkind)
        if step % 3 == 0:
            idx, fresh = overwrites(rng, order.size, 0.01)
        elif step % 3 == 1:
            idx, fresh = overwrites(rng, order.size, 0.0, idx=li["node_idx"][::2])
        else:
            idx, fresh = overwrites(rng, order.size, 0.0, idx=[])
        cap = order.size + 16 if step % 5 != 4 else 2
        what = f"n={n} {kind} f={f} lists={lkind}"
        _, _, launched = res.reorder(POL, order, ins, li, idx, fresh, cap, what)
        if kind == "none":
            assert res.n == 0
        _, _, base, _ = res.empty(POL, f"empty after {what}")
        if res.n:
            assert base == base_launches(POL, res.n), (what, base)
        assert launched == base + (PATCH if idx.size else 0) + REORDER, (what, "launches", launched, base)
        # a plain pod-list delta on the reordered snapshot: list lengths as the host now knows them
        if res.n:
            pk = "same" if step % 2 == 0 else "mixed"
            pl = pods_delta_model.random_lists(rng, res.pods["pod_off"], 0.01, pk)
            pidx, pfresh = overwrites(rng, res.n, 0.01)
            _, _, launched, path = res.pods_delta(POL, pl, pidx, pfresh, res.n + 16, f"pods delta ({pk}) after {what}")
            assert launched == base + (PATCH if pidx.size else 0) + path, (what, "plain launches", launched, base, path)
    order, li, idx, last = tail_reorder(rng, res)
    res.reorder(POL, order, new_nodes(rng, 0), li, idx, last, order.size + 16, f"n={n} tail list")
    assert int(res.pods["pod_off"][-1]) % 8 == 5
    # and a plain delta with the tail list replaced again at a changed length
    li = {"node_idx": np.array([res.n - 1], np.int64), "pod_off": np.array([0, 3], np.int32),
          "pod_flags": pods_delta_model.random_flags(rng, 3)}
    res.pods_delta(POL, li, *overwrites(rng, res.n, 0.0, idx=[]), res.n + 16, f"n={n} plain delta on the tail")
    assert res.paths == {"scatter", "relayout"} or n < 1000, res.paths


def test_reorder_none_is_delta_pods(handle):
    """reorder == NULL gives what ust_apply_state_delta_pods gives, with the same launches."""
    rng = np.random.default_rng(3)
    soa, pods = wide_snapshot(rng, 20_000)
    for kind in ("same", "mixed"):
        li = pods_delta_model.random_lists(rng, pods["pod_off"], 0.01, kind)
        idx, fresh = overwrites(rng, 20_000, 0.01)
        got = []
        for fn in ("apply_state_delta_pods_reorder", "apply_state_delta_pods"):
            PodResident(handle, POL, soa, pods)
            before = handle.launch_count()
            args = (POL, None, li, idx, fresh, soa["ds_rev"], 20_016) if fn.endswith("reorder") else (POL, li, idx, fresh, soa["ds_rev"], 20_016)
            rc, n_out, oi, on, oa, oo, cnt = getattr(handle, fn)(*args)
            got.append((rc, n_out, oi[:n_out].copy(), on[:n_out].copy(), oa[:n_out].copy(), oo[:n_out].copy(), cnt,
                        handle.launch_count() - before))
        a, b = got
        assert a[0] == b[0] and a[1] == b[1] and a[6] == b[6] and a[7] == b[7], (kind, a[0], b[0], a[1], b[1], a[7], b[7])
        for x, y in zip(a[2:6], b[2:6]):
            assert np.array_equal(x, y), kind


def revision_hash_node(rng):
    bad = new_nodes(rng, 1)
    bad["state"][:] = abi.UST_STATE_DONE | abi.UST_HOT_REVISION_HASH_ERROR
    bad["flags"][:] &= ~np.uint32(abi.UST_F_POD_ORPHANED)
    bad["ds_idx"][:] = 0
    return bad


def test_aborts_and_truncation(handle):
    """A revision-hash abort moved through the snapshot, with and without truncation, then UST_ERR_TRUNCATED followed by
    ust_fetch_outputs_pods, then a plain pod-list delta."""
    rng = np.random.default_rng(22)
    soa, pods = wide_snapshot(rng, 30_000)
    res = PodResident(handle, POL, soa, pods)
    order, ins = random_step(rng, res, "mixed", 0.01)
    li = model.random_lists(rng, order, res.pods["pod_off"], 0.01, "mixed")
    rc, _, _ = res.reorder(POL, order, ins, li, np.array([order.size // 3], np.int64), revision_hash_node(rng), order.size + 16, "abort")
    assert rc == REVISION_HASH
    # the aborting node moved to the front: few outputs change, truncated at max_out = 0
    ident = np.arange(res.n, dtype=np.int64)
    order = np.insert(np.delete(ident, res.n // 3), 0, res.n // 3)
    li = model.random_lists(rng, order, res.pods["pod_off"], 0.05, "odd")
    rc, n_out, _ = res.reorder(POL, order, new_nodes(rng, 0), li, np.array([res.n // 2], np.int64), revision_hash_node(rng), 0,
                               "abort moved to the front, truncated")
    assert rc == REVISION_HASH and n_out > 0
    # repair the aborting nodes, shuffle, change lists and truncate
    order = reorder_model.random_order(rng, res.n, "shuffle")
    inv = np.argsort(order)
    idx = np.sort(inv[[0, res.n // 2]]).astype(np.int64)
    fresh = new_nodes(rng, 2)
    fresh["state"] &= np.uint8(abi.UST_HOT_STATE_MASK)
    li = model.random_lists(rng, order, res.pods["pod_off"], 0.3, "mixed")
    rc, n_out, _ = res.reorder(POL, order, new_nodes(rng, 0), li, idx, fresh, 3, "truncated")
    assert rc == TRUNCATED and n_out > 3
    res.pods_delta(POL, pods_delta_model.random_lists(rng, res.pods["pod_off"], 0.01, "same"), *overwrites(rng, res.n, 0.01),
                   cap=res.n, what="after the truncated call")


def test_contract_errors_leave_the_snapshot(handle):
    rng = np.random.default_rng(31)
    soa, pods = wide_snapshot(rng, 5000)
    res = PodResident(handle, POL, soa, pods)
    n = res.n
    none = np.zeros(0, np.int64)
    ins2 = new_nodes(rng, 2)
    f2 = pods_delta_model.random_flags(rng, 2)

    def lists(node_idx, pod_off, n_pods=None):
        pod_off = np.asarray(pod_off, np.int32)
        return {"node_idx": np.asarray(node_idx, np.int64), "pod_off": pod_off,
                "pod_flags": pods_delta_model.random_flags(rng, int(pod_off[-1]) if n_pods is None else n_pods)}

    keep_all = dict(run_src=[0], run_len=[n])
    two_in = dict(run_src=[0, -1], run_len=[n, 2], **ins2)   # new snapshot of n + 2 nodes, n and n + 1 inserted
    ins_lists = lists([n, n + 1], [0, 1, 3])
    big = {"node_idx": np.array([0], np.int64), "pod_off": np.array([0, (1 << 31) - 1], np.int32), "pod_flags": f2}
    bad = [
        ("run length 0", dict(run_src=[0, 5], run_len=[5, 0]), None, none),
        ("overlapping runs", dict(run_src=[0, 100], run_len=[200, 5]), None, none),
        ("old run past the end", dict(run_src=[n - 3], run_len=[4]), None, none),
        ("inserted runs take fewer", dict(run_src=[-1, 0], run_len=[1, n], **ins2), lists([0], [0, 1]), none),
        ("node_idx unsorted", keep_all, lists([5, 3], [0, 1, 2]), none),
        ("node_idx duplicated", keep_all, lists([4, 4], [0, 1, 2]), none),
        ("node_idx outside the new snapshot", dict(run_src=[0], run_len=[n - 3]), lists([n - 3], [0, 2]), none),
        ("an inserted node without a list", two_in, lists([n], [0, 1]), none),
        ("inserted nodes without lists", two_in, None, none),
        ("pod_off[0] != 0", keep_all, lists([3], [1, 2], n_pods=2), none),
        ("pod_off decreasing", keep_all, lists([3, 9], [0, 2, 1], n_pods=1), none),
        ("a pod total of 2^31", keep_all, big, none),
        ("idx outside the new snapshot", dict(run_src=[1], run_len=[n - 1]), None, np.array([n - 1], np.int64)),
    ]
    ref = helpers.oracle_apply(POL, res.soa, res.pods, variant=1)
    for what, ro, li, idx in bad:
        before = handle.launch_count()
        if what == "a pod total of 2^31":   # no array backs the pod count: the raw structure
            rc = _raw_total(handle, ro, li)
        else:
            rc = handle.apply_state_delta_pods_reorder(POL, ro, li, idx, new_nodes(rng, idx.shape[0]), res.soa["ds_rev"], 64)[0]
        assert rc == INVALID, (what, rc, handle.last_error())
        assert handle.launch_count() == before, what
        rc, n_out, *_, cnt = handle.apply_state_delta_pods(POL, None, none, new_nodes(rng, 0), res.soa["ds_rev"], 16)
        assert rc == ref[0] and n_out == 0 and cnt == ref[4], (what, rc, n_out)
    frc, nxt, act, oc = handle.fetch_outputs_pods(n)
    assert frc == 0 and np.array_equal(nxt, ref[1]) and np.array_equal(act, ref[2]) and np.array_equal(oc, ref[3])
    # the next valid call (the same inserted nodes, now with their lists) matches the oracle
    order = np.concatenate([np.arange(n, dtype=np.int64), [-1, -1]])
    res.reorder(POL, order, ins2, ins_lists, none, new_nodes(rng, 0), n + 16, "after the rejected calls")
    # the node-only delta calls still find nothing resident
    assert handle.apply_state_delta_sparse(POL, none, new_nodes(rng, 0), res.soa["ds_rev"], 16)[0] == INVALID
    assert handle.apply_state_delta_reorder(POL, None, none, new_nodes(rng, 0), res.soa["ds_rev"], 16)[0] == INVALID
    assert handle.fetch_outputs(res.n)[0] == INVALID
    res.empty(POL, "the pod-list snapshot is still resident")
    # no resident pod-list snapshot: a call without pods drops it
    handle.apply_state(POL, res.soa)
    before = handle.launch_count()
    rc = handle.apply_state_delta_pods_reorder(POL, dict(run_src=[0], run_len=[1]), None, none, new_nodes(rng, 0), res.soa["ds_rev"], 16)[0]
    assert rc == INVALID and "no resident pod-list snapshot" in handle.last_error()
    assert handle.launch_count() == before


def _raw_total(handle, ro, li):
    """The call with a replacement list of 2^31 - 1 pods that no array backs (only its offsets are read)."""
    import ctypes as C
    src = np.asarray(ro["run_src"], np.int64)
    ln = np.asarray(ro["run_len"], np.int64)
    r = abi.Reorder(int(src.shape[0]), src.ctypes.data, ln.ctypes.data, 0, None, None, None, None)
    ni, off, pf = li["node_idx"], li["pod_off"], li["pod_flags"]
    pl = abi.PodLists(1, ni.ctypes.data, off.ctypes.data, pf.ctypes.data, (1 << 31) - 1)
    ds_rev = np.ones(3, np.int32)
    oi, on, oa, oo = np.zeros(17, np.int64), np.zeros(17, np.uint8), np.zeros(17, np.uint16), np.zeros(17, np.uint8)
    n_out = C.c_int64(0)
    cnt = abi.Counters()
    return handle._lib.ust_apply_state_delta_pods_reorder(
        handle._h, C.addressof(POL), C.addressof(r), C.addressof(pl), 0, None, None, None, None, None, 3, ds_rev.ctypes.data,
        C.c_int64(16), oi.ctypes.data, on.ctypes.data, oa.ctypes.data, oo.ctypes.data, C.addressof(n_out), C.addressof(cnt))


def test_c4_full_size(handle):
    """C4: 10 M nodes and ~300 M pods: 0.1 % of the nodes moved with 1 % of the lists replaced and 1 % re-encoded, then
    0.1 % leaving and 0.1 % joining with their lists."""
    cfg = synth.CONFIGS["C4"]
    soa = synth.make_nodes(cfg["n"], cfg["seed"])
    pods = synth.make_pods_blocked(cfg["n"], cfg["seed"])
    pol = synth.config_policy("C4")
    res = PodResident(handle, pol, soa, pods)
    rng = np.random.default_rng(4)
    n = res.n
    moved = rng.choice(n, size=n // 1000, replace=False)
    keep = np.delete(np.arange(n, dtype=np.int64), moved)
    order = np.insert(keep, np.sort(rng.integers(0, keep.size + 1, size=moved.size)), rng.permutation(moved))
    li = model.random_lists(rng, order, res.pods["pod_off"], 0.01, "mixed")
    res.reorder(pol, order, new_nodes(rng, 0), li, *overwrites(rng, n, 0.01), cap=n // 8, what="C4 moves")
    order = reorder_model.random_order(rng, res.n, "identity", f_remove=0.001, f_insert=0.001)
    li = model.random_lists(rng, order, res.pods["pod_off"], 0.0, "mixed")
    res.reorder(pol, order, new_nodes(rng, int(np.sum(order < 0))), li, *overwrites(rng, order.size, 0.0, idx=[]), cap=n // 8,
                what="C4 joins and leaves")
