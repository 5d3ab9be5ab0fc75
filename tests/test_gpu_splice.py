"""ust_apply_state_delta_splice on the H100: membership changes of the resident snapshot (nodes leave, nodes join) with
overwrites, against the oracle on the numpy-spliced arrays. After every call: the reported nodes are exactly the inserted
ones plus the survivors whose output changed, patching the spliced previous outputs gives the oracle's outputs, the
counters match, and the truncated path hands out the same outputs through ust_fetch_outputs."""
import numpy as np
import pytest

import helpers
import splice_model
from helpers import abi
from ust import lib as ustlib, synth

pytestmark = pytest.mark.gpu

COLS = ("state", "flags", "pod_rev", "ds_idx")
INVALID = abi.K["UST_ERR_INVALID_ARGUMENT"]
TRUNCATED = abi.K["UST_ERR_TRUNCATED"]


@pytest.fixture(scope="module")
def handle():
    h = ustlib.Handle(0)
    yield h
    h.close()


class Resident:
    """What the caller holds: the snapshot the device has resident and the outputs of the last call on it."""

    def __init__(self, handle, pol, soa):
        self.h, self.soa = handle, soa
        rc, self.nxt, self.act, _, cnt = handle.apply_state(pol, soa, want_outcome=False)
        ref = helpers.oracle_apply(pol, soa, variant=1)
        helpers.assert_same((rc, self.nxt, self.act, None, cnt), (ref[0], ref[1], ref[2], None, ref[4]), "full call")

    @property
    def n(self):
        return int(self.soa["state"].shape[0])

    def splice(self, pol, rm, ib, ins, idx, fresh, cap, what=""):
        new = {k: splice_model.splice(self.soa[k], rm, ib, ins[k]) for k in COLS}
        for k in COLS:
            new[k][idx] = fresh[k]
        new["ds_rev"] = self.soa["ds_rev"]
        sp = dict(remove_idx=rm, insert_before=ib, **{k: ins[k] for k in COLS})
        rc, n_out, oi, on, oa, cnt = self.h.apply_state_delta_splice(pol, sp, idx, fresh, new["ds_rev"], cap)
        ref = helpers.oracle_apply(pol, new, variant=1)
        prev_n = splice_model.splice(self.nxt, rm, ib, np.full(ib.shape[0], 0xFF, np.uint8))
        prev_a = splice_model.splice(self.act, rm, ib, np.zeros(ib.shape[0], np.uint16))
        inserted = splice_model.splice(np.zeros(self.n, bool), rm, ib, np.ones(ib.shape[0], bool))
        expect = (ref[1] != prev_n) | (ref[2] != prev_a)
        assert np.all(expect[inserted]), what   # every inserted node is reported
        assert n_out == int(expect.sum()), (what, n_out, int(expect.sum()))
        if n_out > cap:
            # too many changes for the caller's arrays: UST_ERR_TRUNCATED, unless the call aborted (its code wins)
            assert rc == (TRUNCATED if ref[0] == 0 else ref[0]), (what, rc, ref[0])
            frc, nxt, act = self.h.fetch_outputs(ref[1].shape[0])
            assert frc == 0
        else:
            assert rc == ref[0], (what, rc, ref[0])
            assert np.array_equal(oi[:n_out], np.nonzero(expect)[0]), what   # new-index order, exactly those nodes
            nxt, act = prev_n, prev_a
            nxt[oi[:n_out]] = on[:n_out]
            act[oi[:n_out]] = oa[:n_out]
        assert np.array_equal(nxt, ref[1]) and np.array_equal(act, ref[2]), what
        assert cnt == ref[4], (what, cnt, ref[4])
        self.soa, self.nxt, self.act = new, nxt, act
        return rc

    def sparse(self, pol, idx, fresh, cap, what=""):
        for k in COLS:
            self.soa[k][idx] = fresh[k]
        rc, n_out, oi, on, oa, cnt = self.h.apply_state_delta_sparse(pol, idx, fresh, self.soa["ds_rev"], cap)
        ref = helpers.oracle_apply(pol, self.soa, variant=1)
        assert n_out == int(np.sum((ref[1] != self.nxt) | (ref[2] != self.act))), what
        if n_out > cap:
            assert rc == (TRUNCATED if ref[0] == 0 else ref[0])
            _, self.nxt, self.act = self.h.fetch_outputs(self.n)
        else:
            assert rc == ref[0]
            self.nxt[oi[:n_out]] = on[:n_out]
            self.act[oi[:n_out]] = oa[:n_out]
        assert np.array_equal(self.nxt, ref[1]) and np.array_equal(self.act, ref[2]) and cnt == ref[4], what

    def dense(self, pol, what=""):
        empty = {k: self.soa[k][:0] for k in COLS}
        got = self.h.apply_state_delta(pol, self.n, np.zeros(0, np.int64), empty, self.soa["ds_rev"], want_outcome=False)
        ref = helpers.oracle_apply(pol, self.soa, variant=1)
        helpers.assert_same((got[0], got[1], got[2], None, got[4]), (ref[0], ref[1], ref[2], None, ref[4]), what)
        self.nxt, self.act = got[1], got[2]


def overwrites(rng, n, frac, p_err=0.0):
    m = min(n, int(round(n * frac)))
    idx = np.sort(rng.choice(n, size=m, replace=False)).astype(np.int64) if m else np.zeros(0, np.int64)
    fresh, _ = helpers.random_soa(rng, m, wild=True, p_err=p_err)
    return idx, {k: fresh[k] for k in COLS}


def new_nodes(rng, m, p_err=0.0, state=None):
    fresh, _ = helpers.random_soa(rng, m, wild=True, p_err=p_err)
    if state is not None:
        fresh["state"] = np.full(m, state, np.uint8)
    return {k: fresh[k] for k in COLS}


@pytest.mark.parametrize("n", [0, 1, 3071, 3072, 3073, 4097, 700_001])
def test_splice_chains(handle, n):
    """Reconcile chains with removal / insertion fractions 0, 0.001, 0.01 and 0.3 and 1 % overwrites, policy changes, an
    abort, a slot budget that moves; delta and sparse delta calls in between."""
    rng = np.random.default_rng(5000 + n)
    soa, _ = helpers.random_soa(rng, n, wild=True)
    res = Resident(handle, abi.make_policy(max_parallel_upgrades=0, max_unavailable="30%"), soa)
    step = 0
    for frac in (0.0, 0.001, 0.01, 0.3):
        for rep in range(3):
            n_old = res.n
            pol = (helpers.random_policy(rng) if rep == 1 else
                   abi.make_policy(max_parallel_upgrades=max(1, n_old // 9), max_unavailable="55%") if rep == 2 else
                   abi.make_policy(max_parallel_upgrades=0, max_unavailable="30%"))
            rm, ib = splice_model.random_splice(rng, n_old, frac, frac if rep != 1 else frac / 2 + 1e-9)
            if frac and ib.size == 0 and rep == 0:
                ib = np.array([int(rng.integers(0, n_old + 1))], np.int64)   # small snapshots: still one join
            ins = new_nodes(rng, ib.shape[0], p_err=3e-3 if step == 5 else 0.0)
            n_new = n_old - rm.shape[0] + ib.shape[0]
            idx, fresh = overwrites(rng, n_new, 0.01, p_err=2e-4 if step == 5 else 0.0)
            cap = n_new // 4 + 16 if step % 4 != 3 else 2   # some calls overflow the caller's arrays
            res.splice(pol, rm, ib, ins, idx, fresh, cap, f"n={n} frac={frac} rep={rep}")
            step += 1
        res.sparse(pol, *overwrites(rng, res.n, 0.01), cap=res.n // 4 + 16, what=f"sparse after frac={frac}")
        res.dense(pol, f"dense after frac={frac}")


def test_splice_edges(handle):
    """Inserting at 0 and at n, many inserts at one position, removing and inserting at the same position, a new size
    crossing a tile boundary (3072 nodes) both ways, a slot cut that moves because candidates are inserted before it,
    removing every node and inserting into the empty snapshot."""
    rng = np.random.default_rng(77)
    soa, _ = helpers.random_soa(rng, 3072, wild=True)
    pol = abi.make_policy(max_parallel_upgrades=0, max_unavailable="30%")
    res = Resident(handle, pol, soa)
    none = np.zeros(0, np.int64)
    no_ow = (none, new_nodes(rng, 0))

    def go(rm, ib, what, pol=pol, ins=None):
        rm, ib = np.asarray(rm, np.int64), np.asarray(ib, np.int64)
        res.splice(pol, rm, ib, ins if ins is not None else new_nodes(rng, ib.shape[0]), *no_ow, cap=res.n + 64, what=what)

    go(none, [0, 0, 0], "insert at 0")                                                   # 3075: across the boundary
    go(none, [res.n] * 2, "insert at n")
    go(np.arange(0, 6), none, "remove the head")                                        # back to 3071
    go(none, [1500] * 700, "many inserts at one position")
    go([5, 6, 7, 800], [5, 5, 7, 800, 800], "remove and insert at the same positions")
    go(np.arange(res.n - 702, res.n), none, "remove the tail: below the boundary")
    # a limited slot budget: upgrade-required candidates inserted at the head take the slots the cut had granted
    cut = abi.make_policy(max_parallel_upgrades=40, max_unavailable=None)
    go(none, none, "slot budget", pol=cut)
    go(none, np.zeros(120, np.int64), "candidates inserted before the cut", pol=cut,
       ins=new_nodes(rng, 120, state=abi.UST_STATE_UPGRADE_REQUIRED))
    res.dense(cut, "dense after the cut moved")
    go(np.arange(res.n), none, "remove every node")
    assert res.n == 0
    go(none, [0] * 4097, "insert into the empty snapshot")
    res.sparse(pol, *overwrites(rng, res.n, 0.02), cap=16, what="sparse, truncated")


@pytest.mark.parametrize("n", [2048, 4096])
def test_splice_at_a_multiple_of_the_splice_tile(handle, n):
    """n a multiple of the splice kernel's 2048-position tile: its last CTA holds only position n, where the inserts at
    the end go. Inserts at n, at the last tile boundary and around it, with and without removals next to it."""
    rng = np.random.default_rng(900 + n)
    soa, _ = helpers.random_soa(rng, n, wild=True)
    pol = abi.make_policy(max_parallel_upgrades=0, max_unavailable="30%")
    res = Resident(handle, pol, soa)
    none = np.zeros(0, np.int64)
    cases = [(none, [n] * 5, "inserts at n"),
             ([n - 1], [n - 1, n, n], "remove the last node, insert before and after it"),
             ([2047], [2047, 2048, 2048, n + 7], "around the first tile boundary, and at the end")]
    for rm, ib, what in cases:
        rm, ib = np.asarray(rm, np.int64), np.asarray(ib, np.int64)
        assert ib.max() <= res.n
        res.splice(pol, rm, ib, new_nodes(rng, ib.shape[0]), none, new_nodes(rng, 0), res.n + 64, f"n={n}: {what}")
    # back to exactly n nodes, then once more inserts at the end - with overwrites this time
    res.splice(pol, np.arange(res.n - n, dtype=np.int64), none, new_nodes(rng, 0), none, new_nodes(rng, 0), res.n + 64, "shrink")
    assert res.n == n
    idx, fresh = overwrites(rng, n + 4, 0.01)
    res.splice(pol, none, np.full(4, n, np.int64), new_nodes(rng, 4), idx, fresh, n + 64, f"n={n}: inserts at n, overwrites")


def test_splice_noop_is_delta_sparse(handle):
    """splice == NULL and an empty splice behave like ust_apply_state_delta_sparse."""
    rng = np.random.default_rng(3)
    soa, _ = helpers.random_soa(rng, 5000, wild=True)
    pol = abi.make_policy(max_parallel_upgrades=0, max_unavailable="30%")
    res = Resident(handle, pol, soa)
    for sp in (None, dict(remove_idx=np.zeros(0, np.int64), insert_before=np.zeros(0, np.int64))):
        idx, fresh = overwrites(rng, res.n, 0.01)
        launches = handle.launch_count()
        for k in COLS:
            res.soa[k][idx] = fresh[k]
        rc, n_out, oi, on, oa, cnt = handle.apply_state_delta_splice(pol, sp, idx, fresh, res.soa["ds_rev"], 5000)
        ref = helpers.oracle_apply(pol, res.soa, variant=1)
        res.nxt[oi[:n_out]] = on[:n_out]
        res.act[oi[:n_out]] = oa[:n_out]
        assert rc == ref[0] and np.array_equal(res.nxt, ref[1]) and np.array_equal(res.act, ref[2]) and cnt == ref[4]
        # what ust_apply_state_delta_sparse launches: patch, streaming + verification, the three diff kernels - no splice
        assert handle.launch_count() - launches == (1 if idx.size else 0) + 2 + 3


def test_splice_contract_errors_leave_the_snapshot(handle):
    rng = np.random.default_rng(11)
    soa, _ = helpers.random_soa(rng, 4097, wild=True)
    pol = abi.make_policy(max_parallel_upgrades=0, max_unavailable="30%")
    res = Resident(handle, pol, soa)
    n = res.n
    ins2 = new_nodes(rng, 2)
    none = np.zeros(0, np.int64)
    bad = [
        ("unsorted remove_idx", dict(remove_idx=[5, 3], insert_before=none), none),
        ("duplicate remove_idx", dict(remove_idx=[3, 3], insert_before=none), none),
        ("remove_idx out of range", dict(remove_idx=[n], insert_before=none), none),
        ("negative remove_idx", dict(remove_idx=[-1], insert_before=none), none),
        ("insert_before > n", dict(remove_idx=none, insert_before=[0, n + 1], **ins2), none),
        ("decreasing insert_before", dict(remove_idx=none, insert_before=[7, 6], **ins2), none),
        ("NULL insert arrays", dict(remove_idx=none, insert_before=[0, 1]), none),
        ("idx outside the new size", dict(remove_idx=[0, 1, 2], insert_before=none), np.array([n - 3], np.int64)),
    ]
    for what, sp, idx in bad:
        fresh = new_nodes(rng, idx.shape[0])
        rc = handle.apply_state_delta_splice(pol, sp, idx, fresh, res.soa["ds_rev"], 64)[0]
        assert rc == INVALID, (what, rc)
        assert "splice" in handle.last_error() or "outside the snapshot" in handle.last_error(), (what, handle.last_error())
    # the resident snapshot and outputs are what they were: an empty sparse call reports nothing and agrees with the oracle
    res.sparse(pol, none, new_nodes(rng, 0), cap=16, what="after the rejected calls")
    res.splice(pol, np.array([0], np.int64), np.array([n - 1], np.int64), new_nodes(rng, 1), none, new_nodes(rng, 0), 64, "and splices")
    # a rollout simulation leaves the simulated snapshot resident but no outputs of it to compare with
    rc, _, _, _ = handle.simulate_rollout(pol, res.n, 1, want_final=False)
    assert rc not in (abi.K["UST_ERR_CUDA"], INVALID), handle.last_error()
    rc = handle.apply_state_delta_splice(pol, dict(remove_idx=[0], insert_before=none), none, new_nodes(rng, 0), soa["ds_rev"], 16)[0]
    assert rc == INVALID and "no resident outputs" in handle.last_error()
    # no resident snapshot (BuildState shares the staging arrays)
    handle.build_state(soa["state"][:10], np.zeros(10, np.int32), np.array([10], np.int32))
    rc = handle.apply_state_delta_splice(pol, None, none, new_nodes(rng, 0), soa["ds_rev"], 16)[0]
    assert rc == INVALID


def test_splice_c3_10m(handle):
    """A 10 M-node C3 snapshot: 0.1 % leave, 0.1 % join at random positions, 1 % re-encoded."""
    cfg = synth.CONFIGS["C3"]
    soa = synth.make_nodes(cfg["n"], cfg["seed"])
    pol = synth.config_policy("C3")
    res = Resident(handle, pol, soa)
    rng = np.random.default_rng(10)
    for rep in range(2):
        rm, ib = splice_model.random_splice(rng, res.n, 0.001, 0.001)
        ins = {k: v[:ib.shape[0]].copy() for k, v in synth.make_nodes(ib.shape[0], 100 + rep).items() if k in COLS}
        n_new = res.n - rm.shape[0] + ib.shape[0]
        idx = np.sort(rng.choice(n_new, size=n_new // 100, replace=False)).astype(np.int64)
        src = synth.make_nodes(idx.shape[0], 200 + rep)
        fresh = {k: src[k] for k in COLS}
        res.splice(pol, rm, ib, ins, idx, fresh, n_new // 8, f"C3 rep={rep}")
