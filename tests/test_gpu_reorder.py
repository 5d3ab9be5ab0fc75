"""ust_apply_state_delta_reorder on the H100: new node orders of the resident snapshot (runs of old nodes and inserted
nodes) with overwrites, against the oracle on the numpy-reordered arrays. After every call: the reported nodes are exactly
the inserted ones plus the nodes whose output changed wherever they moved, patching the reordered previous outputs gives
the oracle's outputs, the counters match, and the truncated path hands out the same outputs through ust_fetch_outputs."""
import numpy as np
import pytest

import helpers
import reorder_model
import splice_model
from helpers import abi
from ust import lib as ustlib, synth

pytestmark = pytest.mark.gpu

COLS = ("state", "flags", "pod_rev", "ds_idx")
INVALID = abi.K["UST_ERR_INVALID_ARGUMENT"]
TRUNCATED = abi.K["UST_ERR_TRUNCATED"]
TILE = 2048  # new positions per CTA of ust_reorder_kernel
POL = dict(max_parallel_upgrades=0, max_unavailable="30%")


@pytest.fixture(scope="module")
def handle():
    h = ustlib.Handle(0)
    yield h
    h.close()


def new_nodes(rng, m, p_err=0.0, state=None):
    fresh, _ = helpers.random_soa(rng, m, wild=True, p_err=p_err)
    if state is not None:
        fresh["state"] = np.full(m, state, np.uint8)
    return {k: fresh[k] for k in COLS}


def overwrites(rng, n, frac, p_err=0.0):
    m = min(n, int(round(n * frac)))
    idx = np.sort(rng.choice(n, size=m, replace=False)).astype(np.int64) if m else np.zeros(0, np.int64)
    return idx, new_nodes(rng, m, p_err)


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

    def reorder(self, pol, order, ins, idx, fresh, cap, what=""):
        """`order`: the target order (reorder_model.runs_of); `ins`: the inserted nodes' columns."""
        src, ln = reorder_model.runs_of(order)
        launches = self.h.launch_count()
        new = {k: reorder_model.reorder(self.soa[k], src, ln, ins[k]) for k in COLS}
        for k in COLS:
            new[k][idx] = fresh[k]
        new["ds_rev"] = self.soa["ds_rev"]
        ro = dict(run_src=src, run_len=ln, **{k: ins[k] for k in COLS})
        rc, n_out, oi, on, oa, cnt = self.h.apply_state_delta_reorder(pol, ro, idx, fresh, new["ds_rev"], cap)
        n_launch = self.h.launch_count() - launches
        ref = helpers.oracle_apply(pol, new, variant=1)
        n_ins = int(np.sum(order < 0))
        prev_n = reorder_model.reorder(self.nxt, src, ln, np.full(n_ins, 0xFF, np.uint8))
        prev_a = reorder_model.reorder(self.act, src, ln, np.zeros(n_ins, np.uint16))
        inserted = np.asarray(order) < 0
        expect = (ref[1] != prev_n) | (ref[2] != prev_a)
        assert np.all(expect[inserted]), what   # every inserted node is reported
        assert n_out == int(expect.sum()), (what, n_out, int(expect.sum()))
        if n_out > cap:
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
        return n_launch

    def sparse(self, pol, idx, fresh, cap, what=""):
        for k in COLS:
            self.soa[k][idx] = fresh[k]
        launches = self.h.launch_count()
        rc, n_out, oi, on, oa, cnt = self.h.apply_state_delta_sparse(pol, idx, fresh, self.soa["ds_rev"], cap)
        n_launch = self.h.launch_count() - launches
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
        return n_launch

    def splice(self, pol, rm, ib, ins, what=""):
        new = {k: splice_model.splice(self.soa[k], rm, ib, ins[k]) for k in COLS}
        new["ds_rev"] = self.soa["ds_rev"]
        none = np.zeros(0, np.int64)
        rc, n_out, oi, on, oa, cnt = self.h.apply_state_delta_splice(pol, dict(remove_idx=rm, insert_before=ib, **ins), none,
                                                                     new_nodes(np.random.default_rng(0), 0), new["ds_rev"], new["state"].shape[0] + 16)
        ref = helpers.oracle_apply(pol, new, variant=1)
        nxt = splice_model.splice(self.nxt, rm, ib, np.full(ib.shape[0], 0xFF, np.uint8))
        act = splice_model.splice(self.act, rm, ib, np.zeros(ib.shape[0], np.uint16))
        nxt[oi[:n_out]] = on[:n_out]
        act[oi[:n_out]] = oa[:n_out]
        assert rc == ref[0] and np.array_equal(nxt, ref[1]) and np.array_equal(act, ref[2]) and cnt == ref[4], what
        self.soa, self.nxt, self.act = new, nxt, act

    def dense(self, pol, what=""):
        empty = {k: self.soa[k][:0] for k in COLS}
        got = self.h.apply_state_delta(pol, self.n, np.zeros(0, np.int64), empty, self.soa["ds_rev"], want_outcome=False)
        ref = helpers.oracle_apply(pol, self.soa, variant=1)
        helpers.assert_same((got[0], got[1], got[2], None, got[4]), (ref[0], ref[1], ref[2], None, ref[4]), what)
        self.nxt, self.act = got[1], got[2]


KINDS = ("identity", "moves", "swap", "reverse", "shuffle", "none", "insert_only", "mixed")


@pytest.mark.parametrize("n", [0, 1, TILE - 1, TILE, TILE + 1, 3 * TILE, 3 * TILE + 5, 700_001])
def test_reorder_patterns(handle, n):
    """Every run pattern on each size, with 1 % overwrites; the launch count is the sparse delta's plus one."""
    rng = np.random.default_rng(6000 + n)
    soa, _ = helpers.random_soa(rng, n, wild=True)
    pol = abi.make_policy(**POL)
    res = Resident(handle, pol, soa)
    for step, kind in enumerate(KINDS + ("mixed", "shuffle")):
        if res.n == 0 and kind not in ("insert_only", "none", "identity", "mixed"):
            kind = "insert_only"
        f = 0.01 if step == len(KINDS) else (0.2 if kind == "mixed" else 0.0)
        order = reorder_model.random_order(rng, res.n, kind, k=int(rng.integers(1, 12)), f_remove=f, f_insert=f)
        ins = new_nodes(rng, int(np.sum(order < 0)))
        idx, fresh = overwrites(rng, order.size, 0.01)
        cap = order.size // 4 + 16 if step % 4 != 3 else 2
        launches = res.reorder(pol, order, ins, idx, fresh, cap, f"n={n} {kind}")
        sp_launches = res.sparse(pol, idx[:0], new_nodes(rng, 0), res.n + 16, f"sparse after {kind}")
        # reorder = what the sparse delta launches (with its patch when there are overwrites) + the gather kernel
        assert launches == sp_launches + (1 if idx.size else 0) + 1, (kind, launches, sp_launches)
        if kind == "none":
            assert res.n == 0


def test_reorder_slot_cut_and_revision_hash(handle):
    """Upgrade-required candidates moved to the front and to the back under a limited slot budget, so that the slot cut
    crosses many tiles; a node whose revision hash is missing moved ahead of and behind the others (abort)."""
    rng = np.random.default_rng(41)
    n = 40 * TILE + 17
    soa, _ = helpers.random_soa(rng, n, wild=True)
    soa["state"][rng.choice(n, size=n // 5, replace=False)] = abi.UST_STATE_UPGRADE_REQUIRED
    cut = abi.make_policy(max_parallel_upgrades=n // 50, max_unavailable=None)
    res = Resident(handle, cut, soa)
    none = np.zeros(0, np.int64)
    for where in ("front", "back", "front"):
        cand = res.soa["state"] == abi.UST_STATE_UPGRADE_REQUIRED
        rest = np.nonzero(~cand)[0]
        c = np.nonzero(cand)[0]
        order = np.concatenate([c, rest] if where == "front" else [rest, c]).astype(np.int64)
        res.reorder(cut, order, new_nodes(rng, 0), none, new_nodes(rng, 0), res.n + 16, f"candidates to the {where}")
    # a revision-hash error: one node without a readable hash, moved to the head and then to the tail
    idx = np.array([n // 2], np.int64)
    bad = new_nodes(rng, 1, p_err=1.0)
    res.reorder(cut, np.arange(res.n, dtype=np.int64), new_nodes(rng, 0), idx, bad, res.n + 16, "revision-hash node in place")
    ident = np.arange(res.n, dtype=np.int64)
    for what, order in (("ahead of the others", np.insert(np.delete(ident, n // 2), 0, n // 2)),
                        ("behind the others", np.append(np.delete(ident, 0), 0))):
        res.reorder(cut, order, new_nodes(rng, 0), none, new_nodes(rng, 0), 8, f"revision-hash node moved {what}")
    res.dense(cut, "dense after the moves")


def test_reorder_interleaved_with_other_calls(handle):
    """Reorders between delta, sparse delta and splice calls; truncation followed by ust_fetch_outputs at the new size."""
    rng = np.random.default_rng(43)
    soa, _ = helpers.random_soa(rng, 9000, wild=True)
    pol = abi.make_policy(**POL)
    res = Resident(handle, pol, soa)
    for rep in range(3):
        order = reorder_model.random_order(rng, res.n, "mixed", k=30, f_remove=0.05, f_insert=0.07)
        ins = new_nodes(rng, int(np.sum(order < 0)))
        res.reorder(pol, order, ins, *overwrites(rng, order.size, 0.02), cap=4, what=f"truncated reorder {rep}")
        res.sparse(pol, *overwrites(rng, res.n, 0.01), cap=res.n, what="sparse")
        rm, ib = splice_model.random_splice(rng, res.n, 0.01, 0.01)
        res.splice(pol, rm, ib, new_nodes(rng, ib.shape[0]), f"splice {rep}")
        res.dense(pol, "dense")
        order = reorder_model.random_order(rng, res.n, "shuffle")
        res.reorder(pol, order, new_nodes(rng, 0), *overwrites(rng, res.n, 0.01), cap=res.n + 1, what=f"shuffle {rep}")


def test_reorder_noop_is_delta_sparse(handle):
    """reorder == NULL behaves like ust_apply_state_delta_sparse and launches what it launches."""
    rng = np.random.default_rng(3)
    soa, _ = helpers.random_soa(rng, 5000, wild=True)
    pol = abi.make_policy(**POL)
    res = Resident(handle, pol, soa)
    idx, fresh = overwrites(rng, res.n, 0.01)
    launches = handle.launch_count()
    for k in COLS:
        res.soa[k][idx] = fresh[k]
    rc, n_out, oi, on, oa, cnt = handle.apply_state_delta_reorder(pol, None, idx, fresh, res.soa["ds_rev"], 5000)
    ref = helpers.oracle_apply(pol, res.soa, variant=1)
    res.nxt[oi[:n_out]] = on[:n_out]
    res.act[oi[:n_out]] = oa[:n_out]
    assert rc == ref[0] and np.array_equal(res.nxt, ref[1]) and np.array_equal(res.act, ref[2]) and cnt == ref[4]
    assert handle.launch_count() - launches == 1 + 2 + 3   # patch, streaming + verification, the three diff kernels


def test_reorder_contract_errors_leave_the_snapshot(handle):
    rng = np.random.default_rng(11)
    soa, _ = helpers.random_soa(rng, 4097, wild=True)
    pol = abi.make_policy(**POL)
    res = Resident(handle, pol, soa)
    n = res.n
    none = np.zeros(0, np.int64)
    ins2 = new_nodes(rng, 2)
    bad = [
        ("run length 0", dict(run_src=[0, 5], run_len=[5, 0]), none),
        ("negative run length", dict(run_src=[0], run_len=[-3]), none),
        ("run_src below -1", dict(run_src=[-2], run_len=[1]), none),
        ("old run past the end", dict(run_src=[n - 3], run_len=[4]), none),
        ("old run starting at n", dict(run_src=[n], run_len=[1]), none),
        ("overlapping runs", dict(run_src=[0, 100], run_len=[200, 5]), none),
        ("the same node twice", dict(run_src=[7, 7], run_len=[1, 1]), none),
        ("overlap far apart in the list", dict(run_src=[0, 3000, 2999], run_len=[64, 1000, 2]), none),
        ("inserted runs take fewer", dict(run_src=[-1, 0], run_len=[1, n], **ins2), none),
        ("inserted runs take more", dict(run_src=[-1, 0, -1], run_len=[2, n, 1], **ins2), none),
        ("NULL run arrays", None, none),
        ("NULL insert arrays", dict(run_src=[-1], run_len=[2], n_insert=2), none),
        ("new size of 2^40", dict(run_src=[-1], run_len=[1 << 40], n_insert=1 << 40, **ins2), none),
        ("idx outside the new size", dict(run_src=[0], run_len=[n - 3]), np.array([n - 3], np.int64)),
    ]
    for what, ro, idx in bad:
        fresh = new_nodes(rng, idx.shape[0])
        if ro is None:
            rc = _reorder_raw(handle, pol, 3, res.soa["ds_rev"])
        else:
            rc = handle.apply_state_delta_reorder(pol, ro, idx, fresh, res.soa["ds_rev"], 64)[0]
        assert rc == INVALID, (what, rc)
        err = handle.last_error()
        assert "reorder" in err or "outside the snapshot" in err or "too many nodes" in err, (what, err)
        # the resident snapshot and outputs are what they were: an empty sparse call reports nothing
        r = handle.apply_state_delta_sparse(pol, none, new_nodes(rng, 0), res.soa["ds_rev"], 16)
        assert r[0] == 0 and r[1] == 0, (what, r[0], r[1])
        frc, nxt, act = handle.fetch_outputs(n)
        assert frc == 0 and np.array_equal(nxt, res.nxt) and np.array_equal(act, res.act), what
    # and the bitmap of the overlap check was left clean: a valid reorder over the same nodes goes through
    res.reorder(pol, np.arange(n, dtype=np.int64)[::-1].copy(), new_nodes(rng, 0), none, new_nodes(rng, 0), n + 16, "after the rejected calls")
    # a rollout simulation leaves the simulated snapshot resident but no outputs of it to compare with
    rc, _, _, _ = handle.simulate_rollout(pol, res.n, 1, want_final=False)
    assert rc not in (abi.K["UST_ERR_CUDA"], INVALID), handle.last_error()
    rc = handle.apply_state_delta_reorder(pol, dict(run_src=[0], run_len=[1]), none, new_nodes(rng, 0), soa["ds_rev"], 16)[0]
    assert rc == INVALID and "no resident outputs" in handle.last_error()
    # no resident snapshot (BuildState shares the staging arrays)
    handle.build_state(soa["state"][:10], np.zeros(10, np.int32), np.array([10], np.int32))
    rc = handle.apply_state_delta_reorder(pol, dict(run_src=[0], run_len=[1]), none, new_nodes(rng, 0), soa["ds_rev"], 16)[0]
    assert rc == INVALID and "no resident snapshot" in handle.last_error()


def _reorder_raw(handle, pol, n_runs, ds_rev):
    """A ust_reorder with NULL run arrays and n_runs > 0 (the dict form always passes arrays)."""
    import ctypes as C
    ro = abi.Reorder(n_runs, None, None, 0, None, None, None, None)
    ds_rev = np.ascontiguousarray(ds_rev, np.int32)
    oi, on, oa = np.zeros(17, np.int64), np.zeros(17, np.uint8), np.zeros(17, np.uint16)
    n_out = C.c_int64(0)
    cnt = abi.Counters()
    return handle._lib.ust_apply_state_delta_reorder(handle._h, C.addressof(pol), C.addressof(ro), 0, None, None, None, None, None,
                                                     int(ds_rev.shape[0]), ds_rev.ctypes.data, C.c_int64(16), oi.ctypes.data,
                                                     on.ctypes.data, oa.ctypes.data, C.addressof(n_out), C.addressof(cnt))


def test_reorder_c3_10m(handle):
    """A 10 M-node C3 snapshot: 0.1 % of the nodes moved with 1 % re-encoded, the two halves swapped, a full shuffle."""
    cfg = synth.CONFIGS["C3"]
    soa = synth.make_nodes(cfg["n"], cfg["seed"])
    pol = synth.config_policy("C3")
    res = Resident(handle, pol, soa)
    rng = np.random.default_rng(10)
    for what in ("moves", "swap", "shuffle"):
        n = res.n
        if what == "moves":
            moved = rng.choice(n, size=n // 1000, replace=False)
            keep = np.delete(np.arange(n, dtype=np.int64), moved)
            order = np.insert(keep, np.sort(rng.integers(0, keep.size + 1, size=moved.size)), rng.permutation(moved))
        elif what == "swap":
            order = np.concatenate([np.arange(n // 2, n), np.arange(n // 2)]).astype(np.int64)
        else:
            order = rng.permutation(n).astype(np.int64)
        idx = np.sort(rng.choice(n, size=n // 100, replace=False)).astype(np.int64)
        src = synth.make_nodes(idx.shape[0], 300)
        res.reorder(pol, order, new_nodes(rng, 0), idx, {k: src[k] for k in COLS}, n // 8, f"C3 {what}")
