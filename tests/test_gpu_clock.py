"""Clocked pod-list calls on the H100 (ust_apply_state_clocked, ust_apply_state_delta_pods_clocked): the wait-for-completion
and validation timeouts derived on the device from `now` and the resident start times. The oracle is the unclocked call
(ust_apply_state with pod lists, on a second handle) on the same arrays with bits 18 and 27 set on the host from the same
`now` (clock_model): full calls on random snapshots around the tile boundaries, reconciles in which only time passes
(sparse outputs = the diff of two full calls), the reference's wait-timeout timeline replayed through deltas that carry
only the nodes whose objects changed, reorders that move, drop and add nodes with their start times, every refusal, and
one C4-size call."""
import numpy as np
import pytest

import clock_model as cm
import helpers
from helpers import abi
from ust import lib as ustlib, synth

pytestmark = pytest.mark.gpu

INVALID = abi.K["UST_ERR_INVALID_ARGUMENT"]
I64 = np.iinfo(np.int64)
NOW = 1_700_000_000
T = 30
POL_KW = dict(max_parallel_upgrades=0, pod_deletion_enabled=True, pod_deletion={"force": False, "deleteEmptyDir": False},
              drain={"enable": True, "force": False, "deleteEmptyDir": False}, validation_enabled=True,
              wait_for_completion={"podSelector": "app=batch", "timeoutSeconds": T}, evaluate_actuators=True,
              evaluate_validation=True)
COLS = ("state", "flags", "pod_rev", "ds_idx")


@pytest.fixture(scope="module")
def handle():
    h = ustlib.Handle(0)
    yield h
    h.close()


@pytest.fixture(scope="module")
def oracle_handle():
    """A handle of its own for the unclocked reference calls, which leave an unclocked snapshot behind."""
    h = ustlib.Handle(0)
    yield h
    h.close()


def reference(oh, pol, soa, pods, start, now, timeout):
    r = oh.apply_state(pol, cm.derived_soa(soa, start, now, timeout), pods)
    return r


def random_starts(rng, n, now, spread):
    s = now + rng.integers(-spread, spread + 1, n)
    u = rng.random(n)
    s = np.where(u < 0.02, I64.max, s)
    s = np.where((u >= 0.02) & (u < 0.04), I64.min, s)
    s = np.where((u >= 0.04) & (u < 0.05), I64.max - rng.integers(0, 1000, n), s)
    return s.astype(np.int64)


def clocked_snapshot(n, seed, rng, now=NOW):
    """A synthetic snapshot with validation pods, wait-start annotations on most wait-for-jobs-required nodes, start times on
    both sides of the deadlines, and random bits 18 / 27 (which a clocked call ignores)."""
    soa = synth.make_nodes(n, seed, requestor_pct=5.0)
    flags, pods = synth.make_validation_pods(soa, synth.make_pods(n, seed), seed)
    code = soa["state"] & 15
    w = code == abi.UST_STATE_WAIT_FOR_JOBS_REQUIRED
    flags |= np.where(w & (rng.random(n) < 0.8), np.uint32(abi.UST_F_WAIT_START_ANNO), np.uint32(0))
    flags |= np.where(w & (rng.random(n) < 0.02), np.uint32(abi.UST_F_WAIT_START_INVALID), np.uint32(0))
    flags ^= np.where(rng.random(n) < 0.5, np.uint32(cm.TIMED_OUT), np.uint32(0))
    soa["flags"] = flags.astype(np.uint32)
    start = np.where(w, now - rng.integers(-20, 120, n), now - rng.integers(-100, 1300, n)).astype(np.int64)
    return soa, pods, start


def empty_delta():
    return np.zeros(0, np.int64), {k: np.zeros(0, dt) for k, dt in zip(COLS, (np.uint8, np.uint32, np.int32, np.int32))}, \
        np.zeros(0, np.int64)


def check_sparse(got, prev, ref, what, always=()):
    """A sparse result against the full reference: counters and code, the reported set = the nodes whose outputs differ
    from `prev` (plus `always`), and the values reported."""
    rc, n_out, oi, on, oa, oo, cnt = got
    assert rc == ref[0] and cnt == ref[4], (what, rc, ref[0])
    diff = np.nonzero((prev[0] != ref[1]) | (prev[1] != ref[2]) | (prev[2] != ref[3]))[0]
    diff = np.union1d(diff, np.asarray(always, np.int64))
    assert n_out == diff.size, (what, n_out, diff.size)
    assert np.array_equal(oi[:n_out], diff), what
    assert np.array_equal(on[:n_out], ref[1][diff]) and np.array_equal(oa[:n_out], ref[2][diff]) \
        and np.array_equal(oo[:n_out], ref[3][diff]), what
    return n_out


def test_full_calls_random(handle, oracle_handle):
    """Every flag bit random (bits 18 and 27 and the reserved bits too), random starts with the extremes, the wait timeout
    zero and non-zero, UST_EVAL_VALIDATION on and off, revision-hash and validation aborts, sizes around the tiles."""
    rcs = set()
    sizes = [1, 127, 128, 129, 3071, 3072, 3073, 6145, 100_003, 262_145]
    for k, n in enumerate(sizes * 2):
        rng = np.random.default_rng(0xC10C + k)
        soa, pods = helpers.random_soa(rng, n, p_err=0.002 if k % 3 == 0 else 0.0, with_pods=True)
        if k % 3 != 0:  # mostly parsable validation starts, so that not every validation-mode call aborts early
            soa["flags"] &= np.where(rng.random(n) < 0.9995, np.uint32(~abi.UST_F_VALIDATION_START_INVALID & 0xFFFFFFFF),
                                     np.uint32(0xFFFFFFFF))
        pol = helpers.random_policy(rng)
        pol.evaluate_actuators = 3 if k % 2 == 0 else 1
        timeout = int(rng.choice([1, 30, 600, 86_400])) if pol.wait_timeout_nonzero else 0
        now = int(rng.choice([0, NOW, -1000]))
        start = random_starts(rng, n, now, 2 * timeout + 700)
        got = handle.apply_state_clocked(pol, now, timeout, start, soa, pods)
        ref = reference(oracle_handle, pol, soa, pods, start, now, timeout)
        helpers.assert_same(got, ref, f"clocked n={n} k={k}")
        rcs.add(got[0])
    # a validation abort for certain: every validation-required node carries an unparsable start
    rng = np.random.default_rng(0xC10D)
    n = 50_000
    soa, pods = helpers.random_soa(rng, n, with_pods=True)
    v = (soa["state"] & 15) == abi.UST_STATE_VALIDATION_REQUIRED
    soa["flags"] = np.where(v, soa["flags"] | np.uint32(abi.UST_F_VALIDATION_START_ANNO | abi.UST_F_VALIDATION_START_INVALID),
                            soa["flags"]).astype(np.uint32)
    pol = abi.make_policy(**POL_KW)   # no policy-level abort comes first
    start = random_starts(rng, n, NOW, 700)
    got = handle.apply_state_clocked(pol, NOW, T, start, soa, pods)
    helpers.assert_same(got, reference(oracle_handle, pol, soa, pods, start, NOW, T), "validation abort")
    rcs.add(got[0])
    assert {0, abi.K["UST_ERR_REVISION_HASH"], abi.K["UST_ERR_VALIDATION"]} <= rcs, rcs


def test_time_only_reconciles(handle, oracle_handle):
    """A resident clocked snapshot and a run of deltas that carry nothing but the time: forwards past deadlines, once
    backwards (which clears bits again), then far ahead. Each call reports exactly what changed between two full calls."""
    rng = np.random.default_rng(21)
    n = 200_000
    soa, pods, start = clocked_snapshot(n, 0x5EED0021, rng)
    pol = abi.make_policy(**POL_KW)
    got = handle.apply_state_clocked(pol, NOW, T, start, soa, pods)
    ref = reference(oracle_handle, pol, soa, pods, start, NOW, T)
    helpers.assert_same(got, ref, "first call")
    prev = (ref[1], ref[2], ref[3])
    idx, ch, st = empty_delta()
    fired = []
    for now in (NOW + 5, NOW + 31, NOW + 90, NOW + 40, NOW + 700, NOW + 5000):
        got = handle.apply_state_delta_pods_clocked(pol, now, T, None, None, idx, ch, st, soa["ds_rev"], n)
        ref = reference(oracle_handle, pol, soa, pods, start, now, T)
        fired.append(check_sparse(got, prev, ref, f"now={now}"))
        prev = (ref[1], ref[2], ref[3])
    assert all(f > 0 for f in fired[:-1]), fired   # by NOW + 5000 every deadline has passed already
    frc, fn, fa, fo = handle.fetch_outputs_pods(n)
    assert frc == 0 and np.array_equal(fn, prev[0]) and np.array_equal(fa, prev[1]) and np.array_equal(fo, prev[2])


@pytest.mark.parametrize("timeout,dt,steps", [(100, 30, 8), (45, 45, 5), (10, 60, 3)])
def test_wait_timeout_timeline(handle, timeout, dt, steps):
    """helpers.wait_timeout_timeline (the reference's HandleTimeoutOnPodCompletions, pod_manager.go:331-368, reconcile by
    reconcile) replayed through clocked deltas: each reconcile sends only the nodes whose objects changed - a state label or
    a start annotation set or cleared by the previous one - and the device decides when the deadline passes. Final states
    and start annotations must be the golden ones."""
    G = helpers.load_golden()
    pol, _, state_exp, start_exp = helpers.wait_timeout_timeline(G["daemonset_hash"], timeout, dt, steps)
    n = 3
    base = {"ds": True, "pod": {"hash": G["daemonset_hash"], "phase": "Running", "containers": [[True, 0]]}}
    pdict = {"waitForCompletion": {"timeoutSeconds": timeout}}
    job = abi.UST_PHASE_RUNNING | abi.UST_POD_HAS_CONTROLLER | abi.UST_POD_MATCH_WAIT_SELECTOR   # the jobs keep running
    pods = {"pod_off": np.arange(n + 1, dtype=np.int32), "pod_flags": np.full(n, job, np.uint16)}
    state = ["wait-for-jobs-required"] * n
    start = [None] * n
    last, sent = None, []
    for k in range(steps):
        now = k * dt
        vec = [dict(base, state=state[i], **({"anno": {"wait-start": "now-0"}} if start[i] is not None else {})) for i in range(n)]
        cur, _ = helpers.encode_nodes(vec, G["daemonset_hash"], pdict)   # what the encoder sends: no clock involved
        cur["flags"] = np.where((cur["state"] & 15) == 3, cur["flags"] | np.uint32(abi.UST_F_WAIT_PODS_RUNNING),
                                cur["flags"]).astype(np.uint32) & np.uint32(~cm.TIMED_OUT & 0xFFFFFFFF)
        st = np.array([s if s is not None else 0 for s in start], np.int64)
        if last is None:
            rc, nxt, act, oc, _ = handle.apply_state_clocked(pol, now, timeout, st, cur, pods)
        else:
            idx = np.nonzero((cur["state"] != last[0]) | (cur["flags"] != last[1]) | (st != last[2]))[0].astype(np.int64)
            sent.append(idx.size)
            rc = handle.apply_state_delta_pods_clocked(pol, now, timeout, None, None, idx, {c: cur[c][idx] for c in COLS}, st[idx],
                                                       cur["ds_rev"], n)[0]
            frc, nxt, act, oc = handle.fetch_outputs_pods(n)
            assert frc == 0
        assert rc == 0, (k, rc, handle.last_error())
        last = (cur["state"].copy(), cur["flags"].copy(), st.copy())
        for i in range(n):
            if act[i] & abi.UST_A_SET_WAIT_START:
                start[i] = now
            if act[i] & abi.UST_A_CLEAR_WAIT_START:
                start[i] = None
            new = oc[i] if ((act[i] & abi.UST_A_SCHEDULE_WAIT_CHECK) and oc[i] != 0xFF) else nxt[i]
            state[i] = abi.STATE_NAMES[new]
    assert state == state_exp, (state, state_exp)
    assert start == start_exp, (start, start_exp)
    if timeout >= 2 * dt:
        assert 0 in sent, sent   # reconciles in which only time passed carried no node at all


def test_reorder_moves_starts(handle, oracle_handle):
    """Nodes move (the halves swap), leave and join; changed nodes bring new starts. The starts follow their nodes: the
    result is that of a full unclocked call on the reordered arrays, and so is a later time-only call."""
    rng = np.random.default_rng(5)
    n, d, m = 150_000, 100, 50
    soa, pods, start = clocked_snapshot(n, 0x5EED0005, rng)
    pol = abi.make_policy(**POL_KW)
    r0 = handle.apply_state_clocked(pol, NOW, T, start, soa, pods)
    helpers.assert_same(r0, reference(oracle_handle, pol, soa, pods, start, NOW, T), "first call")
    ins, ins_pods, ins_start = clocked_snapshot(m, 0x5EED0105, rng)
    h = n // 2
    ro = {"run_src": np.array([h, -1, 0], np.int64), "run_len": np.array([n - d - h, m, h], np.int64),
          **{c: ins[c] for c in COLS}}
    new_n = n - d + m
    perm = np.concatenate([np.arange(h, n - d), np.arange(0, h)])   # old nodes in new order, inserted ones between
    at = n - d - h
    pos_ins = np.arange(at, at + m)
    soa_r = {c: np.concatenate([soa[c][h:n - d], ins[c], soa[c][:h]]) for c in COLS}
    soa_r["ds_rev"] = soa["ds_rev"]
    start_r = np.concatenate([start[h:n - d], ins_start, start[:h]])
    cnt = np.diff(pods["pod_off"])
    cnt_r = np.concatenate([cnt[h:n - d], np.diff(ins_pods["pod_off"]), cnt[:h]])
    off = pods["pod_off"]
    pods_r = {"pod_off": np.concatenate([[0], np.cumsum(cnt_r)]).astype(np.int32),
              "pod_flags": np.concatenate([pods["pod_flags"][off[h]:off[n - d]], ins_pods["pod_flags"], pods["pod_flags"][:off[h]]])}
    lists = {"node_idx": pos_ins.astype(np.int64), "pod_off": ins_pods["pod_off"], "pod_flags": ins_pods["pod_flags"]}
    stay = np.setdiff1d(np.arange(new_n), pos_ins)
    idx = np.sort(rng.choice(stay, 300, replace=False)).astype(np.int64)
    new_st = start_r[idx] + rng.integers(-900, 900, idx.size)
    start_r[idx] = new_st
    now = NOW + 45
    got = handle.apply_state_delta_pods_clocked(pol, now, T, ro, lists, idx, {c: soa_r[c][idx] for c in COLS}, new_st,
                                                soa["ds_rev"], new_n, insert_start=ins_start)
    ref = reference(oracle_handle, pol, soa_r, pods_r, start_r, now, T)
    prev = [np.full(new_n, 0xFF, np.uint8), np.zeros(new_n, np.uint16), np.full(new_n, 0xFF, np.uint8)]
    keep = np.setdiff1d(np.arange(new_n), pos_ins)
    for j, a in enumerate((r0[1], r0[2], r0[3])):
        prev[j][keep] = a[perm]
    check_sparse(got, prev, ref, "reorder", always=pos_ins)
    # a node whose start did not follow it would change its answer: the snapshot holds many nodes on both sides
    clocked = np.isin(soa_r["state"] & 15, [3, 9])
    derived = cm.derive(soa_r["state"], soa_r["flags"], start_r, now, T)[clocked]
    assert 100 < np.count_nonzero(derived & np.uint32(cm.TIMED_OUT)) < np.count_nonzero(clocked)
    # and they stay with the nodes for the calls after
    idx0, ch0, st0 = empty_delta()
    prev = (ref[1], ref[2], ref[3])
    for later in (now + 700, now - 300):
        got = handle.apply_state_delta_pods_clocked(pol, later, T, None, None, idx0, ch0, st0, soa["ds_rev"], new_n)
        ref = reference(oracle_handle, pol, soa_r, pods_r, start_r, later, T)
        check_sparse(got, prev, ref, f"after the reorder, now={later}")
        prev = (ref[1], ref[2], ref[3])


def test_refusals_before_device_work(handle, oracle_handle):
    """Every refusal returns UST_ERR_INVALID_ARGUMENT without a launch, and leaves the snapshot as it was: the valid call
    that follows gives the right answer."""
    rng = np.random.default_rng(8)
    n = 20_000
    soa, pods, start = clocked_snapshot(n, 0x5EED0008, rng)
    pol = abi.make_policy(**POL_KW)
    idx0, ch0, st0 = empty_delta()
    ds_rev = soa["ds_rev"]
    # an unclocked snapshot: no clocked delta on it
    assert handle.apply_state(pol, soa, pods)[0] == 0
    before = handle.launch_count()
    assert handle.apply_state_delta_pods_clocked(pol, NOW, T, None, None, idx0, ch0, st0, ds_rev, n)[0] == INVALID
    # full clocked calls: no clock, a timeout the policy contradicts, no start, no pod lists, no actuator_outcome
    assert handle.apply_state_clocked(pol, None, T, start, soa, pods)[0] == INVALID
    assert handle.apply_state_clocked(pol, NOW, 0, start, soa, pods)[0] == INVALID
    assert handle.apply_state_clocked(pol, NOW, T, start, soa, pods, clock_start=False)[0] == INVALID
    assert handle.apply_state_clocked(pol, NOW, T, start, soa, None)[0] == INVALID
    out = (np.zeros(n, np.uint8), np.zeros(n, np.uint16), None)
    assert handle.apply_state_clocked(pol, NOW, T, start, soa, pods, out=out)[0] == INVALID
    bad_pods = {"pod_off": pods["pod_off"].copy(), "pod_flags": pods["pod_flags"]}
    bad_pods["pod_off"][5] = bad_pods["pod_off"][6] + 1   # what the unclocked call rejects too
    assert handle.apply_state_clocked(pol, NOW, T, start, soa, bad_pods)[0] == INVALID
    assert handle.launch_count() == before
    # the unclocked snapshot is still resident
    r = handle.apply_state_delta_pods(pol, None, idx0, ch0, ds_rev, n)
    assert r[0] == 0 and r[1] == 0
    # a clocked snapshot: no unclocked delta on it, and every malformed clocked delta refused
    r0 = handle.apply_state_clocked(pol, NOW, T, start, soa, pods)
    helpers.assert_same(r0, reference(oracle_handle, pol, soa, pods, start, NOW, T), "clocked")
    before = handle.launch_count()
    assert handle.apply_state_delta_pods(pol, None, idx0, ch0, ds_rev, n)[0] == INVALID
    assert handle.apply_state_delta_pods_reorder(pol, None, None, idx0, ch0, ds_rev, n)[0] == INVALID
    idx = np.array([3, 17], np.int64)
    ch = {c: soa[c][idx] for c in COLS}
    assert handle.apply_state_delta_pods_clocked(pol, NOW, T, None, None, idx0, ch0, st0, ds_rev, n, clock=False)[0] == INVALID
    assert handle.apply_state_delta_pods_clocked(pol, NOW, 0, None, None, idx0, ch0, st0, ds_rev, n)[0] == INVALID
    assert handle.apply_state_delta_pods_clocked(pol, NOW, T, None, None, idx, ch, None, ds_rev, n)[0] == INVALID
    one = {c: soa[c][:1] for c in COLS}
    ro = {"run_src": np.array([0, -1], np.int64), "run_len": np.array([n, 1], np.int64), **one}
    lists = {"node_idx": np.array([n], np.int64), "pod_off": np.array([0, 0], np.int32), "pod_flags": np.zeros(0, np.uint16)}
    assert handle.apply_state_delta_pods_clocked(pol, NOW, T, ro, lists, idx0, ch0, st0, ds_rev, n + 1)[0] == INVALID
    assert handle.apply_state_delta_pods_clocked(pol, NOW, T, None, None, np.array([n], np.int64), one, start[:1], ds_rev, n)[0] == INVALID
    assert handle.launch_count() == before
    # the clocked snapshot is as it was: a time-only call reports what the clock changed
    got = handle.apply_state_delta_pods_clocked(pol, NOW + 700, T, None, None, idx0, ch0, st0, ds_rev, n)
    check_sparse(got, (r0[1], r0[2], r0[3]), reference(oracle_handle, pol, soa, pods, start, NOW + 700, T), "after refusals")


def test_c4_full_size(handle, oracle_handle):
    """One C4-size clocked call (10 M nodes, ~3 x 10^8 workload pods) with a wait timeout: parity with the unclocked call."""
    cfg = synth.CONFIGS["C4"]
    n = cfg["n"]
    soa = synth.make_nodes(n, cfg["seed"])
    pods = synth.make_pods_blocked(n, cfg["seed"])
    pol = abi.make_policy(auto_upgrade=True, **dict(cfg["policy"], wait_for_completion={"podSelector": "app=batch", "timeoutSeconds": 300}))
    rng = np.random.default_rng(4)
    w = (soa["state"] & 15) == abi.UST_STATE_WAIT_FOR_JOBS_REQUIRED
    soa["flags"] = (soa["flags"] | np.where(w & (rng.random(n) < 0.8), np.uint32(abi.UST_F_WAIT_START_ANNO), np.uint32(0))).astype(np.uint32)
    start = (NOW - rng.integers(0, 700, n)).astype(np.int64)
    got = handle.apply_state_clocked(pol, NOW, 300, start, soa, pods)
    ref = reference(oracle_handle, pol, soa, pods, start, NOW, 300)
    assert got[0] == 0
    helpers.assert_same(got, ref, "C4 clocked")
    assert np.count_nonzero(cm.derive(soa["state"], soa["flags"], start, NOW, 300) & np.uint32(abi.UST_F_WAIT_TIMED_OUT)) > 10_000
