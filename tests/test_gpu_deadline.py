"""ust_next_deadline on the H100: the next deadline every clocked call computes on the device, against deadline_model's flip
model with the unclocked call (ust_apply_state with pod lists, on a second handle) as the reference ApplyState - after full
calls and deltas around the tile sizes, after reorders that move, drop and insert nodes and after aborts; the defining
property walked forward on a 200 k-node snapshot; every refusal; and one C4-size call."""
import numpy as np
import pytest

import deadline_model as dm
import helpers
from helpers import abi
from test_gpu_clock import COLS, NOW, POL_KW, T, clocked_snapshot, empty_delta, random_starts
from ust import lib as ustlib, synth

pytestmark = pytest.mark.gpu

INVALID = abi.K["UST_ERR_INVALID_ARGUMENT"]


@pytest.fixture(scope="module")
def handle():
    h = ustlib.Handle(0)
    yield h
    h.close()


@pytest.fixture(scope="module")
def oracle_handle():
    h = ustlib.Handle(0)
    yield h
    h.close()


def model(oh, pol, soa, pods, start, now, timeout):
    """(next deadline or None, d + 1 per node, the nodes whose outputs change when their bit turns on)"""
    t, at, fire = dm.flip_model(pol, soa, pods, start, now, timeout, apply=lambda p, s, q: oh.apply_state(p, s, q))
    return (None if t == dm.NONE else t), at, fire


def test_full_calls_and_deltas(handle, oracle_handle):
    """Random snapshots around the tile sizes (every bit random, extreme starts, both wait timeouts, UST_EVAL_VALIDATION on
    and off, revision-hash and validation aborts), each followed by a delta that changes some nodes and their starts."""
    found, rcs = 0, set()
    sizes = [1, 127, 128, 129, 3071, 3072, 3073, 6145, 100_003, 262_145]
    for k, n in enumerate(sizes * 2):
        rng = np.random.default_rng(0xDEAD + k)
        soa, pods = helpers.random_soa(rng, n, p_err=0.002 if k % 3 == 0 else 0.0, with_pods=True)
        if k % 3 != 0:
            soa["flags"] &= np.where(rng.random(n) < 0.9995, np.uint32(~abi.UST_F_VALIDATION_START_INVALID & 0xFFFFFFFF),
                                     np.uint32(0xFFFFFFFF))
        pol = helpers.random_policy(rng)
        pol.evaluate_actuators = 3 if k % 2 == 0 else 1
        timeout = int(rng.choice([1, 30, 600, 86_400])) if pol.wait_timeout_nonzero else 0
        now = int(rng.choice([0, NOW, -1000]))
        start = random_starts(rng, n, now, 2 * timeout + 700)
        got = handle.apply_state_clocked(pol, now, timeout, start, soa, pods)
        rcs.add(got[0])
        want = model(oracle_handle, pol, soa, pods, start, now, timeout)[0]
        assert handle.next_deadline() == want, (n, k)
        found += want is not None
        # a delta: some nodes re-encoded with new starts, at a later time
        m = min(n, 50)
        idx = np.sort(rng.choice(n, m, replace=False)).astype(np.int64)
        new, _ = helpers.random_soa(rng, m)
        for c in COLS:
            soa[c][idx] = new[c]
        start[idx] = now + rng.integers(-700, 700, m)
        later = now + int(rng.integers(0, 40))
        r = handle.apply_state_delta_pods_clocked(pol, later, timeout, None, None, idx, {c: soa[c][idx] for c in COLS}, start[idx],
                                                  soa["ds_rev"], n)
        assert r[0] not in (INVALID, abi.K["UST_ERR_CUDA"]), handle.last_error()
        want = model(oracle_handle, pol, soa, pods, start, later, timeout)[0]
        assert handle.next_deadline() == want, (n, k, "delta")
        found += want is not None
    assert found >= 10, found
    assert {0, abi.K["UST_ERR_REVISION_HASH"]} <= rcs, rcs


def test_reorder_and_abort(handle, oracle_handle):
    """After a reorder that moves, drops and inserts nodes (with insert_start), then after a call that aborts in the
    validation pass: the starts and the abort point are those the model sees."""
    rng = np.random.default_rng(55)
    n, d, m = 150_000, 100, 50
    soa, pods, start = clocked_snapshot(n, 0x5EED0055, rng)
    pol = abi.make_policy(**POL_KW)
    assert handle.apply_state_clocked(pol, NOW, T, start, soa, pods)[0] == 0
    assert handle.next_deadline() == model(oracle_handle, pol, soa, pods, start, NOW, T)[0]
    ins, ins_pods, ins_start = clocked_snapshot(m, 0x5EED0155, rng)
    h = n // 2
    ro = {"run_src": np.array([h, -1, 0], np.int64), "run_len": np.array([n - d - h, m, h], np.int64), **{c: ins[c] for c in COLS}}
    new_n = n - d + m
    soa_r = {c: np.concatenate([soa[c][h:n - d], ins[c], soa[c][:h]]) for c in COLS}
    soa_r["ds_rev"] = soa["ds_rev"]
    start_r = np.concatenate([start[h:n - d], ins_start, start[:h]])
    cnt = np.diff(pods["pod_off"])
    cnt_r = np.concatenate([cnt[h:n - d], np.diff(ins_pods["pod_off"]), cnt[:h]])
    off = pods["pod_off"]
    pods_r = {"pod_off": np.concatenate([[0], np.cumsum(cnt_r)]).astype(np.int32),
              "pod_flags": np.concatenate([pods["pod_flags"][off[h]:off[n - d]], ins_pods["pod_flags"], pods["pod_flags"][:off[h]]])}
    at = n - d - h
    lists = {"node_idx": np.arange(at, at + m, dtype=np.int64), "pod_off": ins_pods["pod_off"], "pod_flags": ins_pods["pod_flags"]}
    idx0, ch0, st0 = empty_delta()
    now = NOW + 20
    r = handle.apply_state_delta_pods_clocked(pol, now, T, ro, lists, idx0, ch0, st0, soa["ds_rev"], new_n, insert_start=ins_start)
    assert r[0] == 0
    want = model(oracle_handle, pol, soa_r, pods_r, start_r, now, T)[0]
    assert want is not None and handle.next_deadline() == want
    # a validation abort in the middle of the snapshot: an unparsable start on a node whose one validation pod is not ready;
    # every validation-required node behind it is past the abort
    v = np.nonzero((soa_r["state"] & 15) == abi.UST_STATE_VALIDATION_REQUIRED)[0]
    j = int(v[v.size // 2])
    soa_r["flags"][j] |= np.uint32(abi.UST_F_VALIDATION_START_ANNO | abi.UST_F_VALIDATION_START_INVALID)
    one = np.array([abi.UST_PHASE_RUNNING | abi.UST_POD_MATCH_VALIDATION_SELECTOR], np.uint16)
    o = pods_r["pod_off"]
    pods_r = {"pod_flags": np.concatenate([pods_r["pod_flags"][:o[j]], one, pods_r["pod_flags"][o[j + 1]:]]),
              "pod_off": np.concatenate([o[:j + 1], o[j + 1:] - (o[j + 1] - o[j]) + 1]).astype(np.int32)}
    lists = {"node_idx": np.array([j], np.int64), "pod_off": np.array([0, 1], np.int32), "pod_flags": one}
    idx = np.array([j], np.int64)
    r = handle.apply_state_delta_pods_clocked(pol, now, T, None, lists, idx, {c: soa_r[c][idx] for c in COLS}, start_r[idx],
                                              soa["ds_rev"], new_n)
    assert r[0] == abi.K["UST_ERR_VALIDATION"]
    want_abort = model(oracle_handle, pol, soa_r, pods_r, start_r, now, T)[0]
    assert handle.next_deadline() == want_abort
    # the abort hides deadlines: without it the answer would be the earlier one or the same, never a later one
    assert want_abort is None or want_abort >= want


def test_walk_forward(handle, oracle_handle):
    """The defining property, 25 times on 200 k nodes: with T = ust_next_deadline, a time-only call at T - 1 returns
    nothing, one at T returns exactly the nodes the model says fire at T, and the next query returns a later time or None."""
    rng = np.random.default_rng(77)
    n = 200_000
    soa, pods, start = clocked_snapshot(n, 0x5EED0077, rng)
    pol = abi.make_policy(**POL_KW)
    assert handle.apply_state_clocked(pol, NOW, T, start, soa, pods)[0] == 0
    idx0, ch0, st0 = empty_delta()
    now, steps = NOW, 0
    while steps < 25:
        t = handle.next_deadline()
        want, at, fire = model(oracle_handle, pol, soa, pods, start, now, T)
        assert t == want, (steps, t, want)
        assert t is not None and t > now
        r = handle.apply_state_delta_pods_clocked(pol, t - 1, T, None, None, idx0, ch0, st0, soa["ds_rev"], n)
        assert r[0] == 0 and r[1] == 0, (steps, r[1])
        assert handle.next_deadline() == t
        r = handle.apply_state_delta_pods_clocked(pol, t, T, None, None, idx0, ch0, st0, soa["ds_rev"], n)
        expect = np.nonzero(fire & (at == t))[0]
        assert r[0] == 0 and r[1] == expect.size > 0 and np.array_equal(r[2][:r[1]], expect), (steps, r[1], expect.size)
        now, steps = t, steps + 1
    t = handle.next_deadline()
    assert t is None or t > now


def test_refusals(handle, oracle_handle):
    rng = np.random.default_rng(9)
    n = 20_000
    soa, pods, start = clocked_snapshot(n, 0x5EED0009, rng)
    pol = abi.make_policy(**POL_KW)
    fresh = ustlib.Handle(0)
    try:
        assert fresh.next_deadline(check=False)[0] == INVALID        # nothing resident
        assert "clocked" in fresh.last_error()
    finally:
        fresh.close()
    assert handle.apply_state(pol, soa, pods)[0] == 0                # an unclocked snapshot
    assert handle.next_deadline(check=False)[0] == INVALID
    assert handle.apply_state_clocked(pol, NOW, T, start, soa, pods)[0] == 0
    want = handle.next_deadline()
    assert want == model(oracle_handle, pol, soa, pods, start, NOW, T)[0] and want is not None
    assert ustlib.load().ust_next_deadline(handle._h, None) == INVALID   # a NULL pointer
    assert handle.next_deadline() == want                            # asking again changes nothing
    assert handle.fetch_outputs_pods(n)[0] == 0 and handle.next_deadline() == want
    # a refused clocked call: the snapshot stays resident, its deadline is no longer the last call's
    idx0, ch0, st0 = empty_delta()
    assert handle.apply_state_delta_pods_clocked(pol, NOW, 0, None, None, idx0, ch0, st0, soa["ds_rev"], n)[0] == INVALID
    rc, v = handle.next_deadline(check=False)
    assert rc == INVALID and "last call" in handle.last_error()
    # the next good call answers again; a full clocked call without a clock is refused like the others
    assert handle.apply_state_delta_pods_clocked(pol, NOW + 1, T, None, None, idx0, ch0, st0, soa["ds_rev"], n)[0] == 0
    assert handle.next_deadline() == model(oracle_handle, pol, soa, pods, start, NOW + 1, T)[0]
    assert handle.apply_state_clocked(pol, None, T, start, soa, pods)[0] == INVALID
    assert handle.next_deadline(check=False)[0] == INVALID
    assert handle.apply_state_delta_pods_clocked(pol, NOW + 1, T, None, None, idx0, ch0, st0, soa["ds_rev"], n)[0] == 0
    assert handle.next_deadline() is not None
    # any other call in between: a node-only ApplyState drops the pod-list snapshot
    assert handle.apply_state(abi.make_policy(), soa)[0] == 0
    assert handle.next_deadline(check=False)[0] == INVALID


def test_c4_full_size(handle, oracle_handle):
    """One C4-size clocked call (10 M nodes, ~3 x 10^8 workload pods) with a wait timeout: the deadline equals the model's."""
    cfg = synth.CONFIGS["C4"]
    n = cfg["n"]
    soa = synth.make_nodes(n, cfg["seed"])
    pods = synth.make_pods_blocked(n, cfg["seed"])
    pol = abi.make_policy(auto_upgrade=True, **dict(cfg["policy"], wait_for_completion={"podSelector": "app=batch", "timeoutSeconds": 300}))
    rng = np.random.default_rng(4)
    w = (soa["state"] & 15) == abi.UST_STATE_WAIT_FOR_JOBS_REQUIRED
    soa["flags"] = (soa["flags"] | np.where(w & (rng.random(n) < 0.8), np.uint32(abi.UST_F_WAIT_START_ANNO), np.uint32(0))).astype(np.uint32)
    start = (NOW - rng.integers(0, 700, n)).astype(np.int64)
    assert handle.apply_state_clocked(pol, NOW, 300, start, soa, pods)[0] == 0
    want, at, fire = model(oracle_handle, pol, soa, pods, start, NOW, 300)
    assert want is not None and np.count_nonzero(fire) > 10_000
    assert handle.next_deadline() == want
