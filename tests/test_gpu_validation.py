"""UST_EVAL_VALIDATION on the H100: Validate answered by the pod-summary kernel from the validation pods in list order, for
snapshots of several tiles that mix every outcome (no pod, done, ready-before-not-ready, set, wait, timed out, the abort),
bit for bit against validation_model on ust_apply_state, ust_apply_state_device, ust_apply_state_delta_pods and
ust_apply_state_delta_pods_reorder (sparse outputs = the diff of the full ones). The abort sits mid-array and right before
and after the upgrade-slot cut. With the mode off, pods carrying the validation bits give what the oracle gives."""
import os

import numpy as np
import pytest

import helpers
import pods_delta_model
import validation_model as vm
from helpers import abi
from ust import lib as ustlib, synth

pytestmark = pytest.mark.gpu

INVALID = abi.K["UST_ERR_INVALID_ARGUMENT"]
VALIDATION = abi.K["UST_ERR_VALIDATION"]
N = 300_000
SEED = 0x5EED0009
POL_KW = dict(max_parallel_upgrades=0, pod_deletion_enabled=True, pod_deletion={"force": False, "deleteEmptyDir": False},
              drain={"enable": True, "force": False, "deleteEmptyDir": False}, validation_enabled=True,
              wait_for_completion={"podSelector": "app=batch", "timeoutSeconds": 30}, evaluate_actuators=True,
              evaluate_validation=True)


@pytest.fixture(scope="module")
def handle():
    h = ustlib.Handle(0)
    yield h
    h.close()


def snapshot(n=N, seed=SEED, requestor_pct=5.0):
    soa = synth.make_nodes(n, seed, requestor_pct=requestor_pct)
    flags, pods = synth.make_validation_pods(soa, synth.make_pods(n, seed), seed)
    soa["flags"] = flags
    return soa, pods


def abortable(soa, pods):
    """Validation-required nodes that abort once their annotation is made unparsable: the first validation pod is not ready."""
    off, pf = pods["pod_off"], pods["pod_flags"]
    out = []
    for i in np.nonzero((soa["state"] & 15) == 9)[0].tolist():
        m = [int(p) for p in pf[off[i]:off[i + 1]] if p & abi.UST_POD_MATCH_VALIDATION_SELECTOR]
        if m and not m[0] & abi.UST_POD_READY:
            out.append(i)
    return np.array(out, np.int64)


def with_invalid(soa, nodes):
    s = dict(soa)
    s["flags"] = soa["flags"].copy()
    s["flags"][nodes] |= np.uint32(abi.UST_F_VALIDATION_START_ANNO | abi.UST_F_VALIDATION_START_INVALID)
    return s


def outcome_mix(soa, pods, pol, res):
    """Every Validate outcome is present among the validation-required nodes of a result."""
    v = (soa["state"] & 15) == 9
    act = res[2][v]
    nxt = res[1][v]
    clear, set_ = (act & abi.UST_A_CLEAR_WAIT_START) != 0, (act & abi.UST_A_SET_WAIT_START) != 0
    seen = {
        "done": np.any(clear & np.isin(nxt, [10, 11])),
        "restart": np.any(clear & set_),
        "set": np.any(set_ & ~clear),
        "timed_out": np.any(nxt == 12),
        "wait": np.any((nxt == 9) & ~clear & ~set_),
    }
    assert all(seen.values()), seen


def slot_policy(soa, pods):
    """A budget that cuts through the upgrade-required nodes: returns (policy, index of the last granted node)."""
    pol = abi.make_policy(**POL_KW)
    _, _, _, _, cnt = vm.apply(pol, soa, pods, variant=1)
    kw = dict(POL_KW, max_parallel_upgrades=cnt["in_progress"] + cnt["candidates"] // 2)
    pol = abi.make_policy(**kw)
    res = vm.apply(pol, soa, pods, variant=1)
    # candidates (upgrade-required, schedulable - an unschedulable one moves on without a slot - and not skipped)
    granted = np.nonzero(((soa["state"] & (15 | abi.UST_HOT_SKIP | abi.UST_HOT_UNSCHEDULABLE)) == 1) & (res[1] == 2))[0]
    assert 0 < granted.size < cnt["candidates"]
    return pol, int(granted[-1])


def test_apply_state_every_outcome(handle):
    soa, pods = snapshot()
    pol = abi.make_policy(**POL_KW)
    ref = vm.apply(pol, soa, pods, variant=1)
    assert ref[0] == 0
    outcome_mix(soa, pods, pol, ref)
    helpers.assert_same(handle.apply_state(pol, soa, pods), ref, "validation mode")
    # an empty selector: done without any pod, no annotation call
    pol0 = abi.make_policy(**dict(POL_KW, validation_enabled=False))
    helpers.assert_same(handle.apply_state(pol0, soa, pods), vm.apply(pol0, soa, pods, variant=1), "empty selector")
    # requestor mode
    polr = abi.make_policy(**dict(POL_KW, use_maintenance_operator=True))
    helpers.assert_same(handle.apply_state(polr, soa, pods), vm.apply(polr, soa, pods, variant=1), "requestor mode")


@pytest.mark.parametrize("where", ["mid", "before_cut", "after_cut", "two"])
def test_abort_placements(handle, where):
    soa, pods = snapshot()
    pol, cut = slot_policy(soa, pods)
    cand = abortable(soa, pods)
    if where == "mid":
        nodes = cand[np.searchsorted(cand, N // 2)][None]
    elif where == "before_cut":
        nodes = cand[np.searchsorted(cand, cut) - 1][None]
    elif where == "after_cut":
        nodes = cand[np.searchsorted(cand, cut)][None]
    else:  # the first in pass order wins
        nodes = cand[[len(cand) // 3, 2 * len(cand) // 3]]
    bad = with_invalid(soa, nodes)
    ref = vm.apply(pol, bad, pods, variant=1)
    assert ref[0] == VALIDATION and ref[4]["error_index"] == nodes[0] and ref[4]["error_pass"] == 10
    helpers.assert_same(handle.apply_state(pol, bad, pods), ref, f"abort {where}")


def test_device_entry_point(handle):
    import torch
    soa, pods = snapshot(n=100_003)
    pol, _ = slot_policy(soa, pods)
    bad = with_invalid(soa, abortable(soa, pods)[[7]])
    for s in (soa, bad):
        ref = vm.apply(pol, s, pods, variant=1)
        d = {k: torch.from_numpy(s[k].view(np.int32) if s[k].dtype == np.uint32 else s[k]).cuda() for k in ("state", "flags", "pod_rev", "ds_idx", "ds_rev")}
        off = torch.from_numpy(pods["pod_off"]).cuda()
        pf = torch.from_numpy(pods["pod_flags"].view(np.int16)).cuda()
        n = s["state"].shape[0]
        nxt = torch.zeros(n, dtype=torch.uint8, device="cuda")
        act = torch.zeros(n, dtype=torch.int16, device="cuda")
        oc = torch.zeros(n, dtype=torch.uint8, device="cuda")
        cnt = torch.zeros(32, dtype=torch.int64, device="cuda")
        handle.apply_state_device(pol, n, d["state"].data_ptr(), d["flags"].data_ptr(), d["pod_rev"].data_ptr(),
                                  d["ds_idx"].data_ptr(), int(s["ds_rev"].shape[0]), d["ds_rev"].data_ptr(), nxt.data_ptr(),
                                  act.data_ptr(), oc.data_ptr(), (off.data_ptr(), pf.data_ptr(), int(pf.numel())), cnt.data_ptr())
        handle.sync()
        c = abi.Counters.from_buffer_copy(cnt.cpu().numpy().tobytes()).as_dict()
        got = (c["error_code"], nxt.cpu().numpy(), act.cpu().numpy().view(np.uint16), oc.cpu().numpy(), c)
        helpers.assert_same(got, ref, "device")


def _full_from_sparse(prev, n_out, idx, nxt, act, oc):
    p_n, p_a, p_o = (a.copy() for a in prev)
    p_n[idx[:n_out]], p_a[idx[:n_out]], p_o[idx[:n_out]] = nxt[:n_out], act[:n_out], oc[:n_out]
    return p_n, p_a, p_o


def test_delta_pods_and_reorder(handle):
    rng = np.random.default_rng(11)
    soa, pods = snapshot(n=200_000)
    pol, _ = slot_policy(soa, pods)
    r0 = handle.apply_state(pol, soa, pods)
    helpers.assert_same(r0, vm.apply(pol, soa, pods, variant=1), "first call")
    prev = (r0[1], r0[2], r0[3])
    v = np.nonzero((soa["state"] & 15) == 9)[0]
    for step in range(4):
        # flip readiness of the validation pods of some validation-required nodes, move annotations, abort on step 2
        ni = np.sort(rng.choice(v, size=300, replace=False))
        new_off = [0]
        new_pf = []
        off, pf = pods["pod_off"], pods["pod_flags"]
        for i in ni:
            lst = pf[off[i]:off[i + 1]].copy()
            flip = (lst & abi.UST_POD_MATCH_VALIDATION_SELECTOR) != 0
            lst[flip] ^= np.uint16(abi.UST_POD_READY) * (rng.random(int(flip.sum())) < 0.5).astype(np.uint16)
            if rng.random() < 0.2:
                lst = np.concatenate([lst, [abi.UST_POD_MATCH_VALIDATION_SELECTOR | abi.UST_PHASE_PENDING]]).astype(np.uint16)
            new_pf.append(lst)
            new_off.append(new_off[-1] + lst.size)
        lists = {"node_idx": ni, "pod_off": np.array(new_off, np.int32), "pod_flags": np.concatenate(new_pf).astype(np.uint16)}
        p_off, p_pf = pods_delta_model.replace(off, pf, ni, lists["pod_off"], lists["pod_flags"])
        pods = {"pod_off": p_off, "pod_flags": p_pf}
        idx = np.sort(rng.choice(v, size=200, replace=False)).astype(np.int64)
        ch = {k: soa[k][idx].copy() for k in ("state", "flags", "pod_rev", "ds_idx")}
        ch["flags"] ^= (rng.integers(0, 2, idx.size) * abi.UST_F_VALIDATION_START_ANNO).astype(np.uint32)
        if step == 2:
            ch["flags"][:] |= np.uint32(abi.UST_F_VALIDATION_START_ANNO | abi.UST_F_VALIDATION_START_INVALID)
        soa = dict(soa)
        for k in ch:
            soa[k] = soa[k].copy()
            soa[k][idx] = ch[k]
        ref = vm.apply(pol, soa, pods, variant=1)
        if step == 3:  # a new node order: reversed halves
            n = soa["state"].shape[0]
            h = n // 2
            ro = {"run_src": np.array([h, 0], np.int64), "run_len": np.array([n - h, h], np.int64)}
            perm = np.concatenate([np.arange(h, n), np.arange(0, h)])
            soa_r = {k: (soa[k][perm] if k != "ds_rev" else soa[k]) for k in soa}
            cnts = np.diff(pods["pod_off"])[perm]
            pods_r = {"pod_off": np.concatenate([[0], np.cumsum(cnts)]).astype(np.int32),
                      "pod_flags": np.concatenate([pods["pod_flags"][pods["pod_off"][h]:], pods["pod_flags"][:pods["pod_off"][h]]])}
            inv = np.argsort(perm)
            lists = {"node_idx": inv[ni].astype(np.int64), "pod_off": lists["pod_off"], "pod_flags": lists["pod_flags"]}
            order = np.argsort(lists["node_idx"])
            lists = {"node_idx": lists["node_idx"][order],
                     "pod_off": np.concatenate([[0], np.cumsum(np.diff(lists["pod_off"])[order])]).astype(np.int32),
                     "pod_flags": np.concatenate([new_pf[j] for j in order]).astype(np.uint16)}
            ref = vm.apply(pol, soa_r, pods_r, variant=1)
            prev = tuple(a[perm] for a in prev)
            new_idx = np.sort(inv[idx]).astype(np.int64)
            got = handle.apply_state_delta_pods_reorder(pol, ro, lists, new_idx, {k: soa_r[k][new_idx] for k in ch}, soa["ds_rev"], n)
        else:
            got = handle.apply_state_delta_pods(pol, lists, idx, ch, soa["ds_rev"], soa["state"].shape[0])
        rc, n_out, oi, on, oa, oo, cnt = got
        full = _full_from_sparse(prev, n_out, oi, on, oa, oo)
        helpers.assert_same((rc, *full, cnt), ref, f"delta step {step}")
        diff = np.nonzero((prev[0] != ref[1]) | (prev[1] != ref[2]) | (prev[2] != ref[3]))[0]
        assert np.array_equal(np.sort(oi[:n_out]), diff), f"sparse = diff of full, step {step}"
        prev = (ref[1], ref[2], ref[3])


def test_mode_off_ignores_validation_bits(handle):
    soa, pods = snapshot()
    pol = abi.make_policy(**dict(POL_KW, evaluate_validation=False))
    helpers.assert_same(handle.apply_state(pol, soa, pods), helpers.oracle_apply(pol, soa, pods, variant=1), "mode off")
    soa_plain, pods_plain = synth.make_nodes(N, SEED, requestor_pct=5.0), synth.make_pods(N, SEED)
    # the same snapshot without the validation pods and bits: the same outputs
    helpers.assert_same(handle.apply_state(pol, soa, pods), handle.apply_state(pol, soa_plain, pods_plain), "bits ignored")


def test_rejected_before_device_work(handle):
    soa, pods = snapshot(n=5000)
    two = abi.make_policy(**dict(POL_KW, evaluate_actuators=False))
    assert two.evaluate_actuators == 2
    three = abi.make_policy(**POL_KW)
    before = handle.launch_count()
    assert handle.apply_state(two, soa, pods)[0] == INVALID
    assert handle.apply_state(three, soa, None)[0] == INVALID
    assert handle.apply_state_packed(three, soa)[0] == INVALID
    assert handle.launch_count() == before
    assert handle.apply_state(three, soa, pods)[0] == 0


def test_two_ranks():
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    import torch.multiprocessing as mp
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = 29900 + (os.getpid() % 2000)
    n = 120_000
    procs = [ctx.Process(target=_rank_worker, args=(r, 2, port, n, q)) for r in range(2)]
    for p in procs:
        p.start()
    gathered = q.get(timeout=600)
    for p in procs:
        p.join(timeout=120)
        assert p.exitcode == 0
    soa, pods = snapshot(n=2 * n)
    soa = with_invalid(soa, abortable(soa, pods)[[-3]])  # the abort lives on rank 1
    ref = vm.apply(abi.make_policy(**POL_KW), soa, pods, variant=1)
    nxt = np.concatenate([g[1] for g in gathered])
    act = np.concatenate([g[2] for g in gathered])
    oc = np.concatenate([g[3] for g in gathered])
    for g in gathered:
        assert g[0] == ref[0] and g[4] == ref[4]
    helpers.assert_same((ref[0], nxt, act, oc, ref[4]), ref, "two ranks")


def _rank_worker(rank, world, port, n, q):
    import torch
    import torch.distributed as dist
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", rank))
    h = ustlib.Handle(rank)
    uid = [ustlib.get_unique_id() if rank == 0 else None]
    dist.broadcast_object_list(uid, src=0)
    h.comm_init(rank, world, uid[0])
    soa, pods = snapshot(n=world * n)
    soa = with_invalid(soa, abortable(soa, pods)[[-3]])
    lo, hi = rank * n, (rank + 1) * n
    mine = {k: (soa[k][lo:hi] if k != "ds_rev" else soa[k]) for k in soa}
    off = pods["pod_off"]
    mp_ = {"pod_off": (off[lo:hi + 1] - off[lo]).astype(np.int32), "pod_flags": pods["pod_flags"][off[lo]:off[hi]]}
    res = h.apply_state(abi.make_policy(**POL_KW), mine, mp_)
    out = [None] * world
    dist.all_gather_object(out, res)
    if rank == 0:
        q.put(out)
    h.close()
    dist.destroy_process_group()
