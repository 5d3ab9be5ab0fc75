"""BuildState's driver-pod list on the device (ust_build_state_delta) at 10 M driver pods.

The pods live in pinned host memory. Reported: median host-clock time of the synchronous call for a full
ust_build_state_uids, ust_build_state_delta with 1 % of the pods re-derived, with 0.1 % leaving and 0.1 % joining, with
0.1 % moved, and one full incremental reconcile (ust_build_state_delta with 1 % re-derived + ust_apply_state_delta_splice
on a 10 M-node C3 snapshot with 0.1 % out, 0.1 % in, 1 % re-encoded); the kernels' own times from a separate
torch.profiler run; the GPU name and power limit. The last timed call's outputs are checked against the oracle.
  PODS=10000000 STEPS=30 WARMUP=5 python scripts/micro/build_state_delta_bench.py"""
import json
import os
import subprocess
import sys
import time

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "..", "..", "k8s-operator-libs_b200"))
sys.path.insert(0, os.path.join(HERE, "..", "..", "tests"))
import numpy as np  # noqa: E402
import torch  # noqa: E402

import helpers  # noqa: E402
import reorder_model  # noqa: E402
import splice_model  # noqa: E402
from ust import lib as ustlib, synth  # noqa: E402

n = int(os.environ.get("PODS", "10000000"))
steps = int(os.environ.get("STEPS", "30"))
warm = int(os.environ.get("WARMUP", "5"))
rng = np.random.default_rng(2027)

gpu = torch.cuda.get_device_name(0)
try:
    power = subprocess.check_output(["nvidia-smi", "-i", "0", "--query-gpu=power.limit", "--format=csv,noheader"], text=True).strip()
except (OSError, subprocess.CalledProcessError) as e:
    power = f"unknown ({e})"

N_DS = 4
ds_uid = rng.integers(1, 2 ** 63, size=(N_DS, 2), dtype=np.uint64)


def new_pods(m):
    """m driver pods: 97 % owned by the driver DaemonSets, 2 % orphaned, 1 % owned by something else; states as BuildState
    encodes them (UST_STATE_OTHER, 1 % pending and unscheduled)."""
    state = np.where(rng.random(m) < 0.01, 14, 13).astype(np.uint8)
    owner = ds_uid[rng.integers(0, N_DS, m)]
    k = rng.random(m)
    owner[(k >= 0.97) & (k < 0.99)] = 0
    foreign = k >= 0.99
    owner[foreign] = rng.integers(2 ** 63, 2 ** 64 - 1, size=(int(foreign.sum()), 2), dtype=np.uint64)
    return state, owner


def desired_of(owner):
    ds_idx = helpers.oracle_build_state_uids(np.zeros(owner.shape[0], np.uint8), owner, ds_uid, np.zeros(N_DS, np.int32))[1]
    return np.bincount(ds_idx[ds_idx >= 0], minlength=N_DS).astype(np.int32)


src_state, src_owner = new_pods(n)
state = ustlib.pinned_array(n, np.uint8)
owner = ustlib.pinned_array((n, 2), np.uint64)
state[:] = src_state
owner[:] = src_owner
del src_state, src_owner
desired = desired_of(owner)
h = ustlib.Handle(0)
ds_out = ustlib.pinned_array(n, np.int32)
cap = n // 4
out = (ustlib.pinned_array(cap + 1, np.int64), ustlib.pinned_array(cap + 1, np.int32))


def median_us(ts):
    return float(np.median(ts) * 1e6)


# full ust_build_state_uids (pinned host arrays)
ts = []
for i in range(warm + steps):
    t = time.perf_counter()
    rc = h._lib.ust_build_state_uids(h._h, n, state.ctypes.data, owner.ctypes.data, N_DS, ds_uid.ctypes.data, desired.ctypes.data,
                                     ds_out.ctypes.data, None)
    ts.append(time.perf_counter() - t)
    assert rc == 0, h.last_error()
full_us = median_us(ts[warm:])

# the list made resident: everything as one inserted run
cur = {"state": np.array(state), "owner": np.array(owner)}
rc = h.build_state_delta(dict(run_src=[-1], run_len=[n], state=state, owner_uid=owner), np.zeros(0, np.int64), np.zeros(0, np.uint8),
                         np.zeros((0, 2), np.uint64), ds_uid, desired, cap, out=out)[0]
assert rc == helpers.abi.K["UST_ERR_TRUNCATED"], h.last_error()   # all n pods come back: fetched, not needed here
none = np.zeros(0, np.int64)


def series(calls, kind):
    """`calls` ust_build_state_delta calls of one kind; host-clock seconds per call and the last call's result"""
    global cur
    ts, last = [], None
    for _ in range(calls):
        m = cur["state"].shape[0]
        order, ins = None, (np.zeros(0, np.uint8), np.zeros((0, 2), np.uint64))
        idx = none
        if kind == "rederive":
            idx = np.sort(rng.choice(m, size=m // 100, replace=False)).astype(np.int64)
        elif kind == "membership":
            order = reorder_model.random_order(rng, m, "identity", f_remove=0.001, f_insert=0.001)
            ins = new_pods(int(np.sum(order < 0)))
        elif kind == "moves":
            moved = rng.choice(m, size=m // 1000, replace=False)
            keep = np.delete(np.arange(m, dtype=np.int64), moved)
            order = np.insert(keep, np.sort(rng.integers(0, keep.size + 1, size=moved.size)), rng.permutation(moved))
        new = {k: v for k, v in cur.items()}
        ro = None
        if order is not None:
            run_src, run_len = reorder_model.runs_of(order)
            ro = dict(run_src=run_src, run_len=run_len, state=ins[0], owner_uid=ins[1])
            new["state"] = reorder_model.reorder(cur["state"], run_src, run_len, ins[0])
            new["owner"] = np.stack([reorder_model.reorder(cur["owner"][:, j].copy(), run_src, run_len, ins[1][:, j]) for j in (0, 1)], 1)
        chg = new_pods(idx.size)
        new["state"] = new["state"].copy()
        new["owner"] = new["owner"].copy()
        new["state"][idx] = chg[0]
        new["owner"][idx] = chg[1]
        des = desired_of(new["owner"])
        t = time.perf_counter()
        r = h.build_state_delta(ro, idx, chg[0], chg[1], ds_uid, des, cap, out=out)
        ts.append(time.perf_counter() - t)
        assert r[0] == 0, (r[0], h.last_error())
        cur = new
        last = (r, des)
    return ts, last


res = {}
for kind in ("rederive", "membership", "moves"):
    ts, (last, des) = series(warm + steps, kind)
    res[kind] = median_us(ts[warm:])
# the last timed call against the oracle: counters, and the full owner indices it left resident
orc, ods, ocnt = helpers.oracle_build_state_uids(cur["state"], cur["owner"], ds_uid, des)
frc, full = h.fetch_build_state(cur["state"].shape[0])
assert orc == last[0] == 0 and last[4] == ocnt and frc == 0 and np.array_equal(full, ods), "build-state outputs differ from the oracle"
oi, od = last[2], last[3]
assert np.array_equal(od[:last[1]], ods[oi[:last[1]]]), "sparse owner indices differ from the oracle"

# one full incremental reconcile: BuildState's list (1 % re-derived) + ApplyState's snapshot (0.1 % out, 0.1 % in, 1 % re-encoded)
COLS = ("state", "flags", "pod_rev", "ds_idx")
seed = synth.CONFIGS["C3"]["seed"]
pol = synth.config_policy("C3")
snap = synth.make_nodes(n, seed)
nxt, act = ustlib.pinned_array(n, np.uint8), ustlib.pinned_array(n, np.uint16)
assert h.apply_state(pol, snap, want_outcome=False, out=(nxt, act, None))[0] == 0
aout = (ustlib.pinned_array(cap + 1, np.int64), ustlib.pinned_array(cap + 1, np.uint8), ustlib.pinned_array(cap + 1, np.uint16))
ts = []
for i in range(warm + steps):
    m = snap["state"].shape[0]
    rm, ib = splice_model.random_splice(rng, m, 0.001, 0.001)
    f = synth.make_nodes(ib.shape[0], seed ^ 0xF00D, start=20 * n + i * n)
    ins = {k: f[k] for k in COLS}
    m_new = m - rm.shape[0] + ib.shape[0]
    aidx = np.sort(rng.choice(m_new, size=m_new // 100, replace=False)).astype(np.int64)
    g = synth.make_nodes(aidx.shape[0], seed ^ 0xBEEF, start=40 * n + i * n)
    fr = {k: g[k] for k in COLS}
    bidx = np.sort(rng.choice(cur["state"].shape[0], size=cur["state"].shape[0] // 100, replace=False)).astype(np.int64)
    chg = (cur["state"][bidx], cur["owner"][bidx])   # re-derived, unchanged values
    t = time.perf_counter()
    rb = h.build_state_delta(None, bidx, chg[0], chg[1], ds_uid, des, cap, out=out)[0]
    ra = h.apply_state_delta_splice(pol, dict(remove_idx=rm, insert_before=ib, **ins), aidx, fr, snap["ds_rev"], cap, out=aout)[0]
    ts.append(time.perf_counter() - t)
    assert rb == 0 and ra == 0, (rb, ra, h.last_error())
    new = {k: splice_model.splice(snap[k], rm, ib, ins[k]) for k in COLS}
    for k in COLS:
        new[k][aidx] = fr[k]
    new["ds_rev"] = snap["ds_rev"]
    snap = new
reconcile_us = median_us(ts[warm:])

# the kernels' own times
from torch.profiler import ProfilerActivity, profile  # noqa: E402
with profile(activities=[ProfilerActivity.CUDA]) as prof:
    for kind in ("rederive", "moves"):
        series(5, kind)
    torch.cuda.synchronize()
kernels = {}
for e in prof.events():
    for name in ("ust_build_state_delta_kernel", "ust_build_state_write_kernel", "ust_build_state_reorder_kernel",
                 "ust_build_state_patch_kernel", "ust_diff_scan_kernel", "ust_build_state_finish_kernel"):
        if name in e.name:
            kernels.setdefault(name, []).append(e.time_range.elapsed_us())
kernel_us = {k: round(float(np.median(v)), 1) for k, v in kernels.items()}

print(json.dumps({
    "gpu": gpu, "power_limit": power, "pods": n, "steps": steps, "warmup": warm,
    "build_state_uids_full_us": round(full_us, 1), "build_state_delta_1pct_rederived_us": round(res["rederive"], 1),
    "build_state_delta_0.1pct_out_0.1pct_in_us": round(res["membership"], 1), "build_state_delta_0.1pct_moved_us": round(res["moves"], 1),
    "reconcile_build_state_delta_plus_apply_state_delta_splice_us": round(reconcile_us, 1), "kernel_median_us": kernel_us,
    "oracle_check": "ok",
}))
h.close()
