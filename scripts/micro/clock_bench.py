"""Reconciles in which only time passes, at C4 size (ust_apply_state_delta_pods_clocked).

A 10 M-node C4 snapshot (~300 M workload pods) in pinned host memory, under C4's policy plus a wait-for-completion selector
with a 300 s timeout; 80 % of the wait-for-jobs-required nodes carry a wait-start annotation, and every node a start time
in the last 700 s. Series, each the median and spread (min, max) of the host-clock time of the synchronous call, `now`
advancing 10 s per call:
  time_only_clocked       ust_apply_state_delta_pods_clocked with no node, no list, no reorder: the device derives bits 18
                          and 27 (one extra launch, ust_clock_kernel) and reports the nodes whose timeouts fired;
  resend_unclocked        what a caller does without it: ust_apply_state_delta_pods re-sending every wait-for-jobs-required
                          and validation-required node (~7 % of the snapshot) with bits 18 and 27 derived on the host
                          (the host derivation is not timed);
  time_only_unclocked     ust_apply_state_delta_pods with nothing at all: the floor, wrong once a deadline passes.
Also the clock kernel's own time from a separate torch.profiler run, the bytes it must read and write, and the GPU name,
power limit and SM clocks. The last clocked and re-sending calls' full outputs are checked against each other.
  NODES=10000000 STEPS=20 WARMUP=3 python scripts/micro/clock_bench.py"""
import json
import os
import re
import subprocess
import sys
import time

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "..", "..", "k8s-operator-libs_b200"))
sys.path.insert(0, os.path.join(HERE, "..", "..", "tests"))
import numpy as np  # noqa: E402
import torch  # noqa: E402

import clock_model as cm  # noqa: E402
from ust import abi, lib as ustlib, synth  # noqa: E402

COLS = ("state", "flags", "pod_rev", "ds_idx")
n = int(os.environ.get("NODES", "10000000"))
steps = int(os.environ.get("STEPS", "20"))
warm = int(os.environ.get("WARMUP", "3"))
NOW, TIMEOUT = 1_700_000_000, 300
cfg = synth.CONFIGS["C4"]
pol = abi.make_policy(auto_upgrade=True, **dict(cfg["policy"], wait_for_completion={"podSelector": "app=batch", "timeoutSeconds": TIMEOUT}))

gpu = torch.cuda.get_device_name(0)
try:
    smi = subprocess.check_output(["nvidia-smi", "-i", "0", "--query-gpu=power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                                  text=True).strip()
except (OSError, subprocess.CalledProcessError) as e:
    smi = f"unknown ({e})"


def pinned_copy(a):
    p = ustlib.pinned_array(a.shape[0], a.dtype)
    p[:] = a
    return p


def stats_us(ts):
    t = np.array(ts) * 1e6
    return {"median": round(float(np.median(t)), 1), "min": round(float(t.min()), 1), "max": round(float(t.max()), 1)}


rng = np.random.default_rng(2029)
src = synth.make_nodes(n, cfg["seed"])
code = src["state"] & 15
w = code == abi.UST_STATE_WAIT_FOR_JOBS_REQUIRED
src["flags"] = (src["flags"] | np.where(w & (rng.random(n) < 0.8), np.uint32(abi.UST_F_WAIT_START_ANNO), np.uint32(0))).astype(np.uint32)
soa = {k: pinned_copy(src[k]) for k in COLS}
soa["ds_rev"] = src["ds_rev"]
start = pinned_copy((NOW - rng.integers(0, 700, n)).astype(np.int64))
del src
pods = synth.make_pods_blocked(n, cfg["seed"])
pods = {"pod_off": pinned_copy(pods["pod_off"]), "pod_flags": pinned_copy(pods["pod_flags"])}
clocked_nodes = np.nonzero(np.isin(code, [abi.UST_STATE_WAIT_FOR_JOBS_REQUIRED, abi.UST_STATE_VALIDATION_REQUIRED]))[0].astype(np.int64)
m = clocked_nodes.shape[0]
valid_anno = int(np.count_nonzero(w & ((soa["flags"] & np.uint32(cm.WAIT_BITS)) == abi.UST_F_WAIT_START_ANNO)))

hc, hu = ustlib.Handle(0), ustlib.Handle(0)   # clocked / unclocked snapshot
nxt, act, oc = ustlib.pinned_array(n, np.uint8), ustlib.pinned_array(n, np.uint16), ustlib.pinned_array(n, np.uint8)
cap = n // 8
out = (ustlib.pinned_array(cap + 1, np.int64), ustlib.pinned_array(cap + 1, np.uint8), ustlib.pinned_array(cap + 1, np.uint16),
       ustlib.pinned_array(cap + 1, np.uint8))
none_idx, none, none_st = np.zeros(0, np.int64), {k: soa[k][:0] for k in COLS}, np.zeros(0, np.int64)
# the re-sent nodes of the unclocked alternative, staged in pinned memory like the snapshot
rs_idx = pinned_copy(clocked_nodes)
rs = {k: pinned_copy(soa[k][clocked_nodes]) for k in COLS}
rs_start = start[clocked_nodes]

rc = hc.apply_state_clocked(pol, NOW, TIMEOUT, start, soa, pods, out=(nxt, act, oc))[0]
assert rc == 0, (rc, hc.last_error())
rc = hu.apply_state(pol, cm.derived_soa(soa, start, NOW, TIMEOUT), pods, out=(nxt, act, oc))[0]
assert rc == 0, (rc, hu.last_error())

res = {"time_only_clocked": [], "resend_unclocked": [], "time_only_unclocked": []}
fired = []
now = NOW
for i in range(warm + steps):
    now += 10
    t = time.perf_counter()
    r = hc.apply_state_delta_pods_clocked(pol, now, TIMEOUT, None, None, none_idx, none, none_st, soa["ds_rev"], cap, out=out)
    dt = time.perf_counter() - t
    assert r[0] == 0, (r[0], hc.last_error())
    fired.append(r[1])
    rs["flags"][:] = cm.derive(rs["state"], rs["flags"], rs_start, now, TIMEOUT)
    t2 = time.perf_counter()
    r2 = hu.apply_state_delta_pods(pol, None, rs_idx, rs, soa["ds_rev"], cap, out=out)
    dt2 = time.perf_counter() - t2
    assert r2[0] == 0, (r2[0], hu.last_error())
    if i >= warm:
        res["time_only_clocked"].append(dt)
        res["resend_unclocked"].append(dt2)

# the two snapshots answered the same at the last `now`
a, b = hc.fetch_outputs_pods(n), hu.fetch_outputs_pods(n)
assert a[0] == b[0] == 0 and all(np.array_equal(x, y) for x, y in zip(a[1:], b[1:])), "clocked and re-sending calls disagree"

# the floor: a delta that carries nothing (on the unclocked snapshot, whose bits then stay as they were)
for i in range(warm + steps):
    t = time.perf_counter()
    r = hu.apply_state_delta_pods(pol, None, none_idx, none, soa["ds_rev"], cap, out=out)
    dt = time.perf_counter() - t
    assert r[0] == 0
    if i >= warm:
        res["time_only_unclocked"].append(dt)

# the kernels' own times (medians over the profiled calls): the clocked time-only calls, then the floor
from torch.profiler import ProfilerActivity, profile  # noqa: E402


def kernel_times(call):
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for i in range(10):
            call(i)
        torch.cuda.synchronize()
    names = {}
    for e in prof.events():
        m = re.search(r"(ust_\w+_kernel(?:<[^>]*>)?)", e.name)
        if m:
            names.setdefault(m.group(1), []).append(e.time_range.elapsed_us())
    return {k: round(float(np.median(v)), 1) for k, v in sorted(names.items())}


kernel = kernel_times(lambda i: hc.apply_state_delta_pods_clocked(pol, now + 10 * (i + 1), TIMEOUT, None, None, none_idx, none, none_st,
                                                                  soa["ds_rev"], cap, out=out))
kernel_floor = kernel_times(lambda i: hu.apply_state_delta_pods(pol, None, none_idx, none, soa["ds_rev"], cap, out=out))
clock_us = next((v for k, v in kernel.items() if "ust_clock_kernel" in k), None)
# bytes the clock kernel must move: the hot column, the flags word of every wait-for-jobs / validation-required node, the
# start of those with a valid annotation (validation starts are ignored here: C4 has no validation-mode policy, but the
# kernel reads them by annotation all the same - none carry one), and the words it rewrites (at most every such word)
must_read = n + 4 * m + 8 * valid_anno
print(json.dumps({
    "gpu": gpu, "power_limit_sm_clock_max_sm_clock": smi, "nodes": n, "pods": int(pods["pod_off"][-1]), "steps": steps, "warmup": warm,
    "clocked_nodes": int(m), "clocked_share_pct": round(100.0 * m / n, 2), "valid_wait_annotations": valid_anno,
    "time_only_clocked_us": stats_us(res["time_only_clocked"]), "resend_unclocked_us": stats_us(res["resend_unclocked"]),
    "time_only_unclocked_floor_us": stats_us(res["time_only_unclocked"]),
    "clock_kernel_us": clock_us, "clock_kernel_must_read_bytes": must_read,
    "clock_kernel_GBps_on_must_read": round(must_read / clock_us / 1e3, 1) if clock_us else None,
    "kernel_us_time_only_clocked": kernel, "kernel_us_floor": kernel_floor, "fired_per_call_median": int(np.median(fired[warm:])) if steps else 0, "parity": "ok",
}))
hc.close()
hu.close()
