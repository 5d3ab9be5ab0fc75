"""Reconciles that replace workload pod lists, at C4 size (ust_apply_state_delta_pods).

A 10 M-node C4 snapshot (~300 M workload pods) in pinned host memory. Series, each the median and spread (min, max) of
the host-clock time of the synchronous call: a full ust_apply_state with pod lists; ust_apply_state_delta_pods with 1 % of
the lists replaced at the same lengths (pods changing phase: the in-place scatter); the same with changed lengths (the
relayout); and each of the two delta series with 1 % of the nodes re-encoded as well. Also the kernels' own times from a
separate torch.profiler run (scatter, run table + relayout, the outcome-comparing diff), and the GPU name and power limit.
The last timed call's outputs are checked against the oracle.
  NODES=10000000 STEPS=20 WARMUP=3 python scripts/micro/pods_delta_bench.py"""
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

import helpers  # noqa: E402
import pods_delta_model as model  # noqa: E402
from ust import lib as ustlib, synth  # noqa: E402

COLS = ("state", "flags", "pod_rev", "ds_idx")
n = int(os.environ.get("NODES", "10000000"))
steps = int(os.environ.get("STEPS", "20"))
warm = int(os.environ.get("WARMUP", "3"))
rng = np.random.default_rng(2028)
seed = synth.CONFIGS["C4"]["seed"]
pol = synth.config_policy("C4")

gpu = torch.cuda.get_device_name(0)
try:
    power = subprocess.check_output(["nvidia-smi", "-i", "0", "--query-gpu=power.limit", "--format=csv,noheader"], text=True).strip()
except (OSError, subprocess.CalledProcessError) as e:
    power = f"unknown ({e})"


def pinned_copy(a):
    p = ustlib.pinned_array(a.shape[0], a.dtype)
    p[:] = a
    return p


src = synth.make_nodes(n, seed)
soa = {k: pinned_copy(src[k]) for k in COLS}
soa["ds_rev"] = src["ds_rev"]
del src
pods = synth.make_pods_blocked(n, seed)
pods = {"pod_off": pinned_copy(pods["pod_off"]), "pod_flags": pinned_copy(pods["pod_flags"])}
h = ustlib.Handle(0)
nxt, act, oc = ustlib.pinned_array(n, np.uint8), ustlib.pinned_array(n, np.uint16), ustlib.pinned_array(n, np.uint8)
cap = n // 8
out = (ustlib.pinned_array(cap + 1, np.int64), ustlib.pinned_array(cap + 1, np.uint8), ustlib.pinned_array(cap + 1, np.uint16),
       ustlib.pinned_array(cap + 1, np.uint8))
none_idx, none = np.zeros(0, np.int64), {k: soa[k][:0] for k in COLS}
# the replacement lists of a call, staged in pinned memory like the snapshot
L_CAP, P_CAP = n // 100 + 1, 64 * (n // 100) + 64
pl_idx, pl_off, pl_flags = ustlib.pinned_array(L_CAP, np.int64), ustlib.pinned_array(L_CAP + 1, np.int32), ustlib.pinned_array(P_CAP, np.uint16)


def stats_us(ts):
    t = np.array(ts) * 1e6
    return {"median": round(float(np.median(t)), 1), "min": round(float(t.min()), 1), "max": round(float(t.max()), 1)}


ts = []
for i in range(warm + steps):
    t = time.perf_counter()
    rc = h.apply_state(pol, soa, pods, out=(nxt, act, oc))[0]
    ts.append(time.perf_counter() - t)
    assert rc == 0, (rc, h.last_error())
full = stats_us(ts[warm:])
cur = {k: np.array(soa[k]) for k in COLS}
cur["ds_rev"] = soa["ds_rev"]
cur_pods = {"pod_off": np.array(pods["pod_off"]), "pod_flags": np.array(pods["pod_flags"])}


def one_call(kind, overwrite, i):
    """Lists of 1 % of the nodes (`kind`: same lengths or mixed length changes) and optionally 1 % re-encoded nodes; the
    caller's copy of the snapshot follows."""
    global cur, cur_pods
    li = model.random_lists(rng, cur_pods["pod_off"], 0.01, kind)
    L, P = li["node_idx"].shape[0], li["pod_flags"].shape[0]
    pl_idx[:L], pl_off[:L + 1], pl_flags[:P] = li["node_idx"], li["pod_off"], li["pod_flags"]
    lists = {"node_idx": pl_idx[:L], "pod_off": pl_off[:L + 1], "pod_flags": pl_flags[:P]}
    if overwrite:
        idx = np.sort(rng.choice(n, size=n // 100, replace=False)).astype(np.int64)
        f = synth.make_nodes(idx.shape[0], seed ^ 0xBEEF, start=7 * n + i * (n // 100))
        fr = {k: f[k] for k in COLS}
    else:
        idx, fr = none_idx, none
    t = time.perf_counter()
    r = h.apply_state_delta_pods(pol, lists, idx, fr, cur["ds_rev"], cap, out=out)
    dt = time.perf_counter() - t
    assert r[0] == 0, (r[0], h.last_error())
    if kind == "same":  # offsets stay: the new lists land where the old ones were
        off = cur_pods["pod_off"].astype(np.int64)
        starts = off[li["node_idx"]]
        lens = np.diff(li["pod_off"].astype(np.int64))
        pos = np.repeat(starts - li["pod_off"][:-1], lens) + np.arange(P)
        cur_pods["pod_flags"][pos] = li["pod_flags"]
    else:
        cur_pods["pod_off"], cur_pods["pod_flags"] = model.replace(cur_pods["pod_off"], cur_pods["pod_flags"], li["node_idx"],
                                                                   li["pod_off"], li["pod_flags"])
    for k in COLS:
        cur[k][idx] = fr[k]
    return dt, r


res, last = {}, None
for kind in ("same", "mixed"):
    for overwrite in (False, True):
        ts = []
        for i in range(warm + steps):
            dt, last = one_call(kind, overwrite, i)
            ts.append(dt)
        res[f"{kind}{'_1pct_nodes' if overwrite else ''}"] = stats_us(ts[warm:])

# the last timed call against the oracle: its sparse entries and the full outputs it left resident
frc, fnxt, fact, foc = h.fetch_outputs_pods(n)
ref = helpers.oracle_apply(pol, cur, cur_pods, variant=1)
rc, n_out, oi, on, oa, oo, cnt = last
ok = (frc == 0 and rc == ref[0] and cnt == ref[4] and np.array_equal(fnxt, ref[1]) and np.array_equal(fact, ref[2])
      and np.array_equal(foc, ref[3]) and n_out <= cap and np.array_equal(on[:n_out], ref[1][oi[:n_out]])
      and np.array_equal(oa[:n_out], ref[2][oi[:n_out]]) and np.array_equal(oo[:n_out], ref[3][oi[:n_out]]))
assert ok, "pod-list delta outputs differ from the oracle"

# the kernels' own times (medians over the profiled calls)
from torch.profiler import ProfilerActivity, profile  # noqa: E402
KERNELS = {"scatter": r"ust_pods_scatter_kernel", "run_table": r"ust_pods_runs_kernel", "relayout": r"ust_pods_relayout_kernel",
           "diff_count_outcome": r"ust_diff_count_kernel<true>", "diff_write_outcome": r"ust_diff_write_kernel<true>"}
kernel = {}
for kind in ("same", "mixed"):
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for i in range(5):
            one_call(kind, False, 1000 + i)
        torch.cuda.synchronize()
    for name, pat in KERNELS.items():
        ev = [e.time_range.elapsed_us() for e in prof.events() if re.search(re.escape(pat), e.name)]
        if ev:
            kernel[f"{name} ({kind})"] = round(float(np.median(ev)), 1)

print(json.dumps({
    "gpu": gpu, "power_limit": power, "nodes": n, "pods": int(cur_pods["pod_off"][-1]), "steps": steps, "warmup": warm,
    "full_apply_state_pods_us": full,
    "delta_pods_1pct_lists_same_lengths_us": res["same"], "delta_pods_1pct_lists_changed_lengths_us": res["mixed"],
    "delta_pods_1pct_lists_same_lengths_1pct_nodes_us": res["same_1pct_nodes"],
    "delta_pods_1pct_lists_changed_lengths_1pct_nodes_us": res["mixed_1pct_nodes"],
    "kernel_us": kernel, "last_call_n_out": int(n_out), "oracle_check": "ok",
}))
h.close()
