"""Reconciles in which nodes of the resident pod-list snapshot move, join and leave, at C4 size
(ust_apply_state_delta_pods_reorder).

A 10 M-node C4 snapshot (~300 M workload pods) in pinned host memory. Series, each the median and spread (min, max) of
the host-clock time of the synchronous call, and of the device time of the call by CUDA events on the handle's stream:
  - full: ust_apply_state with pod lists;
  - delta_pods: ust_apply_state_delta_pods with 1 % of the lists replaced (mixed length changes) and 1 % of the nodes
    re-encoded, no moves;
  - moves: 0.1 % of the nodes moved to random positions, with the same 1 % lists and 1 % nodes;
  - joins_leaves: 0.1 % of the nodes leave and 0.1 % join, each inserted node with its list;
  - swap: the two halves swapped;
  - shuffle: a full shuffle (10 M runs of one node).
Also the host time of the list-length pass of each reorder series (ust_debug_pod_pass_ns), the kernels' own times from a
separate torch.profiler run, and the GPU name and power limit read in the same run. The last timed call's outputs are
checked against the oracle.
  NODES=10000000 STEPS=20 WARMUP=3 python scripts/micro/pods_reorder_bench.py"""
import ctypes as C
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
import pods_delta_model  # noqa: E402
import pods_reorder_model as model  # noqa: E402
import reorder_model  # noqa: E402
from ust import lib as ustlib, synth  # noqa: E402

COLS = ("state", "flags", "pod_rev", "ds_idx")
n = int(os.environ.get("NODES", "10000000"))
steps = int(os.environ.get("STEPS", "20"))
warm = int(os.environ.get("WARMUP", "3"))
rng = np.random.default_rng(2029)
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
pass_ns = h._lib.ust_debug_pod_pass_ns
pass_ns.restype = C.c_longlong
pass_ns.argtypes = [C.c_void_p]
stream = torch.cuda.ExternalStream(h.stream())
nxt, act, oc = ustlib.pinned_array(n, np.uint8), ustlib.pinned_array(n, np.uint16), ustlib.pinned_array(n, np.uint8)
cap = n + 1   # a full shuffle may report many nodes
out = (ustlib.pinned_array(cap + 1, np.int64), ustlib.pinned_array(cap + 1, np.uint8), ustlib.pinned_array(cap + 1, np.uint16),
       ustlib.pinned_array(cap + 1, np.uint8))
none_idx, none = np.zeros(0, np.int64), {k: soa[k][:0] for k in COLS}
no_ins = {k: soa[k][:0] for k in COLS}


def pinned_dict(d):
    return {k: pinned_copy(np.ascontiguousarray(v)) if v.size else v for k, v in d.items()}


def stats_us(ts):
    t = np.array(ts) * 1e6
    return {"median": round(float(np.median(t)), 1), "min": round(float(t.min()), 1), "max": round(float(t.max()), 1)}


def timed(call):
    """(host seconds, device seconds by CUDA events on the handle's stream, result) of one synchronous call."""
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(stream)
    t = time.perf_counter()
    r = call()
    dt = time.perf_counter() - t
    e1.record(stream)
    e1.synchronize()
    return dt, e0.elapsed_time(e1) * 1e-3, r


ts, dev = [], []
for i in range(warm + steps):
    dt, dd, r = timed(lambda: h.apply_state(pol, soa, pods, out=(nxt, act, oc)))
    assert r[0] == 0, (r[0], h.last_error())
    ts.append(dt)
    dev.append(dd)
result = {"full_apply_state_pods": {"host_us": stats_us(ts[warm:]), "device_us": stats_us(dev[warm:])}}
cur = {k: np.array(soa[k]) for k in COLS}
cur["ds_rev"] = soa["ds_rev"]
cur_pods = {"pod_off": np.array(pods["pod_off"]), "pod_flags": np.array(pods["pod_flags"])}
perm = None   # swap / shuffle series: the caller's snapshot is cur[perm], materialized once at the end


def churn(m_nodes):
    """1 % re-encoded nodes of a snapshot of m_nodes."""
    idx = np.sort(rng.choice(m_nodes, size=m_nodes // 100, replace=False)).astype(np.int64)
    f = synth.make_nodes(idx.shape[0], seed ^ 0xBEEF, start=int(rng.integers(0, 1 << 30)))
    return idx, {k: f[k] for k in COLS}


def moves_order(m):
    moved = rng.choice(m, size=m // 1000, replace=False)
    keep = np.delete(np.arange(m, dtype=np.int64), moved)
    return np.insert(keep, np.sort(rng.integers(0, keep.size + 1, size=moved.size)), rng.permutation(moved))


def one_call(series):
    """One call of a series; the caller's copy of the snapshot follows. Returns (host s, device s, pass ns, result)."""
    global cur, cur_pods, perm
    m = cur["state"].shape[0]
    if series == "delta_pods":
        li = pinned_dict(pods_delta_model.random_lists(rng, cur_pods["pod_off"], 0.01, "mixed"))
        idx, fr = churn(m)
        dt, dd, r = timed(lambda: h.apply_state_delta_pods(pol, li, idx, fr, cur["ds_rev"], cap, out=out))
        cur_pods["pod_off"], cur_pods["pod_flags"] = pods_delta_model.replace(cur_pods["pod_off"], cur_pods["pod_flags"], li["node_idx"],
                                                                              li["pod_off"], li["pod_flags"])
        for k in COLS:
            cur[k][idx] = fr[k]
        return dt, dd, 0, r
    if series == "moves":
        order = moves_order(m)
        li = model.random_lists(rng, order, cur_pods["pod_off"], 0.01, "mixed")
        idx, fr = churn(m)
        ins = no_ins
    elif series == "joins_leaves":
        order = reorder_model.random_order(rng, m, "identity", f_remove=0.001, f_insert=0.001)
        li = model.random_lists(rng, order, cur_pods["pod_off"], 0.0, "mixed")
        idx, fr = none_idx, none
        f = synth.make_nodes(int(np.sum(order < 0)), seed ^ 0xF00D, start=int(rng.integers(0, 1 << 30)))
        ins = {k: f[k] for k in COLS}
    else:
        order = (np.concatenate([np.arange(m // 2, m), np.arange(m // 2)]) if series == "swap" else rng.permutation(m)).astype(np.int64)
        li, idx, fr, ins = None, none_idx, none, no_ins
    rs, rl = reorder_model.runs_of(order)
    ro = pinned_dict(dict(run_src=rs, run_len=rl, **ins))
    if li is not None:
        li = pinned_dict(li)
    dt, dd, r = timed(lambda: h.apply_state_delta_pods_reorder(pol, ro, li, idx, fr, cur["ds_rev"], cap, out=out))
    ns = pass_ns(h._h)
    if li is None:   # swap / shuffle: a permutation without list or node changes
        perm = order if perm is None else perm[order]
    else:
        assert perm is None
        cur = {k: reorder_model.reorder(cur[k], rs, rl, ins[k]) for k in COLS} | {"ds_rev": cur["ds_rev"]}
        for k in COLS:
            cur[k][idx] = fr[k]
        cur_pods["pod_off"], cur_pods["pod_flags"] = model.reorder(cur_pods["pod_off"], cur_pods["pod_flags"], rs, rl, li["node_idx"],
                                                                   li["pod_off"], li["pod_flags"])
    return dt, dd, ns, r


last = None
for series in ("delta_pods", "moves", "joins_leaves", "swap", "shuffle"):
    ts, dev, ns = [], [], []
    for i in range(warm + steps):
        dt, dd, p, last = one_call(series)
        assert last[0] == 0, (series, last[0], h.last_error())
        ts.append(dt)
        dev.append(dd)
        ns.append(p)
    result[series] = {"host_us": stats_us(ts[warm:]), "device_us": stats_us(dev[warm:])}
    if series != "delta_pods":
        result[series]["list_length_pass_us"] = stats_us(np.array(ns[warm:]) * 1e-9)

# the last timed call against the oracle: its sparse entries and the full outputs it left resident
def permuted_pods(off, flags, p):
    """The CSR with node i taking the list of node p[i], gathered a million nodes at a time."""
    off = off.astype(np.int64)
    lens = np.diff(off)[p]
    new_off = np.zeros(p.size + 1, np.int64)
    np.cumsum(lens, out=new_off[1:])
    o = np.empty(int(new_off[-1]), np.uint16)
    for a in range(0, p.size, 1 << 20):
        b = min(a + (1 << 20), p.size)
        pos = np.repeat(off[p[a:b]] - new_off[a:b], lens[a:b]) + np.arange(new_off[a], new_off[b])
        o[new_off[a]:new_off[b]] = flags[pos]
    return {"pod_off": new_off.astype(np.int32), "pod_flags": o}


if perm is not None:
    cur = {k: cur[k][perm] for k in COLS} | {"ds_rev": cur["ds_rev"]}
    cur_pods = permuted_pods(cur_pods["pod_off"], cur_pods["pod_flags"], perm)
    perm = None
frc, fnxt, fact, foc = h.fetch_outputs_pods(n)
ref = helpers.oracle_apply(pol, cur, cur_pods, variant=1)
rc, n_out, oi, on, oa, oo, cnt = last
ok = (frc == 0 and rc == ref[0] and cnt == ref[4] and np.array_equal(fnxt, ref[1]) and np.array_equal(fact, ref[2])
      and np.array_equal(foc, ref[3]) and n_out <= cap and np.array_equal(on[:n_out], ref[1][oi[:n_out]])
      and np.array_equal(oa[:n_out], ref[2][oi[:n_out]]) and np.array_equal(oo[:n_out], ref[3][oi[:n_out]]))
assert ok, "pod-list reorder outputs differ from the oracle"

# the kernels' own times (medians over the profiled calls), in a run of their own
from torch.profiler import ProfilerActivity, profile  # noqa: E402
KERNELS = {"node_gather": r"ust_reorder_kernel<true>", "pod_run_table": r"ust_pods_reorder_runs_kernel",
           "pod_gather": r"ust_pods_reorder_kernel", "run_table": r"ust_pods_runs_kernel", "relayout": r"ust_pods_relayout_kernel",
           "streaming": r"ust_stream_kernel", "pod_summary": r"ust_pod_summary_kernel",
           "diff_count_outcome": r"ust_diff_count_kernel<true>", "diff_write_outcome": r"ust_diff_write_kernel<true>"}
kernel = {}
for series in ("delta_pods", "moves", "joins_leaves", "swap", "shuffle"):
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for i in range(3):
            one_call(series)
        torch.cuda.synchronize()
    kernel[series] = {}
    for name, pat in KERNELS.items():
        ev = [e.time_range.elapsed_us() for e in prof.events() if re.search(re.escape(pat), e.name)]
        if ev:
            kernel[series][name] = round(float(np.median(ev)), 1)

print(json.dumps({
    "gpu": gpu, "power_limit": power, "nodes": n, "pods": int(cur_pods["pod_off"][-1]), "steps": steps, "warmup": warm,
    "series_us": result, "kernel_us": kernel, "last_call_n_out": int(n_out), "oracle_check": "ok",
}))
h.close()
