"""Reconciles in which nodes move in BuildState's list, at C3 size (ust_apply_state_delta_reorder).

A 10 M-node C3 snapshot in pinned host memory. Series, each the median host-clock time of the synchronous call:
0.1 % of the nodes moved to random positions plus 1 % re-encoded (restarted driver pods under new names); the two halves
swapped plus 1 % re-encoded (two DaemonSets listed in the other order); a full shuffle; beside them a full
ust_apply_state and ust_apply_state_delta_sparse with the same 1 %. Also the gather kernel's own time from a separate
torch.profiler run, and the GPU name and power limit. The last timed reorder call's outputs are checked against the oracle.
  NODES=10000000 STEPS=60 WARMUP=5 python scripts/micro/reorder_bench.py"""
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
from ust import lib as ustlib, synth  # noqa: E402

COLS = ("state", "flags", "pod_rev", "ds_idx")
n = int(os.environ.get("NODES", "10000000"))
steps = int(os.environ.get("STEPS", "60"))
warm = int(os.environ.get("WARMUP", "5"))
rng = np.random.default_rng(2027)
seed = synth.CONFIGS["C3"]["seed"]
pol = synth.config_policy("C3")

gpu = torch.cuda.get_device_name(0)
try:
    power = subprocess.check_output(["nvidia-smi", "-i", "0", "--query-gpu=power.limit", "--format=csv,noheader"], text=True).strip()
except (OSError, subprocess.CalledProcessError) as e:
    power = f"unknown ({e})"

src = synth.make_nodes(n, seed)
soa = {k: ustlib.pinned_array(n, src[k].dtype) for k in COLS}
for k in COLS:
    soa[k][:] = src[k]
soa["ds_rev"] = src["ds_rev"]
del src
h = ustlib.Handle(0)
nxt, act = ustlib.pinned_array(n, np.uint8), ustlib.pinned_array(n, np.uint16)
cap = n // 4
out = (ustlib.pinned_array(cap + 1, np.int64), ustlib.pinned_array(cap + 1, np.uint8), ustlib.pinned_array(cap + 1, np.uint16))
none = {k: soa[k][:0] for k in COLS}


def fresh_nodes(m, start):
    f = synth.make_nodes(m, seed ^ 0xBEEF, start=start)
    return {k: f[k] for k in COLS}


def median_us(ts):
    return float(np.median(ts) * 1e6)


def one_pct(i):
    idx = np.sort(rng.choice(n, size=n // 100, replace=False)).astype(np.int64)
    return idx, fresh_nodes(idx.shape[0], 7 * n + i * n // 100)


ts = []
for i in range(warm + steps):
    t = time.perf_counter()
    rc = h.apply_state(pol, soa, want_outcome=False, out=(nxt, act, None))[0]
    ts.append(time.perf_counter() - t)
    assert rc == 0, rc
full_us = median_us(ts[warm:])

ts = []
for i in range(warm + steps):
    idx, fr = one_pct(i)
    t = time.perf_counter()
    rc = h.apply_state_delta_sparse(pol, idx, fr, soa["ds_rev"], cap, out=out)[0]
    ts.append(time.perf_counter() - t)
    assert rc == 0, rc
    for k in COLS:
        soa[k][idx] = fr[k]
sparse_us = median_us(ts[warm:])
cur = {k: np.array(soa[k]) for k in COLS}
cur["ds_rev"] = soa["ds_rev"]


def target(kind):
    if kind == "moves":  # 0.1 % of the nodes to random positions
        moved = rng.choice(n, size=n // 1000, replace=False)
        keep = np.delete(np.arange(n, dtype=np.int64), moved)
        return np.insert(keep, np.sort(rng.integers(0, keep.size + 1, size=moved.size)), rng.permutation(moved))
    if kind == "swap":
        return np.concatenate([np.arange(n // 2, n), np.arange(n // 2)]).astype(np.int64)
    return rng.permutation(n).astype(np.int64)


def series(kind, calls, overwrite):
    """`calls` reorder calls of one kind; host-clock seconds per call and the last call's result"""
    global cur
    ts, last = [], None
    for i in range(calls):
        src, ln = reorder_model.runs_of(target(kind))
        idx, fr = one_pct(100 + i) if overwrite else (np.zeros(0, np.int64), none)
        ro = dict(run_src=src, run_len=ln, **none)
        t = time.perf_counter()
        r = h.apply_state_delta_reorder(pol, ro, idx, fr, cur["ds_rev"], cap, out=out)
        ts.append(time.perf_counter() - t)
        assert r[0] == 0, (r[0], h.last_error())
        new = {k: reorder_model.reorder(cur[k], src, ln, cur[k][:0]) for k in COLS}
        for k in COLS:
            new[k][idx] = fr[k]
        new["ds_rev"] = cur["ds_rev"]
        cur = new
        last = r
    return ts, last, int(src.shape[0])


res = {}
for kind, overwrite in (("moves", True), ("swap", True), ("shuffle", False)):
    calls = warm + (steps if kind != "shuffle" else max(steps // 3, 10))
    ts, last, runs = series(kind, calls, overwrite)
    res[kind] = (median_us(ts[warm:]), runs)

# the last timed call (a full shuffle) against the oracle: its sparse entries and the full outputs it left resident
frc, fnxt, fact = h.fetch_outputs(n)
ref = helpers.oracle_apply(pol, cur, variant=1)
rc, n_out, oi, on, oa, cnt = last
ok = (frc == 0 and rc == ref[0] and cnt == ref[4] and np.array_equal(fnxt, ref[1]) and np.array_equal(fact, ref[2])
      and (n_out > cap or (np.array_equal(on[:n_out], ref[1][oi[:n_out]]) and np.array_equal(oa[:n_out], ref[2][oi[:n_out]]))))
assert ok, "reorder outputs differ from the oracle"

# the gather kernel's own time
from torch.profiler import ProfilerActivity, profile  # noqa: E402
kernel = {}
for kind in ("moves", "swap", "shuffle"):
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        series(kind, 5, kind != "shuffle")
        torch.cuda.synchronize()
    kern = [e for e in prof.events() if "ust_reorder_kernel" in e.name]
    kernel[kind] = round(float(np.median([e.time_range.elapsed_us() for e in kern])), 1) if kern else None

print(json.dumps({
    "gpu": gpu, "power_limit": power, "nodes": n, "steps": steps, "warmup": warm,
    "full_apply_state_us": round(full_us, 1), "delta_sparse_1pct_us": round(sparse_us, 1),
    "reorder_0.1pct_moved_1pct_us": round(res["moves"][0], 1), "reorder_0.1pct_moved_runs": res["moves"][1],
    "reorder_halves_swapped_1pct_us": round(res["swap"][0], 1),
    "reorder_full_shuffle_us": round(res["shuffle"][0], 1),
    "reorder_kernel_us": kernel, "last_call_n_out": int(n_out), "oracle_check": "ok",
}))
h.close()
