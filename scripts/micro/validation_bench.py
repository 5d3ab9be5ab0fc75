"""The cost of answering Validate on the device (UST_EVAL_VALIDATION), at C4 size.

A 10 M-node C4 snapshot whose validation-required nodes (2 %) carry 0-3 validation pods and start-time bits
(synth.make_validation_pods), in pinned host memory. Series, alternated call by call, each the median and spread (min, max)
of the host-clock time of the synchronous ust_apply_state with pod lists: the C4 policy with the mode off, and with the
mode on. Then, in a separate torch.profiler run, the kernel times of both (the pod-summary kernel among them), and the GPU
name and power limit. The last timed call of each series is checked against validation_model / the oracle. The summary
(validation_bench.json) and the profiler traces go to the directory OUT names (default: a new temporary directory).
  NODES=10000000 STEPS=20 WARMUP=3 OUT=/tmp/validation_bench python scripts/micro/validation_bench.py"""
import json
import os
import re
import subprocess
import sys
import tempfile
import time

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "..", "..", "k8s-operator-libs_b200"))
sys.path.insert(0, os.path.join(HERE, "..", "..", "tests"))
import numpy as np  # noqa: E402
import torch  # noqa: E402

import helpers  # noqa: E402
import validation_model as vm  # noqa: E402
from ust import abi, lib as ustlib, synth  # noqa: E402

COLS = ("state", "flags", "pod_rev", "ds_idx")
n = int(os.environ.get("NODES", "10000000"))
steps = int(os.environ.get("STEPS", "20"))
warm = int(os.environ.get("WARMUP", "3"))
out_dir = os.environ.get("OUT") or tempfile.mkdtemp()
os.makedirs(out_dir, exist_ok=True)
seed = synth.CONFIGS["C4"]["seed"]
kw = dict(synth.CONFIGS["C4"]["policy"], validation_enabled=True)
pols = {"off": abi.make_policy(**kw), "on": abi.make_policy(**kw, evaluate_validation=True)}

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
flags, vpods = synth.make_validation_pods(src, synth.make_pods_blocked(n, seed), seed)
src["flags"] = flags
soa = {k: pinned_copy(src[k]) for k in COLS}
soa["ds_rev"] = src["ds_rev"]
pods = {"pod_off": pinned_copy(vpods["pod_off"]), "pod_flags": pinned_copy(vpods["pod_flags"])}
del src, flags, vpods
h = ustlib.Handle(0)
outs = {m: (ustlib.pinned_array(n, np.uint8), ustlib.pinned_array(n, np.uint16), ustlib.pinned_array(n, np.uint8)) for m in pols}

times = {m: [] for m in pols}
res = {}
for it in range(warm + steps):
    for m in ("off", "on") if it % 2 == 0 else ("on", "off"):
        t0 = time.perf_counter()
        res[m] = h.apply_state(pols[m], soa, pods, out=outs[m], check=True)
        dt = time.perf_counter() - t0
        if it >= warm:
            times[m].append(dt * 1e3)

# kernel times: one profiled call of each after a warm-up
from torch.profiler import ProfilerActivity, profile  # noqa: E402
kernels = {}
for m in pols:
    h.apply_state(pols[m], soa, pods, out=outs[m], check=True)
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(3):
            h.apply_state(pols[m], soa, pods, out=outs[m], check=True)
    torch.cuda.synchronize()
    ev = {}
    for e in prof.events():
        if e.device_type.name == "CUDA" and "ust_" in e.name:
            m_ = re.search(r"(ust_\w+(?:<[^>]*>)?)", e.name)
            ev.setdefault(m_.group(1) if m_ else e.name[:60], []).append(getattr(e, "device_time_total", 0) or e.cuda_time_total)
    kernels[m] = {k: round(float(np.median(v)), 1) for k, v in ev.items()}
    prof.export_chrome_trace(os.path.join(out_dir, f"validation_bench_{m}.pt.trace.json"))

# outputs of the last timed calls against the CPU restatements (at most 2 M nodes: the oracle is single-threaded)
check_n = min(n, 2_000_000)
cut = {k: np.array(soa[k][:check_n]) for k in COLS}
cut["ds_rev"] = soa["ds_rev"]
cpods = {"pod_off": np.array(pods["pod_off"][:check_n + 1]), "pod_flags": np.array(pods["pod_flags"][:int(pods["pod_off"][check_n])])}
checked = {}
for m in pols:
    got = h.apply_state(pols[m], cut, cpods)
    ref = vm.apply(pols[m], cut, cpods, variant=1) if m == "on" else helpers.oracle_apply(pols[m], cut, cpods, variant=1)
    helpers.assert_same(got, ref, f"mode {m}")
    checked[m] = check_n

summary = {
    "gpu": gpu, "power_limit": power, "nodes": n, "pods": int(pods["pod_off"][-1]),
    "validation_required": int(np.sum((soa["state"] & 15) == 9)),
    "call_ms": {m: {"median": round(float(np.median(v)), 3), "min": round(min(v), 3), "max": round(max(v), 3)} for m, v in times.items()},
    "kernel_us": kernels, "checked_nodes": checked,
}
print(json.dumps(summary))
with open(os.path.join(out_dir, "validation_bench.json"), "w") as f:
    json.dump(summary, f, indent=1)
h.close()
