"""Reconciles with membership changes at C3 size (ust_apply_state_delta_splice).

A 10 M-node C3 snapshot in pinned host memory. Each splice call removes 0.1 % of the nodes, inserts 0.1 % at random
positions and re-encodes 1 %. Reported: median host-clock time of the synchronous call, beside ust_apply_state_delta_sparse
with the same 1 % and no membership change, a full ust_apply_state, and splices that change the snapshot size on every
call (the speculation hint is kept per size, so those run without one); the splice kernel's own time from a separate
torch.profiler run; the GPU name and power limit. The last timed splice call's outputs are checked against the oracle.
  NODES=10000000 STEPS=60 WARMUP=5 python scripts/micro/splice_bench.py"""
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
import splice_model  # noqa: E402
from ust import lib as ustlib, synth  # noqa: E402

COLS = ("state", "flags", "pod_rev", "ds_idx")
n = int(os.environ.get("NODES", "10000000"))
steps = int(os.environ.get("STEPS", "60"))
warm = int(os.environ.get("WARMUP", "5"))
rng = np.random.default_rng(2026)
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


def fresh_nodes(m, start):
    f = synth.make_nodes(m, seed ^ 0xF00D, start=start)
    return {k: f[k] for k in COLS}


def median_us(ts):
    return float(np.median(ts) * 1e6)


# full ust_apply_state (host arrays, pinned)
ts = []
for i in range(warm + steps):
    t = time.perf_counter()
    rc = h.apply_state(pol, soa, want_outcome=False, out=(nxt, act, None))[0]
    ts.append(time.perf_counter() - t)
    assert rc == 0, rc
full_us = median_us(ts[warm:])

# ust_apply_state_delta_sparse: 1 % re-encoded, no membership change
cap = n // 4
out = (ustlib.pinned_array(cap + 1, np.int64), ustlib.pinned_array(cap + 1, np.uint8), ustlib.pinned_array(cap + 1, np.uint16))
ts = []
for i in range(warm + steps):
    idx = np.sort(rng.choice(n, size=n // 100, replace=False)).astype(np.int64)
    fr = fresh_nodes(idx.shape[0], 7 * n + i * n // 100)
    t = time.perf_counter()
    rc = h.apply_state_delta_sparse(pol, idx, fr, soa["ds_rev"], cap, out=out)[0]
    ts.append(time.perf_counter() - t)
    assert rc == 0, rc
    for k in COLS:
        soa[k][idx] = fr[k]
sparse_us = median_us(ts[warm:])
cur = {k: np.array(soa[k]) for k in COLS}
cur["ds_rev"] = soa["ds_rev"]


def splice_series(calls, grow):
    """`calls` splice calls (0.1 % out, 0.1 % + `grow` in, 1 % re-encoded); host-clock seconds per call"""
    global cur
    ts, last = [], None
    for i in range(calls):
        m = cur["state"].shape[0]
        rm, ib = splice_model.random_splice(rng, m, 0.001, 0.001)
        if grow:
            ib = np.sort(np.append(ib, rng.integers(0, m + 1))).astype(np.int64)
        ins = fresh_nodes(ib.shape[0], 20 * n + i * n)
        m_new = m - rm.shape[0] + ib.shape[0]
        idx = np.sort(rng.choice(m_new, size=m_new // 100, replace=False)).astype(np.int64)
        fr = fresh_nodes(idx.shape[0], 40 * n + i * n)
        sp = dict(remove_idx=rm, insert_before=ib, **ins)
        t = time.perf_counter()
        r = h.apply_state_delta_splice(pol, sp, idx, fr, cur["ds_rev"], cap, out=out)
        ts.append(time.perf_counter() - t)
        assert r[0] == 0, (r[0], h.last_error())
        new = {k: splice_model.splice(cur[k], rm, ib, ins[k]) for k in COLS}
        for k in COLS:
            new[k][idx] = fr[k]
        new["ds_rev"] = cur["ds_rev"]
        cur = new
        last = r
    return ts, last


ts, last = splice_series(warm + steps, False)
splice_us = median_us(ts[warm:])
# the last timed call against the oracle: its sparse entries and the full outputs it left resident
m = cur["state"].shape[0]
frc, fnxt, fact = h.fetch_outputs(m)
ref = helpers.oracle_apply(pol, cur, variant=1)
rc, n_out, oi, on, oa, cnt = last
ok = (frc == 0 and rc == ref[0] and cnt == ref[4] and np.array_equal(fnxt, ref[1]) and np.array_equal(fact, ref[2])
      and np.array_equal(on[:n_out], ref[1][oi[:n_out]]) and np.array_equal(oa[:n_out], ref[2][oi[:n_out]]))
assert ok, "splice outputs differ from the oracle"
last_n_out = n_out

ts, _ = splice_series(warm + max(steps // 3, 10), True)
resize_us = median_us(ts[warm:])

# the splice kernel's own time
from torch.profiler import ProfilerActivity, profile  # noqa: E402
prof_calls = 10
with profile(activities=[ProfilerActivity.CUDA]) as prof:
    splice_series(prof_calls, False)
    torch.cuda.synchronize()
kern = [e for e in prof.events() if "ust_splice_kernel" in e.name]
kernel_us = float(np.median([e.time_range.elapsed_us() for e in kern])) if kern else None  # device-side span of each launch

print(json.dumps({
    "gpu": gpu, "power_limit": power, "nodes": n, "steps": steps, "warmup": warm,
    "full_apply_state_us": round(full_us, 1), "delta_sparse_1pct_us": round(sparse_us, 1),
    "delta_splice_0.1pct_out_0.1pct_in_1pct_us": round(splice_us, 1),
    "delta_splice_size_change_every_call_us": round(resize_us, 1),
    "splice_kernel_us": None if kernel_us is None else round(kernel_us, 1), "splice_kernel_launches_profiled": len(kern),
    "last_call_n_out": int(last_n_out), "oracle_check": "ok",
}))
h.close()
