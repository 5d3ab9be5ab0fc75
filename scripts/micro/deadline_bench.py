"""What the next-deadline evaluation costs the clocked calls, at C4 size: the same three calls timed with two builds of
libust.so, the one under test and one without the deadline: BASE_TREE, a built checkout of the parent commit, whose own
ust package and libust.so the "before" runs import.

A 10 M-node C4 snapshot (~300 M workload pods) in pinned host memory under C4's policy plus a wait-for-completion selector
with a 300 s timeout; 80 % of the wait-for-jobs-required nodes carry a wait-start annotation, and every node a start time in
the last 700 s (clock_bench.py's snapshot). Series, each the median and spread (min, max) of the host-clock time of the
synchronous call, `now` advancing 10 s per call:
  time_only     ust_apply_state_delta_pods_clocked with no node, no list, no reorder;
  delta_1pct    the same with 1 % of the nodes re-sent (new starts);
  full          ust_apply_state_clocked on the whole snapshot.
Each build runs in its own process, RUNS times in alternation; the result line holds every run's medians, so that
the spread between runs can be told from a difference between the builds. The build under test also reports the value of
ust_next_deadline after its last call.
  BASE_TREE=build/parent_tree NODES=10000000 STEPS=15 WARMUP=3 RUNS=3 python scripts/micro/deadline_bench.py"""
import json
import os
import subprocess
import sys
import time

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.join(HERE, "..", "..")


def child():
    sys.path.insert(0, os.path.join(os.environ.get("UST_TREE", ROOT), "k8s-operator-libs_b200"))
    import numpy as np
    from ust import abi, lib as ustlib, synth

    COLS = ("state", "flags", "pod_rev", "ds_idx")
    n = int(os.environ.get("NODES", "10000000"))
    steps = int(os.environ.get("STEPS", "15"))
    warm = int(os.environ.get("WARMUP", "3"))
    NOW, TIMEOUT = 1_700_000_000, 300
    cfg = synth.CONFIGS["C4"]
    pol = abi.make_policy(auto_upgrade=True, **dict(cfg["policy"], wait_for_completion={"podSelector": "app=batch", "timeoutSeconds": TIMEOUT}))

    def pinned_copy(a):
        p = ustlib.pinned_array(a.shape[0], a.dtype)
        p[:] = a
        return p

    rng = np.random.default_rng(2029)
    src = synth.make_nodes(n, cfg["seed"])
    w = (src["state"] & 15) == abi.UST_STATE_WAIT_FOR_JOBS_REQUIRED
    src["flags"] = (src["flags"] | np.where(w & (rng.random(n) < 0.8), np.uint32(abi.UST_F_WAIT_START_ANNO), np.uint32(0))).astype(np.uint32)
    soa = {c: pinned_copy(src[c]) for c in COLS}
    soa["ds_rev"] = src["ds_rev"]
    pods_src = synth.make_pods_blocked(n, cfg["seed"])
    pods = {"pod_off": pinned_copy(pods_src["pod_off"]), "pod_flags": pinned_copy(pods_src["pod_flags"])}
    start = pinned_copy((NOW - rng.integers(0, 700, n)).astype(np.int64))
    out = tuple(pinned_copy(np.zeros(n, dt)) for dt in (np.uint8, np.uint16, np.uint8))
    sparse = [pinned_copy(np.zeros(n + 1, dt)) for dt in (np.int64, np.uint8, np.uint16, np.uint8)]
    h = ustlib.Handle(0)
    m = n // 100
    empty = np.zeros(0, np.int64), {c: np.zeros(0, src[c].dtype) for c in COLS}, np.zeros(0, np.int64)
    now = NOW
    series = {}

    def timed(fn):
        ts = []
        for k in range(warm + steps):
            t0 = time.perf_counter()
            rc = fn(k)
            dt = time.perf_counter() - t0
            assert rc in (0,), (rc, h.last_error())
            if k >= warm:
                ts.append(dt)
        return round(float(np.median(ts)) * 1e3, 3), round(float(np.min(ts)) * 1e3, 3), round(float(np.max(ts)) * 1e3, 3)

    def full(k):
        return h.apply_state_clocked(pol, NOW + 10 * k, TIMEOUT, start, soa, pods, out=out)[0]

    series["full"] = timed(full)
    assert full(0) == 0

    def time_only(k):
        nonlocal now
        now += 10
        return h.apply_state_delta_pods_clocked(pol, now, TIMEOUT, None, None, *empty[:2], empty[2], soa["ds_rev"], n, out=sparse)[0]

    series["time_only"] = timed(time_only)

    def delta(k):
        nonlocal now
        now += 10
        idx = np.sort(rng.choice(n, m, replace=False)).astype(np.int64)
        ch = {c: src[c][idx] for c in COLS}
        st = (now - rng.integers(0, 700, m)).astype(np.int64)
        return h.apply_state_delta_pods_clocked(pol, now, TIMEOUT, None, None, idx, ch, st, soa["ds_rev"], n, out=sparse)[0]

    series["delta_1pct"] = timed(delta)
    res = {"tree": os.environ.get("UST_TREE", "repo"), "series_ms": series}
    if "UST_TREE" not in os.environ:
        res["next_deadline"] = h.next_deadline()
        res["now"] = now
    h.close()
    print("RESULT " + json.dumps(res))


def main():
    runs = int(os.environ.get("RUNS", "3"))
    base = os.environ.get("BASE_TREE", os.path.join(ROOT, "build", "parent_tree"))
    import torch
    gpu = torch.cuda.get_device_name(0)
    try:
        smi = subprocess.check_output(["nvidia-smi", "-i", "0", "--query-gpu=power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                                      text=True).strip()
    except (OSError, subprocess.CalledProcessError) as e:
        smi = f"unknown ({e})"
    results = {"gpu": gpu, "power_limit,sm_clock,max_sm_clock": smi, "runs": {"after": [], "before": []}}
    for r in range(runs):
        for tag, lib in (("after", None), ("before", base)):
            env = dict(os.environ)
            env.pop("UST_TREE", None)
            if lib:
                env["UST_TREE"] = os.path.abspath(lib)
            p = subprocess.run([sys.executable, os.path.abspath(__file__), "--child"], env=env, capture_output=True, text=True)
            line = [x for x in p.stdout.splitlines() if x.startswith("RESULT ")]
            assert p.returncode == 0 and line, p.stdout + p.stderr
            results["runs"][tag].append(json.loads(line[0][7:]))
    print(json.dumps(results))


if __name__ == "__main__":
    child() if "--child" in sys.argv else main()
