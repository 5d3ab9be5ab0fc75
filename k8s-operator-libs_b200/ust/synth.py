"""Deterministic synthetic ClusterUpgradeState snapshots in the SoA encoding of include/ust.h.

Generator: counter-based splitmix64 (r0 = splitmix64(seed ^ i), r_{k+1} = splitmix64(r_k)), 16-bit fields
of the words drive one categorical / Bernoulli draw each. Distributions: SURVEY.md §8(d) / BASELINE.md §3.
"""
import numpy as np

from . import abi

_M = np.uint64(0xFFFFFFFFFFFFFFFF)


def splitmix64(x):
    x = (x + np.uint64(0x9E3779B97F4A7C15)) & _M
    z = x
    z = ((z ^ (z >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)) & _M
    z = ((z ^ (z >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)) & _M
    return z ^ (z >> np.uint64(31))


def _fields(seed, idx, nwords):
    """nwords*4 independent uint16 fields per index."""
    with np.errstate(over="ignore"):
        r = splitmix64(np.uint64(seed) ^ idx.astype(np.uint64))
        out = []
        for _ in range(nwords):
            for s in (0, 16, 32, 48):
                out.append(((r >> np.uint64(s)) & np.uint64(0xFFFF)).astype(np.uint32))
            r = splitmix64(r)
    return out


def _bern(field, pct):
    return field < np.uint32(round(pct * 655.36))


# state mix in percent: SURVEY.md §8(d)
STATE_MIX = [(0, 5), (1, 35), (2, 5), (3, 5), (4, 5), (5, 5), (8, 10), (9, 2), (10, 5), (11, 20), (12, 3)]
DS_REV = np.array([1001, 1002, 1003, 1004], dtype=np.int32)


def make_nodes(n, seed, start=0, requestor_pct=0.0, error_pct=0.0):
    """SoA arrays for global node indices [start, start+n). Returns dict of numpy arrays."""
    idx = np.arange(start, start + n, dtype=np.uint64)
    f = _fields(seed, idx, 5)
    # categorical state from f[0]
    edges = np.cumsum([p for _, p in STATE_MIX]) * 655.36
    which = np.searchsorted(edges, f[0].astype(np.float64), side="right")
    which = np.minimum(which, len(STATE_MIX) - 1)
    codes = np.array([c for c, _ in STATE_MIX], dtype=np.uint8)[which]
    unsched = _bern(f[1], 10)
    notready = _bern(f[2], 2)
    upgreq = _bern(f[3], 1)
    skip = _bern(f[4], 1)
    safeload = _bern(f[5], 1)
    initial = _bern(f[6], 5)
    requestor = _bern(f[7], requestor_pct)
    orphan = _bern(f[8], 1)
    running = _bern(f[9], 95)
    hasctr = _bern(f[10], 98)
    allready = _bern(f[11], 90)
    failing = _bern(f[12], 1)
    terminating = _bern(f[13], 2)
    ds_idx = (f[14] & np.uint32(3)).astype(np.int32)
    insync = _bern(f[15], 50)
    validation_done = _bern(f[16], 50)
    hasherr = _bern(f[17], error_pct) & ~orphan

    hot = codes.copy()
    hot |= np.where(notready, abi.UST_HOT_NOT_READY, 0).astype(np.uint8)
    hot |= np.where(skip, abi.UST_HOT_SKIP, 0).astype(np.uint8)
    hot |= np.where(unsched, abi.UST_HOT_UNSCHEDULABLE, 0).astype(np.uint8)
    hot |= np.where(hasherr, abi.UST_HOT_REVISION_HASH_ERROR, 0).astype(np.uint8)

    flags = np.zeros(n, dtype=np.uint32)
    for cond, bit in (
        (upgreq, abi.UST_F_UPGRADE_REQUESTED), (validation_done, abi.UST_F_VALIDATION_DONE),
        (safeload, abi.UST_F_SAFE_LOAD), (orphan, abi.UST_F_POD_ORPHANED),
        (running & hasctr & allready, abi.UST_F_POD_READY), (initial, abi.UST_F_INITIAL_STATE_ANNO),
        (requestor, abi.UST_F_REQUESTOR_MODE), (terminating, abi.UST_F_POD_TERMINATING),
        (failing, abi.UST_F_POD_FAILING),
    ):
        flags |= np.where(cond, np.uint32(bit), np.uint32(0))
    ds_idx = np.where(orphan, np.int32(-1), ds_idx).astype(np.int32)
    cur = DS_REV[np.maximum(ds_idx, 0)]
    stale = (cur - np.int32(1) - (f[18] & np.uint32(7)).astype(np.int32)).astype(np.int32)
    pod_rev = np.where(insync, cur, stale).astype(np.int32)
    return {"state": hot, "flags": flags, "pod_rev": pod_rev, "ds_idx": ds_idx, "ds_rev": DS_REV.copy()}


def make_pods(n, seed, start=0, lo=20, hi=40):
    """CSR workload pod lists for nodes [start, start+n): pods/node uniform in [lo, hi]."""
    idx = np.arange(start, start + n, dtype=np.uint64)
    with np.errstate(over="ignore"):
        r = splitmix64(np.uint64(seed ^ 0xC0FFEE) ^ idx)
    cnt = (lo + (r % np.uint64(hi - lo + 1))).astype(np.int64)
    off = np.zeros(n + 1, dtype=np.int64)
    np.cumsum(cnt, out=off[1:])
    total = int(off[-1])
    # global pod id = (node index << 6) + slot, so shards generate identical pods
    node_of = np.repeat(idx, cnt)
    slot = np.arange(total, dtype=np.uint64) - np.repeat(off[:-1].astype(np.uint64), cnt)
    pid = (node_of << np.uint64(6)) + slot
    f = _fields(seed ^ 0xBADC0DE, pid, 2)
    ph = f[0].astype(np.float64) / 655.36
    phase = np.where(ph < 85, abi.UST_PHASE_RUNNING,
                     np.where(ph < 90, abi.UST_PHASE_PENDING,
                              np.where(ph < 97, abi.UST_PHASE_SUCCEEDED, abi.UST_PHASE_FAILED))).astype(np.uint16)
    ctrl = f[1].astype(np.float64) / 655.36
    by_ds = ctrl < 15
    has_ctrl = ctrl < 80
    pf = phase.copy()
    for cond, bit in (
        (has_ctrl, abi.UST_POD_HAS_CONTROLLER), (by_ds, abi.UST_POD_CONTROLLED_BY_DS),
        (_bern(f[2], 0.5) & by_ds, abi.UST_POD_DS_MISSING), (_bern(f[3], 2), abi.UST_POD_MIRROR),
        (_bern(f[4], 20), abi.UST_POD_HAS_EMPTYDIR), (_bern(f[5], 25), abi.UST_POD_MATCH_DELETION_FILTER),
        (_bern(f[6], 30), abi.UST_POD_MATCH_WAIT_SELECTOR), (_bern(f[7], 90), abi.UST_POD_MATCH_DRAIN_SELECTOR),
    ):
        pf |= np.where(cond, np.uint16(bit), np.uint16(0))
    return {"pod_off": off.astype(np.int32), "pod_flags": pf.astype(np.uint16)}


def make_pods_blocked(n, seed, start=0, block=500_000):
    """make_pods() for large n in bounded memory (pods are a pure function of the node index, so blocks agree
    with the one-shot generator bit for bit)."""
    offs = [np.zeros(1, dtype=np.int64)]
    flags = []
    base = 0
    for b0 in range(0, n, block):
        part = make_pods(min(block, n - b0), seed, start=start + b0)
        offs.append(part["pod_off"][1:].astype(np.int64) + base)
        base += int(part["pod_off"][-1])
        flags.append(part["pod_flags"])
    off = np.concatenate(offs)
    assert off[-1] < 2 ** 31, "pod_off is int32"
    return {"pod_off": off.astype(np.int32), "pod_flags": np.concatenate(flags) if flags else np.zeros(0, np.uint16)}


def make_validation_pods(soa, pods, seed, start=0, invalid_pct=0.0):
    """Validation pods for the validation-required nodes of a snapshot (UST_EVAL_VALIDATION): each such node gets 0-3 pods
    matching the validation selector ahead of its workload pods (only their order among themselves matters), each ready
    with 80 % probability, and the validation start-time bits (annotation present 50 %, timed out 20 % of those,
    unparsable `invalid_pct` % of those). Returns (flags, pods) for the same nodes; other nodes keep flags and lists."""
    n = int(soa["state"].shape[0])
    idx = np.arange(start, start + n, dtype=np.uint64)
    f = _fields(seed ^ 0x7A11D, idx, 1)
    val = (soa["state"] & np.uint8(15)) == abi.UST_STATE_VALIDATION_REQUIRED
    anno = val & _bern(f[0], 50)
    flags = soa["flags"] | np.where(anno, np.uint32(abi.UST_F_VALIDATION_START_ANNO), np.uint32(0))
    flags |= np.where(anno & _bern(f[1], 20), np.uint32(abi.UST_F_VALIDATION_TIMED_OUT), np.uint32(0))
    flags |= np.where(anno & _bern(f[2], invalid_pct), np.uint32(abi.UST_F_VALIDATION_START_INVALID), np.uint32(0))
    k = np.where(val, (f[3] & np.uint32(3)).astype(np.int64), 0)
    old_off = pods["pod_off"].astype(np.int64)
    cnt = np.diff(old_off) + k
    off = np.zeros(n + 1, dtype=np.int64)
    np.cumsum(cnt, out=off[1:])
    total = int(off[-1])
    node_of = np.repeat(np.arange(n), cnt)
    slot = np.arange(total, dtype=np.int64) - off[:-1][node_of]
    is_val = slot < k[node_of]
    pf = np.zeros(total, dtype=np.uint16)
    pf[~is_val] = pods["pod_flags"][(old_off[:-1][node_of] + slot - k[node_of])[~is_val]]
    # a validation pod is a pure function of (node index, slot), like make_pods' pods
    g = _fields(seed ^ 0xA11D8, (idx[node_of] << np.uint64(2)) + slot.astype(np.uint64), 1)
    vf = np.where(_bern(g[0], 80), abi.UST_PHASE_RUNNING | abi.UST_POD_READY, abi.UST_PHASE_PENDING).astype(np.uint16)
    pf[is_val] = (vf | np.uint16(abi.UST_POD_MATCH_VALIDATION_SELECTOR))[is_val]
    return flags.astype(np.uint32), {"pod_off": off.astype(np.int32), "pod_flags": pf}


# BASELINE.json configs as concrete inputs (BASELINE.md §3)
CONFIGS = {
    "C1": dict(n=100, seed=0x5EED0001, policy=dict(max_parallel_upgrades=1)),
    "C2": dict(n=1_000_000, seed=0x5EED0002, policy=dict(max_parallel_upgrades=0)),
    "C3": dict(n=10_000_000, seed=0x5EED0003, policy=dict(max_parallel_upgrades=100, max_unavailable="25%")),
    "C4": dict(n=10_000_000, seed=0x5EED0004, pods=True,
               policy=dict(max_parallel_upgrades=100, max_unavailable="25%", pod_deletion_enabled=True,
                           pod_deletion={"force": False, "deleteEmptyDir": False},
                           drain={"enable": True, "force": False, "deleteEmptyDir": False},
                           evaluate_actuators=True)),
    "C5": dict(n=80_000_000, seed=0x5EED0005, policy=dict(max_parallel_upgrades=100, max_unavailable="25%")),
}


def config_policy(name):
    return abi.make_policy(auto_upgrade=True, **CONFIGS[name]["policy"])
