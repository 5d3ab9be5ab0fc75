"""ctypes view of include/ust.h. Constants are parsed out of the header so there is one source of truth."""
import ctypes as C
import os
import re

REPO_ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
HEADER = os.path.join(REPO_ROOT, "include", "ust.h")


def _parse_header(path):
    txt = open(path).read()
    txt = re.sub(r"/\*.*?\*/", "", txt, flags=re.S)
    consts = {}
    for m in re.finditer(r"#define\s+(UST_\w+)\s+(?:\(\s*)?(0x[0-9A-Fa-f]+|\d+)u?(?:\s*<<\s*(\d+)\s*\))?", txt):
        name, base, shift = m.group(1), m.group(2), m.group(3)
        v = int(base, 0)
        if shift:
            v <<= int(shift)
        consts[name] = v
    for m in re.finditer(r"(UST_\w+)\s*=\s*(-?\d+)", txt):
        consts[m.group(1)] = int(m.group(2))
    return consts


K = _parse_header(HEADER)
globals().update(K)

STATE_NAMES = [
    "", "upgrade-required", "cordon-required", "wait-for-jobs-required", "pod-deletion-required",
    "drain-required", "node-maintenance-required", "post-maintenance-required", "pod-restart-required",
    "validation-required", "uncordon-required", "upgrade-done", "upgrade-failed",
]  # reference: pkg/upgrade/consts.go:49-82
STATE_CODE = {n: i for i, n in enumerate(STATE_NAMES)}
ACTION_NAMES = {k[len("UST_A_"):]: v for k, v in K.items() if k.startswith("UST_A_")}
ERROR_NAMES = {v: k[len("UST_ERR_"):] for k, v in K.items() if k.startswith("UST_ERR_")}


class Policy(C.Structure):
    _fields_ = [
        ("auto_upgrade", C.c_int32),
        ("max_unavailable_kind", C.c_int32),
        ("max_parallel_upgrades", C.c_int64),
        ("max_unavailable_value", C.c_int64),
        ("pod_deletion_enabled", C.c_int32),
        ("validation_enabled", C.c_int32),
        ("pod_deletion_spec_present", C.c_int32),
        ("pod_deletion_force", C.c_int32),
        ("pod_deletion_delete_emptydir", C.c_int32),
        ("drain_enabled", C.c_int32),
        ("drain_force", C.c_int32),
        ("drain_delete_emptydir", C.c_int32),
        ("wait_selector_set", C.c_int32),
        ("wait_timeout_nonzero", C.c_int32),
        ("use_maintenance_operator", C.c_int32),
        ("evaluate_actuators", C.c_int32),
    ]


class Counters(C.Structure):
    _fields_ = [
        ("hist", C.c_int64 * 16),
        ("unavailable", C.c_int64),
        ("candidates", C.c_int64),
        ("total_managed", C.c_int64),
        ("in_progress", C.c_int64),
        ("max_unavailable", C.c_int64),
        ("upgrades_available", C.c_int64),
        ("error_code", C.c_int64),
        ("error_index", C.c_int64),
        ("error_pass", C.c_int64),
        ("reserved", C.c_int64 * 7),
    ]

    def as_dict(self):
        d = {"hist": list(self.hist)}
        for name, _ in self._fields_[1:-1]:
            d[name] = getattr(self, name)
        return d


class SimOptions(C.Structure):
    _fields_ = [("seconds_per_reconcile", C.c_int64), ("wait_timeout_seconds", C.c_int64), ("job_seconds", C.c_int64),
                ("validation_seconds", C.c_int64), ("validation_timeout_seconds", C.c_int64), ("maintenance_seconds", C.c_int64)]


class Pods(C.Structure):
    _fields_ = [("pod_off", C.c_void_p), ("pod_flags", C.c_void_p), ("n_pods", C.c_int64)]


class Splice(C.Structure):
    """ust_splice: nodes removed from / inserted into the resident snapshot (raw host addresses)."""
    _fields_ = [("n_remove", C.c_int64), ("remove_idx", C.c_void_p), ("n_insert", C.c_int64), ("insert_before", C.c_void_p),
                ("state", C.c_void_p), ("flags", C.c_void_p), ("pod_rev", C.c_void_p), ("ds_idx", C.c_void_p)]


class Reorder(C.Structure):
    """ust_reorder: a new node order of the resident snapshot as runs of old and inserted nodes (raw host addresses)."""
    _fields_ = [("n_runs", C.c_int64), ("run_src", C.c_void_p), ("run_len", C.c_void_p), ("n_insert", C.c_int64),
                ("state", C.c_void_p), ("flags", C.c_void_p), ("pod_rev", C.c_void_p), ("ds_idx", C.c_void_p)]


class DriverPodReorder(C.Structure):
    """ust_driver_pod_reorder: a new order of the resident driver-pod list as runs of old and joined pods (raw host addresses)."""
    _fields_ = [("n_runs", C.c_int64), ("run_src", C.c_void_p), ("run_len", C.c_void_p), ("n_insert", C.c_int64),
                ("state", C.c_void_p), ("owner_uid", C.c_void_p)]


class PodLists(C.Structure):
    """ust_pod_lists: replacement pod lists for some nodes of the resident pod-list snapshot (raw host addresses)."""
    _fields_ = [("n_lists", C.c_int64), ("node_idx", C.c_void_p), ("pod_off", C.c_void_p), ("pod_flags", C.c_void_p),
                ("n_pods", C.c_int64)]


NO_DEADLINE = -(1 << 63)  # ust_next_deadline: no time-only reconcile will return anything (INT64_MIN)


class Clock(C.Structure):
    """ust_clock: the time of a clocked pod-list call and the start times of the nodes it carries (raw host addresses)."""
    _fields_ = [("now", C.c_int64), ("wait_timeout_seconds", C.c_int64), ("start", C.c_void_p), ("insert_start", C.c_void_p)]


def make_policy(auto_upgrade=True, max_parallel_upgrades=0, max_unavailable=None, pod_deletion_enabled=False,
                validation_enabled=False, pod_deletion=None, drain=None, wait_for_completion=None,
                use_maintenance_operator=False, evaluate_actuators=False, evaluate_validation=False):
    """Flatten a DriverUpgradePolicySpec-like description (api/upgrade/v1alpha1/upgrade_spec.go:27-110).

    max_unavailable: None | int | "NN%" | any other string (=> intstr parse error).
    pod_deletion / drain / wait_for_completion: None or dicts with the spec's json field names.
    evaluate_validation: also answer Validate from the pod lists (UST_EVAL_VALIDATION; needs evaluate_actuators and pods).
    """
    p = Policy()
    p.auto_upgrade = int(bool(auto_upgrade))
    p.max_parallel_upgrades = int(max_parallel_upgrades)
    if max_unavailable is None:
        p.max_unavailable_kind = K["UST_MAXUNAVAIL_NIL"]
    elif isinstance(max_unavailable, int):
        p.max_unavailable_kind = K["UST_MAXUNAVAIL_INT"]
        p.max_unavailable_value = max_unavailable
    else:
        m = re.fullmatch(r"([+-]?\d+)%", max_unavailable)
        if m:
            p.max_unavailable_kind = K["UST_MAXUNAVAIL_PERCENT"]
            p.max_unavailable_value = int(m.group(1))
        else:
            p.max_unavailable_kind = K["UST_MAXUNAVAIL_INVALID"]
    p.pod_deletion_enabled = int(bool(pod_deletion_enabled))
    p.validation_enabled = int(bool(validation_enabled))
    if pod_deletion is not None:
        p.pod_deletion_spec_present = 1
        p.pod_deletion_force = int(bool(pod_deletion.get("force", False)))
        p.pod_deletion_delete_emptydir = int(bool(pod_deletion.get("deleteEmptyDir", False)))
    if drain is not None:
        p.drain_enabled = int(bool(drain.get("enable", False)))
        p.drain_force = int(bool(drain.get("force", False)))
        p.drain_delete_emptydir = int(bool(drain.get("deleteEmptyDir", False)))
    if wait_for_completion is not None:
        p.wait_selector_set = int(bool(wait_for_completion.get("podSelector", "")))
        p.wait_timeout_nonzero = int(wait_for_completion.get("timeoutSeconds", 0) != 0)
    p.use_maintenance_operator = int(bool(use_maintenance_operator))
    p.evaluate_actuators = int(bool(evaluate_actuators)) | (K["UST_EVAL_VALIDATION"] if evaluate_validation else 0)
    return p
