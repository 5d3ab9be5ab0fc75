"""ApplyState with UST_EVAL_VALIDATION (include/ust.h): the CPU oracle (oracle/ust_oracle.cpp) for every pass, with
ProcessValidationRequiredNodes (common_manager.go:573-604) and ValidationManagerImpl.Validate (validation_manager.go:71-175)
restated here for the validation-required nodes. Two independent restatements of that pass:

  variant 0  reference-shaped: per node a corev1.Node-like annotation map and the validation pods as objects (phase,
             container statuses) in list order; Validate and handleTimeout run against a recording provider mock that
             applies its changes to the node (the suite's mocked-provider semantics), and the calls it recorded become
             the node's actions;
  variant 1  over the encoded bits: the outcome read off UST_POD_MATCH_VALIDATION_SELECTOR / UST_POD_READY and the
             UST_F_VALIDATION_* bits.

Every other pass is the oracle's, run with UST_EVAL_VALIDATION cleared: none of them reads the validation bits.
"""
import numpy as np

import helpers
from helpers import abi

TIMEOUT = 600                      # validationTimeoutSeconds, validation_manager.go:32
NOW = 1_760_000_000                # the model's clock (time.Now().Unix())
START_KEY = "nvidia.com/gpu-driver-upgrade-validation-start-time"   # consts.go:40
INITIAL_KEY = "nvidia.com/gpu-driver-upgrade.node-initial-state.unschedulable"   # consts.go:33
REQUESTOR_KEY = "nvidia.com/gpu-driver-upgrade-requestor-mode"        # consts.go:47

A = abi.ACTION_NAMES
S_VALIDATION, S_UNCORDON, S_DONE, S_FAILED = 9, 10, 11, 12


# ---- variant 0: objects ------------------------------------------------------------------------------------------
class Provider:
    """NodeUpgradeStateProvider mock: records the calls and applies them to the node (upgrade_suit_test.go:114-182)."""

    def __init__(self, node):
        self.node, self.calls = node, []

    def change_annotation(self, key, value):
        self.calls.append(("anno", key, value))
        if value == "null":
            self.node["annotations"].pop(key, None)
        else:
            self.node["annotations"][key] = value

    def change_state(self, state):
        self.calls.append(("state", state))
        self.node["state"] = state


def is_pod_ready(pod):  # validation_manager.go:118-136
    if pod["phase"] != "Running":
        return False
    if len(pod["containerStatuses"]) == 0:
        return False
    return all(c["ready"] for c in pod["containerStatuses"])


def parse_int64(s):  # strconv.ParseInt(s, 10, 64)
    import re
    if not re.fullmatch(r"[+-]?[0-9]+", s):
        raise ValueError(s)
    v = int(s)
    if not -(1 << 63) <= v < (1 << 63):
        raise ValueError(s)
    return v


def handle_timeout(node, provider, timeout_seconds):  # validation_manager.go:139-175
    if START_KEY not in node["annotations"]:
        provider.change_annotation(START_KEY, str(NOW))
        return None
    try:
        start = parse_int64(node["annotations"][START_KEY])
    except ValueError:
        return "unable to parse"
    if NOW > start + timeout_seconds:
        provider.change_state("upgrade-failed")
        provider.change_annotation(START_KEY, "null")
    return None


def validate(node, pods, selector, provider):
    """(done, error) of Validate (validation_manager.go:71-116). `pods`: the node's pods in list order with a
    "labels_match" bit standing for the label selector of the List call."""
    if selector == "":
        return True, None
    listed = [p for p in pods if p["labels_match"]]
    if len(listed) == 0:
        return False, None
    done = True
    for pod in listed:
        if not is_pod_ready(pod):
            err = handle_timeout(node, provider, TIMEOUT)
            if err is not None:
                return False, err
            done = False
            break
        provider.change_annotation(START_KEY, "null")
    return done, None


def update_to_uncordon_or_done(node, provider):  # common_manager.go:673-708
    requestor = REQUESTOR_KEY in node["annotations"]
    new = "uncordon-required"
    if INITIAL_KEY in node["annotations"] and not requestor:
        new = "upgrade-done"
    provider.change_state(new)
    if new == "upgrade-done" or requestor:
        provider.change_annotation(INITIAL_KEY, "null")


def node_object(i, fl):
    """The node's annotations as the encoder saw them; where several values encode the same bits, the index picks."""
    ann = {}
    if fl & abi.UST_F_INITIAL_STATE_ANNO:
        ann[INITIAL_KEY] = "true"
    if fl & abi.UST_F_REQUESTOR_MODE:
        ann[REQUESTOR_KEY] = "true"
    if fl & abi.UST_F_SAFE_LOAD:
        ann["nvidia.com/gpu-driver-upgrade.driver-wait-for-safe-load"] = "true"
    if fl & abi.UST_F_VALIDATION_START_ANNO:
        if fl & abi.UST_F_VALIDATION_START_INVALID:
            ann[START_KEY] = ("", "null", "12a", "1.5e9")[i % 4]
        elif fl & abi.UST_F_VALIDATION_TIMED_OUT:
            ann[START_KEY] = str(NOW - TIMEOUT - 1 - i % 7)
        else:
            ann[START_KEY] = str(NOW - TIMEOUT + i % 601)
    return {"state": "validation-required", "annotations": ann}


def pod_objects(i, flags):
    out = []
    for k, pf in enumerate(flags):
        pf = int(pf)
        if pf & abi.UST_POD_READY:
            pod = {"phase": "Running", "containerStatuses": [{"ready": True}] * (1 + (i + k) % 3)}
        else:
            shape = (i + k) % 3
            if shape == 0:
                pod = {"phase": ("Pending", "Succeeded", "Failed", "Unknown")[(i + k) % 4], "containerStatuses": [{"ready": True}]}
            elif shape == 1:
                pod = {"phase": "Running", "containerStatuses": []}
            else:
                pod = {"phase": "Running", "containerStatuses": [{"ready": True}, {"ready": False}]}
        pod["labels_match"] = bool(pf & abi.UST_POD_MATCH_VALIDATION_SELECTOR)
        out.append(pod)
    return out


def pass_objects(i, fl, pod_flags, policy):
    """ProcessValidationRequiredNodes for one node (common_manager.go:577-603): (next_state, actions, error)."""
    node = node_object(i, fl)
    prov = Provider(node)
    actions = 0
    if fl & abi.UST_F_SAFE_LOAD:  # UnblockLoading: the annotation is present (safe_driver_load_manager.go:57-71)
        actions |= A["UNBLOCK_SAFE_LOAD"]
    done, err = validate(node, pod_objects(i, pod_flags), "app=validator" if policy.validation_enabled else "", prov)
    if err is None and done:
        update_to_uncordon_or_done(node, prov)
    nxt = S_VALIDATION
    for c in prov.calls:
        if c[0] == "state":
            nxt = abi.STATE_CODE[c[1]]
        elif c[1] == START_KEY:
            actions |= A["CLEAR_WAIT_START"] if c[2] == "null" else A["SET_WAIT_START"]
        elif c[1] == INITIAL_KEY:
            actions |= A["CLEAR_INITIAL_STATE_ANNO"]
    if nxt != S_VALIDATION:
        actions |= A["SET_STATE"]
    return nxt, actions, err is not None


# ---- variant 1: bits ---------------------------------------------------------------------------------------------
def pass_bits(i, fl, pod_flags, policy):
    actions = A["UNBLOCK_SAFE_LOAD"] if fl & abi.UST_F_SAFE_LOAD else 0
    if policy.validation_enabled:
        m = [int(p) for p in pod_flags if int(p) & abi.UST_POD_MATCH_VALIDATION_SELECTOR]
        first_bad = next((k for k, p in enumerate(m) if not p & abi.UST_POD_READY), None)
        if not m:
            return S_VALIDATION, actions, False
        if first_bad is not None:
            if first_bad > 0:  # the ready ones before it deleted the annotation: handleTimeout sets it anew
                return S_VALIDATION, actions | A["CLEAR_WAIT_START"] | A["SET_WAIT_START"], False
            if not fl & abi.UST_F_VALIDATION_START_ANNO:
                return S_VALIDATION, actions | A["SET_WAIT_START"], False
            if fl & abi.UST_F_VALIDATION_START_INVALID:
                return S_VALIDATION, actions, True
            if fl & abi.UST_F_VALIDATION_TIMED_OUT:
                return S_FAILED, actions | A["CLEAR_WAIT_START"] | A["SET_STATE"], False
            return S_VALIDATION, actions, False
        actions |= A["CLEAR_WAIT_START"]
    requestor = bool(fl & abi.UST_F_REQUESTOR_MODE)
    nxt = S_DONE if (fl & abi.UST_F_INITIAL_STATE_ANNO) and not requestor else S_UNCORDON
    if nxt == S_DONE or requestor:
        actions |= A["CLEAR_INITIAL_STATE_ANNO"]
    return nxt, actions | A["SET_STATE"], False


# ---- ApplyState --------------------------------------------------------------------------------------------------
def apply(policy, soa, pods, variant=0):
    """(rc, next_state, actions, outcome, counters) of ApplyState with `policy` (UST_EVAL_VALIDATION set)."""
    import copy
    base = copy.copy(policy)
    base.evaluate_actuators = int(policy.evaluate_actuators) & ~abi.UST_EVAL_VALIDATION
    rc, nxt, act, oc, cnt = helpers.oracle_apply(base, soa, pods, variant=variant)
    if rc != 0 or not policy.auto_upgrade:
        return rc, nxt, act, oc, cnt  # an earlier pass aborted (passes <= 9), or nothing is processed
    code = soa["state"] & 15
    off, pf = pods["pod_off"], pods["pod_flags"]
    step = pass_objects if variant == 0 else pass_bits
    for i in np.nonzero(code == S_VALIDATION)[0].tolist():  # the bucket in snapshot order
        n_i, a_i, err = step(i, int(soa["flags"][i]), pf[off[i]:off[i + 1]], policy)
        if err:  # ApplyState returns the error here: later nodes of the pass and every later pass stay untouched
            later = (code == S_UNCORDON) | ((code == S_VALIDATION) & (np.arange(code.size) > i))
            nxt = np.where(later, code, nxt).astype(np.uint8)
            act = np.where(later, 0, act).astype(np.uint16)
            oc = np.where(later, 0xFF, oc).astype(np.uint8)
            nxt[i], act[i], oc[i] = S_VALIDATION, (a_i & A["UNBLOCK_SAFE_LOAD"]) | A["ERROR"], 0xFF
            cnt = dict(cnt, error_code=abi.UST_ERR_VALIDATION, error_index=i, error_pass=10)
            return abi.UST_ERR_VALIDATION, nxt, act, oc, cnt
        nxt[i], act[i], oc[i] = n_i, a_i, 0xFF
    return rc, nxt, act, oc, cnt


def node_pass(policy, fl, pod_flags, variant=0, i=0):
    """One validation-required node through pass 10 alone: (next_state, actions, aborts)."""
    return (pass_objects if variant == 0 else pass_bits)(i, int(fl), np.asarray(pod_flags, np.uint16), policy)
