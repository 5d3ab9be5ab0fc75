"""UST_EVAL_VALIDATION without a device: the two restatements of validation_model against the known answers of
tests/golden/validation_vectors.json and against each other, the product's state-9 table in validation mode against
validation_model for every key of its window, and the new ust.h constants against ust/abi.py."""
import ctypes as C
import json
import os
import re

import numpy as np
import pytest

import helpers
import validation_model as vm
from helpers import abi
from ust import lib as ustlib

VECTORS = os.path.join(helpers.ROOT, "tests", "golden", "validation_vectors.json")
A = abi.ACTION_NAMES


def load_vectors():
    with open(VECTORS) as f:
        return json.load(f)["vectors"]


def encode(v):
    """(policy, soa, pods) of a vector. Nodes are synced, ready and not cordoned: only the validation inputs vary."""
    nodes = v["nodes"]
    n = len(nodes)
    state = np.array([abi.STATE_CODE[x["state"]] for x in nodes], np.uint8)
    flags = np.array([sum(abi.K["UST_F_" + b] for b in x["flags"]) | abi.UST_F_POD_READY for x in nodes], np.uint32)
    pf, off = [], [0]
    for x in nodes:
        for p in x["pods"]:
            pf.append(sum(abi.K["UST_PHASE_" + b] if "UST_PHASE_" + b in abi.K else abi.K["UST_POD_" + b] for b in p))
        off.append(len(pf))
    soa = {"state": state, "flags": flags, "pod_rev": np.full(n, 7, np.int32), "ds_idx": np.zeros(n, np.int32),
           "ds_rev": np.array([7], np.int32)}
    pods = {"pod_off": np.array(off, np.int32), "pod_flags": np.array(pf, np.uint16)}
    pol = abi.make_policy(validation_enabled=v["policy"]["validation_enabled"],
                          use_maintenance_operator=v["policy"]["use_maintenance_operator"], evaluate_actuators=True,
                          evaluate_validation=True)
    return pol, soa, pods


def check_vector(v, res):
    rc, nxt, act, oc, cnt = res
    e = v["expect"]
    assert rc == (0 if e["rc"] == "OK" else abi.K["UST_ERR_" + e["rc"]]), (v["name"], rc)
    assert cnt["error_index"] == e["error_index"], (v["name"], cnt["error_index"])
    assert [abi.STATE_NAMES[c] for c in nxt] == e["next_state"], (v["name"], nxt)
    assert act.tolist() == [sum(A[a] for a in names) for names in e["actions"]], (v["name"], act)
    assert (oc == 0xFF).all(), v["name"]  # Validate is synchronous: no actuator outcome
    if e["rc"] == "VALIDATION":
        assert cnt["error_pass"] == 10


@pytest.mark.parametrize("variant", [0, 1])
def test_golden_vectors(variant):
    vs = load_vectors()
    assert len(vs) >= 15 and all(re.search(r"\.go:\d+", v["source"]) for v in vs)
    for v in vs:
        pol, soa, pods = encode(v)
        check_vector(v, vm.apply(pol, soa, pods, variant=variant))


@pytest.mark.parametrize("seed", range(6))
def test_variants_agree(seed):
    rng = np.random.default_rng(seed)
    soa, pods = helpers.random_soa(rng, 3000, with_pods=True)
    soa["state"] = np.where(rng.random(3000) < 0.4, (soa["state"] & 0xF0) | 9, soa["state"]).astype(np.uint8)
    soa["state"] &= np.uint8(0x7F)  # no revision-hash aborts: pass 10 must be reached
    pol = helpers.random_policy(rng)
    pol.evaluate_actuators = 3
    if pol.max_unavailable_kind == abi.UST_MAXUNAVAIL_INVALID:
        pol.max_unavailable_kind = abi.UST_MAXUNAVAIL_NIL
    helpers.assert_same(vm.apply(pol, soa, pods, variant=0), vm.apply(pol, soa, pods, variant=1), f"seed {seed}")


# pods and flags that make the pod-summary kernel write outcome o (ust_lut.h UST_VAL_*); None: not reachable
R = abi.UST_POD_MATCH_VALIDATION_SELECTOR | abi.UST_POD_READY | abi.UST_PHASE_RUNNING
NR = abi.UST_POD_MATCH_VALIDATION_SELECTOR | abi.UST_PHASE_RUNNING
ANNO, INV, TO = abi.UST_F_VALIDATION_START_ANNO, abi.UST_F_VALIDATION_START_INVALID, abi.UST_F_VALIDATION_TIMED_OUT
OUTCOMES = {0: (ANNO, [NR]), 1: (0, [NR]), 2: (0, [R, NR]), 3: (ANNO, [R]), 4: (ANNO | TO, [NR]), 5: (ANNO | INV, [NR])}


@pytest.mark.parametrize("validation_enabled", [0, 1])
@pytest.mark.parametrize("requestor", [0, 1])
def test_validation_table_matches_model(validation_enabled, requestor):
    """Every key of state 9's validation-mode window: the entry == validation_model's pass for a node built to produce
    that summary byte (bits 1-3 outcome, 5-7 SAFE_LOAD / INITIAL_STATE_ANNO / REQUESTOR_MODE)."""
    lib = ustlib.load()
    pol = abi.make_policy(validation_enabled=bool(validation_enabled), use_maintenance_operator=bool(requestor),
                          evaluate_actuators=True, evaluate_validation=True)
    width = C.c_int(0)
    sh = lib.ust_table_window(C.byref(pol), 9, C.byref(width))
    assert (sh, width.value) == (22, 7)
    checked = 0
    for key in range(1 << width.value):
        byte = key << 1
        o = (byte >> 1) & 7
        if byte & 0x10 or o not in OUTCOMES:
            continue  # bit 4 of the byte is never set for state 9; outcomes 6, 7 are never written
        fl, pf = OUTCOMES[o]
        fl |= (abi.UST_F_SAFE_LOAD if byte & 0x20 else 0) | (abi.UST_F_INITIAL_STATE_ANNO if byte & 0x40 else 0) | \
            (abi.UST_F_REQUESTOR_MODE if byte & 0x80 else 0)
        e = lib.ust_table_entry(C.byref(pol), 9, key << sh)
        for variant in (0, 1):
            nxt, act, err = vm.node_pass(pol, fl, pf, variant=variant)
            if err:  # the table entry is what the aborting node keeps; the abort adds UST_A_ERROR
                assert validation_enabled and (e >> 16) & 0xFF == 9 and e & 0xFFFF == act, (key, hex(e), act)
            else:
                assert ((e >> 16) & 0xFF, e & 0xFFFF, e >> 24) == (nxt, act, 0xFF), (key, variant, hex(e), nxt, act)
        checked += 1
    assert checked == 6 * 8


def test_other_windows_unchanged():
    lib = ustlib.load()
    on = abi.make_policy(validation_enabled=True, evaluate_actuators=True, evaluate_validation=True)
    off = abi.make_policy(validation_enabled=True, evaluate_actuators=True)
    width = C.c_int(0)
    for s in range(16):
        assert lib.ust_table_window(C.byref(off), s, None) == lib.ust_table_window_shift(s)
        if s != 9:
            assert lib.ust_table_window(C.byref(on), s, None) == lib.ust_table_window_shift(s)
            for key in range(512):
                w = (key << lib.ust_table_window_shift(s)) & 0xFFFFFFFF
                assert lib.ust_table_entry(C.byref(on), s, w) == lib.ust_table_entry(C.byref(off), s, w)
    assert lib.ust_table_window(C.byref(off), 9, C.byref(width)) == 6 and width.value == 8


def test_header_constants():
    assert abi.UST_EVAL_ACTUATORS == 1 and abi.UST_EVAL_VALIDATION == 2
    assert abi.UST_POD_MATCH_VALIDATION_SELECTOR == 1 << 11 and abi.UST_POD_READY == 1 << 12
    assert (abi.UST_F_VALIDATION_START_ANNO, abi.UST_F_VALIDATION_START_INVALID, abi.UST_F_VALIDATION_TIMED_OUT) == (1 << 25, 1 << 26, 1 << 27)
    for b in (abi.UST_F_VALIDATION_START_ANNO, abi.UST_F_VALIDATION_START_INVALID, abi.UST_F_VALIDATION_TIMED_OUT):
        assert not b & abi.UST_F_INPUT_MASK
    assert abi.UST_ERR_VALIDATION == -10 and abi.ERROR_NAMES[-10] == "VALIDATION"
    assert abi.make_policy(evaluate_actuators=True, evaluate_validation=True).evaluate_actuators == 3
    assert abi.make_policy(evaluate_validation=True).evaluate_actuators == 2
    assert abi.make_policy(evaluate_actuators=True).evaluate_actuators == 1

