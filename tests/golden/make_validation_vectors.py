"""Writes tests/golden/validation_vectors.json: known answers for ApplyState with UST_EVAL_VALIDATION (include/ust.h).

Each vector is one ApplyState over a few nodes, with file:line provenance in the reference (NVIDIA/k8s-operator-libs
pkg/upgrade). The seven ValidationManager specs (validation_manager_test.go:45-171) become vectors of a validation-required
node; a spec that calls Validate twice becomes two vectors, the second with the node as the first call left it. The
ApplyState-level vectors restate ProcessValidationRequiredNodes (common_manager.go:573-604) and
updateNodeToUncordonOrDoneState (:673-708). Mocked-provider semantics (upgrade_suit_test.go:114-182): a state change is the
next state, an annotation change an action.

A node: {"state", "flags": [UST_F_* names], "pods": [[UST_POD_* names / phase], ...] in API List order}.
Expected: rc ("OK" or a UST_ERR_* name), error_index, and per node the next state and the UST_A_* names.

    python tests/golden/make_validation_vectors.py
"""
import json
import os

R = "RUNNING"
READY = ["MATCH_VALIDATION_SELECTOR", "READY", R]                 # Running, every container Ready
NOT_READY = ["MATCH_VALIDATION_SELECTOR", R]                      # Running, a container not Ready
PENDING = ["MATCH_VALIDATION_SELECTOR", "PENDING"]                # not Running
OTHER = [R, "HAS_CONTROLLER"]                                     # a workload pod the selector does not match
V, U = "validation-required", "uncordon-required"


def node(flags=(), pods=(), state=V):
    return {"state": state, "flags": list(flags), "pods": [list(p) for p in pods]}


def vec(name, source, nodes, nxt, actions, rc="OK", error_index=-1, validation_enabled=True, requestor=False):
    return {"name": name, "source": source, "policy": {"validation_enabled": validation_enabled, "use_maintenance_operator": requestor},
            "nodes": nodes, "expect": {"rc": rc, "error_index": error_index, "next_state": nxt, "actions": actions}}


VECTORS = [
    vec("empty podSelector: done without a list", "validation_manager_test.go:52-58, common_manager.go:128",
        [node(pods=[NOT_READY])], [U], [["SET_STATE"]], validation_enabled=False),
    vec("no validation pod: not done, no annotation", "validation_manager_test.go:60-67, validation_manager.go:85-89",
        [node(pods=[OTHER])], [V], [[]]),
    vec("pod Running and Ready: done, annotation removed", "validation_manager_test.go:69-79, validation_manager.go:106-113",
        [node(pods=[READY])], [U], [["SET_STATE", "CLEAR_WAIT_START"]]),
    vec("pod Running but not Ready: start time set", "validation_manager_test.go:81-95, validation_manager.go:141-150",
        [node(pods=[NOT_READY])], [V], [["SET_WAIT_START"]]),
    vec("pod not Running: start time set", "validation_manager_test.go:97-111, validation_manager.go:119-122",
        [node(pods=[PENDING])], [V], [["SET_WAIT_START"]]),
    vec("timeout, call 1: start time set", "validation_manager_test.go:113-133",
        [node(pods=[NOT_READY])], [V], [["SET_WAIT_START"]]),
    vec("timeout, call 2: upgrade-failed, annotation removed", "validation_manager_test.go:135-146, validation_manager.go:161-169",
        [node(["VALIDATION_START_ANNO", "VALIDATION_TIMED_OUT"], [NOT_READY])], ["upgrade-failed"],
        [["SET_STATE", "CLEAR_WAIT_START"]]),
    vec("completion before timeout, call 1: start time set", "validation_manager_test.go:148-163",
        [node(pods=[NOT_READY])], [V], [["SET_WAIT_START"]]),
    vec("completion before timeout, call 2: done, annotation removed", "validation_manager_test.go:165-171",
        [node(["VALIDATION_START_ANNO"], [READY])], [U], [["SET_STATE", "CLEAR_WAIT_START"]]),
    vec("still waiting: annotation present, not timed out", "validation_manager.go:152-171",
        [node(["VALIDATION_START_ANNO"], [PENDING])], [V], [[]]),
    vec("done with the initial-state annotation: upgrade-done", "common_manager.go:593-597, :673-708",
        [node(["INITIAL_STATE_ANNO"], [READY])], ["upgrade-done"],
        [["SET_STATE", "CLEAR_INITIAL_STATE_ANNO", "CLEAR_WAIT_START"]]),
    vec("done in requestor mode: uncordon-required, initial-state annotation removed", "common_manager.go:673-708, util.go:135-138",
        [node(["INITIAL_STATE_ANNO", "REQUESTOR_MODE"], [READY]), node(["REQUESTOR_MODE"], [READY])], [U, U],
        [["SET_STATE", "CLEAR_INITIAL_STATE_ANNO", "CLEAR_WAIT_START"], ["SET_STATE", "CLEAR_INITIAL_STATE_ANNO", "CLEAR_WAIT_START"]],
        requestor=True),
    vec("safe load: the driver is unblocked before Validate", "common_manager.go:578-585, safe_driver_load_manager.go:57-71",
        [node(["SAFE_LOAD"], [NOT_READY]), node(["SAFE_LOAD"], [READY])], [V, U],
        [["UNBLOCK_SAFE_LOAD", "SET_WAIT_START"], ["UNBLOCK_SAFE_LOAD", "SET_STATE", "CLEAR_WAIT_START"]]),
    vec("list order: a ready pod first deletes the annotation, so a timed-out node is not failed",
        "validation_manager.go:99-115, :141-150",
        [node(["VALIDATION_START_ANNO", "VALIDATION_TIMED_OUT"], [READY, OTHER, NOT_READY]),
         node(["VALIDATION_START_ANNO", "VALIDATION_TIMED_OUT"], [NOT_READY, OTHER, READY]),
         node(["VALIDATION_START_ANNO", "VALIDATION_START_INVALID"], [READY, PENDING])],
        [V, "upgrade-failed", V],
        [["CLEAR_WAIT_START", "SET_WAIT_START"], ["SET_STATE", "CLEAR_WAIT_START"], ["CLEAR_WAIT_START", "SET_WAIT_START"]]),
    vec("unparsable start time: ApplyState aborts in pass 10; later nodes of the pass and uncordon-required untouched",
        "validation_manager.go:152-160, common_manager.go:587-590, upgrade_state.go:262-274",
        [node(pods=[READY]), node(["SAFE_LOAD", "VALIDATION_START_ANNO", "VALIDATION_START_INVALID"], [PENDING, READY]),
         node(pods=[READY]), node(state=U)],
        [U, V, V, U], [["SET_STATE", "CLEAR_WAIT_START"], ["UNBLOCK_SAFE_LOAD", "ERROR"], [], []],
        rc="VALIDATION", error_index=1),
]

if __name__ == "__main__":
    out = os.path.join(os.path.dirname(os.path.abspath(__file__)), "validation_vectors.json")
    with open(out, "w") as f:
        json.dump({"reference": "NVIDIA/k8s-operator-libs pkg/upgrade", "vectors": VECTORS}, f, indent=1)
        f.write("\n")
    print(out, len(VECTORS))
