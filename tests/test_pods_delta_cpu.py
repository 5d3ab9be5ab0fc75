"""ust_pod_lists without a GPU: the ctypes mirror against the header, and the numpy model of the CSR after list
replacements (used by the GPU tests) against a direct restatement of the rule in include/ust.h."""
import ctypes as C
import os
import subprocess
import tempfile

import numpy as np
import pytest

import pods_delta_model as model
from helpers import abi


def test_pod_lists_layout_matches_header():
    src = ('#include <stddef.h>\n#include <stdio.h>\n#include "ust.h"\nint main(){printf("%zu %zu %zu %zu %zu %zu\\n", '
           'sizeof(ust_pod_lists), offsetof(ust_pod_lists, n_lists), offsetof(ust_pod_lists, node_idx), '
           'offsetof(ust_pod_lists, pod_off), offsetof(ust_pod_lists, pod_flags), offsetof(ust_pod_lists, n_pods));return 0;}')
    with tempfile.TemporaryDirectory() as d:
        c = os.path.join(d, "t.c")
        with open(c, "w") as f:
            f.write(src)
        exe = os.path.join(d, "t")
        subprocess.check_call(["gcc", "-I", os.path.dirname(abi.HEADER), c, "-o", exe])
        got = [int(x) for x in subprocess.check_output([exe]).split()]
    P = abi.PodLists
    assert got == [C.sizeof(P)] + [getattr(P, f).offset for f, _ in P._fields_]


def restated(pod_off, pod_flags, node_idx, new_off, new_flags):
    """The rule of include/ust.h, node by node: list k replaces the list of node node_idx[k], every other node keeps its
    list; and the offsets as off'[i] = off[i] + sum over k with node_idx[k] < i of (new length - old length)."""
    n = len(pod_off) - 1
    repl = {int(i): k for k, i in enumerate(node_idx)}
    flags = []
    for i in range(n):
        if i in repl:
            k = repl[i]
            flags.extend(new_flags[new_off[k]:new_off[k + 1]])
        else:
            flags.extend(pod_flags[pod_off[i]:pod_off[i + 1]])
    off = []
    for i in range(n + 1):
        d = sum((new_off[k + 1] - new_off[k]) - (pod_off[j + 1] - pod_off[j]) for k, j in enumerate(node_idx) if j < i)
        off.append(pod_off[i] + d)
    return np.array(off, np.int64), np.array(flags, np.uint16)


def check(pod_off, pod_flags, lists):
    got_off, got_flags = model.replace(pod_off, pod_flags, lists["node_idx"], lists["pod_off"], lists["pod_flags"])
    ref_off, ref_flags = restated(pod_off, pod_flags, lists["node_idx"], lists["pod_off"], lists["pod_flags"])
    assert got_off.dtype == np.int32 and got_flags.dtype == np.uint16
    assert np.array_equal(got_off, ref_off) and np.array_equal(got_flags, ref_flags)
    assert got_off[0] == 0 and np.all(np.diff(got_off) >= 0) and got_off[-1] == got_flags.size
    return got_off, got_flags


def csr(lens, rng):
    off = np.zeros(len(lens) + 1, np.int64)
    np.cumsum(lens, out=off[1:])
    return off.astype(np.int32), model.random_flags(rng, int(off[-1]))


def lists(node_idx, lens, rng):
    off = np.zeros(len(lens) + 1, np.int64)
    np.cumsum(lens, out=off[1:])
    return {"node_idx": np.array(node_idx, np.int64), "pod_off": off.astype(np.int32), "pod_flags": model.random_flags(rng, int(off[-1]))}


EDGE = [  # (old lengths, replaced nodes, new lengths)
    ([], [], []),                              # empty snapshot
    ([3], [], []),                             # nothing replaced
    ([3], [0], [3]), ([3], [0], [0]), ([0], [0], [4]), ([0], [0], [0]),
    ([2, 0, 5], [0], [7]),                     # the first node
    ([2, 0, 5], [2], [1]),                     # the last node
    ([2, 0, 5], [0, 1, 2], [0, 0, 0]),         # all nodes, to empty
    ([0, 0, 0], [0, 1, 2], [1, 2, 3]),         # all nodes, from empty
    ([4, 4, 4, 4], [0, 1, 2, 3], [4, 4, 4, 4]),  # all nodes, same lengths
    ([5, 1, 0, 7, 2], [1, 3], [0, 9]),         # neighbours of unchanged stretches
    ([5, 1, 0, 7, 2], [0, 1], [6, 2]),         # adjacent replaced lists
    ([1, 1, 1, 1, 1, 1], [1, 4], [2, 0]),      # shifts by odd counts
]


@pytest.mark.parametrize("old,idx,new", EDGE)
def test_model_edge_cases(old, idx, new):
    rng = np.random.default_rng(len(old) * 31 + len(idx))
    off, flags = csr(old, rng)
    check(off, flags, lists(idx, new, rng))


@pytest.mark.parametrize("seed", range(6))
def test_model_random_chains(seed):
    """Chains of replacements of every kind and fraction, each step checked against the restatement."""
    rng = np.random.default_rng(seed)
    for n in (1, 2, 9, 64, 301):
        off, flags = csr(rng.integers(0, 7, size=n), rng)
        for frac in (0.0, 0.001, 0.01, 0.3, 1.0):
            for kind in model.KINDS:
                li = model.random_lists(rng, off, frac, kind)
                if kind == "same":
                    assert np.array_equal(np.diff(li["pod_off"]), np.diff(off)[li["node_idx"]])
                if kind == "odd":
                    assert np.all((np.diff(li["pod_off"]) - np.diff(off)[li["node_idx"]]) % 2 == 1)
                off, flags = check(off, flags, li)
