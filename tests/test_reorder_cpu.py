"""ust_reorder without a GPU: the ctypes mirror against the header, the numpy model of the new node order (used by the GPU
tests) against a direct restatement of the rule in include/ust.h, and the maximal runs of a target order."""
import ctypes as C
import os
import subprocess
import tempfile

import numpy as np
import pytest

import reorder_model
from helpers import abi


def test_reorder_layout_matches_header():
    src = ('#include <stddef.h>\n#include <stdio.h>\n#include "ust.h"\nint main(){printf("%zu %zu %zu %zu %zu %zu %zu %zu %zu\\n", '
           'sizeof(ust_reorder), offsetof(ust_reorder, n_runs), offsetof(ust_reorder, run_src), offsetof(ust_reorder, run_len), '
           'offsetof(ust_reorder, n_insert), offsetof(ust_reorder, state), offsetof(ust_reorder, flags), '
           'offsetof(ust_reorder, pod_rev), offsetof(ust_reorder, ds_idx));return 0;}')
    with tempfile.TemporaryDirectory() as d:
        c = os.path.join(d, "t.c")
        with open(c, "w") as f:
            f.write(src)
        exe = os.path.join(d, "t")
        subprocess.check_call(["gcc", "-I", os.path.dirname(abi.HEADER), c, "-o", exe])
        got = [int(x) for x in subprocess.check_output([exe]).split()]
    R = abi.Reorder
    assert got == [C.sizeof(R)] + [getattr(R, f).offset for f, _ in R._fields_]


def restated(a, run_src, run_len, ins):
    """The order rule of include/ust.h, element by element."""
    out, k = [], 0
    for s, ln in zip(run_src, run_len):
        for e in range(ln):
            if s >= 0:
                out.append(a[s + e])
            else:
                out.append(ins[k])
                k += 1
    assert k == len(ins)
    return np.array(out, a.dtype)


EDGE = [  # (n, run_src, run_len, n_insert)
    (0, [], [], 0), (0, [-1], [3], 3), (1, [0], [1], 0), (1, [], [], 0), (1, [-1, 0], [2, 1], 2), (1, [0, -1], [1, 1], 1),
    (5, [4, 3, 2, 1, 0], [1, 1, 1, 1, 1], 0), (5, [3, 0], [2, 3], 0), (5, [-1, 2, -1, 0], [1, 3, 2, 1], 3),
    (6, [5, -1, 1], [1, 4, 2], 4), (4, [1], [2], 0),
]


@pytest.mark.parametrize("n,src,ln,n_ins", EDGE)
def test_model_edge_cases(n, src, ln, n_ins):
    a = np.arange(100, 100 + n, dtype=np.int64)
    ins = np.arange(-1, -1 - n_ins, -1, dtype=np.int64)
    got = reorder_model.reorder(a, src, ln, ins)
    assert np.array_equal(got, restated(a, src, ln, ins))
    assert got.shape[0] == sum(ln)


KINDS = ("identity", "moves", "swap", "reverse", "shuffle", "none", "insert_only", "mixed")


@pytest.mark.parametrize("seed", range(8))
def test_model_random(seed):
    """Random target orders of every kind: their maximal runs rebuild them, restate to the same arrays, and are maximal."""
    rng = np.random.default_rng(seed)
    for n in (0, 1, 2, 7, 64, 300):
        for kind in KINDS:
            f = float(rng.choice([0, 0.01, 0.3])) if kind == "mixed" else 0.0
            order = reorder_model.random_order(rng, n, kind, k=int(rng.integers(1, 9)), f_remove=f, f_insert=f)
            src, ln = reorder_model.runs_of(order)
            assert np.all(ln >= 1) and np.all(src >= -1) and int(ln.sum()) == order.size
            assert np.array_equal(reorder_model.order_of(src, ln), order), (seed, n, kind)
            # no old node twice, all in [0, n)
            old = order[order >= 0]
            assert np.unique(old).size == old.size and (old.size == 0 or old.max() < n)
            # maximal: no two neighbouring runs continue each other
            for r in range(1, src.size):
                assert not (src[r] < 0 and src[r - 1] < 0)
                assert not (src[r] >= 0 and src[r - 1] >= 0 and src[r] == src[r - 1] + ln[r - 1])
            a = rng.integers(0, 1 << 30, size=n).astype(np.int64)
            ins = rng.integers(-(1 << 30), 0, size=int(np.sum(order < 0))).astype(np.int64)
            assert np.array_equal(reorder_model.reorder(a, src, ln, ins), restated(a, src, ln, ins)), (seed, n, kind)


def test_identity_is_one_run_and_shuffle_all_ones():
    src, ln = reorder_model.runs_of(np.arange(10))
    assert src.tolist() == [0] and ln.tolist() == [10]
    src, ln = reorder_model.runs_of(np.array([3, 1, 2, -1, -1, 0]))
    assert src.tolist() == [3, 1, -1, 0] and ln.tolist() == [1, 2, 2, 1]
