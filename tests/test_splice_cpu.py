"""ust_splice without a GPU: the ctypes mirror against the header, and the numpy model of the new node order (used by the
GPU tests) against a direct restatement of the rule in include/ust.h."""
import ctypes as C
import os
import subprocess
import tempfile

import numpy as np
import pytest

import splice_model
from helpers import abi


def test_splice_layout_matches_header():
    src = ('#include <stddef.h>\n#include <stdio.h>\n#include "ust.h"\nint main(){printf("%zu %zu %zu %zu %zu %zu %zu %zu %zu\\n", '
           'sizeof(ust_splice), offsetof(ust_splice, n_remove), offsetof(ust_splice, remove_idx), offsetof(ust_splice, n_insert), '
           'offsetof(ust_splice, insert_before), offsetof(ust_splice, state), offsetof(ust_splice, flags), '
           'offsetof(ust_splice, pod_rev), offsetof(ust_splice, ds_idx));return 0;}')
    with tempfile.TemporaryDirectory() as d:
        c = os.path.join(d, "t.c")
        with open(c, "w") as f:
            f.write(src)
        exe = os.path.join(d, "t")
        subprocess.check_call(["gcc", "-I", os.path.dirname(abi.HEADER), c, "-o", exe])
        got = [int(x) for x in subprocess.check_output([exe]).split()]
    S = abi.Splice
    assert got == [C.sizeof(S)] + [getattr(S, f).offset for f, _ in S._fields_]


def restated(a, rm, ib, ins):
    """The order rule of include/ust.h, element by element."""
    removed = set(int(x) for x in rm)
    out = []
    for p in range(len(a) + 1):
        out += [ins[k] for k in range(len(ib)) if ib[k] == p]
        if p < len(a) and p not in removed:
            out.append(a[p])
    return np.array(out, a.dtype)


EDGE = [  # (n, remove_idx, insert_before)
    (0, [], []), (0, [], [0, 0, 0]), (1, [0], []), (1, [0], [0]), (1, [0], [1]), (1, [], [0, 1]),
    (5, [0, 1, 2, 3, 4], []), (5, [0, 1, 2, 3, 4], [0, 2, 5]), (5, [2], [2, 2]), (5, [4], [5, 5]), (5, [0], [0]),
    (6, [1, 3], [1, 3, 3, 6]), (4, [], [0, 4]),
]


@pytest.mark.parametrize("n,rm,ib", EDGE)
def test_model_edge_cases(n, rm, ib):
    a = np.arange(100, 100 + n, dtype=np.int64)
    ins = np.arange(-1, -1 - len(ib), -1, dtype=np.int64)
    got = splice_model.splice(a, rm, ib, ins)
    assert np.array_equal(got, restated(a, rm, ib, ins))
    assert got.shape[0] == n - len(rm) + len(ib)


@pytest.mark.parametrize("seed", range(12))
def test_model_random(seed):
    rng = np.random.default_rng(seed)
    n = int(rng.choice([0, 1, 2, 7, 64, 300]))
    for mode in ("random", "head", "tail", "one_place", "same_place"):
        rm, ib = splice_model.random_splice(rng, n, float(rng.choice([0, 0.01, 0.3, 1.0])), float(rng.choice([0, 0.02, 0.5])), mode)
        a = rng.integers(0, 1 << 30, size=n).astype(np.int64)
        ins = rng.integers(-(1 << 30), 0, size=ib.shape[0]).astype(np.int64)
        assert np.all(np.diff(rm) > 0) and np.all(np.diff(ib) >= 0) and (ib.size == 0 or (ib.min() >= 0 and ib.max() <= n))
        assert np.array_equal(splice_model.splice(a, rm, ib, ins), restated(a, rm, ib, ins)), (seed, mode)
