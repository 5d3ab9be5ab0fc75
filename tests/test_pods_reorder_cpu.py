"""ust_pod_lists under a reorder, without a GPU: the numpy model of the pod-list CSR after a new node order and list
replacements at new indices (used by the GPU tests), against a node-by-node restatement of the rule in include/ust.h."""
import numpy as np
import pytest

import pods_delta_model
import pods_reorder_model as model
import reorder_model

ORDERS = ("identity", "moves", "swap", "reverse", "shuffle", "none", "insert_only", "mixed")


def restated(pod_off, pod_flags, order, lists):
    """New node p takes the list of its old node order[p], unless lists names it (then list k with node_idx[k] == p)."""
    named = {int(i): k for k, i in enumerate(lists["node_idx"])}
    no, nf = lists["pod_off"], lists["pod_flags"]
    flags, off = [], [0]
    for p, o in enumerate(np.asarray(order).tolist()):
        if p in named:
            k = named[p]
            flags.extend(nf[no[k]:no[k + 1]])
        else:
            assert o >= 0, "an inserted node without a list"
            flags.extend(pod_flags[pod_off[o]:pod_off[o + 1]])
        off.append(len(flags))
    return np.array(off, np.int64), np.array(flags, np.uint16)


def check(pod_off, pod_flags, order, lists):
    src, ln = reorder_model.runs_of(order)
    got_off, got_flags = model.reorder(pod_off, pod_flags, src, ln, lists["node_idx"], lists["pod_off"], lists["pod_flags"])
    ref_off, ref_flags = restated(pod_off, pod_flags, order, lists)
    assert got_off.dtype == np.int32 and got_flags.dtype == np.uint16
    assert np.array_equal(got_off, ref_off) and np.array_equal(got_flags, ref_flags)
    return got_off, got_flags


def csr(lens, rng):
    off = np.zeros(len(lens) + 1, np.int64)
    np.cumsum(lens, out=off[1:])
    return off.astype(np.int32), pods_delta_model.random_flags(rng, int(off[-1]))


@pytest.mark.parametrize("order_kind", ORDERS)
@pytest.mark.parametrize("kind", pods_delta_model.KINDS)
def test_model_matches_restatement(order_kind, kind):
    """Every order kind crossed with every list kind, chained over several sizes; every inserted node is named."""
    rng = np.random.default_rng(ORDERS.index(order_kind) * 100 + pods_delta_model.KINDS.index(kind))
    for n in (0, 1, 2, 9, 64, 301):
        off, flags = csr(rng.integers(0, 7, size=n), rng)
        for frac, f_move in ((0.0, 0.0), (0.01, 0.01), (0.3, 0.1), (1.0, 0.0)):
            cur = int(off.size - 1)
            order = reorder_model.random_order(rng, cur, order_kind, k=int(rng.integers(1, 6)), f_remove=f_move, f_insert=f_move)
            li = model.random_lists(rng, order, off, frac, kind)
            assert set(np.nonzero(order < 0)[0].tolist()) <= set(li["node_idx"].tolist())
            assert np.all(np.diff(li["node_idx"]) > 0)
            off, flags = check(off, flags, order, li)


def test_lists_move_with_their_nodes():
    """A hand-made case: lists [a b][][c][d e f] reordered to (3, inserted, 0, 2), node 0 (old 3) replaced by [x]."""
    off = np.array([0, 2, 2, 3, 6], np.int32)
    flags = np.array([1, 2, 3, 4, 5, 6], np.uint16)
    order = np.array([3, -1, 0, 2], np.int64)
    lists = {"node_idx": np.array([0, 1], np.int64), "pod_off": np.array([0, 1, 3], np.int32),
             "pod_flags": np.array([9, 7, 8], np.uint16)}
    got_off, got_flags = check(off, flags, order, lists)
    assert got_off.tolist() == [0, 1, 3, 5, 6] and got_flags.tolist() == [9, 7, 8, 1, 2, 3]
