"""numpy model of ust_splice (include/ust.h): the node order a membership splice of the resident snapshot produces."""
import numpy as np


def splice(a, remove_idx, insert_before, inserted):
    """`a` (one column of the old snapshot) in the new node order: for each old position p = 0..n the inserted values with
    insert_before == p (in the order given), then a[p] unless p is removed."""
    rm = np.asarray(remove_idx, np.int64)
    ib = np.asarray(insert_before, np.int64)
    return np.insert(np.delete(a, rm), ib - np.searchsorted(rm, ib), np.asarray(inserted, a.dtype))


def random_splice(rng, n, f_remove, f_insert, mode="random"):
    """(remove_idx, insert_before) for a snapshot of n nodes. mode: random | head | tail | one_place | same_place."""
    n_rm = min(n, int(round(n * f_remove)))
    rm = np.sort(rng.choice(n, size=n_rm, replace=False)).astype(np.int64) if n_rm else np.zeros(0, np.int64)
    n_ins = int(round(max(n, 1) * f_insert))
    if mode == "head":
        ib = np.zeros(n_ins, np.int64)
    elif mode == "tail":
        ib = np.full(n_ins, n, np.int64)
    elif mode == "one_place":
        ib = np.full(n_ins, int(rng.integers(0, n + 1)), np.int64)
    elif mode == "same_place":  # inserted exactly where nodes are removed
        ib = np.sort(rng.choice(rm, size=n_ins)) if n_rm else np.zeros(n_ins, np.int64)
    else:
        ib = np.sort(rng.integers(0, n + 1, size=n_ins)).astype(np.int64)
    return rm, ib
