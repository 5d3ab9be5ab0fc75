"""numpy model of ust_reorder (include/ust.h): the node order a reorder of the resident snapshot produces, and the maximal
runs that describe a target order."""
import numpy as np


def reorder(a, run_src, run_len, inserted):
    """`a` (one column of the old snapshot) in the new node order: the runs concatenated, old run r = a[run_src[r] :
    run_src[r] + run_len[r]], inserted run r = the next run_len[r] values of `inserted`."""
    src = np.asarray(run_src, np.int64)
    ln = np.asarray(run_len, np.int64)
    inserted = np.asarray(inserted, a.dtype)
    if src.size == 0:
        return a[:0].copy()
    old = src >= 0
    ins_len = np.where(old, 0, ln)
    base = np.where(old, src, np.cumsum(ins_len) - ins_len)  # a run's first index into `a` or into `inserted`
    # per new position: its run's base + its offset in the run
    pos = np.repeat(base - (np.cumsum(ln) - ln), ln) + np.arange(int(ln.sum()))
    from_old = np.repeat(old, ln)
    out = np.empty(int(ln.sum()), a.dtype)
    out[from_old] = a[pos[from_old]]
    out[~from_old] = inserted[pos[~from_old]]
    return out


def runs_of(order):
    """Maximal runs (run_src, run_len) of a target order: order[p] = the old node at new position p, or -1 for the next
    inserted node."""
    o = np.asarray(order, np.int64)
    if o.size == 0:
        return np.zeros(0, np.int64), np.zeros(0, np.int64)
    cont = np.zeros(o.size, bool)
    cont[1:] = ((o[1:] >= 0) & (o[:-1] >= 0) & (o[1:] == o[:-1] + 1)) | ((o[1:] < 0) & (o[:-1] < 0))
    starts = np.nonzero(~cont)[0]
    ln = np.diff(np.append(starts, o.size)).astype(np.int64)
    return o[starts].copy(), ln


def order_of(run_src, run_len):
    """The target order (as in runs_of) that runs describe."""
    src = np.asarray(run_src, np.int64)
    ln = np.asarray(run_len, np.int64)
    if src.size == 0:
        return np.zeros(0, np.int64)
    off = np.repeat(np.cumsum(ln) - ln, ln)
    p = np.arange(int(ln.sum()))
    return np.where(np.repeat(src, ln) >= 0, np.repeat(src, ln) + p - off, -1)


def random_order(rng, n, kind, k=8, f_remove=0.0, f_insert=0.0):
    """A target order for a snapshot of n nodes. kind: identity | moves (k single nodes moved) | swap (two blocks swapped)
    | reverse (blocks in reverse order) | shuffle | none (everything removed) | insert_only | mixed (moves, removals and
    insertions). f_remove / f_insert: nodes removed / inserted besides (mixed)."""
    o = np.arange(n, dtype=np.int64)
    if kind == "identity":
        pass
    elif kind == "moves":
        for _ in range(min(k, n)):
            i, j = int(rng.integers(0, o.size)), int(rng.integers(0, o.size))
            v = o[i]
            o = np.insert(np.delete(o, i), j, v)
    elif kind == "swap":
        c = int(rng.integers(0, n + 1))
        o = np.concatenate([o[c:], o[:c]])
    elif kind == "reverse":
        cuts = np.sort(rng.integers(0, n + 1, size=k))
        o = np.concatenate(np.split(o, cuts)[::-1])
    elif kind == "shuffle":
        o = rng.permutation(n).astype(np.int64)
    elif kind == "none":
        o = o[:0]
    elif kind == "insert_only":
        o = np.full(max(k, 1), -1, np.int64)
    elif kind == "mixed":
        o = random_order(rng, n, "moves", k)
    else:
        raise ValueError(kind)
    if f_remove and o.size:
        o = np.delete(o, rng.choice(o.size, size=min(o.size, int(round(o.size * f_remove))), replace=False))
    n_ins = int(round(max(n, 1) * f_insert))
    if n_ins:
        o = np.insert(o, np.sort(rng.integers(0, o.size + 1, size=n_ins)), -1)
    return o
