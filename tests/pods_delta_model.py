"""numpy model of ust_pod_lists (include/ust.h): the pod-list CSR after the lists of some nodes were replaced, and random
replacement lists of the kinds the GPU tests chain."""
import numpy as np

from helpers import abi


def replace(pod_off, pod_flags, node_idx, new_off, new_flags):
    """(pod_off', pod_flags') after list k of (new_off, new_flags) replaced the list of node node_idx[k]. Built from the
    2 len(node_idx) + 1 slices the new CSR is made of, so it stays within memory at full size."""
    off = np.asarray(pod_off, np.int64)
    ni = np.asarray(node_idx, np.int64)
    no = np.asarray(new_off, np.int64)
    lens = np.diff(off)
    lens[ni] = np.diff(no)
    out_off = np.zeros(off.size, np.int64)
    np.cumsum(lens, out=out_off[1:])
    pieces, end = [], 0  # end: old pod position after the previous replaced list
    for k, i in enumerate(ni.tolist()):
        pieces.append(pod_flags[end:off[i]])
        pieces.append(new_flags[no[k]:no[k + 1]])
        end = int(off[i + 1])
    pieces.append(pod_flags[end:int(off[-1])])
    out = np.concatenate(pieces).astype(np.uint16) if pieces else np.zeros(0, np.uint16)
    assert out.size == out_off[-1]
    return out_off.astype(np.int32), out


def random_flags(rng, m):
    """Pod flags with every UST_POD_* bit i.i.d. and phases 0..5 (the undefined 5 included)."""
    pf = rng.integers(0, 6, size=m).astype(np.uint16)
    for k, v in abi.K.items():
        if k.startswith("UST_POD_") and k != "UST_POD_PHASE_MASK":
            pf |= np.where(rng.random(m) < 0.4, np.uint16(v), np.uint16(0))
    return pf


KINDS = ("same", "grow", "shrink", "zero", "from_zero", "odd", "mixed")


def new_lengths(rng, old, kind):
    """Lengths of replacement lists for lists of lengths `old`."""
    m = old.size
    if kind == "same":
        return old.copy()
    if kind == "grow":
        return old + rng.integers(1, 6, size=m)
    if kind == "shrink":
        return np.maximum(old - rng.integers(1, 6, size=m), 0)
    if kind == "zero":
        return np.zeros(m, np.int64)
    if kind == "from_zero":
        return np.where(old == 0, rng.integers(1, 9, size=m), old)
    if kind == "odd":  # every length moves by an odd count (the CSR behind it shifts by odd pod counts)
        d = rng.choice([-3, -1, 1, 3, 5], size=m)
        d = np.where(old + d < 0, np.abs(d), d)
        return old + d
    assert kind == "mixed"
    return np.stack([new_lengths(rng, old, k) for k in KINDS[:-1]])[rng.integers(0, len(KINDS) - 1, size=m), np.arange(m)]


def random_lists(rng, pod_off, frac=None, kind="mixed", node_idx=None):
    """Replacement lists for a fraction of the nodes (at least one node when frac > 0), or for `node_idx`."""
    off = np.asarray(pod_off, np.int64)
    n = off.size - 1
    if node_idx is None:
        m = min(n, int(np.ceil(n * frac))) if frac > 0 else 0
        node_idx = np.sort(rng.choice(n, size=m, replace=False)) if m else np.zeros(0, np.int64)
    node_idx = np.asarray(node_idx, np.int64)
    lens = new_lengths(rng, np.diff(off)[node_idx], kind).astype(np.int64)
    new_off = np.zeros(node_idx.size + 1, np.int64)
    np.cumsum(lens, out=new_off[1:])
    return {"node_idx": node_idx, "pod_off": new_off.astype(np.int32), "pod_flags": random_flags(rng, int(new_off[-1]))}
