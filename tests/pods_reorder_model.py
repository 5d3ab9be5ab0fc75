"""numpy model of ust_apply_state_delta_pods_reorder's pod lists (include/ust.h): the pod-list CSR after a new node order
(reorder_model) and list replacements at new indices (pods_delta_model), and random replacement lists for it."""
import numpy as np

import pods_delta_model
import reorder_model


def moved(pod_off, pod_flags, run_src, run_len):
    """(pod_off', pod_flags') with every list moved with its node; an inserted node has an empty list. Built from one
    slice per run, so that it stays within memory at full size."""
    off = np.asarray(pod_off, np.int64)
    src = np.asarray(run_src, np.int64)
    ln = np.asarray(run_len, np.int64)
    n_ins = int(ln[src < 0].sum())
    lens = reorder_model.reorder(np.diff(off), src, ln, np.zeros(n_ins, np.int64))
    out_off = np.zeros(lens.size + 1, np.int64)
    np.cumsum(lens, out=out_off[1:])
    pieces = [pod_flags[off[s]:off[s + l]] for s, l in zip(src.tolist(), ln.tolist()) if s >= 0]
    flags = np.concatenate(pieces).astype(np.uint16) if pieces else np.zeros(0, np.uint16)
    assert flags.size == out_off[-1]
    return out_off.astype(np.int32), flags


def reorder(pod_off, pod_flags, run_src, run_len, node_idx, new_off, new_flags):
    """(pod_off', pod_flags') of the new snapshot: the lists moved with their nodes, then list k of (new_off, new_flags)
    replaces the list of new node node_idx[k]."""
    off, flags = moved(pod_off, pod_flags, run_src, run_len)
    return pods_delta_model.replace(off, flags, node_idx, new_off, new_flags)


def random_lists(rng, order, pod_off, frac=0.0, kind="mixed"):
    """Replacement lists for a target order (reorder_model.runs_of): one for every inserted node (0 to 8 pods, none for
    kind "zero") and for a fraction of the nodes that stay (at least one when frac > 0), of pods_delta_model's kind."""
    order = np.asarray(order, np.int64)
    old_len = np.diff(np.asarray(pod_off, np.int64))
    kept = np.nonzero(order >= 0)[0]
    m = min(kept.size, int(np.ceil(kept.size * frac))) if frac > 0 else 0
    chosen = rng.choice(kept, size=m, replace=False) if m else np.zeros(0, np.int64)
    node_idx = np.union1d(chosen, np.nonzero(order < 0)[0]).astype(np.int64)
    lens = np.zeros(node_idx.size, np.int64)
    stay = order[node_idx] >= 0
    lens[stay] = pods_delta_model.new_lengths(rng, old_len[order[node_idx[stay]]], kind)
    lens[~stay] = 0 if kind == "zero" else rng.integers(0, 9, size=int((~stay).sum()))
    new_off = np.zeros(node_idx.size + 1, np.int64)
    np.cumsum(lens, out=new_off[1:])
    return {"node_idx": node_idx, "pod_off": new_off.astype(np.int32),
            "pod_flags": pods_delta_model.random_flags(rng, int(new_off[-1]))}
