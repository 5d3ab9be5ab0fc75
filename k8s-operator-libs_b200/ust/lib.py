"""ctypes binding of libust.so (include/ust.h). Plumbing for tests and bench.py — the product is the .so."""
import ctypes as C
import os

import numpy as np

from . import abi

HERE = os.path.dirname(os.path.abspath(__file__))
SO_PATH = os.environ.get("UST_LIB") or os.path.join(os.path.dirname(HERE), "libust.so")  # UST_LIB: tuning experiments only

_lib = None


class UstError(RuntimeError):
    def __init__(self, code, msg):
        super().__init__(f"{abi.ERROR_NAMES.get(code, code)}: {msg}")
        self.code = code


def load():
    """Load libust.so. There is no fallback: a missing library is an error."""
    global _lib
    if _lib is None:
        if not os.path.exists(SO_PATH):
            raise UstError(abi.UST_ERR_CUDA, f"{SO_PATH} not built (python __graft_entry__.py build)")
        lib = C.CDLL(SO_PATH)
        lib.ust_create.argtypes = [C.POINTER(C.c_void_p), C.c_int]
        lib.ust_destroy.argtypes = [C.c_void_p]
        lib.ust_destroy.restype = None
        lib.ust_last_error.argtypes = [C.c_void_p]
        lib.ust_last_error.restype = C.c_char_p
        lib.ust_create_error.restype = C.c_char_p
        lib.ust_launch_count.argtypes = [C.c_void_p]
        lib.ust_launch_count.restype = C.c_int64
        lib.ust_host_alloc.argtypes = [C.c_size_t]
        lib.ust_host_alloc.restype = C.c_void_p
        lib.ust_host_free.argtypes = [C.c_void_p]
        lib.ust_host_free.restype = None
        lib.ust_sync.argtypes = [C.c_void_p]
        lib.ust_stream.argtypes = [C.c_void_p]
        lib.ust_stream.restype = C.c_void_p
        apply_args = [C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32,
                      C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
        lib.ust_apply_state.argtypes = apply_args
        lib.ust_apply_state_device.argtypes = apply_args + [C.c_void_p]
        lib.ust_apply_state_packed.argtypes = [C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32,
                                               C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
        lib.ust_apply_state_clocked.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p] + apply_args[2:]
        # the delta calls: handle, policy, the call's structs (order change, pod lists, clock), the changed nodes and the
        # DaemonSet table, the outputs; the sparse ones end in out_outcome (pod lists only), n_out and the counters
        vp = C.c_void_p
        nodes = [C.c_int64, vp, vp, vp, vp, vp, C.c_int32, vp]  # n_changed, idx, state, flags, pod_rev, ds_idx, n_ds, ds_rev
        sparse = [C.c_int64, vp, vp, vp]  # max_out, out_idx, out_next_state, out_actions
        lib.ust_apply_state_delta.argtypes = [vp, vp] + nodes + [vp, vp, vp, vp]
        lib.ust_apply_state_delta_sparse.argtypes = [vp, vp] + nodes + sparse + [vp, vp]
        lib.ust_apply_state_delta_splice.argtypes = [vp, vp, vp] + nodes + sparse + [vp, vp]
        lib.ust_apply_state_delta_reorder.argtypes = [vp, vp, vp] + nodes + sparse + [vp, vp]
        lib.ust_apply_state_delta_pods.argtypes = [vp, vp, vp] + nodes + sparse + [vp, vp, vp]
        lib.ust_apply_state_delta_pods_reorder.argtypes = [vp, vp, vp, vp] + nodes + sparse + [vp, vp, vp]
        lib.ust_apply_state_delta_pods_clocked.argtypes = [vp, vp, vp, vp, vp] + nodes + sparse + [vp, vp, vp]
        lib.ust_fetch_outputs.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p]
        lib.ust_fetch_outputs_pods.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
        lib.ust_next_deadline.argtypes = [C.c_void_p, C.c_void_p]
        lib.ust_simulate_rollout.argtypes = [C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
        lib.ust_simulate_rollout_timed.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p,
                                                   C.c_void_p, C.c_void_p]
        lib.ust_build_state.argtypes = [C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p]
        lib.ust_build_state_uids.argtypes = [C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p,
                                             C.c_void_p, C.c_void_p]
        lib.ust_build_state_delta.argtypes = [C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32,
                                              C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
        lib.ust_fetch_build_state.argtypes = [C.c_void_p, C.c_int64, C.c_void_p]
        lib.ust_get_unique_id.argtypes = [C.c_void_p]
        lib.ust_comm_init.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_void_p]
        lib.ust_comm_set_mode.argtypes = [C.c_void_p, C.c_int]
        lib.ust_table_entry.argtypes = [C.c_void_p, C.c_uint, C.c_uint32]
        lib.ust_table_entry.restype = C.c_uint32
        lib.ust_table_window_shift.argtypes = [C.c_uint]
        lib.ust_table_window.argtypes = [C.c_void_p, C.c_uint, C.c_void_p]
        _lib = lib
    return _lib


EXPORTS = ["ust_abi_version", "ust_create", "ust_destroy", "ust_last_error", "ust_create_error", "ust_launch_count",
           "ust_host_alloc", "ust_host_free", "ust_apply_state", "ust_apply_state_device", "ust_stream", "ust_apply_state_packed", "ust_apply_state_delta", "ust_apply_state_delta_sparse", "ust_apply_state_delta_splice", "ust_apply_state_delta_reorder", "ust_apply_state_delta_pods", "ust_apply_state_delta_pods_reorder", "ust_apply_state_clocked", "ust_apply_state_delta_pods_clocked", "ust_fetch_outputs", "ust_fetch_outputs_pods", "ust_next_deadline", "ust_simulate_rollout", "ust_simulate_rollout_timed", "ust_sync",
           "ust_build_state", "ust_build_state_uids", "ust_build_state_delta", "ust_fetch_build_state", "ust_get_unique_id", "ust_comm_init", "ust_comm_set_mode", "ust_table_entry",
           "ust_table_window_shift", "ust_table_window"]


def _p(a):
    if a is None:
        return None
    if isinstance(a, np.ndarray):
        return a.ctypes.data
    return int(a)  # raw address (e.g. torch tensor .data_ptr())


def _ref(s):
    """Address of a ctypes struct, or NULL for None."""
    return C.addressof(s) if s is not None else None


# The ABI structs of the delta calls from the dicts the Handle methods take. Each helper returns the struct (None for None)
# and the arrays it points into, which must stay alive until the call returns.
_NODE_COLUMNS = (("state", np.uint8), ("flags", np.uint32), ("pod_rev", np.int32), ("ds_idx", np.int32))


def _inserted(d):
    """The inserted nodes' columns of a splice or reorder dict (None for a column it lacks)."""
    return [np.ascontiguousarray(d[k], dtype=dt) if k in d else None for k, dt in _NODE_COLUMNS]


def _splice(splice):
    """ust_splice of a dict with remove_idx, insert_before and the inserted nodes' columns."""
    if splice is None:
        return None, []
    rm = np.ascontiguousarray(splice.get("remove_idx", np.zeros(0)), dtype=np.int64)
    ib = np.ascontiguousarray(splice.get("insert_before", np.zeros(0)), dtype=np.int64)
    ins = _inserted(splice)
    return abi.Splice(int(rm.shape[0]), _p(rm), int(ib.shape[0]), _p(ib), *[_p(a) for a in ins]), [rm, ib] + ins


def _reorder(reorder):
    """ust_reorder of a dict with run_src, run_len and the inserted nodes' columns (n_insert defaults to their count)."""
    if reorder is None:
        return None, []
    src = np.ascontiguousarray(reorder.get("run_src", np.zeros(0)), dtype=np.int64)
    ln = np.ascontiguousarray(reorder.get("run_len", np.zeros(0)), dtype=np.int64)
    ins = _inserted(reorder)
    n_ins = reorder.get("n_insert", 0 if ins[0] is None else int(ins[0].shape[0]))
    return abi.Reorder(int(src.shape[0]), _p(src), _p(ln), int(n_ins), *[_p(a) for a in ins]), [src, ln] + ins


def _pod_lists(lists):
    """ust_pod_lists of a dict with node_idx, pod_off and pod_flags."""
    if lists is None:
        return None, []
    ni = np.ascontiguousarray(lists["node_idx"], dtype=np.int64)
    off = np.ascontiguousarray(lists["pod_off"], dtype=np.int32)
    pf = np.ascontiguousarray(lists["pod_flags"], dtype=np.uint16)
    return abi.PodLists(int(ni.shape[0]), _p(ni), _p(off), _p(pf), int(pf.shape[0])), [ni, off, pf]


def _clock(now, wait_timeout_seconds, start, insert_start):
    """ust_clock; a start array that is None is passed as NULL."""
    keep = [np.ascontiguousarray(a, dtype=np.int64) if a is not None else None for a in (start, insert_start)]
    return abi.Clock(int(now), int(wait_timeout_seconds), *[_p(a) for a in keep]), keep


def _changed_nodes(idx, changed, ds_rev):
    """The arguments n_changed .. ds_rev of a delta call: the nodes at `idx` with their columns `changed`, and the
    DaemonSet table."""
    idx = np.ascontiguousarray(idx, dtype=np.int64)
    cols = [np.ascontiguousarray(changed[k], dtype=dt) for k, dt in _NODE_COLUMNS]
    ds_rev = np.ascontiguousarray(ds_rev, dtype=np.int32)
    return [int(idx.shape[0]), _p(idx)] + [_p(a) for a in cols] + [int(ds_rev.shape[0]), _p(ds_rev)], [idx, ds_rev] + cols


def _sparse_outputs(max_out, out, pods):
    """The arguments max_out .. out (counters) of a sparse delta call, and what the call writes: the output arrays (`out`
    reused, or max_out + 1 entries each; out_outcome with pod lists only), n_out and the counters."""
    k = 4 if pods else 3
    if out is None:
        out = [np.zeros(max_out + 1, dt) for dt in (np.int64, np.uint8, np.uint16, np.uint8)[:k]]
    out = tuple(out[:k])
    n_out, cnt = C.c_int64(0), abi.Counters()
    return [C.c_int64(int(max_out))] + [_p(a) for a in out] + [C.addressof(n_out), C.addressof(cnt)], (out, n_out, cnt)


def pinned_array(shape, dtype):
    """numpy array backed by ust_host_alloc (page-locked) memory."""
    lib = load()
    dt = np.dtype(dtype)
    n = int(np.prod(shape)) if not np.isscalar(shape) else int(shape)
    nbytes = max(n * dt.itemsize, 1)
    ptr = lib.ust_host_alloc(nbytes)
    if not ptr:
        raise UstError(abi.UST_ERR_CUDA, "ust_host_alloc failed")
    buf = (C.c_char * nbytes).from_address(ptr)
    arr = np.frombuffer(buf, dtype=dt, count=n).reshape(shape)
    _PINNED[arr.ctypes.data] = ptr
    return arr


_PINNED = {}


def free_pinned(arr):
    ptr = _PINNED.pop(arr.ctypes.data, None)
    if ptr:
        load().ust_host_free(ptr)


class Handle:
    """ust_handle wrapper. One per process per GPU."""

    def __init__(self, device=0):
        lib = load()
        h = C.c_void_p()
        rc = lib.ust_create(C.byref(h), device)
        if rc != 0:
            raise UstError(rc, lib.ust_create_error().decode())
        self._h = h
        self._lib = lib

    def close(self):
        if getattr(self, "_h", None):
            self._lib.ust_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def last_error(self):
        return self._lib.ust_last_error(self._h).decode()

    def launch_count(self):
        return int(self._lib.ust_launch_count(self._h))

    def overlapped_calls(self):
        """diagnostics: how many ust_apply_state_device calls started without waiting for the previous call's tail"""
        fn = self._lib.ust_debug_relaxed_calls
        fn.restype = C.c_longlong
        fn.argtypes = [C.c_void_p]
        return int(fn(self._h))

    def stream_ctas_per_sm(self):
        """diagnostics: streaming CTAs one SM holds (occupancy API at ust_create, fewest over the kernel's variants)"""
        fn = self._lib.ust_debug_stream_ctas_per_sm
        fn.restype = C.c_int
        fn.argtypes = [C.c_void_p]
        return int(fn(self._h))

    def stamps_pair(self, n_ctas):
        """diagnostics (UST_STAMPS set before the handle was created): the streaming CTAs' %globaltimer stamps of the last
        two calls, uint64 array [2 (call before the last, last call), n_ctas, 5 (entry, first tile landed, stream end,
        exit, SM id)]"""
        fn = self._lib.ust_debug_stamps_pair
        fn.argtypes = [C.c_void_p, C.c_void_p, C.c_int]
        out = np.zeros((2, n_ctas, 5), dtype=np.uint64)
        rc = fn(self._h, out.ctypes.data, n_ctas)
        if rc:
            raise UstError(rc, self.last_error())
        return out

    def stream(self):
        """cudaStream_t of the handle's own stream (as an int)."""
        return int(self._lib.ust_stream(self._h))

    def sync(self):
        rc = self._lib.ust_sync(self._h)
        if rc:
            raise UstError(rc, self.last_error())

    def apply_state(self, policy, soa, pods=None, want_outcome=True, out=None, check=False):
        """Host-array entry point (ust_apply_state). Returns (rc, next_state, actions, outcome, counters-dict)."""
        n = int(soa["state"].shape[0])
        if out is None:
            nxt = np.zeros(n, np.uint8)
            act = np.zeros(n, np.uint16)
            oc = np.full(n, 0xFF, np.uint8) if want_outcome else None
        else:
            nxt, act, oc = out
        cnt = abi.Counters()
        ps = None
        if pods is not None:
            off = np.ascontiguousarray(pods["pod_off"], dtype=np.int32)
            pf = np.ascontiguousarray(pods["pod_flags"], dtype=np.uint16)
            ps = abi.Pods(off.ctypes.data, pf.ctypes.data, int(pf.shape[0]))
        rc = self._lib.ust_apply_state(
            self._h, C.addressof(policy) if policy is not None else None, n, _p(soa["state"]), _p(soa["flags"]),
            _p(soa["pod_rev"]), _p(soa["ds_idx"]), int(soa["ds_rev"].shape[0]), _p(soa["ds_rev"]),
            C.addressof(ps) if ps is not None else None, _p(nxt), _p(act), _p(oc), C.addressof(cnt))
        if check and rc:
            raise UstError(rc, self.last_error())
        return rc, nxt, act, oc, cnt.as_dict()

    def apply_state_packed(self, policy, soa, want_outcome=True, out=None, check=False, packed=None):
        """ust_apply_state_packed: the same snapshot with pod_rev as uint16 and ds_idx as int8 on the host side.
        `packed` = (pod_rev16, ds_idx8) arrays to reuse (e.g. pinned); by default they are made from soa."""
        n = int(soa["state"].shape[0])
        if packed is None:
            assert n == 0 or (soa["pod_rev"].min() >= 0 and soa["pod_rev"].max() < 65536 and soa["ds_idx"].min() >= -128 and soa["ds_idx"].max() < 128)
            packed = (np.ascontiguousarray(soa["pod_rev"], dtype=np.uint16), np.ascontiguousarray(soa["ds_idx"], dtype=np.int8))
        if out is None:
            nxt = np.zeros(n, np.uint8)
            act = np.zeros(n, np.uint16)
            oc = np.full(n, 0xFF, np.uint8) if want_outcome else None
        else:
            nxt, act, oc = out
        cnt = abi.Counters()
        rc = self._lib.ust_apply_state_packed(
            self._h, C.addressof(policy) if policy is not None else None, n, _p(soa["state"]), _p(soa["flags"]), _p(packed[0]),
            _p(packed[1]), int(soa["ds_rev"].shape[0]), _p(soa["ds_rev"]), _p(nxt), _p(act), _p(oc), C.addressof(cnt))
        if check and rc:
            raise UstError(rc, self.last_error())
        return rc, nxt, act, oc, cnt.as_dict()

    def apply_state_delta(self, policy, n, idx, changed, ds_rev, want_outcome=True, out=None):
        """ust_apply_state_delta: overwrite nodes `idx` of the resident snapshot (n nodes) with `changed`
        (dict of state / flags / pod_rev / ds_idx arrays of len(idx)) and evaluate it again."""
        nodes, keep = _changed_nodes(idx, changed, ds_rev)  # `keep`: the arrays `nodes` points into, alive until the call returns
        if out is None:
            out = (np.zeros(n, np.uint8), np.zeros(n, np.uint16), np.full(n, 0xFF, np.uint8) if want_outcome else None)
        nxt, act, oc = out
        cnt = abi.Counters()
        rc = self._lib.ust_apply_state_delta(self._h, _ref(policy), *nodes, _p(nxt), _p(act), _p(oc), C.addressof(cnt))
        return rc, nxt, act, oc, cnt.as_dict()

    def _delta_sparse(self, fn, policy, structs, idx, changed, ds_rev, max_out, out, pods=False):
        """One sparse delta call fn(handle, policy, structs, changed nodes, outputs); `structs`: (ctypes struct or None,
        arrays behind it) pairs. Returns (rc, n_out, out_idx, out_next, out_actions[, out_outcome], counters-dict)."""
        nodes, keep = _changed_nodes(idx, changed, ds_rev)  # `keep`: the arrays `nodes` points into, alive until the call returns
        outputs, (out, n_out, cnt) = _sparse_outputs(max_out, out, pods)
        rc = fn(self._h, _ref(policy), *[_ref(s) for s, _ in structs], *nodes, *outputs)
        return (rc, int(n_out.value)) + out + (cnt.as_dict(),)

    def apply_state_delta_sparse(self, policy, idx, changed, ds_rev, max_out, out=None):
        """ust_apply_state_delta_sparse: like apply_state_delta, but only the outputs that differ from the previous call's
        come back. Returns (rc, n_out, out_idx, out_next, out_actions, counters-dict); the arrays hold n_out entries
        when n_out <= max_out."""
        return self._delta_sparse(self._lib.ust_apply_state_delta_sparse, policy, [], idx, changed, ds_rev, max_out, out)

    def apply_state_delta_splice(self, policy, splice, idx, changed, ds_rev, max_out, out=None):
        """ust_apply_state_delta_splice: apply_state_delta_sparse after a membership change of the resident snapshot.
        `splice` is None or a dict with remove_idx, insert_before and the inserted nodes' state / flags / pod_rev / ds_idx;
        `idx` indexes the spliced snapshot. Returns what apply_state_delta_sparse returns, in new-index order."""
        return self._delta_sparse(self._lib.ust_apply_state_delta_splice, policy, [_splice(splice)], idx, changed, ds_rev,
                                  max_out, out)

    def apply_state_delta_reorder(self, policy, reorder, idx, changed, ds_rev, max_out, out=None):
        """ust_apply_state_delta_reorder: apply_state_delta_sparse after the resident snapshot took a new node order.
        `reorder` is None or a dict with run_src, run_len and the inserted nodes' state / flags / pod_rev / ds_idx;
        `idx` indexes the reordered snapshot. Returns what apply_state_delta_sparse returns, in new-index order."""
        return self._delta_sparse(self._lib.ust_apply_state_delta_reorder, policy, [_reorder(reorder)], idx, changed, ds_rev,
                                  max_out, out)

    def apply_state_delta_pods(self, policy, lists, idx, changed, ds_rev, max_out, out=None):
        """ust_apply_state_delta_pods: apply_state_delta_sparse on the resident pod-list snapshot after replacing the pod lists
        of some nodes. `lists` is None or a dict with node_idx, pod_off and pod_flags. Returns (rc, n_out, out_idx, out_next,
        out_actions, out_outcome, counters-dict); the arrays hold n_out entries when n_out <= max_out."""
        return self._delta_sparse(self._lib.ust_apply_state_delta_pods, policy, [_pod_lists(lists)], idx, changed, ds_rev,
                                  max_out, out, pods=True)

    def apply_state_delta_pods_reorder(self, policy, reorder, lists, idx, changed, ds_rev, max_out, out=None):
        """ust_apply_state_delta_pods_reorder: apply_state_delta_pods after the resident pod-list snapshot took a new node
        order. `reorder` is None or a dict as for apply_state_delta_reorder, `lists` None or a dict as for
        apply_state_delta_pods; lists["node_idx"] and `idx` index the reordered snapshot, and every inserted node needs a
        list. Returns what apply_state_delta_pods returns, in new-index order."""
        return self._delta_sparse(self._lib.ust_apply_state_delta_pods_reorder, policy, [_reorder(reorder), _pod_lists(lists)],
                                  idx, changed, ds_rev, max_out, out, pods=True)

    def apply_state_clocked(self, policy, now, wait_timeout_seconds, start, soa, pods, out=None, clock_start=True):
        """ust_apply_state_clocked: apply_state with pod lists, the two timeouts derived on the device from `now` and the
        per-node start times `start` (int64). clock_start=False passes a NULL start (a rejection test); now=None a NULL
        clock. Returns (rc, next_state, actions, outcome, counters-dict)."""
        n = int(soa["state"].shape[0])
        nxt, act, oc = out if out is not None else (np.zeros(n, np.uint8), np.zeros(n, np.uint16), np.full(n, 0xFF, np.uint8))
        # `keep`: the start array `ck` points into, alive until the call returns
        ck, keep = _clock(now, wait_timeout_seconds, start if clock_start else None, None) if now is not None else (None, [])
        ps = None
        if pods is not None:
            off = np.ascontiguousarray(pods["pod_off"], dtype=np.int32)
            pf = np.ascontiguousarray(pods["pod_flags"], dtype=np.uint16)
            ps = abi.Pods(off.ctypes.data, pf.ctypes.data, int(pf.shape[0]))
        cnt = abi.Counters()
        rc = self._lib.ust_apply_state_clocked(
            self._h, _ref(policy), _ref(ck), n,
            _p(soa["state"]), _p(soa["flags"]), _p(soa["pod_rev"]), _p(soa["ds_idx"]), int(soa["ds_rev"].shape[0]),
            _p(soa["ds_rev"]), C.addressof(ps) if ps is not None else None, _p(nxt), _p(act), _p(oc), C.addressof(cnt))
        return rc, nxt, act, oc, cnt.as_dict()

    def apply_state_delta_pods_clocked(self, policy, now, wait_timeout_seconds, reorder, lists, idx, changed, start, ds_rev,
                                       max_out, insert_start=None, out=None, clock=True):
        """ust_apply_state_delta_pods_clocked: apply_state_delta_pods_reorder on a clocked snapshot. `start` holds the start
        times of the nodes at `idx`, `insert_start` those of the reorder's inserted nodes (None: NULL); clock=False passes a
        NULL clock. Returns what apply_state_delta_pods returns."""
        ck = _clock(now, wait_timeout_seconds, start, insert_start) if clock else (None, [])
        return self._delta_sparse(self._lib.ust_apply_state_delta_pods_clocked, policy, [ck, _reorder(reorder), _pod_lists(lists)],
                                  idx, changed, ds_rev, max_out, out, pods=True)

    def next_deadline(self, check=True):
        """ust_next_deadline: the time (int) at which a time-only clocked reconcile on the resident snapshot first returns
        something, or None when no deadline is pending (abi.NO_DEADLINE). check=False returns the code instead of raising:
        (rc, value)."""
        t = C.c_int64(0)
        rc = self._lib.ust_next_deadline(self._h, C.addressof(t))
        v = None if rc or t.value == abi.NO_DEADLINE else int(t.value)
        if not check:
            return rc, v
        if rc:
            raise UstError(rc, self.last_error())
        return v

    def fetch_outputs_pods(self, n):
        """ust_fetch_outputs_pods: (rc, next_state, actions, actuator_outcome) of the last call on the pod-list snapshot."""
        nxt = np.zeros(n, np.uint8)
        act = np.zeros(n, np.uint16)
        oc = np.zeros(n, np.uint8)
        rc = self._lib.ust_fetch_outputs_pods(self._h, _p(nxt), _p(act), _p(oc))
        return rc, nxt, act, oc

    def fetch_outputs(self, n):
        nxt = np.zeros(n, np.uint8)
        act = np.zeros(n, np.uint16)
        rc = self._lib.ust_fetch_outputs(self._h, _p(nxt), _p(act))
        return rc, nxt, act

    def simulate_rollout(self, policy, n, steps, want_final=True):
        """ust_simulate_rollout on the resident snapshot. Returns (rc, steps_done, [counters-dict per step], final dict)."""
        hist = (abi.Counters * max(steps, 1))()
        fin = {"state": np.zeros(n, np.uint8), "flags": np.zeros(n, np.uint32), "pod_rev": np.zeros(n, np.int32)} if want_final else None
        done = C.c_int32(0)
        rc = self._lib.ust_simulate_rollout(
            self._h, C.addressof(policy) if policy is not None else None, int(steps), C.addressof(hist),
            _p(fin["state"]) if fin else None, _p(fin["flags"]) if fin else None, _p(fin["pod_rev"]) if fin else None,
            C.addressof(done))
        return rc, int(done.value), [hist[k].as_dict() for k in range(steps)], fin

    def simulate_rollout_timed(self, policy, options, n, steps, want_final=True):
        """ust_simulate_rollout_timed on the resident snapshot (options: abi.SimOptions)."""
        hist = (abi.Counters * max(steps, 1))()
        fin = {"state": np.zeros(n, np.uint8), "flags": np.zeros(n, np.uint32), "pod_rev": np.zeros(n, np.int32)} if want_final else None
        done = C.c_int32(0)
        rc = self._lib.ust_simulate_rollout_timed(
            self._h, C.addressof(policy) if policy is not None else None, C.addressof(options), int(steps), C.addressof(hist),
            _p(fin["state"]) if fin else None, _p(fin["flags"]) if fin else None, _p(fin["pod_rev"]) if fin else None,
            C.addressof(done))
        return rc, int(done.value), [hist[k].as_dict() for k in range(steps)], fin

    def apply_state_device(self, policy, n, state, flags, pod_rev, ds_idx, n_ds, ds_rev, next_state, actions,
                           outcome=None, pods=None, counters=None, stream=None):
        """Device-pointer entry point (ust_apply_state_device). Arguments are raw device addresses."""
        ps = None
        if pods is not None:
            ps = abi.Pods(int(pods[0]), int(pods[1]), int(pods[2]))
        rc = self._lib.ust_apply_state_device(
            self._h, C.addressof(policy) if policy is not None else None, int(n), _p(state), _p(flags), _p(pod_rev),
            _p(ds_idx), int(n_ds), _p(ds_rev), C.addressof(ps) if ps is not None else None, _p(next_state),
            _p(actions), _p(outcome), _p(counters), _p(stream))
        if rc:
            raise UstError(rc, self.last_error())

    def build_state(self, state, ds_idx, ds_desired):
        cnt = abi.Counters()
        rc = self._lib.ust_build_state(self._h, int(state.shape[0]), _p(state), _p(ds_idx), int(ds_desired.shape[0]),
                                       _p(ds_desired), C.addressof(cnt))
        return rc, cnt.as_dict()

    def build_state_uids(self, state, owner_uid, ds_uid, ds_desired):
        """BuildState with the owner join on the device: owner_uid (n, 2) uint64, ds_uid (n_ds, 2) uint64.
        Returns (rc, ds_idx per pod, counters-dict)."""
        n = int(state.shape[0])
        owner_uid = np.ascontiguousarray(owner_uid, dtype=np.uint64).reshape(n, 2)
        ds_uid = np.ascontiguousarray(ds_uid, dtype=np.uint64).reshape(-1, 2)
        ds_desired = np.ascontiguousarray(ds_desired, dtype=np.int32)
        ds_idx = np.full(n, -3, np.int32)
        cnt = abi.Counters()
        rc = self._lib.ust_build_state_uids(self._h, n, _p(state), _p(owner_uid), int(ds_uid.shape[0]), _p(ds_uid),
                                            _p(ds_desired), _p(ds_idx), C.addressof(cnt))
        return rc, ds_idx, cnt.as_dict()

    def build_state_delta(self, reorder, idx, state, owner_uid, ds_uid, ds_desired, max_out, out=None):
        """ust_build_state_delta on the resident driver-pod list. `reorder` is None or a dict with run_src, run_len and the
        joined pods' state / owner_uid ((n_insert, 2) uint64; n_insert defaults to their count); `idx` (new indices), `state`
        and `owner_uid` are the overwritten pods. Returns (rc, n_out, out_idx, out_ds_idx, counters-dict); the arrays hold
        n_out entries when n_out <= max_out."""
        keep = []

        def arr(a, dt):
            a = np.ascontiguousarray(a, dtype=dt)
            keep.append(a)
            return a

        ro = None
        if reorder is not None:
            src = arr(reorder.get("run_src", np.zeros(0)), np.int64)
            ln = arr(reorder.get("run_len", np.zeros(0)), np.int64)
            ist = arr(reorder["state"], np.uint8) if "state" in reorder else None
            iuid = arr(reorder["owner_uid"], np.uint64) if "owner_uid" in reorder else None
            n_ins = reorder.get("n_insert", 0 if ist is None else int(ist.shape[0]))
            ro = abi.DriverPodReorder(int(src.shape[0]), _p(src), _p(ln), int(n_ins), _p(ist), _p(iuid))
        idx = arr(idx, np.int64)
        state = arr(state, np.uint8)
        owner_uid = arr(owner_uid, np.uint64)
        ds_uid = arr(ds_uid, np.uint64).reshape(-1, 2)
        ds_desired = arr(ds_desired, np.int32)
        if out is None:
            out = (np.zeros(max_out + 1, np.int64), np.zeros(max_out + 1, np.int32))
        n_out = C.c_int64(0)
        cnt = abi.Counters()
        rc = self._lib.ust_build_state_delta(
            self._h, C.addressof(ro) if ro is not None else None, int(idx.shape[0]), _p(idx), _p(state), _p(owner_uid),
            int(ds_uid.shape[0]), _p(ds_uid), _p(ds_desired), C.c_int64(int(max_out)), _p(out[0]), _p(out[1]),
            C.addressof(n_out), C.addressof(cnt))
        return rc, int(n_out.value), out[0], out[1], cnt.as_dict()

    def fetch_build_state(self, n):
        """ust_fetch_build_state: (rc, owner index per pod) of the resident driver-pod list of n pods."""
        ds_idx = np.full(n, -3, np.int32)
        rc = self._lib.ust_fetch_build_state(self._h, int(n), _p(ds_idx))
        return rc, ds_idx

    def comm_init(self, rank, world, unique_id_bytes):
        buf = (C.c_char * abi.UST_UNIQUE_ID_BYTES).from_buffer_copy(unique_id_bytes) if unique_id_bytes else None
        rc = self._lib.ust_comm_init(self._h, rank, world, buf)
        if rc:
            raise UstError(rc, self.last_error())

    def comm_set_mode(self, mode):
        rc = self._lib.ust_comm_set_mode(self._h, mode)
        if rc:
            raise UstError(rc, self.last_error())


def get_unique_id():
    buf = (C.c_char * abi.UST_UNIQUE_ID_BYTES)()
    rc = load().ust_get_unique_id(buf)
    if rc:
        raise UstError(rc, load().ust_create_error().decode())
    return bytes(buf)
