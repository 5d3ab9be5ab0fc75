"""Geometry edges of the streaming kernel against the oracle, for whichever libust.so is loaded (UST_LIB selects a build
variant of scripts/build_variants.py; tests/test_gpu_variants.py runs this module against each one).

The library tiles a snapshot by pick_tile_nodes / pick_grid / pick_static_rounds (ust_api.cu), which are restated
below. The cases sit where that tiling branches: the sizes where the tile size switches, ragged last tiles taken by
ticket, the static / ticket split, the ±64-tile window in which the verification kernel looks for the slot-budget cut
around the previous call's, aborts on tile edges, every instantiation of the streaming kernel, and every hot byte at
every node position of a lane. Every result is bit-exact against the oracle. Run on an H100:
python -m pytest tests/test_gpu_geometry.py -m gpu"""
import ctypes as C
import importlib.util
import os

import numpy as np
import pytest

import helpers
from helpers import abi
from ust import lib as ustlib

pytestmark = pytest.mark.gpu


def _build_variants():
    spec = importlib.util.spec_from_file_location("build_variants", os.path.join(helpers.ROOT, "scripts", "build_variants.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


BV = _build_variants()
# UST_GEOM_<KEY> (set together with UST_LIB) describes the loaded variant; unset, the default build's geometry
GEOM = {k: int(os.environ.get("UST_GEOM_" + k.upper(), v)) for k, v in BV.geometry(BV.DEFAULT).items()}
TILE = GEOM["tile_nodes"]
STATIC_PCT = 75          # ust_handle::static_pct (UST_STATIC_PCT unset)
DS_SMEM_MAX = 1024       # UST_DS_SMEM_MAX (ust_dev.h): DaemonSet tables up to this size live in shared memory
ORACLE_V0_MAX = 300_000  # the reference-shaped oracle takes seconds beyond this


# ---- the library's tiling, restated (ust_api.cu) -------------------------------------------------------------------

def pick_tile_nodes(n, grid_max):
    tn = TILE
    while tn > 128 and n // tn < grid_max:
        tn = max((tn // 2) & ~127, 128)
    return tn


def pick_grid(tiles, grid_max):
    return max(min(tiles, grid_max), 1)


def pick_static_rounds(tiles, grid):
    rounds = tiles // grid
    r = rounds * STATIC_PCT // 100
    if rounds - r < 2:
        r = rounds - 2
    if r < 1 and rounds >= 1:
        r = 1
    return max(r, 0)


def tile_chain():
    """Every tile size the library picks, largest first."""
    chain = [TILE]
    while chain[-1] > 128:
        chain.append(max((chain[-1] // 2) & ~127, 128))
    return chain


CHAIN = tile_chain()


@pytest.fixture(scope="module")
def handle():
    h = ustlib.Handle(0)  # raises (never skips) when the extension or the device is missing
    yield h
    h.close()


@pytest.fixture(scope="module")
def grid_max():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count * GEOM["grid_per_sm"]


# ---- calls and checks ----------------------------------------------------------------------------------------------

def host_apply(handle, pol, soa, pods=None, outcome=True):
    """ust_apply_state; returns the result tuple of helpers.oracle_apply and the tiles the verification redid."""
    n = int(soa["state"].shape[0])
    nxt, act = np.zeros(n, np.uint8), np.zeros(n, np.uint16)
    oc = np.full(n, 0xFF, np.uint8) if outcome else None
    cnt = abi.Counters()
    ps, keep = helpers.pods_struct(pods)
    rc = ustlib.load().ust_apply_state(
        handle._h, C.addressof(pol), n, soa["state"].ctypes.data, soa["flags"].ctypes.data, soa["pod_rev"].ctypes.data,
        soa["ds_idx"].ctypes.data, int(soa["ds_rev"].shape[0]), soa["ds_rev"].ctypes.data,
        C.addressof(ps) if ps is not None else None, nxt.ctypes.data, act.ctypes.data,
        oc.ctypes.data if oc is not None else None, C.addressof(cnt))
    del keep
    return (rc, nxt, act, oc, cnt.as_dict()), int(cnt.reserved[0])


class DeviceCall:
    """One ust_apply_state_device call on inputs and outputs of its own (enqueue, then result() after a sync)."""

    def __init__(self, handle, pol, soa, outcome=True):
        import torch
        dev = torch.device("cuda:0")
        n = int(soa["state"].shape[0])
        self.t = {k: torch.from_numpy(np.ascontiguousarray(v)).to(dev) for k, v in soa.items()}
        self.nxt = torch.empty(n, dtype=torch.uint8, device=dev)
        self.act = torch.empty(n, dtype=torch.int16, device=dev)
        self.oc = torch.empty(n, dtype=torch.uint8, device=dev) if outcome else None
        self.cnt = torch.zeros(C.sizeof(abi.Counters) // 8, dtype=torch.int64, device=dev)
        t = self.t
        handle.apply_state_device(pol, n, t["state"].data_ptr(), t["flags"].data_ptr(), t["pod_rev"].data_ptr(),
                                  t["ds_idx"].data_ptr(), int(soa["ds_rev"].shape[0]), t["ds_rev"].data_ptr(),
                                  self.nxt.data_ptr(), self.act.data_ptr(),
                                  outcome=self.oc.data_ptr() if outcome else None, counters=self.cnt.data_ptr())

    def result(self):
        c = abi.Counters.from_buffer_copy(self.cnt.cpu().numpy().tobytes())
        d = c.as_dict()
        oc = self.oc.cpu().numpy() if self.oc is not None else None
        return (d["error_code"], self.nxt.cpu().numpy(), self.act.cpu().numpy().view(np.uint16), oc, d), int(c.reserved[0])


def device_apply(handle, pol, soa, outcome=True):
    call = DeviceCall(handle, pol, soa, outcome)
    handle.sync()
    return call.result()


def apply(handle, path, pol, soa, pods=None, outcome=True):
    if path == "host":
        return host_apply(handle, pol, soa, pods, outcome)
    assert pods is None
    return device_apply(handle, pol, soa, outcome)


def oracle(pol, soa, pods=None):
    """The oracle's answer; below ORACLE_V0_MAX nodes the SoA oracle and the reference-shaped one must agree."""
    ref = helpers.oracle_apply(pol, soa, pods, variant=1)
    if soa["state"].shape[0] <= ORACLE_V0_MAX:
        helpers.assert_same(helpers.oracle_apply(pol, soa, pods, variant=0), ref, "oracle variants")
    return ref


def check(got, pol, soa, what, pods=None, ref=None):
    helpers.assert_same(got, ref if ref is not None else oracle(pol, soa, pods), what)


def slot_snapshot(rng, n, frac=0.5):
    """Random flags, DaemonSet columns and availability bits; states upgrade-required (a share `frac` of the nodes),
    upgrade-done or unknown only. Nothing is in progress, so under a policy with maxParallelUpgrades = B and a nil
    maxUnavailable the slot budget is exactly B, and it cuts after the B-th candidate in node order."""
    soa, _ = helpers.random_soa(rng, n, wild=True)
    avail_bits = soa["state"] & np.uint8(abi.UST_HOT_NOT_READY | abi.UST_HOT_UNSCHEDULABLE)
    done = abi.STATE_CODE["upgrade-done"]
    code = np.where(rng.random(n) < frac, 1, np.where(rng.random(n) < 0.5, done, 0)).astype(np.uint8)
    skip = np.where((code == 1) & (rng.random(n) < 0.1), abi.UST_HOT_SKIP, 0).astype(np.uint8)
    soa["state"] = (code | avail_bits | skip).astype(np.uint8)
    return soa


def candidates(soa):
    return int(np.sum(((soa["state"] & 15) == 1) & ((soa["state"] & abi.UST_HOT_SKIP) == 0)))


def with_abort_at(soa, i):
    """A copy of `soa` whose node i is upgrade-done with a pod whose revision hash cannot be read (an abort)."""
    s = {k: v.copy() for k, v in soa.items()}
    s["state"][i] = abi.STATE_CODE["upgrade-done"] | abi.UST_HOT_REVISION_HASH_ERROR
    s["flags"][i] &= ~np.uint32(abi.UST_F_POD_ORPHANED)
    return s


# ---- the restatement itself ------------------------------------------------------------------------------------------

def test_tile_chain_and_static_rounds():
    expected = {3072: [3072, 1536, 768, 384, 128], 1536: [1536, 768, 384, 128], 1792: [1792, 896, 384, 128]}
    assert CHAIN == expected[TILE]
    assert all(tn % 128 == 0 for tn in CHAIN)
    # the branches of pick_static_rounds: one round (G, G+1 tiles), two (2G, 2G+1), three (3G+1), many
    g = 132
    assert [pick_static_rounds(t, g) for t in (g, g + 1, 2 * g, 2 * g + 1, 3 * g + 1, 4 * g, 8 * g)] == [1, 1, 1, 1, 1, 2, 6]
    assert pick_static_rounds(5, 5) == 1 and pick_static_rounds(0, 1) == 0


def test_the_build_holds_its_streaming_ctas(handle):
    """A build with two streaming CTAs per SM exists so that the next call's CTA is resident while this call's streams:
    the occupancy the library finds must be the one the build was made for, or none of that is exercised here."""
    assert handle.stream_ctas_per_sm() == GEOM["ctas_per_sm"]


# ---- a. the sizes where the tile size switches -----------------------------------------------------------------------

@pytest.mark.parametrize("level", range(len(CHAIN)))
@pytest.mark.parametrize("delta", [-1, 0, 1])
def test_tile_size_switch(handle, grid_max, level, delta):
    """n = G * tn + delta for every tile size tn of the chain: one node fewer than G full tiles takes the next smaller
    tile size. A random snapshot under a random policy (host path), a slot budget that cuts in the middle (device path),
    and an abort, whose redone-tile count is the library's tile count: it must be the restatement's."""
    tn = CHAIN[level]
    n = grid_max * tn + delta
    rng = np.random.default_rng(100 * level + delta + 7)
    soa, _ = helpers.random_soa(rng, n, n_ds=3, p_err=2e-5)
    pol = helpers.random_policy(rng)
    check(apply(handle, "host", pol, soa)[0], pol, soa, f"n={n} random")
    soa = slot_snapshot(rng, n)
    pol = abi.make_policy(max_parallel_upgrades=candidates(soa) // 2)
    check(apply(handle, "device", pol, soa)[0], pol, soa, f"n={n} cut")
    tn_lib = pick_tile_nodes(n, grid_max)
    assert tn_lib == (tn if delta >= 0 or level + 1 == len(CHAIN) else CHAIN[level + 1])
    aborting = with_abort_at(soa, int(rng.integers(0, n)))
    got, redone = apply(handle, "device", pol, aborting)
    check(got, pol, aborting, f"n={n} abort")
    assert got[0] == abi.K["UST_ERR_REVISION_HASH"]
    assert redone == -(-n // tn_lib), ("tiles of the call", redone, n, tn_lib)


# ---- b. ragged last tiles, taken by ticket ---------------------------------------------------------------------------

@pytest.mark.parametrize("r", [0, 1, 15, 16, 17, 127, 128, 129, "tn-1"])
@pytest.mark.parametrize("path", ["host", "device"])
def test_ragged_tail(handle, grid_max, r, path):
    """n = k * tn + r with more than 2G tiles: the first round of tiles is static, the rest - the ragged last tile among
    them - go by ticket. The host path cuts the snapshot into pipelined segments (n >= 2^19 nodes) of their own grid."""
    tn = TILE
    r = tn - 1 if r == "tn-1" else r
    k = 2 * grid_max + 1
    n = k * tn + r
    assert pick_tile_nodes(n, grid_max) == tn and -(-n // tn) > 2 * grid_max
    rng = np.random.default_rng(r + 31 * (path == "host"))
    soa = slot_snapshot(rng, n)
    soa["state"][-40:] = np.where(rng.random(40) < 0.5, 1, soa["state"][-40:]).astype(np.uint8)
    pol = abi.make_policy(max_parallel_upgrades=candidates(soa) - 7)   # the budget cuts among the last 40 nodes
    check(apply(handle, path, pol, soa)[0], pol, soa, f"n={n} cut in the last tile")
    soa2, _ = helpers.random_soa(rng, n, n_ds=4, p_err=1e-6)
    pol2 = helpers.random_policy(rng)
    check(apply(handle, path, pol2, soa2)[0], pol2, soa2, f"n={n} random")


# ---- c. the static / ticket split ------------------------------------------------------------------------------------

@pytest.mark.parametrize("tiles", ["G", "G+1", "2G", "2G+1", "3G+1"])
@pytest.mark.parametrize("path", ["host", "device"])
def test_static_and_ticket_rounds(handle, grid_max, tiles, path):
    """Tile counts on the branches of pick_static_rounds, with the budget cutting a third of the way in."""
    G = grid_max
    nt = {"G": G, "G+1": G + 1, "2G": 2 * G, "2G+1": 2 * G + 1, "3G+1": 3 * G + 1}[tiles]
    tn = TILE
    n = nt * tn if nt == G else (nt - 1) * tn + tn // 3 + 5
    assert pick_tile_nodes(n, G) == tn and -(-n // tn) == nt
    assert pick_grid(nt, G) == G
    rng = np.random.default_rng(nt + 1000 * (path == "host"))
    soa = slot_snapshot(rng, n)
    pol = abi.make_policy(max_parallel_upgrades=candidates(soa) // 3)
    check(apply(handle, path, pol, soa)[0], pol, soa, f"tiles={nt}")
    soa2, _ = helpers.random_soa(rng, n, n_ds=2, p_err=1e-6, wild=True)
    pol2 = helpers.random_policy(rng)
    check(apply(handle, path, pol2, soa2)[0], pol2, soa2, f"tiles={nt} random")


# ---- d. the window search for the slot-budget cut --------------------------------------------------------------------

WINDOW_TILES = 300
WINDOW_BUDGET = 200


def window_sequence(nT):
    """(cut tile, slots left in it) of consecutive calls; "last": the cut tile's candidates - 1; "all": the budget
    covers every candidate (no cut); "zero": the budget is 0. Each comment gives the move against the previous cut."""
    mid = nT // 2
    return [
        (mid, 0),              # no hint: the policy default (nobody gets a slot) is checked by a full search
        (mid, 0),              # the same tile, no slot left in it
        (mid, 1),              # the same tile, one slot left
        (mid + 1, "last"),     # +1
        (mid, 1),              # -1
        (mid - 64, 0),         # -64: the window's first tile
        (mid - 129, "last"),   # -65: outside the window; now within 64 tiles of the start
        (mid - 66, 1),         # +63: the window's last tile, the window clipped at tile 0
        (mid - 130, 0),        # -64
        (0, None),             # tile 0 (slots left: the whole budget)
        (63, 1),               # a hint of tile 0 opens no window
        (127, "last"),         # +64: outside the window
        (192, 0),              # +65
        (255, 1),              # +63
        (nT - 30, "last"),     # +15: now within 64 tiles of the end
        (nT - 1, 1),           # the ragged last tile, the window clipped at the end
        (nT - 1, "last"),      # the same tile
        (nT - 65, 0),          # -64
        (nT - 1, 0),           # +64: outside the window
        (nT, "all"),           # no cut
        (nT - 20, 1),          # from a hint past the last tile
        (0, "zero"),           # budget 0
        (mid, 1),              # from the cut of a zero budget
    ]


def window_snapshot(rng, base, tn, n, nT, cut, slots):
    """`base` with upgrade candidates laid out so that a budget of WINDOW_BUDGET cuts in tile `cut` with `slots` left.
    Returns (snapshot, cut, slots left) as the verification kernel must find them."""
    B = WINDOW_BUDGET
    cap = [tn] * (nT - 1) + [n - (nT - 1) * tn]
    counts = np.zeros(nT, np.int64)

    def spread(lo, hi, total):
        if hi > lo:
            counts[lo:hi] = total // (hi - lo)
            counts[lo + rng.permutation(hi - lo)[:total % (hi - lo)]] += 1
        else:
            assert total == 0

    in_progress = 0
    if slots == "all":
        spread(0, nT, B - 3)
        cut, left = nT, 0
    elif slots == "zero":
        counts[:] = rng.integers(0, 6, nT)
        in_progress = B   # B nodes in cordon-required: nothing is available
        cut, left = 0, 0
    else:
        if cut == 0:
            left, c_cut = B, B + 2
        else:
            left = 3 if slots == "last" else slots
            c_cut = 4 if slots == "last" else 3
        spread(0, cut, B - left)
        counts[cut] = c_cut
        counts[cut + 1:] = rng.integers(0, 6, nT - cut - 1)
    hot = base["state"].copy()
    for t in range(nT):
        pos = t * tn + rng.choice(cap[t], int(counts[t]), replace=False)
        hot[pos] = (hot[pos] & np.uint8(abi.UST_HOT_NOT_READY | abi.UST_HOT_UNSCHEDULABLE)) | 1
    if in_progress:
        free = np.flatnonzero((hot & 15) != 1)
        pick = rng.choice(free, in_progress, replace=False)
        hot[pick] = (hot[pick] & 0xF0) | abi.STATE_CODE["cordon-required"]
    soa = dict(base)
    soa["state"] = hot
    assert candidates(soa) == int(counts.sum())
    return soa, cut, left


def expected_redone(sc, cut, left, nT, lb, lc):
    """Tiles the verification kernel re-evaluates when the call speculated the cut at tile `sc` (decide(), ust_common.cuh),
    and the hint the call leaves for the next one."""
    need = (lb > 0) if sc <= 0 else ((lb < lc) if sc >= nT else True)
    if not need:
        return 0, sc
    if sc <= cut:
        lo, hi = sc, (cut if cut < nT and left > 0 else cut - 1)
    else:
        lo, hi = cut, sc - 1
    return max(hi - lo + 1, 0), cut


def test_window_search_edges(grid_max):
    """The verification kernel looks for the slot-budget cut in a window of 128 tile counts (-64 .. +63) around the
    cut the previous call of the same size and policy found, and searches every tile when the cut is not in it. The
    data alone moves the cut between calls (the policy, and with it the hint signature, stays): onto the window's
    edges and just past them, the window clipped at either end of the array, tile 0, the ragged last tile, no cut and
    a zero budget, with 0, 1 and all but one of the cut tile's candidates left. Host calls first (each one's hint is the
    previous call's cut: the redone-tile count shows that), then the same snapshots once more as back-to-back device
    calls, which overlap and read the hint of the call before the previous one. Every call is checked bit for bit."""
    import torch
    tn, nT = TILE, WINDOW_TILES
    n = (nT - 1) * tn + tn // 2 + 5
    assert pick_tile_nodes(n, grid_max) == tn and -(-n // tn) == nT
    rng = np.random.default_rng(2024)
    base = slot_snapshot(rng, n, frac=0.0)
    skipped = rng.random(n) < 0.02   # upgrade-required but skipped: in the bucket, never a candidate
    base["state"] = np.where(skipped, (base["state"] & 0xF0) | 1 | abi.UST_HOT_SKIP, base["state"]).astype(np.uint8)
    pol = abi.make_policy(max_parallel_upgrades=WINDOW_BUDGET)
    handle = ustlib.Handle(0)   # a fresh workspace: no hint of an earlier call with this signature
    try:
        snaps, refs, sc = [], [], 0
        for k, (cut, slots) in enumerate(window_sequence(nT)):
            soa, cut, left = window_snapshot(rng, base, tn, n, nT, cut, slots)
            ref = helpers.oracle_apply(pol, soa, variant=1)
            got, redone = host_apply(handle, pol, soa)
            what = f"call {k}: cut {cut} slots left {left}, previous cut {sc}"
            check(got, pol, soa, what, ref=ref)
            lb = max(WINDOW_BUDGET - ref[4]["in_progress"], 0)
            want, sc = expected_redone(sc, cut, left, nT, lb, candidates(soa))
            assert redone == want, (what, "redone tiles", redone, want)
            snaps.append(soa)
            refs.append(ref)
        torch.cuda.synchronize()
        before = handle.overlapped_calls()
        calls = [DeviceCall(handle, pol, soa) for soa in snaps]
        handle.sync()
        assert handle.overlapped_calls() - before >= len(calls) // 2, "the device calls did not overlap"
        for k, call in enumerate(calls):
            check(call.result()[0], pol, snaps[k], f"device call {k}", ref=refs[k])
    finally:
        handle.close()


# ---- e. aborts on tile edges ---------------------------------------------------------------------------------------

@pytest.mark.parametrize("tile_size", ["largest", "smallest"])
@pytest.mark.parametrize("where", ["first node of a tile", "last node of the tile before", "last node"])
@pytest.mark.parametrize("path", ["host", "device"])
def test_abort_on_tile_edges(handle, grid_max, tile_size, where, path):
    """A revision-hash error node on a tile edge aborts the call, and the verification kernel re-evaluates every tile
    step by step: the outputs up to the abort, the error index and the counters are the oracle's."""
    tn = CHAIN[0] if tile_size == "largest" else CHAIN[-1]
    n = (grid_max + 4) * tn + tn // 3 + 1
    assert pick_tile_nodes(n, grid_max) == tn
    j = grid_max + 1   # a tile taken by ticket
    i = {"first node of a tile": j * tn, "last node of the tile before": j * tn - 1, "last node": n - 1}[where]
    rng = np.random.default_rng(i)
    soa = slot_snapshot(rng, n)
    pol = abi.make_policy(max_parallel_upgrades=candidates(soa) // 2)
    soa = with_abort_at(soa, i)
    got, redone = apply(handle, path, pol, soa)
    check(got, pol, soa, f"abort at {i}")
    assert got[0] == abi.K["UST_ERR_REVISION_HASH"] and got[4]["error_index"] == i
    assert redone == -(-n // tn)


# ---- f. every instantiation of the streaming kernel ------------------------------------------------------------------

@pytest.mark.parametrize("n_ds", [1, DS_SMEM_MAX, DS_SMEM_MAX + 1])
@pytest.mark.parametrize("outcome", [False, True])
@pytest.mark.parametrize("pods", [False, True])
def test_every_stream_kernel_instantiation(handle, grid_max, n_ds, outcome, pods):
    """DaemonSet table in shared memory or not (n_ds <= UST_DS_SMEM_MAX), actuator_outcome written or not, pod lists
    or not: the eight launch_variant instantiations, at a ragged size."""
    n = (grid_max + 2) * TILE + 77
    rng = np.random.default_rng(n_ds + 10 * outcome + 100 * pods)
    soa, pl = helpers.random_soa(rng, n, n_ds=n_ds, with_pods=pods)
    pol = abi.make_policy(max_parallel_upgrades=0, max_unavailable="100%", pod_deletion_enabled=True, pod_deletion={"force": True},
                          validation_enabled=True, drain={"enable": True}, wait_for_completion={"podSelector": "app=x", "timeoutSeconds": 30},
                          evaluate_actuators=pods)
    got = host_apply(handle, pol, soa, pl, outcome)[0]
    assert got[0] == 0
    check(got, pol, soa, f"n_ds={n_ds} outcome={outcome} pods={pods}", pods=pl)


# ---- g. every hot byte at every node position of a lane ------------------------------------------------------------

@pytest.mark.parametrize("path", ["host", "device"])
def test_every_hot_byte_at_every_lane_position(handle, grid_max, path):
    """A lane evaluates 4 consecutive nodes, each by a table lookup at an offset shifted out of its byte of the 32-bit
    hot word. Every value 0..255 of the hot byte occurs at each of the four positions (full tiles and the ragged last
    one), with random and reserved flag bits, under policies that do not abort: the revision-hash error bit is set
    only where it does not abort (orphaned driver pods)."""
    n = (grid_max + 1) * TILE + 300
    rng = np.random.default_rng(255 + (path == "device"))
    soa, _ = helpers.random_soa(rng, n, n_ds=3, wild=True)
    u = np.arange(n) // 4
    p = np.arange(n) % 4
    # within each block of 256 consecutive 4-node units, the byte at position p runs through all 256 values
    soa["state"] = ((37 * u + 59 * p + 11 * (u // 256)) % 256).astype(np.uint8)
    code = soa["state"] & 15
    aborting = ((soa["state"] & abi.UST_HOT_REVISION_HASH_ERROR) != 0) & np.isin(code, [0, 8, 11, 12])
    soa["flags"] = np.where(aborting, soa["flags"] | np.uint32(abi.UST_F_POD_ORPHANED), soa["flags"]).astype(np.uint32)
    assert all(len(np.unique(soa["state"][p == q])) == 256 for q in range(4))
    for pol in (abi.make_policy(max_parallel_upgrades=0),
                abi.make_policy(max_parallel_upgrades=0, max_unavailable="100%", pod_deletion_enabled=True, pod_deletion={},
                                drain={"enable": True, "force": True}, wait_for_completion={"podSelector": "app=x"}),
                abi.make_policy(max_parallel_upgrades=5, validation_enabled=True, use_maintenance_operator=True)):
        got = apply(handle, path, pol, soa)[0]
        assert got[0] == 0
        check(got, pol, soa, "hot bytes")
