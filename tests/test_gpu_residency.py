"""Overlapped device calls whose predecessors' verification kernels run long (DESIGN.md §3.3)."""
import ctypes as C

import numpy as np
import pytest

import helpers
from helpers import abi
from ust import lib as ustlib

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def handle():
    h = ustlib.Handle(0)  # raises (never skips) when the extension or the device is missing
    yield h
    h.close()


def test_overlapped_calls_behind_long_repairs(handle):
    """Back-to-back device calls with outputs of their own, every one under a policy the previous call did not have:
    no call has a usable hint, so every verification kernel re-evaluates a third of the tiles while the next two calls'
    streaming kernels are already resident. Each call must still read its own speculation and tile counts (they live
    in the workspace set it shares with the call two before it): all outputs and counters are the oracle's."""
    import torch
    dev = torch.device("cuda:0")
    n = 2_000_003
    rng = np.random.default_rng(77)
    snaps, ins = [], []
    for k in range(2):
        soa, _ = helpers.random_soa(rng, n, all_states=True, wild=(k == 1))
        snaps.append(soa)
        ins.append({key: torch.from_numpy(v).to(dev) for key, v in soa.items()})
    pols = [abi.make_policy(max_parallel_upgrades=0, max_unavailable=f"{p}%") for p in (30, 80, 78, 95, 76, 90, 82, 99)]
    calls = len(pols)
    outs = [{"next": torch.empty(n, dtype=torch.uint8, device=dev), "actions": torch.empty(n, dtype=torch.int16, device=dev),
             "cnt": torch.zeros(C.sizeof(abi.Counters) // 8, dtype=torch.int64, device=dev)} for _ in range(calls)]
    torch.cuda.synchronize()
    before = handle.overlapped_calls()
    for c in range(calls):
        t, o = ins[c % 2], outs[c]
        handle.apply_state_device(pols[c], n, t["state"].data_ptr(), t["flags"].data_ptr(), t["pod_rev"].data_ptr(),
                                  t["ds_idx"].data_ptr(), len(snaps[c % 2]["ds_rev"]), t["ds_rev"].data_ptr(), o["next"].data_ptr(),
                                  o["actions"].data_ptr(), counters=o["cnt"].data_ptr())
    handle.sync()
    assert handle.overlapped_calls() - before >= calls // 2, "the calls did not overlap: nothing was tested"
    redone = [int(abi.Counters.from_buffer_copy(o["cnt"].cpu().numpy().tobytes()).reserved[0]) for o in outs]
    assert max(redone) > 0, "no verification kernel repaired anything: nothing ran long"
    for c in range(calls):
        ref = helpers.oracle_apply(pols[c], snaps[c % 2], variant=1)
        assert np.array_equal(outs[c]["next"].cpu().numpy(), ref[1]), c
        assert np.array_equal(outs[c]["actions"].cpu().numpy().view(np.uint16), ref[2]), c
        assert abi.Counters.from_buffer_copy(outs[c]["cnt"].cpu().numpy().tobytes()).as_dict() == ref[4], c
