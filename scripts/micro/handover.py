#!/usr/bin/env python
"""Call-to-call handover of the streaming kernel, per SM (DESIGN.md §3.3, §9).

Back-to-back ust_apply_state_device calls over rotating buffer sets (bench.py's protocol, C3 data and policy), then the
%globaltimer stamps of the last two calls' streaming CTAs with the SM each ran on. Per SM:

  gap = first tile of call k+1 landed on the SM - last stream end of call k on the SM

A positive gap is time the SM had nothing in flight between the calls; a negative one means call k+1's ring was
already filling while call k still streamed there.

  UST_LIB=build_variants/<name>.so python scripts/micro/handover.py --nodes 10000000 1000000 --steps 1000
"""
import argparse
import json
import os
import sys

os.environ.setdefault("UST_STAMPS", "1024")   # read by ust_create
ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402

import bench  # noqa: E402  (sys.path set-up, DeviceBench)


def per_sm_gaps(st):
    """st: [2, ctas, 5] from Handle.stamps_pair. Returns {sm: gap_ns} over SMs that ran a CTA of both calls."""
    prev, last = st[0].astype(np.int64), st[1].astype(np.int64)
    prev = prev[prev[:, 0] > 0]
    last = last[last[:, 0] > 0]
    end = {}
    for r in prev:
        end[int(r[4])] = max(end.get(int(r[4]), 0), int(r[2]))
    first = {}
    for r in last:
        sm = int(r[4])
        first[sm] = min(first.get(sm, 1 << 62), int(r[1]))
    return {sm: first[sm] - end[sm] for sm in end if sm in first}, prev, last


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--nodes", type=int, nargs="+", default=[10_000_000, 1_000_000])
    ap.add_argument("--steps", type=int, default=1000)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--sets", type=int, default=16)
    args = ap.parse_args()

    import torch
    from ust import abi, lib as ustlib, synth
    if not torch.cuda.is_available():
        raise SystemExit("handover.py needs a CUDA device")
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    sms = torch.cuda.get_device_properties(dev).multi_processor_count
    cfg, pol = synth.CONFIGS["C3"], synth.config_policy("C3")
    for n in args.nodes:
        h = ustlib.Handle(0)
        B = bench.DeviceBench(torch, None, ustlib, abi, dev, 1)
        bufs = B.upload(synth.make_nodes(n, cfg["seed"]), args.sets)
        bound = B.bind(h, pol, bufs)
        ms = B.time_steps(h, lambda i: bound[i % len(bound)], args.steps, args.warmup)
        st = h.stamps_pair(min(2 * sms, 1024))
        gaps, prev, last = per_sm_gaps(st)
        g = np.array(sorted(gaps.values()), dtype=np.float64) / 1e3
        t0 = prev[:, 0].min()
        rel = lambda a: (a - t0) / 1e3  # noqa: E731
        out = {
            "nodes": n, "us_per_call": 1e3 * ms / args.steps, "stream_ctas_per_sm": h.stream_ctas_per_sm(),
            "overlapped_calls": h.overlapped_calls(), "ctas": [int(prev.shape[0]), int(last.shape[0])],
            "sms_with_both_calls": int(g.size),
            "gap_us": {"min": float(g.min()), "median": float(np.median(g)), "max": float(g.max())} if g.size else None,
            "sms_where_next_lands_before_stream_end": int((g < 0).sum()),
            "call_k_us": {"entry_max": float(rel(prev[:, 0]).max()), "first_tile_median": float(np.median(rel(prev[:, 1]))),
                          "stream_end_median": float(np.median(rel(prev[:, 2]))), "stream_end_max": float(rel(prev[:, 2]).max()),
                          "exit_max": float(rel(prev[:, 3]).max())},
            "call_k1_us": {"entry_min": float(rel(last[:, 0]).min()), "entry_median": float(np.median(rel(last[:, 0]))),
                           "first_tile_min": float(rel(last[:, 1]).min()), "first_tile_median": float(np.median(rel(last[:, 1]))),
                           "stream_end_median": float(np.median(rel(last[:, 2])))},
        }
        print(json.dumps(out), flush=True)
        h.close()
        del bufs, bound
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
