#!/usr/bin/env python
"""Tuning: build libust.so variants with different streaming-kernel geometry into build_variants/ (git-ignored). Time
one on a GPU with UST_LIB=build_variants/<name>.so python bench.py --quick --steps 1000 (DESIGN.md §3.1 has the
H100 results)."""
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "k8s-operator-libs_b200", "csrc")
OUT = os.path.join(ROOT, "build_variants")
FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17", "-Xcompiler", "-fPIC",
         "-Xcompiler", "-fvisibility=hidden", "-Xcompiler", "-ffp-contract=off", "--fmad=false"]
TWO_PER_SM = ["-DUST_STREAM_CTAS_PER_SM=2", "-DUST_HOT_REP=1"]   # two streaming CTAs (and a verification CTA) per SM
VARIANTS = {
    "t3072w12s4": [],   # the default geometry: one streaming CTA per SM
    "t3072w8s4": ["-DUST_CONSUMER_WARPS=8"],
    # two streaming CTAs per SM: the next call's CTA fills its ring while the previous call's still streams
    "t1536w6s4": ["-DUST_TILE_NODES=1536", "-DUST_STAGES=4", "-DUST_CONSUMER_WARPS=6"] + TWO_PER_SM,
    "t3072w6s2": ["-DUST_TILE_NODES=3072", "-DUST_STAGES=2", "-DUST_CONSUMER_WARPS=6"] + TWO_PER_SM,
    "t1792w7s3": ["-DUST_TILE_NODES=1792", "-DUST_STAGES=3", "-DUST_CONSUMER_WARPS=7"] + TWO_PER_SM,
    "t1536w6s4g2": ["-DUST_TILE_NODES=1536", "-DUST_STAGES=4", "-DUST_CONSUMER_WARPS=6", "-DUST_STREAM_GRID_PER_SM=2"] + TWO_PER_SM,
    "t1536w6s4v256r64": ["-DUST_TILE_NODES=1536", "-DUST_STAGES=4", "-DUST_CONSUMER_WARPS=6", "-DUST_VERIFY_THREADS=256",
                         "-DUST_VERIFY_MAXREG=64"] + TWO_PER_SM,
}


def main():
    os.makedirs(OUT, exist_ok=True)
    for f in os.listdir(OUT):
        os.remove(os.path.join(OUT, f))
    want = sys.argv[1:] or list(VARIANTS)
    procs = []
    for name in want:
        out = os.path.join(OUT, name + ".so")
        cmd = ["/usr/local/cuda/bin/nvcc"] + FLAGS + VARIANTS[name] + ["-shared", "-o", out] + \
              [os.path.join(CSRC, s) for s in ("ust_stream.cu", "ust_kernels.cu", "ust_api.cu")] + ["-ldl"]
        procs.append((name, subprocess.Popen(cmd)))
    for name, p in procs:
        if p.wait() != 0:
            raise SystemExit(f"variant {name} failed to build")
        print("built", name)


if __name__ == "__main__":
    main()
