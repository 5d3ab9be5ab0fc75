#!/usr/bin/env python
"""Tuning: build libust.so variants with different streaming-kernel geometry into build_variants/ (git-ignored). Time
one on a GPU with UST_LIB=build_variants/<name>.so python bench.py --quick --steps 1000 (DESIGN.md §3.1 has the
H100 results). tests/test_gpu_variants.py builds every variant with build() and runs the GPU suite's geometry cases
against each one."""
import importlib.util
import os
import re
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = os.path.join(ROOT, "k8s-operator-libs_b200")
CSRC = os.path.join(PKG, "csrc")
OUT = os.path.join(ROOT, "build_variants")
SOURCES = ("ust_stream.cu", "ust_kernels.cu", "ust_api.cu")


def _load_build_module():
    spec = importlib.util.spec_from_file_location("ust_build", os.path.join(PKG, "build.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


NVCC_FLAGS = _load_build_module().NVCC_FLAGS   # the library's own flags: a variant differs only in its -D geometry
TWO_PER_SM = ["-DUST_STREAM_CTAS_PER_SM=2", "-DUST_HOT_REP=1"]   # two streaming CTAs (and a verification CTA) per SM
DEFAULT = "t3072w12s4"
VARIANTS = {
    DEFAULT: [],   # the default geometry: one streaming CTA per SM
    "t3072w8s4": ["-DUST_CONSUMER_WARPS=8"],
    # two streaming CTAs per SM: the next call's CTA fills its ring while the previous call's still streams
    "t1536w6s4": ["-DUST_TILE_NODES=1536", "-DUST_STAGES=4", "-DUST_CONSUMER_WARPS=6"] + TWO_PER_SM,
    "t3072w6s2": ["-DUST_TILE_NODES=3072", "-DUST_STAGES=2", "-DUST_CONSUMER_WARPS=6"] + TWO_PER_SM,
    "t1792w7s3": ["-DUST_TILE_NODES=1792", "-DUST_STAGES=3", "-DUST_CONSUMER_WARPS=7"] + TWO_PER_SM,
    "t1536w6s4g2": ["-DUST_TILE_NODES=1536", "-DUST_STAGES=4", "-DUST_CONSUMER_WARPS=6", "-DUST_STREAM_GRID_PER_SM=2"] + TWO_PER_SM,
    "t1536w6s4v256r64": ["-DUST_TILE_NODES=1536", "-DUST_STAGES=4", "-DUST_CONSUMER_WARPS=6", "-DUST_VERIFY_THREADS=256",
                         "-DUST_VERIFY_MAXREG=64"] + TWO_PER_SM,
}

# geometry a test needs to place its cases (macro of csrc/ust_dev.h -> key)
GEOMETRY_MACROS = {"UST_TILE_NODES": "tile_nodes", "UST_STREAM_CTAS_PER_SM": "ctas_per_sm",
                   "UST_STREAM_GRID_PER_SM": "grid_per_sm", "UST_VERIFY_THREADS": "verify_threads"}


def header_defaults():
    """The geometry macros' default values, as csrc/ust_dev.h defines them."""
    with open(os.path.join(CSRC, "ust_dev.h")) as f:
        txt = f.read()
    found = {m.group(1): int(m.group(2)) for m in re.finditer(r"#define\s+(UST_\w+)\s+(\d+)", txt)}
    return {key: found[macro] for macro, key in GEOMETRY_MACROS.items()}


def geometry(name):
    """Geometry of variant `name` from its -D flags, the header's defaults for the macros it does not set:
    {"tile_nodes", "ctas_per_sm", "grid_per_sm", "verify_threads"}."""
    g = header_defaults()
    for flag in VARIANTS[name]:
        m = re.fullmatch(r"-D(UST_\w+)=(\d+)", flag)
        if m and m.group(1) in GEOMETRY_MACROS:
            g[GEOMETRY_MACROS[m.group(1)]] = int(m.group(2))
    return g


def build(names, out_dir):
    """Compile the variants `names` into out_dir/<name>.so, all at once. Returns {name: path}; raises RuntimeError with
    the compiler's output when a variant does not build. Deletes nothing."""
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    os.makedirs(out_dir, exist_ok=True)
    procs = {}
    for name in names:
        out = os.path.join(out_dir, name + ".so")
        cmd = [nvcc] + NVCC_FLAGS + VARIANTS[name] + ["-shared", "-o", out] + [os.path.join(CSRC, s) for s in SOURCES] + ["-ldl"]
        procs[name] = (out, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True))
    failed = []
    for name, (out, p) in procs.items():
        log, _ = p.communicate()
        if p.returncode != 0:
            failed.append(f"variant {name} failed to build:\n{log}")
    if failed:
        raise RuntimeError("\n".join(failed))
    return {name: out for name, (out, _) in procs.items()}


def main():
    os.makedirs(OUT, exist_ok=True)
    for f in os.listdir(OUT):
        os.remove(os.path.join(OUT, f))
    want = sys.argv[1:] or list(VARIANTS)
    try:
        built = build(want, OUT)
    except RuntimeError as e:
        raise SystemExit(str(e))
    for name in built:
        print("built", name)


if __name__ == "__main__":
    main()
