"""The build variants of scripts/build_variants.py (tile size, ring depth, consumer warps, streaming CTAs per SM, hot-byte
table replicas, grid per SM, verification-kernel width). Each one is compiled here, with or without a GPU: a variant
that loses its residency fails the streaming kernel's static_asserts. On a GPU, the geometry cases, the overlapped-call
scenario and the parity suite run in a child process against every variant but the default build (which the GPU suite
itself loads)."""
import importlib.util
import os
import re
import subprocess
import sys
import time

import pytest

import helpers


def _build_variants():
    spec = importlib.util.spec_from_file_location("build_variants", os.path.join(helpers.ROOT, "scripts", "build_variants.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


BV = _build_variants()
OTHERS = [name for name in BV.VARIANTS if name != BV.DEFAULT]
# per variant: the geometry cases, the overlapped calls whose parity sets the verify_done wait protects, and the parity
# suite without its full-size oracle runs
SUITE = ["tests/test_gpu_geometry.py", "tests/test_gpu_residency.py", "tests/test_gpu_parity.py",
         "-k", "not baseline_config and not c4_full_size"]
TIMEOUT_S = 900


@pytest.fixture(scope="module")
def variant_libs(tmp_path_factory):
    return BV.build(list(BV.VARIANTS), str(tmp_path_factory.mktemp("variants")))


def test_every_variant_builds(variant_libs):
    assert len(OTHERS) == len(BV.VARIANTS) - 1 > 0
    assert sorted(variant_libs) == sorted(BV.VARIANTS)
    assert all(os.path.getsize(p) > 0 for p in variant_libs.values())


def test_variant_geometry_follows_the_flags():
    defaults = BV.header_defaults()
    assert BV.geometry(BV.DEFAULT) == defaults == {"tile_nodes": 3072, "ctas_per_sm": 1, "grid_per_sm": 1, "verify_threads": 384}
    assert BV.geometry("t1792w7s3") == dict(defaults, tile_nodes=1792, ctas_per_sm=2)
    assert BV.geometry("t1536w6s4g2") == dict(defaults, tile_nodes=1536, ctas_per_sm=2, grid_per_sm=2)
    assert BV.geometry("t1536w6s4v256r64") == dict(defaults, tile_nodes=1536, ctas_per_sm=2, verify_threads=256)


@pytest.mark.gpu
@pytest.mark.parametrize("name", OTHERS)
def test_variant_passes_the_geometry_and_parity_suite(variant_libs, name):
    env = dict(os.environ, UST_LIB=variant_libs[name])
    for key, value in BV.geometry(name).items():
        env["UST_GEOM_" + key.upper()] = str(value)
    cmd = [sys.executable, "-m", "pytest", "-m", "gpu", "-q", "-p", "no:cacheprovider"] + SUITE
    t0 = time.monotonic()
    res = subprocess.run(cmd, cwd=helpers.ROOT, env=env, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True,
                         timeout=TIMEOUT_S)
    took = time.monotonic() - t0
    tail = res.stdout[-6000:]
    print(f"{name}: {took:.0f} s")
    assert res.returncode == 0, f"{name}: the suite failed ({took:.0f} s)\n{tail}"
    summary = res.stdout.strip().splitlines()[-1]
    passed = re.search(r"(\d+) passed", summary)
    assert passed and int(passed.group(1)) > 0 and "skipped" not in summary, f"{name}: nothing was tested\n{tail}"
