#!/usr/bin/env python
"""Pre-flight of the GPU test tier on a machine without a GPU.

Runs the `-m gpu` test files against tests/hostmodel/libplsvo_hostmodel.so — the product's host code (plsvo_abi.cu, compiled
unchanged) on a model CUDA runtime — with every model kernel answered by the CPU oracle (PLSVO_FAKE_ORACLE).  What this
checks before GPU time is spent: the test files themselves (fixtures, generators, environment switches, assertions), the
Python mirror, and every host path the tests drive (uploads, chunking, the arrival gate, level derivation, frame chains,
the chained track call, the next-row entry points, the ATAN entry points).  What it cannot check: the CUDA kernels — here the oracle is compared
with the oracle, so a green pre-flight says nothing about parity.

Left out, with the reason:
  * test_gpu_shim.py, test_shim_next.py and the shim cases of test_structopt.py and test_gpu_atan.py: the C++ shim harness
    links libplsvo_b200.so directly;
  * depth-only features / bearings derived on the device: outside the oracle's inputs (the digest scenarios of
    tests/test_host_pipeline_cpu.py cover their host paths);
  * the 8 x 1024-pair parity campaign: generation alone takes tens of minutes on a few CPU cores (pass --campaign to run it).

usage: python tools/preflight_gpu_tests.py [--campaign] [pytest args / test files ...]"""
from __future__ import annotations

import importlib.util
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DEFAULT_FILES = ["test_gpu_abi_errors.py", "test_gpu_golden.py", "test_gpu_poseopt.py", "test_gpu_poseopt_cases.py", "test_gpu_track.py", "test_gpu_align.py",
                 "test_gpu_align_variants.py", "test_gpu_atan.py", "test_gpu_atan_cases.py", "test_pyramid.py", "test_gpu_pyramid_cases.py",
                 "test_align2d.py", "test_matcher.py", "test_gpu_direct_match_cases.py", "test_structopt.py", "test_gpu_structopt_cases.py", "test_depth_filter.py", "test_gpu_seed_schedules.py", "test_zz_gpu_chain.py", "test_zz_gpu_word_pitch.py"]
NEEDS_REAL_KERNELS = ("not depths_instead and not bearings_derived and not shim_optimize_structure_on_the_gpu"
                      " and not reference_typed_atan_frames_through_the_shim")


def main(argv):
    campaign = "--campaign" in argv
    argv = [a for a in argv if a != "--campaign"]
    spec = importlib.util.spec_from_file_location("hm_build", os.path.join(ROOT, "tests", "hostmodel", "build.py"))
    hm = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(hm)
    lib = hm.build()
    sys.path.insert(0, os.path.join(ROOT, "oracle"))
    import oracle_lib

    import oracle_atan

    oracle_lib.build()
    oracle_atan.build()  # the model's ATAN kernels find it next to libplsvo_oracle.so
    oracle = os.path.join(ROOT, "oracle", "libplsvo_oracle.so")
    env = dict(os.environ, PLSVO_LIB=lib, PLSVO_FAKE_ORACLE=oracle)
    files = [a for a in argv if a.endswith(".py")] or [os.path.join(ROOT, "tests", f) for f in DEFAULT_FILES]
    extra = [a for a in argv if not a.endswith(".py")]
    k = NEEDS_REAL_KERNELS + ("" if campaign else " and not campaign")
    cmd = [sys.executable, "-m", "pytest", *files, "-m", "gpu", "-q", "-p", "no:cacheprovider", "-k", k, *extra]
    print("[preflight]", " ".join(cmd), flush=True)
    return subprocess.call(cmd, env=env, cwd=ROOT)


if __name__ == "__main__":
    sys.exit(main(sys.argv[1:]))
