"""Builds tests/hostmodel/_build/libplsvo_hostmodel_match_multicam.so: the host-pipeline model of atan_match_model.py (the
stock model plus the ATAN matching kernel's model) plus the model kernel of the per-image-camera findMatchDirect call
(fake_match_multicam.cpp).  Other entry points behave as in the stock model.  TEST INFRASTRUCTURE ONLY (fake_cuda.h)."""
from __future__ import annotations

import importlib.util
import os
import subprocess

HERE = os.path.dirname(os.path.abspath(__file__))
OUT = os.path.join(HERE, "_build", "libplsvo_hostmodel_match_multicam.so")


def _stock():
    spec = importlib.util.spec_from_file_location("plsvo_hostmodel_build", os.path.join(HERE, "build.py"))
    hm = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(hm)
    return hm


def build(force: bool = False, out: str | None = None, abi_source: str | None = None) -> str:
    """abi_source / out: build a variant from another copy of plsvo_abi.cu (the seeded-fault tests mutate one)."""
    hm = _stock()
    out = out or OUT
    sources = [abi_source or hm.SOURCES[0]] + hm.SOURCES[1:] + [os.path.join(HERE, f) for f in ("fake_atan_match.cpp", "fake_match_multicam.cpp")]
    deps = sources + hm.DEPS[len(hm.SOURCES):]
    if not force and os.path.exists(out) and all(os.path.getmtime(out) >= os.path.getmtime(d) for d in deps):
        return out
    os.makedirs(os.path.dirname(out), exist_ok=True)
    subprocess.run(["g++", "-std=c++17", "-O1", "-g", "-fPIC", "-shared", "-Wall", "-Wno-unused-function", "-I" + hm.cuda_include(),
                    "-I" + os.path.join(hm.ROOT, "pl-svo_b200", "csrc"), "-x", "c++", *sources, "-o", out + ".tmp", "-lpthread", "-ldl",
                    "-Wl,-Bsymbolic"], check=True)
    os.replace(out + ".tmp", out)
    return out


if __name__ == "__main__":
    print(build(force=True))
