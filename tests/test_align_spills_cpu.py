"""Register-budget guard for the alignment kernel, on the CPU.

sparse_img_align_kernel<128,4> (the default variant) runs at 128 registers with 27 double accumulators live through
every Gauss-Newton pass, so a small change can push its pass loop back into local memory and slow every pass without
changing a result.  This compiles align_kernel.cu for sm_90a with the library's own flags plus -Xptxas -v and checks
the default variant's stack frame and spill bytes against the figures the kernel has today."""
import importlib.util
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "pl-svo_b200", "csrc")

# <128,4> as of this file's last change; lower them when the kernel gets leaner
MAX_STACK, MAX_SPILL_STORES, MAX_SPILL_LOADS = 320, 256, 544


def _build_module():
    spec = importlib.util.spec_from_file_location("plsvo_build_flags", os.path.join(ROOT, "pl-svo_b200", "build.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def _nvcc():
    return shutil.which("nvcc") or ("/usr/local/cuda/bin/nvcc" if os.path.exists("/usr/local/cuda/bin/nvcc") else None)


@pytest.mark.skipif(_nvcc() is None, reason="nvcc not found")
def test_default_variant_stays_within_its_local_memory_figures(tmp_path):
    flags = [f for f in _build_module().NVCC_FLAGS if f != "-shared"]
    cmd = [_nvcc()] + flags + ["-Xptxas", "-v", "-c", "-o", str(tmp_path / "align_kernel.o"), "align_kernel.cu"]
    res = subprocess.run(cmd, cwd=CSRC, capture_output=True, text=True, check=True)
    log = res.stdout + res.stderr
    m = re.search(r"Compiling entry function '\S*sparse_img_align_kernelILi128ELi4E\S*' for 'sm_90a'\s*\n"
                  r"(?:.*\n)*?\s*(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads\s*\n"
                  r"ptxas info\s*: Used (\d+) registers", log)
    assert m, "no ptxas report for sparse_img_align_kernel<128,4>:\n" + log[-4000:]
    stack, stores, loads, regs = map(int, m.groups())
    assert regs <= 128, f"<128,4> uses {regs} registers: it could no longer keep 4 CTAs per SM"
    assert stack <= MAX_STACK, f"<128,4> stack frame {stack} B > {MAX_STACK} B"
    assert stores <= MAX_SPILL_STORES, f"<128,4> spill stores {stores} B > {MAX_SPILL_STORES} B"
    assert loads <= MAX_SPILL_LOADS, f"<128,4> spill loads {loads} B > {MAX_SPILL_LOADS} B"
