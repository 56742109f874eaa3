"""CPU-side checks of the boundary: the library loads, exports every symbol the header declares,
struct layouts agree with the header, and without a GPU every call fails loudly (no CPU fallback)."""
import ctypes as C
import os
import re
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "include", "plsvo_b200.h")


def test_library_exports_every_declared_symbol(abi):
    lib = abi.load_library()
    text = open(HEADER).read()
    declared = set(re.findall(r"\b(plsvo_[a-z0-9_]+)\s*\(", text))
    declared -= {"plsvo_ctx"}
    assert declared, "no declarations parsed"
    typed = {name for name, _, _ in abi.ABI_SYMBOLS}
    assert declared == typed, f"header vs abi.py mismatch: {declared ^ typed}"
    for name in declared:
        assert hasattr(lib, name), name
    assert b"sm_90a" in lib.plsvo_version()


def test_struct_layout_matches_header(abi, tmp_path):
    """Compile a tiny C program against the header and compare sizeof/offsetof with ctypes."""
    src = tmp_path / "layout.c"
    src.write_text(
        '#include <stdio.h>\n#include <stddef.h>\n#include "plsvo_b200.h"\n'
        "int main(void){\n"
        'printf("%zu %zu %zu %zu %zu %zu %zu\\n", sizeof(plsvo_camera), sizeof(plsvo_align_params), sizeof(plsvo_align_batch),'
        " sizeof(plsvo_align_result), sizeof(plsvo_poseopt_params), sizeof(plsvo_poseopt_batch), sizeof(plsvo_poseopt_result));\n"
        'printf("%zu %zu %zu %zu\\n", offsetof(plsvo_align_batch, T_ref_w), offsetof(plsvo_align_batch, seg_valid),'
        " offsetof(plsvo_poseopt_batch, seg_valid), offsetof(plsvo_align_batch, img_stride));\n"
        'printf("%zu %zu %zu %zu %zu %zu %zu %zu %zu %zu %zu %zu\\n", sizeof(plsvo_pyramid_batch), sizeof(plsvo_pyramid_result),'
        " sizeof(plsvo_align2d_batch), sizeof(plsvo_align2d_result), sizeof(plsvo_align1d_batch), sizeof(plsvo_align1d_result),"
        " sizeof(plsvo_match_batch), sizeof(plsvo_match_result), sizeof(plsvo_structopt_batch), sizeof(plsvo_structopt_result),"
        " sizeof(plsvo_seed_batch), sizeof(plsvo_seed_result));\n"
        'printf("%zu %zu %zu %zu\\n", sizeof(plsvo_line_seed_batch), sizeof(plsvo_line_seed_result), offsetof(plsvo_line_seed_batch, ref_sf),'
        " offsetof(plsvo_line_seed_result, mu_e));\n"
        'printf("%zu %zu %zu %zu\\n", offsetof(plsvo_match_batch, px_cur), offsetof(plsvo_seed_batch, cam),'
        " offsetof(plsvo_seed_batch, sigma2), offsetof(plsvo_structopt_batch, seg_epos));\n"
        "return 0;}\n"
    )
    exe = tmp_path / "layout"
    subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)])
    out = subprocess.check_output([str(exe)]).decode().split()
    sizes = [int(x) for x in out[:7]]
    offs = [int(x) for x in out[7:11]]
    next_sizes = [int(x) for x in out[11:23]]
    line = [int(x) for x in out[23:27]]
    assert line == [C.sizeof(abi.LineSeedBatch), C.sizeof(abi.LineSeedResult), abi.LineSeedBatch.ref_sf.offset, abi.LineSeedResult.mu_e.offset]
    next_offs = [int(x) for x in out[27:]]
    assert next_sizes == [C.sizeof(t) for t in (abi.PyramidBatch, abi.PyramidResult, abi.Align2DBatch, abi.Align2DResult,
                                                 abi.Align1DBatch, abi.Align1DResult, abi.MatchBatch, abi.MatchResult,
                                                 abi.StructOptBatch, abi.StructOptResult, abi.SeedBatch, abi.SeedResult)]
    assert next_offs == [abi.MatchBatch.px_cur.offset, abi.SeedBatch.cam.offset, abi.SeedBatch.sigma2.offset,
                         abi.StructOptBatch.seg_epos.offset]
    assert sizes == [C.sizeof(t) for t in (abi.Camera, abi.AlignParams, abi.AlignBatch, abi.AlignResult,
                                            abi.PoseOptParams, abi.PoseOptBatch, abi.PoseOptResult)]
    assert offs == [abi.AlignBatch.T_ref_w.offset, abi.AlignBatch.seg_valid.offset,
                    abi.PoseOptBatch.seg_valid.offset, abi.AlignBatch.img_stride.offset]


def test_no_cpu_fallback_without_device(abi):
    import torch

    if torch.cuda.is_available():
        pytest.skip("a CUDA device is present")
    lib = abi.load_library()
    h = C.c_void_p()
    rc = lib.plsvo_ctx_create(0, None, C.byref(h))
    assert rc == abi.ERR_NO_DEVICE
    assert b"no CPU fallback" in lib.plsvo_last_error(None)
    assert not h.value


def test_product_never_touches_the_oracle():
    """The oracle is test infrastructure: nothing under pl-svo_b200/ may reference oracle/."""
    pkg = os.path.join(ROOT, "pl-svo_b200")
    for dirpath, _, files in os.walk(pkg):
        for f in files:
            if f.endswith((".py", ".cu", ".cuh", ".h", ".cpp", ".hpp")):
                text = open(os.path.join(dirpath, f), errors="ignore").read()
                assert "oracle_lib" not in text and "libplsvo_oracle" not in text and "plsvo_oracle_" not in text, f


def test_numa_helper_degrades_to_a_no_op_without_a_gpu():
    """plsvo_b200.numa: CPU-list parsing, and no affinity change when the GPU's topology cannot be read (this container)."""
    import os

    from plsvo_b200 import numa

    assert numa._parse_cpulist("0-3,8,10-11\n") == {0, 1, 2, 3, 8, 10, 11}
    assert numa._parse_cpulist("") == set()
    before = os.sched_getaffinity(0)
    saved = numa.bind_to_device(0)
    if saved is None:  # nothing readable: untouched
        assert os.sched_getaffinity(0) == before
    numa.restore(saved)
    assert os.sched_getaffinity(0) == before
    d = numa.describe(0)
    assert set(d) == {"pci_bus_id", "numa_node", "local_cpus", "process_cpus"}


def test_align_variant_list_matches_the_compiled_variants(abi):
    """abi.ALIGN_VARIANTS is what the parity tests iterate over: it must name every variant the library compiles and
    the planner accepts, no more and no fewer."""
    csrc = os.path.join(ROOT, "pl-svo_b200", "csrc")
    kernel = open(os.path.join(csrc, "align_kernel.cu")).read()
    compiled = re.search(r"#define PLSVO_ALIGN_VARIANTS\(X\)(.*)", kernel).group(1)
    plan = re.search(r"kAlignVariants\[\]\[2\] = \{(.*)\};", open(os.path.join(csrc, "plsvo_abi.cu")).read()).group(1)
    want = sorted(abi.ALIGN_VARIANTS)
    assert sorted((int(t), int(b)) for t, b in re.findall(r"X\((\d+), (\d+)\)", compiled)) == want
    assert sorted((int(t), int(b)) for t, b in re.findall(r"\{(\d+), (\d+)\}", plan)) == want
