"""The host side of the C ABI, exercised without a GPU.

`pl-svo_b200/csrc/plsvo_abi.cu` is pure host code (buffer sizing, upload planning, the small-batch staging block, the
arrival-gated stream, device-side pyramid derivation, the frame-chain layout, error exits).  On a
GPU box it is covered by the `-m gpu` parity tests; here it is compiled UNCHANGED as C++ and linked against a
single-threaded model of the CUDA runtime (tests/hostmodel/fake_cudart.cpp: FIFO streams that run as lazily — or, in a
second pass, as eagerly — as events and the arrival gate allow, poisoned and bounds-checked "device" memory) and against
model kernels that digest every byte the real kernels would read (tests/hostmodel/fake_kernels.cpp).  The scenarios
(tests/hostmodel/scenarios.py) drive the product's own Python mirror through that library and compare the digests with
the same digests computed in NumPy from the caller's arrays: whichever host path a call takes, the kernel must be shown
exactly the caller's bytes, every buffer must be large enough, every dependency must be expressed, and no copy from the
caller's arrays may be pending when a call returns.

The second half seeds faults into a copy of plsvo_abi.cu (a dropped wait for the arrival of the copies, an undersized frame
stack, a frame that is never shipped, an arrival flag raised too early, a missing drain on an error exit, pyramid levels
off a 16-byte boundary) and requires the model to notice each of them.

Nothing here is a parity statement about the CUDA kernels — that is what the `-m gpu` tests are for."""
import importlib.util
import json
import os
import subprocess
import sys

import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
HM = os.path.join(HERE, "hostmodel")
ABI_SOURCE = os.path.join(os.path.dirname(HERE), "pl-svo_b200", "csrc", "plsvo_abi.cu")

SCENARIOS = ["plain_upload_launch_download", "small_batch_staging_block", "staging_block_grows_while_a_copy_is_queued", "three_leg_api_and_relaunch",
             "arrival_gated_stream", "padded_host_layouts", "lean_features", "chain_every_host_path", "chain_arrival_gated_stream",
             "chain_padded_host_layouts", "rejected_inputs_leave_nothing_in_flight", "forced_variant_is_the_only_one_tried",
             "seed_schedule_overrides_are_validated", "pose_optimiser_host_paths", "pyramid_call",
             "level_7_derived_from_level_0", "pyramid_call_past_65535_frames", "undistort_past_65535_frames",
             "track_chained_call", "randomised_configurations", "bench_chain_leg"]


def _builder():
    spec = importlib.util.spec_from_file_location("plsvo_hostmodel_build", os.path.join(HM, "build.py"))
    m = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(m)
    return m


def _run(lib, mode, names=()):
    env = dict(os.environ, PLSVO_LIB=lib, PLSVO_FAKE_CUDA=mode)
    for k in [k for k in env if k.startswith("PLSVO_") and k not in ("PLSVO_LIB", "PLSVO_FAKE_CUDA")]:
        del env[k]
    p = subprocess.run([sys.executable, os.path.join(HM, "scenarios.py"), *names], env=env, capture_output=True, text=True, timeout=900)
    lines = [l for l in p.stdout.splitlines() if l.startswith("RESULT ")]
    assert p.returncode == 0 and lines, f"scenario runner failed:\n{p.stdout[-2000:]}\n{p.stderr[-4000:]}"
    return json.loads(lines[-1][7:])


@pytest.fixture(scope="module")
def hostmodel():
    return _builder().build()


@pytest.fixture(scope="module")
def results(hostmodel):
    cache = {}

    def get(mode):
        if mode not in cache:
            cache[mode] = _run(hostmodel, mode)
        return cache[mode]

    return get


def test_scenario_list_is_complete(results):
    assert sorted(results("lazy")) == sorted(SCENARIOS)


@pytest.mark.parametrize("mode", ["lazy", "eager"])
@pytest.mark.parametrize("scenario", SCENARIOS)
def test_host_pipeline(results, scenario, mode):
    """lazy: nothing runs until a synchronising call forces it, other streams advance only as far as events and the
    arrival gate require.  eager: everything runs as early as its dependencies allow."""
    assert results(mode)[scenario] == "ok", results(mode)[scenario]


def test_abi_misuse_tests_of_the_gpu_tier_against_the_host_model(hostmodel):
    """tests/test_gpu_abi_errors.py (state and argument errors, pinned allocation) needs no kernel result: here it runs
    against the host model, so the CPU tier sees the same return codes and messages the GPU tier checks."""
    env = dict(os.environ, PLSVO_LIB=hostmodel, PLSVO_FAKE_CUDA="lazy")
    p = subprocess.run([sys.executable, "-m", "pytest", os.path.join(HERE, "test_gpu_abi_errors.py"), "-q", "-m", "gpu", "-p", "no:cacheprovider"],
                       env=env, capture_output=True, text=True, timeout=600)
    assert p.returncode == 0, p.stdout[-3000:] + p.stderr[-2000:]


def test_fast_gpu_tier_files_against_the_host_model_with_oracle_backed_kernels(hostmodel, oracle):
    """The quick files of the GPU tier (golden fixtures, pose optimiser, and every next-row entry point: pyramid, align2D /
    align1D, findMatchDirect, structure optimisation, depth-filter seeds) run here against the host model with every model
    kernel answered by the CPU oracle (PLSVO_FAKE_ORACLE): a check of those test files, of the Python mirror and of the
    host code of those entry points — the oracle is compared with the oracle, so not of the kernels.  The slower files are
    run the same way by tools/preflight_gpu_tests.py."""
    root = os.path.dirname(HERE)
    env = dict(os.environ, PLSVO_LIB=hostmodel, PLSVO_FAKE_CUDA="lazy", PLSVO_FAKE_ORACLE=os.path.join(root, "oracle", "libplsvo_oracle.so"))
    files = [os.path.join(HERE, f) for f in ("test_gpu_golden.py", "test_gpu_poseopt.py", "test_pyramid.py", "test_align2d.py", "test_matcher.py",
                                             "test_structopt.py", "test_gpu_structopt_cases.py", "test_depth_filter.py")]
    p = subprocess.run([sys.executable, "-m", "pytest", *files, "-q", "-m", "gpu", "-p", "no:cacheprovider", "-k",
                        "not shim_optimize_structure_on_the_gpu"],  # that case links the CUDA library directly
                       env=env, capture_output=True, text=True, timeout=1200)
    assert p.returncode == 0, p.stdout[-3000:] + p.stderr[-2000:]
    assert " passed" in p.stdout and "failed" not in p.stdout


# ---- the model must notice seeded faults -------------------------------------------------------------------------------
FAULTS = {
    # the streamed kernel is launched without its arrival gate: it does not wait for the copies of a chunk to land
    "dropped_event_wait": (
        "  rc = align_launch_kernel(c, plan, c->stream, chunk);  // gated on arrivals\n", "  rc = align_launch_kernel(c, plan, c->stream, 0);\n",
        "lazy", ["arrival_gated_stream"]),
    # a frame chain sized like a two-stack batch: B frames instead of B + 1
    "undersized_frame_stack": (
        "    const size_t n_frames = B + (c->chain ? 1 : 0);\n", "    const size_t n_frames = B;\n",
        "lazy", ["chain_every_host_path"]),
    # the first chunk of a streamed frame chain forgets frame 0
    "chain_frame_never_shipped": (
        "      const size_t f0 = b0 ? b0 + 1 : 0, nf = b1 + 1 - f0;\n", "      const size_t f0 = b0 + 1, nf = b1 + 1 - f0;\n",
        "lazy", ["chain_arrival_gated_stream"]),
    # the arrival flag of a chunk is raised before the chunk's images have been queued
    "arrival_flag_too_early": (
        "  for (int k = 0; k < n_chunks; ++k) {\n    const size_t b0 = (size_t)k * chunk, b1 = std::min<size_t>(b0 + chunk, B);\n",
        "  for (int k = 0; k < n_chunks; ++k) {\n    const size_t b0 = (size_t)k * chunk, b1 = std::min<size_t>(b0 + chunk, B);\n"
        "    CK(cudaMemcpyAsync(d_arrived, &c->h_flags[k], sizeof(unsigned int), cudaMemcpyHostToDevice, c->copy_stream));\n",
        "lazy", ["arrival_gated_stream"]),
    # pyramid levels placed 8 bytes past a 16-byte boundary: the kernel's 16-byte loads and 8-byte stores would fault
    "misaligned_pyramid_level": (
        "    if (l > 0 && !out->level[l]) return fail(c, PLSVO_ERR_INVALID, \"output level missing\");\n"
        "    a.pitch[l] = (uint32_t)((cols + 15) / 16 * 16);\n    a.stride[l] = (size_t)rows * a.pitch[l];\n    total = (total + 255) / 256 * 256;\n    off[l] = total;\n",
        "    if (l > 0 && !out->level[l]) return fail(c, PLSVO_ERR_INVALID, \"output level missing\");\n"
        "    a.pitch[l] = (uint32_t)((cols + 15) / 16 * 16);\n    a.stride[l] = (size_t)rows * a.pitch[l];\n    total = (total + 255) / 256 * 256;\n    off[l] = total + 8;\n",
        "lazy", ["pyramid_call"]),
    # error exits return while copies from the caller's arrays are still queued
    "error_exit_without_drain": (
        "  if (rc == PLSVO_OK || !c) return rc;\n", "  if (true) return rc;\n",
        "lazy", ["rejected_inputs_leave_nothing_in_flight"]),
}


@pytest.mark.parametrize("fault", sorted(FAULTS))
def test_model_notices_seeded_fault(tmp_path, fault):
    old, new, mode, scenarios = FAULTS[fault]
    src = open(ABI_SOURCE).read()
    assert src.count(old) == 1, f"the line this fault is seeded into has changed: {old!r}"
    mutated = tmp_path / "plsvo_abi.cu"
    mutated.write_text(src.replace(old, new))
    lib = _builder().build(force=True, abi_source=str(mutated), out=str(tmp_path / "libplsvo_hostmodel_fault.so"))
    res = _run(lib, mode, scenarios)
    assert any(v != "ok" for v in res.values()), f"{fault}: every scenario still passes — the model is blind to it"
