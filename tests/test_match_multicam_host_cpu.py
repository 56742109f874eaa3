"""The host code of plsvo_match_direct_multicam_batch_run without a GPU, against the host-pipeline model (tests/hostmodel/,
DESIGN §8) with the per-image-camera matching kernel's model (tests/hostmodel/fake_match_multicam.cpp,
match_multicam_model.py): rejected calls leave nothing in flight and the context usable, and an accepted call with mixed
models and sizes shows the kernel only in-bounds bytes (tests/hostmodel/match_multicam_scenarios.py, lazy and eager
stream schedules); two faults seeded into a copy of plsvo_abi.cu are noticed; and tests/test_gpu_match_multicam.py runs
against the model with its kernels answered by the CPU oracle, as tools/preflight_gpu_tests.py runs it — a check of that
test file, the Python mirror and the host path, not of the kernel."""
import importlib.util
import json
import os
import subprocess
import sys

import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
HM = os.path.join(HERE, "hostmodel")
ROOT = os.path.dirname(HERE)


def _model_builder():
    spec = importlib.util.spec_from_file_location("plsvo_hostmodel_match_multicam", os.path.join(HM, "match_multicam_model.py"))
    m = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(m)
    return m


@pytest.fixture(scope="module")
def hostmodel():
    return _model_builder().build()


def _clean_env(**kw):
    env = dict(os.environ)
    for k in [k for k in env if k.startswith("PLSVO_")]:
        del env[k]
    env.update(kw)
    return env


def _scenarios(lib, mode):
    p = subprocess.run([sys.executable, os.path.join(HM, "match_multicam_scenarios.py")],
                       env=_clean_env(PLSVO_LIB=lib, PLSVO_FAKE_CUDA=mode), capture_output=True, text=True, timeout=600)
    lines = [l for l in p.stdout.splitlines() if l.startswith("RESULT ")]
    assert p.returncode == 0 and lines, f"scenario runner failed:\n{p.stdout[-2000:]}\n{p.stderr[-4000:]}"
    return json.loads(lines[-1][7:])


@pytest.mark.parametrize("mode", ["lazy", "eager"])
def test_match_multicam_host_scenarios(hostmodel, mode):
    res = _scenarios(hostmodel, mode)
    assert res and all(v == "ok" for v in res.values()), res


# seeded faults in a copy of plsvo_abi.cu that the model kernel must notice
FAULTS = {
    # the camera indices of the current frames uploaded one image short
    "cam_of_cur_short": ("CK(up(c->m_cam_of_cur, multi->cam_of_cur, (size_t)in->n_cur_images, s, &a.cam_of_cur));",
                         "CK(up(c->m_cam_of_cur, multi->cam_of_cur, (size_t)in->n_cur_images - 1, s, &a.cam_of_cur));"),
    # an ATAN camera's record given s_inv_ in place of s_
    "atan_terms_out_of_order": ("r.s = terms[0], r.s_inv = terms[1],", "r.s = terms[1], r.s_inv = terms[0],"),
}


@pytest.mark.parametrize("fault", FAULTS)
def test_model_notices_seeded_fault(tmp_path, fault):
    src = open(os.path.join(ROOT, "pl-svo_b200", "csrc", "plsvo_abi.cu")).read()
    old, new = FAULTS[fault]
    assert src.count(old) == 1, f"the fault's anchor is not in plsvo_abi.cu: {old!r}"
    mutated = tmp_path / "plsvo_abi.cu"
    mutated.write_text(src.replace(old, new))
    lib = _model_builder().build(force=True, out=str(tmp_path / "libplsvo_hostmodel_match_multicam.so"), abi_source=str(mutated))
    res = _scenarios(lib, "lazy")
    assert res and any(v != "ok" for v in res.values()), f"{fault} went unnoticed"


def test_gpu_match_multicam_file_against_the_host_model_with_oracle_backed_kernels(hostmodel, abi):
    sys.path.insert(0, os.path.join(ROOT, "oracle"))
    import oracle_atan_match
    import oracle_lib
    import oracle_multicam_match

    oracle_lib.build()
    oracle_atan_match.build()
    oracle_multicam_match.build()  # the model kernels find them next to libplsvo_oracle.so
    env = _clean_env(PLSVO_LIB=hostmodel, PLSVO_FAKE_CUDA="lazy", PLSVO_FAKE_ORACLE=os.path.join(ROOT, "oracle", "libplsvo_oracle.so"))
    p = subprocess.run([sys.executable, "-m", "pytest", os.path.join(HERE, "test_gpu_match_multicam.py"), "-q", "-m", "gpu", "-p",
                        "no:cacheprovider"], env=env, capture_output=True, text=True, timeout=1800, cwd=ROOT)
    assert p.returncode == 0, p.stdout[-3000:] + p.stderr[-2000:]
    assert " passed" in p.stdout and "failed" not in p.stdout
