"""Every search schedule of the depth-filter seed kernels against the CPU oracle, on long, tied and odd-sized searches.

seed_update_kernel and line_seed_update_kernel walk the epipolar ZMSSD search (matcher.cpp:354-391) in a schedule chosen
from the batch size: `spw` seeds share a warp (1 ... 32), the first `serial steps` of each search (16 when spw >= 16, else
0) are walked by the seed's own thread, and the whole warp takes the rest, 32 steps per pass, seed after seed.  Every
schedule must give the sequential loop's result: the same winning step, ties to the lowest step, a later pass winning only
with a strictly lower score.  PLSVO_SEEDS_PER_WARP and PLSVO_EPI_SERIAL_STEPS force a schedule; each case's oracle result
is computed once and compared with many forced schedules, with the tolerances of test_gpu_seed_update_matches_the_oracle,
and every schedule's output must be byte-identical to the automatic one's.  Each run is repeated with subpix_refinement
off, so that px_cur and depth show the winning step itself rather than where align2D converged from it.

test_cases_cover_the_schedule_edges (no GPU) uses the oracle's search statistics to keep the cases honest: long searches
in every band around the pass boundaries, ties across passes and across step 16, winners in the own-thread range and late
warp passes, searches nothing wins, every search level of the 5-level cameras and both sides of max_epi_search_steps."""
import dataclasses
import os

import numpy as np
import pytest

KINDS = ("point", "line")
CASES = ["default", "long1", "long3", "boundary", "flat", "striped", "euroc", "odd", "tail1", "tail31", "tail33"]
LONG = ("long1", "long3")
AUTO = (None, None)
# (seeds per warp, serial steps); None: the automatic choice
FEW_SCHEDULES = [AUTO, (32, 16), (32, 0), (1, 0), (5, 17)]
ALL_SCHEDULES = [AUTO] + [(s, t) for s in (1, 2, 3, 8, 16, 31, 32) for t in (0, 1, 15, 16, 17, 48, 100000)]
# step counts (n_steps + 1) either side of step 16 and of the 32-step warp passes
BANDS = [(1, 15), (16, 16), (17, 17), (18, 47), (48, 48), (49, 49), (50, 200), (201, 1 << 30)]


def _take(d, idx):
    """The seeds idx of a batch (frames and pyramids shared)."""
    kw = {}
    for f in d.__dataclass_fields__:
        v = getattr(d, f)
        per_seed = isinstance(v, np.ndarray) and f not in ("T_ref_w", "T_cur_w") and v.shape[:1] == (d.n,)
        kw[f] = np.ascontiguousarray(v[idx]) if per_seed else v
    return type(d)(**kw)


def _stripes(shape, period, axis, phase):
    """Frames constant along one axis and periodic (a fixed sequence of grey values) along the other.  The contrast is low,
    so that the best score of most searches beats PatchScore::threshold() and repeats every period."""
    pattern = (128 + np.array([0, 12, -8, 20, -15, 5, -20, 10, -5, 15, -12])[:period]).astype(np.uint8)
    n, h, w = shape
    along = np.arange(w if axis == 1 else h) + phase
    line = pattern[along % period]
    img = np.broadcast_to(line[None, :] if axis == 1 else line[:, None], (h, w))
    return np.broadcast_to(img, shape)


def _gen(kind, synth, dev, **kw):
    if kind == "point":
        return synth.make_seed_batch(device=dev, **kw)
    return synth.make_line_seed_batch(device=dev, **kw)


def _long(kind, synth, dev, levels):
    """Wide baseline, uncertain depths, no step limit: searches of tens to hundreds of steps."""
    d = _gen(kind, synth, dev, n=2000, seed=9700 + levels + (50 if kind == "line" else 0), n_pyr_levels=levels, baseline=0.3)
    d.sigma2 = (d.sigma2 * 30).astype(np.float32)
    if kind == "line":
        d.sigma2_e = (d.sigma2_e * 30).astype(np.float32)
    d.max_epi_search_steps = 100000
    return d


def _searched(stats):
    """Searches the loop ran (not rejected by max_epi_search_steps)."""
    return (stats["steps"] >= 0) & (stats["rejected"] == 0)


def _make(name, kind, synth, oracle, dev="cpu"):
    """The batch of one case."""
    from plsvo_b200 import abi

    if name == "default":
        return _gen(kind, synth, dev, n=3000, seed=9800 if kind == "point" else 9850)
    if name in LONG:
        return _long(kind, synth, dev, int(name[-1]))
    if name == "boundary":  # max_epi_search_steps equal to the n_steps of some searches, one below that of others
        d = _long(kind, synth, dev, 3)
        steps = oracle.seed_search_stats(abi, d, 8)[1]["steps"]
        steps = steps if steps.ndim == 1 else steps[:, 0]
        count = np.bincount(steps[steps > 0], minlength=2002)
        # n_steps = s - 1 searched, n_steps = s rejected; prefer limits beyond the second warp pass
        ok = [s for s in range(66, 2000) if count[s] >= 2 and count[s + 1] >= 2]
        d.max_epi_search_steps = int(ok[0]) - 1
        return d
    if name in ("flat", "striped"):
        d = _long(kind, synth, dev, 3)
        d.max_epi_search_steps = 1000
        for l, p in d.cur_pyr.items():
            if name == "flat":  # every evaluated step scores the same; align2D meets a singular Hessian
                d.cur_pyr[l] = np.full_like(p, 128)
            else:  # frame 0: vertical stripes of period 7, frame 1: horizontal of period 5, frame 2: vertical of period 11
                d.cur_pyr[l] = np.ascontiguousarray(np.concatenate(
                    [_stripes((1,) + p.shape[1:], per, ax, l) for per, ax in ((7, 1), (5, 0), (11, 1))][: p.shape[0]], 0))
        return d
    if name == "euroc":
        return _gen(kind, synth, dev, n=3000, seed=9900 + (50 if kind == "line" else 0), cam=synth.EUROC, n_pyr_levels=5)
    if name == "odd":
        return _gen(kind, synth, dev, n=3000, seed=9910 + (50 if kind == "line" else 0), cam=synth.ODD, n_pyr_levels=5)
    if name.startswith("tail"):  # 1, 31, 33 seeds, each with a search of more than one warp pass
        d = _long(kind, synth, dev, 3)
        steps = oracle.seed_search_stats(abi, d, 8)[1]["steps"]
        steps = steps if steps.ndim == 1 else steps[:, 0]
        return _take(d, np.nonzero(steps > 40)[0][: int(name[4:])])
    raise KeyError(name)


@pytest.fixture(scope="module")
def case(abi, synth, oracle, gen_device):
    """(name, kind, subpix) -> (data, oracle result), each batch built once and each configuration solved once."""
    data, solved = {}, {}

    def get(name, kind, subpix=True):
        if (name, kind) not in data:
            data[name, kind] = _make(name, kind, synth, oracle, gen_device)
        if (name, kind, subpix) not in solved:
            d = dataclasses.replace(data[name, kind], subpix_refinement=subpix)
            solve = oracle.seed_update if kind == "point" else oracle.line_seed_update
            solved[name, kind, subpix] = (d, solve(abi, d, 8))
        return solved[name, kind, subpix]

    return get


def _outputs(kind):
    return ("status", "converged", "a", "b", "mu", "sigma2", "depth", "px_cur") + (
        ("mu_e", "sigma2_e", "depth_e", "px_cur_e") if kind == "line" else ())


def _run(pkg, monkeypatch, d, kind, schedule):
    spw, serial = schedule
    for var, v in (("PLSVO_SEEDS_PER_WARP", spw), ("PLSVO_EPI_SERIAL_STEPS", serial)):
        if v is None:
            monkeypatch.delenv(var, raising=False)
        else:
            monkeypatch.setenv(var, str(v))
    df = pkg.DepthFilter()
    return df.updatePointSeeds(d) if kind == "point" else df.updateLineSeeds(d)


def _check(abi, kind, out, ref):
    """test_gpu_seed_update_matches_the_oracle's assertions: the branch, the position and the depth exact, the updated
    Gaussian x Beta to the round-off of the libm calls."""
    np.testing.assert_array_equal(out.status, ref.status)
    up = ref.status == abi.SEED_UPDATED
    for f in ("px_cur", "px_cur_e") if kind == "line" else ("px_cur",):
        o, r = getattr(out, f), getattr(ref, f)
        fin = np.isfinite(r).all(axis=1)
        np.testing.assert_array_equal(np.isfinite(o).all(axis=1), fin, err_msg=f)
        np.testing.assert_array_equal(o[fin], r[fin], err_msg=f)
    for f in ("depth", "depth_e") if kind == "line" else ("depth",):
        np.testing.assert_array_equal(getattr(out, f)[up], getattr(ref, f)[up], err_msg=f)
        assert np.isnan(getattr(out, f)[~up]).all(), f
    fields = ("a", "b", "mu", "sigma2") + (("mu_e", "sigma2_e") if kind == "line" else ())
    for f in fields:
        np.testing.assert_array_equal(getattr(out, f)[~up], getattr(ref, f)[~up], err_msg=f)
    ok = up & np.isfinite(ref.a) & np.isfinite(ref.sigma2)
    if kind == "line":
        ok &= np.isfinite(ref.sigma2_e)
    for f in ("mu", "mu_e") if kind == "line" else ("mu",):
        np.testing.assert_allclose(getattr(out, f)[ok], getattr(ref, f)[ok], rtol=2e-6, atol=0, err_msg=f)
    for f in ("sigma2", "sigma2_e") if kind == "line" else ("sigma2",):
        np.testing.assert_allclose(getattr(out, f)[ok], getattr(ref, f)[ok], rtol=2e-4, atol=5e-7, err_msg=f)
    np.testing.assert_allclose(out.a[ok], ref.a[ok], rtol=5e-2)
    np.testing.assert_allclose(out.b[ok], ref.b[ok], rtol=5e-2, atol=1e-3)
    assert (out.converged == ref.converged).mean() > 0.999


def _params():
    for kind in KINDS:
        for name in CASES:
            for schedule in ALL_SCHEDULES if name in LONG else FEW_SCHEDULES:
                for subpix in (True, False):
                    sid = "auto" if schedule == AUTO else f"{schedule[0]}x{schedule[1]}"
                    yield pytest.param(kind, name, schedule, subpix, id=f"{kind}-{name}-{sid}-{'subpix' if subpix else 'nosubpix'}")


@pytest.fixture(scope="module")
def auto_out():
    """(name, kind, subpix) -> output of the automatic schedule (the first schedule of every case)."""
    return {}


@pytest.mark.gpu
@pytest.mark.parametrize("kind,name,schedule,subpix", list(_params()))
def test_schedule_matches_the_oracle(pkg, abi, case, auto_out, monkeypatch, kind, name, schedule, subpix):
    d, ref = case(name, kind, subpix)
    out = _run(pkg, monkeypatch, d, kind, schedule)
    _check(abi, kind, out, ref)
    key = (name, kind, subpix)
    if schedule == AUTO:
        auto_out[key] = out
        return
    if key not in auto_out:  # this schedule ran on its own (-k): take the automatic schedule's output now
        auto_out[key] = _run(pkg, monkeypatch, d, kind, AUTO)
    # after the search every seed's arithmetic runs on its own thread, whatever the schedule: no tolerance
    for f in _outputs(kind):
        assert getattr(out, f).tobytes() == getattr(auto_out[key], f).tobytes(), f"{f} differs from the automatic schedule's"


def _num_sms():
    import torch

    return torch.cuda.get_device_properties(0).multi_processor_count if torch.cuda.is_available() else 132


def _natural_n():
    """A batch the planner gives 32 seeds per warp and 16 serial steps: more than 16 * 8 seeds per SM."""
    return 16 * 8 * _num_sms() + 997


@pytest.mark.gpu
@pytest.mark.parametrize("kind", KINDS)
def test_natural_size_matches_the_oracle(pkg, abi, synth, oracle, gen_device, monkeypatch, kind):
    d = _gen(kind, synth, gen_device, n=_natural_n(), seed=9950 if kind == "point" else 9960)
    ref = (oracle.seed_update if kind == "point" else oracle.line_seed_update)(abi, d, 8)
    _check(abi, kind, _run(pkg, monkeypatch, d, kind, AUTO), ref)


@pytest.mark.gpu
@pytest.mark.skipif(bool(os.environ.get("PLSVO_FAKE_ORACLE")), reason="the host model launches no kernel")
def test_forced_schedule_sets_the_launch_grid(pkg, synth, gen_device, monkeypatch, tmp_path):
    """The grid of seed_update_kernel in a profiler trace is ceil(n / (spw * 4)) (four warps per CTA): the override is
    what ran, and the automatic choice at the natural size is 32 seeds per warp."""
    import json

    import torch

    small = synth.make_seed_batch(n=3000, seed=9970, device=gen_device)
    big = synth.make_seed_batch(n=_natural_n(), seed=9971, device=gen_device)
    runs = [(small, (1, 0), 1), (small, (3, 17), 3), (small, (31, None), 31), (small, (32, 0), 32), (big, AUTO, 32)]
    for i, (d, schedule, spw) in enumerate(runs):
        _run(pkg, monkeypatch, d, "point", schedule)  # warm-up outside the trace
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            _run(pkg, monkeypatch, d, "point", schedule)
        path = tmp_path / f"trace{i}.json"
        prof.export_chrome_trace(str(path))
        events = json.loads(path.read_text())["traceEvents"]
        grids = [e["args"]["grid"] for e in events if e.get("cat") == "kernel" and "seed_update_kernel" in e.get("name", "")
                 and "line_seed_update_kernel" not in e["name"]]
        assert grids, f"no seed_update_kernel launch with a grid in the trace ({len(events)} events)"
        want = -(-d.n // (spw * 4))
        assert grids == [[want, 1, 1]], f"{schedule}: grid {grids}, expected [{want}, 1, 1]"


def test_cases_cover_the_schedule_edges(abi, synth, oracle):
    """The cases contain what the schedules can get wrong (oracle search statistics, CPU-generated batches)."""
    steps, first, last, level5, no_win = [], [], [], set(), 0
    boundary = {}
    for kind in KINDS:
        for name in CASES:
            d = _make(name, kind, synth, oracle)
            st = oracle.seed_search_stats(abi, d, 8)[1]
            ran = _searched(st)
            steps.append(st["steps"][ran]), first.append(st["first_best"][ran]), last.append(st["last_best"][ran])
            no_win += int(st["no_win"][ran].sum())
            if name in ("euroc", "odd"):
                level5 |= set(np.unique(st["level"][ran]).tolist())
            if name == "boundary":
                m = d.max_epi_search_steps
                boundary[kind] = (int((ran & (st["steps"] == m + 1)).sum()), int(((st["rejected"] == 1) & (st["steps"] == m + 2)).sum()))
    s, fb, lb = np.concatenate(steps), np.concatenate(first), np.concatenate(last)
    for lo, hi in BANDS:
        assert ((s >= lo) & (s <= hi)).sum() >= 3, f"fewer than 3 searches of {lo}..{hi} steps"
    won = fb >= 0
    assert (won & (fb < 16)).sum() >= 3, "no winners in the own-thread range"
    assert (won & (fb >= 80)).sum() >= 3, "no winners in the third warp pass or later"
    assert (won & (fb // 32 != lb // 32)).sum() >= 3, "no ties across 32-step passes"
    assert (won & (fb >= 16) & ((fb - 16) // 32 != (lb - 16) // 32)).sum() >= 3, "no ties across passes after 16 own-thread steps"
    assert (won & (fb < 16) & (lb >= 16)).sum() >= 3, "no ties on both sides of step 16"
    assert no_win >= 3, "no search where nothing beat the threshold"
    assert level5 == {0, 1, 2, 3, 4}, f"search levels of the 5-level cameras: {sorted(level5)}"
    for kind, (at, beyond) in boundary.items():
        assert at >= 1 and beyond >= 1, f"{kind}: max_epi_search_steps searched {at} times, rejected {beyond} times one step beyond"
