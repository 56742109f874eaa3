"""The pose-optimiser kernel against the CPU oracle, on the shapes, parameters and frames where it can go wrong.

pose_optimizer_kernel (csrc/poseopt_kernel.cu) gives each frame one CTA of 128 threads.  Features are strided over the
threads, the medians are a radix select over shared-memory keys, the normal equations go through a register LDL^T solve that
hands rejected systems to a pivoted one, and a CTA runs its frames one after another with one shared-memory control block.
Its double sums are not in the reference's order, so it matches the oracle to tolerance (test_gpu_poseopt._check), not bit
for bit.  The cases:

  * the bench shape, 4096 frames of 300 points + 80 segments, two seeds: iteration counts and outlier flags must match.  A
    frame may differ only at a decision whose margin in the oracle (oracle_lib.poseopt_stats) is below 1e-12 relative;
  * feature counts on both sides of the 32-lane and 128-thread strides, the largest count shared memory admits (found by
    bisection through the host's validation) and both sides of the 48 KB dynamic shared-memory point;
  * pyramid levels 0-4, and the grid reproj_thresh x n_iter x n_iter_ref;
  * tied medians at even and odd counts; n/2 and n/2 + 1 exact zeros among the point errors (MAD scale > 0, and = 0: every
    Tukey weight 0, A = 0, the pivoted fallback, a NaN covariance); segments-only frames and frames with a point scale of 0
    (thr_ls infinite); a segment with an exactly zero residual (a NaN step in both loops);
  * layout invariance, GPU against GPU: a frame gives the same bytes alone, among other frames in a large batch (after a
    different frame on the same CTA), padded through pt_count / seg_count, and when the batch runs twice.

Frames with fewer than 8 live observations barely determine the pose (one point: not at all), so their steps and covariance
are round-off.  They are held to the bookkeeping only, as in test_gpu_poseopt.  So are frames whose refinement loop runs on
fewer than 8 inliers (a tight reproj_thresh at an unrefined pose can leave two).  test_cases_cover_the_decisions (no GPU)
uses the oracle's decision statistics to check that the cases keep reaching what they are meant to reach."""
import ctypes as C
from types import SimpleNamespace

import numpy as np
import pytest

from test_gpu_poseopt import FIELDS, ROT_TOL, TRANS_TOL, _check

MARGIN = 1e-12  # a decision this close in the oracle may go either way on the GPU
BOOKKEEPING = ("status", "pt_outlier", "seg_outlier", "num_obs_pt", "num_obs_ls")
LADDER = (1, 2, 31, 32, 33, 127, 128, 129, 255, 256, 257, 1000)
KINDS = ("points", "segments", "mixed")
THRESH = (0.25, 1.0, 2.0, 8.0, 1e6)
N_ITER = (0, 1, 2, 3, 30)
N_ITER_REF = (-1, 0, 1, 3, 10)
BYTES_PER_FEATURE = 25  # poseopt_smem_bytes: three double keys and one alive flag per feature


# ---- frames ------------------------------------------------------------------------------------------------------------
def _kind_shape(kind, n):
    return {"points": (n, 0), "segments": (0, n), "mixed": (n, n)}[kind]


def _plane_frames(synth, B, n_pts, n_segs, seed):
    """Frames at the identity pose with points and segment end points 2-6 m in front of the camera, observed with 1 px of
    noise and 10 % outliers of 20 px, levels 0-2.  Setting pt_f = pt_pos makes a point's residual exactly 0 (project2d
    takes an unnormalised bearing)."""
    rng = np.random.default_rng(seed)
    fx = synth.VGA.fx

    def world(n):
        z = rng.uniform(2.0, 6.0, (B, n, 1))
        return np.concatenate([rng.uniform(-0.6, 0.6, (B, n, 2)) * z, z], -1)

    def noise(n):
        e = rng.normal(0.0, 1.0 / fx, (B, n, 2))
        e[rng.uniform(size=(B, n)) < 0.1] *= 20.0
        return e

    pos = world(n_pts)
    f = pos.copy()
    f[..., :2] += noise(n_pts) * pos[..., 2:]
    spos, epos = world(n_segs), world(n_segs)
    s = np.concatenate([spos[..., :2] / spos[..., 2:] + noise(n_segs), np.ones((B, n_segs, 1))], -1)
    e = np.concatenate([epos[..., :2] / epos[..., 2:] + noise(n_segs), np.ones((B, n_segs, 1))], -1)
    line = np.cross(s, e)
    line /= np.hypot(line[..., 0], line[..., 1])[..., None]
    T = np.tile(np.array([0, 0, 0, 1, 0, 0, 0], np.float64), (B, 1))
    c = np.ascontiguousarray
    return synth.PoseOptData(fx=fx, T_f_w=T, T_f_w_gt=T.copy(), pt_f=c(f), pt_pos=c(pos),
                             pt_level=rng.integers(0, 3, (B, n_pts)).astype(np.int32), seg_line=c(line), seg_spos=c(spos),
                             seg_epos=c(epos), seg_level=rng.integers(0, 3, (B, n_segs)).astype(np.int32))


def _zeros(synth):
    """Rows 0-3 points only, 4-7 with 12 noisy segments: (live points, exact zeros) = (40, 20), (40, 21), (41, 20),
    (41, 21).  n // 2 zeros leave the median on a non-zero error (scale > 0); n // 2 + 1 put it on a zero (scale 0: every
    point weight is tukey(0/0) or tukey(e/0) = 0).  Row 8: 40 points, 12 segments and one segment whose residual is exactly
    0, so that its Jacobian is 0/0 and the step is NaN in both loops."""
    d = _plane_frames(synth, 9, 41, 13, seed=7100)
    d.pt_count = np.array([40, 40, 41, 41] * 2 + [40], np.int32)
    d.seg_count = np.array([0] * 4 + [12] * 4 + [13], np.int32)
    for b, z in enumerate([20, 21, 20, 21] * 2):
        d.pt_f[b, :z] = d.pt_pos[b, :z]
    # x/z = 0.5 at both end points, exactly; the line x = 0.5 goes through both
    d.seg_spos[8, 12], d.seg_epos[8, 12], d.seg_line[8, 12] = (1.0, 0.3, 2.0), (2.0, -1.5, 4.0), (1.0, 0.0, -0.5)
    return d


def _ties(synth):
    """Bench-like frames where 34 of the 45 points repeat one point and 11 of the 21 segments repeat one segment: the run of
    equal keys is longer than half of every live count, so the rank n // 2 of all four medians falls inside it.  Live counts
    (45, 21), (44, 21), (45, 20), (44, 20): even and odd in each median."""
    d = synth.make_poseopt_batch(batch=8, n_pts=45, n_segs=21, seed=7200)
    for b in range(8):
        for a in ("pt_f", "pt_pos", "pt_level"):
            getattr(d, a)[b, 1:34] = getattr(d, a)[b, 0]
        for a in ("seg_line", "seg_spos", "seg_epos", "seg_level"):
            getattr(d, a)[b, 1:11] = getattr(d, a)[b, 0]
    d.pt_count = np.array([45, 44, 45, 44] * 2, np.int32)
    d.seg_count = np.array([21, 21, 20, 20] * 2, np.int32)
    return d


def _pad(synth, d, n_pts, n_segs):
    """d in arrays of n_pts points and n_segs segments per frame: the same feature indices, counts from pt_count / seg_count
    (d's own, or its full widths), and NaN / out-of-range garbage in the padding, which no frame may read."""
    B = d.batch

    def grow(a, n, fill):
        out = np.full((B, n) + a.shape[2:], fill, a.dtype)
        out[:, : a.shape[1]] = a
        return out

    return synth.PoseOptData(
        fx=d.fx, T_f_w=d.T_f_w.copy(), T_f_w_gt=d.T_f_w_gt.copy(), pt_f=grow(d.pt_f, n_pts, np.nan),
        pt_pos=grow(d.pt_pos, n_pts, np.nan), pt_level=grow(d.pt_level, n_pts, 40), seg_line=grow(d.seg_line, n_segs, np.nan),
        seg_spos=grow(d.seg_spos, n_segs, np.nan), seg_epos=grow(d.seg_epos, n_segs, np.nan),
        seg_level=grow(d.seg_level, n_segs, 40),
        pt_valid=None if d.pt_valid is None else grow(d.pt_valid, n_pts, 1),
        seg_valid=None if d.seg_valid is None else grow(d.seg_valid, n_segs, 1),
        pt_count=np.full(B, d.n_pts, np.int32) if d.pt_count is None else d.pt_count.copy(),
        seg_count=np.full(B, d.n_segs, np.int32) if d.seg_count is None else d.seg_count.copy())


def _concat(synth, parts):
    """Frames of several batches of the same widths, in order."""
    cat = lambda f: None if all(getattr(p, f) is None for p in parts) else np.ascontiguousarray(np.concatenate([
        getattr(p, f) if getattr(p, f) is not None else _default(p, f) for p in parts]))
    fields = ("T_f_w", "T_f_w_gt", "pt_f", "pt_pos", "pt_level", "seg_line", "seg_spos", "seg_epos", "seg_level", "pt_valid",
              "seg_valid", "pt_count", "seg_count")
    return synth.PoseOptData(fx=parts[0].fx, **{f: cat(f) for f in fields})


def _default(d, f):
    if f == "pt_valid":
        return np.ones((d.batch, d.n_pts), np.uint8)
    if f == "seg_valid":
        return np.ones((d.batch, d.n_segs), np.uint8)
    return np.full(d.batch, d.n_pts if f == "pt_count" else d.n_segs, np.int32)


def _ragged(d, seed):
    """Dead features (pt_valid / seg_valid) and ragged counts in a bench-like batch."""
    rng = np.random.default_rng(seed)
    d.pt_valid = (rng.uniform(size=(d.batch, d.n_pts)) > 0.1).astype(np.uint8)
    d.seg_valid = (rng.uniform(size=(d.batch, d.n_segs)) > 0.1).astype(np.uint8)
    d.pt_count = rng.integers(d.n_pts // 2, d.n_pts + 1, d.batch).astype(np.int32)
    d.seg_count = rng.integers(0, d.n_segs + 1, d.batch).astype(np.int32)
    return d


def _case(name, synth):
    """(data, list of (reproj_thresh, n_iter, n_iter_ref)) of the named case."""
    if name.startswith("bench"):
        seed = int(name[5:])
        return synth.make_poseopt_batch(batch=4096, n_pts=300, n_segs=80, seed=seed), [(2.0, 10, -1 if seed == 5000 else 3)]
    if name.startswith("ladder-"):
        _, kind, n = name.split("-")
        n_pts, n_segs = _kind_shape(kind, int(n))
        return synth.make_poseopt_batch(batch=8, n_pts=n_pts, n_segs=n_segs, seed=7300 + int(n)), [(2.0, 10, 3)]
    if name.startswith("levels-"):
        n_pts, n_segs = _kind_shape(name[7:], 150)
        return synth.make_poseopt_batch(batch=32, n_pts=n_pts, n_segs=n_segs, seed=7400, max_level=4), [(2.0, 10, -1), (2.0, 10, 3)]
    if name == "grid":
        d = _concat(synth, [synth.make_poseopt_batch(batch=10, n_pts=60, n_segs=20, seed=7500, max_level=4),
                            # noise-free frames: the steps shrink until EPS stops the loop
                            synth.make_poseopt_batch(batch=2, n_pts=60, n_segs=20, seed=7501, max_level=4, noise_px=0.0,
                                                     outlier_frac=0.0)])
        return d, [(t, n, r) for t in THRESH for n in N_ITER for r in N_ITER_REF]
    if name == "zeros":
        return _zeros(synth), [(2.0, 10, -1), (2.0, 10, 3)]
    if name == "ties":
        return _ties(synth), [(2.0, 10, -1), (2.0, 10, 3)]
    raise KeyError(name)


CASES = ["bench5000", "bench5001"] + [f"ladder-{k}-{n}" for k in KINDS for n in LADDER] + [f"levels-{k}" for k in KINDS] + [
    "grid", "zeros", "ties"]


@pytest.fixture(scope="module")
def case(synth):
    made = {}

    def get(name):
        if name not in made:
            made[name] = _case(name, synth)
        return made[name]

    return get


# ---- running and comparing ---------------------------------------------------------------------------------------------
def _live(d):
    def count(valid, n, width):
        v = np.ones((d.batch, width), bool) if valid is None else valid.astype(bool)
        return (v & (np.arange(width)[None, :] < n[:, None])).sum(1)

    pc = np.full(d.batch, d.n_pts) if d.pt_count is None else d.pt_count
    sc = np.full(d.batch, d.n_segs) if d.seg_count is None else d.seg_count
    return count(d.pt_valid, pc, d.n_pts) + count(d.seg_valid, sc, d.n_segs)


def _rows(out, m):
    return SimpleNamespace(**{f: getattr(out, f)[m] for f in FIELDS})


def _gpu(pkg, d, p):
    return pkg.pose_optimizer.optimizeGaussNewton(p[0], p[1], False, d, n_iter_ref=None if p[2] < 0 else p[2])


def _compare(synth, d, gpu, ref, cov=True, skip=(), refined=False):
    """Bookkeeping on every frame; the full _check on frames with at least 8 live observations (rows `skip` excepted) and,
    when the refinement loop ran (refined), at least 8 inliers for it."""
    for f in BOOKKEEPING:
        np.testing.assert_array_equal(np.delete(getattr(gpu, f), list(skip), 0), np.delete(getattr(ref, f), list(skip), 0), err_msg=f)
    empty = _live(d) == 0
    np.testing.assert_array_equal(gpu.T_f_w[empty], d.T_f_w[empty])
    full = _live(d) >= 8
    if refined:
        full &= ref.num_obs_pt + ref.num_obs_ls >= 8
    full[list(skip)] = False
    if full.any():
        _check(synth, _rows(gpu, full), _rows(ref, full), cov=cov)


def _run_case(pkg, abi, synth, oracle, d, p, cov=True):
    gpu = _gpu(pkg, d, p)
    ref = oracle.poseopt(abi, d, abi.poseopt_params(*p), n_threads=8)
    _compare(synth, d, gpu, ref, cov=cov and p[1] > 0, refined=p[2] > 0)
    return gpu, ref


# ---- GPU tests ---------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("name", ["bench5000", "bench5001"])
def test_bench_shape_matches_the_oracle(pkg, abi, synth, oracle, case, name):
    """Iteration counts and outlier flags of every frame, unless the oracle's own decision there was within MARGIN."""
    d, (p,) = case(name)
    gpu = _gpu(pkg, d, p)
    ref, st = oracle.poseopt_stats(abi, d, abi.poseopt_params(*p), n_threads=8)
    excused = set()
    for loop in (0, 1):
        for b in np.nonzero(gpu.iters[:, loop] != ref.iters[:, loop])[0]:
            k = min(gpu.iters[b, loop], ref.iters[b, loop]) - 1  # the first decision the two runs took differently
            m = st["iter_margin"][b, loop, k] if 0 <= k < oracle.PO_STAT_ITERS else np.inf
            assert m < MARGIN, f"frame {b} loop {loop}: {gpu.iters[b, loop]} iterations, oracle {ref.iters[b, loop]} (margin {m:.2e})"
            excused.add(int(b))
    for f, key in (("pt_outlier", "out_margin_pt"), ("seg_outlier", "out_margin_ls")):
        for b in np.nonzero((getattr(gpu, f) != getattr(ref, f)).any(1))[0]:
            if int(b) not in excused:
                assert st[key][b] < MARGIN, f"frame {b}: {f} differs (margin {st[key][b]:.2e})"
                excused.add(int(b))
    skip = sorted(excused)
    print(f"{name}: frames excused by the margin rule: {skip}")
    ang, rel = synth.pose_error(gpu.T_f_w, ref.T_f_w)
    assert ang.max() <= ROT_TOL and rel.max() <= TRANS_TOL
    _compare(synth, d, gpu, ref, skip=skip, refined=p[2] > 0)
    fin = np.isfinite(ref.cov).all(1)
    cov_err = (np.abs(gpu.cov - ref.cov)[fin] / np.abs(ref.cov[fin]).max(1, keepdims=True)).max()
    print(f"{name}: max rotation {ang.max():.3e} rad, max relative translation {rel.max():.3e}, max covariance {cov_err:.3e}")


@pytest.mark.gpu
@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("n", LADDER)
def test_feature_count_ladder(pkg, abi, synth, oracle, case, kind, n):
    d, (p,) = case(f"ladder-{kind}-{n}")
    _run_case(pkg, abi, synth, oracle, d, p)


def _probe(pkg, abi, synth, n):
    """plsvo_poseopt_batch_run on one frame of n points, none of them live -> (rc, message).  Only the host's shared-memory
    validation looks at n; a size it accepts runs one empty frame."""
    ctx = pkg.api.default_context()
    z3 = np.zeros((1, n, 3))
    d = synth.PoseOptData(fx=synth.VGA.fx, T_f_w=np.array([[0, 0, 0, 1, 0, 0, 0.0]]), T_f_w_gt=np.zeros((1, 7)), pt_f=z3,
                          pt_pos=z3, pt_level=np.zeros((1, n), np.int32), seg_line=np.zeros((1, 0, 3)),
                          seg_spos=np.zeros((1, 0, 3)), seg_epos=np.zeros((1, 0, 3)), seg_level=np.zeros((1, 0), np.int32),
                          pt_count=np.zeros(1, np.int32))
    batch, keep = abi.make_poseopt_batch(d)
    out = abi.PoseOptOut(1, n, 0)
    rc = ctx.lib.plsvo_poseopt_batch_run(ctx.handle, C.byref(batch), C.byref(abi.poseopt_params(2.0, 10, -1)), C.byref(out.struct))
    msg = ctx.lib.plsvo_last_error(ctx.handle)
    return rc, (msg.decode() if msg else "")


def _optin_bytes():
    import torch

    if torch.cuda.is_available():
        return int(torch.cuda.get_device_properties(0).shared_memory_per_block_optin)
    return 227 * 1024  # sm_90's opt-in limit, as the host model reports it


@pytest.mark.gpu
def test_shared_memory_limit(pkg, abi, synth, oracle):
    """N = the largest n_pts + n_segs the device admits.  N + 1 is refused with the shared-memory message and the context
    stays usable; frames on both sides of 48 KB (above it the launch raises the kernel's dynamic shared-memory limit) and a
    batch of N-feature frames match the oracle."""
    lo, hi = 1, 1 << 20
    assert _probe(pkg, abi, synth, lo)[0] == abi.OK
    assert _probe(pkg, abi, synth, hi)[0] == abi.ERR_INVALID
    while hi - lo > 1:
        mid = (lo + hi) // 2
        rc, msg = _probe(pkg, abi, synth, mid)
        assert rc in (abi.OK, abi.ERR_INVALID), msg
        lo, hi = (mid, hi) if rc == abi.OK else (lo, mid)
    N = lo
    rc, msg = _probe(pkg, abi, synth, N + 1)
    assert rc == abi.ERR_INVALID and "feature counts exceed shared memory" in msg, (rc, msg)
    print(f"largest frame the device admits: {N} features")
    n48 = N - (_optin_bytes() - 48 * 1024) // BYTES_PER_FEATURE  # the first count above 48 KB, by the kernel's layout
    assert 1000 < n48 < N
    p = (2.0, 10, 3)
    for i, n in enumerate((n48 - 2, n48 - 1, n48, n48 + 1, N)):  # the first call after the refusal, on the same context
        n_segs = n // 5
        d = synth.make_poseopt_batch(batch=2 if n == N else 4, n_pts=n - n_segs, n_segs=n_segs, seed=7600 + i)
        _run_case(pkg, abi, synth, oracle, d, p)


@pytest.mark.gpu
@pytest.mark.parametrize("kind", KINDS)
def test_levels_up_to_four(pkg, abi, synth, oracle, case, kind):
    d, params = case(f"levels-{kind}")
    for p in params:
        _run_case(pkg, abi, synth, oracle, d, p)


@pytest.mark.gpu
@pytest.mark.parametrize("n_iter", N_ITER)
@pytest.mark.parametrize("thresh", THRESH)
def test_parameter_grid(pkg, abi, synth, oracle, case, thresh, n_iter):
    """Every n_iter_ref for this (reproj_thresh, n_iter); n_iter = 0: the reference's covariance is of an A it never set."""
    d, _ = case("grid")
    for r in N_ITER_REF:
        _run_case(pkg, abi, synth, oracle, d, (thresh, n_iter, r))


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["zeros", "ties"])
def test_ties_and_zeros(pkg, abi, synth, oracle, case, name):
    d, params = case(name)
    for p in params:
        gpu, ref = _run_case(pkg, abi, synth, oracle, d, p)
        if name == "zeros":
            scale0 = np.array([0, 1, 0, 1] * 2 + [0], bool)
            assert (gpu.estimated_scale[scale0] == 0).all() and (gpu.estimated_scale[~scale0] > 0).all()
            assert (gpu.iters[[1, 3], 0] == 1).all() and np.isnan(gpu.cov[[1, 3]]).all()


@pytest.mark.gpu
def test_layout_invariance(pkg, abi, synth, case):
    """The same frames, byte for byte: alone, scattered through a 4096-frame batch (each after another frame on its CTA:
    the grid is 16 CTAs per SM), padded to wider arrays, and when the big batch runs a second time."""
    import torch

    sms = torch.cuda.get_device_properties(0).multi_processor_count if torch.cuda.is_available() else 132
    grid = 16 * sms
    frames = _ragged(synth.make_poseopt_batch(batch=12, n_pts=300, n_segs=80, seed=7700), 7701)
    zeros = _pad(synth, case("zeros")[0], 300, 80)
    for f in ("T_f_w", "pt_f", "pt_pos", "pt_level", "seg_line", "seg_spos", "seg_epos", "seg_level", "pt_count", "seg_count"):
        getattr(frames, f)[[4, 5]] = getattr(zeros, f)[[1, 8]]  # a MAD scale of 0, and a NaN step at the first iteration
    frames.pt_valid[[4, 5]], frames.seg_valid[[4, 5]] = 1, 1
    big = _concat(synth, [case("bench5000")[0]])  # a copy
    _ragged(big, 7702)
    # the frame before a test frame on its CTA: degenerate, tied or larger ones, of the same widths
    before = _concat(synth, [_pad(synth, case("zeros")[0], 300, 80), _pad(synth, case("ties")[0], 300, 80)])
    pos = grid + np.arange(12) * 97
    pos[-2:] = (3, grid - 1)  # two in the first wave
    for f in ("T_f_w", "T_f_w_gt", "pt_f", "pt_pos", "pt_level", "seg_line", "seg_spos", "seg_epos", "seg_level", "pt_valid",
              "seg_valid", "pt_count", "seg_count"):
        src, prev = getattr(frames, f), getattr(before, f)
        if prev is None:
            prev = _default(before, f)
        dst = getattr(big, f)
        dst[pos] = src
        dst[pos[:-2] - grid] = prev[np.linspace(0, before.batch - 1, 10).astype(int)]
    p = (2.0, 10, 3)
    out_big = _gpu(pkg, big, p)
    out_again = _gpu(pkg, big, p)
    out_pad = _gpu(pkg, _pad(synth, frames, 450, 133), p)
    outs = ("T_f_w", "cov", "estimated_scale", "error_init", "error_final", "num_obs_pt", "num_obs_ls", "iters", "status",
            "pt_outlier", "seg_outlier")
    for f in outs:
        assert getattr(out_big, f).tobytes() == getattr(out_again, f).tobytes(), f"{f}: the second run differs"
    for i in range(12):
        alone = _gpu(pkg, _concat(synth, [_slice(synth, frames, i)]), p)
        for f in outs:
            a = np.asarray(getattr(alone, f)[0])
            cut = (lambda x: np.asarray(x)[: a.shape[0]]) if a.ndim else np.asarray  # outlier flags: the frame's own width
            assert cut(getattr(out_big, f)[pos[i]]).tobytes() == a.tobytes(), f"frame {i}: {f} differs in the big batch"
            assert cut(getattr(out_pad, f)[i]).tobytes() == a.tobytes(), f"frame {i}: {f} differs when padded"


def _slice(synth, d, i):
    fields = ("T_f_w", "T_f_w_gt", "pt_f", "pt_pos", "pt_level", "seg_line", "seg_spos", "seg_epos", "seg_level", "pt_valid",
              "seg_valid", "pt_count", "seg_count")
    return synth.PoseOptData(fx=d.fx, **{f: None if getattr(d, f) is None else np.ascontiguousarray(getattr(d, f)[i:i + 1])
                                         for f in fields})


# ---- CPU tier ----------------------------------------------------------------------------------------------------------
def _all_runs(synth):
    for name in CASES:
        d, params = _case(name, synth)
        for p in params:
            yield name, d, p


def test_poseopt_stats_leaves_the_outputs_alone(abi, synth, oracle):
    """oracle.poseopt_stats runs the same optimisation: its outputs are byte-identical to oracle.poseopt's."""
    for name in ("grid", "zeros", "ties", "levels-mixed", "ladder-segments-33"):
        d, params = _case(name, synth)
        for p in params[::7] if name == "grid" else params:
            a = oracle.poseopt(abi, d, abi.poseopt_params(*p), n_threads=4)
            b, _ = oracle.poseopt_stats(abi, d, abi.poseopt_params(*p), n_threads=4)
            for f in FIELDS:
                if f == "cov" and p[1] == 0:
                    continue  # the inverse of an A the reference never set
                assert getattr(a, f).tobytes() == getattr(b, f).tobytes(), f"{name} {p}: {f}"


def test_cases_cover_the_decisions(abi, synth, oracle):
    """The cases reach: every exit of both loops, the pivoted fallback, a tie at each median, a MAD scale of 0, outlier
    decisions on both sides of the threshold, levels 3 and 4 for points and segments."""
    exits = {0: set(), 1: set()}
    fallback = np.zeros(2, int)
    ties = np.zeros(4, int)
    scale0, out_pt, in_pt, out_ls, in_ls = 0, 0, 0, 0, 0
    pt_levels, seg_levels = set(), set()
    for name, d, p in _all_runs(synth):
        if name.startswith("bench") and p[2] < 0:
            continue  # a second bench batch adds nothing but time
        out, st = oracle.poseopt_stats(abi, d, abi.poseopt_params(*p), n_threads=8)
        live = out.status == 0
        for loop in (0, 1):
            exits[loop] |= set(np.unique(st["exit"][live, loop]).tolist())
        fallback += st["fallback"][live].sum(0)
        ties += st["med_tie"][live].sum(0)
        scale0 += int(((st["scale_pt"] == 0) & (st["med_count"][:, 0] > 0) & live).sum())
        pv = np.ones(d.pt_f.shape[:2], bool) if d.pt_valid is None else d.pt_valid.astype(bool)
        out_pt += int(out.pt_outlier.sum())
        in_pt += int(out.num_obs_pt.sum())
        out_ls += int(out.seg_outlier.sum())
        in_ls += int(out.num_obs_ls.sum())
        if name.startswith("levels"):
            pt_levels |= set(np.unique(d.pt_level[pv]).tolist())
            seg_levels |= set(np.unique(d.seg_level).tolist())
    every = {oracle.PO_EXIT_NONE, oracle.PO_EXIT_CHI2, oracle.PO_EXIT_NAN, oracle.PO_EXIT_EPS, oracle.PO_EXIT_CAP}
    for loop in (0, 1):
        assert exits[loop] == every, f"loop {loop}: exits {sorted(exits[loop])}"
    assert (fallback >= 3).all(), f"fallback solves per loop: {fallback}"
    assert (ties >= 3).all(), f"ties at the MAD point, MAD segment, initial and final medians: {ties}"
    assert scale0 >= 4, "frames with a MAD point scale of 0"
    assert min(out_pt, in_pt, out_ls, in_ls) >= 10, (out_pt, in_pt, out_ls, in_ls)
    assert pt_levels == seg_levels == {0, 1, 2, 3, 4}, (pt_levels, seg_levels)
