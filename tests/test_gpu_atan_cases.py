"""The ATAN (FOV) alignment kernel (sparse_img_align_atan_kernel) against the oracle's ATAN path at the shapes, cameras
and parameters where it could go wrong unseen by tests/test_gpu_atan.py:

  * every compiled variant (PLSVO_VARIANT) on the cases of test_gpu_align_variants.py, frames and features rendered
    through an ATAN camera with d0 = 0.93 (the planner only ever picks <256,2> or <128,4> by itself);
  * a non-square, off-centre 752x480 camera (fx_ != fy_, cx_ and cy_ off the image centre), aligned and tracked;
  * cam2world's cut-off (no distortion factor for r_d <= 0.01): lean features (bearings formed on the device) and full
    features (bearings of api.ATANCamera.cam2world) must give the same bytes inside the disc, including its centre and a
    pixel with r_d == 0.01 exactly; a ring just outside it is compared with the oracle;
  * world2cam's cut-off (no distortion factor for r < 0.001): pairs whose points stay inside it in every pass must give
    the same bytes with d0 = 0.93 as with d0 = 0, one point projecting to r = 0 exactly;
  * d0 outside the values of the other tests: negative, 1e-9, 1.4 and 2.4, where some feature pixels lie past
    r_d d0 = pi/2 and tan changes sign (valid input: the reference takes such cameras).

The oracle is the reference's own SparseImgAlign through the stand-in camera where oracle/_ref is built, the restated
oracle (oracle/atan_oracle.cpp) otherwise; each case is solved once.  Tolerances and the rule for underdetermined pairs
are those of test_gpu_align_variants.py.  tests/test_atan_cpu.py checks without a GPU that every fixture here reaches the
branch it is built for."""
import copy
import math

import numpy as np
import pytest

from test_gpu_align import ROT_TOL, TRANS_TOL
from test_gpu_align_variants import VARIANTS, _check_all, _make
from test_gpu_atan import atan_for, through

pytestmark = pytest.mark.gpu

D0 = 0.93
FIELDS = ("T_cur_w", "n_tracked", "H", "seg_killed", "iters", "status", "patch_iters", "patch_levels")
VARIANT_CASES = ["vga_full", "vga_lean", "boundaries", "edge", "long_segments", "720p", "levels_5_3", "levels_2_0", "zero_motion",
                 "ragged_pairs_per_cta"]
D0_EDGES = [-0.3, 1e-9, 1.4, 2.4]


@pytest.fixture(scope="module")
def oracle_atan(abi):
    import oracle_atan

    oracle_atan.build()
    oracle_atan.load(abi)
    return oracle_atan


def solve(abi, oracle_atan, cam, data, hi, lo):
    """The oracle's result for `data` seen through `cam` (the reference's own code where oracle/_ref is built)."""
    fn = oracle_atan.ref_align if oracle_atan.ref_available() else oracle_atan.align
    return fn(abi, cam, data, abi.align_params(hi, lo, 30), n_threads=16)


# ------------------------------------------------------------------------------------------------
# fixtures (also checked without a GPU by tests/test_atan_cpu.py)
# ------------------------------------------------------------------------------------------------


def variant_case(pkg, synth, dev, name):
    """(camera, data, max_level, min_level) of a case of test_gpu_align_variants._make rendered through the ATAN camera
    with d0 = 0.93 of its image size.  vga_full ships the bearings, vga_lean does not."""
    data, hi, lo = _make("vga" if name.startswith("vga") else name, synth, dev, atan=lambda cam: atan_for(pkg, cam, D0))
    if name == "vga_lean":
        data = through(None, data, lean=True)
    return atan_for(pkg, data.cam, D0), data, hi, lo


NONSQUARE = (752, 480, 438.06, 384.0, 384.9, 233.5)  # width, height, fx_, fy_, cx_, cy_


def nonsquare_cameras(pkg, d0=D0):
    """The 752x480 camera with fx_ = 438.06, fy_ = 384, principal point (384.9, 233.5), and the same camera with fx and
    fy swapped."""
    w, h, fx, fy, cx, cy = NONSQUARE
    at = lambda a, b: pkg.ATANCamera(w, h, a / w, b / h, (cx + 0.5) / w, (cy + 0.5) / h, d0)
    return at(fx, fy), at(fy, fx)


def nonsquare_batch(pkg, synth, dev, track=False):
    cam = nonsquare_cameras(pkg)[0]
    size = synth.Camera(*NONSQUARE)  # the size only: frames and features go through `cam`
    if track:
        return synth.make_track_batch(cam=size, batch=24, n_pts=300, n_segs=60, seed=9150, device=dev, atan=cam)
    return synth.make_align_batch(cam=size, batch=24, n_pts=300, n_segs=60, seed=9100, device=dev, atan=cam)


def _telephoto(pkg, synth, fx_, d0):
    """A VGA-sized ATAN camera of focal length fx_ (pixels), principal point at the image centre, and a scene whose texture
    is scaled with it, so that the image looks like the VGA scene's: fine structure for the patches at any zoom."""
    cam = pkg.ATANCamera(640, 480, fx_ / 640, fx_ / 480, 0.5, 0.5, d0)
    scene = synth.Scene()
    scene.wvec = scene.wvec * (fx_ / 420.0)
    return cam, scene


def _relift(synth, data, cam, scene, pt_px, spx, epx):
    """Replace the batch's features by these pixels, lifted through `cam`'s rays onto the scene at the reference pose."""
    import torch

    R, t = synth.pose7_to_Rt(torch.tensor(data.T_ref_w))

    def lift(px):
        p = torch.tensor(px)
        d = synth.atan_rays(cam, p[..., 0], p[..., 1])
        return (np.ascontiguousarray(x) for x in ((d / d.norm(dim=-1, keepdim=True)).numpy(), scene.intersect(R, t, d).numpy()))

    data.pt_px, data.seg_spx, data.seg_epx = (np.ascontiguousarray(x) for x in (pt_px, spx, epx))
    data.pt_f, data.pt_pos = lift(pt_px)
    data.seg_sf, data.seg_spos = lift(spx)
    data.seg_ef, data.seg_epos = lift(epx)
    data.seg_length = np.ascontiguousarray(np.linalg.norm(epx - spx, axis=-1))
    return data


def _in_annulus(rng, shape, r0, r1, centre):
    """Pixels uniform in the annulus r0 <= |px - centre| <= r1 (pixels)."""
    rho = np.sqrt(rng.uniform(r0 * r0, r1 * r1, shape))
    phi = rng.uniform(0, 2 * math.pi, shape)
    return np.stack([centre[0] + rho * np.cos(phi), centre[1] + rho * np.sin(phi)], -1)


def rd_of(cam, px):
    """cam2world's distorted radius r_d of pixels, as api.ATANCamera and the kernel compute it."""
    px = np.asarray(px, np.float64)
    x, y = (px[..., 0] - cam.cx_) / cam.fx_, (px[..., 1] - cam.cy_) / cam.fy_
    return np.sqrt(x * x + y * y)


def rd_exactly_001(cam):
    """A pixel (u, cy_) whose r_d is 0.01 in double: stepped by nextafter from cx_ + 0.01 fx_."""
    u0 = cam.cx_ + 0.01 * cam.fx_
    up = down = u0
    for _ in range(64):
        for u in (up, down):
            if rd_of(cam, [u, cam.cy_]) == 0.01:
                return np.array([u, cam.cy_])
        up, down = np.nextafter(up, np.inf), np.nextafter(down, -np.inf)
    raise AssertionError("no pixel with r_d == 0.01 within 64 ulp of cx_ + 0.01 fx_")


C2W_FX = 4000.0  # the r_d <= 0.01 disc is 40 px wide in radius


def cam2world_disc_batch(pkg, synth, dev, ring=False):
    """(camera, data): every feature pixel (points and segment endpoints) has r_d <= 0.01 — pixel 0 of every pair at the
    principal point, pixel 1 at r_d == 0.01 exactly — or, with ring, 0.01 < r_d <= 0.011."""
    cam, scene = _telephoto(pkg, synth, C2W_FX, D0)
    s = 420.0 / C2W_FX
    data = synth.make_align_batch(batch=16, n_pts=120, n_segs=24, seed=9300 + ring, device=dev, atan=cam, scene=scene,
                                  motion_t=0.03 * s, motion_r=0.01 * s)
    rng = np.random.default_rng(9301 + ring)
    B, centre = data.batch, (cam.cx_, cam.cy_)
    r0, r1 = (0.01 * C2W_FX * 1.0005, 0.011 * C2W_FX * 0.9995) if ring else (0.0, 0.01 * C2W_FX * 0.999)
    pt_px = _in_annulus(rng, (B, data.n_pts), r0, r1, centre)
    spx, epx = (_in_annulus(rng, (B, data.n_segs), r0, r1, centre) for _ in range(2))
    if not ring:
        pt_px[:, 0] = centre
        pt_px[:, 1] = rd_exactly_001(cam)
    return cam, _relift(synth, data, cam, scene, pt_px, spx, epx)


W2C_FX = 80000.0  # the r < 0.0005 disc is 40 px wide in radius
W2C_R = 0.00045   # every feature pixel within this r_d (= r at the initial pose) of the principal point


def world2cam_disc_batch(pkg, synth, dev, d0=D0):
    """(camera, data): every point projects within r < 0.0005 of the principal point at the initial pose, with motion
    small enough that r stays below 0.001.  Pair 0 has the identity reference pose and its initial current pose moved
    along the optical axis, and its point 0 at (cx_, cy_): it projects to r = 0 exactly."""
    import torch

    cam, scene = _telephoto(pkg, synth, W2C_FX, d0)
    s = 420.0 / W2C_FX
    B = 12
    rng = np.random.default_rng(9400)
    xi_ref = np.concatenate([rng.uniform(-0.2, 0.2, (B, 3)), rng.uniform(-0.03, 0.03, (B, 3))], -1)
    xi_ref[0] = 0.0
    xi_mot = np.concatenate([rng.uniform(-0.03 * s, 0.03 * s, (B, 3)), rng.uniform(-0.01 * s, 0.01 * s, (B, 3))], -1)
    R_ref, t_ref = synth.se3_exp_Rt(torch.tensor(xi_ref))
    R_m, t_m = synth.se3_exp_Rt(torch.tensor(xi_mot))
    T_ref = synth.pose7_from_Rt(R_ref, t_ref).numpy()
    T_cur = synth.pose7_from_Rt(R_m @ R_ref, (R_m @ t_ref[..., None])[..., 0] + t_m).numpy()
    T_ref[0] = [0, 0, 0, 1, 0, 0, 0]
    data = synth.make_align_batch(batch=B, n_pts=96, n_segs=16, seed=9401, device=dev, atan=cam, scene=scene,
                                  T_ref_w_gt=T_ref, T_cur_w_gt=T_cur)
    data.T_cur_w[0] = [0, 0, 0, 1, 0, 0, 2e-4]  # moved along the optical axis: the centre pixel's point stays at r = 0
    centre = (cam.cx_, cam.cy_)
    r1 = W2C_R * W2C_FX
    pt_px = _in_annulus(rng, (B, data.n_pts), 0.0, r1, centre)
    pt_px[0, 0] = centre
    spx, epx = (_in_annulus(rng, (B, data.n_segs), 0.0, r1, centre) for _ in range(2))
    return cam, _relift(synth, data, cam, scene, pt_px, spx, epx)


def projected_r(data, T_cur_w):
    """r = |(x/z, y/z)| of every point and segment endpoint in the current frame at the poses T_cur_w [B, 7]."""
    import torch

    from plsvo_b200 import synth

    R, t = synth.pose7_to_Rt(torch.tensor(T_cur_w))
    out = []
    for P in (data.pt_pos, data.seg_spos, data.seg_epos):
        X = (torch.tensor(P) @ R.transpose(-1, -2) + t[:, None, :]).numpy()
        out.append(np.hypot(X[..., 0] / X[..., 2], X[..., 1] / X[..., 2]).reshape(data.batch, -1))
    return np.concatenate(out, 1)


def d0_edge_batch(pkg, synth, dev, d0):
    cam = atan_for(pkg, synth.VGA, d0)
    return cam, synth.make_align_batch(batch=24, n_pts=300, n_segs=60, seed=9500, device=dev, atan=cam)


def feature_px(data):
    return np.concatenate([data.pt_px.reshape(-1, 2), data.seg_spx.reshape(-1, 2), data.seg_epx.reshape(-1, 2)])


# ------------------------------------------------------------------------------------------------
# every variant
# ------------------------------------------------------------------------------------------------


@pytest.fixture(scope="module")
def case(pkg, abi, synth, oracle_atan, gen_device):
    """name -> (camera, data, max_level, min_level, oracle result), each built and solved once."""
    cache = {}

    def get(name):
        if name not in cache:
            cam, data, hi, lo = variant_case(pkg, synth, gen_device, name)
            cache[name] = (cam, data, hi, lo, solve(abi, oracle_atan, cam, data, hi, lo))
        return cache[name]

    return get


@pytest.mark.parametrize("name", VARIANT_CASES)
@pytest.mark.parametrize("variant", VARIANTS)
def test_every_atan_variant_matches_the_oracle(pkg, synth, case, monkeypatch, variant, name):
    cam, data, hi, lo, ref = case(name)
    monkeypatch.setenv("PLSVO_VARIANT", variant)
    al = pkg.SparseImgAlign(hi, lo, 30)
    if name == "ragged_pairs_per_cta":
        monkeypatch.setenv("PLSVO_CTAS_PER_SM", "1")
    gpu = al.run(data, camera=cam)
    if name == "zero_motion":  # NaN step on every pair: status 2, the pose stays where it was
        for f in ("status", "iters", "n_tracked", "seg_killed"):
            np.testing.assert_array_equal(getattr(gpu, f), getattr(ref, f), err_msg=f)
        assert (gpu.status == 2).all()
        for other in (ref.T_cur_w, data.T_cur_w):
            ang, rel = synth.pose_error(gpu.T_cur_w, other)
            assert ang.max() < 1e-12 and rel.max() < 1e-12, (ang.max(), rel.max())
        return
    _check_all(synth, data, gpu, ref)
    if name == "edge":
        assert gpu.status[3] == 1 and gpu.n_tracked[3] == 0
        np.testing.assert_array_equal(gpu.T_cur_w[3], data.T_cur_w[3])


# ------------------------------------------------------------------------------------------------
# non-square, off-centre camera
# ------------------------------------------------------------------------------------------------


@pytest.mark.parametrize("lean", [False, True])
def test_nonsquare_offcentre_camera_alignment(pkg, abi, synth, oracle_atan, gen_device, lean):
    cam = nonsquare_cameras(pkg)[0]
    data = through(cam, nonsquare_batch(pkg, synth, gen_device), lean)
    ref = solve(abi, oracle_atan, cam, data, 4, 2)
    gpu = pkg.SparseImgAlign(4, 2, 30).run(data, camera=cam)
    _check_all(synth, data, gpu, ref)
    assert gpu.n_tracked.min() > 0


def test_nonsquare_offcentre_camera_track(pkg, abi, synth, oracle, oracle_atan, gen_device):
    """The track call with the pose optimiser's errorMultiplier2 = fx_ (not fy_) of the non-square camera."""
    cam = nonsquare_cameras(pkg)[0]
    al, po = nonsquare_batch(pkg, synth, gen_device, track=True)
    al = through(cam, al, lean=False)
    po = copy.copy(po)
    po.fx = cam.errorMultiplier2()
    assert po.fx == cam.fx_ != cam.fy_
    ao, pout = pkg.api.track(al, po, camera=cam)
    ra = solve(abi, oracle_atan, cam, al, 4, 2)
    _check_all(synth, al, ao, ra)
    po3 = copy.copy(po)
    po3.T_f_w = np.ascontiguousarray(ra.T_cur_w)
    rp = oracle.poseopt(abi, po3, abi.poseopt_params(2.0, 10, -1), n_threads=16)
    ang, rel = synth.pose_error(pout.T_f_w, rp.T_f_w)
    assert ang.max() <= ROT_TOL and rel.max() <= TRANS_TOL, (ang.max(), rel.max())
    for f in ("num_obs_pt", "num_obs_ls", "pt_outlier", "seg_outlier", "iters", "status"):
        np.testing.assert_array_equal(getattr(pout, f), getattr(rp, f), err_msg=f)


# ------------------------------------------------------------------------------------------------
# the two cut-offs
# ------------------------------------------------------------------------------------------------


def test_cam2world_cutoff_lean_and_full_bearings_are_byte_identical(pkg, synth, gen_device):
    """Inside r_d <= 0.01 no distortion factor is applied: the bearings the kernel forms (lean) are those of
    api.ATANCamera.cam2world (full) bit for bit, so every output is the same byte for byte."""
    cam, data = cam2world_disc_batch(pkg, synth, gen_device)
    assert rd_of(cam, feature_px(data)).max() <= 0.01
    al = pkg.SparseImgAlign(4, 2, 30)
    lean = al.run(through(cam, data, lean=True), camera=cam)
    full = al.run(through(cam, data, lean=False), camera=cam)
    for f in FIELDS:
        np.testing.assert_array_equal(getattr(lean, f), getattr(full, f), err_msg=f)
    assert lean.n_tracked.min() > 0


@pytest.mark.parametrize("lean", [False, True])
def test_cam2world_ring_outside_the_cutoff_matches_the_oracle(pkg, abi, synth, oracle_atan, gen_device, lean):
    """Decisions exactly, poses within the tolerance.  H is not held to 1e-9 here: every feature lies in a cone of 0.011
    rad, where the last bits of the inputs move H far more: one ulp of the point bearings moves the oracle's own pose by
    6e-7 rad and its H by 2.7e-6 relative, and the kernel's H differs from the oracle's by 3e-6 (H100)."""
    cam, data = cam2world_disc_batch(pkg, synth, gen_device, ring=True)
    data = through(cam, data, lean)
    gpu = pkg.SparseImgAlign(4, 2, 30).run(data, camera=cam)
    ref = solve(abi, oracle_atan, cam, data, 4, 2)
    ang, rel = synth.pose_error(gpu.T_cur_w, ref.T_cur_w)
    assert ang.max() <= ROT_TOL and rel.max() <= TRANS_TOL, (ang.max(), rel.max())
    for f in ("n_tracked", "seg_killed", "status", "iters") + (("patch_iters", "patch_levels") if ref.patch_levels.any() else ()):
        np.testing.assert_array_equal(getattr(gpu, f), getattr(ref, f), err_msg=f)


def world2cam_inside_pairs(abi, oracle_atan, cam, flat, data):
    """Pairs whose projections stayed inside r < 0.001 in every pass of the oracle: its outputs with d0 = 0.93 and d0 = 0
    are the same bytes (just outside the cut-off the factor differs from 1 by tans_/s_ - 1 = 8 %).  The steps of these
    narrow-cone pairs are poorly conditioned, and a few of them leave the disc."""
    a, b = (oracle_atan.align(abi, c, data, n_threads=16) for c in (cam, flat))
    same = np.ones(data.batch, bool)
    for f in FIELDS:
        x, y = getattr(a, f), getattr(b, f)
        same &= np.array([np.array_equal(u, v) for u, v in zip(x, y)])
    # and the pose change bounds the last pass's projections: a pair that lost every point is the same bytes too
    return same & (projected_r(data, a.T_cur_w).max(1) < 0.001) & (a.n_tracked > 0), a


def test_world2cam_cutoff_d0_and_no_distortion_are_byte_identical(pkg, abi, synth, oracle_atan):
    """Inside r < 0.001 world2cam applies no distortion factor: on pairs whose projections stay there in every pass, d0 =
    0.93 and d0 = 0 give the same bytes.  Point 0 of pair 0 projects to r = 0 exactly (0/0 without the guard).  The batch
    is generated on the CPU so that the pairs are those tests/test_atan_cpu.py checks."""
    cam, data = world2cam_disc_batch(pkg, synth, "cpu")
    flat = _telephoto(pkg, synth, W2C_FX, 0.0)[0]
    data = through(cam, data, lean=False)
    inside, ref = world2cam_inside_pairs(abi, oracle_atan, cam, flat, data)
    assert inside[0] and inside.sum() >= data.batch // 2, inside
    assert projected_r(data, ref.T_cur_w)[inside].max() < 0.001
    al = pkg.SparseImgAlign(4, 2, 30)
    got, zero = al.run(data, camera=cam), al.run(data, camera=flat)
    for f in FIELDS:
        np.testing.assert_array_equal(getattr(got, f)[inside], getattr(zero, f)[inside], err_msg=f)
    assert got.n_tracked[inside].min() > 0


# ------------------------------------------------------------------------------------------------
# d0 edges
# ------------------------------------------------------------------------------------------------


@pytest.mark.parametrize("lean", [False, True])
@pytest.mark.parametrize("d0", D0_EDGES)
def test_d0_edges_match_the_oracle(pkg, abi, synth, oracle_atan, gen_device, d0, lean):
    cam, data = d0_edge_batch(pkg, synth, gen_device, d0)
    if d0 == 2.4:  # tan(r_d d0) changes sign for some feature pixels: valid input, as in the reference
        assert (rd_of(cam, feature_px(data)) * d0 > math.pi / 2).any()
    data = through(cam, data, lean)
    gpu = pkg.SparseImgAlign(4, 2, 30).run(data, camera=cam)
    ref = solve(abi, oracle_atan, cam, data, 4, 2)
    _check_all(synth, data, gpu, ref)
    assert np.isfinite(gpu.T_cur_w).all()
