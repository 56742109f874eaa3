"""Deterministic synthetic inputs for the PL-SVO hot path (SURVEY.md §8d).

The reference ships no dataset and no tests; these generators produce inputs with exact ground
truth: an analytic textured surface rendered by per-pixel ray/surface intersection, truncating
2x2 half-sample pyramids (vk::halfSample scalar path, called from src/frame.cpp:171-180),
reference-frame point / segment features with their exact 3D positions, and pose-optimiser
observation sets with noise and outliers.

Everything here is *input generation* (torch is used only as an array library so the same code
runs on the CPU for tests and on the GPU for the benchmark); nothing is on the product path.
"""
from __future__ import annotations

import math
from dataclasses import dataclass, field, replace

import numpy as np
import torch

# ------------------------------------------------------------------------------------------------
# cameras (SURVEY.md §8d)
# ------------------------------------------------------------------------------------------------


@dataclass(frozen=True)
class Camera:
    width: int
    height: int
    fx: float
    fy: float
    cx: float
    cy: float


VGA = Camera(640, 480, 420.0, 420.0, 319.5, 239.5)
HD720 = Camera(1280, 720, 840.0, 840.0, 639.5, 359.5)
QVGA = Camera(320, 240, 210.0, 210.0, 159.5, 119.5)  # small case for fast CPU tests
ODD = Camera(641, 479, 420.0, 420.0, 320.0, 239.0)  # odd sizes: no level is a multiple of 16 pixels wide
# 640x480 cameras with the published TUM RGB-D freiburg1/2/3 intrinsics: with VGA, the four of a mixed (multicam) batch
TUM_FR1 = Camera(640, 480, 517.3, 516.5, 318.6, 255.3)
TUM_FR2 = Camera(640, 480, 520.9, 521.0, 325.1, 249.7)
TUM_FR3 = Camera(640, 480, 535.4, 539.2, 320.1, 247.6)
MULTICAM_K4 = (VGA, TUM_FR1, TUM_FR2, TUM_FR3)


# ------------------------------------------------------------------------------------------------
# SE3 helpers (float64, batched).  Pose layout = [qx,qy,qz,qw,tx,ty,tz] as in include/plsvo_b200.h
# ------------------------------------------------------------------------------------------------


def _hat(w: torch.Tensor) -> torch.Tensor:
    z = torch.zeros_like(w[..., 0])
    return torch.stack(
        [
            torch.stack([z, -w[..., 2], w[..., 1]], -1),
            torch.stack([w[..., 2], z, -w[..., 0]], -1),
            torch.stack([-w[..., 1], w[..., 0], z], -1),
        ],
        -2,
    )


def se3_exp_Rt(xi: torch.Tensor):
    """xi [...,6] = (upsilon, omega) -> R [...,3,3], t [...,3]  (closed form, float64)."""
    ups, om = xi[..., :3], xi[..., 3:]
    th = om.norm(dim=-1, keepdim=True).clamp_min(1e-300)
    W = _hat(om)
    W2 = W @ W
    th2 = (th * th)[..., None]
    th_ = th[..., None]
    small = th_ < 1e-8
    a = torch.where(small, 1.0 - th2 / 6, torch.sin(th_) / th_)
    b = torch.where(small, 0.5 - th2 / 24, (1 - torch.cos(th_)) / th2)
    c = torch.where(small, 1.0 / 6 - th2 / 120, (th_ - torch.sin(th_)) / (th2 * th_))
    I = torch.eye(3, dtype=xi.dtype, device=xi.device).expand(W.shape)
    R = I + a * W + b * W2
    V = I + b * W + c * W2
    t = (V @ ups[..., None])[..., 0]
    return R, t


def R_to_quat(R: torch.Tensor) -> torch.Tensor:
    """Rotation matrices [...,3,3] -> unit quaternions [...,4] as (x,y,z,w), w >= 0 (small rotations)."""
    m = R
    w = 0.5 * torch.sqrt((1.0 + m[..., 0, 0] + m[..., 1, 1] + m[..., 2, 2]).clamp_min(1e-30))
    x = (m[..., 2, 1] - m[..., 1, 2]) / (4 * w)
    y = (m[..., 0, 2] - m[..., 2, 0]) / (4 * w)
    z = (m[..., 1, 0] - m[..., 0, 1]) / (4 * w)
    q = torch.stack([x, y, z, w], -1)
    return q / q.norm(dim=-1, keepdim=True)


def quat_to_R(q: torch.Tensor) -> torch.Tensor:
    x, y, z, w = q.unbind(-1)
    return torch.stack(
        [
            torch.stack([1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w)], -1),
            torch.stack([2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w)], -1),
            torch.stack([2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)], -1),
        ],
        -2,
    )


def pose7_from_Rt(R: torch.Tensor, t: torch.Tensor) -> torch.Tensor:
    return torch.cat([R_to_quat(R), t], -1)


def pose7_to_Rt(p: torch.Tensor):
    return quat_to_R(p[..., :4]), p[..., 4:]


def pose_error(p_a, p_b):
    """Parity metric of SURVEY.md §8d: (rotation angle of R_a R_b^T in rad, ||t_a-t_b|| / max(||t_b||,1e-12))."""
    p_a = torch.as_tensor(p_a, dtype=torch.float64)
    p_b = torch.as_tensor(p_b, dtype=torch.float64)
    Ra, ta = pose7_to_Rt(p_a)
    Rb, tb = pose7_to_Rt(p_b)
    dR = Ra @ Rb.transpose(-1, -2)
    # angle from the skew part (accurate for tiny angles)
    s = 0.5 * torch.stack([dR[..., 2, 1] - dR[..., 1, 2], dR[..., 0, 2] - dR[..., 2, 0], dR[..., 1, 0] - dR[..., 0, 1]], -1)
    sn = s.norm(dim=-1)
    cs = 0.5 * (dR[..., 0, 0] + dR[..., 1, 1] + dR[..., 2, 2] - 1.0)
    ang = torch.atan2(sn, cs)
    rel_t = (ta - tb).norm(dim=-1) / tb.norm(dim=-1).clamp_min(1e-12)
    return ang.numpy(), rel_t.numpy()


# ------------------------------------------------------------------------------------------------
# scene: Z(X,Y) = 2.0 + 0.15 sin(1.3X+0.4) cos(0.9Y), texture = 127 + sum_k a_k sin(w_k.(X,Y) + phi_k)
# ------------------------------------------------------------------------------------------------


@dataclass
class Scene:
    seed: int = 1001
    n_waves: int = 24
    amp: np.ndarray = field(init=False)
    wvec: np.ndarray = field(init=False)
    phase: np.ndarray = field(init=False)

    def __post_init__(self):
        rng = np.random.Generator(np.random.PCG64(self.seed))
        self.amp = rng.uniform(2.0, 10.0, self.n_waves)
        mag = rng.uniform(4.0, 60.0, self.n_waves)
        ang = rng.uniform(0.0, 2 * math.pi, self.n_waves)
        self.wvec = np.stack([mag * np.cos(ang), mag * np.sin(ang)], -1)
        self.phase = rng.uniform(0.0, 2 * math.pi, self.n_waves)

    @staticmethod
    def surface(X, Y):
        return 2.0 + 0.15 * torch.sin(1.3 * X + 0.4) * torch.cos(0.9 * Y)

    @staticmethod
    def surface_grad(X, Y):
        zx = 0.15 * 1.3 * torch.cos(1.3 * X + 0.4) * torch.cos(0.9 * Y)
        zy = -0.15 * 0.9 * torch.sin(1.3 * X + 0.4) * torch.sin(0.9 * Y)
        return zx, zy

    def texture(self, X, Y):
        I = torch.full_like(X, 127.0)
        for k in range(self.n_waves):
            I = I + float(self.amp[k]) * torch.sin(float(self.wvec[k, 0]) * X + float(self.wvec[k, 1]) * Y + float(self.phase[k]))
        return I

    def intersect(self, R_f_w, t_f_w, dirs_c):
        """World points where camera rays hit the surface.
        R_f_w [B,3,3], t_f_w [B,3], dirs_c [B,N,3] (camera-frame directions, z=1) -> P_w [B,N,3]."""
        Rt = R_f_w.transpose(-1, -2)
        C = -(Rt @ t_f_w[..., None])[..., 0]  # camera centre in world [B,3]
        d = dirs_c @ R_f_w  # rows: (R^T d_c)^T = d_c^T R  -> [B,N,3]
        lam = torch.full(d.shape[:-1], 2.0, dtype=d.dtype, device=d.device)
        Cx, Cy, Cz = C[:, None, 0], C[:, None, 1], C[:, None, 2]
        for _ in range(12):
            X = Cx + lam * d[..., 0]
            Y = Cy + lam * d[..., 1]
            g = Cz + lam * d[..., 2] - self.surface(X, Y)
            zx, zy = self.surface_grad(X, Y)
            gp = d[..., 2] - (zx * d[..., 0] + zy * d[..., 1])
            lam = lam - g / gp
        return torch.stack([Cx + lam * d[..., 0], Cy + lam * d[..., 1], Cz + lam * d[..., 2]], -1)

    def render(self, cam: Camera, pose7: torch.Tensor, chunk: int = 64, atan=None) -> torch.Tensor:
        """pose7 [B,7] (T_f_w) -> u8 images [B,H,W].  atan: an ATAN (FOV) camera (api.ATANCamera) of cam's size: each
        pixel's ray is then its cam2world (atan_rays) instead of the pinhole's."""
        dev = pose7.device
        B = pose7.shape[0]
        u = torch.arange(cam.width, dtype=torch.float64, device=dev)
        v = torch.arange(cam.height, dtype=torch.float64, device=dev)
        vv, uu = torch.meshgrid(v, u, indexing="ij")
        if atan is not None:
            dirs = atan_rays(atan, uu, vv).reshape(1, -1, 3)
        else:
            dirs = torch.stack([(uu - cam.cx) / cam.fx, (vv - cam.cy) / cam.fy, torch.ones_like(uu)], -1).reshape(1, -1, 3)
        out = torch.empty(B, cam.height, cam.width, dtype=torch.uint8, device=dev)
        for s in range(0, B, chunk):
            R, t = pose7_to_Rt(pose7[s : s + chunk])
            P = self.intersect(R, t, dirs.expand(R.shape[0], -1, -1))
            I = self.texture(P[..., 0], P[..., 1])
            out[s : s + chunk] = I.round().clamp(0, 255).to(torch.uint8).reshape(-1, cam.height, cam.width)
        return out


def atan_rays(atan, u: torch.Tensor, v: torch.Tensor) -> torch.Tensor:
    """Rays (x, y, 1) of pixels (u, v) of the ATAN (FOV) camera `atan` (api.ATANCamera): its cam2world scaled to z = 1.
    Scenes rendered and features lifted through these rays are what that camera sees, distortion included."""
    x, y = (u - atan.cx_) / atan.fx_, (v - atan.cy_) / atan.fy_
    rd = torch.sqrt(x * x + y * y)
    r = torch.tan(rd * atan.s_) * atan.tans_inv_ if atan.s_ != 0.0 else rd
    factor = torch.where(rd > 0.01, r / torch.where(rd > 0.01, rd, torch.ones_like(rd)), torch.ones_like(rd))
    return torch.stack([factor * x, factor * y, torch.ones_like(x)], -1)


def half_sample(img: torch.Tensor) -> torch.Tensor:
    """vk::halfSample, scalar path: truncating mean of each 2x2 block (u8 [B,H,W] -> [B,H/2,W/2])."""
    B, H, W = img.shape
    h, w = H // 2, W // 2
    x = img[:, : 2 * h, : 2 * w].to(torch.int32)
    s = x[:, 0::2, 0::2] + x[:, 0::2, 1::2] + x[:, 1::2, 0::2] + x[:, 1::2, 1::2]
    return (s // 4).to(torch.uint8)


def build_pyramid(img0: torch.Tensor, n_levels: int):
    """frame_utils::createImgPyramid (src/frame.cpp:171-180)."""
    pyr = [img0]
    for _ in range(1, n_levels):
        pyr.append(half_sample(pyr[-1]))
    return pyr


# ------------------------------------------------------------------------------------------------
# alignment batches
# ------------------------------------------------------------------------------------------------


@dataclass
class AlignData:
    """Host (numpy) arrays of one alignment batch, shaped as include/plsvo_b200.h describes."""

    cam: Camera
    max_level: int
    min_level: int
    ref_pyr: dict  # level -> u8 [B,h,w]
    cur_pyr: dict
    T_ref_w: np.ndarray  # [B,7]
    T_cur_w: np.ndarray  # [B,7] initial guess (= T_ref_w, frame_handler_mono.cpp:266)
    T_cur_w_gt: np.ndarray  # [B,7]
    pt_px: np.ndarray
    pt_f: np.ndarray
    pt_pos: np.ndarray
    seg_spx: np.ndarray
    seg_epx: np.ndarray
    seg_sf: np.ndarray
    seg_ef: np.ndarray
    seg_spos: np.ndarray
    seg_epos: np.ndarray
    seg_length: np.ndarray
    pt_valid: np.ndarray | None = None
    seg_valid: np.ndarray | None = None
    pt_count: np.ndarray | None = None
    seg_count: np.ndarray | None = None
    # frame chain (PLSVO_ALIGN_FRAME_CHAIN, include/plsvo_b200.h): level -> u8 [B+1,h,w]; pair b = (frame b, frame b+1).
    # When set, the ABI call ships this one stack instead of ref_pyr + cur_pyr.
    frame_pyr: dict | None = None

    @property
    def batch(self):
        return self.T_ref_w.shape[0]

    @property
    def n_pts(self):
        return self.pt_px.shape[1]

    @property
    def n_segs(self):
        return self.seg_spx.shape[1]


def _bearing(cam: Camera, px: torch.Tensor) -> torch.Tensor:
    """vk::PinholeCamera::cam2world: normalised ((u-cx)/fx, (v-cy)/fy, 1)."""
    d = torch.stack([(px[..., 0] - cam.cx) / cam.fx, (px[..., 1] - cam.cy) / cam.fy, torch.ones_like(px[..., 0])], -1)
    return d / d.norm(dim=-1, keepdim=True)


def make_align_batch(
    cam: Camera = VGA,
    batch: int = 8,
    n_pts: int = 300,
    n_segs: int = 80,
    max_level: int = 4,
    min_level: int = 2,
    n_pyr_levels: int | None = None,
    seed: int = 3000,
    device: str | torch.device = "cpu",
    motion_t: float = 0.03,
    motion_r: float = 0.01,
    margin: int | None = None,
    scene: Scene | None = None,
    keep_levels_only: bool = True,
    T_ref_w_gt: np.ndarray | None = None,
    T_cur_w_gt: np.ndarray | None = None,
    chain: bool = False,
    atan=None,
) -> AlignData:
    """SURVEY.md §8d config C2 generator: B independent frame pairs, each with its own reference view,
    features and motion (seeds derived from `seed`).  atan: an ATAN (FOV) camera (api.ATANCamera) of cam's size — the
    frames are rendered and the features lifted through it (bearings = its cam2world), so the batch is what that camera
    sees; `cam` then only gives the image size."""
    dev = torch.device(device)
    scene = scene or Scene()
    n_pyr_levels = n_pyr_levels or (max_level + 1)
    margin = margin if margin is not None else 4 * (1 << max_level)
    rng = np.random.Generator(np.random.PCG64(seed))
    f64 = dict(dtype=torch.float64, device=dev)

    # reference views: small random pose around the origin so that every pair sees different pixels
    xi_ref = np.concatenate([rng.uniform(-0.2, 0.2, (batch, 3)), rng.uniform(-0.03, 0.03, (batch, 3))], -1)
    xi_mot = np.concatenate([rng.uniform(-motion_t, motion_t, (batch, 3)), rng.uniform(-motion_r, motion_r, (batch, 3))], -1)
    R_ref, t_ref = se3_exp_Rt(torch.tensor(xi_ref, **f64))
    R_m, t_m = se3_exp_Rt(torch.tensor(xi_mot, **f64))
    R_cur = R_m @ R_ref  # T_cur_w = T_cur_from_ref * T_ref_w
    t_cur = (R_m @ t_ref[..., None])[..., 0] + t_m
    if T_ref_w_gt is not None:  # given poses (frame sequences): the random draws above keep the stream position
        R_ref, t_ref = pose7_to_Rt(torch.tensor(np.asarray(T_ref_w_gt), **f64))
        R_cur, t_cur = pose7_to_Rt(torch.tensor(np.asarray(T_cur_w_gt), **f64))
    T_ref_w = pose7_from_Rt(R_ref, t_ref)
    T_cur_w_gt = pose7_from_Rt(R_cur, t_cur)

    if chain:
        # one trajectory (the given poses satisfy T_ref_w_gt[b+1] == T_cur_w_gt[b]): every frame is rendered ONCE and the two
        # stacks are views of the one sequence, so "cur of pair b" and "ref of pair b+1" are the same bytes by construction
        # rather than by the renderer happening to be bit-reproducible across batch positions
        frames = build_pyramid(scene.render(cam, torch.cat([T_ref_w, T_cur_w_gt[-1:]], 0), atan=atan), n_pyr_levels)
        ref_pyr = [f[:-1] for f in frames]
        cur_pyr = [f[1:] for f in frames]
    else:
        ref0 = scene.render(cam, T_ref_w, atan=atan)
        cur0 = scene.render(cam, T_cur_w_gt, atan=atan)
        ref_pyr = build_pyramid(ref0, n_pyr_levels)
        cur_pyr = build_pyramid(cur0, n_pyr_levels)
    levels = range(min_level, max_level + 1) if keep_levels_only else range(n_pyr_levels)

    lo_u, hi_u = margin, cam.width - margin
    lo_v, hi_v = margin, cam.height - margin
    pt_px = np.stack([rng.uniform(lo_u, hi_u, (batch, n_pts)), rng.uniform(lo_v, hi_v, (batch, n_pts))], -1)
    # segments: start point uniform in the box, direction uniform, length U[60,240] clipped to the box
    spx = np.stack([rng.uniform(lo_u, hi_u, (batch, n_segs)), rng.uniform(lo_v, hi_v, (batch, n_segs))], -1)
    epx = np.empty_like(spx)
    max_len = min(240.0, 0.5 * min(hi_u - lo_u, hi_v - lo_v))
    min_len = min(60.0, 0.5 * max_len)
    for b in range(batch):
        for j in range(n_segs):
            while True:
                L = rng.uniform(min_len, max_len)
                a = rng.uniform(0, 2 * math.pi)
                e = spx[b, j] + L * np.array([math.cos(a), math.sin(a)])
                if lo_u <= e[0] < hi_u and lo_v <= e[1] < hi_v:
                    epx[b, j] = e
                    break

    def lift(px_np):
        px = torch.tensor(px_np, **f64)
        if atan is not None:
            d = atan_rays(atan, px[..., 0], px[..., 1])
            return d / d.norm(dim=-1, keepdim=True), scene.intersect(R_ref, t_ref, d)
        d = torch.stack([(px[..., 0] - cam.cx) / cam.fx, (px[..., 1] - cam.cy) / cam.fy, torch.ones_like(px[..., 0])], -1)
        return _bearing(cam, px), scene.intersect(R_ref, t_ref, d)

    pt_f, pt_pos = lift(pt_px)
    seg_sf, seg_spos = lift(spx)
    seg_ef, seg_epos = lift(epx)

    npy = lambda t: np.ascontiguousarray(t.detach().cpu().numpy())
    return AlignData(
        cam=cam,
        max_level=max_level,
        min_level=min_level,
        ref_pyr={l: npy(ref_pyr[l]) for l in levels},
        cur_pyr={l: npy(cur_pyr[l]) for l in levels},
        T_ref_w=npy(T_ref_w),
        T_cur_w=npy(T_ref_w).copy(),
        T_cur_w_gt=npy(T_cur_w_gt),
        pt_px=np.ascontiguousarray(pt_px),
        pt_f=npy(pt_f),
        pt_pos=npy(pt_pos),
        seg_spx=np.ascontiguousarray(spx),
        seg_epx=np.ascontiguousarray(epx),
        seg_sf=npy(seg_sf),
        seg_ef=npy(seg_ef),
        seg_spos=npy(seg_spos),
        seg_epos=npy(seg_epos),
        seg_length=np.ascontiguousarray(np.linalg.norm(epx - spx, axis=-1)),
    )


# ------------------------------------------------------------------------------------------------
# pose-optimiser batches (SURVEY.md §8d config C3)
# ------------------------------------------------------------------------------------------------


@dataclass
class PoseOptData:
    fx: float
    T_f_w: np.ndarray  # [B,7] initial (perturbed) pose
    T_f_w_gt: np.ndarray
    pt_f: np.ndarray
    pt_pos: np.ndarray
    pt_level: np.ndarray
    seg_line: np.ndarray
    seg_spos: np.ndarray
    seg_epos: np.ndarray
    seg_level: np.ndarray
    pt_valid: np.ndarray | None = None
    seg_valid: np.ndarray | None = None
    pt_count: np.ndarray | None = None
    seg_count: np.ndarray | None = None

    @property
    def batch(self):
        return self.T_f_w.shape[0]

    @property
    def n_pts(self):
        return self.pt_f.shape[1]

    @property
    def n_segs(self):
        return self.seg_line.shape[1]


def make_poseopt_batch(
    cam: Camera = VGA,
    batch: int = 8,
    n_pts: int = 300,
    n_segs: int = 80,
    seed: int = 5000,
    noise_px: float = 0.5,
    outlier_frac: float = 0.10,
    pert_t: float = 0.02,
    pert_r: float = 0.01,
    scene: Scene | None = None,
    T_gt: np.ndarray | None = None,
    max_level: int = 2,
) -> PoseOptData:
    """B frames; observations = GT projection + N(0,(noise_px/fx)^2) on the unit plane, 10 % outliers
    (U[5,30] px), level in {0, ..., max_level}; initial pose = exp(delta) * T_gt.  T_gt [B,7]: ground-truth poses to use (the
    chained align -> pose-opt case observes the features in the alignment's current frame)."""
    scene = scene or Scene()
    rng = np.random.Generator(np.random.PCG64(seed))
    f64 = dict(dtype=torch.float64)
    xi_gt = np.concatenate([rng.uniform(-0.2, 0.2, (batch, 3)), rng.uniform(-0.03, 0.03, (batch, 3))], -1)
    R_gt, t_gt = se3_exp_Rt(torch.tensor(xi_gt, **f64))
    if T_gt is not None:
        assert T_gt.shape == (batch, 7)
        R_gt, t_gt = pose7_to_Rt(torch.tensor(np.asarray(T_gt), **f64))
    xi_d = np.concatenate([rng.uniform(-pert_t, pert_t, (batch, 3)), rng.uniform(-pert_r, pert_r, (batch, 3))], -1)
    R_d, t_d = se3_exp_Rt(torch.tensor(xi_d, **f64))
    R0 = R_d @ R_gt
    t0 = (R_d @ t_gt[..., None])[..., 0] + t_d

    def world_points(px_np):
        px = torch.tensor(px_np, **f64)
        d = torch.stack([(px[..., 0] - cam.cx) / cam.fx, (px[..., 1] - cam.cy) / cam.fy, torch.ones_like(px[..., 0])], -1)
        return scene.intersect(R_gt, t_gt, d), d

    def perturb(uv1, n):
        """uv1 [B,n,3] unit-plane coords -> noisy, with outliers."""
        uv = uv1[..., :2].clone()
        uv += torch.tensor(rng.normal(0.0, noise_px / cam.fx, uv.shape), **f64)
        out = rng.uniform(0, 1, (batch, n)) < outlier_frac
        mag = rng.uniform(5.0, 30.0, (batch, n)) / cam.fx
        ang = rng.uniform(0, 2 * math.pi, (batch, n))
        off = torch.tensor(np.stack([mag * np.cos(ang), mag * np.sin(ang)], -1) * out[..., None], **f64)
        return uv + off

    m = 16
    pt_px = np.stack([rng.uniform(m, cam.width - m, (batch, n_pts)), rng.uniform(m, cam.height - m, (batch, n_pts))], -1)
    pt_pos, d = world_points(pt_px)
    uv = perturb(d, n_pts)
    f = torch.cat([uv, torch.ones_like(uv[..., :1])], -1)
    pt_f = f / f.norm(dim=-1, keepdim=True)
    pt_level = rng.integers(0, max_level + 1, (batch, n_pts)).astype(np.int32)

    spx = np.stack([rng.uniform(m, cam.width - m, (batch, n_segs)), rng.uniform(m, cam.height - m, (batch, n_segs))], -1)
    epx = np.stack([rng.uniform(m, cam.width - m, (batch, n_segs)), rng.uniform(m, cam.height - m, (batch, n_segs))], -1)
    seg_spos, ds = world_points(spx)
    seg_epos, de = world_points(epx)
    s_uv = perturb(ds, n_segs)
    e_uv = perturb(de, n_segs)
    sf = torch.cat([s_uv, torch.ones_like(s_uv[..., :1])], -1)
    ef = torch.cat([e_uv, torch.ones_like(e_uv[..., :1])], -1)
    sf = sf / sf.norm(dim=-1, keepdim=True)
    ef = ef / ef.norm(dim=-1, keepdim=True)
    line = torch.linalg.cross(sf, ef)  # src/feature.cpp:93-107
    line = line / torch.sqrt(line[..., 0:1] ** 2 + line[..., 1:2] ** 2)
    seg_level = rng.integers(0, max_level + 1, (batch, n_segs)).astype(np.int32)

    npy = lambda t: np.ascontiguousarray(t.detach().cpu().numpy())
    return PoseOptData(
        fx=cam.fx,
        T_f_w=npy(pose7_from_Rt(R0, t0)),
        T_f_w_gt=npy(pose7_from_Rt(R_gt, t_gt)),
        pt_f=npy(pt_f),
        pt_pos=npy(pt_pos),
        pt_level=pt_level,
        seg_line=npy(line),
        seg_spos=npy(seg_spos),
        seg_epos=npy(seg_epos),
        seg_level=seg_level,
    )


def make_track_batch(cam: Camera = VGA, batch: int = 8, n_pts: int = 300, n_segs: int = 80, seed: int = 3000,
                     device: str | torch.device = "cpu", **align_kw):
    """BASELINE config 4 ("combined align+pose path"): an alignment batch and, for every pair's current frame, a
    pose-optimiser batch whose features are observed at that frame's ground-truth pose (noise + outliers as in C3).
    Chained use: the pose optimiser starts from the alignment's result (frame_handler_mono.cpp:272-274 -> :327-329)."""
    al = make_align_batch(cam=cam, batch=batch, n_pts=n_pts, n_segs=n_segs, seed=seed, device=device, **align_kw)
    po = make_poseopt_batch(cam=cam, batch=batch, n_pts=n_pts, n_segs=n_segs, seed=seed + 7919, T_gt=al.T_cur_w_gt)
    return al, po


def scatter_batches(parts, index, batch: int):
    """One batch of `batch` entries from per-group batches of the same dataclass: entry index[k][i] of the result is
    entry i of parts[k].  Arrays of batch-first shape and dicts of them (pyramids) are scattered; the rest comes from
    parts[0]."""
    def merge(vals):
        v0 = vals[0]
        if isinstance(v0, dict):
            return {key: merge([v[key] for v in vals]) for key in v0}
        if isinstance(v0, np.ndarray):
            out = np.empty((batch,) + v0.shape[1:], v0.dtype)
            for v, idx in zip(vals, index):
                out[idx] = v
            return out
        return v0

    return type(parts[0])(**{f: merge([getattr(p, f) for p in parts]) for f in parts[0].__dataclass_fields__})


def take_pairs(data, idx):
    """Entries idx of a batch (AlignData or PoseOptData) as a batch of their own: every batch-first array attribute is
    sliced, the two-stack pyramids (ref_pyr, cur_pyr) included; the rest (the camera, fx) is shared.  A frame chain
    (frame_pyr set) raises ValueError: its stack has B+1 frames, so the pairs of a subset are not a chain."""
    import copy

    if getattr(data, "frame_pyr", None) is not None:
        raise ValueError("take_pairs does not take frame chains (frame_pyr): take the pairs of the two-stack batch")
    out = copy.copy(data)
    B = data.batch
    for f, v in vars(data).items():  # the dataclass fields and any array set on the instance (pt_depth, seg_sdepth, ...)
        if isinstance(v, dict):
            setattr(out, f, {k: np.ascontiguousarray(a[idx]) for k, a in v.items()})
        elif isinstance(v, np.ndarray) and v.shape[:1] == (B,):
            setattr(out, f, np.ascontiguousarray(v[idx]))
    return out


def merge_sizes(parts, index, slot: Camera | None = None, fill=0, raws=None):
    """One batch of pairs of several image sizes from one AlignData per size (part k's pairs go to positions index[k],
    as scatter_batches places them).  Every pair's frames sit in a slot of `slot`'s size (default: the largest width and
    height of the parts' cameras), the pair's own part.cam.width x height in its top-left corner: the layout of the
    multicam calls with `sizes=`.  The padding of every level is `fill`, a byte, or a numpy Generator for random bytes.
    raws: optionally one (ref, cur) pair of raw u8 [B_k, H_k, W_k] stacks per part, merged into slot-sized stacks the
    same way.  Frame chains are not merged (a chain's pairs share frames, so they have one size).  Returns (AlignData
    with cam = slot, sizes [B, 2] int32 of (width, height)), plus the merged (ref, cur) raw stacks when `raws` is given.
    Pose-optimiser batches have no images: scatter_batches merges them."""
    if any(getattr(p, "frame_pyr", None) is not None for p in parts):
        raise ValueError("merge_sizes does not take frame chains (frame_pyr)")
    if slot is None:
        c0 = parts[0].cam
        slot = Camera(max(p.cam.width for p in parts), max(p.cam.height for p in parts), c0.fx, c0.fy, c0.cx, c0.cy)
    if any(p.cam.width > slot.width or p.cam.height > slot.height for p in parts):
        raise ValueError("every part's camera must fit inside the slot")
    B = sum(len(i) for i in index)

    def pad(stacks, W, H):
        shape = (B, H, W)
        out = fill.integers(0, 256, shape, dtype=np.uint8) if isinstance(fill, np.random.Generator) else np.full(shape, fill, np.uint8)
        for s, idx in zip(stacks, index):
            out[np.asarray(idx), : s.shape[1], : s.shape[2]] = s
        return out

    al = scatter_batches([replace(p, ref_pyr={}, cur_pyr={}) for p in parts], index, B)
    levels = set.intersection(*(set(p.ref_pyr) for p in parts)) if parts[0].ref_pyr else set()
    al.ref_pyr = {l: pad([p.ref_pyr[l] for p in parts], slot.width >> l, slot.height >> l) for l in sorted(levels)}
    al.cur_pyr = {l: pad([p.cur_pyr[l] for p in parts], slot.width >> l, slot.height >> l) for l in sorted(levels)}
    al.cam = slot
    sizes = np.zeros((B, 2), np.int32)
    for p, idx in zip(parts, index):
        sizes[np.asarray(idx)] = (p.cam.width, p.cam.height)
    if raws is None:
        return al, sizes
    raw = tuple(pad([r[i] for r in raws], slot.width, slot.height) for i in range(2))
    return al, sizes, raw


def multicam_cameras(cams, cam_of_pair) -> np.ndarray:
    """[B, 4] (fx, fy, cx, cy) of every pair: row b is cams[cam_of_pair[b]] (the `cameras=` argument of the API)."""
    k = np.array([[c.fx, c.fy, c.cx, c.cy] for c in cams], np.float64)
    return np.ascontiguousarray(k[np.asarray(cam_of_pair)])


def make_multicam_batch(cams, cam_of_pair, n_pts: int = 300, n_segs: int = 80, seed: int = 3000, poseopt: bool = False,
                        **align_kw):
    """A mixed batch from several undistorted pinhole cameras of one image size: pair b is rendered and its features are
    lifted through cams[cam_of_pair[b]].  Each camera's pairs are one make_align_batch (make_track_batch when `poseopt`)
    of its own, scattered to their places in the batch.  Returns (AlignData, cameras [B, 4]) — AlignData.cam is cams[0]
    and gives only the image size — or (AlignData, PoseOptData, cameras) when `poseopt`; the pose optimiser of frame b
    then takes errorMultiplier2 = cameras[b, 0]."""
    cam_of_pair = np.asarray(cam_of_pair)
    if len({(c.width, c.height) for c in cams}) != 1:
        raise ValueError("every camera of a multicam batch has the same image size")
    groups = [np.flatnonzero(cam_of_pair == k) for k in range(len(cams))]
    used = [k for k in range(len(cams)) if len(groups[k])]
    al_parts, po_parts = [], []
    for k in used:
        kw = dict(cam=cams[k], batch=len(groups[k]), n_pts=n_pts, n_segs=n_segs, seed=seed + 104729 * k, **align_kw)
        if poseopt:
            al, po = make_track_batch(**kw)
            po_parts.append(po)
        else:
            al = make_align_batch(**kw)
        al_parts.append(al)
    B = len(cam_of_pair)
    index = [groups[k] for k in used]
    al = scatter_batches(al_parts, index, B)
    al.cam = cams[0]
    cameras = multicam_cameras(cams, cam_of_pair)
    if not poseopt:
        return al, cameras
    return al, scatter_batches(po_parts, index, B), cameras


def make_atan_multicam_batch(cams, cam_of_pair, slot: Camera | None = None, fill=0, poseopt: bool = False, n_pts: int = 300,
                             n_segs: int = 80, seed: int = 3000, **align_kw):
    """A batch of pairs from several ATAN (FOV) cameras (api.ATANCamera), of one size or several: pair b is rendered and its
    features are lifted through cams[cam_of_pair[b]] (make_align_batch(atan=), make_track_batch when `poseopt`), at that
    camera's size.  The per-camera parts are padded into one slot batch with merge_sizes (slot, fill as there).  Returns
    (AlignData, parts, groups), or (AlignData, PoseOptData, parts, po_parts, groups) when `poseopt`: parts[i] is the
    AlignData of camera used[i] = the i-th camera that has pairs, at its own size, and groups[i] the positions of its pairs
    in the batch.  The pose optimiser of frame b then takes errorMultiplier2 = its camera's fx_."""
    cam_of_pair = np.asarray(cam_of_pair)
    groups = [np.flatnonzero(cam_of_pair == k) for k in range(len(cams))]
    used = [k for k in range(len(cams)) if len(groups[k])]
    al_parts, po_parts = [], []
    for k in used:
        a = cams[k]
        cam = Camera(a.width, a.height, a.fx_, a.fy_, a.cx_, a.cy_)
        kw = dict(cam=cam, batch=len(groups[k]), n_pts=n_pts, n_segs=n_segs, seed=seed + 104729 * k, atan=a, **align_kw)
        if poseopt:
            al, po = make_track_batch(**kw)
            po.fx = a.errorMultiplier2()
            po_parts.append(po)
        else:
            al = make_align_batch(**kw)
        al_parts.append(al)
    index = [groups[k] for k in used]
    al, _ = merge_sizes(al_parts, index, slot=slot, fill=fill)
    if not poseopt:
        return al, al_parts, index
    return al, scatter_batches(po_parts, index, len(cam_of_pair)), al_parts, po_parts, index


def make_any_camera_batch(cams, cam_of_pair, slot: Camera | None = None, fill=0, poseopt: bool = False, n_pts: int = 300,
                          n_segs: int = 80, seed: int = 3000, **align_kw):
    """A batch of pairs from pinhole and ATAN (FOV) cameras (a sequence of Camera, the undistorted pinhole, and
    api.ATANCamera), of one size or several: pair b is rendered and its features are lifted through cams[cam_of_pair[b]]
    with that camera's own model at its own size (make_align_batch, with atan= for an ATAN camera; make_track_batch when
    `poseopt`).  The per-camera parts are padded into one slot batch with merge_sizes (slot, fill as there).  Returns
    what make_atan_multicam_batch returns: (AlignData, parts, groups), or (AlignData, PoseOptData, parts, po_parts,
    groups) when `poseopt`, parts[i] and groups[i] those of the i-th camera that has pairs.  The pose optimiser of frame b
    then takes errorMultiplier2 = |fx| of a pinhole camera, fx_ of an ATAN camera."""
    cam_of_pair = np.asarray(cam_of_pair)
    groups = [np.flatnonzero(cam_of_pair == k) for k in range(len(cams))]
    used = [k for k in range(len(cams)) if len(groups[k])]
    al_parts, po_parts = [], []
    for k in used:
        a = cams[k]
        if isinstance(a, Camera):
            cam, model = a, {}
        else:
            cam, model = Camera(a.width, a.height, a.fx_, a.fy_, a.cx_, a.cy_), {"atan": a}
        kw = dict(cam=cam, batch=len(groups[k]), n_pts=n_pts, n_segs=n_segs, seed=seed + 104729 * k, **model, **align_kw)
        if poseopt:
            al, po = make_track_batch(**kw)
            po.fx = abs(a.fx) if isinstance(a, Camera) else a.errorMultiplier2()
            po_parts.append(po)
        else:
            al = make_align_batch(**kw)
        al_parts.append(al)
    index = [groups[k] for k in used]
    al, _ = merge_sizes(al_parts, index, slot=slot, fill=fill)
    if not poseopt:
        return al, al_parts, index
    return al, scatter_batches(po_parts, index, len(cam_of_pair)), al_parts, po_parts, index


def make_sequence(cam: Camera = VGA, n_seq: int = 4, n_frames: int = 20, n_pts: int = 300, n_segs: int = 80, seed: int = 1000,
                  device: str | torch.device = "cpu", noise_px: float = 0.3, outlier_frac: float = 0.05):
    """BASELINE config 1 / SURVEY 8d C1: n_seq independent sequences of n_frames views along the smooth trajectory
    T_k = exp(k * (0.02, 0.005, 0.01, 0.004, -0.006, 0.002)) * T_0.  Returns the ground-truth poses [n_seq, n_frames, 7] and,
    for every step k = 1..n_frames-1, (AlignData, PoseOptData): the alignment of frame k-1 (reference, with its features)
    against frame k, and frame k's matched features for the pose optimiser.  A sequence driver overwrites the poses of
    each step with its own estimates (run_sequence)."""
    f64 = dict(dtype=torch.float64)
    rng = np.random.Generator(np.random.PCG64(seed))
    xi0 = np.concatenate([rng.uniform(-0.15, 0.15, (n_seq, 3)), rng.uniform(-0.02, 0.02, (n_seq, 3))], -1)
    R0, t0 = se3_exp_Rt(torch.tensor(xi0, **f64))
    step = np.array([0.02, 0.005, 0.01, 0.004, -0.006, 0.002])
    poses = np.zeros((n_seq, n_frames, 7))
    for k in range(n_frames):
        Rk, tk = se3_exp_Rt(torch.tensor(np.tile(k * step, (n_seq, 1)), **f64))
        poses[:, k] = pose7_from_Rt(Rk @ R0, (Rk @ t0[..., None])[..., 0] + tk).numpy()
    steps = []
    for k in range(1, n_frames):
        al = make_align_batch(cam=cam, batch=n_seq, n_pts=n_pts, n_segs=n_segs, seed=seed + 31 * k, device=device,
                              T_ref_w_gt=poses[:, k - 1], T_cur_w_gt=poses[:, k])
        po = make_poseopt_batch(cam=cam, batch=n_seq, n_pts=n_pts, n_segs=n_segs, seed=seed + 31 * k + 7, noise_px=noise_px,
                                outlier_frac=outlier_frac, T_gt=poses[:, k])
        steps.append((al, po))
    return poses, steps


def chain_frames(data: AlignData, levels=None) -> dict:
    """One stack of B+1 frames per level for a batch whose pairs are consecutive frames of one sequence
    (cur of pair b is the same image as ref of pair b+1; src/frame_handler_mono.cpp:176,272): level -> u8 [B+1,h,w].
    Raises if the batch is not such a chain."""
    out = {}
    for l in (levels if levels is not None else sorted(data.ref_pyr)):
        r, c = data.ref_pyr[l], data.cur_pyr[l]
        if not np.array_equal(c[:-1], r[1:]):
            raise ValueError("not a frame chain: cur image of pair b differs from the ref image of pair b+1")
        out[l] = np.ascontiguousarray(np.concatenate([r, c[-1:]], 0))
    return out


def make_chain_batch(cam: Camera = VGA, batch: int = 8, n_pts: int = 300, n_segs: int = 80, seed: int = 3000, step_t: float = 0.03,
                     step_r: float = 0.01, device: str | torch.device = "cpu", **kw) -> AlignData:
    """B pairs that replay ONE camera trajectory of B+1 frames: pair b aligns frame b+1 to frame b, starting (like
    FrameHandlerMono::processFrame, src/frame_handler_mono.cpp:266) from the previous frame's pose.  The two-stack arrays
    (ref_pyr / cur_pyr) are filled as usual, so the same object feeds the oracle; `chain_frames` gives the one-stack form."""
    rng = np.random.Generator(np.random.PCG64(seed + 77))
    f64 = dict(dtype=torch.float64)
    R, t = se3_exp_Rt(torch.tensor(np.concatenate([rng.uniform(-0.2, 0.2, 3), rng.uniform(-0.03, 0.03, 3)])[None], **f64))
    poses = [pose7_from_Rt(R, t)]
    # a bounded walk: steps of up to (step_t, step_r) whose drift is pulled back towards the start
    drift = np.zeros(6)
    for _ in range(batch):
        xi = np.concatenate([rng.uniform(-step_t, step_t, 3), rng.uniform(-step_r, step_r, 3)]) - 0.1 * drift
        drift += xi
        Rm, tm = se3_exp_Rt(torch.tensor(xi[None], **f64))
        R, t = Rm @ R, (Rm @ t[..., None])[..., 0] + tm
        poses.append(pose7_from_Rt(R, t))
    poses = torch.cat(poses, 0).numpy()
    return make_align_batch(cam=cam, batch=batch, n_pts=n_pts, n_segs=n_segs, seed=seed, device=device,
                            T_ref_w_gt=poses[:-1], T_cur_w_gt=poses[1:], chain=True, **kw)


# EuRoC's cam0 as config/dataset_params.yaml gives it: the undistorted pinhole camera and its Brown-Conrady coefficients
# (k1, k2, p1, p2, k3) = vk::PinholeCamera's d0..d4
EUROC = Camera(752, 480, 416.401549, 416.375319, 385.554786, 237.640332)
EUROC_DIST = (-0.27797, 0.060647, -0.002097, 0.000373, 0.0)


def undistort_points(cam: Camera, dist, u: torch.Tensor, v: torch.Tensor, iters: int = 20):
    """cv::undistortPoints for raw pixels (u, v) of the distorted pinhole camera `cam` with (k1, k2, p1, p2, k3) = dist:
    OpenCV's fixed-point iteration x = (x0 - delta(x)) / radial(x), in float64 -> normalised undistorted (x, y)."""
    k1, k2, p1, p2, k3 = (float(d) for d in dist)
    x0, y0 = (u - cam.cx) / cam.fx, (v - cam.cy) / cam.fy
    x, y = x0.clone(), y0.clone()
    for _ in range(iters):
        r2 = x * x + y * y
        icdist = 1.0 / (1.0 + ((k3 * r2 + k2) * r2 + k1) * r2)
        dx = 2.0 * p1 * x * y + p2 * (r2 + 2.0 * x * x)
        dy = p1 * (r2 + 2.0 * y * y) + 2.0 * p2 * x * y
        x, y = (x0 - dx) * icdist, (y0 - dy) * icdist
    return x, y


def render_distorted(scene: Scene, cam: Camera, dist, pose7: torch.Tensor, chunk: int = 64) -> torch.Tensor:
    """Raw frames of the analytic scene as a lens with Brown-Conrady distortion `dist` sees it: pose7 [B,7] (T_f_w) ->
    u8 [B,H,W].  Each raw pixel's ray is its undistorted normalised coordinate (undistort_points), so rectifying these
    frames with PinholeCamera(cam, *dist).undistortImage approximates Scene.render(cam, pose7) away from the border."""
    dev = pose7.device
    B = pose7.shape[0]
    u = torch.arange(cam.width, dtype=torch.float64, device=dev)
    v = torch.arange(cam.height, dtype=torch.float64, device=dev)
    vv, uu = torch.meshgrid(v, u, indexing="ij")
    x, y = undistort_points(cam, dist, uu, vv)
    dirs = torch.stack([x, y, torch.ones_like(x)], -1).reshape(1, -1, 3)
    out = torch.empty(B, cam.height, cam.width, dtype=torch.uint8, device=dev)
    for s in range(0, B, chunk):
        R, t = pose7_to_Rt(pose7[s : s + chunk])
        P = scene.intersect(R, t, dirs.expand(R.shape[0], -1, -1))
        I = scene.texture(P[..., 0], P[..., 1])
        out[s : s + chunk] = I.round().clamp(0, 255).to(torch.uint8).reshape(-1, cam.height, cam.width)
    return out


def make_raw_chain_batch(cam: Camera = EUROC, dist=EUROC_DIST, batch: int = 8, n_pts: int = 300, n_segs: int = 80,
                         seed: int = 3000, device: str | torch.device = "cpu", scene: Scene | None = None, **kw):
    """make_chain_batch whose frames are also rendered raw through a distorting lens: returns (AlignData, raw u8
    [B+1,H,W]).  Features, poses and ground truth are those of the undistorted camera `cam` (what the pipeline's
    handler sees after rectification); the AlignData's own pyramids are Scene.render's undistorted frames."""
    scene = scene or Scene()
    data = make_chain_batch(cam=cam, batch=batch, n_pts=n_pts, n_segs=n_segs, seed=seed, device=device, scene=scene, **kw)
    poses = torch.tensor(np.concatenate([data.T_ref_w, data.T_cur_w_gt[-1:]], 0), dtype=torch.float64, device=torch.device(device))
    raw = render_distorted(scene, cam, dist, poses)
    return data, np.ascontiguousarray(raw.cpu().numpy())


def make_raw_multicam_batch(cams, dists, cam_of_pair, n_pts: int = 300, n_segs: int = 80, seed: int = 3000,
                            poseopt: bool = False, scene: Scene | None = None, **align_kw):
    """make_multicam_batch whose frames are also rendered raw, each pair through its own lens: pair b's reference frame
    (at T_ref_w) and current frame (at the ground truth T_cur_w_gt) through cams[k] with Brown-Conrady distortion
    dists[k], k = cam_of_pair[b].  Features, poses and ground truth are those of the undistorted cameras.  Returns
    (AlignData, (ref_raw, cur_raw) u8 [B,H,W], cameras [B, 4]), or (AlignData, PoseOptData, raw, cameras) when
    `poseopt`."""
    scene = scene or Scene()
    cam_of_pair = np.asarray(cam_of_pair)
    out = make_multicam_batch(cams, cam_of_pair, n_pts=n_pts, n_segs=n_segs, seed=seed, poseopt=poseopt, scene=scene, **align_kw)
    al = out[0]
    B, cam = len(cam_of_pair), cams[0]
    ref = np.empty((B, cam.height, cam.width), np.uint8)
    cur = np.empty_like(ref)
    for k in np.unique(cam_of_pair):
        idx = np.flatnonzero(cam_of_pair == k)
        for poses, dst in ((al.T_ref_w, ref), (al.T_cur_w_gt, cur)):
            pose = torch.tensor(poses[idx], dtype=torch.float64, device=torch.device(align_kw.get("device", "cpu")))
            dst[idx] = render_distorted(scene, cams[k], dists[k], pose).cpu().numpy()
    return out[:-1] + ((ref, cur),) + out[-1:]


def make_raw_any_camera_batch(cams, cam_of_pair, slot: Camera | None = None, fill=0, poseopt: bool = False, n_pts: int = 300,
                              n_segs: int = 80, seed: int = 3000, scene: Scene | None = None, **align_kw):
    """A batch of raw pairs from distorted lenses (api.PinholeCamera) and ATAN (FOV) cameras (api.ATANCamera), of one size
    or several, for the raw any-camera calls.  A lens pair is make_raw_multicam_batch's: features, poses, ground truth and
    pyramids of the undistorted camera (the lens's size and fx..cy), its raw frames rendered through the lens
    (render_distorted).  An ATAN pair is make_any_camera_batch's, its raw frames the level 0 it renders through its model
    (the pipeline does not rectify FOV frames).  The per-camera parts and raw stacks are padded into one slot with
    merge_sizes (slot, fill as there).  Returns (AlignData, (ref_raw, cur_raw) u8 [B, H, W], parts, groups), or
    (AlignData, PoseOptData, raw, parts, po_parts, groups) when `poseopt`: parts[i] and groups[i] those of the i-th camera
    that has pairs.  The pose optimiser of frame b then takes errorMultiplier2 = |fx| of a lens, fx_ of an ATAN camera."""
    scene = scene or Scene()
    cam_of_pair = np.asarray(cam_of_pair)
    dev = torch.device(align_kw.get("device", "cpu"))
    groups = [np.flatnonzero(cam_of_pair == k) for k in range(len(cams))]
    used = [k for k in range(len(cams)) if len(groups[k])]
    al_parts, po_parts, raws = [], [], []
    for k in used:
        a = cams[k]
        atan = a if hasattr(a, "fx_") else None
        if atan is not None:
            cam = Camera(a.width, a.height, a.fx_, a.fy_, a.cx_, a.cy_)
        else:
            s = a.struct
            cam, dist = Camera(s.width, s.height, s.fx, s.fy, s.cx, s.cy), tuple(s.d)
        kw = dict(cam=cam, batch=len(groups[k]), n_pts=n_pts, n_segs=n_segs, seed=seed + 104729 * k, scene=scene, atan=atan,
                  **align_kw)
        if poseopt:
            al, po = make_track_batch(**kw)
            po.fx = a.errorMultiplier2() if atan is not None else abs(cam.fx)
            po_parts.append(po)
        else:
            al = make_align_batch(**kw)
        al_parts.append(al)
        pair = []
        for poses in (al.T_ref_w, al.T_cur_w_gt):
            pose = torch.tensor(poses, dtype=torch.float64, device=dev)
            img = scene.render(cam, pose, atan=atan) if atan is not None else render_distorted(scene, cam, dist, pose)
            pair.append(np.ascontiguousarray(img.cpu().numpy()))
        raws.append(tuple(pair))
    index = [groups[k] for k in used]
    al, _, raw = merge_sizes(al_parts, index, slot=slot, fill=fill, raws=raws)
    if not poseopt:
        return al, raw, al_parts, index
    return al, scatter_batches(po_parts, index, len(cam_of_pair)), raw, al_parts, po_parts, index


def run_sequence(poses, steps, track_fn):
    """The frame-to-frame chain of FrameHandlerMono::processFrame (src/frame_handler_mono.cpp:263-340) over a sequence:
    new_frame.T_f_w = last_frame.T_f_w (:266), sparse image alignment, pose optimisation, and the result becomes the
    reference pose of the next step.  track_fn(AlignData, PoseOptData) -> (AlignOut, PoseOptOut) runs one step (chained
    on the GPU, or the two reference calls on the CPU).  Returns estimated poses [n_seq, n_frames, 7], the per-step
    alignment iteration counts and pose-optimiser outlier flags."""
    import copy

    n_seq, n_frames = poses.shape[:2]
    est = np.zeros_like(poses)
    est[:, 0] = poses[:, 0]  # the first frame's pose is given
    iters, outliers = [], []
    for k, (al, po) in enumerate(steps, start=1):
        al = copy.copy(al)
        po = copy.copy(po)
        al.T_ref_w = np.ascontiguousarray(est[:, k - 1])
        al.T_cur_w = np.ascontiguousarray(est[:, k - 1])  # initial guess = last frame's pose (:266)
        po.T_f_w = np.ascontiguousarray(est[:, k - 1])    # placeholder; the step function starts from the aligned pose
        ao, pout = track_fn(al, po)
        est[:, k] = pout.T_f_w
        iters.append(ao.iters.copy())
        outliers.append(pout.pt_outlier.copy())
    return est, np.stack(iters, 1), np.stack(outliers, 1)


# ---- Matcher::findMatchDirect candidates (SURVEY §8f rank 1) -----------------------------------------
@dataclass
class MatchData:
    """Host arrays of one findMatchDirect batch, shaped as plsvo_match_batch describes."""

    cam: Camera
    n_pyr_levels: int
    ref_pyr: dict  # level -> u8 [n_ref,h,w]
    cur_pyr: dict  # level -> u8 [n_cur,h,w]
    T_ref_w: np.ndarray
    T_cur_w: np.ndarray
    ref_index: np.ndarray
    cur_index: np.ndarray
    ref_px: np.ndarray
    ref_f: np.ndarray
    ref_level: np.ndarray
    is_edgelet: np.ndarray
    ref_grad: np.ndarray
    pos: np.ndarray
    px_cur: np.ndarray
    px_cur_gt: np.ndarray
    n_iter: int = 10

    @property
    def n(self):
        return self.ref_index.shape[0]


def make_match_batch(cam: Camera = VGA, n: int = 2000, n_ref: int = 3, n_cur: int = 3, n_pyr_levels: int = 3, seed: int = 7000,
                     device: str | torch.device = "cpu", motion_t: float = 0.08, motion_r: float = 0.04,
                     edgelet_frac: float = 0.25, noise_px: float = 1.5, scene: Scene | None = None, atan=None) -> MatchData:
    """n reprojection candidates: a reference observation (keyframe r, pixel, bearing, level), its 3D point on the
    synthetic surface, and the projection into current frame c perturbed by up to `noise_px` (what the reprojector
    hands to findMatchDirect).  A few candidates sit at the image border / far outside to exercise the early-outs.
    atan: an ATAN (FOV) camera (api.ATANCamera) of cam's size.  Both pyramids are then rendered through it, the bearings
    are its cam2world and px_cur_gt its world2cam; the random draws are the same as without it."""
    dev = torch.device(device)
    scene = scene or Scene()
    rng = np.random.Generator(np.random.PCG64(seed))
    f64 = dict(dtype=torch.float64, device=dev)
    xi_ref = np.concatenate([rng.uniform(-0.2, 0.2, (n_ref, 3)), rng.uniform(-0.03, 0.03, (n_ref, 3))], -1)
    xi_cur = np.concatenate([rng.uniform(-0.2 - motion_t, 0.2 + motion_t, (n_cur, 3)), rng.uniform(-motion_r, motion_r, (n_cur, 3))], -1)
    xi_cur[:, 2] = rng.uniform(-0.05, 0.45, n_cur)  # some frames closer to the scene: search levels above 0
    R_ref, t_ref = se3_exp_Rt(torch.tensor(xi_ref, **f64))
    R_cur, t_cur = se3_exp_Rt(torch.tensor(xi_cur, **f64))
    T_ref_w, T_cur_w = pose7_from_Rt(R_ref, t_ref), pose7_from_Rt(R_cur, t_cur)
    ref_pyr = {l: np.ascontiguousarray(p.cpu().numpy()) for l, p in enumerate(build_pyramid(scene.render(cam, T_ref_w, atan=atan), n_pyr_levels))}
    cur_pyr = {l: np.ascontiguousarray(p.cpu().numpy()) for l, p in enumerate(build_pyramid(scene.render(cam, T_cur_w, atan=atan), n_pyr_levels))}
    ref_index = rng.integers(0, n_ref, n).astype(np.int32)
    cur_index = rng.integers(0, n_cur, n).astype(np.int32)
    ref_level = rng.integers(0, n_pyr_levels, n).astype(np.int32)
    ref_px = np.stack([rng.uniform(20, cam.width - 20, n), rng.uniform(20, cam.height - 20, n)], -1)
    k = min(8, n)
    ref_px[:k] = [[3.0, 50.0], [cam.width - 4.0, 50.0], [100.0, 2.0], [100.0, cam.height - 3.0], [6.0 * 4, 6.0 * 4],
                  [cam.width / 2, cam.height / 2], [7.9, 200.0], [cam.width - 7.0, cam.height - 7.0]][:k]
    px_t = torch.tensor(ref_px, **f64)
    if atan is None:
        d = torch.stack([(px_t[:, 0] - cam.cx) / cam.fx, (px_t[:, 1] - cam.cy) / cam.fy, torch.ones_like(px_t[:, 0])], -1)
        ref_f = d / d.norm(dim=-1, keepdim=True)
    else:
        d = atan_rays(atan, px_t[:, 0], px_t[:, 1])
        ref_f = torch.tensor(atan.cam2world(ref_px), **f64)
    ridx = torch.tensor(ref_index, device=dev, dtype=torch.long)
    cidx = torch.tensor(cur_index, device=dev, dtype=torch.long)
    pos = scene.intersect(R_ref[ridx], t_ref[ridx], d[:, None, :])[:, 0, :]
    p_cur = (R_cur[cidx] @ pos[..., None])[..., 0] + t_cur[cidx]
    if atan is None:
        px_gt = torch.stack([cam.fx * p_cur[:, 0] / p_cur[:, 2] + cam.cx, cam.fy * p_cur[:, 1] / p_cur[:, 2] + cam.cy], -1).cpu().numpy()
    else:
        px_gt = atan.world2cam(p_cur.cpu().numpy())
    px_cur = px_gt + rng.uniform(-noise_px, noise_px, (n, 2))
    is_edgelet = (rng.uniform(size=n) < edgelet_frac).astype(np.uint8)
    ang = rng.uniform(0, 2 * math.pi, n)
    ref_grad = np.stack([np.cos(ang), np.sin(ang)], -1)
    c = lambda a, t: np.ascontiguousarray(a.cpu().numpy() if isinstance(a, torch.Tensor) else a, dtype=t)  # noqa: E731
    return MatchData(cam=cam, n_pyr_levels=n_pyr_levels, ref_pyr=ref_pyr, cur_pyr=cur_pyr, T_ref_w=c(T_ref_w, np.float64),
                     T_cur_w=c(T_cur_w, np.float64), ref_index=ref_index, cur_index=cur_index, ref_px=c(ref_px, np.float64),
                     ref_f=c(ref_f, np.float64), ref_level=ref_level, is_edgelet=is_edgelet, ref_grad=c(ref_grad, np.float64),
                     pos=c(pos, np.float64), px_cur=c(px_cur, np.float64), px_cur_gt=c(px_gt, np.float64))


def make_match_multicam_batch(cams, cam_of_ref, cam_of_cur, n: int = 2000, n_pyr_levels: int = 3, seed: int = 7100,
                              device: str | torch.device = "cpu", slot: Camera | None = None, fill=0, same_camera_frac: float = 0.5,
                              motion_t: float = 0.08, motion_r: float = 0.04, edgelet_frac: float = 0.25, noise_px: float = 1.5,
                              scene: Scene | None = None):
    """n reprojection candidates over keyframes and current frames from several cameras, the batch of
    plsvo_match_direct_multicam_batch_run.  cams: undistorted pinholes (Camera) or ATAN cameras (api.ATANCamera), of any
    sizes; ref image r is seen through cams[cam_of_ref[r]] and current image c through cams[cam_of_cur[c]].  Every image
    is rendered through its own camera at that camera's size and padded into a slot of `slot`'s size (default: the largest
    width and height), in the top-left corner, as merge_sizes pads; the padding is `fill`, a byte or a numpy Generator
    for random bytes.  Each reference pixel lies inside its ref camera's size (the first few on its borders), its bearing is
    that camera's cam2world and px_cur_gt the current camera's world2cam.  A share `same_camera_frac` of the candidates
    picks a current image of its keyframe's camera where one exists; the others pick any, so many pair two cameras.
    Returns (MatchData with cam = slot, parts, groups): for camera k, groups[k] are the positions of the candidates whose
    two images are both seen through cams[k], and parts[k] their one-camera MatchData, its images cut out of the slots
    at k's own size (None when groups[k] is empty)."""
    dev = torch.device(device)
    scene = scene or Scene()
    rng = np.random.Generator(np.random.PCG64(seed))
    f64 = dict(dtype=torch.float64, device=dev)
    cam_of_ref, cam_of_cur = np.asarray(cam_of_ref, np.int32), np.asarray(cam_of_cur, np.int32)
    n_ref, n_cur = len(cam_of_ref), len(cam_of_cur)
    is_atan = [hasattr(c, "s_") for c in cams]
    size = [Camera(c.width, c.height, 1.0, 1.0, 0.0, 0.0) for c in cams]
    if slot is None:
        slot = Camera(max(c.width for c in cams), max(c.height for c in cams), 1.0, 1.0, 0.0, 0.0)
    if any(c.width > slot.width or c.height > slot.height for c in cams):
        raise ValueError("every camera must fit inside the slot")
    xi_ref = np.concatenate([rng.uniform(-0.2, 0.2, (n_ref, 3)), rng.uniform(-0.03, 0.03, (n_ref, 3))], -1)
    xi_cur = np.concatenate([rng.uniform(-0.2 - motion_t, 0.2 + motion_t, (n_cur, 3)), rng.uniform(-motion_r, motion_r, (n_cur, 3))], -1)
    xi_cur[:, 2] = rng.uniform(-0.05, 0.45, n_cur)
    R_ref, t_ref = se3_exp_Rt(torch.tensor(xi_ref, **f64))
    R_cur, t_cur = se3_exp_Rt(torch.tensor(xi_cur, **f64))
    T_ref_w, T_cur_w = pose7_from_Rt(R_ref, t_ref), pose7_from_Rt(R_cur, t_cur)

    def pyramids(T, cam_of):
        pyr = {l: (fill.integers(0, 256, (len(cam_of), slot.height >> l, slot.width >> l), dtype=np.uint8)
                   if isinstance(fill, np.random.Generator) else np.full((len(cam_of), slot.height >> l, slot.width >> l), fill, np.uint8))
               for l in range(n_pyr_levels)}
        for k in np.unique(cam_of):
            idx = np.flatnonzero(cam_of == k)
            img = scene.render(cams[k] if not is_atan[k] else size[k], T[torch.as_tensor(idx, device=dev)],
                               atan=cams[k] if is_atan[k] else None)
            for l, p in enumerate(build_pyramid(img, n_pyr_levels)):
                pyr[l][idx, : p.shape[1], : p.shape[2]] = p.cpu().numpy()
        return pyr

    ref_pyr, cur_pyr = pyramids(T_ref_w, cam_of_ref), pyramids(T_cur_w, cam_of_cur)
    ref_index = rng.integers(0, n_ref, n).astype(np.int32)
    cur_index = rng.integers(0, n_cur, n).astype(np.int32)
    same = rng.uniform(size=n) < same_camera_frac
    for i in np.flatnonzero(same):
        mine = np.flatnonzero(cam_of_cur == cam_of_ref[ref_index[i]])
        if len(mine):
            cur_index[i] = mine[rng.integers(0, len(mine))]
    ref_level = rng.integers(0, n_pyr_levels, n).astype(np.int32)
    kr, kc = cam_of_ref[ref_index], cam_of_cur[cur_index]
    W = np.array([c.width for c in cams], np.float64)
    H = np.array([c.height for c in cams], np.float64)
    ref_px = np.stack([rng.uniform(20, W[kr] - 20), rng.uniform(20, H[kr] - 20)], -1)
    k = min(8, n)  # the borders of the ref camera, as make_match_batch places them in its one camera
    w, h = W[kr[:8]], H[kr[:8]]
    if k == 8:
        ref_px[:8] = np.stack([[3.0, w[1] - 4.0, 100.0, 100.0, 24.0, w[5] / 2, 7.9, w[7] - 7.0],
                               [50.0, 50.0, 2.0, h[3] - 3.0, 24.0, h[5] / 2, 200.0, h[7] - 7.0]], -1)
    d = torch.empty(n, 3, **f64)
    ref_f = np.empty((n, 3))
    for kk in np.unique(kr):
        sel = np.flatnonzero(kr == kk)
        c = cams[kk]
        px_t = torch.tensor(ref_px[sel], **f64)
        if is_atan[kk]:
            d[sel] = atan_rays(c, px_t[:, 0], px_t[:, 1])
            ref_f[sel] = c.cam2world(ref_px[sel])
        else:
            dd = torch.stack([(px_t[:, 0] - c.cx) / c.fx, (px_t[:, 1] - c.cy) / c.fy, torch.ones_like(px_t[:, 0])], -1)
            d[sel] = dd
            ref_f[sel] = (dd / dd.norm(dim=-1, keepdim=True)).cpu().numpy()
    ridx = torch.tensor(ref_index, device=dev, dtype=torch.long)
    cidx = torch.tensor(cur_index, device=dev, dtype=torch.long)
    pos = scene.intersect(R_ref[ridx], t_ref[ridx], d[:, None, :])[:, 0, :]
    p_cur = ((R_cur[cidx] @ pos[..., None])[..., 0] + t_cur[cidx]).cpu().numpy()
    px_gt = np.empty((n, 2))
    for kk in np.unique(kc):
        sel = np.flatnonzero(kc == kk)
        c = cams[kk]
        if is_atan[kk]:
            px_gt[sel] = c.world2cam(p_cur[sel])
        else:
            px_gt[sel] = np.stack([c.fx * p_cur[sel, 0] / p_cur[sel, 2] + c.cx, c.fy * p_cur[sel, 1] / p_cur[sel, 2] + c.cy], -1)
    px_cur = px_gt + rng.uniform(-noise_px, noise_px, (n, 2))
    is_edgelet = (rng.uniform(size=n) < edgelet_frac).astype(np.uint8)
    ang = rng.uniform(0, 2 * math.pi, n)
    ref_grad = np.stack([np.cos(ang), np.sin(ang)], -1)
    c64 = lambda a: np.ascontiguousarray(a.cpu().numpy() if isinstance(a, torch.Tensor) else a, dtype=np.float64)  # noqa: E731
    data = MatchData(cam=slot, n_pyr_levels=n_pyr_levels, ref_pyr=ref_pyr, cur_pyr=cur_pyr, T_ref_w=c64(T_ref_w), T_cur_w=c64(T_cur_w),
                     ref_index=ref_index, cur_index=cur_index, ref_px=c64(ref_px), ref_f=c64(ref_f), ref_level=ref_level,
                     is_edgelet=is_edgelet, ref_grad=c64(ref_grad), pos=c64(pos), px_cur=c64(px_cur), px_cur_gt=c64(px_gt))
    groups, parts = [], []
    for kk, c in enumerate(cams):
        g = np.flatnonzero((kr == kk) & (kc == kk))
        groups.append(g)
        if not len(g):
            parts.append(None)
            continue
        refs, curs = np.flatnonzero(cam_of_ref == kk), np.flatnonzero(cam_of_cur == kk)
        rmap, cmap = np.full(n_ref, -1, np.int32), np.full(n_cur, -1, np.int32)
        rmap[refs], cmap[curs] = np.arange(len(refs)), np.arange(len(curs))
        one = c if not is_atan[kk] else Camera(c.width, c.height, c.fx_, c.fy_, c.cx_, c.cy_)
        parts.append(MatchData(cam=one, n_pyr_levels=n_pyr_levels,
                               ref_pyr={l: im[refs][:, : c.height >> l, : c.width >> l] for l, im in ref_pyr.items()},
                               cur_pyr={l: im[curs][:, : c.height >> l, : c.width >> l] for l, im in cur_pyr.items()},
                               T_ref_w=data.T_ref_w[refs], T_cur_w=data.T_cur_w[curs], ref_index=rmap[ref_index[g]],
                               cur_index=cmap[cur_index[g]], ref_px=data.ref_px[g], ref_f=data.ref_f[g], ref_level=ref_level[g],
                               is_edgelet=is_edgelet[g], ref_grad=data.ref_grad[g], pos=data.pos[g], px_cur=data.px_cur[g],
                               px_cur_gt=data.px_cur_gt[g]))
    return data, parts, groups


# ---- structure optimisation: Point::optimize / LineSeg::optimize (SURVEY §8f rank 3) -------------------
@dataclass
class StructOptData:
    """Host arrays of one structure-optimisation batch, shaped as plsvo_structopt_batch describes."""

    T_f_w: np.ndarray
    pt_obs_begin: np.ndarray
    pt_obs_frame: np.ndarray
    pt_obs_f: np.ndarray
    pt_pos: np.ndarray
    pt_pos_gt: np.ndarray
    seg_obs_begin: np.ndarray
    seg_obs_frame: np.ndarray
    seg_obs_sf: np.ndarray
    seg_obs_ef: np.ndarray
    seg_spos: np.ndarray
    seg_epos: np.ndarray
    seg_spos_gt: np.ndarray
    seg_epos_gt: np.ndarray
    n_iter_pts: int = 5
    n_iter_segs: int = 5


def make_structopt_batch(n_points: int = 2000, n_segs: int = 500, n_frames: int = 12, max_obs: int = 10, seed: int = 8000,
                         noise: float = 1e-3, pert: float = 0.05, cam: Camera = VGA) -> StructOptData:
    """3D points / segments around z ~ 2 observed from n_frames keyframes on a small baseline; observations are unit
    bearing vectors of the true position with unit-plane noise `noise`; the entry position is perturbed by `pert`.
    A few features get a single observation (rank-deficient normal equations) or coincident views."""
    rng = np.random.Generator(np.random.PCG64(seed))
    xi = np.concatenate([rng.uniform(-0.4, 0.4, (n_frames, 3)) * [1, 1, 0.2], rng.uniform(-0.05, 0.05, (n_frames, 3))], -1)
    R, t = se3_exp_Rt(torch.tensor(xi, dtype=torch.float64))
    T = pose7_from_Rt(R, t).numpy()
    R, t = R.numpy(), t.numpy()

    def observe(P, frames):  # P [3], frames [k] -> unit bearings [k,3]
        pc = (R[frames] @ P) + t[frames]
        uv = pc[:, :2] / pc[:, 2:3] + rng.normal(0, noise, (len(frames), 2))
        d = np.concatenate([uv, np.ones((len(frames), 1))], -1)
        return d / np.linalg.norm(d, axis=-1, keepdims=True)

    def world_points(n):
        return np.stack([rng.uniform(-1.2, 1.2, n), rng.uniform(-0.9, 0.9, n), rng.uniform(1.5, 3.0, n)], -1)

    def csr(n, gt_list):
        begin, frame, obs = [0], [], [[] for _ in gt_list]
        for i in range(n):
            k = int(rng.integers(2, max_obs + 1))
            if i % 97 == 5:
                k = 1  # single observation: singular A, the pivoted LDLT still returns a step
            fr = rng.choice(n_frames, size=min(k, n_frames), replace=False)
            if i % 97 == 11:
                fr = np.repeat(fr[:1], 3)  # the same view three times
            frame.extend(fr.tolist())
            for g, o in zip(gt_list, obs):
                o.append(observe(g[i], fr))
            begin.append(len(frame))
        cat = lambda o: np.ascontiguousarray(np.concatenate(o, 0)) if o else np.zeros((0, 3))  # noqa: E731
        return (np.asarray(begin, np.int32), np.asarray(frame, np.int32), [cat(o) for o in obs])

    P = world_points(n_points)
    pb, pf, (pobs,) = csr(n_points, [P])
    S, E = world_points(n_segs), None
    E = S + rng.uniform(-0.3, 0.3, (n_segs, 3)) * [1, 1, 0.3]
    sb, sf_, (sobs, eobs) = csr(n_segs, [S, E])
    c = np.ascontiguousarray
    return StructOptData(T_f_w=c(T), pt_obs_begin=pb, pt_obs_frame=pf, pt_obs_f=pobs, pt_pos=c(P + rng.normal(0, pert, P.shape)),
                         pt_pos_gt=c(P), seg_obs_begin=sb, seg_obs_frame=sf_, seg_obs_sf=sobs, seg_obs_ef=eobs,
                         seg_spos=c(S + rng.normal(0, pert, S.shape)), seg_epos=c(E + rng.normal(0, pert, E.shape)),
                         seg_spos_gt=c(S), seg_epos_gt=c(E))


# ---- depth-filter point seeds (SURVEY §8f rank 4) ---------------------------------------------------------
@dataclass
class SeedData:
    """Host arrays of one depth-filter seed batch, shaped as plsvo_seed_batch describes."""

    cam: Camera
    n_pyr_levels: int
    ref_pyr: dict
    cur_pyr: dict
    T_ref_w: np.ndarray
    T_cur_w: np.ndarray
    ref_index: np.ndarray
    cur_index: np.ndarray
    ref_px: np.ndarray
    ref_f: np.ndarray
    ref_level: np.ndarray
    is_edgelet: np.ndarray
    ref_grad: np.ndarray
    a: np.ndarray
    b: np.ndarray
    mu: np.ndarray
    z_range: np.ndarray
    sigma2: np.ndarray
    depth_gt: np.ndarray
    n_iter: int = 10
    max_epi_search_steps: int = 1000
    align_1d: bool = False
    subpix_refinement: bool = True
    edgelet_filtering: bool = True
    edgelet_max_angle: float = 0.7
    convergence_thresh: float = 200.0

    @property
    def n(self):
        return self.ref_index.shape[0]


def make_seed_batch(cam: Camera = VGA, n: int = 2000, n_ref: int = 3, n_cur: int = 3, n_pyr_levels: int = 3, seed: int = 9000,
                    device: str | torch.device = "cpu", baseline: float = 0.12, edgelet_frac: float = 0.2,
                    scene: Scene | None = None) -> SeedData:
    """n depth-filter seeds: a feature in keyframe r (pixel, bearing, level), a Gaussian x Beta prior on its inverse
    depth at various stages of convergence (so that epipolar segments range from sub-pixel to hundreds of pixels),
    and a current frame c a small baseline away.  A few seeds are invisible in c, far outside or nearly converged."""
    dev = torch.device(device)
    scene = scene or Scene()
    rng = np.random.Generator(np.random.PCG64(seed))
    f64 = dict(dtype=torch.float64, device=dev)
    xi_ref = np.concatenate([rng.uniform(-0.15, 0.15, (n_ref, 3)), rng.uniform(-0.03, 0.03, (n_ref, 3))], -1)
    xi_cur = np.concatenate([rng.uniform(-0.15 - baseline, 0.15 + baseline, (n_cur, 3)), rng.uniform(-0.04, 0.04, (n_cur, 3))], -1)
    xi_cur[:, 2] = rng.uniform(-0.05, 0.15, n_cur)
    R_ref, t_ref = se3_exp_Rt(torch.tensor(xi_ref, **f64))
    R_cur, t_cur = se3_exp_Rt(torch.tensor(xi_cur, **f64))
    T_ref_w, T_cur_w = pose7_from_Rt(R_ref, t_ref), pose7_from_Rt(R_cur, t_cur)
    ref_pyr = {l: np.ascontiguousarray(p.cpu().numpy()) for l, p in enumerate(build_pyramid(scene.render(cam, T_ref_w), n_pyr_levels))}
    cur_pyr = {l: np.ascontiguousarray(p.cpu().numpy()) for l, p in enumerate(build_pyramid(scene.render(cam, T_cur_w), n_pyr_levels))}
    ref_index = rng.integers(0, n_ref, n).astype(np.int32)
    cur_index = rng.integers(0, n_cur, n).astype(np.int32)
    ref_level = rng.integers(0, n_pyr_levels, n).astype(np.int32)
    ref_px = np.stack([rng.uniform(24, cam.width - 24, n), rng.uniform(24, cam.height - 24, n)], -1)
    px_t = torch.tensor(ref_px, **f64)
    d = torch.stack([(px_t[:, 0] - cam.cx) / cam.fx, (px_t[:, 1] - cam.cy) / cam.fy, torch.ones_like(px_t[:, 0])], -1)
    ref_f = d / d.norm(dim=-1, keepdim=True)
    ridx = torch.tensor(ref_index, device=dev, dtype=torch.long)
    pos = scene.intersect(R_ref[ridx], t_ref[ridx], d[:, None, :])[:, 0, :]
    p_ref = (R_ref[ridx] @ pos[..., None])[..., 0] + t_ref[ridx]
    depth = p_ref.norm(dim=-1).cpu().numpy()  # distance along the unit bearing
    z_range = np.full(n, 1.0 / 1.2, np.float32)  # 1 / depth_min of the scene
    stage = rng.uniform(0.0, 3.0, n)  # decades of variance reduction already achieved
    sigma2 = (z_range.astype(np.float64) ** 2 / 36.0 * 10.0 ** (-stage)).astype(np.float32)
    mu = (1.0 / depth + rng.normal(0, 1, n) * np.sqrt(sigma2) * 0.5).astype(np.float32)
    mu = np.maximum(mu, 0.05).astype(np.float32)
    a = (10.0 + rng.uniform(0, 20, n)).astype(np.float32)
    b = (10.0 + rng.uniform(0, 5, n)).astype(np.float32)
    k = min(6, n)
    mu[:k] = [1e-3, 5.0, 0.4, 0.5, 0.45, 0.6][:k]        # far beyond the scene / in front of it / plausible
    sigma2[:k] = [1e-8, 1e-4, 1e-9, 2e-2, 1e-12, 4e-2][:k]  # already converged ... very uncertain (long epipolar segments)
    is_edgelet = (rng.uniform(size=n) < edgelet_frac).astype(np.uint8)
    ang = rng.uniform(0, 2 * math.pi, n)
    ref_grad = np.stack([np.cos(ang), np.sin(ang)], -1)
    c = lambda x, t: np.ascontiguousarray(x.cpu().numpy() if isinstance(x, torch.Tensor) else x, dtype=t)  # noqa: E731
    return SeedData(cam=cam, n_pyr_levels=n_pyr_levels, ref_pyr=ref_pyr, cur_pyr=cur_pyr, T_ref_w=c(T_ref_w, np.float64),
                    T_cur_w=c(T_cur_w, np.float64), ref_index=ref_index, cur_index=cur_index, ref_px=c(ref_px, np.float64),
                    ref_f=c(ref_f, np.float64), ref_level=ref_level, is_edgelet=is_edgelet, ref_grad=c(ref_grad, np.float64),
                    a=a, b=b, mu=mu, z_range=z_range, sigma2=sigma2, depth_gt=c(depth, np.float64))


@dataclass
class LineSeedData(SeedData):
    """SeedData for the segment's mid-point feature and start-point Gaussian + the end-point fields (plsvo_line_seed_batch)."""

    ref_sf: np.ndarray = None
    ref_ef: np.ndarray = None
    mu_e: np.ndarray = None
    z_range_e: np.ndarray = None
    sigma2_e: np.ndarray = None
    depth_e_gt: np.ndarray = None


def make_line_seed_batch(cam: Camera = VGA, n: int = 1500, seed: int = 9500, half_len_px: float = 18.0, device: str | torch.device = "cpu",
                         **kw) -> LineSeedData:
    """Line seeds: a point-seed batch for the segment mid points (px, f) plus end-point bearings sf / ef a few pixels either
    side of the mid point and an independent inverse-depth Gaussian for the end point."""
    base = make_seed_batch(cam=cam, n=n, seed=seed, device=device, edgelet_frac=0.0, **kw)
    rng = np.random.Generator(np.random.PCG64(seed + 17))
    ang = rng.uniform(0, 2 * math.pi, n)
    off = np.stack([np.cos(ang), np.sin(ang)], -1) * rng.uniform(0.4, 1.0, (n, 1)) * half_len_px
    spx, epx = base.ref_px - off, base.ref_px + off

    def bearing(px):
        d = np.stack([(px[:, 0] - cam.cx) / cam.fx, (px[:, 1] - cam.cy) / cam.fy, np.ones(n)], -1)
        return np.ascontiguousarray(d / np.linalg.norm(d, axis=-1, keepdims=True))

    stage = rng.uniform(0.0, 3.0, n)
    z_range_e = base.z_range.copy()
    sigma2_e = (z_range_e.astype(np.float64) ** 2 / 36.0 * 10.0 ** (-stage)).astype(np.float32)
    mu_e = np.maximum(1.0 / base.depth_gt + rng.normal(0, 1, n) * np.sqrt(sigma2_e) * 0.5, 0.05).astype(np.float32)
    fields = {f: getattr(base, f) for f in base.__dataclass_fields__}
    return LineSeedData(**fields, ref_sf=bearing(spx), ref_ef=bearing(epx), mu_e=mu_e, z_range_e=z_range_e, sigma2_e=sigma2_e,
                        depth_e_gt=base.depth_gt.copy())
