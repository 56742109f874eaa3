"""The structure-optimisation kernel against the CPU oracle, on the pivots, exits and degenerate features where it can go wrong.

structopt_kernel (csrc/structopt_kernel.cu) gives each point, and each segment with both its end points, one thread of a
128-thread CTA: points first, then segments.  Every thread runs Point::optimize / LineSeg::optimize in exact double
arithmetic with Eigen's pivoted 3x3 LDLT, so its positions and iteration counts must be byte-identical to the oracle's.
The cases are built so that each decision of the loop and of the LDLT is taken on purpose:

  * pivots: every transposition pair (tr[0], tr[1]) of the LDLT, for points and both segment ends.  Views with exact 0/±1
    rotations (identity, (½,½,½,½), (−½,−½,−½,½) and the 180° turns (1,0,0,0), (0,1,0,0)) put the depth of each view on
    a chosen world axis, and their distances order the diagonal of A;
  * zeros: a point on the optical axis of one view (A = diag(1/z², 1/z², 0): the pseudo-inverse zeroes D[2]) and features
    without observations (A = 0: the k == 0 early return, dp = 0, an EPS exit after one iteration);
  * nans: an entry on a keyframe's principal plane, an observation with f.z = 0, a NaN entry, and segments with one NaN end
    (both ends roll back);
  * rollbacks: far entries that make Gauss-Newton overshoot (chi2 rises at it = 1 and later), segments whose s end
    converges while the e end does not, and segments whose e end rises while the s end falls;
  * params: n_iter 0, 1, 2, 5 (the Config default) and 100, and n_iter_pts != n_iter_segs;
  * shapes: 1, 127, 128 and 129 features, the point/segment boundary inside a CTA and on a CTA edge, 1000 observations,
    1 and 4096 frames, observation lists that start past 0, quaternions scaled by 3 and 1e-3, and 2^20 features;
  * layout invariance, GPU against GPU, and every rejection of the host's validation.

Positions are also checked against a solve that shares nothing with the three LDLT transcriptions (kernel, oracle and the
Eigen stand-in the reference compiles against): the first step of every well-conditioned feature is compared with the exact
solution of A dp = b, recomputed from the input doubles with mpmath.  test_cases_cover_the_decisions (no GPU) uses the
oracle's decision statistics to check that the cases keep reaching what they are meant to reach."""
import ctypes as C
import itertools

import numpy as np
import pytest

# rotations whose matrices are exactly 0/±1, as (x, y, z, w).  A view's depth lies along world z for Q_ID, Q_X180 and
# Q_Y180 (-z for the last two), along world y for Q_CYC and along world x for Q_ICYC.
Q_ID, Q_CYC, Q_ICYC, Q_X180, Q_Y180 = (0, 0, 0, 1), (0.5, 0.5, 0.5, 0.5), (-0.5, -0.5, -0.5, 0.5), (1, 0, 0, 0), (0, 1, 0, 0)
N_ITER = (0, 1, 2, 5, 100)
BIG = 1 << 20
EXACT_COND = 1e8  # the exact-solve check covers first steps whose A is better conditioned than this


def _R(q):
    x, y, z, w = np.asarray(q, np.float64) / np.linalg.norm(q)
    return np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w)],
                     [2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w)],
                     [2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)]])


class _Builder:
    """Features with explicit observation lists; frames are (quaternion, translation), deduplicated."""

    def __init__(self):
        self.frames, self.points, self.segs = [], [], []

    def frame(self, q, t):
        T = tuple(float(v) for v in tuple(q) + tuple(t))
        if T not in self.frames:
            self.frames.append(T)
        return self.frames.index(T)

    def cam(self, k, X):
        """X in frame k's camera coordinates (for observations: the bearing need not be unit, only f / f.z is used)."""
        T = np.array(self.frames[k])
        return _R(T[:4]) @ np.asarray(X, np.float64) + T[4:]

    def point(self, entry, obs):
        self.points.append((np.asarray(entry, np.float64), [(k, np.asarray(f, np.float64)) for k, f in obs]))

    def seg(self, s, e, obs):
        self.segs.append((np.asarray(s, np.float64), np.asarray(e, np.float64),
                          [(k, np.asarray(sf, np.float64), np.asarray(ef, np.float64)) for k, sf, ef in obs]))

    def data(self, synth, n_iter_pts=5, n_iter_segs=5):
        c = np.ascontiguousarray
        pb = np.cumsum([0] + [len(o) for _, o in self.points]).astype(np.int32)
        sb = np.cumsum([0] + [len(o) for _, _, o in self.segs]).astype(np.int32)
        pf = np.array([k for _, o in self.points for k, _ in o], np.int32)
        pobs = np.array([f for _, o in self.points for _, f in o], np.float64).reshape(-1, 3)
        sf = np.array([k for _, _, o in self.segs for k, _, _ in o], np.int32)
        sobs = np.array([f for _, _, o in self.segs for _, f, _ in o], np.float64).reshape(-1, 3)
        eobs = np.array([f for _, _, o in self.segs for _, _, f in o], np.float64).reshape(-1, 3)
        P = np.array([p for p, _ in self.points], np.float64).reshape(-1, 3)
        S = np.array([s for s, _, _ in self.segs], np.float64).reshape(-1, 3)
        E = np.array([e for _, e, _ in self.segs], np.float64).reshape(-1, 3)
        return synth.StructOptData(T_f_w=c(np.array(self.frames, np.float64).reshape(-1, 7)), pt_obs_begin=pb, pt_obs_frame=pf,
                                   pt_obs_f=c(pobs), pt_pos=c(P), pt_pos_gt=P.copy(), seg_obs_begin=sb, seg_obs_frame=sf,
                                   seg_obs_sf=c(sobs), seg_obs_ef=c(eobs), seg_spos=c(S), seg_epos=c(E), seg_spos_gt=S.copy(),
                                   seg_epos_gt=E.copy(), n_iter_pts=n_iter_pts, n_iter_segs=n_iter_segs)


# ---- cases -------------------------------------------------------------------------------------------------------------
def _view(b, axis, d, z_turn=Q_ID):
    """A view whose depth lies along world axis `axis`, d in front of the world origin."""
    q = {0: Q_ICYC, 1: Q_CYC, 2: z_turn}[axis]
    return b.frame(q, (0.0, 0.0, d))


def _pivots(synth):
    """For each order of the diagonal of A (6 permutations) and several offsets: a point and a segment near the world origin
    seen from one view per world axis.  A view whose depth is along axis a adds ~1/d² to the other two diagonal entries,
    so the axis seen from farthest away gets the largest diagonal entry; off-axis offsets fill the off-diagonal entries.
    Entries and truths are dyadic, so A and b carry little round-off."""
    b = _Builder()
    offsets = [(0.25, -0.125, 0.375), (-0.375, 0.25, 0.125), (0.125, 0.375, -0.25), (0.5, -0.25, -0.125)]
    deltas = [(0.125, -0.0625, 0.09375), (-0.09375, 0.125, -0.0625)]
    for n, order in enumerate(itertools.permutations(range(3))):
        dist = {order[0]: 4.0, order[1]: 2.0, order[2]: 1.0}  # largest diagonal first
        for m, o in enumerate(offsets):
            turn = (Q_ID, Q_X180, Q_Y180)[(n + m) % 3]
            views = [_view(b, a, dist[a] + 0.5 * m, turn) for a in range(3)]
            if m % 2:
                views.append(views[m % 3])  # one view twice
            truth = np.array(o)
            entry = truth + deltas[m % 2]
            b.point(entry, [(k, b.cam(k, truth)) for k in views])
            e_truth = truth + (0.125, 0.0625, -0.0625)
            b.seg(entry, e_truth + deltas[(m + 1) % 2], [(k, b.cam(k, truth), b.cam(k, e_truth)) for k in views])
    return b.data(synth)


def _zeros(synth):
    """0: on the optical axis of the identity view, one observation: A = diag(1/4, 1/4, 0) exactly.  1: the same with an
    observation straight up, so dp[0] = 0 while dp[1] != 0.  2: no observation.  Segments: no observation, and both ends on
    the optical axis of one view."""
    b = _Builder()
    k = b.frame(Q_ID, (0.0, 0.0, 2.0))
    k2 = b.frame(Q_X180, (0.0, 0.0, 4.0))
    b.point((0.0, 0.0, 0.0), [(k, (1 / 64, -1 / 32, 1.0))])
    b.point((0.0, 0.0, 0.0), [(k, (0.0, 1 / 32, 1.0))])
    b.point((0.25, 0.5, 0.125), [])
    b.point((0.0, 0.0, 1.0), [(k2, (1 / 16, 1 / 8, 1.0))])  # on the axis of a 180° view
    b.seg((0.25, 0.5, 0.125), (1.0, 2.0, 3.0), [])
    b.seg((0.0, 0.0, 0.0), (0.0, 0.0, 0.5), [(k, (1 / 64, 1 / 64, 1.0), (-1 / 32, 0.0, 1.0))])
    return b.data(synth)


def _nans(synth):
    """Points: an entry on the principal plane of a keyframe (p.z = 0), an observation with f.z = 0, a NaN entry.
    Segments: a NaN s entry with a healthy e end, the same the other way round, and an f.z = 0 observation of the e end."""
    b = _Builder()
    k0, k1, k2 = b.frame(Q_ID, (0.0, 0.0, 2.0)), b.frame(Q_CYC, (0.0, 0.0, 3.0)), b.frame(Q_ICYC, (0.0, 0.0, 2.5))
    good = lambda X: [(k, b.cam(k, X)) for k in (k0, k1, k2)]  # noqa: E731
    b.point((0.25, 0.125, -2.0), good((0.25, 0.125, 0.0)))
    b.point((0.25, 0.125, 0.0), good((0.25, 0.125, 0.0))[:2] + [(k2, (0.125, 0.0625, 0.0))])
    b.point((np.nan, 0.0, 0.0), good((0.0, 0.0, 0.0)))
    S, E = np.array([0.125, -0.25, 0.0]), np.array([0.375, 0.25, 0.125])
    obs = [(k, b.cam(k, S), b.cam(k, E)) for k in (k0, k1, k2)]
    b.seg((np.nan, -0.25, 0.0), E + 0.0625, obs)
    b.seg(S + 0.0625, (0.375, np.nan, 0.125), obs)
    b.seg(S + 0.0625, E + 0.0625, obs[:2] + [(k2, b.cam(k2, S), (0.125, 0.25, 0.0))])
    return b.data(synth)


def _concat(synth, parts, n_iter_pts=5, n_iter_segs=5):
    """Several batches as one: frames, points and segments in order, observation lists re-based."""
    nf = np.cumsum([0] + [p.T_f_w.shape[0] for p in parts])
    c = np.ascontiguousarray

    def csr(begin, frame):
        b, f, base = [np.zeros(1, np.int32)], [], 0
        for i, p in enumerate(parts):
            pb = getattr(p, begin)
            b.append((pb[1:] - pb[0] + base).astype(np.int32))
            f.append(getattr(p, frame)[pb[0]:pb[-1]] + nf[i])
            base += int(pb[-1] - pb[0])
        return np.concatenate(b).astype(np.int32), np.concatenate(f).astype(np.int32)

    def obs(begin, name):
        return c(np.concatenate([getattr(p, name)[getattr(p, begin)[0]:getattr(p, begin)[-1]] for p in parts]).reshape(-1, 3))

    cat = lambda name: c(np.concatenate([getattr(p, name) for p in parts]).reshape(-1, 3))  # noqa: E731
    pb, pf = csr("pt_obs_begin", "pt_obs_frame")
    sb, sf = csr("seg_obs_begin", "seg_obs_frame")
    return synth.StructOptData(T_f_w=c(np.concatenate([p.T_f_w for p in parts])), pt_obs_begin=pb, pt_obs_frame=pf,
                               pt_obs_f=obs("pt_obs_begin", "pt_obs_f"), pt_pos=cat("pt_pos"), pt_pos_gt=cat("pt_pos_gt"),
                               seg_obs_begin=sb, seg_obs_frame=sf, seg_obs_sf=obs("seg_obs_begin", "seg_obs_sf"),
                               seg_obs_ef=obs("seg_obs_begin", "seg_obs_ef"), seg_spos=cat("seg_spos"), seg_epos=cat("seg_epos"),
                               seg_spos_gt=cat("seg_spos_gt"), seg_epos_gt=cat("seg_epos_gt"), n_iter_pts=n_iter_pts,
                               n_iter_segs=n_iter_segs)


def _take(synth, d, pts, segs):
    """The points `pts` and segments `segs` of d, with all of d's frames."""
    c = np.ascontiguousarray

    def csr(begin, frame, names, idx):
        b, f, o = [0], [], {n: [] for n in names}
        for i in idx:
            lo, hi = getattr(d, begin)[i], getattr(d, begin)[i + 1]
            f.append(getattr(d, frame)[lo:hi])
            for n in names:
                o[n].append(getattr(d, n)[lo:hi])
            b.append(b[-1] + hi - lo)
        cat = lambda a, s: c(np.concatenate(a)) if a else np.zeros(s)  # noqa: E731
        return np.array(b, np.int32), cat(f, 0).astype(np.int32), {n: cat(v, (0, 3)).reshape(-1, 3) for n, v in o.items()}

    pb, pf, po = csr("pt_obs_begin", "pt_obs_frame", ["pt_obs_f"], pts)
    sb, sf, so = csr("seg_obs_begin", "seg_obs_frame", ["seg_obs_sf", "seg_obs_ef"], segs)
    rows = lambda a, idx: c(a[list(idx)].reshape(-1, 3))  # noqa: E731
    return synth.StructOptData(T_f_w=d.T_f_w.copy(), pt_obs_begin=pb, pt_obs_frame=pf, pt_obs_f=po["pt_obs_f"], pt_pos=rows(d.pt_pos, pts),
                               pt_pos_gt=rows(d.pt_pos_gt, pts), seg_obs_begin=sb, seg_obs_frame=sf, seg_obs_sf=so["seg_obs_sf"],
                               seg_obs_ef=so["seg_obs_ef"], seg_spos=rows(d.seg_spos, segs), seg_epos=rows(d.seg_epos, segs),
                               seg_spos_gt=rows(d.seg_spos_gt, segs), seg_epos_gt=rows(d.seg_epos_gt, segs),
                               n_iter_pts=d.n_iter_pts, n_iter_segs=d.n_iter_segs)


def _rollbacks(synth):
    """Far entries (0.5 m): Gauss-Newton overshoots, so chi2 rises at it = 1 (back to the entry) and later.  Segments with a
    noise-free, exact s end and a far e end (s converges at once, e does not), and with a near s end and a far e end (e rises
    while s falls)."""
    far = synth.make_structopt_batch(n_points=1500, n_segs=500, seed=8300, pert=0.5)
    conv = synth.make_structopt_batch(n_points=0, n_segs=200, seed=8301, noise=0.0)
    conv.seg_spos = conv.seg_spos_gt.copy()
    conv.seg_epos = np.ascontiguousarray(conv.seg_epos_gt + np.random.default_rng(8302).normal(0, 0.2, conv.seg_epos.shape))
    mixed = synth.make_structopt_batch(n_points=0, n_segs=600, seed=8303)
    mixed.seg_epos = np.ascontiguousarray(mixed.seg_epos_gt + np.random.default_rng(8304).normal(0, 0.5, mixed.seg_epos.shape))
    return _concat(synth, [far, conv, mixed])


def _shifted(synth, d, n_pt, n_seg):
    """d with n_pt / n_seg unused observations in front of each list: pt_obs_begin[0] > 0 and seg_obs_begin[0] > 0."""
    c = np.ascontiguousarray
    pad = lambda a, n, v: c(np.concatenate([np.full((n,) + a.shape[1:], v, a.dtype), a]))  # noqa: E731
    return synth.StructOptData(T_f_w=d.T_f_w, pt_obs_begin=(d.pt_obs_begin + n_pt).astype(np.int32),
                               pt_obs_frame=pad(d.pt_obs_frame, n_pt, 0), pt_obs_f=pad(d.pt_obs_f, n_pt, np.nan), pt_pos=d.pt_pos,
                               pt_pos_gt=d.pt_pos_gt, seg_obs_begin=(d.seg_obs_begin + n_seg).astype(np.int32),
                               seg_obs_frame=pad(d.seg_obs_frame, n_seg, 0), seg_obs_sf=pad(d.seg_obs_sf, n_seg, np.nan),
                               seg_obs_ef=pad(d.seg_obs_ef, n_seg, np.nan), seg_spos=d.seg_spos, seg_epos=d.seg_epos,
                               seg_spos_gt=d.seg_spos_gt, seg_epos_gt=d.seg_epos_gt, n_iter_pts=d.n_iter_pts, n_iter_segs=d.n_iter_segs)


def _long(synth):
    """A point and a segment with 1000 observations each (every frame many times over), next to short ones."""
    d = synth.make_structopt_batch(n_points=3, n_segs=3, n_frames=12, seed=8400)
    rng = np.random.default_rng(8401)
    b = _Builder()
    b.frames = [tuple(T) for T in d.T_f_w.tolist()]
    ks = rng.integers(0, 12, 1000)
    P, S, E = d.pt_pos_gt[0], d.seg_spos_gt[0], d.seg_epos_gt[0]
    noisy = lambda k, X: b.cam(k, X) + np.r_[rng.normal(0, 1e-3, 2) * b.cam(k, X)[2], 0.0]  # noqa: E731
    b.point(d.pt_pos[0], [(int(k), noisy(k, P)) for k in ks])
    b.seg(d.seg_spos[0], d.seg_epos[0], [(int(k), noisy(k, S), noisy(k, E)) for k in ks])
    return _concat(synth, [b.data(synth), d])


def _count(synth, n, kind, seed):
    n_pts, n_segs = {"points": (n, 0), "segments": (0, n), "mixed": (n - n // 2, n // 2)}[kind]
    return synth.make_structopt_batch(n_points=n_pts, n_segs=n_segs, seed=seed)


def _scaled_quaternions(synth):
    """Every third frame's quaternion times 3, every third (from the second) times 1e-3: Sophus normalises them."""
    d = synth.make_structopt_batch(n_points=400, n_segs=100, n_frames=12, seed=8500)
    d.T_f_w = d.T_f_w.copy()
    d.T_f_w[0::3, :4] *= 3.0
    d.T_f_w[1::3, :4] *= 1e-3
    return d


def _big(synth):
    """2^20 features: 128 copies of a 6144-point + 2048-segment batch, copy c's point entries moved by c mm along x (so that
    a feature read from the wrong copy shows)."""
    base = synth.make_structopt_batch(n_points=6144, n_segs=2048, n_frames=32, seed=8600)
    d = _concat(synth, [base] * 128)
    d.pt_pos[:, 0] += np.repeat(np.arange(128) * 1e-3, 6144)
    return d


def _case(name, synth):
    if name == "pivots":
        return _pivots(synth)
    if name == "zeros":
        return _zeros(synth)
    if name == "nans":
        return _nans(synth)
    if name == "rollbacks":
        return _rollbacks(synth)
    if name.startswith("iter-"):
        n_pts, n_segs = (int(v) for v in name[5:].split("-"))
        d = synth.make_structopt_batch(n_points=800, n_segs=250, seed=8700, pert=0.2)
        d.n_iter_pts, d.n_iter_segs = n_pts, n_segs
        return d
    if name.startswith("count-"):
        _, kind, n = name.split("-")
        return _count(synth, int(n), kind, 8800 + int(n))
    if name == "boundary-mid-cta":
        return synth.make_structopt_batch(n_points=192, n_segs=100, seed=8900)
    if name == "boundary-cta-edge":
        return synth.make_structopt_batch(n_points=256, n_segs=100, seed=8901)
    if name == "long":
        return _long(synth)
    if name == "frames-1":
        return synth.make_structopt_batch(n_points=200, n_segs=60, n_frames=1, seed=8902)
    if name == "frames-4096":
        return synth.make_structopt_batch(n_points=3000, n_segs=800, n_frames=4096, seed=8903)
    if name == "shifted":
        return _shifted(synth, _concat(synth, [_pivots(synth), _zeros(synth)]), 5, 7)
    if name == "quaternions":
        return _scaled_quaternions(synth)
    if name == "big":
        return _big(synth)
    raise KeyError(name)


COUNTS = [f"count-{k}-{n}" for k in ("points", "segments", "mixed") for n in (1, 127, 128, 129)]
ITERS = [f"iter-{n}-{n}" for n in N_ITER] + ["iter-3-7", "iter-7-3", "iter-0-5", "iter-5-0"]
SMALL = ["pivots", "zeros", "nans", "rollbacks", "boundary-mid-cta", "boundary-cta-edge", "long", "frames-1", "frames-4096",
         "shifted", "quaternions"]
CASES = SMALL + ITERS + COUNTS + ["big"]
# cases whose first steps the exact-solve check covers: zeros, nans and frames-1 (one view) have no nonsingular finite system,
# the others repeat these generators at other sizes
EXACT = ["pivots", "rollbacks", "long", "shifted", "quaternions"]


@pytest.fixture(scope="module")
def case(synth):
    made = {}

    def get(name):
        if name not in made:
            made[name] = _case(name, synth)
        return made[name]

    return get


def _with_iters(synth, d, n_pts, n_segs):
    return _concat(synth, [d], n_pts, n_segs)


# ---- comparing -----------------------------------------------------------------------------------------------------------
OUTS = ("pt_pos", "seg_spos", "seg_epos", "pt_iters", "seg_iters")


def _same(got, want, what=""):
    for f in OUTS:
        a, b = getattr(got, f), getattr(want, f)
        if a.tobytes() != b.tobytes():
            bad = np.nonzero((a != b) & ~(np.isnan(a) & np.isnan(b)) if a.dtype.kind == "f" else a != b)[0]
            raise AssertionError(f"{what}: {f} differs at {len(bad)} rows, first {bad[:8].tolist()}: {a[bad[:2]]} vs {b[bad[:2]]}")


def _exact_step(frames, obs, pos):
    """dp of A dp = b at pos for one point (or segment end), from the input doubles at 60 digits: the pose action, the
    Jacobian, A and b as the reference writes them, and dp by Cramer's rule (no LDLT).  Also |A^-1|inf * |beta|inf, where
    beta = sum |J|^T (|f / f.z| + |p / p.z|) bounds, in units of the double round-off, the error of forming b: a residual
    that is itself round-off (an entry already at a noise-free truth) has no correct digits to pass on to dp."""
    import mpmath as mp

    mp.mp.dps = 60
    A = mp.zeros(3, 3)
    b = mp.zeros(3, 1)
    beta = mp.zeros(3, 1)
    P = mp.matrix([mp.mpf(float(v)) for v in pos])
    for k, f in obs:
        T = frames[k]
        q = [mp.mpf(float(v)) for v in T[:4]]
        n = mp.sqrt(sum(v * v for v in q))
        x, y, z, w = (v / n for v in q)
        R = mp.matrix([[1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w)],
                       [2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w)],
                       [2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)]])
        p = R * P + mp.matrix([mp.mpf(float(v)) for v in T[4:]])
        zi = 1 / p[2]
        Pj = mp.matrix([[zi, 0, -p[0] * zi * zi], [0, zi, -p[1] * zi * zi]])
        J = -(Pj * R)
        fv = [mp.mpf(float(v)) for v in f]
        e = mp.matrix([fv[0] / fv[2] - p[0] / p[2], fv[1] / fv[2] - p[1] / p[2]])
        A += J.T * J
        b -= J.T * e
        for r in range(3):
            beta[r] += abs(J[0, r]) * (abs(fv[0] / fv[2]) + abs(p[0] / p[2])) + abs(J[1, r]) * (abs(fv[1] / fv[2]) + abs(p[1] / p[2]))
    det = mp.det(A)
    dp = []
    for i in range(3):
        Ai = A.copy()
        for r in range(3):
            Ai[r, i] = b[r]
        dp.append(mp.det(Ai) / det)
    inv = A ** -1
    return dp, max(sum(abs(inv[r, c]) for c in range(3)) for r in range(3)) * max(abs(v) for v in beta)


def _exact_targets(d, pst, sst):
    """(kind, index, end) of every point and segment end whose first-iteration A is finite and nonsingular with a condition
    number below EXACT_COND and whose b is finite (a segment needs both ends so, since a NaN end rolls both back)."""
    def ok(st):
        return np.isfinite(st["b"]).all(-1) & (st["cond"] < EXACT_COND) & (st["exit"] != 2)

    pts = np.nonzero(ok(pst))[0]
    segs = np.nonzero(ok(sst).all(1))[0] if len(sst["exit"]) else np.zeros(0, int)
    return pts, segs


def _check_exact_steps(d, out, pst, sst, limit=None):
    """|(out - entry) - dp_exact|inf <= 64 2^-53 (kappa |dp_exact|inf + |A^-1|inf |beta|inf) + 2 ulp(entry) for the first
    step (out: n_iter = 1): the LDLT's backward error, the round-off of b (see _exact_step) and the rounding of the sum."""
    import mpmath as mp

    pts, segs = _exact_targets(d, pst, sst)
    if limit is not None:
        pts, segs = pts[:: max(1, len(pts) // limit)], segs[:: max(1, len(segs) // limit)]
    frames = d.T_f_w.tolist()
    worst, checked = 0.0, 0

    def one(entry, got, obs, cond, what):
        nonlocal worst, checked
        dp, b_err = _exact_step(frames, obs, entry)
        dpn = max(abs(v) for v in dp)
        for c in range(3):
            err = abs((mp.mpf(float(got[c])) - mp.mpf(float(entry[c]))) - dp[c])
            tol = 64 * mp.mpf(2) ** -53 * (cond * dpn + b_err) + 2 * mp.mpf(float(np.spacing(abs(entry[c]))))
            assert err <= tol, f"{what}: component {c}: step error {mp.nstr(err, 5)} > {mp.nstr(tol, 5)} (cond {cond:.3g}, " \
                               f"step {[mp.nstr(v, 17) for v in dp]}, got {(got - entry).tolist()})"
            worst = max(worst, float(err / tol) if tol > 0 else 0.0)
        checked += 1

    for i in pts:
        lo, hi = d.pt_obs_begin[i], d.pt_obs_begin[i + 1]
        obs = [(int(d.pt_obs_frame[o]), d.pt_obs_f[o]) for o in range(lo, hi)]
        one(d.pt_pos[i], out.pt_pos[i], obs, pst["cond"][i], f"point {i}")
    for i in segs:
        lo, hi = d.seg_obs_begin[i], d.seg_obs_begin[i + 1]
        for e, (entry, got, fobs) in enumerate(((d.seg_spos[i], out.seg_spos[i], d.seg_obs_sf), (d.seg_epos[i], out.seg_epos[i], d.seg_obs_ef))):
            obs = [(int(d.seg_obs_frame[o]), fobs[o]) for o in range(lo, hi)]
            one(entry, got, obs, sst["cond"][i, e], f"segment {i} end {'se'[e]}")
    return checked, worst


# ---- GPU tests -----------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("name", SMALL + ITERS + COUNTS)
def test_case_is_bit_identical_to_the_oracle(pkg, abi, synth, oracle, case, name):
    d = case(name)
    _same(pkg.optimizeStructure(d), oracle.structopt(abi, d, 8), name)


@pytest.mark.gpu
def test_two_to_the_twenty_features(pkg, abi, synth, oracle, case):
    d = case("big")
    assert d.pt_pos.shape[0] + d.seg_spos.shape[0] >= BIG
    _same(pkg.optimizeStructure(d), oracle.structopt(abi, d, 0), "big")


@pytest.mark.gpu
@pytest.mark.parametrize("name", EXACT)
def test_first_step_solves_the_normal_equations_exactly(pkg, abi, synth, oracle, case, name):
    """The kernel's first step against the exact solution of its normal equations (no LDLT involved)."""
    d = _with_iters(synth, case(name), 1, 1)
    ref, pst, sst = oracle.structopt_stats(abi, d, 8)
    out = pkg.optimizeStructure(d)
    _same(out, ref, name)
    checked, worst = _check_exact_steps(d, out, pst, sst, limit=None if name != "rollbacks" else 150)
    print(f"{name}: {checked} first steps within {worst:.3f} of the bound")
    assert checked > 0


@pytest.mark.gpu
def test_layout_invariance(pkg, abi, synth, case):
    """A feature gives the same bytes alone, at another index inside a large batch, and when that batch runs twice on one
    context."""
    picks = {"pivots": ([0, 7, 13, 23], [1, 8, 14, 22]), "zeros": ([0, 1, 2], [0, 1]), "nans": ([0, 1, 2], [0, 1, 2]),
             "rollbacks": ([3, 700, 1499], [0, 499, 650, 1200])}
    parts = [_take(synth, case(n), p, s) for n, (p, s) in picks.items()]
    feats = _concat(synth, parts)
    big = case("frames-4096")
    # the test features go after 1000 points and 300 segments of a large batch, so they land on other CTAs and lanes
    host = _concat(synth, [_take(synth, big, range(1000), range(300)), feats, _take(synth, big, range(1000, 3000), range(300, 800))])
    run1 = pkg.optimizeStructure(host)
    run2 = pkg.optimizeStructure(host)
    for f in OUTS:
        assert getattr(run1, f).tobytes() == getattr(run2, f).tobytes(), f"{f}: the second run differs"
    n_p, n_s = feats.pt_pos.shape[0], feats.seg_spos.shape[0]
    for i in range(n_p):
        alone = pkg.optimizeStructure(_take(synth, feats, [i], []))
        assert run1.pt_pos[1000 + i].tobytes() == alone.pt_pos[0].tobytes() and run1.pt_iters[1000 + i] == alone.pt_iters[0], f"point {i}"
    for i in range(n_s):
        alone = pkg.optimizeStructure(_take(synth, feats, [], [i]))
        for f in ("seg_spos", "seg_epos"):
            assert getattr(run1, f)[300 + i].tobytes() == getattr(alone, f)[0].tobytes(), f"segment {i}: {f}"
        assert run1.seg_iters[300 + i] == alone.seg_iters[0], f"segment {i}: iters"


def _run(ctx, b, out):
    return ctx.lib.plsvo_structopt_batch_run(ctx.handle, C.byref(b), C.byref(out.struct))


def _rejections():
    """(what, mutate(batch, result) -> None, message) for every rejection of structopt_batch_run_body."""
    null_d, null_i = C.POINTER(C.c_double)(), C.POINTER(C.c_int32)()
    desc, pts, segs, obs = "structopt batch description", "structopt point arrays missing", "structopt segment arrays missing", \
        "structopt observation arrays missing"

    def setf(obj, field, value):
        return lambda b, o: setattr(b if obj == "b" else o, field, value)

    cases = [("negative n_points", setf("b", "n_points", -1), desc), ("negative n_segs", setf("b", "n_segs", -1), desc),
             ("n_frames 0", setf("b", "n_frames", 0), desc), ("negative n_iter_pts", setf("b", "n_iter_pts", -1), desc),
             ("negative n_iter_segs", setf("b", "n_iter_segs", -1), desc), ("no T_f_w", setf("b", "T_f_w", null_d), desc),
             ("no pt_obs_begin", setf("b", "pt_obs_begin", null_i), pts), ("no pt_pos", setf("b", "pt_pos", null_d), pts),
             ("no out pt_pos", setf("o", "pt_pos", null_d), pts),
             ("no seg_obs_begin", setf("b", "seg_obs_begin", null_i), segs), ("no seg_spos", setf("b", "seg_spos", null_d), segs),
             ("no seg_epos", setf("b", "seg_epos", null_d), segs), ("no out seg_spos", setf("o", "seg_spos", null_d), segs),
             ("no out seg_epos", setf("o", "seg_epos", null_d), segs),
             ("no pt_obs_frame", setf("b", "pt_obs_frame", null_i), obs), ("no pt_obs_f", setf("b", "pt_obs_f", null_d), obs),
             ("no seg_obs_frame", setf("b", "seg_obs_frame", null_i), obs), ("no seg_obs_sf", setf("b", "seg_obs_sf", null_d), obs),
             ("no seg_obs_ef", setf("b", "seg_obs_ef", null_d), obs)]
    return cases


@pytest.mark.gpu
def test_validation_rejects_before_queueing(pkg, abi, synth, oracle):
    """Every rejection returns PLSVO_ERR_INVALID with its message and launches nothing; the context then runs a valid call.
    A call with no feature returns OK."""
    ctx = pkg.api.default_context()
    d = synth.make_structopt_batch(n_points=40, n_segs=12, n_frames=6, seed=9000)
    ref = oracle.structopt(abi, d)

    def expect(b, out, msg, what):
        n0 = ctx.launch_count()
        assert _run(ctx, b, out) == abi.ERR_INVALID, what
        m = ctx.lib.plsvo_last_error(ctx.handle)
        assert m and msg in m.decode(), f"{what}: {m!r}"
        assert ctx.launch_count() == n0, f"{what}: a kernel was launched"
        _same(pkg.optimizeStructure(d), ref, f"the call after {what}")

    for what, mutate, msg in _rejections():
        b, keep = abi.make_structopt_batch(d)
        out = abi.StructOptOut(b.n_points, b.n_segs)
        mutate(b, out.struct)
        expect(b, out, msg, what)
    for begin, msg in (("pt_obs_begin", "pt_obs_begin not monotone"), ("seg_obs_begin", "seg_obs_begin not monotone")):
        for i, v in ((3, None), (0, -1)):  # an offset above the next one, and a negative first offset
            bad = _concat(synth, [d])
            arr = getattr(bad, begin)
            arr[i] = arr[i + 1] + 1 if v is None else v
            b, keep = abi.make_structopt_batch(bad)
            expect(b, abi.StructOptOut(b.n_points, b.n_segs), msg, f"{begin}[{i}]")
    for frame in ("pt_obs_frame", "seg_obs_frame"):
        for v in (-1, d.T_f_w.shape[0]):
            bad = _concat(synth, [d])
            getattr(bad, frame)[5] = v
            b, keep = abi.make_structopt_batch(bad)
            expect(b, abi.StructOptOut(b.n_points, b.n_segs), "observation refers to a missing frame", f"{frame} = {v}")
    empty = _take(synth, d, [], [])
    b, keep = abi.make_structopt_batch(empty)
    n0 = ctx.launch_count()
    assert _run(ctx, b, abi.StructOptOut(0, 0)) == abi.OK
    assert ctx.launch_count() == n0


# ---- CPU tier ------------------------------------------------------------------------------------------------------------
def _runs(synth):
    """(name, data) of every case the GPU tests run, big excepted, at its own n_iter and at n_iter = 1."""
    for name in SMALL + ITERS + COUNTS:
        d = _case(name, synth)
        yield name, d
        if name in EXACT:
            yield name + "@1", _with_iters(synth, d, 1, 1)


def test_structopt_stats_leaves_the_outputs_alone(abi, synth, oracle):
    """oracle.structopt_stats runs the same optimisation: positions and iteration counts byte-identical to oracle.structopt."""
    for name in ("pivots", "zeros", "nans", "rollbacks", "iter-0-0", "iter-100-100", "iter-3-7", "shifted", "long"):
        d = _case(name, synth)
        a = oracle.structopt(abi, d, 4)
        b, pst, sst = oracle.structopt_stats(abi, d, 4)
        _same(b, a, name)
        assert (pst["exit_it"] + 1 == np.where(pst["exit"] == oracle.SO_EXIT_NONE, 0, a.pt_iters)).all()
        assert (sst["exit_it"][:, 0] + 1 == np.where(sst["exit"][:, 0] == oracle.SO_EXIT_NONE, 0, a.seg_iters)).all()


def test_cases_cover_the_decisions(abi, synth, oracle):
    """The cases reach all six pivot sequences for points and both segment ends, every exit (for segments, caused by either
    end), chi2 rises at it = 1 and later, the early return of an all-zero A and a D entry the pseudo-inverse zeroes."""
    pivots = np.zeros((3, 6), int)
    exits = {k: np.zeros(5, int) for k in ("pt", "seg")}
    rise1 = rise_late = zero = zeroed = s_only_eps = e_only_rise = 0
    for name, d in _runs(synth):
        _, pst, sst = oracle.structopt_stats(abi, d, 8)
        for r, st in enumerate((pst, {k: v[:, 0] for k, v in sst.items()}, {k: v[:, 1] for k, v in sst.items()})):
            for k in range(6):
                pivots[r, k] += int(((st["pivots"] >> k) & 1).sum())
            zero += int(st["zero"].sum())
            zeroed += int(st["d_zeroed"].sum())
        exits["pt"] += np.bincount(pst["exit"], minlength=5)
        exits["seg"] += np.bincount(sst["exit"][:, 0], minlength=5) if len(sst["exit"]) else 0
        for st, ex in ((pst, pst["exit"]), (sst, sst["exit"][:, 0] if len(sst["exit"]) else np.zeros(0, int))):
            it = st["exit_it"] if st is pst else st["exit_it"][:, 0]
            rise1 += int(((ex == oracle.SO_EXIT_CHI2) & (it == 1)).sum())
            rise_late += int(((ex == oracle.SO_EXIT_CHI2) & (it >= 2)).sum())
        if len(sst["exit"]):
            c = sst["cause"]
            s_only_eps += int(((sst["exit"][:, 0] == oracle.SO_EXIT_EPS) & (c[:, 0] == 4) & (c[:, 1] == 0)).sum())
            e_only_rise += int(((sst["exit"][:, 0] == oracle.SO_EXIT_CHI2) & (c[:, 0] == 0) & (c[:, 1] == 1) & (sst["exit_it"][:, 0] >= 1)).sum())
    print("pivot pairs (points, s ends, e ends):", pivots.tolist(), "exits:", {k: v.tolist() for k, v in exits.items()})
    assert (pivots >= 8).all(), f"pivot pairs {oracle.SO_PIVOTS}: {pivots.tolist()}"
    for k in ("pt", "seg"):
        assert (exits[k] >= 3).all(), f"{k} exits (none, chi2, NaN, EPS, cap): {exits[k].tolist()}"
    assert rise1 >= 10 and rise_late >= 10, (rise1, rise_late)
    assert zero >= 3 and zeroed >= 3, (zero, zeroed)
    assert s_only_eps >= 10 and e_only_rise >= 10, (s_only_eps, e_only_rise)


@pytest.mark.parametrize("name", EXACT)
def test_oracle_first_step_solves_the_normal_equations_exactly(abi, synth, oracle, name):
    """The oracle's first step against the exact solution: catches a transcription error that the oracle, the Eigen stand-in
    and the kernel share.  Every pivot sequence is among the checked steps."""
    d = _with_iters(synth, _case(name, synth), 1, 1)
    out, pst, sst = oracle.structopt_stats(abi, d, 8)
    checked, worst = _check_exact_steps(d, out, pst, sst, limit=None if name != "rollbacks" else 150)
    print(f"{name}: {checked} first steps within {worst:.3f} of the bound")
    assert checked > 0
    if name == "pivots":
        pts, segs = _exact_targets(d, pst, sst)
        for mask in (pst["pivots"][pts], sst["pivots"][segs, 0], sst["pivots"][segs, 1]):
            assert np.bitwise_or.reduce(mask) == 0b111111, f"pivot pairs among the checked steps: {np.bitwise_or.reduce(mask):06b}"


@pytest.mark.parametrize("name", CASES)
def test_oracle_is_bit_identical_to_the_reference_tu(abi, synth, oracle, name):
    """Every case, and every case of the exact-solve check at n_iter = 1, through the reference's own feature3D_impl.cpp."""
    if not oracle.have_ref():
        pytest.skip("oracle/_ref is not built and no recorded outputs of it are present")
    d = _case(name, synth)
    runs = [d] + ([_with_iters(synth, d, 1, 1)] if name in EXACT else [])
    for run in runs:
        o = oracle.structopt(abi, run, 0)
        r = oracle.ref_structopt(abi, run)
        for f in ("pt_pos", "seg_spos", "seg_epos"):
            oracle.assert_ref_equal(getattr(o, f), r, f, err_msg=name)
