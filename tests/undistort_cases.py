"""The cameras, sizes and frames of tests/test_gpu_undistort_cases.py, shared with the fixture generator
tests/golden/make_undistort_cases_golden.py.  A camera is (width, height, fx, fy, cx, cy, d0, d1, d2, d3, d4), the
arguments of vk::PinholeCamera."""
import numpy as np

# both sides of the remap tile (64 x 16, four pixels per thread) and of the fused kernel's 64 x 64 tile
WIDTHS = (1, 2, 3, 4, 5, 7, 8, 9, 15, 16, 17, 63, 64, 65, 127, 128, 129, 641, 752, 1280)
HEIGHTS = (1, 2, 3, 15, 16, 17, 63, 64, 65, 479)
# the out-of-range cameras: the VGA frame of their definition, one row and column more, small frames with and without a
# tail of columns past OpenCV 4's eight-column vector blocks, and frames narrower than one block
OOR_SIZES = ((640, 480), (641, 479), (61, 45), (7, 5), (3, 2))
SMALL_OOR_SIZES = OOR_SIZES[2:]
# the sizes of the in-range cameras in the committed OpenCV digests
DIGEST_SIZES = ((641, 479), (129, 63), (17, 15), (3, 2))


def in_range(W, H):
    """Cameras whose every map entry lies well inside the int16 range at any size: the VGA calibrations below with fx,
    cx scaled by W / 640 and fy, cy by H / 480, so that the normalised coordinates span what they span at 640 x 480."""
    sx, sy = W / 640.0, H / 480.0
    c = (W / 2 - 0.3, H / 2 + 0.7)
    return {
        "barrel": (W, H, 420.0 * sx, 421.5 * sy, *c, -0.42, 0.21, 0.0, 0.0, -0.06),
        "pincushion": (W, H, 300.0 * sx, 300.0 * sy, W / 2, H / 2, 0.9, 0.6, 0.0, 0.0, 0.3),
        "tangential_only": (W, H, 500.0 * sx, 500.0 * sy, (W - 1) / 2, (H - 1) / 2, 1e-6, 0.0, 0.004, -0.003, 0.0),
        "non_square": (W, H, 520.0 * sx, 380.0 * sy, *c, -0.2, 0.05, 0.001, -0.0005, 0.0),
        "centre_off": (W, H, 400.0 * sx, 400.0 * sy, 0.2 * W, 0.8 * H, -0.25, 0.07, 0.0, 0.0, 0.0),
        "centre_outside": (W, H, 400.0 * sx, 400.0 * sy, -0.35 * W, 1.4 * H, -0.1, 0.02, 0.0, 0.0, 0.0),
        "neg_fx": (W, H, -420.0 * sx, 421.5 * sy, *c, -0.3, 0.1, 0.0, 0.0, 0.0),
        "neg_fy": (W, H, 420.0 * sx, -421.5 * sy, *c, -0.3, 0.1, 0.002, 0.0, 0.0),
        "neg_fx_fy": (W, H, -420.0 * sx, -421.5 * sy, *c, 0.3, 0.1, 0.0, 0.001, 0.0),
        # PinholeCamera's distortion_ flag is fabs(d0) > 1e-7: exactly 1e-7 is a copy whatever d1..d4 are, one step more a map
        "d0_1e-7_copy": (W, H, 420.0 * sx, 421.5 * sy, *c, 1e-7, 0.2, 0.001, 0.001, 0.05),
        "d0_-1e-7_copy": (W, H, 420.0 * sx, 421.5 * sy, *c, -1e-7, 0.2, 0.001, 0.001, 0.05),
        "d0_1.0000001e-7_map": (W, H, 420.0 * sx, 421.5 * sy, *c, 1.0000001e-7, 0.2, 0.001, 0.001, 0.05),
        "d0_-1.0000001e-7_map": (W, H, 420.0 * sx, 421.5 * sy, *c, -1.0000001e-7, 0.2, 0.001, 0.001, 0.05),
    }


# dyadic parameters at integer c: the map arithmetic is exact, and u * 32 or v * 32 lands exactly on a rounding tie
TIES = {
    "tie_k1": (640, 480, 256.0, 256.0, 320.0, 240.0, 2.0 ** -12, 0.0, 0.0, 0.0, 0.0),
    "tie_k1_k2": (640, 480, 256.0, 256.0, 320.0, 240.0, -2.0 ** -10, 2.0 ** -14, 0.0, 0.0, 0.0),
    "tie_neg_fx_p1": (640, 480, -256.0, 256.0, 320.0, 240.0, 2.0 ** -12, 0.0, 2.0 ** -12, 0.0, 0.0),
}


def out_of_range(W, H):
    """Cameras with map entries outside the int16 range (and outside int, and infinite), all accepted by the parameter
    checks; at 640 x 480 they are the cameras of DESIGN.md's table, at other sizes scaled as in_range."""
    sx, sy = W / 640.0, H / 480.0
    return {
        "oor_wrap": (W, H, 300.0 * sx, 300.0 * sy, W / 2, H / 2, 50.0, 80.0, 0.0, 0.0, 100.0),
        "oor_huge": (W, H, 300.0 * sx, 300.0 * sy, W / 2, H / 2, 1e6, 1e6, 0.0, 0.0, 1e8),
        "oor_f60": (W, H, 60.0 * sx, 60.0 * sy, W / 2, H / 2, 0.5, 0.5, 0.0, 0.0, 0.5),
        # fx is subnormal as a float, but not zero
        "oor_subnormal_fx": (W, H, 2.0 ** -140 * sx, 256.0 * sy, W / 2, 100.0 * sy, 0.5, 0.0, 0.0, 0.0, 1.0),
    }


# u or v infinite (k3 * r2^3 overflows double); a NaN would take the same cvRound branch
INF = (64, 48, 2.0 ** -140, 2.0 ** -140, 32.0, 24.0, 0.5, 0.0, 0.0, 0.0, 3e38)


def special():
    """name@WxH -> camera: the tie cameras, the out-of-range cameras at every size of OOR_SIZES and the infinite one."""
    out = {f"{n}@640x480": p for n, p in TIES.items()}
    for W, H in OOR_SIZES:
        out.update({f"{n}@{W}x{H}": p for n, p in out_of_range(W, H).items()})
    out["inf@64x48"] = INF
    return out


def frames(B, H, W, seed):
    """B random frames, then one of all 255 (the largest weighted sum) and a 0/255 checkerboard: [B + 2, H, W] u8."""
    rng = np.random.default_rng(seed)
    out = np.empty((B + 2, H, W), np.uint8)
    out[:B] = rng.integers(0, 256, (B, H, W), dtype=np.uint8)
    out[B] = 255
    y, x = np.mgrid[:H, :W]
    out[B + 1] = ((x + y) % 2 * 255).astype(np.uint8)
    return out
