"""Host-side model of the kernel's exact-order chi2 (align_kernel.cu, phase 1a + walker).

The reference sums chi2 in a float accumulator, sequentially over all pixels of all point patches
(src/sparse_img_align.cpp:484).  The kernel reproduces that float bit for bit in parallel: inside one binade
`s -> fl(s + t)` depends only on the parity of s's mantissa, so the 16 additions of a patch collapse to
"add A[parity] ulps", these maps compose associatively, and the few patches that may cross a power of two are
chained term by term.  This test runs the same decision rules (margin delta, binade classification, map
composition, walker) in NumPy and compares with the plain sequential float32 sum on adversarial inputs."""
import numpy as np
import pytest

F = np.float32


def seq_sum(terms):
    s = F(0)
    for t in terms.reshape(-1):
        s = F(s + t)
    return s


def chain16(s, t):
    for k in range(16):
        s = F(s + t[k])
    return s


def bits(x):
    return int(np.array([x], dtype=np.float32).view(np.uint32)[0])


def from_bits(b):
    return np.array([b & 0xFFFFFFFF], dtype=np.uint32).view(np.float32)[0]


def align_opq_cap(n_pts):
    """Opaque slots per pass of a batch with n_pts points: align_opq_cap, pl-svo_b200/csrc/internal.h."""
    return 48 + n_pts * n_pts // 131072


def kernel_model(terms, nt=128, opq_cap=None):
    """terms: [np, 16] float32 >= 0.  Returns (float32 sum, number of opaque patches)."""
    n_p = terms.shape[0]
    opq_cap = align_opq_cap(n_p) if opq_cap is None else opq_cap
    nw = nt // 32
    rounds = (n_p + nt - 1) // nt
    n_chunks = (n_p + 31) // 32
    items = [[] for _ in range(n_chunks)]
    n_opq = 0
    prefix_rounds = 0.0
    for r in range(rounds):
        chunk_tot = []
        Tf_all = {}
        for w in range(nw):
            c = r * nw + w
            tot = 0.0
            for lane in range(32):
                p = c * 32 + lane
                t = terms[p] if p < n_p else np.zeros(16, F)
                Tf = chain16(F(0), t)
                Tf_all[p] = (t, Tf, tot)  # tot = exclusive prefix inside the chunk
                tot += float(Tf)
            chunk_tot.append(tot)
        for w in range(nw):
            c = r * nw + w
            if c >= n_chunks:
                continue
            base = prefix_rounds + sum(chunk_tot[:w])
            lanes = []
            for lane in range(32):
                p = c * 32 + lane
                t, Tf, excl = Tf_all[p]
                P = base + excl
                delta = (16 * (p + 2)) * 6.0e-8 + 2.0e-6
                lo, hi = P * (1.0 - delta), (P + float(Tf)) * (1.0 + delta)
                ef = Ae = Ao = 0
                opaque = False
                if Tf == 0:
                    # no terms, or 16 terms that are all +0: the identity, never opaque.  It takes the estimate's binade,
                    # or a group of its own (255) next to a power of two.
                    if P != 0.0:
                        e_lo, e_hi = int(np.floor(np.log2(lo))), int(np.floor(np.log2(hi)))
                        ef = e_lo + 127 if e_lo == e_hi and -100 <= e_lo <= 100 else 255
                elif P == 0.0:
                    opaque = True
                else:
                    e_lo, e_hi = int(np.floor(np.log2(lo))), int(np.floor(np.log2(hi)))
                    if e_lo != e_hi or e_lo < -100 or e_lo > 100:
                        opaque = True
                    else:
                        ef = e_lo + 127
                        b0 = ef << 23
                        s0, s1 = chain16(from_bits(b0), t), chain16(from_bits(b0 | 1), t)
                        Ae, Ao = bits(s0) - b0, bits(s1) - (b0 | 1)
                lanes.append([Ae, Ao, ef, opaque, t])
            # segmented composition
            run = None
            for lane in range(32):
                Ae, Ao, ef, opaque, t = lanes[lane]
                head = lane == 0 or opaque or lanes[lane - 1][3] or ef != lanes[lane - 1][2]
                if head:
                    if run is not None:
                        items[c].append(run)
                    run = ["opq", t] if opaque else ["map", Ae, Ao, ef]
                    n_opq += int(opaque)
                else:
                    pAe, pAo = run[1], run[2]
                    run[1] = pAe + (Ao if (pAe & 1) else Ae)
                    run[2] = pAo + (Ae if (pAo & 1) else Ao)
            items[c].append(run)
        prefix_rounds += sum(chunk_tot)
    assert n_opq <= opq_cap
    s = F(0)
    for c in range(n_chunks):
        for it in items[c]:
            if it[0] == "opq":
                s = chain16(s, it[1])
            elif it[1] != 0 or it[2] != it[1]:  # the walker skips identity maps
                b = bits(s)
                assert (b >> 23) == it[3] or (it[3] == 0 and b == 0), "binade check"
                assert abs(it[2] - it[1]) < 32768
                b += it[2] if (b & 1) else it[1]
                assert (b >> 23) == it[3] or (it[3] == 0 and b == 0), "binade check"
                s = from_bits(b)
    return s, n_opq


def _residual_like(rng, n_p, scale=1.0):
    res = (rng.standard_normal((n_p, 16)) * 6 * scale).astype(F)
    w = (1.0 / (1.0 + np.abs(res).astype(np.float64))).astype(F)
    return (res * res * w).astype(F)


@pytest.mark.parametrize("n_p,nt", [(300, 128), (300, 96), (64, 64), (500, 128), (37, 256)])
def test_exact_order_on_residual_like_terms(n_p, nt):
    rng = np.random.default_rng(n_p * 1000 + nt)
    for trial in range(6):
        terms = _residual_like(rng, n_p)
        if trial == 1:
            terms[rng.random(n_p) < 0.3] = 0  # invisible / out-of-frame patches
        if trial == 2:
            terms[: n_p // 3] = 0  # leading zeros
        if trial == 3:
            terms = _residual_like(rng, n_p, scale=1e-3)  # near-perfect alignment: tiny residuals
        if trial == 4:
            terms[:, ::2] = 0  # exact zeros inside patches
        if trial == 5:
            terms = (terms * F(40)).astype(F)  # saturated residuals
        got, n_opq = kernel_model(terms, nt)
        want = seq_sum(terms)
        assert bits(got) == bits(want), (trial, float(got), float(want))
        assert n_opq < 40


def test_exact_order_with_ties_and_dyadic_terms():
    # dyadic terms create exact ties in the rounding (the parity-dependent case of the map)
    rng = np.random.default_rng(7)
    for trial in range(8):
        n_p = 200
        k = rng.integers(0, 12, (n_p, 16))
        terms = (rng.integers(1, 64, (n_p, 16)) * (2.0 ** -k.astype(np.float64))).astype(F)
        got, _ = kernel_model(terms, 128)
        assert bits(got) == bits(seq_sum(terms))


def test_exact_order_all_zero_and_single_patch():
    z = np.zeros((300, 16), F)
    got, n_opq = kernel_model(z, 128)
    assert bits(got) == 0 and n_opq == 0
    one = np.zeros((300, 16), F)
    one[123] = F(0.37)
    got, n_opq = kernel_model(one, 128)
    assert bits(got) == bits(seq_sum(one)) and n_opq == 1


def test_exact_order_growing_magnitudes():
    # every patch much larger than the sum so far: every patch crosses binades -> many opaque patches
    n_p = 30
    terms = np.zeros((n_p, 16), F)
    for p in range(n_p):
        terms[p] = F(3.0 ** p * 1e-6)
    got, n_opq = kernel_model(terms, 128)
    assert bits(got) == bits(seq_sum(terms))
    assert n_opq <= 48


# More points than this cannot fit in the 227 KB of shared memory of an sm_90a CTA, whatever the variant and the segments:
# every point takes at least 33 bytes of it (its 3-D point, 24; its chi2 item, 8; its visibility, 1; make_layout).
MAX_PTS_SMEM = 232448 // 33


@pytest.mark.parametrize("nt", [64, 96, 128, 160, 192, 256])
@pytest.mark.parametrize("n_p", [2048, 4096, MAX_PTS_SMEM])
def test_opaque_buffer_scales_with_the_point_count(n_p, nt):
    """The classification margin grows with the patch index, so the opaque patches grow with the square of the point
    count: at 4096 residual-like patches there are more than the 48 slots the buffer once had.  The sized buffer keeps
    a factor of two in hand, and the sum stays the sequential one bit for bit."""
    rng = np.random.default_rng(n_p + nt)
    worst = 0
    for trial in range(2):
        terms = _residual_like(rng, n_p)
        got, n_opq = kernel_model(terms, nt)
        assert bits(got) == bits(seq_sum(terms)), (trial, float(got))
        assert n_opq <= align_opq_cap(n_p) // 2, (trial, n_opq, align_opq_cap(n_p))
        worst = max(worst, n_opq)
    if n_p >= 4096:
        assert worst > 48  # what a fixed buffer of 48 slots could not hold


def test_zero_patches_next_to_a_power_of_two_are_not_opaque():
    """80 evaluated patches whose terms are all +0, right below a power of two: they are the identity and take no
    opaque slot, so the list has no more opaque patches than without them."""
    rng = np.random.default_rng(1)
    terms = _residual_like(rng, 600)
    k = 250
    before = terms[:k].astype(np.float64).sum()
    terms[k] = F((2.0 ** np.ceil(np.log2(before)) * (1 - 1e-5) - before) / 16)  # the sum ends just below 2^e
    without = np.delete(terms, np.s_[k + 1:k + 81], axis=0)
    terms[k + 1:k + 81] = 0
    for nt in (64, 128, 256):
        got, n_opq = kernel_model(terms, nt)
        assert bits(got) == bits(seq_sum(terms))
        got0, n_opq0 = kernel_model(without, nt)
        assert bits(got0) == bits(got)
        assert n_opq <= n_opq0, (nt, n_opq, n_opq0)
