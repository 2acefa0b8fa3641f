"""Seeded frame families for the ContourDetector and LSD front ends, built to reach what the kernels can get wrong:
ties and plateaus, frames without a defined gradient, lists that fall into one bucket across many chunks, more than
1024 buckets, mirrors that wrap several times, and the epsilon guard of the edge test.  Shared by the reference pins
(test_frontend_cases_cpu.py, tests/golden/make_golden_frontend.py) and the GPU parity tests (test_frontend_cases_gpu.py).

Every case is (family, case id, frame [Y, X], parameters).  Frames that are whole numbers in 0..255 are uint8 and also
go through the u8 entries; the others are float64."""
import math

import numpy as np

from image_b200 import synth

LSD_DEFAULTS = dict(scale=0.8, sigma_scale=0.6, quant=2.0, ang_th=22.5, n_bins=1024)
CHUNK = 2048                       # elements of the LSD list per chunk of the bucket kernels (csrc/lsd.cu LSD_CHUNK)
GREATER_EPS = 1000 * np.finfo(np.float64).eps


def lsd_params(**kw):
    p = dict(LSD_DEFAULTS)
    p.update(kw)
    return p


def lsd_size(n, scale):
    """The scaled size of an axis of n pixels, as the sampler computes it (lsd.c:623-624)."""
    return int(math.ceil(n * scale))


def lsd_halfwidth(scale, sigma_scale):
    """Half width of the sampler's kernel (lsd.c:629-640)."""
    sigma = sigma_scale / scale if scale < 1.0 else sigma_scale
    return int(math.ceil(sigma * math.sqrt(2.0 * 3.0 * math.log(10.0))))


def contour_offset(sigma):
    """Half width of the contour blur (smooth_contours.c:206-210)."""
    return int(math.ceil(sigma * math.sqrt(2.0 * 3.0 * math.log(10.0))))


def _axis_for(n_out, scale):
    """The smallest input size whose scaled size is n_out."""
    n = max(1, int(n_out / scale) - 2)
    while lsd_size(n, scale) < n_out:
        n += 1
    assert lsd_size(n, scale) == n_out
    return n


def _list_shape(total, scale):
    """(Y, X) of a frame whose LSD list has exactly `total` elements: (N - 1)(M - 1) == total with N - 1 the divisor
    of `total` nearest to its square root."""
    a = min((d for d in range(1, int(math.isqrt(total)) + 1) if total % d == 0), key=lambda d: abs(d - math.isqrt(total)))
    return _axis_for(total // a + 1, scale), _axis_for(a + 1, scale)


def _ramp(Y, X, sx, sy=0.0):
    y, x = np.indices((Y, X), dtype=np.float64)
    return sx * x + sy * y


def lsd_cases():
    # no defined gradient: every modulus at or below rho, so the frame's max_grad stays 0
    yield "notdef", "shapes01_120x160", synth.frame_shapes(3, 120, 160) / 255.0, lsd_params()
    yield "notdef", "const0_120x160", np.zeros((120, 160), np.uint8), lsd_params()
    yield "notdef", "const7_120x160", np.full((120, 160), 7, np.uint8), lsd_params()
    f = np.zeros((120, 160), np.uint8)
    f[:, 80:] = np.random.default_rng(21).integers(0, 4, (120, 80))
    yield "notdef", "flat_and_low_noise_120x160", f, lsd_params()
    yield "natural", "shapes_120x160", synth.frame_shapes(3, 120, 160), lsd_params()
    yield "natural", "shapes_noise_333x517", synth.frame_shapes(8, 333, 517) + np.random.default_rng(8).random((333, 517)), lsd_params()
    # one or a few buckets over many chunks
    # (the ramps are steep enough for a defined angle everywhere: a step above rho = 5.23 per sample)
    x = np.indices((1960, 85))[1]
    yield "buckets", "ramp_x_1960x85", (3 * x).astype(np.uint8), lsd_params(scale=0.5)
    yield "buckets", "ramp_diag_500x640", _ramp(500, 640, 3.7, 1.1), lsd_params(scale=0.5)
    r = _ramp(420, 600, 4.0)
    r[:, 300:] = 1200.0 + 10.0 * (r[:, 300:] / 4.0 - 300.0)
    yield "buckets", "two_slopes_420x600", r, lsd_params(scale=0.5)
    yield "buckets", "nbins1_shapes_333x517", synth.frame_shapes(9, 333, 517), lsd_params(n_bins=1)
    for k, d in ((8, -1), (8, 0), (8, 1), (1, -1), (1, 0), (1, 1)):
        total = CHUNK * k + d
        Y, X = _list_shape(total, 0.5)
        yield "buckets", "ramp_list_%d" % total, _ramp(Y, X, 4.0, 2.0), lsd_params(scale=0.5)
    # more than 1024 buckets: the bucket starts carry across passes of 1024
    nat = synth.frame_shapes(10, 333, 517) + np.random.default_rng(10).random((333, 517))
    for nb in (1025, 2048, 3000, 4096):
        yield "bins", "shapes_noise_333x517_bins%d" % nb, nat, lsd_params(n_bins=nb)
        yield "bins", "ramp_diag_300x400_bins%d" % nb, _ramp(300, 400, 3.7, 1.1), lsd_params(scale=0.5, n_bins=nb)
    # sampler edges
    yield "sampler", "scale0.3_200x260", synth.frame_shapes(11, 200, 260), lsd_params(scale=0.3)
    yield "sampler", "scale1.5_60x80", synth.frame_shapes(12, 60, 80), lsd_params(scale=1.5)
    yield "sampler", "scale1.7_61x83", synth.frame_shapes(13, 61, 83), lsd_params(scale=1.7)
    yield "sampler", "taps63_90x120", synth.frame_shapes(14, 90, 120), lsd_params(sigma_scale=6.6)
    yield "sampler", "M2_2x40", synth.frame_shapes(15, 2, 40), lsd_params()
    yield "sampler", "N2_40x3", synth.frame_shapes(16, 40, 3), lsd_params(scale=0.5)
    yield "sampler", "Y3_wrap_3x40", synth.frame_shapes(17, 3, 40), lsd_params(sigma_scale=2.0)
    yield "sampler", "X2_wrap_40x2", synth.frame_shapes(18, 40, 2), lsd_params(sigma_scale=2.0)
    yield "sampler", "Y1_wrap_1x33", synth.frame_shapes(19, 1, 33), lsd_params(scale=1.5)
    yield "sampler", "X1_wrap_30x1", synth.frame_shapes(20, 30, 1), lsd_params(scale=1.5, sigma_scale=1.6)
    yield "sampler", "2x2_wrap", synth.frame_shapes(22, 2, 2), lsd_params(scale=1.5, sigma_scale=1.6)
    # thresholds
    f = synth.frame_shapes(23, 150, 210)
    f[:, :70] = 0
    yield "thresholds", "quant0_150x210", f, lsd_params(quant=0.0)
    yield "thresholds", "quant_huge_150x210", synth.frame_shapes(24, 150, 210), lsd_params(quant=1e6)
    yield "thresholds", "quant5_ang60_150x210", synth.frame_shapes(25, 150, 210), lsd_params(quant=5.0, ang_th=60.0)


def contour_cases():
    """(family, id, frame, sigma); sigma None = the reference's default."""
    yield "ties", "integer_shapes_97x131", synth.frame_shapes(30, 97, 131), None
    yield "ties", "quantised_120x160", synth.frame_shapes(31, 120, 160) // 16 * 16, None
    chk = (np.indices((64, 80)).sum(0) % 2 * 255).astype(np.uint8)
    yield "ties", "checker1_64x80_s0.3", chk, 0.3
    yield "ties", "checker1_64x80", chk, None
    yield "ties", "checker2_64x80", (((np.indices((64, 80)) // 2).sum(0) % 2) * 255).astype(np.uint8), None
    x = np.indices((70, 90))[1]
    yield "ties", "stripes1_70x90_s0.3", (x % 2 * 200).astype(np.uint8), 0.3
    yield "ties", "stripes3_70x90", (x // 3 % 2 * 200).astype(np.uint8), None
    yield "ties", "stripes3_t_90x70", (x // 3 % 2 * 200).astype(np.uint8).T.copy(), 0.5
    # isolated dots of a power of two: the blur is bitwise symmetric about each dot, so on its diagonals a pixel that is
    # both a horizontal and a vertical maximum sees min(L, R) == min(U, D) exactly
    d = np.zeros((120, 160), np.uint8)
    d[6::12, 6::12] = 128
    yield "ties", "dots128_every12_120x160_s1.5", d, 1.5
    for p, q in ((4, 2), (3, 4)):
        d = np.zeros((120, 160), np.uint8)
        d[::p, ::q] = 255
        yield "density", "dots%dx%d_120x160" % (p, q), d, None
    # around the greater_eps guard (1000 DBL_EPSILON) and far from 0
    base = synth.frame_shapes(32, 100, 140).astype(np.float64)
    yield "eps", "scaled1e-12_100x140", base * 1e-12, None
    yield "eps", "scaled3e-13_noise_100x140", (base + np.random.default_rng(33).random((100, 140))) * 3e-13, None
    yield "eps", "offset1e6_100x140", 1e6 + base / 64.0, None
    yield "eps", "negative_100x140", base - 300.0, None
    # kernel width: 65 taps (off = 32) and frames narrower than the half width
    yield "width", "taps65_64x200", synth.frame_shapes(34, 64, 200), 8.6
    yield "width", "taps65_3x40", synth.frame_shapes(35, 3, 40), 8.6
    for k, (Y, X) in enumerate(((5, 40), (40, 5), (1, 30), (30, 1), (3, 3), (2, 64), (64, 4), (6, 6))):
        yield "width", "narrow_%dx%d_s8" % (Y, X), synth.frame_shapes(36 + k, Y, X), 8.0


def is_u8(img):
    return img.dtype == np.uint8


# ------------------------------------------------------------------------------------------ oracle runs and pins

def lsd_oracle(po, img, p, impl="oracle"):
    """(scaled, angles, modgrad, list) of the oracle (or of the reference build, impl='ref')."""
    s = po.lsd_sampler(img, scale=p["scale"], sigma_scale=p["sigma_scale"], impl=impl)
    a, m, lst = po.lsd_ll_angle(s, threshold=po.lsd_rho(p["quant"], p["ang_th"]), n_bins=p["n_bins"], impl=impl)
    return s, a, m, lst


def lsd_digests(po, out):
    s, a, m, lst = out
    return dict(scaled=po.digest(s), angle_mod=po.digest(a, m), list=po.digest(lst))


EDGE_KEYS = ("idx", "Ex", "Ey", "Gx", "Gy")


def contour_oracle(po, img, sigma, impl="oracle"):
    g = po.contour_gaussian(img, sigma=sigma, impl=impl)
    return g, po.contour_edge_points(g, impl=impl)


def contour_digests(po, out):
    g, e = out
    return dict(gauss=po.digest(g), edges=po.digest(*[e[k] for k in EDGE_KEYS]))


def all_digests(po, impl):
    d = {}
    for fam, cid, img, p in lsd_cases():
        d["lsd/%s/%s" % (fam, cid)] = lsd_digests(po, lsd_oracle(po, img, p, impl))
    for fam, cid, img, sigma in contour_cases():
        d["contour/%s/%s" % (fam, cid)] = contour_digests(po, contour_oracle(po, img, sigma, impl))
    return d


# ------------------------------------------------------------------------------------------ what makes a case hard

def bucket_of(modgrad, max_grad, n_bins):
    """The bucket of every gradient pixel as the x86-64 reference computes it (the quotient truncated through int64)."""
    m = modgrad[:-1, :-1]
    with np.errstate(divide="ignore", invalid="ignore"):
        q = m * float(n_bins) / max_grad
    b = np.where(np.isfinite(q), q, 0.0).astype(np.int64)
    return np.minimum(b, n_bins - 1)


def contour_moduli(g):
    """|G| of the blurred plane as compute_gradient forms it (interior; 0 on the border)."""
    mod = np.zeros_like(g)
    gx = g[1:-1, 2:] - g[1:-1, :-2]
    gy = g[2:, 1:-1] - g[:-2, 1:-1]
    mod[1:-1, 1:-1] = np.sqrt(gx * gx + gy * gy)
    return mod


def diagonal_ties(g):
    """Pixels that are horizontal and vertical maxima with min(L, R) == min(U, D) and L != R, where the tie-break of
    compute_edge_points (smooth_contours.c:467-470) picks the direction of the sub-pixel offset."""
    mod = contour_moduli(g)
    c, L, R = mod[2:-2, 2:-2], mod[2:-2, 1:-3], mod[2:-2, 3:-1]
    D, U = mod[1:-3, 2:-2], mod[3:-1, 2:-2]

    def greater(a, b):
        return (a > b) & ~(a - b < GREATER_EPS)
    both = greater(c, L) & ~greater(R, c) & greater(c, D) & ~greater(U, c)
    return int((both & (np.minimum(L, R) == np.minimum(U, D)) & (L != R)).sum())


def guard_straddles(g):
    """(comparisons the epsilon guard turns to 'not greater', comparisons above the guard) among the horizontal and
    vertical neighbour pairs of |G| that the edge test reads."""
    mod = contour_moduli(g)[1:-1, 1:-1]
    pairs = [(mod[:, 1:], mod[:, :-1]), (mod[:, :-1], mod[:, 1:]), (mod[1:, :], mod[:-1, :]), (mod[:-1, :], mod[1:, :])]
    guarded = sum(int(((a > b) & (a - b < GREATER_EPS)).sum()) for a, b in pairs)
    above = sum(int((a - b >= GREATER_EPS).sum()) for a, b in pairs)
    return guarded, above
