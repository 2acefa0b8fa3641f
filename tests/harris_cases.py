"""Harris parameter sets beyond the defaults, shared by the CPU tests (oracle against the reference build, emulated error
bound) and the GPU tests (CUDA against the oracle), and the rules that decide which kernels a parameter set reaches.

The rules restate the C code in float32 where it computes in float32: the half-width of the Gaussian taps is
(int)(3 * sigma) (gaussian.cpp:306-329), the NMS window radius (int)(2 * sigma_i + 0.5) (harris.cpp:523).  The fused
kernel exists for sigma_d taps of half-width 3 and sigma_i taps of half-width 3 or 7 (harris_fused_supported), and the
certified corner path additionally needs the Harris measure and an NMS radius of 2, 3 or 5 (harris_certified_supported).
"""
import numpy as np

F = np.float32


def taps_halfwidth(sigma):
    return int(F(3) * F(sigma))


def nms_radius(sigma_i):
    return int(float(F(2) * F(sigma_i)) + 0.5)


def sigma_below(n):
    """The largest float32 sigma whose taps have half-width n - 1 (3 * sigma rounds below n)."""
    s = F(n / 3.0)
    while taps_halfwidth(s) >= n:
        s = np.nextafter(s, F(0))
    while taps_halfwidth(np.nextafter(s, F(100))) < n:
        s = np.nextafter(s, F(100))
    return s


def sigma_above(n):
    """The smallest float32 sigma whose taps have half-width n."""
    return np.nextafter(sigma_below(n), F(100))


# sigma_i: radius 2 (1.0, 1.2), radius 3 (1.25, 1.3, just below 4/3), radius 5 (just above 7/3, 2.34, 2.5, 2.65), and
# the float32 neighbours of 4/3 and 7/3 on the staged side (half-widths 4 and 6: no fused kernel)
SIGMA_I = [F(1.0), F(1.2), F(1.25), F(1.3), sigma_below(4), sigma_above(4), sigma_below(7), sigma_above(7),
           F(2.34), F(2.5), F(2.65)]
SIGMA_D = [F(1.0), F(1.15), F(1.33)]
K = [0.0, 0.04, 0.06, 0.15, -0.05, -2.0]


def fused_supported(nx, ny, sigma_d=1.0, sigma_i=2.5, gaussian=0, **_):
    return (gaussian == 0 and sigma_d > 0 and sigma_i > 0 and taps_halfwidth(sigma_d) == 3
            and taps_halfwidth(sigma_i) in (3, 7) and nx >= 32 and ny >= 32)


def certified_supported(nx, ny, sigma_d=1.0, sigma_i=2.5, gaussian=0, measure=0, **_):
    r = nms_radius(sigma_i)
    return (fused_supported(nx, ny, sigma_d, sigma_i, gaussian) and measure == 0 and r in (2, 3, 5)
            and ny > 2 * r + 1 and nx > 2 * r + 1)


def levels(nx, ny, Nscales=1, sigma_i=2.5, **_):
    """(nx, ny, sigma_i) of every level harris_scale (harris.cpp:554-608) computes, coarsest first."""
    if Nscales <= 1 or nx <= 64 or ny <= 64:
        return [(nx, ny, F(sigma_i))]
    return levels(nx // 2, ny // 2, Nscales - 1, F(sigma_i) / F(2)) + [(nx, ny, F(sigma_i))]


def any_level_certified(nx, ny, **kw):
    return any(certified_supported(x, y, **dict(kw, sigma_i=s)) for x, y, s in levels(nx, ny, **kw))


def reference_cases():
    """(key, image, detect_corners keywords) of the parameter sets whose oracle output is pinned to the reference build
    (tests/golden/ref_digests.json): every sigma_i, sigma_d and k above, both gradients, the sub-pixel modes and output
    strategies, two and three scales, and float input (scaled, shifted, non-integer)."""
    from image_b200 import synth
    img = synth.frame_shapes(700, 96, 136)
    big = synth.frame_shapes(701, 272, 300)
    for j, s in enumerate(SIGMA_I):
        for g in (0, 1):
            yield "harris_p_si%d_g%d" % (j, g), img, dict(threshold=10, sigma_i=float(s), gradient=g)
    for j, s in enumerate(SIGMA_D):
        for si in (F(1.0), F(1.3), F(2.5)):
            yield "harris_p_sd%d_si%s" % (j, si), img, dict(threshold=10, sigma_d=float(s), sigma_i=float(si))
    for j, k in enumerate(K):
        for si in (F(1.2), F(2.5)):
            yield "harris_p_k%d_si%s" % (j, si), img, dict(threshold=10, k=k, sigma_i=float(si))
    for pr in (0, 1, 2):
        for st in (0, 1, 2, 3):
            yield "harris_p_pr%d_st%d" % (pr, st), img, dict(threshold=10, precision=pr, strategy=st, Nselect=20, cells=4,
                                                            sigma_i=1.2 if st % 2 else 2.5)
    for ns in (2, 3):
        for si in (F(2.5), F(2.4)):
            yield "harris_p_ns%d_si%s" % (ns, si), big, dict(threshold=20, Nscales=ns, sigma_i=float(si), precision=ns - 1)
    x = img.astype(np.float64)
    rng = np.random.default_rng(8)
    for name, v, th in (("unit", x / 255.0, 10 / 255.0 ** 4), ("u16", x * 257.0, 10 * 257.0 ** 4), ("centred", x - 128.0, 10),
                        ("noisy", x + rng.uniform(-0.5, 0.5, x.shape), 10)):
        for si in (F(1.2), F(2.5)):
            yield "harris_p_%s_si%s" % (name, si), v, dict(threshold=th, sigma_i=float(si), precision=2)
