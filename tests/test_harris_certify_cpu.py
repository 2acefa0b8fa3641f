"""CPU check of the certified Harris fast path's error bound (harris_eps, image_b200/csrc/harris_kernels3.cuh):
the fused kernel's fp32 arithmetic, emulated operation by operation in numpy (tests/harris_emul.py), stays within
eps of the oracle's R (double accumulation, reference order) on adversarial frames, evaluated per 8x8 block exactly
like the kernel (block maximum of the trace, maximum |pixel| of the neighbourhood that can reach the block)."""
import numpy as np
import pytest
from scipy.ndimage import maximum_filter

import harris_emul as E


def _frames():
    rng = np.random.default_rng(42)
    ny, nx = 136, 200
    yy, xx = np.mgrid[0:ny, 0:nx]
    out = {}
    out["noise_full_range"] = rng.integers(0, 256, (ny, nx)).astype(np.uint8)
    out["checker_1px"] = (((yy + xx) & 1) * 255).astype(np.uint8)
    out["checker_8px"] = ((((yy >> 3) + (xx >> 3)) & 1) * 255).astype(np.uint8)
    out["bright_flat_with_impulses"] = np.full((ny, nx), 255, np.uint8)
    out["bright_flat_with_impulses"][rng.integers(0, ny, 40), rng.integers(0, nx, 40)] = 0
    out["bright_small_noise"] = (250 + rng.integers(0, 6, (ny, nx))).astype(np.uint8)
    out["ramp_plus_noise"] = np.clip(xx * 255.0 / nx + rng.integers(0, 4, (ny, nx)), 0, 255).astype(np.uint8)
    step = np.where(xx > nx // 2, 255, 0).astype(np.uint8)
    step[yy > ny // 2] = 255 - step[yy > ny // 2]
    out["step_corner"] = step
    from image_b200 import synth
    out["shapes"] = synth.frame_shapes(7, ny, nx)
    return out


@pytest.mark.parametrize("grad", [0, 1])
@pytest.mark.parametrize("name", list(_frames().keys()))
def test_fp32_chain_stays_within_the_certified_bound(oracle, name, grad):
    img = _frames()[name]
    Rf, tr = E.fused_response(img, grad=grad)
    Ro, _ = oracle.harris_response(img, grad=grad, measure=0)
    ny, nx = img.shape
    c = 16                                                       # emulation ignores the frame border
    # per 8x8 block: max trace; M = max |pixel| within the 12-pixel halo of the block (<= the kernel's tile maximum)
    by, bx = ny // 8, nx // 8
    T = tr[: by * 8, : bx * 8].reshape(by, 8, bx, 8).max(axis=(1, 3))
    M = maximum_filter(img.astype(np.float32), size=8 + 24 + 1)[4: by * 8: 8, 4: bx * 8: 8]
    eps = np.kron(E.eps(T, M), np.ones((8, 8), np.float32))
    diff = np.abs(Rf[: by * 8, : bx * 8].astype(np.float64) - Ro[: by * 8, : bx * 8].astype(np.float64))
    ratio = (diff / eps)[c:-c, c:-c]
    assert ratio.max() < 1.0, (name, grad, float(ratio.max()))
    # the bound is not vacuous: it stays below 2 % of the local response scale wherever the response is significant
    scale = maximum_filter(np.abs(Ro), size=15)[: by * 8, : bx * 8]
    sig = scale > 1.0
    if sig.any():
        assert np.median(eps[sig] / scale[sig]) < 2e-2


def _grid():
    """(sigma_d, sigma_i, k) beyond the defaults: every sigma_i of the fused kernel, every sigma_d, every k."""
    import harris_cases as H
    out = [(1.0, float(s), 0.06) for s in H.SIGMA_I if H.fused_supported(64, 64, 1.0, s)]
    out += [(float(d), s, 0.06) for d in H.SIGMA_D[1:] for s in (1.0, 1.3, 2.5)]
    out += [(1.15, s, k) for k in H.K for s in (1.2, 2.5)]
    return out


def _worst_ratio(oracle, img, sigma_d, sigma_i, k, grad):
    """max |R_fp32 - R_oracle| / eps over the interior, eps per 8x8 block as the kernel evaluates it (M = max |pixel|)."""
    Rf, tr = E.fused_response(img, k=k, sigma_d=sigma_d, sigma_i=sigma_i, grad=grad)
    Ro, _ = oracle.harris_response(img, grad=grad, measure=0, k=k, sigma_d=sigma_d, sigma_i=sigma_i)
    ny, nx = img.shape
    by, bx = ny // 8, nx // 8
    T = tr[: by * 8, : bx * 8].reshape(by, 8, bx, 8).max(axis=(1, 3))
    M = maximum_filter(np.abs(img.astype(np.float32)), size=8 + 24 + 1)[4: by * 8: 8, 4: bx * 8: 8]
    eps = np.kron(E.eps(T, M, k), np.ones((8, 8), np.float32))
    diff = np.abs(Rf[: by * 8, : bx * 8].astype(np.float64) - Ro[: by * 8, : bx * 8].astype(np.float64))
    return float((diff / eps)[16:-16, 16:-16].max())


@pytest.mark.parametrize("sigma_d,sigma_i,k", _grid())
def test_bound_holds_beyond_the_default_parameters(oracle, sigma_d, sigma_i, k):
    """The bound is derived for any k (through |k|) and any normalised taps: checked on every adversarial frame, both
    gradients, over the sigma / k grid the certified path accepts (sigma_i of both window radii families, k = 0, k < 0)."""
    worst = 0.0
    for name, img in _frames().items():
        for grad in (0, 1):
            worst = max(worst, _worst_ratio(oracle, img, sigma_d, sigma_i, k, grad))
    assert worst < 1.0, worst


@pytest.mark.parametrize("sigma_i,k", [(1.0, 0.06), (1.3, -0.05), (2.5, 0.06), (2.5, 0.15)])
def test_bound_holds_on_float_input(oracle, sigma_i, k):
    """Float frames (where M is the largest |pixel| of the tile): [0, 1] images, 16-bit ranges, negative values and
    non-integer values."""
    rng = np.random.default_rng(4)
    worst = 0.0
    for name in ("noise_full_range", "checker_8px", "shapes", "step_corner"):
        x = _frames()[name].astype(np.float32)
        for img in (x / np.float32(255), x * np.float32(257), x - np.float32(128),
                    x + rng.uniform(-0.5, 0.5, x.shape).astype(np.float32)):
            for grad in (0, 1):
                worst = max(worst, _worst_ratio(oracle, img.astype(np.float32), 1.15, sigma_i, k, grad))
    assert worst < 1.0, worst


def test_bound_fails_when_shrunk(oracle):
    """The check above has teeth: the bound is a worst-case one (every rounding at its maximum, all with the same sign)
    and sits a few hundred times above the observed error; divided by 1000 it is violated somewhere."""
    img = _frames()["noise_full_range"]
    Rf, tr = E.fused_response(img)
    Ro, _ = oracle.harris_response(img, grad=0, measure=0)
    by, bx = img.shape[0] // 8, img.shape[1] // 8
    T = tr[: by * 8, : bx * 8].reshape(by, 8, bx, 8).max(axis=(1, 3))
    eps = np.kron(E.eps(T, np.float32(255.0)), np.ones((8, 8), np.float32)) / 1000.0
    diff = np.abs(Rf[: by * 8, : bx * 8].astype(np.float64) - Ro[: by * 8, : bx * 8].astype(np.float64))
    assert (diff / eps)[16:-16, 16:-16].max() > 1.0


@pytest.mark.parametrize("Th", [1.0, 130.0, 5000.0])
@pytest.mark.parametrize("name", list(_frames().keys()))
def test_trace_cut_only_removes_pixels_below_the_threshold(oracle, name, Th):
    """harris_trace_cut: a pixel whose fused (fp32) trace is below the cut has a reference response below the threshold,
    so the certified path may drop it (it is stored as -FLT_MAX).  Checked against the oracle's R on the adversarial
    frames; frames with gentle content make the cut bite (most of their pixels fall under it)."""
    img = _frames()[name]
    c = 16
    for grad in (0, 1):
        _, tr = E.fused_response(img, grad=grad)
        Ro, _ = oracle.harris_response(img, grad=grad, measure=0)
        cut = E.trace_cut(Th)
        assert cut > 0
        below = (tr < cut)[c:-c, c:-c]
        assert np.all(Ro[c:-c, c:-c][below] < np.float32(Th)), (name, grad, Th)
        # the margin of the certificate: the largest reference response among the removed pixels stays well below Th
        if below.any():
            assert float(Ro[c:-c, c:-c][below].max()) <= Th * 1.0


def test_trace_cut_bites_on_flat_noise_and_is_tight_enough(oracle):
    """On small-noise content nearly every pixel is certified below Th = 130 by its trace alone; and the cut is not
    vacuous the other way: no pixel with a reference response >= Th has a trace below 2*sqrt(Th) at all."""
    rng = np.random.default_rng(5)
    img = (100 + rng.integers(0, 8, (136, 200))).astype(np.uint8)
    _, tr = E.fused_response(img)
    Ro, _ = oracle.harris_response(img, grad=0, measure=0)
    cut = E.trace_cut(130.0)
    assert (tr < cut)[16:-16, 16:-16].mean() > 0.99
    img2 = _frames()["noise_full_range"]
    _, tr2 = E.fused_response(img2)
    Ro2, _ = oracle.harris_response(img2, grad=0, measure=0)
    hot = Ro2[16:-16, 16:-16] >= 130.0
    assert hot.any() and tr2[16:-16, 16:-16][hot].min() >= 2 * np.sqrt(130.0)
