"""CPU tests: the oracle restatement (oracle/*_oracle.c) against (a) the golden vectors frozen from
the unmodified reference on its own fixtures, (b) the in-place reference build oracle/_ref when it
is present.  No GPU, no product code."""
import ast

import numpy as np
import pytest

HARRIS_CASES = ["default", "cpp_default", "sobel_shi_sorted", "harmonic_quartic_top50", "grid100_quadratic",
                "two_scales", "no_gaussian"]


@pytest.mark.parametrize("fixture", ["chairs", "building"])
@pytest.mark.parametrize("case", HARRIS_CASES)
def test_harris_oracle_matches_golden(oracle, golden, fixture, case):
    g = golden("harris_" + fixture)
    kw = ast.literal_eval(str(g[case + "_args"]))
    x, y, s = oracle.harris_detect(g["image"], impl="oracle", **kw)
    assert len(x) == len(g[case + "_x"])
    # bit-exact: same corners, same order, same float strengths
    assert np.array_equal(x, g[case + "_x"]) and np.array_equal(y, g[case + "_y"])
    assert np.array_equal(s, g[case + "_s"])


def test_harris_oracle_response_matches_golden(oracle, golden):
    g = golden("harris_chairs")
    R, _ = oracle.harris_response(g["image"], impl="oracle")
    assert np.array_equal(R, g["R_default"])


def test_harris_window_predicate_equals_scan_on_tie_free_maps(oracle):
    """SURVEY §8a-H6: on tie-free data the order-free window predicate (what the CUDA kernel
    implements) reproduces the reference scan exactly."""
    rng = np.random.default_rng(7)
    for trial in range(30):
        ny, nx = rng.integers(24, 90), rng.integers(24, 90)
        R = rng.standard_normal((ny, nx)).astype(np.float32) * 100
        r = int(rng.integers(1, 7))
        a = oracle.harris_nms(R, 10.0, r)
        b = oracle.harris_nms(R, 10.0, r, window=True)
        assert np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1]) and np.array_equal(a[2], b[2])
        assert b[3].sum() == 0


def test_harris_nms_small_image_returns_nothing(oracle):
    R = np.ones((11, 40), np.float32) * 1000
    assert len(oracle.harris_nms(R, 1.0, 5)[0]) == 0        # ny <= 2r+1  (harris.cpp:151)


@pytest.mark.parametrize("case", ["default", "cpp_default", "fractional_thr"])
def test_canny_oracle_matches_golden(oracle, golden, case):
    g = golden("canny_chairs")
    kw = ast.literal_eval(str(g[case + "_args"]))
    e, nz = oracle.canny(g["image"], impl="oracle", **kw)
    ref = np.unpackbits(g[case + "_edges"])[: e.size].reshape(e.shape).astype(bool)
    assert nz == int(g[case + "_nonzero"])
    assert np.array_equal(e == 255, ref)          # integer edge map: bit-exact
    assert set(np.unique(e)) <= {0, 255}


def test_canny_taps_are_symmetric_and_normalised(oracle):
    c, w = oracle.canny_taps(1920, 2.0)
    assert c[0] == -c[-1] and np.allclose(w, w[::-1], rtol=0, atol=0)
    assert abs(w.sum() - 1) < 1e-15
    assert len(c) == 27                            # |c| <= 13 for s = 2  (exp(-c^2/4) >= 2^-64)


# ------------------------------------------------------------------ against the reference build's frozen outputs
# (oracle/_ref run on these inputs by tests/golden/make_golden_ref.py: digests in ref_digests.json, Canny blur planes in
# canny_blur_ref.npz)

def harris_random_cases():
    from image_b200 import synth
    for seed, (ny, nx) in enumerate([(120, 200), (97, 131), (256, 64), (70, 70)]):
        img = synth.frame_shapes(100 + seed, ny, nx)
        for j, kw in enumerate([dict(), dict(gaussian=1), dict(gradient=1, measure=2, precision=1), dict(Nscales=2, strategy=1)]):
            yield "harris_%d_%d" % (seed, j), img, dict(threshold=10, **kw)


def harris_tiny_cases():
    rng = np.random.default_rng(3)
    for ny, nx in [(2, 50), (50, 2), (9, 9), (12, 30), (30, 12), (13, 13)]:
        yield "harris_tiny_%dx%d" % (ny, nx), rng.integers(0, 255, (ny, nx)), dict(threshold=0.001)


def canny_cases():
    from image_b200 import synth
    for seed, (ny, nx) in enumerate([(108, 192), (75, 101), (64, 64), (9, 7)]):
        yield "canny_%d" % seed, synth.frame_shapes(200 + seed, ny, nx)


def test_harris_oracle_equals_reference_on_random_frames(oracle, ref_digests):
    for key, img, kw in harris_random_cases():
        assert oracle.digest(*oracle.harris_detect(img, impl="oracle", **kw)) == ref_digests[key], key


def test_harris_tiny_images_match_reference(oracle, ref_digests):
    for key, img, kw in harris_tiny_cases():
        assert oracle.digest(*oracle.harris_detect(img, impl="oracle", **kw)) == ref_digests[key], key


def test_harris_oracle_equals_reference_beyond_default_parameters(oracle, ref_digests):
    """The parameter sets the GPU tests compare against the oracle (tests/harris_cases.py): other sigma_i (both sides of
    the tap half-width boundaries 4/3 and 7/3), sigma_d and k (zero and negative), sub-pixel modes, strategies, scales,
    float input — the oracle's lists and strengths are the reference's bit for bit."""
    import harris_cases
    keys = []
    for key, img, kw in harris_cases.reference_cases():
        assert oracle.digest(*oracle.harris_detect(img, impl="oracle", **kw)) == ref_digests[key], key
        keys.append(key)
    assert len(keys) == len(set(keys)) > 60


def test_canny_oracle_equals_reference_shim(oracle, golden, ref_digests):
    """The restatement (direct circular convolution) against the reference's own tools.c driven by
    the DFT shim: blurred planes may differ in float rounding for ~1e-7 of the pixels; edge maps
    must agree (a flip would need a blur flip AND a gradient tie)."""
    blur_ref = golden("canny_blur_ref")
    for key, img in canny_cases():
        for acc in (True, False):
            eo, no, blur, _ = oracle.canny(img, impl="oracle", accGrad=acc, stages=True)
            flips = int((blur_ref[key] != blur).sum())
            assert flips <= max(1, img.size // 100000)
            assert oracle.digest(eo, np.int64(no)) == ref_digests["%s_%d" % (key, acc)], (key, acc)
