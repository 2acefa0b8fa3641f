"""GPU parity tests of NL-means denoising (image.DenoiseNLMeans) against the serial reference build (oracle/_ref) and
its frozen digests (tests/golden/nlmeans_digests.json).  Every comparison is bit for bit on the float32 results."""
import ctypes as C
import json
import os
import subprocess

import numpy as np
import pytest

import nlmeans_cases as nc

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def ref(oracle):
    from oracle import ref_nlmeans as rn
    if not rn.have_ref():
        rn.build()
    if not rn.have_ref():
        pytest.skip("oracle/_ref/libref_nlmeans.so not built (reference tree absent)")
    return rn


def _same(got, want):
    assert got["channels"] == want["channels"]
    assert (got["window"], got["bloc"]) == (want["window"], want["bloc"])
    assert np.float32(got["filter"]) == np.float32(want["filter"])
    g = np.asarray(got["denoised"], np.float32)
    w = np.asarray(want["denoised"], np.float32)
    assert g.shape == w.shape
    bad = np.flatnonzero(g.view(np.uint32) != w.view(np.uint32))
    assert bad.size == 0, "%d of %d values differ, first at %d: %r vs %r" % (bad.size, g.size, bad[0], g[bad[0]], w[bad[0]])


def _run_both(ref, img, sigma, args_auto=True, win=1, bloc=10, filt=0.4):
    from image_b200.nlmeans import rcpp_nlmeans
    c, h, w = img.shape
    got = rcpp_nlmeans(img.ravel(), w, h, c, sigma, args_auto, win, bloc, filt)
    want = ref.nlmeans(img.ravel(), w, h, c, sigma, args_auto, win, bloc, filt)
    _same(got, want)
    return got


def _rgb(seed, h, w, std):
    from image_b200 import synth
    return nc.noisy(synth.frame_rgb(seed, h, w).transpose(2, 0, 1), std, seed)


def _grey(seed, h, w, std):
    from image_b200 import synth
    return nc.noisy(synth.frame_shapes(seed, h, w)[None], std, seed)


# every row of both tables, and sigma <= 0 (which takes the last row)
@pytest.mark.parametrize("sigma,shape", [(10, (48, 64)), (20, (48, 64)), (40, (40, 56)), (60, (36, 48)), (90, (36, 48)),
                                         (-5, (30, 40))])
def test_auto_table_grey(ref, sigma, shape):
    _run_both(ref, _grey(int(abs(sigma)) + 3, *shape, max(abs(sigma), 1)), sigma)


@pytest.mark.parametrize("sigma,shape", [(10, (48, 64)), (40, (40, 56)), (80, (36, 48)), (-5, (30, 40))])
def test_auto_table_colour(ref, sigma, shape):
    _run_both(ref, _rgb(int(abs(sigma)) + 4, *shape, abs(sigma)), sigma)


def test_auto_table_larger_frame(ref):
    _run_both(ref, _rgb(5, 120, 160, 15), 15)


@pytest.mark.parametrize("c,win,bloc,filt,sigma", [(1, 0, 5, 0.5, 12), (3, 0, 4, 0.7, 9), (1, 2, 0, 0.4, 10), (3, 1, 0, 0.4, 10),
                                                   (1, 7, 4, 0.5, 20), (3, 4, 3, 0.45, 25), (1, 3, 6, 1.2, 5), (3, 2, 5, 0.4, 30)])
def test_explicit_parameters(ref, c, win, bloc, filt, sigma):
    img = _grey(win + bloc, 33, 41, sigma) if c == 1 else _rgb(win + bloc, 29, 37, sigma)
    _run_both(ref, img, sigma, False, win, bloc, filt)


@pytest.mark.parametrize("h,w", [(1, 1), (1, 9), (9, 1), (2, 7), (7, 2), (13, 11), (19, 20), (37, 23), (23, 37)])
def test_shapes(ref, h, w):
    _run_both(ref, _rgb(h * 100 + w, h, w, 20), 20)              # colour: win 1, bloc 10 (wider than most of these)
    _run_both(ref, _grey(h * 100 + w, h, w, 50), 50)             # grey: win 4, bloc 17
    _run_both(ref, _grey(h + w, h, w, 10), 10, False, 3, 2, 0.6)


def test_flat_frame(ref):
    for c in (1, 3):
        img = np.full((c, 30, 44), 117, np.int32)
        if c == 3:
            img[1] += 3
        r = _run_both(ref, img, 10)
        assert np.all(r["denoised"] == np.repeat(img.reshape(c, -1).astype(np.float64), 1, axis=1).ravel())


def test_zero_weights_leave_pixels_uncounted(ref):
    """A random texture with sigma 1: every candidate weighs 0, the total stays at 0 <= fTiny, those centres add nothing
    and their pixels keep the input value (count 0)."""
    rng = np.random.default_rng(11)
    img = rng.integers(0, 256, (1, 40, 60)).astype(np.int32)
    img[:, :, :20] = 90
    r = _run_both(ref, img, 1.0, False, 1, 6, 0.5)
    out = r["denoised"].reshape(40, 60)
    same = out == img[0]
    assert same[:, 30:].mean() > 0.9                              # uncounted pixels exist and take the input


def test_lut_cell_boundaries_and_cut(ref):
    """win 0, filter 1, sigma 1: fH2 = C and the offset 2C, so integer differences put d on LUT cell boundaries; in
    colour a squared distance of 93 gives d = 29.0f exactly, the cut of wxSLUT.  Grey win 1 reaches it at 279."""
    rng = np.random.default_rng(12)
    img3 = rng.integers(0, 10, (3, 24, 30)).astype(np.int32)
    d2 = lambda a, b: sum(((a[k] - b[k]).astype(np.int64) ** 2) for k in range(3))
    hits = sum(int(np.count_nonzero(d2(img3[:, :, dx:], img3[:, :, :30 - dx]) == 93)) for dx in range(1, 5))
    assert hits > 0
    _run_both(ref, img3, 1.0, False, 0, 4, 1.0)
    _run_both(ref, img3[:1], 1.0, False, 0, 4, 1.0)
    _run_both(ref, rng.integers(0, 7, (1, 24, 30)).astype(np.int32), 1.0, False, 1, 4, 1.0)


def test_colour_test(ref):
    from image_b200.nlmeans import rcpp_nlmeans
    g = _grey(31, 26, 34, 20)[0]
    img = np.stack([g, g, g])
    r = _run_both(ref, img, 20)
    assert r["channels"] == 1 and r["window"] == 2                    # grey table row, one plane out
    img2 = img.copy()
    img2[2, -1, -1] += 1
    r2 = _run_both(ref, img2, 20)
    assert r2["channels"] == 3 and r2["window"] == 1
    # channels 2 uses plane 0 only, channels 4 the first three planes
    four = np.concatenate([img2, img2[:1]])
    _same(rcpp_nlmeans(four.ravel(), 34, 26, 4, 20), ref.nlmeans(four.ravel(), 34, 26, 4, 20))
    _same(rcpp_nlmeans(img2[:2].ravel(), 34, 26, 2, 20), ref.nlmeans(img2[:2].ravel(), 34, 26, 2, 20))


def test_sigma_above_100_raises_the_reference_message(oracle):
    from image_b200 import B2FError
    from image_b200.nlmeans import rcpp_nlmeans
    msg = "error :: algorithm parametrized only for values of sigma less than 100.0"
    for c in (1, 3):
        img = np.arange(c * 12).astype(np.int32)
        with pytest.raises(B2FError, match="sigma less than 100.0") as e:
            rcpp_nlmeans(img, 4, 3, c, 100.5)
        assert msg in str(e.value)
        from oracle import ref_nlmeans as rn
        if rn.have_ref():
            with pytest.raises(ValueError, match="sigma less than 100.0"):
                rn.nlmeans(img, 4, 3, c, 100.5)
    rcpp_nlmeans(np.arange(36).astype(np.int32), 4, 3, 3, 100.5, False, 1, 2, 0.4)      # explicit parameters: no limit


@pytest.fixture(scope="module")
def digests():
    with open(os.path.join(ROOT, "tests", "golden", "nlmeans_digests.json")) as f:
        return json.load(f)


def test_frozen_digests(oracle, digests):
    import torch
    from image_b200.nlmeans import nlmeans_dev, nlmeans_resolve, rcpp_nlmeans
    for key, img, sigma in nc.digest_cases():
        c, h, w = img.shape
        r = rcpp_nlmeans(img.ravel(), w, h, c, sigma)
        assert nc.digest_of(oracle, r) == digests[key], key
        win, bloc, filt = nlmeans_resolve(c, sigma)
        d = torch.from_numpy(np.ascontiguousarray(img, dtype=np.uint8)).cuda()
        out = torch.empty((c, h, w), dtype=torch.float32, device="cuda")
        nlmeans_dev(d, 1, c, w, h, win, bloc, sigma, filt, out)
        torch.cuda.synchronize()
        rd = dict(denoised=out.cpu().numpy().ravel().astype(np.float64), channels=c, window=win, bloc=bloc, filter=filt)
        assert nc.digest_of(oracle, rd) == digests[key], key


def _dev_frames():
    from image_b200 import synth
    h, w = 45, 61
    fs = [_rgb(40, h, w, 25), np.full((3, h, w), 200, np.int32), np.random.default_rng(41).integers(0, 256, (3, h, w)),
          synth.frame_rgb(42, h, w).transpose(2, 0, 1), _rgb(43, h, w, 5)]
    return np.stack(fs).astype(np.uint8)


@pytest.mark.parametrize("c,win,bloc", [(3, 1, 10), (3, 2, 6), (1, 3, 17), (1, 6, 3)])
def test_dev_batch_equals_single_calls_on_a_caller_stream(c, win, bloc):
    import torch
    from image_b200.nlmeans import nlmeans_dev
    f = _dev_frames()[:, :c]
    n, _, h, w = f.shape
    d = torch.from_numpy(np.ascontiguousarray(f)).cuda()
    guard = 4096
    buf = torch.full((2 * guard + n * c * h * w,), -7.25, dtype=torch.float32, device="cuda")
    out = buf[guard:guard + n * c * h * w]
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        nlmeans_dev(d, n, c, w, h, win, bloc, 25.0, 0.4, out, stream=s.cuda_stream)
    s.synchronize()
    g = buf.cpu().numpy()
    assert np.all(g[:guard] == -7.25) and np.all(g[-guard:] == -7.25)
    batch = out.cpu().numpy().reshape(n, c, h, w)
    for i in range(n):
        one = torch.empty((c, h, w), dtype=torch.float32, device="cuda")
        nlmeans_dev(d[i], 1, c, w, h, win, bloc, 25.0, 0.4, one)
        torch.cuda.synchronize()
        assert np.array_equal(batch[i].view(np.uint32), one.cpu().numpy().view(np.uint32)), i


def test_dev_matches_reference_with_channel_mapping(ref):
    import torch
    from image_b200.nlmeans import nlmeans_dev
    f = _dev_frames()[[0, 2]]                                            # two colour frames
    n, _, h, w = f.shape
    d = torch.from_numpy(np.ascontiguousarray(np.concatenate([f, f[:, :1]], axis=1))).cuda()   # 4 planes: the first 3 are used
    out = torch.empty((n, 3, h, w), dtype=torch.float32, device="cuda")
    nlmeans_dev(d, n, 4, w, h, 2, 7, 18.0, 0.5, out)
    torch.cuda.synchronize()
    for i in range(n):
        want = ref.nlmeans(f[i].astype(np.int32).ravel(), w, h, 3, 18.0, False, 2, 7, 0.5)
        assert want["channels"] == 3
        _same(dict(denoised=out[i].cpu().numpy().ravel(), channels=3, window=2, bloc=7, filter=0.5), want)


def test_dev_rejects_bad_arguments():
    import torch
    from image_b200 import B2FError
    from image_b200.nlmeans import nlmeans_dev
    d = torch.zeros((1, 3, 8, 8), dtype=torch.uint8, device="cuda")
    out = torch.zeros((3, 8, 8), dtype=torch.float32, device="cuda")
    for args in [(1, 3, 8, 8, -1, 3), (1, 3, 8, 8, 1, -1), (1, 0, 8, 8, 1, 3), (0, 3, 8, 8, 1, 3), (1, 3, 0, 8, 1, 3),
                 (1, 3, 8, -2, 1, 3), (1, 3, 8, 8, 20000, 3)]:
        with pytest.raises(B2FError):
            nlmeans_dev(d, *args, 10.0, 0.4, out)
    nlmeans_dev(d, 1, 3, 8, 8, 1, 3, 10.0, 0.4, out)                     # the context still works
    torch.cuda.synchronize()
    assert torch.all(out == 0)


HARNESS = r"""
#include <Rcpp.h>
#include <cstring>
Rcpp::List rcpp_nlmeans(Rcpp::IntegerVector image, int width, int height, int channels, float sigma, bool args_auto, int win,
                        int bloc, float fFiltPar);
extern "C" int shim_nlmeans(const int *img, int w, int h, int c, float sigma, int args_auto, int win, int bloc, float filt,
                            double *out, int *meta, float *fs) {
  try {
    Rcpp::IntegerVector v(img, (size_t)w * h * c);
    Rcpp::List l = rcpp_nlmeans(v, w, h, c, sigma, args_auto != 0, win, bloc, filt);
    const std::vector<double> &d = l.get("denoised").data;
    for (size_t i = 0; i < d.size(); i++) out[i] = d[i];
    meta[0] = (int)l.get("channels").data[0]; meta[1] = (int)l.get("window").data[0]; meta[2] = (int)l.get("bloc").data[0];
    meta[3] = (int)l.get("width").data[0]; meta[4] = (int)l.get("height").data[0];
    fs[0] = (float)l.get("sigma").data[0]; fs[1] = (float)l.get("filter").data[0];
    return 0;
  } catch (std::exception &e) { return -1; }
}
"""


def test_rshim(ref, tmp_path):
    src = tmp_path / "harness.cpp"
    src.write_text(HARNESS)
    lib = str(tmp_path / "libnlshim.so")
    subprocess.check_call(["g++", "-O1", "-std=c++17", "-fPIC", "-shared", "-I" + os.path.join(ROOT, "oracle", "stubs"),
                           "-I" + os.path.join(ROOT, "include"), "-I" + os.path.join(ROOT, "image_b200", "rshim"), str(src),
                           os.path.join(ROOT, "image_b200", "rshim", "rcpp_nlmeans.cpp"), "-L" + os.path.join(ROOT, "image_b200"),
                           "-lb200feat", "-Wl,-rpath," + os.path.join(ROOT, "image_b200"), "-o", lib])
    shim = C.CDLL(lib)
    shim.shim_nlmeans.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_float, C.c_int, C.c_int, C.c_int, C.c_float,
                                  C.c_void_p, C.c_void_p, C.c_void_p]
    for img, sigma in [(_rgb(50, 40, 52, 30), 30.0), (_grey(51, 40, 52, 45), 45.0)]:
        c, h, w = img.shape
        v = np.ascontiguousarray(img.ravel(), np.int32)
        out = np.zeros(c * h * w)
        meta = np.zeros(5, np.int32)
        fs = np.zeros(2, np.float32)
        assert shim.shim_nlmeans(v.ctypes.data, w, h, c, sigma, 1, 1, 10, 0.4, out.ctypes.data, meta.ctypes.data, fs.ctypes.data) == 0
        want = ref.nlmeans(v, w, h, c, sigma)
        assert (meta[3], meta[4], fs[0]) == (w, h, np.float32(want["sigma"]))
        _same(dict(denoised=out[:meta[0] * h * w], channels=int(meta[0]), window=int(meta[1]), bloc=int(meta[2]), filter=fs[1]), want)


def test_image_denoise_nlmeans_mirror(ref):
    from image_b200 import image_denoise_nlmeans
    g = nc.garden()[:60, :80]
    r = image_denoise_nlmeans(g)
    want = ref.nlmeans(g.transpose(2, 0, 1).astype(np.int32).ravel(), 80, 60, 3, 10.0)
    assert r["x"].shape == g.shape and (r["window"], r["bloc"]) == (want["window"], want["bloc"])
    assert np.array_equal(r["x"], np.minimum(want["denoised"], 255).reshape(3, 60, 80).transpose(1, 2, 0))
    r2 = image_denoise_nlmeans(g, sigma=10, win=2, bloc=5, filter=0.3)                # all three given: no table
    assert (r2["window"], r2["bloc"], np.float32(r2["filter"])) == (2, 5, np.float32(0.3))
    r3 = image_denoise_nlmeans(g, sigma=10, win=2)                                    # one missing: the table
    assert (r3["window"], r3["bloc"]) == (1, 10)
    grey = g[:, :, 1]
    r4 = image_denoise_nlmeans(grey, sigma=20)
    want4 = ref.nlmeans(np.stack([grey] * 3).astype(np.int32).ravel(), 80, 60, 3, 20.0)
    assert want4["channels"] == 1 and np.array_equal(r4["x"], np.minimum(want4["denoised"], 255).reshape(60, 80))
