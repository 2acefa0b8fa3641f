"""Face detection on the H100 against the reference build (oracle/_ref/libref_facedetect.so), exactly: the per-frame maximum
of all 16 ReLU layers, the candidate records of the head pass, and the 15 ints of every detection in order."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from image_b200 import _lib, synth
from image_b200.facedetect import FaceModel, detect_faces, facedetect_batch, facedetect_dev, image_detect_faces, load_model, read_layers
from oracle import ref_facedetect as rf

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "facedetect_handshake.npz")
pytestmark = [pytest.mark.gpu, pytest.mark.skipif(not rf.have_ref(), reason="reference build oracle/_ref/libref_facedetect.so absent")]
CAP = 600000


@pytest.fixture(scope="module")
def model():
    m = load_model(rf.SO_PATH)
    yield m
    m.free()


def handshake():
    return np.load(GOLDEN)["rgb"]


def mosaic(tile, H=2160, W=3840):
    ry, rx = -(-H // tile.shape[0]), -(-W // tile.shape[1])
    return np.ascontiguousarray(np.tile(tile, (ry, rx, 1))[:H, :W])


def downscale(a, k):
    h, w = a.shape[0] // k * k, a.shape[1] // k * k
    return a[:h, :w].reshape(h // k, k, w // k, k, 3).mean(axis=(1, 3)).round().astype(np.uint8)


def run_dev(frames, model):
    import torch
    a = np.ascontiguousarray(np.stack(frames), dtype=np.uint8)
    d = torch.from_numpy(a).cuda()
    n, h, w = a.shape[:3]
    out = facedetect_dev(d, n, w, h, model, layer_max=True, cand_cap=CAP)
    torch.cuda.synchronize()
    return out


def check_against_oracle(frames, model):
    """Every frame of one device batch against the layer driver; returns the driver's results."""
    out = run_dev(frames, model)
    lays = []
    for f, fr in enumerate(frames):
        lay = rf.layers(fr)
        lays.append(lay)
        assert np.array_equal(out["layer_max"][f], lay["nmax"]), (f, out["layer_max"][f], lay["nmax"])
        want = rf.candidates(lay)
        assert out["n_cand"][f] == len(want), f
        assert np.array_equal(out["cand"][f, :len(want)], want), f
        n = out["n_faces"][f]
        assert n == len(lay["ints"]) and np.array_equal(out["faces"][f, :n], lay["ints"]), f
        assert not out["faces"][f, n:].any()
    return out, lays


def test_handshake(model):
    fr = handshake()
    out, lays = check_against_oracle([fr], model)
    g = np.load(GOLDEN)["faces"]
    assert out["n_faces"][0] == len(g) == 3 and np.array_equal(out["faces"][0, :3], g)


def test_mosaic_4k(model):
    out, lays = check_against_oracle([mosaic(handshake())], model)
    assert out["n_faces"][0] == 100 and lays[0]["n_nms"] > 100


def test_dense_mosaic_hits_top_k_and_keep_top_k(model):
    fr = mosaic(downscale(handshake(), 3))
    out, lays = check_against_oracle([fr], model)
    assert lays[0]["n_above"] > 1000, "top_k branch not reached"
    assert lays[0]["n_nms"] > 100, "keep_top_k branch not reached"
    assert out["n_faces"][0] == 100


@pytest.mark.parametrize("h,w", [(64, 64), (63, 65), (97, 131), (128, 200), (301, 257), (480, 640)])
def test_synthetic_sizes(model, h, w):
    check_against_oracle([synth.frame_rgb(h * 7 + w, h, w), synth.frame_rgb(h + w, h, w, noise=200)], model)


@pytest.mark.parametrize("other", [64, 200])
def test_sizes_across_pool_collapse(model, other):
    for s in range(56, 73):
        for h, w in ((s, other), (other, s)):
            out, lays = check_against_oracle([synth.frame_rgb(s * 31 + other, h, w, noise=120)], model)
            runs = (lays[0]["nmax"] >= 0).all()
            assert runs == (s >= 63), (h, w)            # the fifth pool needs 63 px in each dimension


def test_degenerate_content_in_one_batch(model, capsys):
    h, w = 160, 224
    rng = np.random.default_rng(9)
    frames = [np.full((h, w, 3), v, np.uint8) for v in (0, 128, 255)]
    frames.append(rng.integers(0, 2, (h, w, 3)).astype(np.uint8))                 # a [0, 1]-valued frame
    frames.insert(2, synth.frame_rgb(11, h, w))
    frames.append(mosaic(downscale(handshake(), 4), h, w))
    out, lays = check_against_oracle(frames, model)
    zero = [(f, int(np.nonzero(l["nmax"] == 0)[0][0])) for f, l in enumerate(lays) if (l["nmax"] == 0).any()]
    with capsys.disabled():
        print("\nframes with a layer of nMax == 0 (frame, first layer):", zero or "none")


def test_r32_narrowing_wraps(model):
    fr = handshake()[:200, :300]
    rng = np.random.default_rng(3)
    x = fr.astype(np.int32) + 256 * rng.integers(-3, 4, fr.shape).astype(np.int32)
    r = image_detect_faces(x, model)
    want = rf.facedetect_cnn((x & 255).astype(np.uint8))
    assert r["nr"] == len(want)
    for k, c in enumerate(("confidence", "x", "y", "width", "height")):
        assert np.array_equal(r["detections"][c], want[:, k])


def test_forms_agree_across_chunks(model):
    # 4K frames need ~0.4 GB of scratch each: six of them make two chunks of the batch entry
    base = mosaic(handshake())
    frames = np.stack([np.roll(base, (37 * i, 91 * i), axis=(0, 1)) for i in range(6)])
    nf, faces = facedetect_batch(frames, model)
    dev = run_dev(list(frames), model)
    assert np.array_equal(nf, dev["n_faces"]) and np.array_equal(faces, dev["faces"])
    for i in (0, 5):
        r = detect_faces(frames[i].astype(np.int32).ravel(), 3840, 2160, 3 * 3840, model)
        assert r["nr"] == nf[i] and np.array_equal(r["detections"]["x"], faces[i, :nf[i], 1])
    assert nf.min() > 0


def test_bad_arguments(model):
    lib, tab = read_layers(rf.SO_PATH)
    bad = (type(tab))()
    C.memmove(bad, tab, C.sizeof(tab))
    bad[3].channels = 16
    with pytest.raises(_lib.B2FError) as e:
        FaceModel(bad)
    assert e.value.code == _lib.B2F_EINVAL
    C.memmove(bad, tab, C.sizeof(tab))
    bad[5].pad = 1
    with pytest.raises(_lib.B2FError) as e:
        FaceModel(bad)
    assert e.value.code == _lib.B2F_EINVAL
    h = C.c_void_p()
    assert _lib.load().b2f_facedet_model_create(_lib.context(), C.cast(tab, C.c_void_p), 23, C.byref(h)) == _lib.B2F_EINVAL
    fr = handshake()[:100, :100].astype(np.int32).ravel()
    with pytest.raises(_lib.B2FError) as e:
        detect_faces(fr, 100, 100, 301, model)
    assert e.value.code == _lib.B2F_EINVAL
    with pytest.raises(_lib.B2FError) as e:
        detect_faces(fr[:-1], 100, 100, 300, model)
    assert e.value.code == _lib.B2F_EINVAL
    assert detect_faces(fr, 0, 100, 0, model)["nr"] == 0
    assert detect_faces(fr, 100, 100, 300, model)["nr"] == len(rf.facedetect_cnn(handshake()[:100, :100]))   # context still works


HARNESS = r"""
#include <Rcpp.h>
#include <cstring>
Rcpp::List detect_faces(Rcpp::IntegerVector x, int width, int height, int step);
extern "C" int shim_detect(const int *x, int n, int w, int h, int step, int *out) {
  try {
    Rcpp::IntegerVector v(x, (size_t)n);
    Rcpp::List l = detect_faces(v, w, h, step);
    const Rcpp::Value &d = l.get("detections");
    for (size_t i = 0; i < d.data.size(); i++) out[i] = (int)d.data[i];
    return (int)l.get("nr").data[0] * 1000 + (int)d.nc;
  } catch (std::exception &e) { return -1; }
}
"""


def test_rshim(tmp_path):
    src = tmp_path / "harness.cpp"
    src.write_text(HARNESS)
    lib = str(tmp_path / "libfdshim.so")
    subprocess.check_call(["g++", "-O1", "-std=c++17", "-fPIC", "-shared", "-I" + os.path.join(ROOT, "oracle", "stubs"),
                           "-I" + os.path.join(ROOT, "include"), "-I" + os.path.join(ROOT, "image_b200", "rshim"), str(src),
                           os.path.join(ROOT, "image_b200", "rshim", "rcpp_libfacedetection.cpp"), rf.SO_PATH,
                           "-L" + os.path.join(ROOT, "image_b200"), "-lb200feat",
                           "-Wl,-rpath," + os.path.join(ROOT, "image_b200") + ":" + os.path.dirname(rf.SO_PATH), "-o", lib])
    shim = C.CDLL(lib)
    for fr in (handshake(), synth.frame_rgb(4, 90, 120)):
        h, w = fr.shape[:2]
        v = np.ascontiguousarray(fr.astype(np.int32).ravel())
        out = np.zeros(256 * 15, np.int32)
        rc = shim.shim_detect(v.ctypes.data_as(C.c_void_p), v.size, w, h, 3 * w, out.ctypes.data_as(C.c_void_p))
        want = rf.facedetect_cnn(fr)
        assert rc == len(want) * 1000 + 15
        cols = out[:15 * len(want)].reshape(15, len(want)).T          # x, y, width, height, confidence, landmarks
        assert np.array_equal(cols[:, [4, 0, 1, 2, 3] + list(range(5, 15))], want)
