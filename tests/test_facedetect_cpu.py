"""CPU checks of the face-detection oracle (oracle/_ref/libref_facedetect.so, the reference build) and of the facts the GPU
path relies on: the layer driver reproduces facedetect_cnn, the golden detections reproduce, the weight table has the
network's shapes, and the candidate pre-filter (a prior with conf ints i1 <= i0 is never kept) holds with libm's expf."""
import ctypes as C
import ctypes.util
import os

import numpy as np
import pytest

from image_b200 import synth
from image_b200.facedetect import read_layers
from oracle import ref_facedetect as rf

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "facedetect_handshake.npz")
pytestmark = pytest.mark.skipif(not rf.have_ref(), reason="reference build oracle/_ref/libref_facedetect.so absent")

SHAPES = [(3, 3, 32), (1, 32, 16), (3, 16, 32), (1, 32, 32), (3, 32, 64), (1, 64, 32), (3, 32, 64), (3, 64, 128),
          (1, 128, 64), (3, 64, 128), (3, 128, 256), (1, 256, 128), (3, 128, 256), (3, 256, 256), (1, 256, 256),
          (3, 256, 256), (3, 64, 42), (3, 64, 6), (3, 128, 28), (3, 128, 4), (3, 256, 28), (3, 256, 4), (3, 256, 42),
          (3, 256, 6)]


def _frames():
    g = np.load(GOLDEN)
    yield g["rgb"]
    for seed, h, w in [(1, 64, 64), (2, 97, 131), (3, 120, 160)]:
        yield synth.frame_rgb(seed, h, w)


def test_layer_driver_matches_facedetect_cnn():
    for fr in _frames():
        assert np.array_equal(rf.layers(fr)["ints"], rf.facedetect_cnn(fr))


def test_golden_detections_reproduce():
    g = np.load(GOLDEN)
    assert g["rgb"].shape == (192, 592, 3) and len(g["faces"]) == 3
    assert np.array_equal(rf.facedetect_cnn(g["rgb"]), g["faces"])


def test_load_model_reads_the_table():
    _, tab = read_layers(rf.SO_PATH)
    assert len(tab) == 24
    for l, (k, c, n) in enumerate(SHAPES):
        assert (tab[l].kernel_size, tab[l].channels, tab[l].num) == (k, c, n), l
        assert tab[l].weights and tab[l].bias and np.isfinite(tab[l].scale) and tab[l].scale > 0
        if l > 0:
            assert (tab[l].stride, tab[l].pad) == (1, 1 if k == 3 else 0), l


def _expf():
    libm = C.CDLL(ctypes.util.find_library("m"))
    libm.expf.restype = C.c_float
    libm.expf.argtypes = [C.c_float]
    return libm.expf


def _softmax_conf(i0, i1, s, expf):
    """softmax1vector2class (facedetectcnn.cpp:716-728) on the floats convertInt2Float makes of i0, i1"""
    c0, c1 = np.float32(np.float32(i0) * s), np.float32(np.float32(i1) * s)
    vm = c1 if c0 < c1 else c0
    e0, e1 = np.float32(expf(np.float32(c0 - vm))), np.float32(expf(np.float32(c1 - vm)))
    return np.float32(e1 / np.float32(e0 + e1))


def test_prefilter_rule_holds_against_libm_expf():
    expf = _expf()
    rng = np.random.default_rng(5)
    lay = rf.layers(np.load(GOLDEN)["rgb"])
    scales = [np.float32(1.0) / lay["head_scale"][k] for k in (1, 3, 5, 7)]
    scales += [np.float32(x) for x in rng.uniform(1e-7, 10.0, 20)]
    for s in scales:
        i0 = rng.integers(-2 ** 26, 2 ** 26, 400)
        d = rng.integers(0, 3000, 400)
        for a, b in zip(i0, i0 - d):                 # b <= a
            assert not _softmax_conf(a, b, s, expf) > np.float32(0.5)
    # and the rule is tight: i1 = i0 + 1 can pass for a coarse scale
    assert _softmax_conf(0, 1, np.float32(1.0), expf) > np.float32(0.5)
