"""darknet on the H100 against the reference build (oracle/_ref/libref_darknet.so), exactly: per-layer outputs, the region
input and output, probs and boxes after NMS, the count above the threshold, and the classifier's top-k, on the package's
images decoded by the reference's stb, synthetic frames of awkward sizes and content, and random-weight models."""
import os

import numpy as np
import pytest
import torch

from image_b200 import _lib
from image_b200 import darknet as dn
from oracle import ref_darknet as rd
from darknet_cases import RANDOM_MODELS, random_model, random_weights

pytestmark = [pytest.mark.gpu, pytest.mark.skipif(not rd.have_ref(), reason="reference build oracle/_ref/libref_darknet.so absent")]


@pytest.fixture(scope="module")
def yolo():
    m = dn.load_network(rd.path("tiny-yolo-voc.cfg"), rd.path("tiny-yolo-voc.weights"))
    yield m
    m.free()


@pytest.fixture(scope="module")
def tiny():
    m = dn.load_network(rd.path("tiny.cfg"), rd.path("tiny.weights"))
    yield m
    m.free()


def dev(frames):
    a = np.ascontiguousarray(frames, dtype=np.uint8)
    if a.ndim == 3:
        a = a[None]
    return torch.from_numpy(a).cuda(), a.shape[0], a.shape[2], a.shape[1]


def check_detect(m, cfg, weights, frame):
    rd.load(cfg, weights)
    want = rd.detect(frame)
    probs, boxes, cnt = dn.detect_batch(frame, m)
    assert np.array_equal(probs[0], want["probs"]) and np.array_equal(boxes[0], want["boxes"]) and cnt[0] == want["count"]
    return want


def check_classify(m, cfg, weights, frame, resize, top=5):
    rd.load(cfg, weights)
    want = rd.classify(frame, resize, top)
    idx, prob = dn.classify_batch(frame, m, resize, top)
    assert np.array_equal(idx[0], want["index"]) and np.array_equal(prob[0], want["probability"])
    return want


def check_layers(m, cfg, weights, frame, mode):
    """Every layer's output (the region / softmax layers as the reference leaves l.output) and the network input."""
    rd.load(cfg, weights)
    outs = rd.forward(frame, mode)
    d, n, w, h = dev(frame)
    assert np.array_equal(dn.layer_dev(d, n, w, h, m, mode, -1)[0], rd.network_input(frame, mode))
    for i, L in enumerate(m.net["layers"]):
        if L["type"] == dn.B2F_DN_COST:
            continue
        got = dn.layer_dev(d, n, w, h, m, mode, i)[0].ravel()
        assert np.array_equal(got, outs[i]), "layer %d (%s) differs" % (i, L["name"])


@pytest.mark.parametrize("name", rd.IMAGES)
def test_detect_package_images(yolo, name):
    im = rd.decode(name)
    check_detect(yolo, rd.path("tiny-yolo-voc.cfg"), rd.path("tiny-yolo-voc.weights"), im)


@pytest.mark.parametrize("name", rd.IMAGES)
def test_classify_package_images(tiny, name):
    im = rd.decode(name)
    for resize in (True, False):
        check_classify(tiny, rd.path("tiny.cfg"), rd.path("tiny.weights"), im, resize)


def test_layers_of_both_models_on_dog(yolo, tiny):
    im = rd.decode("dog.jpg")
    check_layers(yolo, rd.path("tiny-yolo-voc.cfg"), rd.path("tiny-yolo-voc.weights"), im, 0)
    for mode in (1, 2):
        check_layers(tiny, rd.path("tiny.cfg"), rd.path("tiny.weights"), im, mode)


def synthetic(shape, seed):
    return np.random.default_rng(seed).integers(0, 256, shape, dtype=np.uint8)


SIZES = [(1, 37), (41, 1), (2, 3), (416, 416), (224, 224), (900, 120), (130, 700), (2160, 3840)]


@pytest.mark.parametrize("h,w", SIZES)
def test_synthetic_sizes(yolo, tiny, h, w):
    f = synthetic((h, w, 3), h * 7 + w)
    check_detect(yolo, rd.path("tiny-yolo-voc.cfg"), rd.path("tiny-yolo-voc.weights"), f)
    for resize in (True, False):
        check_classify(tiny, rd.path("tiny.cfg"), rd.path("tiny.weights"), f, resize)


def test_224_frame_is_its_own_resize_min(tiny):
    f = synthetic((224, 300, 3), 3)
    check_layers(tiny, rd.path("tiny.cfg"), rd.path("tiny.weights"), f, 1)


@pytest.mark.parametrize("value", [0, 128, 255])
def test_constant_frames(yolo, tiny, value):
    f = np.full((120, 160, 3), value, np.uint8)
    check_detect(yolo, rd.path("tiny-yolo-voc.cfg"), rd.path("tiny-yolo-voc.weights"), f)
    check_classify(tiny, rd.path("tiny.cfg"), rd.path("tiny.weights"), f, True)


def test_batch_dev_and_single_agree_across_chunks(yolo, tiny):
    """Frames of different content in one batch; the host batch cuts them into chunks (2 GB of scratch each), the device
    form runs them in one pass, and each agrees with the single-frame form and the reference."""
    rng = np.random.default_rng(11)
    h, w = 48, 64
    n = 100
    frames = rng.integers(0, 256, (n, h, w, 3), dtype=np.uint8)
    frames[3] = 0
    frames[7] = rd.decode("dog.jpg")[:h, :w]
    probs, boxes, cnt = dn.detect_batch(frames, yolo)
    d, _, _, _ = dev(frames)
    p2, b2, c2 = dn.detect_dev(d, n, w, h, yolo)
    assert np.array_equal(probs, p2) and np.array_equal(boxes, b2) and np.array_equal(cnt, c2)
    for i in (0, 3, 7, 88, n - 1):
        p1, b1, c1 = dn.detect_batch(frames[i], yolo)
        assert np.array_equal(p1[0], probs[i]) and np.array_equal(b1[0], boxes[i]) and c1[0] == cnt[i]
    for i in (3, 7, n - 1):
        rd.load(rd.path("tiny-yolo-voc.cfg"), rd.path("tiny-yolo-voc.weights"))
        want = rd.detect(frames[i])
        assert np.array_equal(probs[i], want["probs"]) and np.array_equal(boxes[i], want["boxes"]) and cnt[i] == want["count"]
    idx, prob = dn.classify_batch(frames, tiny, True, 5)
    i2, q2 = dn.classify_dev(d, n, w, h, tiny, True, 5)
    assert np.array_equal(idx, i2) and np.array_equal(prob, q2)
    for i in (0, 7, n - 1):
        rd.load(rd.path("tiny.cfg"), rd.path("tiny.weights"))
        want = rd.classify(frames[i], True, 5)
        assert np.array_equal(idx[i], want["index"]) and np.array_equal(prob[i], want["probability"])


@pytest.mark.parametrize("cfg,w,h", RANDOM_MODELS)
def test_random_weight_models(tmp_path, cfg, w, h):
    c, wt = random_model(rd.path, str(tmp_path), cfg, w, h)
    m = dn.load_network(c, wt)
    try:
        for seed, shape in ((1, (h + 7, w - 5, 3)), (2, (h // 2, w * 2, 3))):
            f = synthetic(shape, seed)
            if m.boxes:
                check_detect(m, c, wt, f)
                check_layers(m, c, wt, f, 0)
            else:
                check_classify(m, c, wt, f, True, 7)
                check_layers(m, c, wt, f, 1)
    finally:
        m.free()


def test_bad_arguments(tmp_path, yolo, tiny):
    yv = random_weights(rd.path("yolo-voc.cfg"), os.path.join(str(tmp_path), "yolo-voc.weights"), 3)
    with pytest.raises(_lib.B2FError, match="route") as e:
        dn.DarknetModel(yv)
    assert e.value.code == _lib.B2F_EINVAL
    net = dn.parse_cfg(rd.path("tiny.cfg"))
    dn.read_weights(rd.path("tiny.weights"), net)
    net["layers"][2]["weights"] = net["layers"][2]["weights"][:-1]
    with pytest.raises(_lib.B2FError, match="weights hold") as e:
        dn.DarknetModel(net)
    assert e.value.code == _lib.B2F_EINVAL
    f = synthetic((50, 60, 3), 4)
    for top in (0, -1, 1001):
        with pytest.raises(_lib.B2FError, match="top") as e:
            dn.classify_batch(f, tiny, True, top) if top > 0 else dn.classify_dev(*dev(f), tiny, True, top)
        assert e.value.code == _lib.B2F_EINVAL
    lib = _lib.load()
    probs = np.zeros((1, yolo.boxes, yolo.classes + 1), np.float32)
    boxes = np.zeros((1, yolo.boxes, 4), np.float32)
    cnt = np.zeros(1, np.int32)
    for n, w, h in ((0, 60, 50), (1, 0, 50), (1, 60, -1)):
        rc = lib.b2f_darknet_detect_batch_rgb(yolo.ctx, yolo.handle, _lib.ptr(f), n, w, h, 0.3, 0.5, _lib.ptr(probs),
                                              _lib.ptr(boxes), _lib.ptr(cnt))
        assert rc == _lib.B2F_EINVAL
    with pytest.raises(_lib.B2FError):
        dn.detect_batch(f, tiny)                     # no region layer
    with pytest.raises(_lib.B2FError):
        dn.classify_batch(f, yolo)                   # a detector
