"""darknet on the CPU: the Python cfg / .weights reader against the reference's parser, the reference driver against its
own full detect and classify paths and the frozen golden values, and a numpy emulation of the exact-order convolution
that pins the argument for skipping padded taps (DESIGN.md §5)."""
import json
import os

import numpy as np
import pytest

from image_b200 import darknet as dn
from oracle import ref_darknet as rd
from darknet_cases import RANDOM_MODELS, random_model

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
pytestmark = pytest.mark.skipif(not rd.have_ref(), reason="reference build oracle/_ref/libref_darknet.so absent")
GPU_TYPES = {dn.B2F_DN_CONV: rd.CONVOLUTIONAL, dn.B2F_DN_MAXPOOL: rd.MAXPOOL, dn.B2F_DN_AVGPOOL: rd.AVGPOOL,
             dn.B2F_DN_SOFTMAX: rd.SOFTMAX, dn.B2F_DN_REGION: rd.REGION, dn.B2F_DN_COST: rd.COST}


def check_reader(cfg, weights):
    net = dn.parse_cfg(cfg)
    dn.read_weights(weights, net)
    rd.load(cfg, weights)
    info = rd.net_info()
    assert (net["w"], net["h"], len(net["layers"])) == (info["w"], info["h"], info["n"])
    for i, L in enumerate(net["layers"]):
        R = rd.layer_info(i)
        assert GPU_TYPES[L["type"]] == R["type"], i
        keys = {dn.B2F_DN_CONV: ("c", "h", "w", "out_c", "out_h", "out_w", "size", "stride", "pad", "batch_normalize"),
                dn.B2F_DN_MAXPOOL: ("c", "h", "w", "out_c", "out_h", "out_w", "size", "stride", "pad"),
                dn.B2F_DN_AVGPOOL: ("c", "h", "w"), dn.B2F_DN_REGION: ("h", "w", "n", "classes", "coords", "softmax")}
        for k in keys.get(L["type"], ()):
            assert L["num" if k == "n" else k] == R[k], (i, k)
        if L["type"] == dn.B2F_DN_CONV:
            assert R["activation"] == (7 if L["activation"] == 1 else 3), i        # darknet's LEAKY / LINEAR
        for k, v in rd.params(i).items():
            assert np.array_equal(v, L[k]), (i, k)
    return net


@pytest.mark.parametrize("cfg,weights", [("tiny-yolo-voc.cfg", "tiny-yolo-voc.weights"), ("tiny.cfg", "tiny.weights")])
def test_reader_matches_the_reference_parser(cfg, weights):
    check_reader(rd.path(cfg), rd.path(weights))


@pytest.mark.parametrize("cfg,w,h", RANDOM_MODELS)
def test_random_weight_models_load_run_and_round_trip(tmp_path, cfg, w, h):
    c, wt = random_model(rd.path, str(tmp_path), cfg, w, h)
    net = check_reader(c, wt)
    again = os.path.join(str(tmp_path), "again.weights")
    dn.write_weights(again, net)
    with open(wt, "rb") as a, open(again, "rb") as b:
        assert a.read() == b.read()
    frame = np.random.default_rng(1).integers(0, 256, (h + 7, w - 5, 3), dtype=np.uint8)
    outs = rd.forward(frame, 0)
    assert all(np.isfinite(o).all() for o in outs)
    last = max(i for i in range(len(outs)) if rd.layer_info(i)["type"] != rd.COST)
    assert outs[last].std() > 0


def test_short_weights_file_is_refused(tmp_path):
    raw = open(rd.path("tiny.weights"), "rb").read()
    p = os.path.join(str(tmp_path), "short.weights")
    open(p, "wb").write(raw[:-4])
    with pytest.raises(ValueError, match="end inside"):
        dn.read_weights(p, dn.parse_cfg(rd.path("tiny.cfg")))


def test_unsupported_layers_are_kept_by_name():
    net = dn.parse_cfg(rd.path("yolo-voc.cfg"))
    names = {L["name"] for L in net["layers"] if L["type"] == dn.B2F_DN_OTHER}
    assert names == {"route", "reorg"}


def test_driver_detect_matches_the_layers_and_the_golden_values():
    golden = json.load(open(os.path.join(ROOT, "tests", "golden", "darknet_golden.json")))
    for name in rd.IMAGES:
        im = rd.decode(name)
        g = golden[name]
        assert list(im.shape) == g["shape"]
        rd.load(rd.path("tiny-yolo-voc.cfg"), rd.path("tiny-yolo-voc.weights"))
        d = rd.detect(im)
        nz = np.argwhere(d["probs"] != 0)
        assert d["count"] == g["count"] and nz.tolist() == g["nonzero"]
        assert ["%x" % v for v in d["probs"][nz[:, 0], nz[:, 1]].view(np.uint32)] == g["probs"]
        assert ["%x" % v for v in np.ascontiguousarray(d["boxes"][nz[:, 0]]).ravel().view(np.uint32)] == g["boxes"]
        rd.load(rd.path("tiny.cfg"), rd.path("tiny.weights"))
        for rs in (True, False):
            c = rd.classify(im, rs, 5)
            assert c["index"].tolist() == g["top5_resize%d" % rs]
            assert ["%x" % v for v in c["probability"].view(np.uint64)] == g["prob5_resize%d" % rs]
            # network_predict's output is the softmax layer's
            outs = rd.forward(im, 1 if rs else 2)
            assert np.array_equal(outs[-2], c["predictions"])


def test_dog_finds_the_car_and_the_dog():
    rd.load(rd.path("tiny-yolo-voc.cfg"), rd.path("tiny-yolo-voc.weights"))
    d = rd.detect(rd.decode("dog.jpg"))
    labels = open(rd.path("voc.names")).read().split()
    found = {labels[c]: round(float(d["probs"][i, c]), 3) for i, c in np.argwhere(d["probs"][:, :20] > 0.3)}
    assert found == {"car": 0.758, "dog": 0.785}


def emulate_conv(x, L, skip_padded):
    """forward_convolutional_layer in numpy float32: every output a sequential sum over k = (c, ky, kx) from +0 with the
    product and the add rounded separately, then normalize_cpu in double, scale_bias, add_bias, leaky in double.  With
    skip_padded the taps outside the frame are left out instead of added as w * 0."""
    c, h, w = x.shape
    s, st, p, n = L["size"], L["stride"], L["pad"], L["filters"]
    oh, ow = (h + 2 * p - s) // st + 1, (w + 2 * p - s) // st + 1
    xp = np.zeros((c, h + 2 * p, w + 2 * p), np.float32)
    xp[:, p:p + h, p:p + w] = x
    inside = np.zeros((h + 2 * p, w + 2 * p), bool)
    inside[p:p + h, p:p + w] = True
    W = L["weights"].reshape(n, c, s, s)
    acc = np.zeros((n, oh, ow), np.float32)
    for ci in range(c):
        for ky in range(s):
            for kx in range(s):
                col = xp[ci, ky:ky + st * oh:st, kx:kx + st * ow:st]
                prod = W[:, ci, ky, kx][:, None, None] * col[None]
                if skip_padded:
                    m = inside[ky:ky + st * oh:st, kx:kx + st * ow:st]
                    acc = np.where(m[None], acc + prod, acc).astype(np.float32)
                else:
                    acc = (acc + prod).astype(np.float32)
    v = acc
    if L["batch_normalize"]:
        den = np.sqrt(L["rolling_variance"].astype(np.float64)) + np.float64(np.float32(1e-6))
        v = ((v - L["rolling_mean"][:, None, None]).astype(np.float64) / den[:, None, None]).astype(np.float32)
        v = (v * L["scales"][:, None, None]).astype(np.float32)
    v = (v + L["biases"][:, None, None]).astype(np.float32)
    if L["activation"] == 1:
        v = np.where(v > 0, v, (0.1 * v.astype(np.float64)).astype(np.float32))
    return v


@pytest.mark.parametrize("skip_padded", [False, True])
def test_exact_order_convolution_emulation_equals_the_reference(skip_padded):
    """Layer 0 of tiny (3x3 pad 1 over the 224-min input) and layer 4 (1x1) bit for bit, with and without the padded taps:
    a padded tap adds w * 0 = +-0 to an accumulator that starts at +0 and so is never -0, which leaves it unchanged."""
    net = dn.parse_cfg(rd.path("tiny.cfg"))
    dn.read_weights(rd.path("tiny.weights"), net)
    rd.load(rd.path("tiny.cfg"), rd.path("tiny.weights"))
    im = rd.decode("eagle.jpg")
    x = rd.network_input(im, 1)
    outs = rd.forward(im, 1)
    y0 = emulate_conv(x, net["layers"][0], skip_padded)
    assert np.array_equal(y0.ravel(), outs[0])
    R = rd.layer_info(3)
    pooled = outs[3].reshape(R["out_c"], R["out_h"], R["out_w"])
    y4 = emulate_conv(pooled, net["layers"][4], skip_padded)
    assert np.array_equal(y4.ravel(), outs[4])
