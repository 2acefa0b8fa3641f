"""TEST INFRASTRUCTURE — ctypes front-end to the reference build of image.darknet (oracle/_ref/libref_darknet.so, made by
oracle/darknet.mk) and the model files it copies into oracle/_ref/darknet/.  The reference holds one network at a time
(load()); every call runs batch 1, as the R glue does.  Only tests/, smoke() and tools may import this module; the
product package image_b200 never does."""
import ctypes as C
import os
import subprocess

import numpy as np

from . import pyoracle as po

HERE = os.path.dirname(os.path.abspath(__file__))
SO_PATH = os.path.join(HERE, "_ref", "libref_darknet.so")
DATA = os.path.join(HERE, "_ref", "darknet")
IMAGES = ("dog.jpg", "eagle.jpg", "giraffe.jpg", "horses.jpg", "person.jpg", "scream.jpg")
# darknet's LAYER_TYPE values (layer.h) of the layers the engine runs
CONVOLUTIONAL, MAXPOOL, SOFTMAX, COST, AVGPOOL, REGION = 0, 3, 4, 9, 11, 21
_loaded = [None]


def build():
    """(Re)build oracle/_ref/libref_darknet.so and the model files when the reference tree exists."""
    subprocess.check_call(["make", "-s", "-f", os.path.join(HERE, "darknet.mk")])
    po._cache.pop("ref_darknet", None)


def have_ref():
    return po.have_ref("darknet") and os.path.exists(os.path.join(DATA, "tiny-yolo-voc.weights"))


def path(name):
    return os.path.join(DATA, name)


def _lib():
    lib = po.lib("ref_darknet")
    lib.ref_dn_detect.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_float, C.c_float, C.c_void_p, C.c_void_p]
    return lib


def load(cfg, weights=None):
    """Parse cfg (a path) and load weights (a path or None) into the reference; no-op when already loaded."""
    key = (cfg, weights, os.path.getmtime(weights) if weights else 0)
    if _loaded[0] != key:
        _lib().ref_dn_load(cfg.encode(), (weights or "").encode())
        _loaded[0] = key


def decode(name):
    """A file decoded by the reference's stbi_load(.., 3): u8 [h, w, 3]."""
    f = name if os.path.isabs(name) else path(name)
    w, h = C.c_int(), C.c_int()
    assert _lib().ref_dn_decode(f.encode(), C.byref(w), C.byref(h), None) == 0, f
    out = np.zeros((h.value, w.value, 3), np.uint8)
    _lib().ref_dn_decode(f.encode(), C.byref(w), C.byref(h), out.ctypes.data_as(C.c_void_p))
    return out


def _rgb(frame):
    a = np.ascontiguousarray(frame, dtype=np.uint8)
    assert a.ndim == 3 and a.shape[2] == 3, "frames are [h, w, 3] u8"
    return a


def net_info():
    info = np.zeros(5, np.int32)
    _lib().ref_dn_net(info.ctypes.data_as(C.c_void_p))
    return dict(n=int(info[0]), w=int(info[1]), h=int(info[2]), c=int(info[3]), outputs=int(info[4]))


def network_input(frame, mode):
    """The planar float input a frame becomes: mode 0 = detect, 1 = classify with resize, 2 = without; [3, h, w]."""
    a = _rgb(frame)
    dims = np.zeros(3, np.int32)
    n = _lib().ref_dn_input(a.ctypes.data_as(C.c_void_p), a.shape[1], a.shape[0], mode, None, dims.ctypes.data_as(C.c_void_p))
    out = np.zeros(n, np.float32)
    _lib().ref_dn_input(a.ctypes.data_as(C.c_void_p), a.shape[1], a.shape[0], mode, out.ctypes.data_as(C.c_void_p),
                        dims.ctypes.data_as(C.c_void_p))
    return out.reshape(dims)


INFO = ("type", "c", "h", "w", "out_c", "out_h", "out_w", "n", "size", "stride", "pad", "batch_normalize", "activation",
        "outputs", "classes", "coords", "softmax", "groups")


def layer_info(i):
    info = np.zeros(len(INFO), np.int32)
    _lib().ref_dn_layer(i, info.ctypes.data_as(C.c_void_p), None)
    return dict(zip(INFO, (int(v) for v in info)))


def forward(frame, mode):
    """network_predict of one frame; returns every layer's output (float32, flat) in layer order."""
    a = _rgb(frame)
    lib = _lib()
    lib.ref_dn_forward(a.ctypes.data_as(C.c_void_p), a.shape[1], a.shape[0], mode)
    outs = []
    for i in range(net_info()["n"]):
        info = np.zeros(len(INFO), np.int32)
        n = lib.ref_dn_layer(i, info.ctypes.data_as(C.c_void_p), None)
        o = np.zeros(n, np.float32)
        lib.ref_dn_layer(i, info.ctypes.data_as(C.c_void_p), o.ctypes.data_as(C.c_void_p))
        outs.append(o)
    return outs


def params(i):
    """The parameter arrays of layer i as load_weights left them."""
    L = layer_info(i)
    if L["type"] == CONVOLUTIONAL:
        n, k = L["n"], L["c"] * L["size"] * L["size"]
        b, s, m, v = (np.zeros(n, np.float32) for _ in range(4))
        w = np.zeros(n * k, np.float32)
        bn = L["batch_normalize"]
        _lib().ref_dn_params(i, b.ctypes.data_as(C.c_void_p), s.ctypes.data_as(C.c_void_p) if bn else None,
                             m.ctypes.data_as(C.c_void_p), v.ctypes.data_as(C.c_void_p), w.ctypes.data_as(C.c_void_p), None)
        return dict(biases=b, weights=w, **(dict(scales=s, rolling_mean=m, rolling_variance=v) if bn else {}))
    if L["type"] == REGION:
        a = np.zeros(2 * L["n"], np.float32)
        _lib().ref_dn_params(i, None, None, None, None, None, a.ctypes.data_as(C.c_void_p))
        return dict(anchors=a)
    return {}


def detect(frame, thresh=0.3, hier_thresh=0.5):
    """darknet_test_detector on one frame: dict(probs [total, classes + 1], boxes [total, 4], count)."""
    a = _rgb(frame)
    L = layer_info(net_info()["n"] - 1)
    total = L["w"] * L["h"] * L["n"]
    probs = np.zeros((total, L["classes"] + 1), np.float32)
    boxes = np.zeros((total, 4), np.float32)
    cnt = _lib().ref_dn_detect(a.ctypes.data_as(C.c_void_p), a.shape[1], a.shape[0], thresh, hier_thresh,
                               probs.ctypes.data_as(C.c_void_p), boxes.ctypes.data_as(C.c_void_p))
    return dict(probs=probs, boxes=boxes, count=cnt)


def classify(frame, resize=True, top=5):
    """darknet_predict_classifier on one frame: dict(index int32 [top], probability float64 [top], predictions)."""
    a = _rgb(frame)
    outputs = net_info()["outputs"]
    idx = np.zeros(top, np.int32)
    sc = np.zeros(top, np.float64)
    pred = np.zeros(outputs, np.float32)
    _lib().ref_dn_classify(a.ctypes.data_as(C.c_void_p), a.shape[1], a.shape[0], int(bool(resize)), top,
                           idx.ctypes.data_as(C.c_void_p), sc.ctypes.data_as(C.c_void_p), pred.ctypes.data_as(C.c_void_p))
    return dict(index=idx, probability=sc, predictions=pred)
