"""Host-side mirror of image.darknet: image_darknet_model, image_darknet_detect and image_darknet_classify (R/*.R) over the
C ABI of include/b2f.h (b2f_darknet_*).  The cfg INI parser and the .weights reader here follow darknet's file formats
(parser.c): the engine itself only sees the parsed layers.  Frames are decoded RGB arrays [h, w, 3] u8; the product has no
image decoder.  No CPU path."""
import ctypes as C
import os

import numpy as np

from . import _lib

B2F_DN_OTHER, B2F_DN_CONV, B2F_DN_MAXPOOL, B2F_DN_AVGPOOL, B2F_DN_SOFTMAX, B2F_DN_REGION, B2F_DN_COST = range(7)
_SECTIONS = {"[conv]": B2F_DN_CONV, "[convolutional]": B2F_DN_CONV, "[max]": B2F_DN_MAXPOOL, "[maxpool]": B2F_DN_MAXPOOL,
             "[avg]": B2F_DN_AVGPOOL, "[avgpool]": B2F_DN_AVGPOOL, "[soft]": B2F_DN_SOFTMAX, "[softmax]": B2F_DN_SOFTMAX,
             "[region]": B2F_DN_REGION, "[cost]": B2F_DN_COST}
_ACT = {"linear": 0, "leaky": 1}
PRESETS = ("tiny.cfg", "alexnet.cfg", "darknet.cfg", "vgg-16.cfg", "extraction.cfg", "darknet19.cfg", "darknet19_448.cfg",
           "yolo.cfg", "tiny-yolo.cfg", "yolo-voc", "tiny-yolo-voc.cfg")


class DarknetLayer(C.Structure):
    """b2f_darknet_layer."""
    _fields_ = [("type", C.c_int), ("name", C.c_char_p), ("filters", C.c_int), ("size", C.c_int), ("stride", C.c_int),
                ("pad", C.c_int), ("batch_normalize", C.c_int), ("activation", C.c_int), ("groups", C.c_int),
                ("temperature", C.c_float), ("classes", C.c_int), ("coords", C.c_int), ("num", C.c_int),
                ("softmax", C.c_int), ("tree", C.c_int), ("biases", C.c_void_p), ("scales", C.c_void_p),
                ("rolling_mean", C.c_void_p), ("rolling_variance", C.c_void_p), ("weights", C.c_void_p),
                ("n_weights", C.c_size_t), ("anchors", C.c_void_p)]


def read_cfg(path):
    """darknet's read_cfg: [(section, {key: value})], every whitespace character removed from each line, lines starting
    with '#', ';' or nothing skipped."""
    sections = []
    with open(path, "r", errors="replace") as f:
        for line in f:
            s = "".join(line.split())
            if not s or s[0] in "#;":
                continue
            if s[0] == "[":
                sections.append((s, {}))
            elif "=" in s and sections:
                k, v = s.split("=", 1)
                sections[-1][1][k] = v
    return sections


def _int(opts, k, d):
    return int(_atof(opts[k])) if k in opts else d


def _atof(v):
    """C atof/atoi on the leading number of v (0 when there is none)."""
    import re
    m = re.match(r"[+-]?(\d+\.?\d*([eE][+-]?\d+)?|\.\d+([eE][+-]?\d+)?)", v)
    return float(m.group(0)) if m else 0.0


def _float(opts, k, d):
    return _atof(opts[k]) if k in opts else d


def parse_cfg(path):
    """The network of a cfg file: dict(w, h, c, layers), each layer a dict with darknet's geometry (c, h, w, out_c, out_h,
    out_w at the cfg size) and options.  Sections the engine does not run keep type B2F_DN_OTHER and their name."""
    secs = read_cfg(path)
    if not secs or secs[0][0] not in ("[net]", "[network]"):
        raise ValueError("%s: the first section must be [net] or [network]" % path)
    net = secs[0][1]
    w, h, c = _int(net, "width", 0), _int(net, "height", 0), _int(net, "channels", 0)
    adam = _int(net, "adam", 0)
    layers = []
    for name, o in secs[1:]:
        t = _SECTIONS.get(name, B2F_DN_OTHER)
        L = dict(type=t, name=name.strip("[]"), c=c, h=h, w=w)
        oc, oh, ow = c, h, w
        if t == B2F_DN_CONV:
            size, stride = _int(o, "size", 1), _int(o, "stride", 1)
            pad = size // 2 if _int(o, "pad", 0) else _int(o, "padding", 0)
            act = o.get("activation", "logistic")
            L.update(filters=_int(o, "filters", 1), size=size, stride=stride, pad=pad,
                     batch_normalize=_int(o, "batch_normalize", 0), activation=_ACT.get(act, 2), activation_name=act)
            if _int(o, "binary", 0) or _int(o, "xnor", 0) or _int(o, "flipped", 0) or adam:
                L["activation"] = 2                    # binary, xnor, flipped and adam layers are not run by the engine
            L["skips_weights"] = bool(_int(o, "dontload", 0) or _int(o, "dontloadscales", 0))
            oc = L["filters"]
            oh = (h + 2 * pad - size) // stride + 1 if stride else 0
            ow = (w + 2 * pad - size) // stride + 1 if stride else 0
        elif t == B2F_DN_MAXPOOL:
            stride = _int(o, "stride", 1)
            size = _int(o, "size", stride)
            pad = _int(o, "padding", (size - 1) // 2)
            L.update(size=size, stride=stride, pad=pad)
            oh, ow = ((h + 2 * pad) // stride, (w + 2 * pad) // stride) if stride else (0, 0)
        elif t == B2F_DN_AVGPOOL:
            oh = ow = 1
        elif t == B2F_DN_SOFTMAX:
            L.update(groups=_int(o, "groups", 1), temperature=_float(o, "temperature", 1.0), tree=int("tree" in o))
        elif t == B2F_DN_REGION:
            L.update(coords=_int(o, "coords", 4), classes=_int(o, "classes", 20), num=_int(o, "num", 1),
                     softmax=_int(o, "softmax", 0), tree=int("tree" in o))
            anchors = np.full(2 * L["num"], 0.5, np.float32)
            if "anchors" in o:
                vals = [np.float32(_atof(v)) for v in o["anchors"].split(",")]
                anchors[:len(vals)] = vals[:2 * L["num"]]
            L["anchors"] = anchors
        L.update(out_c=oc, out_h=oh, out_w=ow)
        layers.append(L)
        c, h, w = oc, oh, ow
    return dict(w=_int(net, "width", 0), h=_int(net, "height", 0), c=_int(net, "channels", 0), layers=layers)


def read_weights(path, net):
    """darknet's load_weights on the parsed net: a header of four int32 (major, minor, revision, seen), then per
    convolutional layer biases, [scales, rolling_mean, rolling_variance when batch_normalize], weights.  Fills the
    arrays into net's layers and returns the header; a file too short for the layers raises ValueError."""
    raw = np.fromfile(path, np.uint8)
    if raw.size < 16:
        raise ValueError("%s: %d bytes, shorter than the header" % (path, raw.size))
    header = raw[:16].view(np.int32).copy()
    data = raw[16:16 + (raw.size - 16) // 4 * 4].view(np.float32)
    off = 0

    def take(n, what, i):
        nonlocal off
        if off + n > data.size:
            raise ValueError("%s: the weights end inside the %s of layer %d" % (path, what, i))
        a = data[off:off + n].copy()
        off += n
        return a

    for i, L in enumerate(net["layers"]):
        if L["type"] != B2F_DN_CONV:
            continue
        if L.get("skips_weights"):
            # load_weights would leave this layer's (or its batch-norm) parameters at their random initial values
            raise ValueError("%s: layer %d sets dontload or dontloadscales, which this reader does not support" % (path, i))
        n = L["filters"]
        L["biases"] = take(n, "biases", i)
        if L["batch_normalize"]:
            L["scales"] = take(n, "scales", i)
            L["rolling_mean"] = take(n, "rolling_mean", i)
            L["rolling_variance"] = take(n, "rolling_variance", i)
        L["weights"] = take(n * L["c"] * L["size"] * L["size"], "weights", i)
    return dict(major=int(header[0]), minor=int(header[1]), revision=int(header[2]), seen=int(header[3]))


def write_weights(path, net, header=(0, 1, 0, 0)):
    """The inverse of read_weights (for tests that make random-weight models)."""
    with open(path, "wb") as f:
        f.write(np.asarray(header, np.int32).tobytes())
        for L in net["layers"]:
            if L["type"] != B2F_DN_CONV:
                continue
            for k in ("biases", "scales", "rolling_mean", "rolling_variance", "weights") if L["batch_normalize"] else ("biases", "weights"):
                f.write(np.ascontiguousarray(L[k], np.float32).tobytes())


class DarknetModel:
    """A b2f_darknet_model: the parsed network with its weights on the device of `ctx`.  free() releases it."""

    def __init__(self, net, ctx=None):
        self.net = net
        self.ctx = ctx or _lib.context()
        n = len(net["layers"])
        tab = (DarknetLayer * n)()
        self._keep = []
        for i, L in enumerate(net["layers"]):
            d = tab[i]
            d.type = L["type"]
            d.name = L["name"].encode()
            for k in ("filters", "size", "stride", "pad", "batch_normalize", "activation", "groups", "classes", "coords",
                      "num", "softmax", "tree"):
                setattr(d, k, int(L.get(k, 0)))
            d.temperature = float(L.get("temperature", 1.0))
            for k in ("biases", "scales", "rolling_mean", "rolling_variance", "weights", "anchors"):
                if L.get(k) is not None:
                    a = np.ascontiguousarray(L[k], np.float32)
                    self._keep.append(a)
                    setattr(d, k, a.ctypes.data)
            d.n_weights = L["weights"].size if L.get("weights") is not None else 0
        self.handle = C.c_void_p()
        _lib.check(_lib.load().b2f_darknet_model_create(self.ctx, C.cast(tab, C.c_void_p), n, int(net["w"]), int(net["h"]),
                                                        C.byref(self.handle)))
        dims = np.zeros(3, np.int32)
        _lib.check(_lib.load().b2f_darknet_model_dims(self.handle, _lib.ptr(dims)))
        self.boxes, self.classes, self.outputs = (int(v) for v in dims)

    def free(self):
        if self.handle:
            _lib.load().b2f_darknet_model_free(self.handle)
            self.handle = C.c_void_p()


def load_network(cfg, weights, ctx=None):
    """A DarknetModel of a cfg file and a .weights file."""
    net = parse_cfg(cfg)
    if net["c"] != 3:
        raise ValueError("%s: %d channels; the engine runs RGB networks" % (cfg, net["c"]))
    read_weights(weights, net)
    return DarknetModel(net, ctx)


def image_darknet_model(type="classify", model=None, weights=None, labels=None, resize=True, cfg_dir=None, ctx=None):
    """image_darknet_model with R's argument rules.  A preset name (tiny.cfg, ...) is looked up in cfg_dir (the R package's
    include/darknet/cfg).  labels: a list of labels, or one path to a file of them."""
    if type not in ("classify", "detect"):
        raise ValueError("type must be 'classify' or 'detect'")
    if model in PRESETS and cfg_dir is not None:
        model = os.path.join(cfg_dir, model)
    if not (model and os.path.exists(model)):
        raise ValueError("file.exists(model) is not TRUE")
    if not (weights and os.path.exists(weights)):
        raise ValueError("file.exists(weights) is not TRUE")
    if isinstance(labels, str):
        labels = [labels]
    if labels is None or not all(isinstance(v, str) for v in labels):
        raise ValueError("is.character(labels) is not TRUE")
    if len(labels) == 1:
        if not os.path.exists(labels[0]):
            raise ValueError("file.exists(labels) is not TRUE")
        with open(labels[0]) as f:
            labels = f.read().splitlines()
        if len(labels) <= 1:
            raise ValueError("length(labels) > 1 is not TRUE")
    out = dict(type=type, cfgfile=model, weightfile=weights, labels=list(labels), network=load_network(model, weights, ctx))
    if type == "classify":
        out["resize"] = bool(resize)
    return out


def _frames(frames):
    a = np.ascontiguousarray(frames, dtype=np.uint8)
    if a.ndim == 3:
        a = a[None]
    if a.ndim != 4 or a.shape[3] != 3:
        raise ValueError("frames must be [h, w, 3] or [n, h, w, 3] u8")
    return a


def detect_batch(frames, net, threshold=0.3, hier_threshold=0.5):
    """b2f_darknet_detect_batch_rgb on host frames [n, h, w, 3]: (probs [n, boxes, classes + 1], boxes [n, boxes, 4],
    count [n])."""
    a = _frames(frames)
    n, h, w = a.shape[:3]
    probs = np.zeros((n, net.boxes, net.classes + 1), np.float32)
    boxes = np.zeros((n, net.boxes, 4), np.float32)
    cnt = np.zeros(n, np.int32)
    _lib.check(_lib.load().b2f_darknet_detect_batch_rgb(net.ctx, net.handle, _lib.ptr(a), n, w, h, float(threshold),
                                                        float(hier_threshold), _lib.ptr(probs), _lib.ptr(boxes), _lib.ptr(cnt)))
    return probs, boxes, cnt


def detect_dev(d_frames, n_frames, width, height, net, threshold=0.3, hier_threshold=0.5, stream=None):
    """b2f_darknet_detect_dev on u8 frames [n, h, w, 3] on the device (a pointer or a tensor)."""
    n = int(n_frames)
    probs = np.zeros((n, net.boxes, net.classes + 1), np.float32)
    boxes = np.zeros((n, net.boxes, 4), np.float32)
    cnt = np.zeros(n, np.int32)
    _lib.check(_lib.load().b2f_darknet_detect_dev(net.ctx, net.handle, _lib.ptr(d_frames), n, int(width), int(height),
                                                  float(threshold), float(hier_threshold), _lib.ptr(probs), _lib.ptr(boxes),
                                                  _lib.ptr(cnt), C.c_void_p(stream) if stream is not None else None))
    return probs, boxes, cnt


def classify_batch(frames, net, resize=True, top=5):
    """b2f_darknet_classify_batch_rgb on host frames [n, h, w, 3]: (index int32 [n, top], prob float64 [n, top])."""
    a = _frames(frames)
    n, h, w = a.shape[:3]
    idx = np.zeros((n, max(int(top), 0)), np.int32)
    prob = np.zeros((n, max(int(top), 0)), np.float64)
    _lib.check(_lib.load().b2f_darknet_classify_batch_rgb(net.ctx, net.handle, _lib.ptr(a), n, w, h, int(bool(resize)), int(top),
                                                          _lib.ptr(idx), _lib.ptr(prob)))
    return idx, prob


def classify_dev(d_frames, n_frames, width, height, net, resize=True, top=5, stream=None):
    """b2f_darknet_classify_dev on u8 frames [n, h, w, 3] on the device."""
    n = int(n_frames)
    idx = np.zeros((n, max(int(top), 0)), np.int32)
    prob = np.zeros((n, max(int(top), 0)), np.float64)
    _lib.check(_lib.load().b2f_darknet_classify_dev(net.ctx, net.handle, _lib.ptr(d_frames), n, int(width), int(height),
                                                    int(bool(resize)), int(top), _lib.ptr(idx), _lib.ptr(prob),
                                                    C.c_void_p(stream) if stream is not None else None))
    return idx, prob


def layer_dev(d_frames, n_frames, width, height, net, mode, layer, stream=None):
    """b2f_darknet_layer_dev: the output of `layer` (-1 = the network input) as float32 [n, c, h, w]; mode 0 = detect,
    1 = classify with resize, 2 = classify without."""
    n = int(n_frames)
    dims = np.zeros(3, np.int32)
    lib = _lib.load()
    st = C.c_void_p(stream) if stream is not None else None
    _lib.check(lib.b2f_darknet_layer_dev(net.ctx, net.handle, _lib.ptr(d_frames), n, int(width), int(height), int(mode), int(layer),
                                         None, 0, _lib.ptr(dims), st))
    out = np.zeros((n,) + tuple(int(v) for v in dims), np.float32)
    _lib.check(lib.b2f_darknet_layer_dev(net.ctx, net.handle, _lib.ptr(d_frames), n, int(width), int(height), int(mode), int(layer),
                                         _lib.ptr(out), out.size, _lib.ptr(dims), st))
    return out


def _detections(probs, boxes, labels, threshold):
    """draw_detections' choice per box: its best class when that probability is above the threshold."""
    rows = []
    for i in range(probs.shape[0]):
        cls = _max_index(probs[i, :-1])
        p = probs[i, cls]
        if p > np.float32(threshold):
            rows.append(dict(label=labels[cls] if cls < len(labels) else str(cls), probability=float(p),
                             x=float(boxes[i, 0]), y=float(boxes[i, 1]), w=float(boxes[i, 2]), h=float(boxes[i, 3])))
    return rows


def _max_index(a):
    """utils.c max_index: the first maximum under '>'."""
    mi, mx = 0, a[0]
    for j in range(1, a.size):
        if a[j] > mx:
            mi, mx = j, a[j]
    return mi


def image_darknet_detect(frame, object, threshold=0.3, hier_threshold=0.5):
    """image_darknet_detect on a decoded frame [h, w, 3] u8: dict(detections = [(label, probability, box)], count, probs,
    boxes) — the boxes draw_detections prints and the reference's arrays after NMS."""
    if object["type"] != "detect":
        raise ValueError("object$type == \"detect\" is not TRUE")
    probs, boxes, cnt = detect_batch(frame, object["network"], threshold, hier_threshold)
    return dict(detections=_detections(probs[0], boxes[0], object["labels"], threshold), count=int(cnt[0]),
                probs=probs[0], boxes=boxes[0])


def image_darknet_classify(frame, object, top=5):
    """image_darknet_classify on a decoded frame [h, w, 3] u8: dict(type = dict(label, probability)), the columns of R's
    data.frame."""
    if object["type"] != "classify":
        raise ValueError("object$type == \"classify\" is not TRUE")
    idx, prob = classify_batch(frame, object["network"], object["resize"], int(top))
    labels = object["labels"]
    return dict(type=dict(label=[labels[i] for i in idx[0]], probability=prob[0]), index=idx[0])
