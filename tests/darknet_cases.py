"""Shared helpers of the darknet tests: random-weight models of the package's cfgs at reduced input sizes, written as
.weights files the reference and image_b200.darknet both read."""
import os

import numpy as np

from image_b200 import darknet as dn


def shrink_cfg(src, dst, width, height):
    """A copy of cfg src with the [net] width and height replaced."""
    out, in_net = [], False
    with open(src) as f:
        for line in f:
            s = "".join(line.split())
            if s.startswith("["):
                in_net = s in ("[net]", "[network]")
            if in_net and s.startswith("width="):
                line = "width=%d\n" % width
            elif in_net and s.startswith("height="):
                line = "height=%d\n" % height
            out.append(line)
    with open(dst, "w") as f:
        f.writelines(out)
    return dst


def random_weights(cfg, dst, seed):
    """A .weights file of random parameters for cfg: He-scaled weights, scales near 1, positive variances, so that the
    activations stay of order 1 through the network.  Returns the parsed net with the arrays."""
    rng = np.random.default_rng(seed)
    net = dn.parse_cfg(cfg)
    for L in net["layers"]:
        if L["type"] != dn.B2F_DN_CONV:
            continue
        n, k = L["filters"], L["c"] * L["size"] * L["size"]
        L["biases"] = rng.normal(0, 0.1, n).astype(np.float32)
        if L["batch_normalize"]:
            L["scales"] = rng.normal(1, 0.1, n).astype(np.float32)
            L["rolling_mean"] = rng.normal(0, 0.1, n).astype(np.float32)
            L["rolling_variance"] = rng.uniform(0.5, 2, n).astype(np.float32)
        L["weights"] = (rng.normal(0, 1, n * k) * np.sqrt(2.0 / k)).astype(np.float32)
    dn.write_weights(dst, net)
    return net


RANDOM_MODELS = (("darknet19.cfg", 96, 96), ("extraction.cfg", 96, 112), ("tiny-yolo.cfg", 160, 128))


def random_model(ref_path, tmpdir, cfg, w, h, seed=5):
    """(cfg path, weights path) of a random-weight copy of the package cfg at w x h."""
    c = shrink_cfg(ref_path(cfg), os.path.join(tmpdir, "%dx%d-%s" % (w, h, cfg)), w, h)
    wt = os.path.join(tmpdir, "%dx%d-%s.weights" % (w, h, cfg))
    random_weights(c, wt, seed)
    return c, wt
