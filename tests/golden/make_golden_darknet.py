"""Freezes the reference build's darknet outputs on the package's sample images into tests/golden/darknet_golden.json:
per image the tiny-yolo-voc detection count, the non-zero probabilities after NMS (box index, class, value) with their
boxes, and the tiny classifier's top 5 with resize TRUE and FALSE.  Values are stored as the hex of their float32 /
float64 bits.  Run from the repository root after `python __graft_entry__.py build`:
    python tests/golden/make_golden_darknet.py"""
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from oracle import ref_darknet as rd  # noqa: E402


def bits(a):
    a = np.ascontiguousarray(a)
    return ["%x" % v for v in a.ravel().view(np.uint32 if a.dtype == np.float32 else np.uint64)]


def golden():
    out = {}
    for name in rd.IMAGES:
        im = rd.decode(name)
        rd.load(rd.path("tiny-yolo-voc.cfg"), rd.path("tiny-yolo-voc.weights"))
        d = rd.detect(im)
        nz = np.argwhere(d["probs"] != 0)
        g = dict(shape=list(im.shape), count=int(d["count"]), nonzero=nz.tolist(),
                 probs=bits(d["probs"][nz[:, 0], nz[:, 1]]), boxes=bits(d["boxes"][nz[:, 0]]))
        rd.load(rd.path("tiny.cfg"), rd.path("tiny.weights"))
        for rs in (True, False):
            c = rd.classify(im, rs, 5)
            g["top5_resize%d" % rs] = c["index"].tolist()
            g["prob5_resize%d" % rs] = bits(c["probability"])
        out[name] = g
    return out


if __name__ == "__main__":
    with open(os.path.join(ROOT, "tests", "golden", "darknet_golden.json"), "w") as f:
        json.dump(golden(), f, indent=1, sort_keys=True)
