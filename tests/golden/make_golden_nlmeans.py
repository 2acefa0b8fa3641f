"""Frozen NL-means outputs of the serial reference build (oracle/_ref/libref_nlmeans.so) on frames too large for a test
to run the CPU reference on (tests/nlmeans_cases.py).  Run where oracle/_ref/libref_nlmeans.so has been built
(make -f oracle/nlmeans.mk) and the reference tree is present (for the garden fixture):

    python tests/golden/make_golden_nlmeans.py

writes tests/golden/nlmeans_garden.npz (the decoded img_garden.png) and tests/golden/nlmeans_digests.json.  The serial
reference takes several minutes on the 1080p frames; the cases run in parallel processes."""
import json
import os
import sys
from multiprocessing import Pool

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path[:0] = [ROOT, os.path.dirname(HERE)]
GARDEN_PNG = "/root/reference/image.DenoiseNLMeans/inst/extdata/img_garden.png"


def _one(case):
    from oracle import pyoracle as po, ref_nlmeans as rn
    import nlmeans_cases as nc
    key, img, sigma = case
    c, h, w = img.shape
    return key, nc.digest_of(po, rn.nlmeans(img.ravel(), w, h, c, sigma))


def main():
    from oracle import ref_nlmeans as rn
    assert rn.have_ref(), "build oracle/_ref/libref_nlmeans.so first (make -f oracle/nlmeans.mk)"
    if os.path.exists(GARDEN_PNG):
        from PIL import Image
        img = np.asarray(Image.open(GARDEN_PNG).convert("RGB"), dtype=np.uint8)
        np.savez_compressed(os.path.join(HERE, "nlmeans_garden.npz"), image=img)
    import nlmeans_cases as nc
    with Pool(min(os.cpu_count() or 1, 5)) as pool:
        d = dict(pool.map(_one, list(nc.digest_cases())))
    with open(os.path.join(HERE, "nlmeans_digests.json"), "w") as f:
        json.dump(d, f, indent=0, sort_keys=True)
        f.write("\n")


if __name__ == "__main__":
    main()
