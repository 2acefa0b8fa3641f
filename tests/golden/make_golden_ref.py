"""Frozen outputs of the reference build (oracle/_ref) on the inputs of the reference-parity tests, so that those tests
need neither the reference tree nor oracle/_ref at run time.  Run where oracle/_ref has been built (oracle/Makefile `ref`):

    python tests/golden/make_golden_ref.py

writes tests/golden/ref_digests.json (oracle.digest of every reference output) and tests/golden/canny_blur_ref.npz (the
reference's Canny blur planes, which the test compares value by value)."""
import json
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path[:0] = [ROOT, os.path.dirname(HERE)]

from oracle import pyoracle as po  # noqa: E402
import harris_cases  # noqa: E402
import test_oracle_contour_lsd as tcl  # noqa: E402
import test_oracle_dlib as tdl  # noqa: E402
import test_oracle_harris_canny as thc  # noqa: E402


def main():
    assert all(po.have_ref(w) for w in ("harris", "canny", "dlib", "otsu", "contour", "lsd")), "build oracle/_ref first"
    d, blur = {}, {}
    for key, img, kw in list(thc.harris_random_cases()) + list(thc.harris_tiny_cases()) + list(harris_cases.reference_cases()):
        d[key] = po.digest(*po.harris_detect(img, impl="ref", **kw))
    for key, img in thc.canny_cases():
        blur[key] = po.canny_blur_ref(img, 2.0).astype(np.float32)
        for acc in (True, False):
            e, nz = po.canny(img, impl="ref", accGrad=acc)
            d["%s_%d" % (key, acc)] = po.digest(e, np.int64(nz))
    for k, img in enumerate(tcl._frames()):
        g = po.contour_gaussian(img, impl="ref")
        d["contour_gauss_%d" % k] = po.digest(g)
        e = po.contour_edge_points(g, impl="ref")
        for name in tcl.EDGE_KEYS:
            d["contour_%s_%d" % (name, k)] = po.digest(e[name])
        s = po.lsd_sampler(img, impl="ref")
        d["lsd_sampler_%d" % k] = po.digest(s)
        a, m, lst = po.lsd_ll_angle(s, impl="ref")
        d["lsd_angle_mod_%d" % k] = po.digest(a, m)
        d["lsd_list_%d" % k] = po.digest(lst)
    for key, im, args in tdl.fhog_cases():
        d[key] = po.digest(po.fhog(im, *args, impl="ref"))
    for key, img, args in tdl.surf_cases():
        r = po.surf(img, *args, impl="ref")
        d[key] = po.digest(*[r[k] for k in tdl.SURF_KEYS])
    for key, x, args in tdl.otsu_cases():
        out, t = po.otsu(x, *args, impl="ref")
        d[key] = po.digest(out, np.int64(t))
    with open(os.path.join(HERE, "ref_digests.json"), "w") as f:
        json.dump(d, f, indent=0, sort_keys=True)
        f.write("\n")
    np.savez_compressed(os.path.join(HERE, "canny_blur_ref.npz"), **blur)


if __name__ == "__main__":
    main()
