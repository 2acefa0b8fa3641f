"""TEST INFRASTRUCTURE — ctypes front-end to the serial reference build of image.DenoiseNLMeans
(oracle/_ref/libref_nlmeans.so, made by oracle/nlmeans.mk).  There is no C restatement of NL-means: the reference build is
the authority, and tests/golden/nlmeans_digests.json freezes its output on the large frames.  Only tests/, smoke() and
tools may import this module; the product package image_b200 never does."""
import ctypes as C
import os
import subprocess

import numpy as np

from . import pyoracle as po

HERE = os.path.dirname(os.path.abspath(__file__))


def build():
    """(Re)build oracle/_ref/libref_nlmeans.so when the reference tree exists."""
    subprocess.check_call(["make", "-s", "-f", os.path.join(HERE, "nlmeans.mk")])
    po._cache.pop("ref_nlmeans", None)


def have_ref():
    return po.have_ref("nlmeans")


def nlmeans(image, width, height, channels, sigma, args_auto=True, win=1, bloc=10, filter=0.4):
    """rcpp_nlmeans of image.DenoiseNLMeans, serial build.  image = the width*height*channels R integers, channel-planar.
    Returns the glue's list as a dict; raises ValueError with the Rcpp::stop message."""
    v = np.ascontiguousarray(np.asarray(image).ravel(), dtype=np.int32)
    if v.size != int(width) * int(height) * int(channels):
        raise ValueError("image must hold width * height * channels values")
    out = np.zeros(max(int(width) * int(height) * min(max(int(channels), 1), 3), 1), np.float64)
    oc, w, b = C.c_int(0), C.c_int(0), C.c_int(0)
    f, s = C.c_float(0), C.c_float(0)
    err = C.create_string_buffer(512)
    fn = po.lib("ref_nlmeans").ref_nlmeans
    fn.restype = C.c_int
    rc = fn(v.ctypes.data_as(C.c_void_p), int(width), int(height), int(channels), C.c_float(sigma), int(bool(args_auto)),
            int(win), int(bloc), C.c_float(filter), out.ctypes.data_as(C.c_void_p), C.byref(oc), C.byref(w), C.byref(b),
            C.byref(f), C.byref(s), err, 512)
    if rc != 0:
        raise ValueError(err.value.decode())
    n = int(width) * int(height) * oc.value
    return dict(width=int(width), height=int(height), channels=oc.value, denoised=out[:n].copy(), sigma=s.value,
                filter=f.value, window=w.value, bloc=b.value)
