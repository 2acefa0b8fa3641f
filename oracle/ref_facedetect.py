"""TEST INFRASTRUCTURE — ctypes front-end to the reference build of image.libfacedetection
(oracle/_ref/libref_facedetect.so, made by oracle/facedetect.mk): facedetect_cnn, and the layer driver of
oracle/ref_wrap_facedetect.cpp.  Only tests/, smoke() and tools may import this module; the product package image_b200
never does."""
import ctypes as C
import os
import subprocess

import numpy as np

from . import pyoracle as po

HERE = os.path.dirname(os.path.abspath(__file__))
SO_PATH = os.path.join(HERE, "_ref", "libref_facedetect.so")
HEAD_SIZES = (3, 2, 2, 3)       # prior sizes per head (L16/17 .. L22/23)


def build():
    """(Re)build oracle/_ref/libref_facedetect.so when the reference tree exists."""
    subprocess.check_call(["make", "-s", "-f", os.path.join(HERE, "facedetect.mk")])
    po._cache.pop("ref_facedetect", None)


def have_ref():
    return po.have_ref("facedetect")


def _lib():
    return po.lib("ref_facedetect")


def _rgb(frame):
    a = np.ascontiguousarray(frame, dtype=np.uint8)
    assert a.ndim == 3 and a.shape[2] == 3, "frames are [h, w, 3] u8"
    return a


def facedetect_cnn(frame):
    """facedetect_cnn on an [h, w, 3] u8 frame (step = 3w): int32 [n, 15] as detect_faces reads the result buffer."""
    a = _rgb(frame)
    h, w = a.shape[:2]
    out = np.zeros((256, 15), np.int32)
    n = _lib().ref_facedetect_cnn(a.ctypes.data_as(C.c_void_p), w, h, 3 * w, out.ctypes.data_as(C.c_void_p))
    return out[:n].copy()


def layers(frame):
    """The layer driver on one frame.  Returns dict(nmax int32[16] (-1 = layer did not run), scale float32[16],
    bias int32[16], heads = 8 int32 arrays [h, w, c] (None where the head did not run), head_scale float32[8],
    faces float32 [n, 15] (detection_output's floats), ints int32 [n, 15] (facedetect_cnn's result), n_above, n_nms)."""
    a = _rgb(frame)
    h, w = a.shape[:2]
    lib = _lib()
    n = lib.ref_fd_run(a.ctypes.data_as(C.c_void_p), w, h, 3 * w)
    nmax, bias = np.zeros(16, np.int32), np.zeros(16, np.int32)
    scale = np.zeros(16, np.float32)
    lib.ref_fd_trunk(nmax.ctypes.data_as(C.c_void_p), scale.ctypes.data_as(C.c_void_p), bias.ctypes.data_as(C.c_void_p))
    heads, hs = [], np.zeros(8, np.float32)
    for k in range(8):
        dims = np.zeros(3, np.int32)
        s = C.c_float()
        lib.ref_fd_head(k, dims.ctypes.data_as(C.c_void_p), C.byref(s), None)
        hs[k] = s.value
        if dims.prod() == 0:
            heads.append(None)
            continue
        plane = np.zeros((dims[1], dims[0], dims[2]), np.int32)
        lib.ref_fd_head(k, dims.ctypes.data_as(C.c_void_p), C.byref(s), plane.ctypes.data_as(C.c_void_p))
        heads.append(plane)
    faces, ints = np.zeros((n, 15), np.float32), np.zeros((n, 15), np.int32)
    if n:
        lib.ref_fd_faces(faces.ctypes.data_as(C.c_void_p), ints.ctypes.data_as(C.c_void_p))
    na, nn = C.c_int(), C.c_int()
    lib.ref_fd_counts(C.byref(na), C.byref(nn))
    return dict(nmax=nmax, scale=scale, bias=bias, heads=heads, head_scale=hs, faces=faces, ints=ints,
                n_above=na.value, n_nms=nn.value)


def candidates(lay):
    """The candidate records a head pass must emit, from the driver's head planes: int32 [m, 17] = (prior index in
    concatenation order, conf int 0, conf int 1, 14 loc ints), every prior whose conf ints satisfy i1 > i0, or every prior
    of a head whose 1/scale of the conf plane is not a positive finite float."""
    recs, base = [], 0
    for hd, ns in enumerate(HEAD_SIZES):
        loc, conf = lay["heads"][2 * hd], lay["heads"][2 * hd + 1]
        if loc is None or conf is None:
            return np.zeros((0, 17), np.int32)
        npix = conf.shape[0] * conf.shape[1]
        c = conf.reshape(npix * ns, 2)
        l = loc.reshape(npix * ns, 14)
        with np.errstate(divide="ignore", over="ignore", invalid="ignore"):
            inv = np.float32(1.0) / lay["head_scale"][2 * hd + 1]
        keep = np.ones(npix * ns, bool) if not (np.isfinite(inv) and inv > 0) else c[:, 1] > c[:, 0]
        idx = np.nonzero(keep)[0]
        recs.append(np.concatenate([(base + idx)[:, None].astype(np.int32), c[idx], l[idx]], axis=1))
        base += npix * ns
    return np.concatenate(recs, axis=0).astype(np.int32)
