"""Host-side mirror of image.CannyEdges::image_canny_edge_detector
(reference: image.CannyEdges/R/canny_edges_detector.R:63-67) over the C ABI."""
import ctypes as C

import numpy as np

from . import _lib


class CannyResult(dict):
    """list(edges, pixels_nonzero, nx, ny, s, low_thr, high_thr, accGrad), class 'image_canny'
    (rcpp_canny.cpp:236-244; print method R/canny_edges_detector.R:71-79)."""

    def __repr__(self):
        return ("Canny edge detector\n  %s x %s matrix\n  number of pixels on edge %s\n  sigma %s\n  low_thr %s\n"
                "  high_thr %s\n  accGrad %s" % (self["nx"], self["ny"], self["pixels_nonzero"], self["s"],
                                                 self["low_thr"], self["high_thr"], self["accGrad"]))


def canny_edge_detector(image, X, Y, s=2.0, low_thr=3.0, high_thr=10.0, accGrad=False):
    """The Rcpp export (rcpp_canny.cpp:122-126; note its accGrad default is false, the R wrapper's
    is TRUE).  image: length X*Y integer vector, index y*X + x; values are narrowed to unsigned
    char like `(unsigned char)image[i]` (rcpp_canny.cpp:137)."""
    lib = _lib.load()
    v = np.asarray(image).ravel()
    if v.size != X * Y:
        raise ValueError("image has %d elements, expected X*Y = %d" % (v.size, X * Y))
    u8 = np.ascontiguousarray(v.astype(np.int64) & 0xFF, dtype=np.uint8)
    edges = np.zeros(X * Y, np.uint8)
    nz = C.c_int(0)
    _lib.check(lib.b2f_canny_host(_lib.context(), _lib.ptr(u8), int(X), int(Y), float(s), float(low_thr),
                                  float(high_thr), int(bool(accGrad)), _lib.ptr(edges), C.byref(nz)))
    # NumericMatrix(nx, ny) filled in the input's linear order (rcpp_canny.cpp:226-229): R-style [X, Y]
    out = edges.astype(np.float64).reshape(Y, X).T
    return CannyResult(edges=out, pixels_nonzero=int(nz.value), nx=int(X), ny=int(Y), s=float(s),
                       low_thr=float(low_thr), high_thr=float(high_thr), accGrad=bool(accGrad))


def image_canny_edge_detector(x, s=2, low_thr=3, high_thr=10, accGrad=True):
    """image_canny_edge_detector(x, s = 2, low_thr = 3, high_thr = 10, accGrad = TRUE) as in R.
    `x` is an R-style integer matrix [nrow, ncol] (first index fastest, i.e. the image x
    coordinate); `edges` comes back in the same orientation with values 0 / 255."""
    a = np.asarray(x)
    if a.ndim != 2:
        raise ValueError("x must be a matrix")
    return canny_edge_detector(a.ravel(order="F"), a.shape[0], a.shape[1], s, low_thr, high_thr, accGrad)


def canny_batch(frames, s=2.0, low_thr=3.0, high_thr=10.0, accGrad=True, out=None, ctx=None):
    """Batch form (new surface): uint8 [n, ny, nx] host frames -> (edges uint8 [n, ny, nx], nonzero int32 [n]).
    `out` may be a preallocated (e.g. pinned) uint8 array of the same shape."""
    lib = _lib.load()
    f = np.ascontiguousarray(frames, dtype=np.uint8)
    n, ny, nx = f.shape
    edges = out if out is not None else np.empty_like(f)
    nz = np.zeros(n, np.int32)
    _lib.check(lib.b2f_canny_batch(ctx or _lib.context(), _lib.ptr(f), n, nx, ny, float(s), float(low_thr), float(high_thr),
                                   int(bool(accGrad)), _lib.ptr(edges), _lib.ptr(nz)))
    return edges, nz


def canny_dev(d_frames, n_frames, nx, ny, d_edges, d_nonzero, s=2.0, low_thr=3.0, high_thr=10.0, accGrad=True, stream=None, ctx=None):
    lib = _lib.load()
    _lib.check(lib.b2f_canny_dev(ctx or _lib.context(), _lib.ptr(d_frames), n_frames, nx, ny, float(s), float(low_thr),
                                 float(high_thr), int(bool(accGrad)), _lib.ptr(d_edges), _lib.ptr(d_nonzero),
                                 _lib.ptr(stream) if stream is not None else None))


def canny_hysteresis_dev(d_cls, n_frames, nx, ny, d_edges, d_nonzero, stream=None, ctx=None):
    """The hysteresis stage alone on device-resident class maps (uint8 [n, ny, nx]: 0 = no edge, 2 = strong,
    any other non-zero = weak) -> edge map (0 / 255) and per-frame edge counts, as canny_dev writes them."""
    lib = _lib.load()
    _lib.check(lib.b2f_canny_hysteresis_dev(ctx or _lib.context(), _lib.ptr(d_cls), n_frames, nx, ny, _lib.ptr(d_edges),
                                            _lib.ptr(d_nonzero), _lib.ptr(stream) if stream is not None else None))


def canny_tier2_pixels(ctx=None):
    """Pixels of this context's Canny calls that went to the exact fp64 tier (b2f_canny_stats)."""
    lib = _lib.load()
    n = C.c_ulonglong(0)
    _lib.check(lib.b2f_canny_stats(ctx or _lib.context(), C.byref(n)))
    return int(n.value)
