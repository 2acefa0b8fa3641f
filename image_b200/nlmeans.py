"""Host-side mirror of image.DenoiseNLMeans: image_denoise_nlmeans(image, sigma = 10, win = 1, bloc = 10, filter = 0.4)
(R/pkg.R) and its Rcpp export rcpp_nlmeans over the C ABI of include/b2f.h (b2f_nlmeans_*).  No CPU path."""
import ctypes as C

import numpy as np

from . import _lib


def nlmeans_resolve(channels, sigma, args_auto=True, win=1, bloc=10, filter=0.4):
    """The glue's parameter table (b2f_nlmeans_resolve): (win, bloc, filter) a call with these arguments runs with.
    channels = the channel count after the colour test (1 = grey).  Raises B2FError for sigma > 100 when args_auto."""
    w, b, f = C.c_int(int(win)), C.c_int(int(bloc)), C.c_float(filter)
    _lib.check(_lib.load().b2f_nlmeans_resolve(int(channels), C.c_float(sigma), int(bool(args_auto)), C.byref(w), C.byref(b), C.byref(f)))
    return w.value, b.value, f.value


def rcpp_nlmeans(image, width, height, channels, sigma, args_auto=True, win=1, bloc=10, fFiltPar=0.4):
    """The Rcpp export rcpp_nlmeans: image = width*height*channels integers, channel-planar (x + w*y + w*h*c, R's
    aperm(image_data, c(2, 1, 3))).  Returns the glue's list: dict(width, height, channels, denoised = float64 vector of
    channels planes, sigma, filter, window, bloc)."""
    lib = _lib.load()
    v = np.ascontiguousarray(np.asarray(image).ravel(), dtype=np.int32)
    if v.size != int(width) * int(height) * int(channels):
        raise ValueError("image must hold width * height * channels values")
    out = np.empty(max(int(width) * int(height) * min(max(int(channels), 1), 3), 1), np.float32)
    oc, w, b, f = C.c_int(0), C.c_int(0), C.c_int(0), C.c_float(0)
    _lib.check(lib.b2f_nlmeans_host_r32(_lib.context(), _lib.ptr(v), int(width), int(height), int(channels), C.c_float(sigma),
                                        int(bool(args_auto)), int(win), int(bloc), C.c_float(fFiltPar), _lib.ptr(out),
                                        C.byref(oc), C.byref(w), C.byref(b), C.byref(f)))
    n = int(width) * int(height) * oc.value
    return dict(width=int(width), height=int(height), channels=oc.value, denoised=out[:n].astype(np.float64),
                sigma=float(np.float32(sigma)), filter=f.value, window=w.value, bloc=b.value)


def image_denoise_nlmeans(x, sigma=10, win=None, bloc=None, filter=None):
    """image_denoise_nlmeans for an [h, w, 3] or [h, w] array of 0..255 values (R/pkg.R): the parameter table is used
    unless win, bloc and filter are all given (R's missing() rule); denoised values above 255 are set to 255.  Returns
    dict(x = float64 array of the input's shape, sigma, filter, window, bloc).  A grey result is recycled over the three
    planes of an [h, w, 3] input, as R's array(ok, dim = c(width, height, 3)) does."""
    a = np.asarray(x)
    if a.ndim == 2:
        a3 = np.repeat(a[:, :, None], 3, axis=2)
    elif a.ndim == 3 and a.shape[2] == 3:
        a3 = a
    else:
        raise ValueError("x must be [h, w] or [h, w, 3]")
    h, w = a3.shape[:2]
    args_auto = win is None or bloc is None or filter is None
    r = rcpp_nlmeans(np.ascontiguousarray(a3.transpose(2, 0, 1)).astype(np.int32), w, h, 3, sigma, args_auto,
                     1 if win is None else win, 10 if bloc is None else bloc, 0.4 if filter is None else filter)
    ok = np.minimum(r["denoised"], 255.0)
    planes = np.resize(ok, 3 * w * h).reshape(3, h, w)                  # R recycles a single plane
    out = planes[0] if a.ndim == 2 else planes.transpose(1, 2, 0)
    return dict(x=np.ascontiguousarray(out), sigma=r["sigma"], filter=r["filter"], window=r["window"], bloc=r["bloc"])


def nlmeans_dev(d_frames, n_frames, channels, width, height, win, bloc, sigma, filter, d_out, stream=None, ctx=None):
    """b2f_nlmeans_dev: u8 [n, channels, h, w] frames on the device -> float32 [n, C, h, w] (C = 1 for channels 1 or 2,
    else 3), explicit parameters, asynchronous on `stream` (a cudaStream_t as int; None = the context's stream)."""
    lib = _lib.load()
    _lib.check(lib.b2f_nlmeans_dev(ctx or _lib.context(), _lib.ptr(d_frames), int(n_frames), int(channels), int(width), int(height),
                                   int(win), int(bloc), C.c_float(sigma), C.c_float(filter), _lib.ptr(d_out),
                                   C.c_void_p(stream) if stream is not None else None))
