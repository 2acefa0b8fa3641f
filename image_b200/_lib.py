"""ctypes binding of libb200feat.so (the C ABI declared in include/b2f.h).

The CUDA library IS the product: there is no CPU fallback.  Importing this module only loads
the shared object (possible on a CPU-only box, for symbol checks); the first call that needs a
device creates a context with b2f_init, which raises B2FError when no H100 is present.
"""
import ctypes as C
import os
import threading

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(HERE, "libb200feat.so")

B2F_OK, B2F_EINVAL, B2F_ECUDA, B2F_ENOMEM, B2F_ECAP, B2F_EUNSUP = 0, -1, -2, -3, -4, -5


class B2FError(RuntimeError):
    """Raised for every non-zero status of the C ABI (the Rcpp shim turns these into Rcpp::stop)."""

    def __init__(self, code, msg):
        super().__init__("libb200feat error %d: %s" % (code, msg))
        self.code = code


class HarrisParams(C.Structure):
    _fields_ = [("k", C.c_float), ("sigma_d", C.c_float), ("sigma_i", C.c_float), ("threshold", C.c_float),
                ("gaussian", C.c_int), ("gradient", C.c_int), ("strategy", C.c_int), ("Nselect", C.c_int),
                ("measure", C.c_int), ("Nscales", C.c_int), ("precision", C.c_int), ("cells", C.c_int),
                ("verbose", C.c_int), ("exact", C.c_int)]


class CannyParams(C.Structure):
    _fields_ = [("s", C.c_double), ("low_thr", C.c_double), ("high_thr", C.c_double), ("acc_grad", C.c_int)]


class SurfPoint(C.Structure):
    _fields_ = [("x", C.c_double), ("y", C.c_double), ("angle", C.c_double), ("scale", C.c_double),
                ("score", C.c_double), ("laplacian", C.c_double), ("des", C.c_double * 64)]


_lib = None
_lock = threading.Lock()
_ctx = {}


def load():
    """Load libb200feat.so; fails loudly when it has not been built (python __graft_entry__.py build)."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise ImportError("image_b200: %s is missing — build it with `make -C image_b200/csrc` "
                          "(or __graft_entry__.build()); there is no CPU fallback" % LIB_PATH)
    lib = C.CDLL(LIB_PATH)
    vp, ip, fp = C.c_void_p, C.POINTER(C.c_int), C.POINTER(C.c_float)
    lib.b2f_last_error.restype = C.c_char_p
    lib.b2f_version.restype = C.c_char_p
    lib.b2f_init.argtypes = [C.c_int, C.POINTER(vp)]
    lib.b2f_shutdown.argtypes = [vp]
    lib.b2f_free.argtypes = [vp]
    lib.b2f_stream.argtypes = [vp]
    lib.b2f_stream.restype = vp
    lib.b2f_launch_count.argtypes = [vp]
    lib.b2f_launch_count.restype = C.c_longlong
    lib.b2f_set_chunk_bytes.argtypes = [vp, C.c_size_t]
    lib.b2f_otsu_host.argtypes = [vp, vp, C.c_int, C.c_int, C.c_int, vp, ip]
    lib.b2f_otsu_batch_u8.argtypes = [vp, vp, C.c_int, C.c_int, C.c_int, C.c_int, vp, vp]
    lib.b2f_otsu_dev.argtypes = [vp, vp, C.c_int, C.c_int, C.c_int, C.c_int, vp, vp, vp]
    lib.b2f_harris_default_params.argtypes = [C.POINTER(HarrisParams)]
    lib.b2f_harris_host.argtypes = [vp, vp, C.c_int, C.c_int, C.POINTER(HarrisParams), C.POINTER(fp), C.POINTER(fp), C.POINTER(fp), ip]
    lib.b2f_harris_batch_u8.argtypes = [vp, vp, C.c_int, C.c_int, C.c_int, C.POINTER(HarrisParams), C.c_int, vp, vp, vp, vp]
    lib.b2f_harris_response_dev.argtypes = [vp, vp, C.c_int, C.c_int, C.c_int, C.c_int, C.POINTER(HarrisParams), vp, vp]
    lib.b2f_harris_corners_dev.argtypes = [vp, vp, C.c_int, C.c_int, C.c_int, C.c_int, C.POINTER(HarrisParams), C.c_int, vp, vp, vp, vp, vp]
    lib.b2f_harris_cert_stats.argtypes = [vp, C.POINTER(C.c_ulonglong)]
    lib.b2f_harris_response_eps_dev.argtypes = [vp, vp, C.c_int, C.c_int, C.c_int, C.c_int, C.POINTER(HarrisParams), vp, vp, vp]
    lib.b2f_harris_nms_dev.argtypes = [vp, vp, C.c_int, C.c_int, C.c_int, C.c_float, C.c_int, C.c_int, vp, vp, vp, vp]
    for name, args in [
        ("b2f_canny_host", [vp, vp, C.c_int, C.c_int, C.c_double, C.c_double, C.c_double, C.c_int, vp, ip]),
        ("b2f_canny_batch", [vp, vp, C.c_int, C.c_int, C.c_int, C.c_double, C.c_double, C.c_double, C.c_int, vp, vp]),
        ("b2f_canny_dev", [vp, vp, C.c_int, C.c_int, C.c_int, C.c_double, C.c_double, C.c_double, C.c_int, vp, vp, vp]),
        ("b2f_canny_hysteresis_dev", [vp, vp, C.c_int, C.c_int, C.c_int, vp, vp, vp]),
        ("b2f_canny_stats", [vp, C.POINTER(C.c_ulonglong)]),
        ("b2f_fhog_size", [C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, ip, ip]),
        ("b2f_fhog_host", [vp, vp, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, vp]),
        ("b2f_fhog_batch", [vp, vp, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, vp]),
        ("b2f_fhog_dev", [vp, vp, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, vp, vp]),
        ("b2f_surf_host", [vp, vp, C.c_int, C.c_int, C.c_long, C.c_double, C.POINTER(C.POINTER(SurfPoint)), ip]),
        ("b2f_surf_batch", [vp, vp, C.c_int, C.c_int, C.c_int, C.c_long, C.c_double, C.c_int, vp, vp]),
        ("b2f_harris_host_r64", [vp, vp, C.c_int, C.c_int, C.POINTER(HarrisParams), C.POINTER(fp), C.POINTER(fp), C.POINTER(fp), ip]),
        ("b2f_canny_host_r32", [vp, vp, C.c_int, C.c_int, C.c_double, C.c_double, C.c_double, C.c_int, vp, ip]),
        ("b2f_fhog_host_r32", [vp, vp, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, vp]),
        ("b2f_surf_host_r32", [vp, vp, C.c_int, C.c_int, C.c_long, C.c_double, C.POINTER(C.POINTER(SurfPoint)), ip]),
        ("b2f_surf_dev", [vp, vp, C.c_int, C.c_int, C.c_int, C.c_long, C.c_double, C.c_int, vp, vp, vp]),
        ("b2f_features_batch_rgb", [vp, vp, C.c_int, C.c_int, C.c_int, C.POINTER(HarrisParams), C.c_int, vp, vp, vp, vp,
                                    C.POINTER(CannyParams), vp, vp, C.c_int, C.c_int, C.c_int, vp]),
        ("b2f_features_batch_grey", [vp, vp, C.c_int, C.c_int, C.c_int, C.POINTER(HarrisParams), C.c_int, vp, vp, vp, vp,
                                     C.POINTER(CannyParams), vp, vp]),
        ("b2f_lsd_front_size", [C.c_int, C.c_int, C.c_double, ip, ip]),
        ("b2f_lsd_front_host", [vp, vp, C.c_int, C.c_int, C.c_double, C.c_double, C.c_double, C.c_double, C.c_int, vp, vp, vp, ip, vp]),
        ("b2f_lsd_front_dev", [vp, vp, C.c_int, C.c_int, C.c_int, C.c_int, C.c_double, C.c_double, C.c_double, C.c_double, C.c_int, vp, vp, vp, vp, vp]),
        ("b2f_contour_edge_points_host", [vp, vp, C.c_int, C.c_int, C.c_double, vp, C.POINTER(ip), C.POINTER(C.POINTER(C.c_double)),
                                          C.POINTER(C.POINTER(C.c_double)), C.POINTER(C.POINTER(C.c_double)), C.POINTER(C.POINTER(C.c_double)), ip]),
        ("b2f_contour_edge_points_batch_u8", [vp, vp, C.c_int, C.c_int, C.c_int, C.c_double, C.c_int, vp, vp, vp, vp, vp, vp]),
        ("b2f_contour_edge_points_dev", [vp, vp, C.c_int, C.c_int, C.c_int, C.c_int, C.c_double, C.c_int, vp, vp, vp, vp, vp, vp, vp, vp]),
    ]:
        if hasattr(lib, name):
            getattr(lib, name).argtypes = args
    _lib = lib
    return lib


def check(rc):
    if rc != B2F_OK:
        raise B2FError(rc, load().b2f_last_error().decode("utf-8", "replace"))


def context(device=None):
    """One context per (thread, device), created lazily (R_init_<pkg> does the same in the R build)."""
    lib = load()
    if device is None:      # one process per GPU: B2F_DEVICE, else torchrun's LOCAL_RANK, else 0
        device = int(os.environ.get("B2F_DEVICE", os.environ.get("LOCAL_RANK", "0")))
    key = (threading.get_ident(), device)
    with _lock:
        if key not in _ctx:
            h = C.c_void_p()
            check(lib.b2f_init(int(device), C.byref(h)))
            _ctx[key] = h
        return _ctx[key]


def new_context(device=None):
    """An additional context (own stream + scratch arena) on `device`; calls on different contexts may
    run concurrently (bench.py gives each detector its own).  Released by shutdown()."""
    lib = load()
    if device is None:
        device = int(os.environ.get("B2F_DEVICE", os.environ.get("LOCAL_RANK", "0")))
    h = C.c_void_p()
    check(lib.b2f_init(int(device), C.byref(h)))
    with _lock:
        _ctx[("extra", len(_ctx), device)] = h
    return h


def shutdown():
    lib = load()
    with _lock:
        for h in _ctx.values():
            lib.b2f_shutdown(h)
        _ctx.clear()


def ptr(a):
    """void* of a numpy array or an int (device pointer) or an object with data_ptr() (torch tensor)."""
    if a is None:
        return None
    if isinstance(a, int):
        return C.c_void_p(a)
    if isinstance(a, np.ndarray):
        return a.ctypes.data_as(C.c_void_p)
    if hasattr(a, "data_ptr"):
        return C.c_void_p(a.data_ptr())
    raise TypeError("cannot take a pointer of %r" % type(a))


EXPORTS = [
    "b2f_init", "b2f_shutdown", "b2f_last_error", "b2f_version", "b2f_device_count", "b2f_free", "b2f_stream",
    "b2f_launch_count", "b2f_set_chunk_bytes", "b2f_harris_default_params", "b2f_harris_host", "b2f_harris_batch_u8",
    "b2f_harris_response_dev", "b2f_harris_nms_dev", "b2f_harris_corners_dev", "b2f_harris_cert_stats",
    "b2f_harris_response_eps_dev", "b2f_canny_host", "b2f_canny_batch", "b2f_canny_dev", "b2f_canny_hysteresis_dev", "b2f_canny_stats",
    "b2f_fhog_size", "b2f_fhog_host", "b2f_fhog_batch", "b2f_fhog_dev", "b2f_surf_host", "b2f_surf_batch", "b2f_surf_dev",
    "b2f_otsu_host", "b2f_otsu_batch_u8", "b2f_otsu_dev",
    "b2f_harris_host_r64", "b2f_canny_host_r32", "b2f_fhog_host_r32", "b2f_surf_host_r32", "b2f_features_batch_rgb", "b2f_features_batch_grey", "b2f_lsd_front_size", "b2f_lsd_front_host", "b2f_lsd_front_dev",
    "b2f_contour_edge_points_host", "b2f_contour_edge_points_batch_u8", "b2f_contour_edge_points_dev",
]
