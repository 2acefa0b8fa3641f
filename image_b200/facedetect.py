"""Host-side mirror of image.libfacedetection: image_detect_faces(x) (R/pkg.R) and its Rcpp export detect_faces over the C
ABI of include/b2f.h (b2f_facedet_*).  The library ships no weights: load_model reads the package's own table
(param_pConvInfo) from a shared object that contains it.  No CPU path."""
import ctypes as C

import numpy as np

from . import _lib

N_LAYERS = 24
COLUMNS = ("x", "y", "width", "height", "confidence", "landmark1_x", "landmark1_y", "landmark2_x", "landmark2_y",
           "landmark3_x", "landmark3_y", "landmark4_x", "landmark4_y", "landmark5_x", "landmark5_y")
_FIELD = (1, 2, 3, 4, 0, 5, 6, 7, 8, 9, 10, 11, 12, 13, 14)     # column -> index in the 15 ints of a face


class ConvLayer(C.Structure):
    """b2f_conv_layer, laid out like the reference's ConvInfoStruct."""
    _fields_ = [("pad", C.c_int), ("stride", C.c_int), ("kernel_size", C.c_int), ("channels", C.c_int), ("num", C.c_int),
                ("scale", C.c_float), ("weights", C.c_void_p), ("bias", C.c_void_p)]


def read_layers(so_path):
    """(library handle, ConvLayer[24]) of the param_pConvInfo table exported by the shared object so_path."""
    lib = C.CDLL(so_path)
    return lib, (ConvLayer * N_LAYERS).in_dll(lib, "param_pConvInfo")


class FaceModel:
    """A b2f_facedet_model: the weights repacked on the device of `ctx`.  free() releases it."""

    def __init__(self, layers, ctx=None, keep=None):
        self.ctx = ctx or _lib.context()
        self._keep = keep
        self.handle = C.c_void_p()
        _lib.check(_lib.load().b2f_facedet_model_create(self.ctx, C.cast(layers, C.c_void_p), len(layers), C.byref(self.handle)))

    def free(self):
        if self.handle:
            _lib.load().b2f_facedet_model_free(self.handle)
            self.handle = C.c_void_p()


def load_model(so_path, ctx=None):
    """The model of the param_pConvInfo table in so_path (the R package's shared object, or any library exporting it)."""
    lib, tab = read_layers(so_path)
    return FaceModel(tab, ctx, keep=lib)


def _faces(n, f):
    return dict(nr=int(n), detections={c: f[:n, i].astype(np.int64) for c, i in zip(COLUMNS, _FIELD)})


def detect_faces(x, width, height, step, model):
    """The Rcpp export detect_faces: x = the interleaved RGB frame as integers (R's aperm(x, c(3, 2, 1))).  Returns
    dict(nr, detections = dict of the data frame's 15 integer columns)."""
    v = np.ascontiguousarray(np.asarray(x).ravel(), dtype=np.int32)
    n = C.c_int(0)
    f = np.zeros((256, 15), np.int32)
    _lib.check(_lib.load().b2f_facedet_host_r32(model.ctx, model.handle, _lib.ptr(v), v.size, int(width), int(height), int(step),
                                                C.byref(n), _lib.ptr(f)))
    return _faces(n.value, f)


def image_detect_faces(x, model):
    """image_detect_faces for an [h, w, 3] array (R/pkg.R): aperm to interleaved RGB, step = 3w."""
    a = np.asarray(x)
    if a.ndim != 3 or a.shape[2] != 3:
        raise ValueError("x must be [h, w, 3]")
    h, w = a.shape[:2]
    return detect_faces(a.astype(np.int32).ravel(), w, h, 3 * w, model)


def facedetect_batch(frames, model):
    """b2f_facedet_batch_rgb: u8 frames [n, h, w, 3] in host memory -> (n_faces int32 [n], faces int32 [n, 256, 15])."""
    a = np.ascontiguousarray(frames, dtype=np.uint8)
    n, h, w = a.shape[:3]
    nf = np.zeros(n, np.int32)
    f = np.zeros((n, 256, 15), np.int32)
    _lib.check(_lib.load().b2f_facedet_batch_rgb(model.ctx, model.handle, _lib.ptr(a), n, w, h, _lib.ptr(nf), _lib.ptr(f)))
    return nf, f


def facedetect_dev(d_frames, n_frames, width, height, model, layer_max=False, cand_cap=0, stream=None):
    """b2f_facedet_dev: u8 frames [n, h, w, 3] on the device (a pointer or a tensor).  Returns dict(n_faces, faces) and,
    when asked, layer_max int32 [n, 16] and the candidate records cand int32 [n, cand_cap, 17] with n_cand [n]."""
    n = int(n_frames)
    nf = np.zeros(n, np.int32)
    f = np.zeros((n, 256, 15), np.int32)
    lm = np.zeros((n, 16), np.int32) if layer_max else None
    cand = np.zeros((n, cand_cap, 17), np.int32) if cand_cap else None
    nc = np.zeros(n, np.int32) if cand_cap else None
    _lib.check(_lib.load().b2f_facedet_dev(model.ctx, model.handle, _lib.ptr(d_frames), n, int(width), int(height), _lib.ptr(nf),
                                           _lib.ptr(f), _lib.ptr(lm), _lib.ptr(cand), int(cand_cap), _lib.ptr(nc),
                                           C.c_void_p(stream) if stream is not None else None))
    out = dict(n_faces=nf, faces=f)
    if layer_max:
        out["layer_max"] = lm
    if cand_cap:
        out["cand"], out["n_cand"] = cand, nc
    return out
