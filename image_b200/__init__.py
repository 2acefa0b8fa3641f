"""image_b200 — H100-native (sm_90a) engine for the per-pixel feature-detection hot path of
bnosac/image (image.CornerDetectionHarris, image.CannyEdges, image.dlib FHOG/SURF).

The product is the CUDA shared library image_b200/libb200feat.so (C ABI: include/b2f.h).  This
package is the host-side mirror of the reference's R functions over that ABI, used by the parity
tests and the benchmark; the R packages themselves bind the same ABI through the Rcpp shims in
image_b200/rshim/ (see INTEGRATION.md).  There is no CPU fallback.
"""
from ._lib import B2FError, load, context, shutdown  # noqa: F401
from .harris import image_harris, detect_corners, harris_batch_u8  # noqa: F401
from .canny import image_canny_edge_detector, canny_edge_detector, canny_batch  # noqa: F401
from .dlib import image_fhog, image_surf, dlib_fhog, dlib_surf_points, fhog_batch, surf_batch  # noqa: F401
from .otsu import image_otsu, otsu_batch  # noqa: F401   (the export mirror otsu() stays in image_b200.otsu: same name as the module)
from .nlmeans import image_denoise_nlmeans, rcpp_nlmeans, nlmeans_dev  # noqa: F401
from .facedetect import image_detect_faces, detect_faces, facedetect_batch, facedetect_dev, load_model  # noqa: F401
from .darknet import image_darknet_model, image_darknet_detect, image_darknet_classify  # noqa: F401

__all__ = ["image_harris", "detect_corners", "harris_batch_u8", "image_canny_edge_detector", "canny_edge_detector",
           "canny_batch", "image_fhog", "image_surf", "dlib_fhog", "dlib_surf_points", "fhog_batch", "surf_batch",
           "image_otsu", "otsu_batch", "image_denoise_nlmeans", "rcpp_nlmeans", "nlmeans_dev", "image_detect_faces", "detect_faces", "facedetect_batch", "facedetect_dev", "load_model", "image_darknet_model", "image_darknet_detect", "image_darknet_classify", "B2FError", "load", "context", "shutdown"]
