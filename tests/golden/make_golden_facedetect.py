"""Writes tests/golden/facedetect_handshake.npz: the RGB pixels of the three faces of image.libfacedetection's example
image inst/images/handshake.jpg (the 592x192 region x 240..831, y 96..287 of the 1024x683 photo, which keeps the file
small), decoded once with PIL so that no JPEG decoder is needed where the tests run, and the reference's detections on it
(facedetect_cnn of oracle/_ref/libref_facedetect.so: int32 [n, 15], confidence, x, y, w, h, 5 landmarks).
Run from the repository root where the reference tree and its build exist:
    python tests/golden/make_golden_facedetect.py /path/to/image.libfacedetection/inst/images/handshake.jpg"""
import os
import sys

import numpy as np
from PIL import Image

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from oracle import ref_facedetect as rf  # noqa: E402

Y0, Y1, X0, X1 = 96, 288, 240, 832

rgb = np.ascontiguousarray(np.asarray(Image.open(sys.argv[1]).convert("RGB"))[Y0:Y1, X0:X1], dtype=np.uint8)
faces = rf.facedetect_cnn(rgb)
np.savez_compressed(os.path.join(ROOT, "tests", "golden", "facedetect_handshake.npz"), rgb=rgb, faces=faces)
print(rgb.shape, len(faces), "faces")
