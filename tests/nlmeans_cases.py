"""Seeded NL-means inputs shared by tests/golden/make_golden_nlmeans.py (which freezes the serial reference's output on
them as digests) and the tests that compare the GPU with those digests.  Images are channel-planar int32 [c, h, w]."""
import os

import numpy as np

from image_b200 import synth

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def noisy(img, std, seed):
    """img + N(0, std) from a seeded numpy generator, rounded and clipped to 0..255 (the reference's own fiAddNoise seeds
    from the clock)."""
    rng = np.random.default_rng(seed)
    return np.clip(np.rint(img.astype(np.float64) + rng.normal(0.0, std, img.shape)), 0, 255).astype(np.int32)


def garden():
    """The reference's fixture img_garden.png (640x478 RGB), decoded: uint8 [h, w, 3]."""
    return np.load(os.path.join(GOLDEN, "nlmeans_garden.npz"))["image"]


def digest_cases():
    """(key, image [c, h, w] int32, sigma) of the frozen digests, smallest first; all run with the parameter table."""
    g = garden().transpose(2, 0, 1).astype(np.int32)
    yield "garden_sigma10", g, 10.0
    yield "garden_noise20_sigma20", noisy(g, 20.0, 7), 20.0
    grey = noisy(synth.frame_shapes(501, 1024, 1024)[None], 60.0, 8)
    yield "grey1024_sigma60", grey, 60.0
    rgb = synth.frame_rgb(502, 1080, 1920).transpose(2, 0, 1)
    yield "rgb1080_sigma10", noisy(rgb, 10.0, 9), 10.0
    yield "rgb1080_sigma40", noisy(rgb, 40.0, 10), 40.0


def digest_of(po, r):
    """Digest of an rcpp_nlmeans result: the denoised doubles, then (channels, window, bloc) and the filter."""
    return po.digest(np.asarray(r["denoised"], np.float64), np.array([r["channels"], r["window"], r["bloc"]], np.int64),
                     np.float32(r["filter"]))
