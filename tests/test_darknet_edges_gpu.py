"""darknet on the H100: a classification batch that crosses a chunk boundary, and a network taller than wide classified
without resize, where a frame whose resize_min planes are shorter than the network input is refused."""
import os

import numpy as np
import pytest
import torch

from image_b200 import _lib
from image_b200 import darknet as dn
from oracle import ref_darknet as rd
from darknet_cases import shrink_cfg

pytestmark = [pytest.mark.gpu, pytest.mark.skipif(not rd.have_ref(), reason="reference build oracle/_ref/libref_darknet.so absent")]


def test_classify_batch_crosses_chunks():
    """About 9 MB of scratch per 298x224 frame: 2 GB chunks hold some 230 frames, so 300 frames make two chunks."""
    m = dn.load_network(rd.path("tiny.cfg"), rd.path("tiny.weights"))
    try:
        rng = np.random.default_rng(12)
        n, h, w = 300, 48, 64
        frames = rng.integers(0, 256, (n, h, w, 3), dtype=np.uint8)
        frames[250] = rd.decode("eagle.jpg")[100:100 + h, 200:200 + w]
        idx, prob = dn.classify_batch(frames, m, True, 5)
        d = torch.from_numpy(frames).cuda()
        i2, p2 = dn.classify_dev(d, n, w, h, m, True, 5)
        assert np.array_equal(idx, i2) and np.array_equal(prob, p2)
        rd.load(rd.path("tiny.cfg"), rd.path("tiny.weights"))
        for i in (0, 228, 229, 230, 250, n - 1):
            want = rd.classify(frames[i], True, 5)
            assert np.array_equal(idx[i], want["index"]) and np.array_equal(prob[i], want["probability"])
    finally:
        m.free()


def test_tall_network_without_resize(tmp_path):
    cfg = shrink_cfg(rd.path("tiny.cfg"), str(tmp_path / "tall.cfg"), 224, 300)
    m = dn.load_network(cfg, rd.path("tiny.weights"))
    try:
        wide = np.random.default_rng(5).integers(0, 256, (100, 400, 3), dtype=np.uint8)   # planes 896x224: enough
        idx, prob = dn.classify_batch(wide, m, False, 5)
        rd.load(cfg, rd.path("tiny.weights"))
        want = rd.classify(wide, False, 5)
        assert np.array_equal(idx[0], want["index"]) and np.array_equal(prob[0], want["probability"])
        short = np.random.default_rng(6).integers(0, 256, (224, 250, 3), dtype=np.uint8)  # planes 250x224 < 224x300
        with pytest.raises(_lib.B2FError, match="fewer floats") as e:
            dn.classify_batch(short, m, False, 5)
        assert e.value.code == _lib.B2F_EUNSUP
        dn.classify_batch(short, m, True, 5)                                            # with resize it runs
    finally:
        m.free()
