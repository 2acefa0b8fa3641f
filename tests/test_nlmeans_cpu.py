"""CPU tests of the NL-means parameter table (b2f_nlmeans_resolve needs no device) against the serial reference build,
and of the reference build against the smallest frozen digest."""
import json
import os

import numpy as np
import pytest

import nlmeans_cases as nc

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GREY_EDGES = [15.0, 30.0, 45.0, 75.0, 100.0]
COLOUR_EDGES = [25.0, 55.0, 100.0]


def _grid(edges):
    s = [0.0, -0.0, -1e-30, -5.0, -1e6, np.float32(1e-45), 1.0, 150.0, 1e30, np.inf, -np.inf, np.nan]
    for e in [0.0] + edges:
        e = np.float32(e)
        s += [e, np.nextafter(e, np.float32(-np.inf)), np.nextafter(e, np.float32(np.inf))]
    return [float(np.float32(v)) for v in s]


def _resolve(c, sigma):
    from image_b200 import B2FError
    from image_b200.nlmeans import nlmeans_resolve
    try:
        return nlmeans_resolve(c, sigma)
    except B2FError as e:
        assert "algorithm parametrized only for values of sigma less than 100.0" in str(e)
        return None


def test_resolve_table():
    assert _resolve(1, 10) == (1, 10, np.float32(0.4)) and _resolve(1, 30) == (2, 10, np.float32(0.4))
    assert _resolve(1, 31) == (3, 17, np.float32(0.35)) and _resolve(1, 75) == (4, 17, np.float32(0.35))
    assert _resolve(1, 100) == (5, 17, np.float32(0.3)) and _resolve(1, 0) == (5, 17, np.float32(0.3))
    assert _resolve(3, 25) == (1, 10, np.float32(0.55)) and _resolve(3, 26) == (2, 17, np.float32(0.4))
    assert _resolve(3, -3) == (3, 17, np.float32(0.35)) and _resolve(3, 100.5) is None and _resolve(1, np.nan) is None
    assert _resolve(2, 20) == _resolve(1, 20) and _resolve(4, 20) == _resolve(3, 20)       # the glue's channel mapping
    from image_b200.nlmeans import nlmeans_resolve
    assert nlmeans_resolve(3, 500.0, False, 7, 3, 0.25) == (7, 3, np.float32(0.25))     # explicit: left as given
    from image_b200 import B2FError
    with pytest.raises(B2FError):
        nlmeans_resolve(0, 10.0)


@pytest.fixture(scope="module")
def ref(oracle):
    from oracle import ref_nlmeans as rn
    if not rn.have_ref():
        rn.build()
    if not rn.have_ref():
        pytest.skip("oracle/_ref/libref_nlmeans.so not built (reference tree absent)")
    return rn


@pytest.mark.parametrize("channels", [1, 3])
def test_resolve_agrees_with_reference(ref, channels):
    img = np.arange(channels, dtype=np.int32)            # 1x1 frame: no candidates, the glue's table is all that runs
    for s in _grid(GREY_EDGES if channels == 1 else COLOUR_EDGES):
        mine = _resolve(channels, s)
        try:
            r = ref.nlmeans(img, 1, 1, channels, s)
            want = (r["window"], r["bloc"], r["filter"])
            assert r["channels"] == channels
        except ValueError as e:
            assert "sigma less than 100.0" in str(e)
            want = None
        assert mine == want, (channels, s, mine, want)


def test_reference_reproduces_smallest_digest(oracle, ref):
    with open(os.path.join(ROOT, "tests", "golden", "nlmeans_digests.json")) as f:
        d = json.load(f)
    key, img, sigma = next(nc.digest_cases())
    c, h, w = img.shape
    assert nc.digest_of(oracle, ref.nlmeans(img.ravel(), w, h, c, sigma)) == d[key]
