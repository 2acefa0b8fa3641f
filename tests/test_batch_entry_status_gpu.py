"""Status codes of the single-detector host batches (b2f_harris_batch_u8, b2f_canny_batch, b2f_fhog_batch): what each
entry refuses, what it serves, and what it reports when a frame has more corners than the caller made room for."""
import ctypes as C

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

NY, NX = 120, 160


def _harris(frames, cap, n=None, nx=NX, ny=NY, out=True, **kw):
    """b2f_harris_batch_u8 on frames [n, ny, nx]: (status, x, y, strength, counts)."""
    from image_b200 import _lib
    from image_b200.harris import _params
    n = len(frames) if n is None else n
    k = max(len(frames), 1)
    x, y, s = (np.empty((k, max(cap, 1)), np.float32) for _ in range(3))
    cnt = np.zeros(k, np.int32)
    f = np.ascontiguousarray(frames, dtype=np.uint8)
    rc = _lib.load().b2f_harris_batch_u8(_lib.context(), _lib.ptr(f) if f.size else None, n, nx, ny, C.byref(_params(kw)), cap,
                                         _lib.ptr(x) if out else None, _lib.ptr(y), _lib.ptr(s), _lib.ptr(cnt))
    return rc, x, y, s, cnt


def _canny(frames, n=None, nx=NX, ny=NY, edges=True, nonzero=True):
    from image_b200 import _lib
    n = len(frames) if n is None else n
    f = np.ascontiguousarray(frames, dtype=np.uint8)
    e = np.empty((max(len(frames), 1), ny, nx), np.uint8)
    nz = np.zeros(max(len(frames), 1), np.int32)
    return _lib.load().b2f_canny_batch(_lib.context(), _lib.ptr(f) if f.size else None, n, nx, ny, 2.0, 3.0, 10.0, 1,
                                       _lib.ptr(e) if edges else None, _lib.ptr(nz) if nonzero else None)


def _fhog(frames, rows, cols, cell=8, n=None, hog=True):
    from image_b200 import _lib
    n = len(frames) if n is None else n
    f = np.ascontiguousarray(frames, dtype=np.uint8)
    h = np.empty(max(len(frames), 1) * 200 * 200 * 31, np.float32)
    return _lib.load().b2f_fhog_batch(_lib.context(), _lib.ptr(f) if f.size else None, n, rows, cols, cell, 1, 1,
                                      _lib.ptr(h) if hog else None)


def _grey(n):
    from image_b200 import synth
    return np.stack([synth.frame_shapes(610 + i, NY, NX) for i in range(n)])


def test_harris_batch_refusals():
    from image_b200._lib import B2F_EINVAL, B2F_EUNSUP
    g = _grey(1)
    assert _harris(g, 64, out=False)[0] == B2F_EINVAL
    assert _harris(np.zeros((0, NY, NX), np.uint8), 64)[0] == B2F_EINVAL
    assert _harris(g, 64, n=0)[0] == B2F_EINVAL
    assert _harris(g, 0)[0] == B2F_EINVAL
    assert _harris(g, 64, nx=0)[0] == B2F_EINVAL
    for kw in (dict(strategy=2), dict(precision=1), dict(Nscales=2)):
        assert _harris(g, 64, **kw)[0] == B2F_EUNSUP, kw
    rc, x, y, s, cnt = _harris(g, 4096, threshold=60.0)                    # the context still serves a valid call
    assert rc == 0 and cnt[0] > 0


def test_harris_batch_reports_a_frame_over_cap(oracle):
    """B2F_ECAP, and counts[f] is the frame's true count (not cap + 1), also on the certified path, whose candidate
    records are sized by the cap."""
    from image_b200._lib import B2F_ECAP
    noise = np.random.default_rng(11).integers(0, 256, (NY, NX), dtype=np.uint8)
    flat = np.full((NY, NX), 90, np.uint8)
    cap = 16
    n_true = len(oracle.harris_detect(noise, threshold=1.0, sigma_i=1.0)[0])
    for mode in (0, 1):
        rc, _, _, _, cnt = _harris(np.stack([noise, flat]), cap, threshold=1.0, sigma_i=1.0, exact=mode)
        assert rc == B2F_ECAP
        assert cnt[0] == n_true > cap + 1 and cnt[1] == 0, (mode, cnt, n_true)


def test_harris_batch_exact_modes_give_the_same_lists():
    """exact = 0 (certified path), 1 (staged kernels) and 3 (treated as the default) return the same corner lists; 2 is
    the uncertified fp32 path and is not expected to match bit for bit."""
    g = _grey(1)
    outs = []
    for mode in (0, 1, 3):
        rc, x, y, s, cnt = _harris(g, 8192, threshold=30.0, exact=mode)
        assert rc == 0 and cnt[0] > 0, mode
        m = cnt[0]
        outs.append((x[0, :m].copy(), y[0, :m].copy(), s[0, :m].copy()))
    for mode, o in zip((1, 3), outs[1:]):
        for q in range(3):
            assert np.array_equal(o[q], outs[0][q]), mode


def test_canny_batch_refusals():
    from image_b200._lib import B2F_EINVAL
    g = _grey(1)
    assert _canny(np.zeros((0, NY, NX), np.uint8)) == B2F_EINVAL
    assert _canny(g, n=0) == B2F_EINVAL
    assert _canny(g, edges=False) == B2F_EINVAL
    assert _canny(g, nonzero=False) == B2F_EINVAL
    assert _canny(g, ny=0) == B2F_EINVAL
    assert _canny(g) == 0


def test_fhog_batch_refusals_and_empty_geometry():
    from image_b200 import synth
    from image_b200._lib import B2F_EINVAL
    rgb = synth.frame_rgb(620, 64, 64)[None]
    assert _fhog(np.zeros((0, 64, 64, 3), np.uint8), 64, 64) == B2F_EINVAL
    assert _fhog(rgb, 64, 64, n=0) == B2F_EINVAL
    assert _fhog(rgb, 64, 64, cell=0) == B2F_EINVAL
    assert _fhog(rgb, 64, 64, hog=False) == B2F_EINVAL                   # a non-empty output needs somewhere to go
    tiny = synth.frame_rgb(621, 8, 8)[None]
    assert _fhog(tiny, 8, 8, hog=False) == 0                              # empty output: nothing to write
    assert _fhog(rgb, 64, 64) == 0
