"""Chunked / pipelined host batches (b2f_*_batch): cutting a batch into several chunks that overlap
upload, kernels and download must not change a single byte, and concurrent calls on separate
contexts from separate host threads must not disturb each other."""
import threading

import numpy as np
import pytest

pytestmark = pytest.mark.gpu


@pytest.fixture()
def small_chunks():
    from image_b200 import _lib
    lib = _lib.load()
    ctx = _lib.new_context()
    _lib.check(lib.b2f_set_chunk_bytes(ctx, 3 * 150 * 210))       # 3 grey frames (1 RGB frame) per chunk
    yield ctx
    lib.b2f_shutdown(ctx)


def _frames(n, ny=150, nx=210):
    from image_b200 import synth
    return np.stack([synth.frame_shapes(900 + i, ny, nx) for i in range(n)])


def test_canny_batch_chunked_equals_oracle(oracle, small_chunks):
    from image_b200.canny import canny_batch
    f = _frames(8)
    edges, nz = canny_batch(f, ctx=small_chunks)                   # chunks of 1, 3, 3, 1 frames
    one, nz1 = canny_batch(f)                                       # default context: a single chunk
    assert np.array_equal(edges, one) and np.array_equal(nz, nz1)
    for i in (0, 3, 7):
        e, cnt = oracle.canny(f[i])
        assert int(nz[i]) == cnt and np.array_equal(edges[i], e)


def test_harris_batch_chunked_equals_single_chunk(small_chunks):
    from image_b200.harris import harris_batch_u8
    f = _frames(7)
    a = harris_batch_u8(f, cap=4096, raw=True, ctx=small_chunks, threshold=10.0)
    b = harris_batch_u8(f, cap=4096, raw=True, threshold=10.0)
    assert np.array_equal(a[3], b[3]) and a[3].sum() > 0
    for i, m in enumerate(a[3]):          # only the first counts[i] entries of a padded row are written
        for q in range(3):
            assert np.array_equal(a[q][i, :m], b[q][i, :m])


def test_fhog_batch_chunked_equals_oracle(oracle, small_chunks):
    from image_b200 import synth
    from image_b200.dlib import fhog_batch
    f = np.stack([synth.frame_rgb(950 + i, 150, 210) for i in range(5)])
    a = fhog_batch(f, ctx=small_chunks)                             # 5 chunks of one frame
    b = fhog_batch(f)
    assert np.array_equal(a, b)
    for i in (0, 4):
        assert np.array_equal(a[i], oracle.fhog(f[i]))


def test_fhog_tables_follow_the_geometry(oracle):
    """The vote tables are cached per (rows, cols, cell): alternate geometries on one context."""
    from image_b200 import synth
    from image_b200.dlib import fhog_batch
    for (ny, nx, cell) in [(96, 128, 8), (97, 131, 8), (96, 128, 4), (96, 128, 8), (64, 200, 6)]:
        f = synth.frame_rgb(7, ny, nx)[None]
        assert np.array_equal(fhog_batch(f, cell=cell)[0], oracle.fhog(f[0], cell=cell)), (ny, nx, cell)


def test_three_detectors_from_three_threads(oracle):
    from image_b200 import _lib, synth
    from image_b200.canny import canny_batch
    from image_b200.dlib import fhog_batch
    from image_b200.harris import harris_batch_u8
    lib = _lib.load()
    rgb = np.stack([synth.frame_rgb(980 + i, 270, 480) for i in range(6)])
    grey = (rgb.astype(np.uint16).sum(axis=3) // 3).astype(np.uint8)
    ctxs = [_lib.new_context() for _ in range(3)]
    for c in ctxs:
        _lib.check(lib.b2f_set_chunk_bytes(c, 2 * 270 * 480))
    out = {}
    errs = []

    def run(name, fn):
        try:
            for _ in range(3):
                out[name] = fn()
        except Exception as ex:      # surfaced below
            errs.append((name, ex))
    th = [threading.Thread(target=run, args=("harris", lambda: harris_batch_u8(grey, cap=8192, raw=True, ctx=ctxs[0], threshold=10.0))),
          threading.Thread(target=run, args=("canny", lambda: canny_batch(grey, ctx=ctxs[1]))),
          threading.Thread(target=run, args=("fhog", lambda: fhog_batch(rgb, ctx=ctxs[2])))]
    for t in th:
        t.start()
    for t in th:
        t.join()
    assert not errs, errs
    ref_h = harris_batch_u8(grey, cap=8192, raw=True, threshold=10.0)
    assert np.array_equal(out["harris"][3], ref_h[3])
    for i, m in enumerate(ref_h[3]):
        for q in range(3):
            assert np.array_equal(out["harris"][q][i, :m], ref_h[q][i, :m])
    e, cnt = oracle.canny(grey[2])
    assert np.array_equal(out["canny"][0][2], e) and int(out["canny"][1][2]) == cnt
    assert np.array_equal(out["fhog"][5], oracle.fhog(rgb[5]))
    for c in ctxs:
        lib.b2f_shutdown(c)


def test_combined_rgb_batch_equals_the_single_detector_calls(oracle):
    """b2f_features_batch_rgb: one upload of the RGB frames, grey derived on the device; results equal the three
    single-detector batch calls (and therefore the oracle) — also for a frame size whose planes are not 16-byte multiples
    and with a chunk size that cuts the batch."""
    from image_b200 import synth, harris_batch_u8, _lib
    from image_b200.canny import canny_batch
    from image_b200.dlib import fhog_batch
    from image_b200.features import features_batch
    lib = _lib.load()
    for (rows, cols) in [(216, 320), (131, 203)]:
        rgb = np.stack([synth.frame_rgb(40 + i, rows, cols) for i in range(5)])
        grey = (rgb.astype(np.uint16).sum(axis=3) // 3).astype(np.uint8)
        lib.b2f_set_chunk_bytes(_lib.context(), 2 * rows * cols * 3)
        try:
            o = features_batch(rgb, harris=dict(threshold=60.0), canny=dict(s=2.0, low_thr=3.0, high_thr=10.0, accGrad=True), fhog=dict(cell=8))
        finally:
            lib.b2f_set_chunk_bytes(_lib.context(), 48 << 20)
        hs = harris_batch_u8(grey, threshold=60.0)
        e, nz = canny_batch(grey, accGrad=True)
        h = fhog_batch(rgb)
        x, y, s, cnt = o["corners"]
        for i in range(5):
            assert cnt[i] == len(hs[i]["x"]) and np.array_equal(x[i, :cnt[i]], hs[i]["x"]) and np.array_equal(y[i, :cnt[i]], hs[i]["y"])
            assert np.array_equal(s[i, :cnt[i]], hs[i]["strength"])
        assert np.array_equal(o["edges"], e) and np.array_equal(o["nonzero"], nz)
        assert np.array_equal(o["hog"], h)
        ox, oy, os_ = oracle.harris_detect(grey[2], threshold=60.0, gaussian=0, precision=0)
        assert np.array_equal(x[2, :cnt[2]], ox) and np.array_equal(s[2, :cnt[2]], os_)


def test_combined_batch_long_corner_lists_and_uneven_chunk_schedules(oracle):
    """The chunk schedule (half-size first and last chunk) over batch sizes that do not divide, and corner lists longer
    than the head that rides home with each chunk (4096 entries): the lists still equal the single-detector call."""
    from image_b200 import synth, harris_batch_u8, _lib
    from image_b200.canny import canny_batch
    from image_b200.features import features_batch
    lib = _lib.load()
    rows, cols = 480, 800
    for n, per_chunk in [(7, 3), (5, 2), (1, 4), (6, 4), (3, 1)]:
        grey = np.stack([synth.frame_shapes(70 + i, rows, cols) for i in range(n)])
        grey[0] = np.random.default_rng(7).integers(0, 256, (rows, cols), dtype=np.uint8)     # noise: thousands of corners
        lib.b2f_set_chunk_bytes(_lib.context(), per_chunk * rows * cols)
        try:
            o = features_batch(grey, harris=dict(threshold=1.0, sigma_i=1.0), canny=dict(s=2.0, low_thr=3.0, high_thr=10.0, accGrad=True), corner_cap=60000)
        finally:
            lib.b2f_set_chunk_bytes(_lib.context(), 48 << 20)
        hs = harris_batch_u8(grey, threshold=1.0, sigma_i=1.0, cap=60000)
        e, nz = canny_batch(grey, accGrad=True)
        x, y, s, cnt = o["corners"]
        assert cnt[0] > 4096, cnt
        for i in range(n):
            assert cnt[i] == len(hs[i]["x"]) and np.array_equal(x[i, :cnt[i]], hs[i]["x"]) and np.array_equal(y[i, :cnt[i]], hs[i]["y"])
            assert np.array_equal(s[i, :cnt[i]], hs[i]["strength"])
        assert np.array_equal(o["edges"], e) and np.array_equal(o["nonzero"], nz)


def test_surf_batch_chunked_equals_oracle(oracle):
    """b2f_surf_batch / b2f_surf_dev run their frames through a two-deep chunk pipeline (GPU stages of chunk c+1 under the host
    tail of chunk c): 5 frames in chunks of 2, 2, 1 give the oracle's lists, and the same records as one chunk."""
    from image_b200 import synth, _lib
    from image_b200.dlib import surf_batch
    lib = _lib.load()
    rows, cols = 300, 417
    frames = np.stack([synth.frame_blobs(700 + i, rows, cols) for i in range(5)])
    ctx = _lib.new_context()
    try:
        _lib.check(lib.b2f_set_chunk_bytes(ctx, rows * cols * 3))       # SURF takes twice the usual chunk: 2 frames
        rec_a, cnt_a = surf_batch(frames, 10000, 10.0, raw=True, ctx=ctx)
    finally:
        lib.b2f_shutdown(ctx)
    rec_b, cnt_b = surf_batch(frames, 10000, 10.0, raw=True)
    assert np.array_equal(cnt_a, cnt_b) and cnt_a.min() > 0
    for i in range(5):
        assert np.array_equal(rec_a[i, :cnt_a[i]], rec_b[i, :cnt_b[i]])
        ref = oracle.surf(frames[i], 10000, 10.0)
        assert cnt_a[i] == len(ref["x"]) and np.array_equal(rec_a[i, :cnt_a[i], 0], ref["x"]) and np.array_equal(rec_a[i, :cnt_a[i], 4], ref["score"])


def test_surf_flat_frames_rerun_with_a_larger_candidate_capacity(oracle, small_chunks):
    """A constant image makes every interior sample a 3x3x3 'maximum' (ties survive, hessian_pyramid.h:343-356) when the
    threshold is 0: far more candidates than the first capacity guess; the call reruns and returns what dlib returns."""
    from image_b200.dlib import surf_batch
    frames = np.full((3, 150, 210, 3), 90, np.uint8)
    outs = surf_batch(frames, 50, 0.0, ctx=small_chunks)
    ref = oracle.surf(frames[0], 50, 0.0)
    for o in outs:
        assert o["points"] == len(ref["x"]) and np.array_equal(o["x"], ref["x"]) and np.array_equal(o["y"], ref["y"])
