"""The default Harris path (certified: fused fp32 kernel, per-block error bound, tolerant NMS, exact patches) away from its
default parameters, against the oracle bit for bit — lists, order and strengths — through the host entry (float input)
and the u8 batch:
 * sigma_i of every NMS radius the certified path has (2, 3, 5: nms_tolerant_kernel<2|3|5>) and both fused kernel
   instances (sigma_i taps of half-width 3 and 7), with the float32 neighbours of 4/3 and 7/3 (tests/harris_cases.py);
 * other sigma_d, k = 0 (the trace cut still on) and k < 0 (trace cut off), both gradients, a threshold equal to an exact
   strength, tiled frames (equal maxima), sub-pixel fits (quartic: the exact patches' 3x3 neighbourhoods), the output
   strategies, two and three scales, float input ([0, 1], 16-bit, negative, non-integer);
 * the fp32 plane of the sigma_i half-width-3 kernel within its certified bound on every pixel;
 * candidate records that overflow: the host entry's fallback, and the batch entries' counts, which are the true counts
   (B2F_ECAP only when a frame really has more corners than the caller's cap).
Wherever the certified path applies, cert_stats() shows that it ran (candidates grow) and that the bound held
(violations stay 0): a silent fallback to the staged kernels does not pass."""
import ctypes as C

import numpy as np
import pytest

import harris_cases as H

pytestmark = pytest.mark.gpu

F = np.float32
SHAPES = [(32, 32), (31, 64), (33, 47), (64, 200), (270, 480), (541, 963)]


def _stats():
    from image_b200.harris import cert_stats
    return cert_stats()


def _same(got, want, what):
    ox, oy, os_ = want
    assert len(got["x"]) == len(ox), (what, len(got["x"]), len(ox))
    assert np.array_equal(got["x"], ox) and np.array_equal(got["y"], oy), what
    assert np.array_equal(got["strength"], os_), what


def _certified_ran(before, n_oracle, certified, what):
    """After a call: the bound held; where the certified path applies and the frame has corners, it really ran."""
    after = _stats()
    assert after["violations"] == 0, what
    if certified and n_oracle:
        assert after["candidates"] > before["candidates"], ("certified path did not run", what)


def _host(oracle, img, **kw):
    """Host entry (detect_corners: float input, every strategy / precision / scale) against the oracle."""
    from image_b200 import detect_corners
    ny, nx = img.shape
    kw = dict(dict(gaussian=0, precision=0), **kw)
    before = _stats()
    got = detect_corners(np.asarray(img, np.float64).ravel(), nx, ny, **kw)
    want = oracle.harris_detect(img, **kw)
    _same(got, want, (img.shape, kw))
    _certified_ran(before, len(want[0]), H.certified_supported(nx, ny, **kw), (img.shape, kw))
    return want


def _batch(oracle, frames, **kw):
    """harris_batch_u8 on u8 frames [n, ny, nx] against the oracle frame by frame."""
    from image_b200 import harris_batch_u8
    n, ny, nx = frames.shape
    before = _stats()
    outs = harris_batch_u8(frames, cap=nx * ny, **kw)
    tot = 0
    for i in range(n):
        want = oracle.harris_detect(frames[i], **dict(dict(gaussian=0, precision=0), **kw))
        _same(outs[i], want, (frames.shape, i, kw))
        tot += len(want[0])
    _certified_ran(before, tot, H.certified_supported(nx, ny, **kw), (frames.shape, kw))
    return tot


def _adversarial():
    from test_harris_certify_cpu import _frames
    return _frames()


def _tiled():
    from image_b200 import synth
    return np.tile(synth.frame_shapes(32, 64, 96), (4, 4))


# ------------------------------------------------------------------------------------------ parameters


@pytest.mark.parametrize("j", range(len(H.SIGMA_I)), ids=["si%r" % float(s) for s in H.SIGMA_I])
def test_sigma_i_every_window_radius_and_kernel_instance(oracle, j):
    """Every sigma_i, both gradients: a 270x480 frame through the host entry, one frame of the shape list through the u8
    batch (aligned and unaligned widths, below the fused minimum) and a frame just one row taller than the window."""
    from image_b200 import synth
    s = float(H.SIGMA_I[j])
    r = H.nms_radius(s)
    ny, nx = SHAPES[j % len(SHAPES)]
    for grad in (0, 1):
        _host(oracle, synth.frame_shapes(40 + j, 270, 480), threshold=50, sigma_i=s, gradient=grad)
        _batch(oracle, synth.frame_shapes(60 + j, ny, nx)[None], threshold=1.0, sigma_i=s, gradient=grad)
        _batch(oracle, synth.frame_shapes(80 + j, 2 * r + 2, 100)[None], threshold=1.0, sigma_i=s, gradient=grad)
    for ny, nx in SHAPES:
        if H.certified_supported(nx, ny, sigma_i=s):
            break
    else:
        return
    # the radius of this sigma reaches the certified path somewhere in the shape list
    assert _batch(oracle, synth.frame_shapes(90 + j, ny, nx)[None], threshold=1.0, sigma_i=s) > 0


GRID = ([(float(d), si, 0.06) for d in H.SIGMA_D for si in (1.0, 1.3, 2.5)] +
        [(1.15, si, k) for k in H.K for si in (1.2, 2.5)])


@pytest.mark.parametrize("sigma_d,sigma_i,k", GRID)
def test_sigma_d_and_k_on_adversarial_frames(oracle, sigma_d, sigma_i, k):
    """sigma_d, sigma_i and k (zero, negative) on the adversarial frames of the CPU bound check, both gradients, thresholds
    1, 50 and 130; and a threshold equal to one corner's exact strength through the host entry."""
    fr = _adversarial()
    frames = np.stack(list(fr.values()))
    kw = dict(sigma_d=sigma_d, sigma_i=sigma_i, k=k)
    for grad in (0, 1):
        for th in (1.0, 50.0, 130.0):
            _batch(oracle, frames, threshold=th, gradient=grad, **kw)
    _, _, s = oracle.harris_detect(fr["shapes"], threshold=50.0, **kw)
    assert len(s) > 2
    _host(oracle, fr["shapes"], threshold=float(np.sort(s)[len(s) // 2]), **kw)


@pytest.mark.parametrize("sigma_i", [1.0, 1.2, 1.3, 2.5])
@pytest.mark.parametrize("k", [-0.05, -2.0])
def test_corner_tied_with_its_left_neighbour(oracle, sigma_i, k):
    """k < 0 makes straight edges positive ridges of exactly equal values.  The last pixel of such a run can be the maximum
    of its window (ties on the left are allowed) and yet the reference's row scan passes over it (harris.cpp:175-176: it
    walks down the leading run of the row).  The certified path leaves such frames to the staged kernels: count -1 from
    the device entry, the reference's list from the others."""
    import torch
    from image_b200.harris import harris_corners_dev
    img = _adversarial()["step_corner"]
    ny, nx = img.shape
    for grad in (0, 1):
        kw = dict(threshold=1.0, sigma_d=1.15, sigma_i=sigma_i, k=k, gradient=grad)
        _host(oracle, img, **kw)
        _batch(oracle, img[None], **kw)
        want = oracle.harris_detect(img, **kw)
        cap = nx * ny
        xy = torch.zeros((1, cap), dtype=torch.int32, device="cuda")
        st = torch.zeros((1, cap), dtype=torch.float32, device="cuda")
        cnt = torch.zeros(1, dtype=torch.int32, device="cuda")
        harris_corners_dev(torch.from_numpy(img).cuda(), True, 1, nx, ny, cap, xy, st, cnt, **kw)
        torch.cuda.synchronize()
        c = int(cnt[0])
        assert c in (-1, len(want[0])), (grad, c, len(want[0]))
        if c > 0:
            q = xy[0, :c].cpu().numpy()
            assert np.array_equal(q % nx, want[0].astype(np.int64)) and np.array_equal(st[0, :c].cpu().numpy(), want[2])


def test_nms_follows_the_row_scan_on_ridges_of_equal_values(oracle):
    """The staged NMS (every radius kernel) on maps with exact ties at maxima: a ridge of equal values that starts the
    row (the scan walks down all of it and keeps nothing there, although its last pixel is a window maximum), a ridge
    after an ascent (its last pixel is a corner), a plateau.  Lists and counts equal the reference scan's."""
    import torch
    from scipy.ndimage import gaussian_filter
    from image_b200 import harris as Hh
    rng = np.random.default_rng(21)
    differs = 0
    for ny, nx, r in [(64, 200, 2), (64, 200, 3), (80, 300, 5), (40, 97, 1), (64, 200, 7)]:
        R = np.stack([gaussian_filter(rng.standard_normal((ny, nx)), 1.5) * 100 for _ in range(2)]).astype(np.float32)
        R[0, 30, : nx // 3] = 1000
        R[0, 29, : nx // 3] = R[0, 31, : nx // 3] = 900
        R[1, 20, nx // 2: nx // 2 + 30] = 1000
        R[1, 19, nx // 2: nx // 2 + 30] = R[1, 21, nx // 2: nx // 2 + 30] = 900
        R[1, 30:38, 10:40] = 500
        for th in (20.0, -1e9):
            cap = nx * ny
            xy = torch.zeros((2, cap), dtype=torch.int32, device="cuda")
            st = torch.zeros((2, cap), dtype=torch.float32, device="cuda")
            cnt = torch.zeros(2, dtype=torch.int32, device="cuda")
            Hh.harris_nms_dev(torch.from_numpy(R).cuda(), 2, nx, ny, th, r, cap, xy, st, cnt)
            torch.cuda.synchronize()
            for f in range(2):
                ox, oy, os_ = oracle.harris_nms(R[f], th, r)
                differs += len(oracle.harris_nms(R[f], th, r, window=True)[0]) != len(ox)
                n = int(cnt[f])
                assert n == len(ox), (ny, nx, r, th, f, n, len(ox))
                q = xy[f, :n].cpu().numpy()
                assert np.array_equal(q % nx, ox.astype(np.int64)) and np.array_equal(q // nx, oy.astype(np.int64))
                assert np.array_equal(st[f, :n].cpu().numpy(), os_)
    assert differs > 0, "no map where the row scan and the window predicate disagree"


@pytest.mark.parametrize("sigma_i", [1.0, 1.3, 2.5])
def test_threshold_at_an_exact_strength_and_equal_maxima(oracle, sigma_i):
    from image_b200 import synth
    base = synth.frame_shapes(31, 256, 384)
    _, _, s = oracle.harris_detect(base, threshold=50.0, sigma_i=sigma_i)
    th = float(np.sort(s)[len(s) // 2])
    for grad in (0, 1):
        _host(oracle, base, threshold=th, sigma_i=sigma_i, gradient=grad)
        _batch(oracle, base[None], threshold=th, sigma_i=sigma_i, gradient=grad)
        _batch(oracle, _tiled()[None], threshold=50.0, sigma_i=sigma_i, gradient=grad)
        _host(oracle, _tiled().astype(np.float64), threshold=50.0, sigma_i=sigma_i, gradient=grad)


@pytest.mark.parametrize("precision", [0, 1, 2])
@pytest.mark.parametrize("strategy", [0, 1, 2, 3])
def test_subpixel_fits_and_output_strategies(oracle, precision, strategy):
    """Quadratic and quartic fits on the 3x3 neighbourhoods the exact patches return, every strategy, at each certified
    window radius."""
    from image_b200 import synth
    img = synth.frame_shapes(17, 270, 480)
    for s in (1.2, 1.3, 2.5):
        _host(oracle, img, threshold=50, sigma_i=s, precision=precision, strategy=strategy, Nselect=50, cells=5)


@pytest.mark.parametrize("Nscales", [2, 3])
@pytest.mark.parametrize("sigma_i", [2.5, 2.4])
def test_scales(oracle, Nscales, sigma_i):
    """Two and three scales; the second level of sigma_i = 2.4 (1.2) lands on window radius 2."""
    from image_b200 import synth
    img = synth.frame_shapes(19, 541, 963)
    lv = H.levels(963, 541, Nscales, sigma_i)
    assert len(lv) == Nscales and all(H.certified_supported(x, y, sigma_i=s) for x, y, s in lv[-2:])
    assert [H.nms_radius(s) for _, _, s in lv[-2:]] == ([3, 5] if sigma_i == 2.5 else [2, 5])
    for precision in (0, 2):
        _host(oracle, img, threshold=50, sigma_i=sigma_i, Nscales=Nscales, precision=precision)


@pytest.mark.parametrize("sigma_i", [1.2, 1.3, 2.5])
def test_float_input(oracle, sigma_i):
    """A u8 frame in [0, 1] (threshold scaled by 255^-4), in a 16-bit range (threshold by 257^4), minus 128, and plus
    non-integer noise: the bound's M is then the tile's largest |pixel| and the trace cut is off."""
    from image_b200 import synth
    x = synth.frame_shapes(23, 270, 480).astype(np.float64)
    noisy = x + np.random.default_rng(5).uniform(-0.5, 0.5, x.shape)
    for img, th in ((x / 255.0, 50.0 / 255.0 ** 4), (x * 257.0, 50.0 * 257.0 ** 4), (x - 128.0, 50.0), (noisy, 50.0)):
        img = img.astype(np.float32)
        for grad in (0, 1):
            assert len(_host(oracle, img, threshold=th, sigma_i=sigma_i, gradient=grad, precision=2)[0]) > 10


# ------------------------------------------------------------------------------------------ the fp32 plane and its bound


@pytest.mark.parametrize("sigma_i", [1.0, 1.3])
@pytest.mark.parametrize("k", [0.0, 0.15, -0.05])
def test_plane_within_certified_bound_half_width_3_kernel(oracle, sigma_i, k):
    """The fused kernel with sigma_i taps of half-width 3 (sigma_d = 1.15): every pixel of the fp32 plane within the
    certified per-block bound of the oracle's R, for u8 and float input (negative, [0, 1]), aligned and unaligned widths,
    both gradients, on the adversarial frames."""
    import torch
    from image_b200 import harris as Hh
    fr = np.stack(list(_adversarial().values()))
    for nx in (200, 197):
        u8 = np.ascontiguousarray(fr[:, :, :nx])
        n, ny, _ = u8.shape
        for src in (u8, u8.astype(np.float32) - F(128), u8.astype(np.float32) / F(255)):
            is_u8 = src.dtype == np.uint8
            for grad in (0, 1):
                kw = dict(sigma_d=1.15, sigma_i=sigma_i, k=k, gradient=grad)
                d = torch.from_numpy(src).cuda()
                R = torch.empty((n, ny, nx), dtype=torch.float32, device="cuda")
                eps = torch.empty((n, (ny + 7) // 8, (nx + 7) // 8), dtype=torch.float32, device="cuda")
                Hh.harris_response_eps_dev(d, is_u8, n, nx, ny, R, eps, **kw)
                torch.cuda.synchronize()
                R, eps = R.cpu().numpy(), eps.cpu().numpy()
                for i in range(n):
                    Ro, _ = oracle.harris_response(src[i], grad=grad, measure=0, k=k, sigma_d=1.15, sigma_i=sigma_i)
                    e = np.kron(eps[i], np.ones((8, 8), np.float32))[:ny, :nx].astype(np.float64)
                    diff = np.abs(R[i].astype(np.float64) - Ro.astype(np.float64))
                    assert np.all(diff <= e), (nx, src.dtype, grad, i, float((diff / e).max()))


# ------------------------------------------------------------------------------------------ candidate capacity


def _plateaus():
    flat = np.full((64, 64), 90.0)
    shapes = np.full((96, 160), 100.0)
    shapes[20:34, 30:50] = 200.0
    shapes[60:70, 100:140] = 30.0
    return flat, shapes


@pytest.mark.parametrize("sigma_i", [1.0, 1.3, 2.5])
@pytest.mark.parametrize("threshold", [0.0, -1.0])
def test_host_entry_candidate_overflow_falls_back(oracle, sigma_i, threshold):
    """A threshold of 0 or below over plateaus: every flat pixel is a candidate, more than the host entry's records
    ((nx/2+1)(ny/2+1)); the result is still the oracle's (staged fallback), and the candidate counter shows that the
    certified path ran and overflowed (the patch kernel counts min(candidates, records))."""
    from image_b200 import detect_corners
    for img in _plateaus():
        ny, nx = img.shape
        before = _stats()
        got = detect_corners(img.ravel(), nx, ny, threshold=threshold, sigma_i=sigma_i, gaussian=0, precision=0)
        after = _stats()
        _same(got, oracle.harris_detect(img, threshold=threshold, sigma_i=sigma_i), (img.shape, threshold))
        assert after["violations"] == 0
        assert after["candidates"] - before["candidates"] == (nx // 2 + 1) * (ny // 2 + 1)


def _entry(entry, frames, cap, ctx, **kw):
    """One of the three batch entries with Harris on u8 frames [n, ny, nx] (RGB entry: frames [n, ny, nx, 3]):
    (status, x, y, strength, counts)."""
    from image_b200 import _lib
    from image_b200.harris import _params
    lib = _lib.load()
    f = np.ascontiguousarray(frames, dtype=np.uint8)
    n, ny, nx = f.shape[:3]
    x, y, s = (np.zeros((n, cap), np.float32) for _ in range(3))
    cnt = np.zeros(n, np.int32)
    p = _params(kw)
    outs = (cap, _lib.ptr(x), _lib.ptr(y), _lib.ptr(s), _lib.ptr(cnt))
    if entry == "harris":
        rc = lib.b2f_harris_batch_u8(ctx, _lib.ptr(f), n, nx, ny, C.byref(p), *outs)
    elif entry == "grey":
        rc = lib.b2f_features_batch_grey(ctx, _lib.ptr(f), n, nx, ny, C.byref(p), *outs, None, None, None)
    else:
        rc = lib.b2f_features_batch_rgb(ctx, _lib.ptr(f), n, ny, nx, C.byref(p), *outs, None, None, None, 0, 0, 0, None)
    return rc, x, y, s, cnt


@pytest.fixture(scope="module")
def one_frame_chunks():
    from image_b200 import _lib
    lib = _lib.load()
    ctx = _lib.new_context()
    _lib.check(lib.b2f_set_chunk_bytes(ctx, 120 * 160))             # one frame per chunk, grey or RGB
    yield ctx
    lib.b2f_shutdown(ctx)


@pytest.mark.parametrize("entry", ["harris", "grey", "rgb"])
@pytest.mark.parametrize("chunked", [False, True])
@pytest.mark.parametrize("sigma_i", [1.0, 2.5])
def test_batch_counts_are_true_counts_when_candidates_overflow(oracle, one_frame_chunks, entry, chunked, sigma_i):
    """The certified path sizes its candidate records by the caller's cap, and undecided candidates outnumber the kept
    corners on noise at a low threshold.  With cap = the frame's true count the entry returns B2F_OK and the oracle's
    list; with one less it reports B2F_ECAP and the true count.  exact = 0 and 1 agree on status and counts."""
    from image_b200 import _lib, synth
    from image_b200._lib import B2F_ECAP, B2F_OK
    ctx = one_frame_chunks if chunked else _lib.context()
    rng = np.random.default_rng(11)
    if entry == "rgb":
        rgb = np.stack([rng.integers(0, 256, (120, 160, 3)).astype(np.uint8), synth.frame_rgb(12, 120, 160, noise=0),
                        rng.integers(0, 256, (120, 160, 3)).astype(np.uint8)])
        grey = (rgb.astype(np.int32).sum(axis=3) // 3).astype(np.uint8)
        frames = rgb
    else:
        grey = np.stack([rng.integers(0, 256, (120, 160)).astype(np.uint8), synth.frame_shapes(12, 120, 160, noise=0),
                         rng.integers(0, 256, (120, 160)).astype(np.uint8)])
        frames = grey
    kw = dict(threshold=1.0, sigma_i=sigma_i)
    want = [oracle.harris_detect(g, **kw) for g in grey]
    n_true = np.array([len(w[0]) for w in want])
    cap = int(n_true.max())
    assert n_true[1] < cap
    # with room for everything: the oracle's counts; and the frame with the most corners has more candidates than corners,
    # so that cap = its count overflows the records (the next step is not vacuous)
    from image_b200.harris import cert_stats
    rc, x, y, s, cnt = _entry(entry, frames, 160 * 120, ctx, **kw)
    assert rc == B2F_OK and np.array_equal(cnt, n_true)
    before = cert_stats(ctx)
    rc, x, y, s, cnt = _entry(entry, frames[np.argmax(n_true)][None], 160 * 120, ctx, **kw)
    after = cert_stats(ctx)
    assert rc == B2F_OK and cnt[0] == cap and after["kept"] - before["kept"] == cap
    assert after["candidates"] - before["candidates"] > cap
    assert after["violations"] == 0
    for c in (cap, cap - 1):
        res = [_entry(entry, frames, c, ctx, exact=e, **kw) for e in (0, 1)]
        for e, (rc, x, y, s, cnt) in enumerate(res):
            assert np.array_equal(cnt, n_true), (c, e, cnt, n_true)
            assert rc == (B2F_OK if c == cap else B2F_ECAP), (c, e, rc)
            for i in range(len(grey)):
                if n_true[i] <= c:
                    m = n_true[i]
                    assert np.array_equal(x[i, :m], want[i][0]) and np.array_equal(y[i, :m], want[i][1]), (c, e, i)
                    assert np.array_equal(s[i, :m], want[i][2]), (c, e, i)


@pytest.mark.parametrize("is_u8", [True, False])
def test_corners_dev_reports_overflow_never_a_wrong_count(oracle, is_u8):
    """b2f_harris_corners_dev on the certified path: a cap below the candidate count gives -1 (the documented 'records
    overflowed'), never a wrong positive count; a cap of nx*ny gives the oracle's lists."""
    import torch
    from image_b200.harris import harris_corners_dev
    rng = np.random.default_rng(13)
    frames = rng.integers(0, 256, (2, 120, 160)).astype(np.uint8)
    n, ny, nx = frames.shape
    kw = dict(threshold=1.0, sigma_i=1.0)
    want = [oracle.harris_detect(f, **kw) for f in frames]
    src = torch.from_numpy(frames if is_u8 else frames.astype(np.float32)).cuda()
    for cap in (1, 16, len(want[0][0]), nx * ny):
        xy = torch.zeros((n, cap), dtype=torch.int32, device="cuda")
        st = torch.zeros((n, cap), dtype=torch.float32, device="cuda")
        cnt = torch.zeros(n, dtype=torch.int32, device="cuda")
        harris_corners_dev(src, is_u8, n, nx, ny, cap, xy, st, cnt, **kw)
        torch.cuda.synchronize()
        for f in range(n):
            c = int(cnt[f])
            true = len(want[f][0])
            assert c == -1 or c == true, (cap, f, c, true)
            if cap < true:
                assert c == -1, (cap, f, c)
            if cap == nx * ny:
                assert c == true
                q = xy[f, :c].cpu().numpy()
                assert np.array_equal(q % nx, want[f][0].astype(np.int64)) and np.array_equal(q // nx, want[f][1].astype(np.int64))
                assert np.array_equal(st[f, :c].cpu().numpy(), want[f][2])
    assert _stats()["violations"] == 0
