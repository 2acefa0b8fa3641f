"""GPU parity of the ContourDetector and LSD front ends on the adversarial frame families of frontend_cases.py, bit for
bit against the oracle (which test_frontend_cases_cpu.py pins to the reference build on the same frames).

LSD: the sampled plane, the modulus, the NOTDEF pattern and the bucket list of the host entry and of the device entry
(u8 and double frames), on frames without a defined gradient, single-bucket ramps over many chunks, lists of 2048 k - 1,
2048 k and 2048 k + 1 elements, 1025-4096 buckets, scales 0.3-1.7, the 63-tap kernel and frames whose mirror wraps more
than once; mixed frames in one device batch; the error paths.  Contour: the blurred plane and the edge-point records of
the host, batch and device entries on ties, plateaus, lattices, frames around the epsilon guard, the 65-tap kernel and
frames narrower than the half width; record capacity overflow into guarded buffers; the error path."""
import ctypes as C

import numpy as np
import pytest

import frontend_cases as fc

pytestmark = pytest.mark.gpu

LSD = list(fc.lsd_cases())
CONTOUR = list(fc.contour_cases())
G = 64                      # guard elements on each side of a device or host output
I_SENT, D_SENT = -7, -7.5


# ------------------------------------------------------------------------------------------ LSD

def check_lsd(cid, o, ref):
    s, a, m, lst = ref
    assert np.array_equal(o["scaled"], s), "%s: sampled plane" % cid
    assert np.array_equal(o["modgrad"], m), "%s: modulus" % cid
    nd = a == -1024.0
    assert np.array_equal(o["angles"] == -1024.0, nd), "%s: NOTDEF pattern" % cid
    assert np.max(np.abs(o["angles"][~nd] - a[~nd]), initial=0.0) < 1e-12, "%s: angles" % cid
    assert len(o["list"]) == len(lst), cid
    bad = np.flatnonzero(o["list"] != lst)
    assert bad.size == 0, "%s: bucket list differs at %d of %d positions, first %d" % (cid, bad.size, len(lst), bad[0])


def lsd_dev(frames, p):
    """The device entry on frames [n, Y, X] (u8 or double), with the list in a guarded buffer."""
    import torch
    from image_b200.lsd import lsd_front_dev
    n, Y, X = frames.shape
    N, M = fc.lsd_size(X, p["scale"]), fc.lsd_size(Y, p["scale"])
    total = (N - 1) * (M - 1)
    d = torch.from_numpy(np.ascontiguousarray(frames)).cuda()
    ang = torch.empty((n, M, N), dtype=torch.float64, device="cuda")
    mod, sc = torch.empty_like(ang), torch.empty_like(ang)
    buf = torch.full((n * total + 2 * G,), I_SENT, dtype=torch.int32, device="cuda")
    lsd_front_dev(d, frames.dtype == np.uint8, n, X, Y, ang, mod, buf.data_ptr() + 4 * G, d_scaled=sc, **p)
    torch.cuda.synchronize()
    b = buf.cpu().numpy()
    assert (b[:G] == I_SENT).all() and (b[G + n * total:] == I_SENT).all(), "list written outside its buffer"
    lst = b[G:G + n * total].reshape(n, total)
    return [dict(scaled=sc[i].cpu().numpy(), angles=ang[i].cpu().numpy(), modgrad=mod[i].cpu().numpy(), list=lst[i])
            for i in range(n)]


@pytest.mark.parametrize("family", sorted({c[0] for c in LSD}))
def test_lsd_family_equals_the_oracle(oracle, family):
    from image_b200.lsd import lsd_front
    n = 0
    for fam, cid, img, p in LSD:
        if fam != family:
            continue
        ref = fc.lsd_oracle(oracle, img, p)
        Y, X = img.shape
        check_lsd(cid + " host", lsd_front(img.astype(np.float64).ravel(), X, Y, want_scaled=True, **p), ref)
        check_lsd(cid + " dev f64", lsd_dev(img.astype(np.float64)[None], p)[0], ref)
        if fc.is_u8(img):
            check_lsd(cid + " dev u8", lsd_dev(img[None], p)[0], ref)
        n += 1
    assert n > 0


def test_lsd_mixed_frames_in_one_device_batch(oracle):
    """Frames without a defined angle next to ordinary ones: max_grad and the buckets are per frame."""
    by_id = {cid: (img, p) for _, cid, img, p in LSD}
    p = by_id["shapes_120x160"][1]
    u8 = ["const7_120x160", "shapes_120x160", "flat_and_low_noise_120x160", "const0_120x160", "shapes_120x160"]
    frames = np.stack([by_id[c][0] for c in u8])
    for cid, o in zip(u8, lsd_dev(frames, p)):
        check_lsd(cid + " u8 batch", o, fc.lsd_oracle(oracle, by_id[cid][0], p))
    f64 = ["shapes_120x160", "shapes01_120x160", "quant0_150x210"]
    frames = np.stack([by_id[c][0].astype(np.float64)[:120, :160] for c in f64])
    for cid, img, o in zip(f64, frames, lsd_dev(frames, p)):
        check_lsd(cid + " f64 batch", o, fc.lsd_oracle(oracle, img, p))


def test_lsd_rejects_what_the_library_does_not_serve(oracle):
    from image_b200 import synth
    from image_b200._lib import B2F_EINVAL, B2F_EUNSUP, B2FError
    from image_b200.lsd import lsd_front
    img = synth.frame_shapes(40, 60, 80).astype(np.float64)
    for kw, code in [(dict(n_bins=4097), B2F_EINVAL), (dict(n_bins=0), B2F_EINVAL), (dict(n_bins=-3), B2F_EINVAL),
                     (dict(sigma_scale=6.7), B2F_EUNSUP)]:
        with pytest.raises(B2FError) as e:
            lsd_front(img.ravel(), 80, 60, **kw)
        assert e.value.code == code, kw
        with pytest.raises(B2FError) as e:
            lsd_dev(img[None], fc.lsd_params(**kw))
        assert e.value.code == code, kw
    for Y, X in ((1, 40), (40, 1)):                      # scaled size 1: the library refuses it
        f = synth.frame_shapes(41, Y, X).astype(np.float64)
        with pytest.raises(B2FError) as e:
            lsd_front(f.ravel(), X, Y)
        assert e.value.code == B2F_EUNSUP, (Y, X)
    # the context still works after the refusals
    o = lsd_front(img.ravel(), 80, 60, want_scaled=True, n_bins=4096, sigma_scale=6.6)
    check_lsd("after the refusals", o, fc.lsd_oracle(oracle, img, fc.lsd_params(n_bins=4096, sigma_scale=6.6)))


# ------------------------------------------------------------------------------------------ contour

def check_edges(cid, o, r, n=None):
    n = len(r["idx"]) if n is None else n
    assert len(o["idx"]) == n, "%s: %d edge points, oracle %d" % (cid, len(o["idx"]), len(r["idx"]))
    for key in fc.EDGE_KEYS:
        assert np.array_equal(o[key], r[key][:n]), "%s: %s" % (cid, key)


def contour_dev(frames, sigma, cap):
    """The device entry on frames [n, Y, X] (u8 or double); every output sits in a guarded buffer, and the part of a
    frame's record slots past its count must stay untouched."""
    import torch
    from image_b200.contour import contour_edge_points_dev
    n, Y, X = frames.shape
    d = torch.from_numpy(np.ascontiguousarray(frames)).cuda()
    idx = torch.full((n * cap + 2 * G,), I_SENT, dtype=torch.int32, device="cuda")
    val = [torch.full((n * cap + 2 * G,), D_SENT, dtype=torch.float64, device="cuda") for _ in range(4)]
    cnt = torch.full((n + 2 * G,), I_SENT, dtype=torch.int32, device="cuda")
    gauss = torch.empty((n, Y, X), dtype=torch.float64, device="cuda")
    contour_edge_points_dev(d, frames.dtype == np.uint8, n, X, Y, cap, idx.data_ptr() + 4 * G,
                            *[v.data_ptr() + 8 * G for v in val], cnt.data_ptr() + 4 * G, d_gauss=gauss, sigma=sigma or 0.0)
    torch.cuda.synchronize()
    counts = cnt.cpu().numpy()
    assert (counts[:G] == I_SENT).all() and (counts[G + n:] == I_SENT).all(), "counts written outside d_counts"
    arrs = [idx.cpu().numpy()] + [v.cpu().numpy() for v in val]
    outs = []
    for f in range(n):
        m = min(int(counts[G + f]), cap)
        rec = {}
        for key, a, sent in zip(fc.EDGE_KEYS, arrs, (I_SENT,) + (D_SENT,) * 4):
            assert (a[:G] == sent).all() and (a[G + n * cap:] == sent).all(), "%s written outside its buffer" % key
            row = a[G + f * cap:G + (f + 1) * cap]
            assert (row[m:] == sent).all(), "%s written past the frame's count" % key
            rec[key] = row[:m].copy()
        outs.append(rec)
    return outs, counts[G:G + n], gauss.cpu().numpy()


def contour_batch_raw(frames, sigma, cap):
    """b2f_contour_edge_points_batch_u8 into guarded host buffers -> (status, counts, records per frame)."""
    from image_b200 import _lib
    lib = _lib.load()
    n, Y, X = frames.shape
    idx = np.full(n * cap + 2 * G, I_SENT, np.int32)
    val = [np.full(n * cap + 2 * G, D_SENT) for _ in range(4)]
    cnt = np.full(n + 2 * G, I_SENT, np.int32)
    off = lambda a: C.c_void_p(a.ctypes.data + a.itemsize * G)            # noqa: E731
    rc = lib.b2f_contour_edge_points_batch_u8(_lib.context(), _lib.ptr(np.ascontiguousarray(frames)), n, X, Y, float(sigma or 0.0),
                                              cap, off(idx), *[off(v) for v in val], off(cnt))
    assert (cnt[:G] == I_SENT).all() and (cnt[G + n:] == I_SENT).all()
    outs = []
    for f in range(n):
        m = min(int(cnt[G + f]), cap)
        rec = {}
        for key, a, sent in zip(fc.EDGE_KEYS, [idx] + val, (I_SENT,) + (D_SENT,) * 4):
            assert (a[:G] == sent).all() and (a[G + n * cap:] == sent).all(), "%s written outside its buffer" % key
            row = a[G + f * cap:G + (f + 1) * cap]
            assert (row[m:] == sent).all(), "%s written past the frame's count" % key
            rec[key] = row[:m].copy()
        outs.append(rec)
    return rc, cnt[G:G + n], outs


@pytest.mark.parametrize("family", sorted({c[0] for c in CONTOUR}))
def test_contour_family_equals_the_oracle(oracle, family):
    from image_b200._lib import B2F_ECAP, B2F_OK, B2FError
    from image_b200.contour import contour_edge_points
    n = 0
    for fam, cid, img, sigma in CONTOUR:
        if fam != family:
            continue
        g, r = fc.contour_oracle(oracle, img, sigma)
        Y, X = img.shape
        if len(r["idx"]) <= X * Y // 2:
            o = contour_edge_points(img.astype(np.float64).ravel(), X, Y, sigma=sigma or 0.0, want_gauss=True)
            assert np.array_equal(o["gauss"], g), "%s: blurred plane" % cid
            check_edges(cid + " host", o, r)
        else:                                            # more edge points than the host entry's records hold
            with pytest.raises(B2FError) as e:
                contour_edge_points(img.astype(np.float64).ravel(), X, Y, sigma=sigma or 0.0)
            assert e.value.code == B2F_ECAP, cid
        frames = img[None] if not fc.is_u8(img) else np.stack([img, img[::-1]])
        refs = [r] + [fc.contour_oracle(oracle, f, sigma)[1] for f in frames[1:]]
        outs, counts, gauss = contour_dev(frames, sigma, X * Y)
        assert np.array_equal(gauss[0], g), "%s: blurred plane (dev)" % cid
        for f, (o, rr) in enumerate(zip(outs, refs)):
            assert counts[f] == len(rr["idx"]), cid
            check_edges("%s dev %s frame %d" % (cid, img.dtype, f), o, rr)
        if fc.is_u8(img):                                # the u8 entries give the records of the double host form
            outs, _, _ = contour_dev(frames.astype(np.float64), sigma, X * Y)
            rc, counts, bouts = contour_batch_raw(frames, sigma, X * Y)
            assert rc == B2F_OK, cid
            for f, rr in enumerate(refs):
                assert counts[f] == len(rr["idx"]), cid
                check_edges("%s dev f64 frame %d" % (cid, f), outs[f], rr)
                check_edges("%s batch frame %d" % (cid, f), bouts[f], rr)
        n += 1
    assert n > 0


@pytest.mark.parametrize("cap", [1, 777, 9047, 9048])
def test_contour_record_capacity(oracle, cap):
    """The batch and device entries with fewer record slots than edge points: true counts, the first `cap` records,
    B2F_ECAP from the batch entry, and nothing written outside the slots."""
    from image_b200._lib import B2F_ECAP, B2F_OK
    by_id = {cid: img for _, cid, img, _ in CONTOUR}
    frames = np.stack([by_id["dots4x2_120x160"], by_id["dots3x4_120x160"], by_id["quantised_120x160"]])
    refs = [fc.contour_oracle(oracle, f, None)[1] for f in frames]
    rc, counts, outs = contour_batch_raw(frames, None, cap)
    assert rc == (B2F_OK if all(len(r["idx"]) <= cap for r in refs) else B2F_ECAP)
    douts, dcounts, _ = contour_dev(frames, None, cap)
    for f, r in enumerate(refs):
        assert counts[f] == dcounts[f] == len(r["idx"]), f
        check_edges("batch frame %d" % f, outs[f], r, min(cap, len(r["idx"])))
        check_edges("dev frame %d" % f, douts[f], r, min(cap, len(r["idx"])))


def test_contour_rejects_a_kernel_beyond_65_taps(oracle):
    from image_b200 import synth
    from image_b200._lib import B2F_EUNSUP, B2FError
    from image_b200.contour import contour_edge_points, contour_edge_points_batch
    img = synth.frame_shapes(42, 40, 60)
    with pytest.raises(B2FError) as e:
        contour_edge_points(img.astype(np.float64).ravel(), 60, 40, sigma=8.61)
    assert e.value.code == B2F_EUNSUP
    with pytest.raises(B2FError) as e:
        contour_edge_points_batch(img[None], sigma=8.61)
    assert e.value.code == B2F_EUNSUP
    o = contour_edge_points(img.astype(np.float64).ravel(), 60, 40, sigma=8.6, want_gauss=True)
    g, r = fc.contour_oracle(oracle, img, 8.6)
    assert np.array_equal(o["gauss"], g)
    check_edges("after the refusal", o, r)
