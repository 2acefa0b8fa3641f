"""The oracle's ContourDetector and LSD front ends against the reference build's frozen outputs on the adversarial frame
families of frontend_cases.py (tests/golden/frontend_digests.json, tests/golden/make_golden_frontend.py), and checks
that each family really contains the case it is meant to test, so that the GPU comparisons are not vacuous."""
import json
import os

import numpy as np
import pytest

import frontend_cases as fc

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LSD = {cid: (fam, img, p) for fam, cid, img, p in fc.lsd_cases()}
CONTOUR = {cid: (fam, img, s) for fam, cid, img, s in fc.contour_cases()}


@pytest.fixture(scope="module")
def frontend_digests():
    with open(os.path.join(ROOT, "tests", "golden", "frontend_digests.json")) as f:
        return json.load(f)


def test_every_case_is_pinned(frontend_digests):
    keys = {"lsd/%s/%s" % (fam, cid) for cid, (fam, _, _) in LSD.items()}
    keys |= {"contour/%s/%s" % (fam, cid) for cid, (fam, _, _) in CONTOUR.items()}
    assert len(keys) == len(LSD) + len(CONTOUR) and keys == set(frontend_digests)


@pytest.mark.parametrize("family", sorted({fam for fam, _, _ in LSD.values()}))
def test_lsd_oracle_reproduces_the_reference(oracle, frontend_digests, family):
    for cid, (fam, img, p) in LSD.items():
        if fam == family:
            got = fc.lsd_digests(oracle, fc.lsd_oracle(oracle, img, p))
            assert got == frontend_digests["lsd/%s/%s" % (fam, cid)], cid


@pytest.mark.parametrize("family", sorted({fam for fam, _, _ in CONTOUR.values()}))
def test_contour_oracle_reproduces_the_reference(oracle, frontend_digests, family):
    for cid, (fam, img, s) in CONTOUR.items():
        if fam == family:
            got = fc.contour_digests(oracle, fc.contour_oracle(oracle, img, s))
            assert got == frontend_digests["contour/%s/%s" % (fam, cid)], cid


def _lsd(oracle, cid):
    fam, img, p = LSD[cid]
    s, a, m, lst = fc.lsd_oracle(oracle, img, p)
    nd = a[:-1, :-1] == -1024.0
    max_grad = m[:-1, :-1][~nd].max(initial=0.0)
    return p, m[:-1, :-1], nd, max_grad, fc.bucket_of(m, max_grad, p["n_bins"]), lst


def test_lsd_families_reach_the_hard_cases(oracle):
    for cid in ("shapes01_120x160", "const7_120x160", "flat_and_low_noise_120x160", "quant_huge_150x210"):
        p, m, nd, max_grad, b, lst = _lsd(oracle, cid)
        assert nd.all() and max_grad == 0.0, cid
        # positive moduli are where a saturating conversion of +inf would move pixels to the top bucket
        assert (m > 0).any(), cid
    for cid in ("shapes01_120x160", "flat_and_low_noise_120x160"):
        m = _lsd(oracle, cid)[1]
        assert (m == 0).any() and (m > 0).any(), cid
    m = _lsd(oracle, "quant0_150x210")[1]
    assert 0 < (m == 0).sum() < m.size
    # one bucket holding more than 90 % of a list that spans at least 20 chunks; pixels at exactly max_grad (q == n_bins)
    for cid in ("ramp_x_1960x85", "ramp_diag_500x640"):
        p, m, nd, max_grad, b, lst = _lsd(oracle, cid)
        top = np.bincount(b.ravel(), minlength=p["n_bins"]).max()
        assert len(lst) >= 20 * fc.CHUNK and top > 0.9 * len(lst), cid
        assert (m == max_grad).sum() > 1 and not nd.all(), cid
    b = _lsd(oracle, "two_slopes_420x600")[4]
    assert 2 <= len(np.unique(b)) <= 16
    for k in (1, 8):
        for d in (-1, 0, 1):
            assert len(_lsd(oracle, "ramp_list_%d" % (fc.CHUNK * k + d))[5]) == fc.CHUNK * k + d
    # more than 1024 buckets in use, and buckets below the first 1024 from the top occupied
    for nb in (1025, 2048, 3000, 4096):
        p, m, nd, max_grad, b, lst = _lsd(oracle, "shapes_noise_333x517_bins%d" % nb)
        assert (b < nb - 1024).any() and (nb == 1025 or len(np.unique(b)) > 1024), nb
    # the sampler: the 63-tap kernel, scaled sizes of 2, and mirrors that wrap more than once (h >= 2 * size)
    assert fc.lsd_halfwidth(0.8, 6.6) == 31 and fc.lsd_halfwidth(0.8, 6.7) == 32
    for cid in ("Y3_wrap_3x40", "X2_wrap_40x2", "Y1_wrap_1x33", "X1_wrap_30x1", "2x2_wrap"):
        _, img, p = LSD[cid]
        assert fc.lsd_halfwidth(p["scale"], p["sigma_scale"]) >= 2 * min(img.shape), cid
    for cid in ("M2_2x40", "N2_40x3", "Y1_wrap_1x33", "X1_wrap_30x1"):
        _, img, p = LSD[cid]
        assert min(fc.lsd_size(img.shape[0], p["scale"]), fc.lsd_size(img.shape[1], p["scale"])) == 2, cid


def test_contour_families_reach_the_hard_cases(oracle):
    def run(cid):
        _, img, s = CONTOUR[cid]
        return fc.contour_oracle(oracle, img, s)
    # a 1-px checkerboard at sigma 0.3: the comparisons are ties that the epsilon guard decides, no edge point
    g, e = run("checker1_64x80_s0.3")
    guarded, above = fc.guard_straddles(g)
    assert len(e["idx"]) == 0 and guarded > 100
    # exact ties between min(L, R) and min(U, D) that decide the direction of the offset
    assert fc.diagonal_ties(run("dots128_every12_120x160_s1.5")[0]) > 100
    # the densest lattice is above the host entry's record capacity (X*Y/2), the other below it
    for cid, lo, hi in (("dots3x4_120x160", 0.5, 1.0), ("dots4x2_120x160", 0.3, 0.5)):
        n = len(run(cid)[1]["idx"])
        assert lo * 120 * 160 < n <= hi * 120 * 160, (cid, n)
    # the epsilon guard decides comparisons, and others are above it
    for cid in ("scaled1e-12_100x140", "scaled3e-13_noise_100x140"):
        guarded, above = fc.guard_straddles(run(cid)[0])
        assert guarded > 100 and above > 100, cid
    assert (CONTOUR["negative_100x140"][1] < 0).any()
    # 65 taps, and frames narrower than the half width (the mirror wraps more than once)
    assert fc.contour_offset(8.6) == 32 and fc.contour_offset(8.61) == 33
    for cid, (fam, img, s) in CONTOUR.items():
        if cid.startswith("narrow_") or cid == "taps65_3x40":
            assert fc.contour_offset(s) >= 2 * min(img.shape), cid
    assert sum(len(run(cid)[1]["idx"]) > 0 for cid in CONTOUR if cid.startswith("narrow_")) >= 2
