"""CPU checks of the hysteresis test maps (tests/hyst_maps.py) and of the two references the GPU tests compare with:
the oracle's flood fill from the strong seeds (orc_canny_hysteresis) and scipy's 8-connected labelling must agree on
every map, each designed map must keep what it was built to keep, and each family must contain the feature it is
there for (long single-seed chains, corner-only contacts that decide a component, the limits of the run encoding)."""
import numpy as np
import pytest

import hyst_maps as H

pytest.importorskip("scipy.ndimage")

CASES = list(H.cases(big=False))


@pytest.mark.parametrize("family", sorted({c[0] for c in CASES}))
def test_flood_fill_and_labelling_agree(oracle, family):
    for fam, cid, maps, expected in CASES:
        if fam != family:
            continue
        for f in range(maps.shape[0]):
            e_o, n_o = oracle.canny_hysteresis(maps[f])
            e_s, n_s = H.scipy_hysteresis(maps[f])
            assert np.array_equal(e_o, e_s), (cid, f)
            assert n_o == n_s == int((e_o == 255).sum()), (cid, f)
            assert not np.any(e_o[maps[f] == 0]), (cid, f)
            if maps[f].size <= 10 ** 5:
                assert np.array_equal(H.graph_hysteresis(maps[f])[0], e_o), (cid, f)
            if expected is not None:
                assert np.array_equal(e_o == 255, expected[f]), (cid, f)


def test_path_family_has_long_single_seed_chains():
    spans = {cid: H.longest_single_seed_span(m[0]) for fam, cid, m, _ in CASES if fam == "path" and ("_seed_far_" in cid or "_seed_near_" in cid)}
    assert len(spans) == 12
    assert min(spans.values()) >= 50, spans                    # every tile of a 70- / 80-tile frame
    cut = [m[0] for fam, cid, m, _ in CASES if fam == "path" and "_cut_" in cid]
    assert all(H.scipy_hysteresis(m)[1] < (m != 0).sum() for m in cut)


def test_corner_families_have_deciding_corner_contacts():
    for fam, cid, m, _ in CASES:
        if fam != "corner":
            continue
        full = H.graph_hysteresis(m[0])[0]
        no_br = H.graph_hysteresis(m[0], corners=("bl",))[0]
        no_bl = H.graph_hysteresis(m[0], corners=("br",))[0]
        if cid.startswith("diagonal") or cid.startswith("pairs"):
            assert not np.array_equal(full, no_br), cid        # a bottom-right corner link decides a component
        if cid.startswith("anti_diagonal") or cid.startswith("pairs"):
            assert not np.array_equal(full, no_bl), cid        # a bottom-left corner link decides a component
    a = H.anti_diagonals(256, 320) != 0
    contacts = a[31:-1:32, 32::32] & a[32::32, 31:-1:32]       # (32i, 32j - 1) - (32i - 1, 32j)
    assert int(contacts.sum()) == 63


def image_features(oracle):
    """The features of the designed Canny images (tests/test_canny_gpu.py), measured on the oracle's class maps."""
    c = oracle.canny(H.spiral_image(), stages=True)[3]
    span = H.longest_single_seed_span(c)
    deciding = []
    for anti, keep in [(False, ("bl",)), (True, ("br",))]:
        c = oracle.canny(H.diagonal_stripes(anti=anti), stages=True)[3]
        deciding.append(int((H.graph_hysteresis(c)[0] != H.graph_hysteresis(c, corners=keep)[0]).sum()))
    c = oracle.canny(H.fine_grating(), s=1.0, low_thr=1.0, high_thr=5.0, stages=True)[3]
    return span, deciding, H.max_runs_per_row(c)


def test_designed_images_reach_the_hard_cases(oracle):
    span, deciding, runs = image_features(oracle)
    assert span >= 50                                          # one weak chain over >= 50 tiles, seeded in one tile
    assert min(deciding) > 0, deciding                         # both corner kinds decide kept pixels
    assert runs >= 10


def test_limit_families_reach_the_encoding_limits():
    by_id = {cid: m for _, cid, m, _ in CASES}
    assert H.max_components_per_tile(by_id["lattice_96x128"][0]) == 256
    assert H.max_runs_per_row(by_id["checkerboard_96x128"][0]) == 16
    fr = by_id["full_rows_96x128"][0]
    assert (fr[0, :32] != 0).all() and H.scipy_hysteresis(fr)[1] > 0
    cb = by_id["checkerboard_96x128"]
    assert H.scipy_hysteresis(cb[0])[1] == int((cb[0] != 0).sum())   # one component, held by diagonals only
    assert H.scipy_hysteresis(cb[1])[1] == 0
