"""The Canny hysteresis kernels on given class maps (b2f_canny_hysteresis_dev, the stage after NMS), compared bit for
bit with two references: the oracle's flood fill from the strong seeds and scipy's 8-connected labelling.  The maps
(tests/hyst_maps.py) are built to hit what the tiled design can get wrong: diagonal links at tile corners, chains
across tens of tiles seeded in one, the limits of the per-tile run encoding, seams that must not link, and many tiny
frames in one call.  Every call writes into a guarded buffer, so stray stores outside the output are caught too."""
import numpy as np
import pytest

import hyst_maps as H

pytestmark = pytest.mark.gpu

SENT = 0x5A           # sentinel byte around the edge map
GUARD = 4096          # bytes of guard on each side (keeps the edge map 16-byte aligned)
NZ_SENT, NZ_GUARD = -7, 64

CASES = list(H.cases(big=True))


def run_stage(maps, offset=0):
    """Upload the maps, run the stage with the edge map at byte `offset` past a 16-byte boundary; check the guards."""
    import torch
    from image_b200.canny import canny_hysteresis_dev
    n, ny, nx = maps.shape
    size = n * ny * nx
    d_cls = torch.from_numpy(np.ascontiguousarray(maps)).cuda()
    buf = torch.full((size + 2 * GUARD + 16,), SENT, dtype=torch.uint8, device="cuda")
    nzb = torch.full((n + 2 * NZ_GUARD,), NZ_SENT, dtype=torch.int32, device="cuda")
    assert buf.data_ptr() % 16 == 0
    torch.cuda.synchronize()
    canny_hysteresis_dev(d_cls, n, nx, ny, buf.data_ptr() + GUARD + offset, nzb.data_ptr() + 4 * NZ_GUARD)
    torch.cuda.synchronize()
    b, z = buf.cpu().numpy(), nzb.cpu().numpy()
    lo = GUARD + offset
    assert (b[:lo] == SENT).all() and (b[lo + size:] == SENT).all(), "bytes written outside the edge map"
    assert (z[:NZ_GUARD] == NZ_SENT).all() and (z[NZ_GUARD + n:] == NZ_SENT).all(), "counts written outside d_nonzero"
    return b[lo:lo + size].reshape(n, ny, nx), z[NZ_GUARD:NZ_GUARD + n]


def check(oracle, cid, maps, edges, nz, expected=None):
    assert set(np.unique(edges).tolist()) <= {0, 255}, cid
    for f in range(maps.shape[0]):
        e_o, n_o = oracle.canny_hysteresis(maps[f])
        e_s, n_s = H.scipy_hysteresis(maps[f])
        assert np.array_equal(e_o, e_s) and n_o == n_s, (cid, f)
        bad = int((edges[f] != e_o).sum())
        assert bad == 0, "%s frame %d: %d pixels differ from the references" % (cid, f, bad)
        assert int(nz[f]) == int((edges[f] == 255).sum()) == n_o, (cid, f, int(nz[f]), n_o)
        assert not edges[f][maps[f] == 0].any(), (cid, f)
        if expected is not None:
            assert np.array_equal(edges[f] == 255, expected[f]), (cid, f)


@pytest.mark.parametrize("family", sorted({c[0] for c in CASES}))
def test_stage_equals_references(oracle, family):
    n = 0
    for fam, cid, maps, expected in CASES:
        if fam == family:
            edges, nz = run_stage(maps)
            check(oracle, cid, maps, edges, nz, expected)
            n += 1
    assert n > 0


def test_families_reach_the_hard_cases():
    """The maps contain what they are meant to test (so that the comparisons above are not vacuous)."""
    by_id = {cid: m for _, cid, m, _ in CASES}
    assert H.longest_single_seed_span(by_id["spiral_seed_far_256x320"][0]) >= 50
    assert H.longest_single_seed_span(by_id["serpentine_v_seed_near_200x333"][0]) >= 50
    for cid, keep in [("diagonal_256x320", ("bl",)), ("anti_diagonal_256x320", ("br",)), ("pairs_200x333", ("bl",)),
                      ("pairs_200x333", ("br",))]:
        m = by_id[cid][0]
        assert not np.array_equal(H.graph_hysteresis(m)[0], H.graph_hysteresis(m, corners=keep)[0]), cid
    assert H.max_components_per_tile(by_id["lattice_96x128"][0]) == 256
    assert H.max_runs_per_row(by_id["checkerboard_70x100"][0]) == 16


@pytest.mark.parametrize("ny,nx,offset", [(96, 128, 1), (33, 32, 1), (40, 48, 7), (70, 100, 0), (70, 100, 3), (31, 33, 1)])
def test_edge_map_alignment(oracle, ny, nx, offset):
    """nx % 16 == 0 with a misaligned d_edges takes the scalar stores of hyst_emit_kernel; so does nx % 16 != 0."""
    rng = np.random.default_rng(ny * 1000 + nx + offset)
    maps = np.concatenate([H.random_maps(rng, 3, ny, nx, 0.45, 0.01), H.checkerboard(ny, nx, True)[None]])
    edges, nz = run_stage(maps, offset)
    check(oracle, (ny, nx, offset), maps, edges, nz)


def test_stage_equals_full_canny_on_nms_classes(oracle):
    """On the class map of a real image the stage gives what canny_batch gives (same kernels after the NMS)."""
    from image_b200 import synth
    from image_b200.canny import canny_batch
    frames = np.stack([synth.frame_shapes(900 + i, 150, 210) for i in range(3)])
    cls = np.stack([oracle.canny(f, stages=True)[3] for f in frames])
    edges, nz = run_stage(cls)
    e_full, nz_full = canny_batch(frames)
    assert np.array_equal(edges, e_full) and np.array_equal(nz, nz_full)


def test_bad_arguments_are_refused():
    import torch
    from image_b200 import _lib
    from image_b200.canny import canny_hysteresis_dev
    d = torch.zeros(64, dtype=torch.uint8, device="cuda")
    z = torch.zeros(2, dtype=torch.int32, device="cuda")
    for n, nx, ny in [(0, 8, 8), (1, 0, 8), (1, 8, -1)]:
        with pytest.raises(_lib.B2FError):
            canny_hysteresis_dev(d, n, nx, ny, d, z)
    with pytest.raises(_lib.B2FError):
        canny_hysteresis_dev(None, 1, 8, 8, d, z)
