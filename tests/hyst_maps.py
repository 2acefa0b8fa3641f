"""Seeded class maps for testing Canny hysteresis on its own, and two plain references for it.

A class map is uint8 [n, ny, nx]: 0 = no edge, 2 = strong edge, any other value = weak edge (the NMS stage
only writes 1, but the hysteresis must treat 3..255 as weak too).  The families aim at what the tiled
hysteresis of image_b200/csrc/canny.cu can get wrong: 32x32 tile seams and corners, long chains across many
tiles, the limits of the per-tile run encoding, frame boundaries in a batch, and many tiny frames per call.

`cases()` lists every map as (family, case id, map, expected-or-None).  `expected` is a handle on what the
map was built to show (the pixels that must be kept), checked against both references by the CPU suite.
"""
import numpy as np

T = 32                                  # hysteresis tile edge

# ------------------------------------------------------------------------------------------ references


def scipy_hysteresis(cls):
    """8-connected labelling of the edge pixels (scipy.ndimage.label); a label is kept iff it holds a class-2 pixel.
    cls: [ny, nx] -> (edges uint8 0/255, number of 255s)."""
    from scipy import ndimage
    lab, n = ndimage.label(cls != 0, structure=np.ones((3, 3), int))
    keep = np.zeros(n + 1, bool)
    keep[np.unique(lab[cls == 2])] = True
    keep[0] = False
    e = np.where(keep[lab], 255, 0).astype(np.uint8)
    return e, int(keep[lab].sum())


def graph_hysteresis(cls, corners=("br", "bl")):
    """Hysteresis on an explicit pixel graph (scipy.sparse.csgraph), with the option of leaving out the diagonal links
    that cross a tile corner: 'br' = (x, y)-(x+1, y+1) with x % 32 == 31 and y % 32 == 31, 'bl' = (x, y)-(x-1, y+1)
    with x % 32 == 0 and y % 32 == 31.  With both kinds kept this is plain 8-connected hysteresis."""
    from scipy.sparse import coo_matrix
    from scipy.sparse.csgraph import connected_components
    ny, nx = cls.shape
    ed = cls != 0
    idx = np.full((ny, nx), -1, np.int64)
    idx[ed] = np.arange(int(ed.sum()))
    yy, xx = np.mgrid[0:ny, 0:nx]
    a, b = [], []
    for dy, dx, kind in [(0, 1, None), (1, 0, None), (1, 1, "br"), (1, -1, "bl")]:
        ys, xs = slice(0, ny - dy), slice(max(0, -dx), nx - max(0, dx))
        yt, xt = slice(dy, ny), slice(max(0, dx), nx - max(0, -dx))
        m = ed[ys, xs] & ed[yt, xt]
        if kind is not None and kind not in corners:
            cx = (xx[ys, xs] % T == T - 1) if dx == 1 else (xx[ys, xs] % T == 0)
            m &= ~(cx & (yy[ys, xs] % T == T - 1))
        a.append(idx[ys, xs][m]); b.append(idx[yt, xt][m])
    nv = int(ed.sum())
    out = np.zeros((ny, nx), np.uint8)
    if nv == 0:
        return out, 0
    a, b = np.concatenate(a), np.concatenate(b)
    g = coo_matrix((np.ones(a.size, np.int8), (a, b)), shape=(nv, nv))
    _, lab = connected_components(g, directed=False)
    keep = np.zeros(lab.max() + 1, bool)
    keep[lab[idx[cls == 2]]] = True
    out[ed] = np.where(keep[lab], 255, 0)
    return out, int((out == 255).sum())


# ------------------------------------------------------------------------------------------ measures of a map


def tile_of(ny, nx):
    """Tile number (ty * TX + tx) of every pixel."""
    TX = -(-nx // T)
    yy, xx = np.mgrid[0:ny, 0:nx]
    return (yy // T) * TX + xx // T


def longest_single_seed_span(cls):
    """Over the kept components whose class-2 pixels all lie in ONE tile: the largest number of tiles a component touches."""
    from scipy import ndimage
    ny, nx = cls.shape
    lab, n = ndimage.label(cls != 0, structure=np.ones((3, 3), int))
    if n == 0:
        return 0
    tl = tile_of(ny, nx)
    nt = int(tl.max()) + 1
    sel = lab > 0
    span = np.bincount(np.unique(lab[sel].astype(np.int64) * nt + tl[sel]) // nt, minlength=n + 1)
    st = cls == 2
    seeds = np.bincount(np.unique(lab[st].astype(np.int64) * nt + tl[st]) // nt, minlength=n + 1)
    ok = seeds == 1
    return int(span[ok].max()) if ok.any() else 0


def max_components_per_tile(cls):
    """The largest number of 8-connected components of edge pixels inside one 32x32 tile (components cut at seams)."""
    from scipy import ndimage
    ny, nx = cls.shape
    TY, TX = -(-ny // T), -(-nx // T)
    pad = np.zeros((TY * T, TX * T), bool)
    pad[:ny, :nx] = cls != 0
    tiles = pad.reshape(TY, T, TX, T).transpose(0, 2, 1, 3).reshape(TY * TX, T, T)
    st = np.zeros((3, 3, 3), int)
    st[1] = 1                                           # no links between tiles
    lab, n = ndimage.label(tiles, structure=st)
    per = [len(np.unique(lab[i][lab[i] > 0])) for i in range(TY * TX)]
    return max(per) if per else 0


def max_runs_per_row(cls):
    """The largest number of runs of edge pixels in one 32-pixel row of a tile."""
    ny, nx = cls.shape
    TX = -(-nx // T)
    b = np.zeros((ny, TX, T), bool)
    b.reshape(ny, TX * T)[:, :nx] = cls != 0
    prev = np.zeros_like(b)
    prev[..., 1:] = b[..., :-1]
    return int((b & ~prev).sum(axis=2).max())


# ------------------------------------------------------------------------------------------ generators


def random_maps(rng, n, ny, nx, density, strong_frac):
    """Edges with probability `density`; each edge strong with probability `strong_frac`; a quarter of the weak ones
    carry a byte in 3..255 instead of 1."""
    e = rng.random((n, ny, nx)) < density
    s = e & (rng.random((n, ny, nx)) < strong_frac)
    w = np.where(rng.random((n, ny, nx)) < 0.25, rng.integers(3, 256, (n, ny, nx)), 1)
    return np.where(s, 2, np.where(e, w, 0)).astype(np.uint8)


def serpentine_path(ny, nx):
    """A 1-pixel path over rows 0, 2, 4, ... joined alternately at the right and the left border; it visits every tile."""
    path = []
    for k, y in enumerate(range(0, ny, 2)):
        xs = range(nx) if k % 2 == 0 else range(nx - 1, -1, -1)
        path += [(y, x) for x in xs]
        if y + 2 < ny:
            path.append((y + 1, nx - 1 if k % 2 == 0 else 0))
    return path


def spiral_path(ny, nx):
    """An inward rectangular spiral, one empty pixel between its rings (a turtle that keeps one pixel of clearance)."""
    seen = np.zeros((ny, nx), bool)
    dirs = [(0, 1), (1, 0), (0, -1), (-1, 0)]
    y, x, d = 0, 0, 0
    seen[0, 0] = True
    path = [(0, 0)]

    def free(yy, xx):
        return 0 <= yy < ny and 0 <= xx < nx and not seen[yy, xx]

    def can(yy, xx, dd):
        cy, cx = yy + dirs[dd][0], xx + dirs[dd][1]
        if not free(cy, cx):
            return False
        fy, fx = cy + dirs[dd][0], cx + dirs[dd][1]      # keep one pixel of clearance ahead
        return not (0 <= fy < ny and 0 <= fx < nx and seen[fy, fx])

    while True:
        if not can(y, x, d):
            d = (d + 1) % 4
            if not can(y, x, d):
                break
        y, x = y + dirs[d][0], x + dirs[d][1]
        seen[y, x] = True
        path.append((y, x))
    return path


def path_variants(path, ny, nx):
    """The four variants of a 1-pixel path: (name, map, expected kept mask)."""
    def draw(pts, seed):
        m = np.zeros((ny, nx), np.uint8)
        if pts:
            yy, xx = np.array(pts).T
            m[yy, xx] = 1
        if seed is not None:
            m[seed] = 2
        return m
    allp = draw(path, None) != 0
    out = [("seed_far", draw(path, path[-1]), allp), ("seed_near", draw(path, path[0]), allp),
           ("no_seed", draw(path, None), np.zeros_like(allp))]
    # cut: a pixel in the middle of a straight stretch, so that nothing else bridges the gap
    i = len(path) // 2
    while not all(path[j][0] == path[i][0] for j in range(i - 2, i + 3)) and \
            not all(path[j][1] == path[i][1] for j in range(i - 2, i + 3)):
        i += 1
    m = draw(path[:i] + path[i + 1:], path[-1])
    out.append(("cut", m, draw(path[i + 1:], None) != 0))
    return out


def diagonal_lines(ny, nx):
    """45-degree lines y = x + 32k: every link between tiles is a bottom-right tile corner.  Every other line has a
    strong pixel at its upper end, the rest none."""
    yy, xx = np.mgrid[0:ny, 0:nx]
    d = yy - xx
    m = np.where(d % T == 0, 1, 0).astype(np.uint8)
    for k, dd in enumerate(sorted(set(d[m != 0].tolist()))):
        if k % 2 == 0:
            y0 = max(dd, 0)
            m[y0, y0 - dd] = 2
    return m


def anti_diagonals(ny, nx):
    """Anti-diagonals x + y = 31 (mod 32): every link between tiles is a bottom-left tile corner.  Every other line has
    a strong pixel at its upper (right) end."""
    yy, xx = np.mgrid[0:ny, 0:nx]
    s = xx + yy
    m = np.where(s % T == T - 1, 1, 0).astype(np.uint8)
    for k, ss in enumerate(sorted(set(s[m != 0].tolist()))):
        if k % 2 == 0:
            x0 = min(ss, nx - 1)
            m[ss - x0, x0] = 2
    return m


def corner_pairs(ny, nx):
    """A diagonal pixel pair at every inner tile corner, in the four orientations in turn (bottom-right pair with the
    strong pixel above-left or below-right, bottom-left pair with it above-right or below-left)."""
    m = np.zeros((ny, nx), np.uint8)
    k = 0
    for Y in range(T, ny, T):
        for X in range(T, nx, T):
            if k % 4 < 2:
                a, b = (Y - 1, X - 1), (Y, X)            # "\" : the bottom-right corner of the upper-left tile
            else:
                a, b = (Y - 1, X), (Y, X - 1)            # "/" : the bottom-left corner of the upper-right tile
            if k % 2:
                a, b = b, a
            m[a], m[b] = 2, 1
            k += 1
    return m


def lattice(rng, ny, nx):
    """Isolated pixels on the even-even lattice: 256 components in every full tile; a third of them strong."""
    m = np.zeros((ny, nx), np.uint8)
    m[::2, ::2] = np.where(rng.random(m[::2, ::2].shape) < 1 / 3, 2, 1)
    return m


def checkerboard(ny, nx, seed):
    """(x + y) % 2 == 0: one component held together only by diagonals, 16 runs in every row of a tile."""
    yy, xx = np.mgrid[0:ny, 0:nx]
    m = ((xx + yy) % 2 == 0).astype(np.uint8)
    if seed:
        m[(ny - 1), (nx - 1) - ((nx - 1 + ny - 1) % 2)] = 2
    return m


def full_rows(ny, nx):
    """Full rows (every bit of a 32-pixel row set) alternating with empty rows.  In the upper half the odd rows hold one
    pixel at column 3*nx//5, joining the rows into one comb with a single strong pixel at the far corner; in the lower
    half every full row is its own component, every third one with a strong pixel."""
    m = np.zeros((ny, nx), np.uint8)
    m[::2] = 1
    h = ny // 2
    m[1:h - 1:2, 3 * nx // 5] = 1
    m[h - (h % 2) - 2, nx - 1] = 2
    for i, y in enumerate(range(h + (h % 2), ny, 2)):
        if i % 3 == 0:
            m[y, (7 * i) % nx] = 2
    return m


def frame_seam_batch(ny, nx, n=3):
    """A batch whose frames have a weak last row and a strong first row: nothing may link across the frame boundary,
    so every last row stays 0."""
    m = np.zeros((n, ny, nx), np.uint8)
    m[:, -1, :] = 1
    m[:, 0, :] = 2
    m[:, 0, 1::3] = 0                                   # (a dashed strong row: several runs)
    return m


def row_wrap_seams(ny, nx):
    """Column 0 strong in even tile rows, column nx-1 weak in odd tile rows: the last tile of a tile row and the first tile
    of the next are neighbours in tile order but not in the image, so column nx-1 must stay 0."""
    m = np.zeros((ny, nx), np.uint8)
    for r in range(-(-ny // T)):
        if r % 2 == 0:
            m[r * T:(r + 1) * T, 0] = 2
        else:
            m[r * T:(r + 1) * T, nx - 1] = 1
    return m


def tiny_frames(rng, ny, nx, n=40):
    """n frames of one tiny size with distinct content: empty, full, single pixels and random densities."""
    out = []
    for i in range(n):
        k = i % 5
        if k == 0:
            f = np.zeros((ny, nx), np.uint8)
            if i % 10 == 5:
                f[rng.integers(ny), rng.integers(nx)] = 2
        elif k == 1:
            f = np.ones((ny, nx), np.uint8)
            if i % 2:
                f[rng.integers(ny), rng.integers(nx)] = 2
        else:
            f = random_maps(rng, 1, ny, nx, rng.choice([0.1, 0.3, 0.6, 0.9]), rng.choice([0.02, 0.1, 0.3]))[0]
        out.append(f)
    return np.stack(out)


# ------------------------------------------------------------------------------------------ images
# Images whose Canny class maps (default s = 2, thresholds 3 / 10, accGrad) reach the same hard cases through the
# real blur and NMS.  The parameters were tuned against the oracle's class maps; the tests re-check the features.


def spiral_image(ny=320, nx=384, period=24.0, a0=10.0, a1=3.0):
    """A two-armed Archimedean spiral (cos profile) whose contrast fades from a0 at the centre to a1 at the far
    corners: the inner turns are strong edges, the outer ones weak, so each arm is one long weak chain with its
    strong pixels in a single tile near the centre."""
    yy, xx = np.mgrid[0:ny, 0:nx].astype(np.float64)
    cy, cx = (ny - 1) / 2, (nx - 1) / 2
    r = np.hypot(yy - cy, xx - cx)
    ph = 2 * np.pi * r / period - np.arctan2(yy - cy, xx - cx)
    A = a0 * np.exp(np.log(a1 / a0) * np.sqrt(r / r.max()))
    return np.clip(np.round(128 + A * np.cos(ph)), 0, 255).astype(np.uint8)


def diagonal_stripes(ny=256, nx=320, anti=False):
    """45-degree stripes of period 32 (cos profile) placed so that the edge lines are x - y = 0 (mod 16) or, with
    anti=True, x + y = 15 (mod 16): they cross tile corners diagonally.  The contrast fades along the lines, so the
    strong head of a line reaches its weak tail only through those corners."""
    yy, xx = np.mgrid[0:ny, 0:nx].astype(np.float64)
    u, off = ((xx + yy), 9.0) if anti else ((xx - yy), 8.0)
    v = yy / ny if anti else (xx + yy) / (nx + ny)
    A = 10.0 * np.exp(np.log(3.5 / 10.0) * np.clip(v / 0.5, 0, 1))
    return np.clip(np.round(128 + A * np.cos(2 * np.pi * (u + off) / 32)), 0, 255).astype(np.uint8)


def fine_grating(ny=96, nx=128, period=3):
    """A vertical square-wave grating of period 3 (use s = 1, thresholds 1 / 5): rows with 10 and more runs per tile row."""
    yy, xx = np.mgrid[0:ny, 0:nx]
    return np.clip(128 + np.where((xx % period) < period // 2, 100, -100) + (yy // 8) % 3, 0, 255).astype(np.uint8)


# ------------------------------------------------------------------------------------------ the catalogue

RANDOM_SHAPES = [(1, 1), (1, 64), (64, 1), (31, 33), (32, 32), (33, 65), (96, 64), (100, 1000), (257, 511), (1080, 1920)]
DENSITIES = [0.02, 0.1, 0.3, 0.5, 0.7, 0.9]
STRONG_FRACS = [1e-3, 1e-2]
TINY_SHAPES = [(1, 1), (7, 5), (20, 20), (32, 32), (33, 33), (40, 1), (1, 40), (2, 3)]


def cases(big=True):
    """Every map: yields (family, case id, map uint8 [n, ny, nx], expected kept mask [n, ny, nx] bool or None).
    big=False leaves out the 4 x (2160, 3840) batch."""
    rng = np.random.default_rng(20261015)
    for ny, nx in RANDOM_SHAPES:
        combos = [(d, s) for d in DENSITIES for s in STRONG_FRACS]
        if ny * nx > 10 ** 5:                            # large frames: a batch with one combination per frame
            combos = combos[1::3]
        n = len(combos) if ny * nx <= 10 ** 5 else 2
        for j in range(0, len(combos), n):
            m = np.concatenate([random_maps(rng, 1, ny, nx, d, s) for d, s in combos[j:j + n]])
            yield "random", "%dx%d_%d" % (ny, nx, j), m, None
    if big:
        m = np.concatenate([random_maps(rng, 1, 2160, 3840, d, s) for d, s in [(0.1, 1e-2), (0.3, 1e-3), (0.5, 1e-3), (0.9, 1e-2)]])
        yield "random", "4x2160x3840", m, None
    for ny, nx in [(256, 320), (200, 333)]:
        for shape_name, path, sh in [("serpentine_h", serpentine_path(ny, nx), (ny, nx)),
                                     ("serpentine_v", [(x, y) for y, x in serpentine_path(nx, ny)], (ny, nx)),
                                     ("spiral", spiral_path(ny, nx), (ny, nx))]:
            for vname, m, keep in path_variants(path, *sh):
                yield "path", "%s_%s_%dx%d" % (shape_name, vname, ny, nx), m[None], keep[None]
    for ny, nx in [(256, 320), (200, 333)]:
        yield "corner", "diagonal_%dx%d" % (ny, nx), diagonal_lines(ny, nx)[None], None
        yield "corner", "anti_diagonal_%dx%d" % (ny, nx), anti_diagonals(ny, nx)[None], None
        yield "corner", "pairs_%dx%d" % (ny, nx), corner_pairs(ny, nx)[None], None
    for ny, nx in [(96, 128), (70, 100)]:
        yield "limits", "lattice_%dx%d" % (ny, nx), lattice(rng, ny, nx)[None], None
        yield "limits", "checkerboard_%dx%d" % (ny, nx), np.stack([checkerboard(ny, nx, True), checkerboard(ny, nx, False)]), None
        yield "limits", "full_rows_%dx%d" % (ny, nx), full_rows(ny, nx)[None], None
        one = np.ones((2, ny, nx), np.uint8)
        one[0, ny // 3, nx // 3] = 2
        yield "limits", "all_weak_%dx%d" % (ny, nx), one, np.stack([np.ones((ny, nx), bool), np.zeros((ny, nx), bool)])
    for ny, nx in [(64, 96), (64, 100)]:
        m = frame_seam_batch(ny, nx)
        keep = m == 2
        yield "seam", "frames_%dx%d" % (ny, nx), m, keep
    for ny, nx in [(160, 96), (160, 100), (150, 64)]:
        m = row_wrap_seams(ny, nx)
        yield "seam", "row_wrap_%dx%d" % (ny, nx), m[None], (m == 2)[None]
    for ny, nx in TINY_SHAPES:
        yield "tiny", "40x%dx%d" % (ny, nx), tiny_frames(rng, ny, nx), None
