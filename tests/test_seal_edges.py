"""The seal search at the edges of its contract, on the host: builds every input test_gpu_seal_edges.py runs on the device and
proves with the numpy twin that each one reaches the edge it is tagged with -- chroma 63 against 64 in every channel order, cells
of 1 and 2 seal pixels, last cells of width and height 1 to 3, components joined only through NE and NW cell diagonals across
cell-tile borders, exact (bin, sector) counts on both sides of every band and arc threshold, pixels on the sector rays and at
rho = k / 32 exactly, and the 4096-side candidates.  Histogram and table values are asserted, not only final tables.

Exact counts are painted as the first n pixels, in raster order, of a chosen (bin, sector) set of a fixed box, with bins 30-32
(the ring) fully painted in all 72 sectors so that the candidate's box stays the whole crop."""
import functools

import numpy as np
import pytest

from oracle import seal_pages as S
from oracle import spread_pages as SP

from test_seal_pages import BOX, PAPER, RED, stamp

RING3 = range(30, 33)
RAYS = {0: 0, 45: 9, 90: 18, 180: 36, 270: 54}       # ray angle -> the sector whose first direction it is


@functools.lru_cache(maxsize=None)
def grid(A, B):
    """(k, s): the radial bin and sector of each pixel of an A x B box (B rows), read-only."""
    X, Y, a, b = S.ellipse_coords((0, 0, A, B))
    k, s = (np.ascontiguousarray(v) for v in np.broadcast_arrays(S.radial_bin(X, Y, a, b), S.sector(X * b, -Y * a)))
    k.flags.writeable = s.flags.writeable = False
    return k, s


def lhs(A, B):
    """1024 (X^2 B^2 + Y^2 A^2) per pixel of an A x B box, and A^2 B^2."""
    X, Y, a, b = S.ellipse_coords((0, 0, A, B))
    return 1024 * (X * X * b * b + Y * Y * a * a), a * a * b * b


def first(mask, n):
    """The first n pixels of ``mask`` in raster order (it must hold them)."""
    idx = np.flatnonzero(mask)[:n]
    assert len(idx) == n
    out = np.zeros(mask.shape, bool)
    out.flat[idx] = True
    return out


def sel(A, B, ks, secs):
    k, s = grid(A, B)
    return np.isin(k, list(ks)) & np.isin(s, list(secs))


def page(A, B, *masks, ring=range(72), colour=RED):
    """An A x B crop, seal red on bins 30-32 of the sectors ``ring`` and on each of ``masks``."""
    img = np.full((B, A, 3), PAPER, np.uint8)
    img[sel(A, B, RING3, ring)] = colour
    for m in masks:
        img[m] = colour
    return img


def ring_crop(A, B):
    """A big A x B crop whose bins 30-32 are seal red, from the bins alone (no sectors)."""
    X, Y, a, b = S.ellipse_coords((0, 0, A, B))
    q = 1024 * (X * X * b * b + Y * Y * a * a)
    img = np.full((B, A, 3), PAPER, np.uint8)
    img[(q >= 900 * a * a * b * b) & (q < 1089 * a * a * b * b)] = RED
    return img


def record(img, seal_size=8, box=None):
    """The twin's record of the candidate ``box`` (default: the whole crop) of find_seals(img)."""
    t = S.find_seals(img, seal_size)
    box = box or (0, 0, img.shape[1], img.shape[0])
    (r,) = [r for r in t["seals"] if (r["x0"], r["y0"], r["x1"], r["y1"]) == box]
    return r


def ink_area(img, box=None):
    box = box or (0, 0, img.shape[1], img.shape[0], 0)
    return S.histograms(img, box)


# ---- colour and cells ----------------------------------------------------------------------------------------------------
CHROMA_LEVELS = ((0, 63), (0, 64), (192, 255), (191, 255), (100, 163), (100, 164))


def chroma_colours():
    """(colour, chroma) for max - min of 63 and 64 with the max and the min channel in each position, at grey 0, 255 and mid."""
    out = []
    for lo, hi in CHROMA_LEVELS:
        for imax in range(3):
            for imin in range(3):
                if imin != imax:
                    c = [(lo + hi) // 2] * 3
                    c[imax], c[imin] = hi, lo
                    out.append((tuple(c), hi - lo))
    return out


def chroma_page():
    """The 200 x 200 ring with one probe pixel of each chroma colour inside, 8 pixels apart (one to a cell)."""
    img = page(200, 200)
    pos = [(70 + 8 * (j % 8), 70 + 8 * (j // 8)) for j in range(len(chroma_colours()))]
    for (c, _), (x, y) in zip(chroma_colours(), pos):
        img[y, x] = c
    return img, pos


def frame(img, x0, y0, x1, y1, t=2, colour=RED):
    img[y0:y1, x0:x0 + t] = img[y0:y1, x1 - t:x1] = img[y0:y0 + t, x0:x1] = img[y1 - t:y1, x0:x1] = colour


def cells_page():
    """Frames of side 40 (seal size 8) with, beside their right edge: one seal pixel in the next cell (off), two (on), a 2-pixel
    run across the next cells' border (both off); and two frames one off cell apart."""
    img = np.full((100, 160, 3), PAPER, np.uint8)
    for x0, y0 in ((4, 4), (60, 4), (4, 56), (60, 56), (104, 56)):
        frame(img, x0, y0, x0 + 40, y0 + 40)
    img[20, 45] = RED                               # cell 11: one pixel
    img[20, 101] = img[20, 102] = RED               # cell 25: two pixels
    img[76, 47] = img[76, 48] = RED                 # cells 11 and 12: one each
    return img


def last_cell_pages():
    """Crops of w, h = 1, 2, 3 mod 4 and w = 0 mod 128 (one cell tile is 128 x 32 pixels): a 1-pixel frame on the crop's border
    (the last cells hold its last column and row) around the ring of the whole crop."""
    out = []
    for w, h in ((61, 62), (62, 63), (63, 61), (256, 201)):
        img = ring_crop(w, h)
        frame(img, 0, 0, w, h, t=1)
        out.append(img)
    return out


def chain_page():
    """Two chains of cells with two seal pixels each on a 150 x 60 crop (38 cells wide, the last 2 pixels): one joined only through
    NE diagonals, across the cell-tile borders cx = 31 | 32 and cy = 8 | 7 and into the last cell column; one only through NW
    diagonals across cy = 7 | 8."""
    img = np.full((60, 150, 3), PAPER, np.uint8)
    for cx, cy in [(28 + i, 12 - i) for i in range(10)] + [(2 + i, 2 + i) for i in range(10)]:
        img[4 * cy + 1, 4 * cx] = img[4 * cy, 4 * cx + 1] = RED
    return img


def arcs_page():
    """Two concentric quarter arcs around the corner (10, 10): both candidates' boxes start at (10, 10)."""
    img = np.full((70, 70, 3), PAPER, np.uint8)
    dy, dx = np.mgrid[0:60, 0:60]
    d2 = dx * dx + dy * dy
    for r in (20, 40):
        img[10:70, 10:70][(d2 >= r * r) & (d2 < (r + 3) ** 2)] = RED
    return img


def size_page():
    """Frames of side 8 and 7 at seal size 8."""
    img = np.full((20, 40, 3), PAPER, np.uint8)
    frame(img, 4, 4, 12, 12)
    frame(img, 20, 4, 27, 11)
    return img


def test_chroma_probes():
    img, pos = chroma_page()
    m = S.seal_mask(img)
    copy = S.layout_copy(img, [BOX])
    seen = set()
    for (c, ch), (x, y) in zip(chroma_colours(), pos):
        assert m[y, x] == (ch >= 64) and int(max(c)) - int(min(c)) == ch
        assert (tuple(copy[y, x]) == (255, 255, 255)) == (ch >= 64)
        seen.add((c.index(max(c)), c.index(min(c)), min(c) == 0 or max(c) == 255))
    assert len(seen) == 12 and len(chroma_colours()) == 36
    with pytest.MonkeyPatch.context() as mp:
        mp.setattr(S, "CHROMA", 63)
        assert not (S.layout_copy(img, [BOX]) == copy).all()


def test_cells():
    img = cells_page()
    n, cands = S.candidates(img, 8)
    assert [c[:4] for c in cands] == [(4, 4, 44, 44), (60, 4, 103, 44), (4, 56, 44, 96), (60, 56, 100, 96), (104, 56, 144, 96)]
    for w, h in ((61, 62), (62, 63), (63, 61), (256, 201)):
        assert (w % 4, h % 4) in ((1, 2), (2, 3), (3, 1), (0, 1))
    for img in last_cell_pages():
        h, w = img.shape[:2]
        r = record(img)
        assert r["found"] and (r["x0"], r["y0"], r["x1"], r["y1"]) == (0, 0, w, h)


def test_diagonal_chains():
    img = chain_page()
    assert S.candidates(img, 8)[1] == [(8, 8, 46, 46, 2 * 38 + 2), (112, 12, 150, 50, 3 * 38 + 37)]
    from scipy import ndimage
    with pytest.MonkeyPatch.context() as mp:              # 4-connected cells find no candidate
        mp.setattr(S, "ndimage", _four_connected(ndimage))
        assert S.candidates(img, 8) == (0, [])


def _four_connected(ndimage):
    import types
    return types.SimpleNamespace(label=lambda a, structure=None: ndimage.label(a), minimum=ndimage.minimum,
                                 find_objects=ndimage.find_objects)


def test_root_ties_and_sizes():
    n, cands = S.candidates(arcs_page(), 8)
    assert n == 2 and [c[:2] for c in cands] == [(10, 10), (10, 10)] and cands[0][4] < cands[1][4]
    assert cands[0][2] < cands[1][2]
    assert S.candidates(size_page(), 8)[1] == [(4, 4, 12, 12, 1 * 10 + 1)]


# ---- ring, band and arc: exact counts -------------------------------------------------------------------------------------
def band_pages():
    """(name, crop, facts) on the 200 x 200 box: facts the twin's record and histogram values each page must show."""
    A = B = 200
    k, s = grid(A, B)
    area = np.bincount(k[k < 33], minlength=33)
    out = []
    out.append(("band 32 ink == area", page(A, B, first(sel(A, B, [20], range(72)), area[20] // 32)), (20, 20)))
    out.append(("band 32 ink == area - 1", page(A, B, first(sel(A, B, [20], range(72)), area[20] // 32 - 1)), None))
    # bin 29 at 4 ink == area ends the ring run, one pixel less hands it to the edge run: the band is the same either way
    out.append(("ring inner 4 ink == area", page(A, B, first(sel(A, B, [29], range(72)), area[29] // 4),
                                                 sel(A, B, [20], range(72))), (20, 20)))
    out.append(("ring inner 4 ink == area - 1", page(A, B, first(sel(A, B, [29], range(72)), area[29] // 4 - 1),
                                                     sel(A, B, [20], range(72))), (20, 20)))
    out.append(("band stops at 10", page(A, B, sel(A, B, range(8, 15), range(72))), (10, 14)))
    out.append(("band bin 10 exact", page(A, B, first(sel(A, B, [10], range(72)), area[10] // 32)), (10, 10)))
    out.append(("no gap", page(A, B, *[first(sel(A, B, [j], range(72)), -(-area[j] // 32)) for j in range(10, 30)]), None))
    text = first(sel(A, B, range(18, 21), range(36)), 1438)
    two = first(sel(A, B, [19], [50]), 2)
    out.append(("720 sec == band_ink", page(A, B, text, two), (18, 20)))
    out.append(("720 sec == band_ink + 1", page(A, B, text, first(sel(A, B, [19], [50]), 1)), (18, 20)))
    for name, secs in (("gap 1", set(range(72)) - {40}), ("gap 2", set(range(72)) - {40, 41}), ("text 8", range(10, 18)),
                       ("text 9", range(10, 19)), ("gap wraps 71 | 0", range(10, 61)),
                       ("tied gaps", list(range(0, 10)) + list(range(36, 46)))):
        out.append((name, page(A, B, sel(A, B, [20], secs)), (20, 20)))
    return out


def empty_page():
    """A 12 x 15 crop whose bins 26-32 are seal red: its band (bin 23) holds no pixel, so all 72 sectors are empty."""
    k, _ = grid(12, 15)
    img = np.full((15, 12, 3), PAPER, np.uint8)
    img[k >= 26] = RED
    return img


RING53 = set(range(72)) - set(range(4, 9)) - set(range(22, 27)) - set(range(40, 45)) - set(range(58, 62))


def ring_pages():
    """Rings of bins 30-32 over 53 and 54 sectors inside a 2-pixel frame of the crop, which joins them into one component
    whose box is the crop; the frame's pixels at rho < 33 / 32 lie within 15 degrees of the axes, in sectors of the ring."""
    out = []
    for secs in (RING53, RING53 | {61}):
        img = page(200, 200, ring=sorted(secs))
        frame(img, 0, 0, 200, 200)
        out.append(img)
    return out


def test_band_pages():
    A = B = 200
    k, _ = grid(A, B)
    area = np.bincount(k[k < 33], minlength=33)
    assert area[20] == 32 * 40 and area[10] == 32 * 20 and area[29] % 4 == 0
    for name, img, band in band_pages():
        r = record(img)
        ink, ar = ink_area(img)
        ink_k = ink.sum(axis=1)
        assert (ar == area).all() and r["found"] and r["ring"] == 72, name
        assert ((r["k_bottom"], r["k_top"]) if r["k_top"] >= 0 else None) == band, name
        if name.startswith("band 32"):
            assert 32 * ink_k[20] - area[20] == (0 if "- 1" not in name else -32)
        if name.startswith("ring inner"):
            assert 4 * ink_k[29] - area[29] == (0 if "- 1" not in name else -4)
        if name == "band stops at 10":
            assert (ink_k[8:10] == area[8:10]).all()
        if name == "no gap":
            assert r["why"] == S.NO_BAND and all(32 * ink_k[j] >= area[j] for j in range(10, 33))
        if name.startswith("720"):
            sec = ink[18:21].sum(axis=0)
            assert 720 * sec[50] - r["band_ink"] == (0 if "+ 1" not in name else -719)
            assert r["band_ink"] > 720 and (r["g0"], r["n_gap"]) == ((51, 24) if "+ 1" not in name else (33, 42))
        if name.startswith(("gap", "text", "tied")):
            want = {"gap 1": (40, 1, S.NO_GAP), "gap 2": (40, 2, 0), "text 8": (18, 64, S.SHORT), "text 9": (19, 63, 0),
                    "gap wraps 71 | 0": (61, 21, 0), "tied gaps": (10, 26, 0)}[name]
            assert (r["g0"], r["n_gap"], r["why"]) == want, name
    r = record(empty_page())
    assert (r["found"], r["ring"], r["k_top"], r["band_ink"], r["g0"], r["n_gap"], r["why"]) == (1, 54, 23, 0, 0, 72, S.SHORT)
    assert ink_area(empty_page())[1][23] == 0
    for img, n in zip(ring_pages(), (53, 54)):
        r = record(img)
        assert (r["ring"], r["found"]) == (n, int(n == 54))


def _band_gt(ink_k, area):
    """S.band with the band density's >= passed as >."""
    k = S.BINS - 1
    while k >= 0 and S.RING_DENSITY * ink_k[k] < area[k]:
        k -= 1
    while k >= 0 and S.RING_DENSITY * ink_k[k] >= area[k]:
        k -= 1
    while k >= 0 and S.BAND_DENSITY * ink_k[k] > area[k]:
        k -= 1
    gap_top = k
    while k >= S.BAND_MIN_K and S.BAND_DENSITY * ink_k[k] <= area[k]:
        k -= 1
    if gap_top < S.BAND_MIN_K or k < S.BAND_MIN_K:
        return None
    top = k
    while k >= S.BAND_MIN_K and S.BAND_DENSITY * ink_k[k] > area[k]:
        k -= 1
    return k + 1, top


def _arc_gap_le(sec):
    """S.arc_gap with the empty-sector test's < passed as <=."""
    band_ink = int(sec.sum())
    empty = S.EMPTY_DIV * sec <= max(S.EMPTY_DIV, band_ink)
    if empty.all():
        return 0, S.SECTORS
    g0 = n = 0
    for s in range(S.SECTORS):
        if not empty[s] or empty[s - 1]:
            continue
        m = 0
        while empty[(s + m) % S.SECTORS]:
            m += 1
        if m > n:
            g0, n = s, m
    return g0, n


def layout_copy_le(crop, boxes):
    """S.layout_copy with its rho < 33 / 32 passed as rho <= 33 / 32."""
    out = crop.copy()
    m = S.seal_mask(crop)
    h, w = crop.shape[:2]
    for box in boxes:
        x0, y0, x1, y1 = box[:4]
        bx0, by0, bx1, by1 = max(x0, 0), max(y0, 0), min(x1, w), min(y1, h)
        if bx0 >= bx1 or by0 >= by1:
            continue
        X, Y, A, B = S.ellipse_coords(box)
        inside = 1024 * (X * X * B * B + Y * Y * A * A) <= S.BINS * S.BINS * A * A * B * B
        inside = inside[by0 - y0:by1 - y0, bx0 - x0:bx1 - x0] & m[by0:by1, bx0:bx1]
        out[by0:by1, bx0:bx1][inside] = 255
    return out


def test_controls_disagree_with_the_twin_on_their_pages():
    pages = {name: img for name, img, _ in band_pages()}
    for name, attr, value in (("band 32 ink == area", "band", _band_gt), ("720 sec == band_ink", "arc_gap", _arc_gap_le),
                              (None, "RING_SECTORS", 53)):
        img = pages[name] if name else ring_pages()[0]
        want = record(img)
        with pytest.MonkeyPatch.context() as mp:
            mp.setattr(S, attr, value)
            assert record(img) != want, attr


# ---- histograms: rays, centre, exact rho -----------------------------------------------------------------------------------
def ray_pages():
    """(name, crop, (x, y), sector) on odd boxes, square 201 x 201 and oval 195 x 165: the ring; a probe pixel on the ray (cross
    = 0 with its sector's first direction) at a band bin kb; and bin kb painted in the three sectors before it.  The arc's gap
    then starts right after the probe's sector.  The square page also paints its centre pixel (p = 0)."""
    out = []
    for A, B in ((201, 201), (195, 165)):
        k, s = grid(A, B)
        X, Y, a, b = S.ellipse_coords((0, 0, A, B))
        px, py = np.broadcast_arrays(X * b, -Y * a)
        for deg, sec in RAYS.items():
            d = S.DIRS[sec % 36] * (1 if sec < 36 else -1)
            on = (d[0] * py - d[1] * px == 0) & (k >= 12) & (k <= 24) & (s == sec)
            y, x = np.argwhere(on)[0]
            kb = int(k[y, x])
            img = page(A, B, sel(A, B, [kb], [(sec - j) % 72 for j in (1, 2, 3)]))
            img[y, x] = RED
            if A == B:
                img[B // 2, A // 2] = RED
            out.append((f"{deg} degrees, {'square' if A == B else 'oval'}", img, (int(x), int(y)), sec))
    return out


def exact_rho_pages():
    """(crop, probes): the ring of a 44 x 48 box with its pixels at rho = 10 / 32 and 26 / 32 exactly, and of a 160 x 120 box
    with those at rho = 33 / 32 exactly and the largest rho under it.  (rho = 1 holds no pixel centre: X / A = +-1 lies on the
    box's edge, and a rational point of the unit circle has one even and one odd numerator over an odd denominator, which the
    parities of X against A and Y against B exclude.)"""
    out = []
    for (A, B), ks in (((44, 48), (10, 26)), ((160, 120), (33,))):
        q, ab = lhs(A, B)
        q = np.broadcast_to(q, (B, A))
        img = page(A, B)
        probes = {}
        for kk in ks:
            probes[kk] = [tuple(p) for p in np.argwhere(q == kk * kk * ab)]
            for y, x in probes[kk]:
                img[y, x] = (40, 60, 190)
        if 33 in ks:
            inside = q[q < 1089 * ab].max()
            probes["under 33"] = [tuple(p) for p in np.argwhere(q == inside)]
            for y, x in probes["under 33"]:
                img[y, x] = (40, 60, 190)
        out.append((img, probes))
    return out


def test_ray_and_exact_rho_pages():
    for name, img, (x, y), sec in ray_pages():
        A, B = img.shape[1], img.shape[0]
        k, s = grid(A, B)
        r = record(img)
        assert r["found"] and r["k_top"] == r["k_bottom"] == k[y, x], name
        assert (r["g0"], r["n_gap"]) == ((sec + 1) % 72, 68), name
    for img, probes in exact_rho_pages():
        A, B = img.shape[1], img.shape[0]
        k, _ = grid(A, B)
        q, ab = lhs(A, B)
        q = np.broadcast_to(q, (B, A))
        copy = S.layout_copy(img, [(0, 0, A, B)])
        for kk, pts in probes.items():
            assert pts
            for y, x in pts:
                if kk == "under 33":
                    assert k[y, x] == 32 and (copy[y, x] == 255).all()
                else:
                    assert q[y, x] == kk * kk * ab and k[y, x] == kk
                    assert (copy[y, x] == 255).all() == (kk < 33)
        if 33 in probes:
            assert not (layout_copy_le(img, [(0, 0, A, B)]) == copy).all()


# ---- 4096-side candidates ------------------------------------------------------------------------------------------------
BIG = ((4096, 4096, 4096, True), (4095, 4095, 4096, False), (4097, 4097, 8, False), (4096, 2731, 8, True),
       (2731, 4096, 8, True), (4096, 2730, 8, False), (2730, 4096, 8, False))


def test_big_candidates():
    """The candidate test only: the histograms of the 16.7 M-pixel box run against the twin in the device test."""
    for A, B, ss, cand in BIG:
        img = ring_crop(A, B)
        n, c = S.candidates(img, ss)
        assert n == int(cand), (A, B)
        if cand:
            assert c[0][:4] == (0, 0, A, B)


# ---- windowed twin ----------------------------------------------------------------------------------------------------------
def windowed(win, ox, oy, w, seal_size):
    """find_seals of a crop w pixels wide that is paper outside ``win``, its window at (ox, oy) (multiples of 4, every seal
    pixel at least 4 pixels inside the window): the window's table with boxes and roots moved to the crop."""
    assert ox % 4 == 0 and oy % 4 == 0
    t = S.find_seals(win, seal_size)
    wcw, cw = -(-win.shape[1] // 4), -(-w // 4)
    seals = []
    for r in t["seals"]:
        cy, cx = divmod(r["root"], wcw)
        seals.append(dict(r, x0=r["x0"] + ox, y0=r["y0"] + oy, x1=r["x1"] + ox, y1=r["y1"] + oy,
                          root=(cy + oy // 4) * cw + cx + ox // 4))
    return dict(t, seals=seals)


def stamp_window():
    """A 260 x 260 window holding one drawn stamp 8 pixels inside its border."""
    win = np.full((260, 260, 3), PAPER, np.uint8)
    stamp(win, 130, 130, 118, 118)
    m = S.seal_mask(win)
    assert not m[:8].any() and not m[-8:].any() and not m[:, :8].any() and not m[:, -8:].any()
    return win


def test_windowed_twin_equals_the_whole_crop():
    win = stamp_window()
    for (H, W), (ox, oy) in (((700, 900), (400, 300)), ((600, 500), (0, 0)), ((264, 264), (4, 4))):
        img = np.full((H, W, 3), PAPER, np.uint8)
        img[oy:oy + 260, ox:ox + 260] = win
        want = S.find_seals(img, 100)
        assert want["n_seals"] == 1 and windowed(win, ox, oy, W, 100) == want


# ---- spines ---------------------------------------------------------------------------------------------------------------
def key_plane(n, x1, x2):
    """A label plane of n x n (as a boolean mask): every pixel of the page except the first n - 1 rows of columns x1 and x2,
    and the quad (0, -n), (n, -n), (n, 2n), (0, 2n) set by hand: t(x) = 0 except t(x1) = t(x2) = n - 1, b(x) = n.  Corners
    inside the image give |D| <= n^2 < 2^30; these lie n rows above and below it, so D = n (2n - 1) nears the key's 2^31."""
    m = np.ones((n, n), bool)
    m[:n - 1, x1] = m[:n - 1, x2] = False
    return m, [(0, -n), (n, -n), (n, 2 * n), (0, 2 * n)]


def key_expected(n, x1, x2):
    """The closed form of the spine of key_plane: D = n (t(x1) + n) at x1 (the tie's smaller column), E = n (2n - n) = n^2 at
    the first column of the middle half, ceil(n / 4)."""
    lo = -(-n // 4)
    return dict(found=True, st=(x1, n - 1), sb=(lo, n), D=n * (2 * n - 1), E=n * n)


def test_key_plane_closed_form():
    for n in (67, 101, 4 * 33 + 3):
        x1, x2 = n // 2 - 3, n // 2 + 5
        m, quad = key_plane(n, x1, x2)
        assert SP.spine(m, quad) == key_expected(n, x1, x2)
    n = 32767
    assert 2 ** 30 <= n * (2 * n - 1) < 2 ** 31 and n * n < 2 ** 30      # in-image corners reach at most 32767^2 < 2^30
