"""Numpy twin of the seal search (DESIGN.md section 7b, "Seals"), written from the definition, exact in integers so that the
device's seal tables and layout copies equal it bit for bit.  Layered on the page twins: a seal page's layout is the layout of
its layout copy (``layout_image``) under oracle.pages / oracle.panel_pages.  Test infrastructure only."""
import math

import numpy as np
from scipy import ndimage

CHROMA, CELL, CELL_MIN, MAX_SIDE = 64, 4, 2, 4096
BINS, SECTORS, RING_K, RING_SECTORS = 33, 72, 26, 54
RING_DENSITY, BAND_DENSITY, BAND_MIN_K = 4, 32, 10
EMPTY_DIV, MIN_GAP, MIN_TEXT, MAX_SEALS = 720, 2, 9, 64
NO_BAND, NO_GAP, SHORT = 1, 2, 3
DIRS = np.array([(round(2 ** 20 * math.cos(math.radians(5 * j))), round(2 ** 20 * math.sin(math.radians(5 * j))))
                 for j in range(SECTORS // 2)], np.int64)


def default_seal_size(w, h):
    return max(24, min(w, h) // 12)


def seal_mask(img):
    """max(c) - min(c) >= CHROMA per pixel of a uint8 [h, w, 3] image."""
    c = img.astype(np.int16)
    return c.max(axis=2) - c.min(axis=2) >= CHROMA


def candidates(crop, seal_size):
    """(n_cand, candidates): every component of on cells whose box passes the size test, as (x0, y0, x1, y1, root) in crop
    pixels, sorted by (y0, x0, root)."""
    h, w = crop.shape[:2]
    m = seal_mask(crop)
    ch, cw = -(-h // CELL), -(-w // CELL)
    pad = np.zeros((ch * CELL, cw * CELL), bool)
    pad[:h, :w] = m
    on = pad.reshape(ch, CELL, cw, CELL).sum(axis=(1, 3)) >= CELL_MIN
    lab, n = ndimage.label(on, structure=np.ones((3, 3), bool))
    if not n:
        return 0, []
    idx = np.arange(ch * cw).reshape(ch, cw)
    roots = ndimage.minimum(idx, lab, np.arange(1, n + 1)).astype(np.int64)
    plab = np.repeat(np.repeat(lab, CELL, 0), CELL, 1)[:h, :w] * m
    out = []
    for c, sl in enumerate(ndimage.find_objects(plab)):
        if sl is None:
            continue
        y0, y1, x0, x1 = sl[0].start, sl[0].stop, sl[1].start, sl[1].stop
        A, B = x1 - x0, y1 - y0
        if min(A, B) >= seal_size and max(A, B) <= MAX_SIDE and 2 * max(A, B) <= 3 * min(A, B):
            out.append((x0, y0, x1, y1, int(roots[c])))
    out.sort(key=lambda e: (e[1], e[0], e[4]))
    return len(out), out


def ellipse_coords(box):
    """(X, Y, A, B) int64 grids of the box's pixels."""
    x0, y0, x1, y1 = box[:4]
    X = 2 * np.arange(x0, x1, dtype=np.int64) + 1 - (x0 + x1)
    Y = 2 * np.arange(y0, y1, dtype=np.int64) + 1 - (y0 + y1)
    return X[None, :], Y[:, None], np.int64(x1 - x0), np.int64(y1 - y0)


def radial_bin(X, Y, A, B):
    """floor(32 rho), exact: floor(sqrt(floor(1024 (X^2 B^2 + Y^2 A^2) / (A^2 B^2))))."""
    q = 1024 * (X * X * B * B + Y * Y * A * A) // (A * A * B * B)
    k = np.floor(np.sqrt(q.astype(np.float64))).astype(np.int64)
    k -= k * k > q
    k += (k + 1) * (k + 1) <= q
    return k


def sector(px, py):
    """The 5-degree sector of (px, py) between DIRS' directions, by cross products only; (0, 0) is sector 0."""
    px, py = np.broadcast_arrays(np.asarray(px, np.int64), np.asarray(py, np.int64))
    upper = (py > 0) | ((py == 0) & (px > 0))
    qx, qy = np.where(upper, px, -px), np.where(upper, py, -py)
    s = np.zeros(px.shape, np.int64)
    for dx, dy in DIRS[1:]:
        s += dx * qy - dy * qx >= 0
    s = np.where(upper, s, SECTORS // 2 + s)
    return np.where((px == 0) & (py == 0), 0, s)


def histograms(crop, box):
    """ink [BINS, SECTORS] and area [BINS] of a candidate's box."""
    X, Y, A, B = ellipse_coords(box)
    k = radial_bin(X, Y, A, B)
    s = sector(X * B, -Y * A)
    x0, y0, x1, y1 = box[:4]
    m = seal_mask(crop[y0:y1, x0:x1])
    keep = k < BINS
    area = np.bincount(k[keep], minlength=BINS)
    sel = keep & m
    ink = np.bincount((k * SECTORS + s)[sel], minlength=BINS * SECTORS).reshape(BINS, SECTORS)
    return ink, area


def band(ink_k, area):
    """(k_bottom, k_top) of the arc-text band, or None."""
    k = BINS - 1
    while k >= 0 and RING_DENSITY * ink_k[k] < area[k]:
        k -= 1
    while k >= 0 and RING_DENSITY * ink_k[k] >= area[k]:
        k -= 1
    while k >= 0 and BAND_DENSITY * ink_k[k] >= area[k]:
        k -= 1
    gap_top = k
    while k >= BAND_MIN_K and BAND_DENSITY * ink_k[k] < area[k]:
        k -= 1
    if gap_top < BAND_MIN_K or k < BAND_MIN_K:
        return None
    top = k
    while k >= BAND_MIN_K and BAND_DENSITY * ink_k[k] >= area[k]:
        k -= 1
    return k + 1, top


def arc_gap(sec):
    """(g0, n): the longest circular run of empty sectors, ties to the smallest g0."""
    band_ink = int(sec.sum())
    empty = EMPTY_DIV * sec < max(EMPTY_DIV, band_ink)
    if empty.all():
        return 0, SECTORS
    g0 = n = 0
    for s in range(SECTORS):
        if not empty[s] or empty[s - 1]:
            continue
        m = 0
        while empty[(s + m) % SECTORS]:
            m += 1
        if m > n:
            g0, n = s, m
    return g0, n


def seal_record(crop, cand):
    """The mn_seal fields of a candidate (x0, y0, x1, y1, root), as a dict."""
    ink, area = histograms(crop, cand)
    ring = int((ink[RING_K:].sum(axis=0) > 0).sum())
    r = dict(x0=cand[0], y0=cand[1], x1=cand[2], y1=cand[3], root=cand[4], ring=ring, found=int(ring >= RING_SECTORS),
             k_bottom=-1, k_top=-1, g0=-1, n_gap=-1, why=0, band_ink=0)
    if not r["found"]:
        return r
    bd = band(ink.sum(axis=1), area)
    if bd is None:
        r["why"] = NO_BAND
        return r
    r["k_bottom"], r["k_top"] = bd
    sec = ink[bd[0]:bd[1] + 1].sum(axis=0)
    r["band_ink"] = int(sec.sum())
    r["g0"], r["n_gap"] = arc_gap(sec)
    n = r["n_gap"]
    r["why"] = NO_GAP if n < MIN_GAP else SHORT if SECTORS - n < MIN_TEXT else 0
    return r


def find_seals(crop, seal_size):
    """The mn_seal_table of a page crop: dict(error, n_cand, n_seals, seals), seals the records of the candidates in order
    (empty with error 1 over MAX_SEALS candidates)."""
    n, cands = candidates(crop, seal_size)
    if n > MAX_SEALS:
        return dict(error=1, n_cand=n, n_seals=0, seals=[])
    seals = [seal_record(crop, c) for c in cands]
    return dict(error=0, n_cand=n, n_seals=sum(s["found"] for s in seals), seals=seals)


def layout_copy(crop, boxes):
    """The crop with every seal-coloured pixel at rho < 33/32 of one of ``boxes`` (crop pixels) set to 255."""
    out = crop.copy()
    m = seal_mask(crop)
    h, w = crop.shape[:2]
    for box in boxes:
        x0, y0, x1, y1 = box[:4]
        bx0, by0, bx1, by1 = max(x0, 0), max(y0, 0), min(x1, w), min(y1, h)
        if bx0 >= bx1 or by0 >= by1:
            continue
        X, Y, A, B = ellipse_coords(box)
        inside = 1024 * (X * X * B * B + Y * Y * A * A) < BINS * BINS * A * A * B * B
        inside = inside[by0 - y0:by1 - y0, bx0 - x0:bx1 - x0] & m[by0:by1, bx0:bx1]
        out[by0:by1, bx0:bx1][inside] = 255
    return out


def layout_image(img, rect, boxes):
    """The whole image with its crop ``rect`` replaced by the crop's layout copy for seal ``boxes`` in image pixels: the page
    twins run on it with the same rect."""
    x0, y0, x1, y1 = rect
    out = img.copy()
    out[y0:y1, x0:x1] = layout_copy(img[y0:y1, x0:x1], [(a - x0, b - y0, c - x0, d - y0) for a, b, c, d in boxes])
    return out


def page_seals(img, rect=None, seal_size=None):
    """find_seals of a page crop with its found seals' boxes in image coordinates: (table, boxes)."""
    H, W = img.shape[:2]
    x0, y0, x1, y1 = rect or (0, 0, W, H)
    t = find_seals(img[y0:y1, x0:x1], seal_size or default_seal_size(x1 - x0, y1 - y0))
    return t, [(s["x0"] + x0, s["y0"] + y0, s["x1"] + x0, s["y1"] + y0) for s in t["seals"] if s["found"]]
