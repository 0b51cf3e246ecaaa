"""numpy twin of pipeline.find_blocks and find_lines for skewed pages and windowed blocks (DESIGN.md section 7b, "Skewed pages"):
the page's angle searched as a skewed block's, the XY-cut of oracle/pages.py on the bitmap of rotated-frame cells, and the lines
of each block, the pixels of the page whose cell lies in the block's window.  Vectorised numpy fp64, every operation rounded on
its own; written from the definition, not from the kernels.
TEST INFRASTRUCTURE ONLY."""
import math

import numpy as np

from . import blocks as B
from . import pages as P
from . import skewed_blocks as SB


def layout(ink, vertical, gap_x=None, gap_y=None):
    """Steps 4 to 6 of "Text pages" on the boolean [h, w] mask ``ink`` (oracle/pages.find_blocks' text size, XY-cut, rejection
    and growth, on a mask): (blocks, rejected, text_size, gap_x, gap_y) in mask cells, blocks in reading order, grown and
    clipped to the mask.  A mask without a leaf of size >= 2 gives ([], [], 0, 0, 0).  Raises ValueError over a limit."""
    sizes = sorted(s for s in (max(x1 - x0, y1 - y0) for x0, y0, x1, y1 in P.xy_cut(ink, vertical, 1, 1)) if s >= 2)
    if not sizes:
        return [], [], 0, 0, 0
    S = sizes[(len(sizes) - 1) // 2]
    wide, narrow = S, max(1, S // 2)
    g_x = gap_x or (narrow if vertical else wide)
    g_y = gap_y or (wide if vertical else narrow)
    q = (min(g_x, g_y) - 1) // 2
    h, w = ink.shape
    blocks, rejected = [], []
    for x0, y0, x1, y1 in P.xy_cut(ink, vertical, g_x, g_y):
        n = int(ink[y0:y1, x0:x1].sum())
        if 2 * n > (y1 - y0) * (x1 - x0) or min(y1 - y0, x1 - x0) < max(1, S // 3):
            rejected.append((x0, y0, x1, y1))
        else:
            blocks.append((max(0, x0 - q), max(0, y0 - q), min(w, x1 + q), min(h, y1 + q)))
    if len(blocks) > P.MAX_BLOCKS:
        raise ValueError(f"{len(blocks)} blocks exceed the {P.MAX_BLOCKS} a text page may hold")
    return blocks, rejected, S, g_x, g_y


def ink_of(img, rect=None, polarity="auto"):
    """Steps 1 to 3 on the page ``rect`` (None: the whole image): (rect, ink mask, threshold, polarity)."""
    H, W = img.shape[:2]
    X0, Y0, X1, Y1 = rect if rect is not None else (0, 0, W, H)
    g = B.grey(img[Y0:Y1, X0:X1])
    t = B.otsu(g)
    if polarity == "auto":
        polarity = "dark" if 2 * int((g <= t).sum()) <= g.size else "light"
    return (X0, Y0, X1, Y1), (g <= t if polarity == "dark" else g > t), t, polarity


def table(skew, max_skew, vertical):
    """(idx, deg, c, s) of the search: the angle table's indices, the frame angles in degrees (a given angle negated for a
    vertical page, whose frame is the transposed crop) and their fp64 cos and sin."""
    tab = SB.angles(skew, max_skew)
    idx = [i for i, _ in tab]
    deg = [(-th if vertical and not isinstance(skew, str) else th) for _, th in tab]
    c = np.array([math.cos(math.radians(d)) for d in deg], np.float64)
    s = np.array([math.sin(math.radians(d)) for d in deg], np.float64)
    return idx, deg, c, s


def cells(h, w, c, s):
    """(k, j, L, M, u_min, v_min) of every pixel of an h x w crop in the frame (c, s): [h, w] int64 bins and indices."""
    u_min, v_min, L, M = (a[0] for a in SB.frame(h, w, np.array([c]), np.array([s])))
    ys, xs = np.mgrid[0:h, 0:w].astype(np.float64)
    u, v = SB._uv(ys, xs, h, w, c, s)
    k = np.clip(np.floor(v - v_min), 0, L - 1).astype(np.int64)
    j = np.clip(np.floor(u - u_min), 0, M - 1).astype(np.int64)
    return k, j, int(L), int(M), float(u_min), float(v_min)


def frame_bitmap(ink, c, s):
    """The L x M bitmap of frame cells of the boolean [h, w] mask ``ink`` at (c, s): a cell is set iff an ink pixel falls in it."""
    h, w = ink.shape
    k, j, L, M, _, _ = cells(h, w, c, s)
    bits = np.zeros((L, M), bool)
    bits[k[ink], j[ink]] = True
    return bits


def find_blocks(img, rect=None, direction="horizontal", polarity="auto", gap_x=None, gap_y=None, skew="auto", max_skew=10.0):
    """The skewed text page ``rect`` of ``img`` -> dict(blocks, rejected, threshold, ink, text_size, gap_x, gap_y, skew, detail).
    When the chosen entry's s is 0 this is oracle/pages.find_blocks' dict plus skew.  Otherwise blocks and rejected are windows
    (c0, l0, c1, l1) of the block frame (the transposed crop at the negated angle for a vertical page), blocks in reading order.
    detail: the table's i, c, s, the scores (None for a one-entry table), the chosen position, the bitmap's frame (u_min, v_min,
    L, M) (the untransposed frame of a vertical page) and its leaves (x0, y0, x1, y1, rejected) in bitmap cells."""
    (X0, Y0, X1, Y1), ink, t, polarity = ink_of(img, rect, polarity)
    vertical = direction == "vertical"
    idx, deg, c, s = table(skew, max_skew, vertical)
    search = ink.T if vertical else ink
    _, _, Ls, Ms = SB.frame(*search.shape, c, s)
    if max(Ls.max(), Ms.max()) > 32767:
        raise ValueError(f"a frame side of {max(Ls.max(), Ms.max())} exceeds 32767")
    if len(idx) > 1:
        scores = [SB.score(r) for r in SB.profiles(search, c, s)]
        p = SB.choose(idx, scores)
    else:
        scores, p = None, 0
    angle = float(skew) if not isinstance(skew, str) else 0.0 - deg[p] if vertical else deg[p]
    detail = dict(i=idx, c=c, s=s, scores=scores, chosen=p)
    if s[p] == 0:
        out = P.find_blocks(img, rect, direction, polarity, gap_x, gap_y)
        return dict(out, skew=angle, detail=dict(detail, frame=None, leaves=None))
    cb, sb = c[p], -s[p] if vertical else s[p]                  # the axis swap: (c, -s) on the untransposed crop
    u_min, v_min, L, M = (a[0] for a in SB.frame(*ink.shape, np.array([cb]), np.array([sb])))
    bits = frame_bitmap(ink, cb, sb)
    blocks, rejected, S, g_x, g_y = layout(bits, vertical, gap_x, gap_y)
    swap = (lambda r: (r[1], r[0], r[3], r[2])) if vertical else (lambda r: tuple(r))
    leaves = [tuple(r) + (False,) for r in blocks] + [tuple(r) + (True,) for r in rejected]
    return dict(blocks=[swap(r) for r in blocks], rejected=[swap(r) for r in rejected], threshold=t, ink=polarity, text_size=S,
                gap_x=g_x, gap_y=g_y, skew=angle,
                detail=dict(detail, frame=(float(u_min), float(v_min), int(L), int(M)), leaves=leaves))


def block_frame(h, w, vertical, skew):
    """(c, s, u_min, v_min, L, M) of a windowed block's frame: the crop's (transposed for a vertical block) at the given angle
    (negated for a vertical block)."""
    _, _, c, s = table(skew, 10.0, vertical)
    ht, wt = (w, h) if vertical else (h, w)
    u_min, v_min, L, M = (a[0] for a in SB.frame(ht, wt, c, s))
    return float(c[0]), float(s[0]), float(u_min), float(v_min), int(L), int(M)


def members(h, w, vertical, skew, window):
    """The boolean [h, w] mask of the crop's pixels whose frame cell lies in ``window`` = (c0, l0, c1, l1)."""
    c, s, *_ = block_frame(h, w, vertical, skew)
    ht, wt = (w, h) if vertical else (h, w)
    k, j, *_ = cells(ht, wt, c, s)
    c0, l0, c1, l1 = window
    m = (k >= l0) & (k < l1) & (j >= c0) & (j < c1)
    return m.T if vertical else m


def footprint(h, w, vertical, skew, window):
    """The crop pixels [px0, px1) x [py0, py1) that hold the window's pixel set: the fp64 bounding box of its corners' pixel
    centres, padded by one pixel and clipped."""
    c, s, u_min, v_min, _, _ = block_frame(h, w, vertical, skew)
    ht, wt = (w, h) if vertical else (h, w)
    c0, l0, c1, l1 = window
    xs, ys = [], []
    for u in (u_min + c0, u_min + c1):
        for v in (v_min + l0, v_min + l1):
            xs.append(u * c + v * s + wt / 2 - 0.5)
            ys.append(v * c - u * s + ht / 2 - 0.5)
    fx0, fx1 = max(0, math.floor(min(xs)) - 1), min(wt, math.floor(max(xs)) + 2)
    fy0, fy1 = max(0, math.floor(min(ys)) - 1), min(ht, math.floor(max(ys)) + 2)
    return (fy0, fx0, fy1, fx1) if vertical else (fx0, fy0, fx1, fy1)


def find_lines(img, rect, window, skew, direction="horizontal", min_ink=None, gap=None, min_height=None, polarity="auto"):
    """The windowed text block (rect, skew, window) of ``img`` -> dict(lines, threshold, ink, skew, detail): Otsu's threshold
    over the window's pixel set, polarity from 2 D <= n, the profile in bins k - l0 and indices j - c0, and the lines as
    oracle/skewed_blocks.find_lines gives them (integer rectangles when s is 0).  detail: the frame lines in window cells and
    the set's ink mask."""
    x0, y0, x1, y1 = rect
    vertical = direction == "vertical"
    g = B.grey(img[y0:y1, x0:x1])
    m = members(y1 - y0, x1 - x0, vertical, skew, window)
    vals = g[m]
    t = B.otsu(vals) if vals.size else 0
    if polarity == "auto":
        polarity = "dark" if 2 * int((vals <= t).sum()) <= vals.size else "light"
    ink = m & (g <= t if polarity == "dark" else g > t)
    c, s, u_min, v_min, L, M = block_frame(y1 - y0, x1 - x0, vertical, skew)
    inkf = ink.T if vertical else ink
    ht, wt = inkf.shape
    k, j, *_ = cells(ht, wt, c, s)
    c0, l0, c1, l1 = window
    kk, jj = k[inkf] - l0, j[inkf] - c0
    Lw, Mw = l1 - l0, c1 - c0
    r = np.bincount(kk, minlength=Lw)
    lo = np.full(Lw, np.iinfo(np.int64).max)
    hi = np.full(Lw, -1)
    np.minimum.at(lo, kk, jj)
    np.maximum.at(hi, kk, jj)
    frame_lines = SB._segment(r, lo, hi, Lw, Mw, min_ink, gap, min_height)
    shifted = [(c0 + a, l0 + b, c0 + e, l0 + f) for a, b, e, f in frame_lines]
    if s == 0:
        if vertical:
            lines = [(x0 + b, y0 + a, x0 + f, y0 + e) for a, b, e, f in shifted][::-1]
        else:
            lines = [(x0 + a, y0 + b, x0 + e, y0 + f) for a, b, e, f in shifted]
    elif vertical:
        O = (y0 + (y1 - y0) / 2, x0 + (x1 - x0) / 2)
        lines = []
        for q in shifted:
            tl, tr, bl = SB.corners(q, c, s, u_min, v_min, O)
            lines.append((tl[::-1], bl[::-1], tr[::-1]))
        lines = lines[::-1]
    else:
        O = (x0 + (x1 - x0) / 2, y0 + (y1 - y0) / 2)
        lines = [SB.corners(q, c, s, u_min, v_min, O) for q in shifted]
    return dict(lines=lines, threshold=t, ink=polarity, skew=float(skew), detail=dict(frame_lines=frame_lines, ink=ink))
