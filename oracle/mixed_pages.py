"""numpy twin of pipeline.find_blocks for pages with block_direction="auto" (DESIGN.md section 7b, "Mixed directions"): the
blocks of oracle/pages.py (with the rules of oracle/ruled_pages.py and the figures of oracle/figure_pages.py when asked), and
each kept leaf's own direction from the row and column bands of its ink.  Written from the definition, not from the kernels:
plain run lengths over the leaf's profiles.
TEST INFRASTRUCTURE ONLY."""
import numpy as np

from . import blocks as B
from . import figure_pages as FP
from . import pages as P
from . import ruled_pages as RP
from .quad_regions import rectify


def bands(nw):
    """(n, b, G) of a boolean profile of non-white indices: the number of bands (maximal runs of non-white indices), the longest
    and the white indices between the first and the last non-white one; (0, 0, 0) when none is non-white."""
    idx = np.nonzero(nw)[0]
    if len(idx) == 0:
        return 0, 0, 0
    run = nw[idx[0]:idx[-1] + 1].astype(np.int8)
    d = np.diff(np.concatenate(([0], run, [0])))
    starts, ends = np.nonzero(d == 1)[0], np.nonzero(d == -1)[0]
    return len(starts), int((ends - starts).max()), int(len(run) - run.sum())


def leaf_bands(ink, rule, leaf):
    """((n_r, b_r, G_y), (n_c, b_c, G_x)) of the ungrown leaf (x0, y0, x1, y1): a row is white when its ink is under
    max(1, w // 128), a column when under max(1, h // 128), and on a ruled page a rule index (2 u >= the extent, u its U
    pixels in the leaf) is white too, as in the XY-cut."""
    x0, y0, x1, y1 = leaf
    h, w = y1 - y0, x1 - x0
    sub, u = ink[y0:y1, x0:x1], rule[y0:y1, x0:x1]
    rows = (sub.sum(axis=1) >= max(1, w // 128)) & ~(2 * u.sum(axis=1) >= w)
    cols = (sub.sum(axis=0) >= max(1, h // 128)) & ~(2 * u.sum(axis=0) >= h)
    return bands(rows), bands(cols)


def decide(h, w, row_bands, col_bands):
    """"horizontal", "vertical" or None (undecided) for a leaf of h x w with its row and column bands: horizontal iff A > B and
    vertical iff A < B, (A, B) = (w, h) for one band each way, (2 b_c, h) for one row band and more column bands, (w, 2 b_r)
    for one column band and more row bands, and (G_y (n_c - 1), G_x (n_r - 1)) for a grid, its mean gap between row bands
    against its mean gap between column bands; undecided when A = B or a profile has no band."""
    (nr, br, gy), (nc, bc, gx) = row_bands, col_bands
    if nr == 0 or nc == 0:
        return None
    if nr == 1 and nc == 1:
        a, b = w, h
    elif nr == 1:
        a, b = 2 * bc, h
    elif nc == 1:
        a, b = w, 2 * br
    else:
        a, b = gy * (nc - 1), gx * (nr - 1)
    return None if a == b else "horizontal" if a > b else "vertical"


def leaf_direction(ink, rule, leaf, direction):
    """(the leaf's direction, whether its test was undecided and it took the page's ``direction``)."""
    x0, y0, x1, y1 = leaf
    d = decide(int(y1 - y0), int(x1 - x0), *leaf_bands(ink, rule, leaf))
    return (direction, True) if d is None else (d, False)


def find_blocks(img, rect=None, direction="horizontal", polarity="auto", gap_x=None, gap_y=None, rules=False, rule_length=None,
                figures=False, figure_size=None):
    """oracle.pages.find_blocks (with ``rules`` oracle.ruled_pages', with ``figures`` oracle.figure_pages') of a page with
    block_direction="auto": the same dict with block_direction ("auto"), directions (each block's) and undecided (the indices
    of the blocks that took the page's direction).  Raises ValueError over a limit."""
    H, W = img.shape[:2]
    X0, Y0, X1, Y1 = rect if rect is not None else (0, 0, W, H)
    g = B.grey(img[Y0:Y1, X0:X1])
    t = B.otsu(g)
    if polarity == "auto":
        polarity = "dark" if 2 * int((g <= t).sum()) <= g.size else "light"
    ink = g <= t if polarity == "dark" else g > t
    h, w = ink.shape
    out = dict(blocks=[], rejected=[], threshold=t, ink=polarity, text_size=0, gap_x=0, gap_y=0)
    rule = np.zeros_like(ink)
    if rules:
        length = rule_length or RP.default_rule_length(w, h)
        rule = RP.rule_pixels(ink, length)
        out.update(rule_length=length, rule_pixels=int(rule.sum()))
    ink = ink & ~rule
    vertical = direction == "vertical"
    if figures:
        out.update(figure_size=0, figures=[])
    out.update(block_direction="auto", undecided=[], directions=[])
    leaves = RP.xy_cut(ink, rule, vertical, 1, 1)
    sizes = sorted(s for s in (max(x1 - x0, y1 - y0) for x0, y0, x1, y1 in leaves) if s >= 2)
    if not sizes:
        return out
    S = sizes[(len(sizes) - 1) // 2]
    F = np.zeros_like(ink)
    if figures:
        f = figure_size or 3 * S
        figs = [r for r in leaves if min(r[2] - r[0], r[3] - r[1]) >= f]
        if len(figs) > FP.MAX_FIGURES:
            raise ValueError(f"{len(figs)} figures exceed the {FP.MAX_FIGURES} a text page may hold")
        for x0, y0, x1, y1 in figs:
            F[y0:y1, x0:x1] = True
        ink = ink & ~F
        out.update(figure_size=f, figures=[(X0 + x0, Y0 + y0, X0 + x1, Y0 + y1) for x0, y0, x1, y1 in figs])
    wide, narrow = S, max(1, S // 2)
    g_x = gap_x or (narrow if vertical else wide)
    g_y = gap_y or (wide if vertical else narrow)
    q = (min(g_x, g_y) - 1) // 2
    for x0, y0, x1, y1 in RP.xy_cut(ink, rule, vertical, g_x, g_y):
        n = int(ink[y0:y1, x0:x1].sum())
        if 2 * n > (y1 - y0) * (x1 - x0) or min(y1 - y0, x1 - x0) < max(1, S // 3):
            out["rejected"].append((X0 + x0, Y0 + y0, X0 + x1, Y0 + y1))
            continue
        d, undecided = leaf_direction(ink, rule, (x0, y0, x1, y1), direction)
        if undecided:
            out["undecided"].append(len(out["blocks"]))
        out["directions"].append(d)
        a, b, c, e = RP._grow(rule | F, (x0, y0, x1, y1), q)
        out["blocks"].append((X0 + a, Y0 + b, X0 + c, Y0 + e))
    if len(out["blocks"]) > P.MAX_BLOCKS:
        raise ValueError(f"{len(out['blocks'])} blocks exceed the {P.MAX_BLOCKS} a text page may hold")
    return dict(out, text_size=S, gap_x=g_x, gap_y=g_y)


def find_quad_blocks(img, quad, direction="horizontal", polarity="auto", gap_x=None, gap_y=None, rules=False, rule_length=None,
                     figures=False, figure_size=None):
    """The blocks of a quad page with block_direction="auto": find_blocks on its whole rectified crop R, blocks (and figures)
    being rectangles of R, as oracle.quad_pages.find_blocks."""
    R = rectify(img, quad)
    res = find_blocks(R, None, direction, polarity, gap_x, gap_y, rules, rule_length, figures, figure_size)
    return dict(res, quad=tuple((float(x), float(y)) for x, y in quad), size=(R.shape[1], R.shape[0]))
