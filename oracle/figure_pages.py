"""numpy twin of pipeline.find_blocks for pages with figures (DESIGN.md section 7b, "Figures"): the pass-1 leaves of a page whose
shorter side is at least the figure size f are its figures; their rectangles F leave the ink before pass 2, and blocks stop
growing at them as at rules.  Written from the definition, not from the kernels, with oracle/ruled_pages.py's XY-cut and growth.
TEST INFRASTRUCTURE ONLY."""
import numpy as np

from . import blocks as B
from . import pages as P
from . import ruled_pages as RP
from .quad_regions import rectify

MAX_FIGURES = 1024


def find_blocks(img, rect=None, direction="horizontal", polarity="auto", gap_x=None, gap_y=None, rules=False, rule_length=None,
                figure_size=None):
    """oracle.pages.find_blocks (oracle.ruled_pages.find_blocks with ``rules``) of a page with figures: the same dict with
    figure_size (the f used: ``figure_size`` or 3 S; 0 without a text size) and figures (their rectangles in image
    coordinates, in leaf order).  Raises ValueError over a limit."""
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
    out.update(figure_size=0, figures=[])
    leaves = RP.xy_cut(ink, rule, vertical, 1, 1)
    sizes = sorted(s for s in (max(x1 - x0, y1 - y0) for x0, y0, x1, y1 in leaves) if s >= 2)
    if not sizes:
        return out
    S = sizes[(len(sizes) - 1) // 2]
    f = figure_size or 3 * S
    figures = [r for r in leaves if min(r[2] - r[0], r[3] - r[1]) >= f]
    if len(figures) > MAX_FIGURES:
        raise ValueError(f"{len(figures)} figures exceed the {MAX_FIGURES} a text page may hold")
    F = np.zeros_like(ink)
    for x0, y0, x1, y1 in figures:
        F[y0:y1, x0:x1] = True
    ink = ink & ~F
    out.update(figure_size=f, figures=[(X0 + x0, Y0 + y0, X0 + x1, Y0 + y1) for x0, y0, x1, y1 in figures])
    wide, narrow = S, max(1, S // 2)
    g_x = gap_x or (narrow if vertical else wide)
    g_y = gap_y or (wide if vertical else narrow)
    q = (min(g_x, g_y) - 1) // 2
    for x0, y0, x1, y1 in RP.xy_cut(ink, rule, vertical, g_x, g_y):
        n = int(ink[y0:y1, x0:x1].sum())
        if 2 * n > (y1 - y0) * (x1 - x0) or min(y1 - y0, x1 - x0) < max(1, S // 3):
            out["rejected"].append((X0 + x0, Y0 + y0, X0 + x1, Y0 + y1))
        else:
            a, b, c, d = RP._grow(rule | F, (x0, y0, x1, y1), q)
            out["blocks"].append((X0 + a, Y0 + b, X0 + c, Y0 + d))
    if len(out["blocks"]) > P.MAX_BLOCKS:
        raise ValueError(f"{len(out['blocks'])} blocks exceed the {P.MAX_BLOCKS} a text page may hold")
    return dict(out, text_size=S, gap_x=g_x, gap_y=g_y)


def find_quad_blocks(img, quad, direction="horizontal", polarity="auto", gap_x=None, gap_y=None, rules=False, rule_length=None,
                     figure_size=None):
    """The blocks of a quad page with figures: find_blocks on its whole rectified crop R, figures and blocks being rectangles of
    R, as oracle.quad_pages.find_blocks."""
    R = rectify(img, quad)
    res = find_blocks(R, None, direction, polarity, gap_x, gap_y, rules, rule_length, figure_size)
    return dict(res, quad=tuple((float(x), float(y)) for x, y in quad), size=(R.shape[1], R.shape[0]))
