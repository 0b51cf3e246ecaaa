"""numpy twin of pipeline.find_blocks for pages with panels="auto" (DESIGN.md section 7b, "Reversed panels"): the pass-1 leaves of
at least the panel size p that are over half ink and flat-filled are panels; inside each, the layout ink is the page's paper
(J = not I) minus the rectangle's outline, which joins the rules, and the blocks found there take the opposite polarity.
Layered on oracle/ruled_pages.py (XY-cut, growth), oracle/figure_pages.py (figures) and oracle/mixed_pages.py (directions).
Written from the definition, not from the kernels.
TEST INFRASTRUCTURE ONLY."""
import numpy as np

from . import blocks as B
from . import figure_pages as FP
from . import mixed_pages as MP
from . import pages as P
from . import ruled_pages as RP
from .quad_regions import rectify

MAX_PANELS = 1024
FLAT = 8                                                # a flat fill: over half of its greys within FLAT of its mode


def flat(g, leaf):
    """Whether the rectangle (x0, y0, x1, y1) of the grey crop ``g`` is flat-filled: m its modal grey (ties to the smaller),
    more than half of its pixels have a grey in [m - 8, m + 8]."""
    x0, y0, x1, y1 = leaf
    hist = np.bincount(g[y0:y1, x0:x1].reshape(-1), minlength=256)
    m = int(np.argmax(hist))
    return 2 * int(hist[max(0, m - FLAT):m + FLAT + 1].sum()) > (y1 - y0) * (x1 - x0)


def is_panel(ink, g, leaf, p):
    """The panel test of a pass-1 leaf: shorter side at least p, over half ink (2 |I' & leaf| > h w) and flat."""
    x0, y0, x1, y1 = leaf
    h, w = y1 - y0, x1 - x0
    return min(h, w) >= p and 2 * int(ink[y0:y1, x0:x1].sum()) > h * w and flat(g, leaf)


def find_blocks(img, rect=None, direction="horizontal", polarity="auto", gap_x=None, gap_y=None, rules=False, rule_length=None,
                figures=False, figure_size=None, block_direction=False, panel_size=None):
    """oracle.pages.find_blocks of a page with panels="auto" (with ``rules`` oracle.ruled_pages', with ``figures``
    oracle.figure_pages', with ``block_direction`` oracle.mixed_pages'): the same dict with panel_size (the p used, 0 without a
    text size), panels (their rectangles in image coordinates, in leaf order) and polarities (each block's: the opposite of
    the page's ink for a block whose ungrown leaf lies inside a panel, else ``polarity``).  Raises ValueError over a limit."""
    H, W = img.shape[:2]
    X0, Y0, X1, Y1 = rect if rect is not None else (0, 0, W, H)
    g = B.grey(img[Y0:Y1, X0:X1])
    t = B.otsu(g)
    if polarity == "auto":
        ink_pol = "dark" if 2 * int((g <= t).sum()) <= g.size else "light"
    else:
        ink_pol = polarity
    I = g <= t if ink_pol == "dark" else g > t
    h, w = I.shape
    out = dict(blocks=[], rejected=[], threshold=t, ink=ink_pol, text_size=0, gap_x=0, gap_y=0)
    rule = np.zeros_like(I)
    if rules:
        length = rule_length or RP.default_rule_length(w, h)
        rule = RP.rule_pixels(I, length)
        out.update(rule_length=length, rule_pixels=int(rule.sum()))
    ink = I & ~rule
    vertical = direction == "vertical"
    if figures:
        out.update(figure_size=0, figures=[])
    if block_direction:
        out.update(block_direction="auto", undecided=[], directions=[])
    out.update(panel_size=0, panels=[], polarities=[])
    leaves = RP.xy_cut(ink, rule, vertical, 1, 1)
    sizes = sorted(s for s in (max(x1 - x0, y1 - y0) for x0, y0, x1, y1 in leaves) if s >= 2)
    if not sizes:
        return out
    S = sizes[(len(sizes) - 1) // 2]
    p = panel_size or S
    panels = [r for r in leaves if is_panel(ink, g, r, p)]
    if len(panels) > MAX_PANELS:
        raise ValueError(f"{len(panels)} panels exceed the {MAX_PANELS} a text page may hold")
    F = np.zeros_like(ink)
    if figures:
        f = figure_size or 3 * S
        figs = [r for r in leaves if min(r[2] - r[0], r[3] - r[1]) >= f and r not in panels]
        if len(figs) > FP.MAX_FIGURES:
            raise ValueError(f"{len(figs)} figures exceed the {FP.MAX_FIGURES} a text page may hold")
        for x0, y0, x1, y1 in figs:
            F[y0:y1, x0:x1] = True
        out.update(figure_size=f, figures=[(X0 + x0, Y0 + y0, X0 + x1, Y0 + y1) for x0, y0, x1, y1 in figs])
    layout = rule.copy()
    for x0, y0, x1, y1 in panels:                       # J = not I inside, the outline out of the ink and into U
        ink[y0:y1, x0:x1] = ~I[y0:y1, x0:x1]
        edge = np.zeros((y1 - y0, x1 - x0), bool)
        edge[[0, -1], :] = edge[:, [0, -1]] = True
        ink[y0:y1, x0:x1] &= ~edge
        layout[y0:y1, x0:x1] |= edge
    ink &= ~F
    out.update(panel_size=p, panels=[(X0 + x0, Y0 + y0, X0 + x1, Y0 + y1) for x0, y0, x1, y1 in panels])
    wide, narrow = S, max(1, S // 2)
    g_x = gap_x or (narrow if vertical else wide)
    g_y = gap_y or (wide if vertical else narrow)
    q = (min(g_x, g_y) - 1) // 2
    opposite = "light" if ink_pol == "dark" else "dark"
    for x0, y0, x1, y1 in RP.xy_cut(ink, layout, vertical, g_x, g_y):
        n = int(ink[y0:y1, x0:x1].sum())
        if 2 * n > (y1 - y0) * (x1 - x0) or min(y1 - y0, x1 - x0) < max(1, S // 3):
            out["rejected"].append((X0 + x0, Y0 + y0, X0 + x1, Y0 + y1))
            continue
        if block_direction:
            d, undecided = MP.leaf_direction(ink, layout, (x0, y0, x1, y1), direction)
            if undecided:
                out["undecided"].append(len(out["blocks"]))
            out["directions"].append(d)
        inside = any(a <= x0 and b <= y0 and x1 <= c and y1 <= e for a, b, c, e in panels)
        out["polarities"].append(opposite if inside else polarity)
        a, b, c, e = RP._grow(layout | F, (x0, y0, x1, y1), q)
        out["blocks"].append((X0 + a, Y0 + b, X0 + c, Y0 + e))
    if len(out["blocks"]) > P.MAX_BLOCKS:
        raise ValueError(f"{len(out['blocks'])} blocks exceed the {P.MAX_BLOCKS} a text page may hold")
    return dict(out, text_size=S, gap_x=g_x, gap_y=g_y)


def find_quad_blocks(img, quad, direction="horizontal", polarity="auto", gap_x=None, gap_y=None, rules=False, rule_length=None,
                     figures=False, figure_size=None, block_direction=False, panel_size=None):
    """The blocks of a quad page with panels="auto": find_blocks on its whole rectified crop R, blocks, panels (and figures)
    being rectangles of R, as oracle.quad_pages.find_blocks."""
    R = rectify(img, quad)
    res = find_blocks(R, None, direction, polarity, gap_x, gap_y, rules, rule_length, figures, figure_size, block_direction,
                      panel_size)
    return dict(res, quad=tuple((float(x), float(y)) for x, y in quad), size=(R.shape[1], R.shape[0]))
