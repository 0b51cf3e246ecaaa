"""numpy twin of pipeline's page turns (DESIGN.md section 7b, "Page turns"): the vote statistics of each kept leaf of a page laid
out as oracle/panel_pages.py lays it out (rules, figures and panels as asked; directions from oracle/mixed_pages.py), the
page's scores and turn, and the turned quad, whose rectified crop (oracle/quad_pages.py) is the upright page.  Written from the
definition with plain loops, not from the kernels.
TEST INFRASTRUCTURE ONLY."""
import numpy as np

from . import blocks as B
from . import figure_pages as FP
from . import mixed_pages as MP
from . import panel_pages as PP
from . import ruled_pages as RP
from .quad_regions import rectify

# (page vertical, leaf vertical, D > 0) -> the turn a leaf's |D| votes for
VOTE = {(False, False, True): 0, (False, False, False): 180, (False, True, True): 270, (False, True, False): 90,
        (True, True, True): 0, (True, True, False): 180, (True, False, True): 90, (True, False, False): 270}


def turn_quad(rect, k):
    """The corners (tl, tr, br, bl) of the rectangle (x0, y0, x1, y1) (or of four corners) rotated right by k places."""
    if len(rect) == 4 and not hasattr(rect[0], "__len__"):
        x0, y0, x1, y1 = rect
        rect = [(x0, y0), (x1, y0), (x1, y1), (x0, y1)]
    pts = [(float(x), float(y)) for x, y in rect]
    return [pts[(m - k) % 4] for m in range(4)]


def leaf_stats(ink, rule, leaf, vertical):
    """(n, E_lo, E_hi) of the ungrown leaf (x0, y0, x1, y1) along its direction: its bands are the maximal runs of non-white
    rows (columns when ``vertical``) under oracle.mixed_pages.leaf_bands' white rule; band k spans [lo_k, hi_k] across, the
    least and largest column (row) of an ink pixel of its rows (columns) inside the leaf; E_lo = sum (lo_k - min lo),
    E_hi = sum (max hi - hi_k).  (0, 0, 0) without a band."""
    x0, y0, x1, y1 = leaf
    sub, u = ink[y0:y1, x0:x1], rule[y0:y1, x0:x1]
    if vertical:
        sub, u = sub.T, u.T
    n_idx, ext = sub.shape
    m = max(1, ext // 128)
    bands, cur = [], None
    for i in range(n_idx):
        nonwhite = int(sub[i].sum()) >= m and not 2 * int(u[i].sum()) >= ext
        if not nonwhite:
            cur = None
            continue
        cols = np.nonzero(sub[i])[0]
        lo, hi = int(cols[0]), int(cols[-1])
        if cur is None:
            cur = [lo, hi]
            bands.append(cur)
        else:
            cur[0], cur[1] = min(cur[0], lo), max(cur[1], hi)
    if not bands:
        return 0, 0, 0
    min_lo, max_hi = min(b[0] for b in bands), max(b[1] for b in bands)
    return len(bands), sum(b[0] - min_lo for b in bands), sum(max_hi - b[1] for b in bands)


def layout(img, rect=None, direction="horizontal", polarity="auto", gap_x=None, gap_y=None, rules=False, rule_length=None,
           figures=False, figure_size=None, panels=False, panel_size=None):
    """The kept pass-2 leaves of a page as oracle/panel_pages.py cuts it (panels only when asked), with the planes the direction
    test reads: [(leaf, ink, layout)] share one (ink, layout) pair; returns (leaves, ink, layout)."""
    H, W = img.shape[:2]
    X0, Y0, X1, Y1 = rect if rect is not None else (0, 0, W, H)
    g = B.grey(img[Y0:Y1, X0:X1])
    t = B.otsu(g)
    pol = polarity if polarity != "auto" else "dark" if 2 * int((g <= t).sum()) <= g.size else "light"
    I = g <= t if pol == "dark" else g > t
    h, w = I.shape
    rule = np.zeros_like(I)
    if rules:
        rule = RP.rule_pixels(I, rule_length or RP.default_rule_length(w, h))
    ink = I & ~rule
    vertical = direction == "vertical"
    leaves = RP.xy_cut(ink, rule, vertical, 1, 1)
    sizes = sorted(s for s in (max(x1 - x0, y1 - y0) for x0, y0, x1, y1 in leaves) if s >= 2)
    if not sizes:
        return [], ink, rule
    S = sizes[(len(sizes) - 1) // 2]
    pans = [r for r in leaves if PP.is_panel(ink, g, r, panel_size or S)] if panels else []
    F = np.zeros_like(ink)
    if figures:
        f = figure_size or 3 * S
        figs = [r for r in leaves if min(r[2] - r[0], r[3] - r[1]) >= f and r not in pans]
        assert len(figs) <= FP.MAX_FIGURES
        for x0, y0, x1, y1 in figs:
            F[y0:y1, x0:x1] = True
    lay = rule.copy()
    for x0, y0, x1, y1 in pans:
        ink[y0:y1, x0:x1] = ~I[y0:y1, x0:x1]
        edge = np.zeros((y1 - y0, x1 - x0), bool)
        edge[[0, -1], :] = edge[:, [0, -1]] = True
        ink[y0:y1, x0:x1] &= ~edge
        lay[y0:y1, x0:x1] |= edge
    ink &= ~F
    wide, narrow = S, max(1, S // 2)
    g_x = gap_x or (narrow if vertical else wide)
    g_y = gap_y or (wide if vertical else narrow)
    kept = []
    for x0, y0, x1, y1 in RP.xy_cut(ink, lay, vertical, g_x, g_y):
        n = int(ink[y0:y1, x0:x1].sum())
        if not (2 * n > (y1 - y0) * (x1 - x0) or min(y1 - y0, x1 - x0) < max(1, S // 3)):
            kept.append((x0, y0, x1, y1))
    return kept, ink, lay


def votes(img, rect=None, direction="horizontal", **kw):
    """dict(stats, directions, undecided, votes, turn) of a page: per kept leaf in reading order its (n, E_lo, E_hi) along its
    direction, its direction and whether its test was undecided; the scores (V_0, V_90, V_180, V_270) and the turn, the
    largest score's, ties to the least."""
    leaves, ink, lay = layout(img, rect, direction, **kw)
    out = dict(stats=[], directions=[], undecided=[], votes=[0, 0, 0, 0])
    for leaf in leaves:
        d, undecided = MP.leaf_direction(ink, lay, leaf, direction)
        n, e_lo, e_hi = leaf_stats(ink, lay, leaf, d == "vertical")
        out["stats"].append((n, e_lo, e_hi))
        out["directions"].append(d)
        out["undecided"].append(undecided)
        D = e_hi - e_lo
        if not undecided and n >= 2 and D != 0:
            out["votes"][VOTE[(direction == "vertical", d == "vertical", D > 0)] // 90] += abs(D)
    out["votes"] = tuple(out["votes"])
    out["turn"] = 90 * max(range(4), key=lambda k: (out["votes"][k], -k))
    return out


def upright(img, rect, turn):
    """The rectified crop of the rectangle's turned quad: np.rot90(crop, -turn // 90) for a page turned ``turn`` degrees."""
    return rectify(img, turn_quad(rect, turn // 90))
