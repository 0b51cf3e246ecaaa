"""numpy twin of pipeline.find_blocks for pages with rules (DESIGN.md section 7b, "Ruled pages"): the rule pixels U of a page's
ink (its maximal row and column runs of at least the rule length), the XY-cut of oracle/pages.py on the ink without them, in
which a rule index is white and any white run holding one cuts, and blocks whose growth stops at a rule.  Written from the
definition, not from the kernels: plain run lengths and recursion.
TEST INFRASTRUCTURE ONLY."""
import numpy as np

from . import blocks as B
from . import pages as P
from .quad_regions import rectify


def default_rule_length(w, h):
    """The rule length of a w x h frame when none is given: max(32, min(w, h) // 16)."""
    return max(32, min(w, h) // 16)


def row_runs(mask, length):
    """The pixels of the boolean [h, w] ``mask`` that lie in a maximal run of ones at least ``length`` long in their row."""
    h, w = mask.shape
    flat = np.zeros((h, w + 1), np.int8)                 # a zero after every row: runs end at the row's end
    flat[:, :w] = mask
    d = np.diff(np.concatenate(([0], flat.ravel())))
    starts, ends = np.nonzero(d == 1)[0], np.nonzero(d == -1)[0]
    keep = ends - starts >= length
    mark = np.zeros(flat.size + 1, np.int64)
    np.add.at(mark, starts[keep], 1)
    np.add.at(mark, ends[keep], -1)
    return (np.cumsum(mark)[:flat.size] > 0).reshape(h, w + 1)[:, :w]


def rule_pixels(ink, length):
    """U: the ink pixels in a maximal row run or column run of at least ``length``."""
    return row_runs(ink, length) | row_runs(ink.T, length).T


def _attempt(ink, rule, rect, rows, g, vertical):
    """oracle.pages' attempt on the node ``rect`` with the layout ink ``ink`` (I'): an index is white when its ink is under
    max(1, extent // 128) or when it is a rule index (2 u >= extent, u its U pixels inside the node), and a white run between
    two ink indices cuts when it is at least g long or holds a rule index."""
    x0, y0, x1, y1 = rect
    axis = 1 if rows else 0
    ext = x1 - x0 if rows else y1 - y0
    p = ink[y0:y1, x0:x1].sum(axis=axis)
    r = 2 * rule[y0:y1, x0:x1].sum(axis=axis) >= ext
    nw = np.nonzero((p >= max(1, ext // 128)) & ~r)[0]
    if len(nw) == 0:
        return None
    rc = np.concatenate(([0], np.cumsum(r)))            # rule indices in [a, b): rc[b] - rc[a]
    at = [k for k in range(len(nw) - 1) if nw[k + 1] - nw[k] - 1 >= g or rc[nw[k + 1]] - rc[nw[k] + 1] > 0]
    starts = [int(nw[0])] + [int(nw[k + 1]) for k in at]
    ends = [int(nw[k]) + 1 for k in at] + [int(nw[-1]) + 1]
    lo = y0 if rows else x0
    if rows:
        spans = [(x0, lo + a, x1, lo + e) for a, e in zip(starts, ends)]
    else:
        spans = [(lo + a, y0, lo + e, y1) for a, e in zip(starts, ends)]
        if vertical:
            spans = spans[::-1]
    return spans[0] if len(spans) == 1 else None, spans if len(spans) > 1 else []


def xy_cut(ink, rule, vertical, g_x, g_y):
    """The leaves of the XY-cut of the layout ink ``ink`` with the rule pixels ``rule``, in reading order, as oracle.pages.xy_cut
    (the same levels, node bound and limit)."""
    h, w = ink.shape
    cap = min(P.MAX_NODES, (h + 1) * (w + 1) // 4)
    nodes = [((0, 0, w, h), not vertical, False, False)]
    for depth in range(P.LEVELS):
        if all(leaf for *_, leaf in nodes):
            break
        out = []
        for rect, rows, failed, leaf in nodes:
            if leaf:
                out.append((rect, rows, failed, True))
                continue
            res = _attempt(ink, rule, rect, rows, g_y if rows else g_x, vertical)
            if res is None:
                continue
            trimmed, children = res
            last = depth + 1 == P.LEVELS
            if children:
                out += [(c, not rows, False, last) for c in children]
            else:
                out.append((trimmed, not rows, True, failed or last))
        if len(out) > cap:
            raise ValueError(f"more than {P.MAX_NODES} nodes in one level")
        nodes = out
    return [rect for rect, *_ in nodes]


def _grow(rule, leaf, q):
    """A kept leaf (x0, y0, x1, y1) grown by q on each side and clipped to the page, each side stopping short of the nearest
    row (column) of its margin that holds a U pixel in the leaf's columns (rows)."""
    h, w = rule.shape
    x0, y0, x1, y1 = leaf
    top, bottom, left, right = max(0, y0 - q), min(h, y1 + q), max(0, x0 - q), min(w, x1 + q)
    hit = np.nonzero(rule[top:y0, x0:x1].any(axis=1))[0]
    top = top + int(hit[-1]) + 1 if len(hit) else top
    hit = np.nonzero(rule[y1:bottom, x0:x1].any(axis=1))[0]
    bottom = y1 + int(hit[0]) if len(hit) else bottom
    hit = np.nonzero(rule[y0:y1, left:x0].any(axis=0))[0]
    left = left + int(hit[-1]) + 1 if len(hit) else left
    hit = np.nonzero(rule[y0:y1, x1:right].any(axis=0))[0]
    right = x1 + int(hit[0]) if len(hit) else right
    return left, top, right, bottom


def find_blocks(img, rect=None, direction="horizontal", polarity="auto", gap_x=None, gap_y=None, rule_length=None):
    """oracle.pages.find_blocks of a page with rules: the same dict with rule_length (the length used: ``rule_length`` or
    default_rule_length of the crop) and rule_pixels (|U|).  Raises ValueError over a limit."""
    H, W = img.shape[:2]
    X0, Y0, X1, Y1 = rect if rect is not None else (0, 0, W, H)
    g = B.grey(img[Y0:Y1, X0:X1])
    t = B.otsu(g)
    if polarity == "auto":
        polarity = "dark" if 2 * int((g <= t).sum()) <= g.size else "light"
    ink = g <= t if polarity == "dark" else g > t
    h, w = ink.shape
    length = rule_length or default_rule_length(w, h)
    rule = rule_pixels(ink, length)
    ink = ink & ~rule
    vertical = direction == "vertical"
    out = dict(blocks=[], rejected=[], threshold=t, ink=polarity, text_size=0, gap_x=0, gap_y=0, rule_length=length,
               rule_pixels=int(rule.sum()))
    sizes = sorted(s for s in (max(x1 - x0, y1 - y0) for x0, y0, x1, y1 in xy_cut(ink, rule, vertical, 1, 1)) if s >= 2)
    if not sizes:
        return out
    S = sizes[(len(sizes) - 1) // 2]
    wide, narrow = S, max(1, S // 2)
    g_x = gap_x or (narrow if vertical else wide)
    g_y = gap_y or (wide if vertical else narrow)
    q = (min(g_x, g_y) - 1) // 2
    for x0, y0, x1, y1 in xy_cut(ink, rule, vertical, g_x, g_y):
        n = int(ink[y0:y1, x0:x1].sum())
        if 2 * n > (y1 - y0) * (x1 - x0) or min(y1 - y0, x1 - x0) < max(1, S // 3):
            out["rejected"].append((X0 + x0, Y0 + y0, X0 + x1, Y0 + y1))
        else:
            a, b, c, d = _grow(rule, (x0, y0, x1, y1), q)
            out["blocks"].append((X0 + a, Y0 + b, X0 + c, Y0 + d))
    if len(out["blocks"]) > P.MAX_BLOCKS:
        raise ValueError(f"{len(out['blocks'])} blocks exceed the {P.MAX_BLOCKS} a text page may hold")
    return dict(out, text_size=S, gap_x=g_x, gap_y=g_y)


def find_quad_blocks(img, quad, direction="horizontal", polarity="auto", gap_x=None, gap_y=None, rule_length=None):
    """The blocks of a quad page with rules: find_blocks on its whole rectified crop R (the default rule length of R), as
    oracle.quad_pages.find_blocks."""
    R = rectify(img, quad)
    res = find_blocks(R, None, direction, polarity, gap_x, gap_y, rule_length)
    return dict(res, quad=tuple((float(x), float(y)) for x, y in quad), size=(R.shape[1], R.shape[0]))
