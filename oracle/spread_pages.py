"""numpy twin of pipeline's book spreads (DESIGN.md section 7b, "Book spreads"): the spine of an open book, searched on the page
component and corners of oracle.quad_pages.find_corners -- each column's first and last row of the component, the deepest
top and bottom notch over the middle half of the quad's top and bottom edges, ties to the smallest column, exact in Python
integers -- and the spread's two halves, each flattened by oracle.flat_pages as a FlatPage with its quad given.  Written from
the definition, not from the kernels.
TEST INFRASTRUCTURE ONLY."""
import math

import numpy as np

from . import flat_pages as F
from . import quad_pages as QP


def column_extents(members):
    """(t, b): per column x of the boolean mask ``members``, its first row and its last row + 1; -1 where it holds no pixel."""
    has = members.any(axis=0)
    t = np.where(has, np.argmax(members, axis=0), -1)
    b = np.where(has, members.shape[0] - np.argmax(members[::-1], axis=0), -1)
    return t, b


def _cross(o, a, c):
    return (a[0] - o[0]) * (c[1] - o[1]) - (a[1] - o[1]) * (c[0] - o[0])


def _deepest(p, q, pts, sign):
    """(depth, point): the largest sign * cross(q - p, point - p) over ``pts`` (x, y) whose x lies in the middle half of p.x ..
    q.x, ties to the smallest x; (None, (-1, -1)) when none does."""
    best = (None, (-1, -1))
    span = q[0] - p[0]
    for x, y in pts:
        if 4 * (x - p[0]) >= span and 4 * (q[0] - x) >= span:
            d = sign * _cross(p, q, (x, y))
            if best[0] is None or d > best[0]:
                best = (d, (x, y))
    return best


def deep_enough(d, p, q):
    """The acceptance test of one notch: d > 0, d^2 >= 4 |q - p|^2 and 100 d >= |q - p|^2 (depth d / |q - p| at least
    max(2, |q - p| / 100) pixels)."""
    l2 = (q[0] - p[0]) ** 2 + (q[1] - p[1]) ** 2
    return d is not None and d > 0 and d * d >= 4 * l2 and 100 * d >= l2


def spine(members, quad):
    """The spine record of a page component ``members`` with corners ``quad`` (tl, tr, br, bl as integer (x, y)):
    dict(found, st, sb, D, E), D and E None when no column lies in their range."""
    tl, tr, br, bl = [(int(x), int(y)) for x, y in quad]
    t, b = column_extents(members)
    xs = [int(x) for x in np.nonzero(t >= 0)[0]]
    D, st = _deepest(tl, tr, [(x, int(t[x])) for x in xs], 1)
    E, sb = _deepest(bl, br, [(x, int(b[x])) for x in xs], -1)
    return dict(found=deep_enough(D, tl, tr) and deep_enough(E, bl, br), st=st, sb=sb, D=D, E=E)


def find_spine(img, polarity="auto"):
    """The corner search of oracle.quad_pages and the spine on its component: find_corners' dict with ``spine``; spine None when
    no pixel is paper."""
    res = QP.find_corners(img, polarity)
    if res["quad"] is None:
        return dict(res, spine=None)
    _, _, members = QP.page_component(QP.paper(img, polarity)[0])
    return dict(res, spine=spine(members, res["quad"]))


def halves(quad, st, sb):
    """The left and right halves (tl, st, sb, bl) and (st, tr, br, sb) as QuadRegions of floats."""
    from marconet_b200.pipeline import QuadRegion
    tl, tr, br, bl = quad
    return tuple(QuadRegion(*((float(x), float(y)) for x, y in q)) for q in ((tl, st, sb, bl), (st, tr, br, sb)))


def flatten(img, fp):
    """The spread dict of FlatPage ``fp`` (spread="auto") of ``img`` as pipeline.flatten_pages gives it: kind, quad, spine,
    depth and the two pages in reading order, each oracle.flat_pages.flatten of FlatPage(quad=half) with ``side``.  Raises
    ValueError without a page or a spine found."""
    res = find_spine(img, fp.polarity)
    if QP.accepted(res, img.shape) is None:
        raise ValueError("no page found")
    sp = res["spine"]
    if not sp["found"]:
        raise ValueError("no spread found")
    quad = [(int(x), int(y)) for x, y in res["quad"]]
    tl, tr, br, bl = quad
    depth = (sp["D"] / math.hypot(tr[0] - tl[0], tr[1] - tl[1]), sp["E"] / math.hypot(br[0] - bl[0], br[1] - bl[1]))
    pages = [dict(F.flatten(img, fp._replace(quad=q, spread=None)), side=side)
             for q, side in zip(halves(quad, sp["st"], sp["sb"]), ("left", "right"))]
    if fp.direction == "vertical":
        pages = pages[::-1]
    return dict(kind="spread", quad=tuple((float(x), float(y)) for x, y in quad), spine=(sp["st"], sp["sb"]), depth=depth,
                pages=pages)
