"""numpy twin of pipeline's perspective pages (DESIGN.md section 7b, "Perspective pages"): the page-corner search of
TextPage(quad="auto") -- Otsu's paper mask, its largest 4-connected component (scipy.ndimage.label), the monotone-chain hull of
that component's row ends and the brute-force largest quad on it -- and the blocks and lines of a quad page or block, found on its
rectified crop with oracle.pages and oracle.blocks and mapped back through the quad's homography.  Written from the definition,
not from the kernels.
TEST INFRASTRUCTURE ONLY."""
import numpy as np
from scipy import ndimage

from . import blocks as B
from . import pages as P
from .quad_regions import rectify


def paper(img, polarity="auto"):
    """(mask, t): the paper of a uint8 [H, W, 3] image, grey > t (grey <= t with polarity "light"), t Otsu's threshold."""
    g = B.grey(img)
    t = B.otsu(g)
    return (g <= t if polarity == "light" else g > t), t


def page_component(mask):
    """(label, size, members) of the 4-connected component of ``mask`` with the most pixels, ties to the smallest label, a
    component's label being the smallest raster index of its pixels; (-1, 0, None) when the mask is empty."""
    lab, n = ndimage.label(mask)
    if n == 0:
        return -1, 0, None
    first = np.full(n + 1, mask.size, np.int64)
    np.minimum.at(first, lab.ravel(), np.arange(mask.size))
    size = np.bincount(lab.ravel(), minlength=n + 1)
    k = 1 + int(np.lexsort((first[1:], -size[1:]))[0])
    return int(first[k]), int(size[k]), lab == k


def row_points(members):
    """The pixel-square corners of each row's ends, sorted by (y, x): for y from the first row to one past the last, the least
    left end and the largest right end + 1 over rows y - 1 and y."""
    rows = np.nonzero(members.any(axis=1))[0]
    y0, y1 = int(rows[0]), int(rows[-1])
    xl = {y: int(np.argmax(members[y])) for y in range(y0, y1 + 1)}
    xr = {y: members.shape[1] - 1 - int(np.argmax(members[y, ::-1])) for y in range(y0, y1 + 1)}
    pts = []
    for y in range(y0, y1 + 2):
        rs = [r for r in (y - 1, y) if y0 <= r <= y1]
        pts += [(min(xl[r] for r in rs), y), (max(xr[r] for r in rs) + 1, y)]
    return pts


def _cross(o, a, b):
    return (a[0] - o[0]) * (b[1] - o[1]) - (a[1] - o[1]) * (b[0] - o[0])


def monotone_chain(pts):
    """Andrew's monotone chain over points sorted by (y, x), collinear points dropped: the hull's vertices, the first sweep's
    chain from the first point, then the return sweep's."""
    h = []
    for p in pts:
        while len(h) >= 2 and _cross(h[-2], h[-1], p) <= 0:
            h.pop()
        h.append(p)
    lo = len(h) + 1
    for p in pts[-2::-1]:
        while len(h) >= lo and _cross(h[-2], h[-1], p) <= 0:
            h.pop()
        h.append(p)
    return h[:-1]


def largest_quad(hull):
    """(area2, (i, a, j, b)): the four hull vertices i < a < j < b of the largest doubled area, ties to the lexicographically
    smallest index tuple, by brute force: every diagonal i-j and every apex on each side."""
    v = np.array(hull, np.int64)
    k = len(v)
    best = (-1, None)
    for i in range(k - 3):
        d = v - v[i]
        c = np.abs(d[:, 0, None] * d[None, :, 1] - d[:, 1, None] * d[None, :, 0])    # c[m, j]: the doubled area of i, m, j
        m = np.arange(k)[:, None]
        j = np.arange(k)[None, :]
        left = np.where((m > i) & (m < j), c, -1)
        right = np.where(m > j, c, -1)
        a, b = left.argmax(axis=0), right.argmax(axis=0)
        s = left.max(axis=0) + right.max(axis=0)
        for jj in range(i + 2, k - 1):
            cand = (int(s[jj]), (i, int(a[jj]), jj, int(b[jj])))
            if cand[0] > best[0] or (cand[0] == best[0] and cand[1] < best[1]):
                best = cand
    return best


def order_corners(hull, idx):
    """The quad's vertices clockwise on screen (y down), from tl: the smallest x + y, then the smallest y."""
    i, a, j, b = idx
    cw = _cross(hull[i], hull[a], hull[j]) > 0
    c = [hull[i], hull[a if cw else b], hull[j], hull[b if cw else a]]
    s = min(range(4), key=lambda m: (c[m][0] + c[m][1], c[m][1], m))
    return [c[(s + m) % 4] for m in range(4)]


def find_corners(img, polarity="auto"):
    """The corner search of one image: dict(threshold, label, size, hull, idx, area2, quad), quad the corners tl, tr, br, bl as
    integer (x, y) points; hull [] and quad None when no pixel is paper."""
    mask, t = paper(img, polarity)
    label, size, members = page_component(mask)
    out = dict(threshold=t, label=label, size=size, hull=[], idx=None, area2=0, quad=None)
    if members is None:
        return out
    hull = monotone_chain(row_points(members))
    area2, idx = largest_quad(hull)
    return dict(out, hull=hull, idx=idx, area2=area2, quad=order_corners(hull, idx))


def accepted(res, shape):
    """The found quad as a QuadRegion of floats when it is a page: at least a quarter of the image and valid under _plan_quad;
    else None."""
    from marconet_b200.pipeline import QuadRegion, _plan_quad
    H, W = shape[:2]
    if res["quad"] is None or 2 * res["area2"] < H * W:
        return None
    q = QuadRegion(*((float(x), float(y)) for x, y in res["quad"]))
    try:
        _plan_quad(q, H, W, 1, "page")
    except ValueError:
        return None
    return q


def homography(quad):
    """Heckbert's unit square -> quad homography as rows (a, b, c), (d, e, f), (g, h, 1), in fp64."""
    (x0, y0), (x1, y1), (x2, y2), (x3, y3) = [(float(x), float(y)) for x, y in quad]
    sx, sy = x0 - x1 + x2 - x3, y0 - y1 + y2 - y3
    dx1, dx2, dy1, dy2 = x1 - x2, x3 - x2, y1 - y2, y3 - y2
    den = dx1 * dy2 - dx2 * dy1
    g = (sx * dy2 - sy * dx2) / den
    h = (dx1 * sy - dy1 * sx) / den
    return (x1 - x0 + g * x1, x3 - x0 + h * x3, x0), (y1 - y0 + g * y1, y3 - y0 + h * y3, y0), (g, h, 1.0)


def line_quad(quad, size, rect):
    """The line rectangle (x0, y0, x1, y1) of a quad's rectified crop of ``size`` (w_r, h_r) as image corners tl, tr, br, bl:
    H(x0 / w_r, y0 / h_r), H(x1 / w_r, y0 / h_r), H(x1 / w_r, y1 / h_r), H(x0 / w_r, y1 / h_r)."""
    (a, b, c), (d, e, f), (g, h, _) = homography(quad)
    w_r, h_r = size
    x0, y0, x1, y1 = rect

    def at(u, v):
        w = g * u + h * v + 1.0
        return ((a * u + b * v + c) / w, (d * u + e * v + f) / w)
    return (at(x0 / w_r, y0 / h_r), at(x1 / w_r, y0 / h_r), at(x1 / w_r, y1 / h_r), at(x0 / w_r, y1 / h_r))


def find_blocks(img, quad, direction="horizontal", polarity="auto", gap_x=None, gap_y=None):
    """The blocks of a quad page: oracle.pages.find_blocks on its whole rectified crop R.  Returns that dict, blocks and rejected
    being windows of R, with quad and size (w_r, h_r)."""
    R = rectify(img, quad)
    res = P.find_blocks(R, None, direction, polarity, gap_x, gap_y)
    return dict(res, quad=tuple((float(x), float(y)) for x, y in quad), size=(R.shape[1], R.shape[0]))


def find_lines(img, quad, window=None, direction="horizontal", min_ink=None, gap=None, min_height=None, polarity="auto"):
    """The lines of a quad block: oracle.blocks.find_lines on the window of its rectified crop R (all of R without one), each
    line's rectangle of R as its image corners (line_quad).  Returns that dict, lines as corner 4-tuples and ``rects`` the
    rectangles of R."""
    R = rectify(img, quad)
    size = (R.shape[1], R.shape[0])
    res = B.find_lines(R, window or (0, 0) + size, direction, min_ink, gap, min_height, polarity)
    return dict(res, rects=res["lines"], lines=[line_quad(quad, size, q) for q in res["lines"]])
