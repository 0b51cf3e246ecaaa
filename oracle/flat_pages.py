"""numpy twin of pipeline.flatten_pages (DESIGN.md section 7b, "Flat pages"): a page's frame (its crop, its crop warped upright
with oracle.warp_affine, or its rectified crop R with oracle.quad_pages), and for a curled page the dewarp field built from
the lines oracle.pages and oracle.curled_blocks find on that frame, composed with the frame's map and sampled with
oracle.remap.  The line table is pipeline.flat_line_table, shared with the pipeline as curve_lines is; the field and the maps
are built here in fp64, vectorised over pixels, in the operation order the definition fixes.  Written from the definition, not
from the kernels.
TEST INFRASTRUCTURE ONLY."""
import numpy as np

from . import curled_blocks as CB
from . import pages as P
from . import quad_pages as QP
from . import skewed_pages as SP
from .remap import remap_cubic_u8
from .warp_affine import warp_affine_cubic_u8


def column_values(lines, w):
    """(cover [n, w] bool, M [n, w] fp64): whether line k's block holds column x, and m_k at the column's centre."""
    from marconet_b200.pipeline import _bezier_1d
    xc = np.arange(w, dtype=np.float64) + 0.5
    n = len(lines)
    cover = np.zeros((n, w), bool)
    M = np.zeros((n, w), np.float64)
    for k, L in enumerate(lines):
        t = np.clip((xc - L[0]) / (L[1] - L[0]), 0.0, 1.0)
        M[k] = _bezier_1d(L[2:6], t)
        cover[k, int(L[7]):int(L[8])] = True
    return cover, M


def _rows(Y, Mx, yc):
    """The source rows of row centres yc in a column with (Y, M) pairs sorted by Y (at least one)."""
    n = len(Y)
    k = np.searchsorted(Y, yc, side="right") - 1
    above = yc + (Mx[0] - Y[0])
    below = yc + (Mx[-1] - Y[-1])
    kk = np.clip(k, 0, max(n - 2, 0))
    kn = np.minimum(kk + 1, n - 1)
    with np.errstate(divide="ignore", invalid="ignore"):
        mid = Mx[kk] + ((yc - Y[kk]) * (Mx[kn] - Mx[kk])) / (Y[kn] - Y[kk])
    return np.where(k < 0, above, np.where(k >= n - 1, below, mid))


def field(lines, w, h):
    """fp64 [h, w]: the source row of every frame pixel of a w x h frame under the line table ``lines`` (the identity without
    lines)."""
    yc = np.arange(h, dtype=np.float64) + 0.5
    src = np.repeat(yc[:, None], w, axis=1)
    if len(lines) == 0:
        return src
    cover, M = column_values(lines, w)
    Y = lines[:, 6]
    covered = cover.any(axis=0)
    for x in np.nonzero(covered)[0]:
        src[:, x] = _rows(Y[cover[:, x]], M[cover[:, x], x], yc)
    cols = np.nonzero(covered)[0]
    for x in np.nonzero(~covered)[0]:
        li, ri = np.searchsorted(cols, x) - 1, np.searchsorted(cols, x)
        l = int(cols[li]) if li >= 0 else -1
        r = int(cols[ri]) if ri < len(cols) else -1
        if l >= 0 and r >= 0:
            dl, dr = src[:, l] - yc, src[:, r] - yc
            d = dl + (float(x - l) * (dr - dl)) / float(r - l)
        elif l >= 0 or r >= 0:
            d = src[:, max(l, r)] - yc
        else:
            d = np.zeros_like(yc)
        src[:, x] = yc + d
    return src


def maps(lines, w, h, kind, m):
    """fp64 (mapx, mapy) [h, w] of a curled page: the field's frame point (xc, src) through the frame map (kind "rect" with m =
    (x0, y0), or "quad" with m = H's a .. h) minus 0.5."""
    xc = np.arange(w, dtype=np.float64)[None, :] + 0.5
    src = field(lines, w, h)
    if kind == "rect":
        X, Y = m[0] + xc + 0 * src, m[1] + src
    else:
        a, b, c, d, e, f, g, hh = (float(v) for v in m)
        u, v = xc / w, src / h
        den = (g * u + hh * v) + 1.0
        X, Y = ((a * u + b * v) + c) / den, ((d * u + e * v) + f) / den
    return X - 0.5, Y - 0.5


def flatten(img, fp):
    """The flat page of FlatPage ``fp`` of the uint8 [H, W, 3] image ``img``: dict(image, kind, size, quad | skew, lines) as
    pipeline.flatten_pages gives it.  Raises ValueError for a quad="auto" page without a page found or a block over a limit."""
    from marconet_b200.pipeline import (CurvedRegion, QuadRegion, _quad_homography, flat_line_table, flat_strips,
                                        skew_flat_matrix)
    from marconet_b200 import ops
    H, W = img.shape[:2]
    quad = fp.quad
    if isinstance(quad, str):
        quad = QP.accepted(QP.find_corners(img, fp.polarity), img.shape)
        if quad is None:
            raise ValueError("no page found")
    if quad is not None:
        q = QuadRegion(*((float(x), float(y)) for x, y in quad))
        frame, kind, out = QP.rectify(img, q), "quad", dict(quad=tuple(q))
    else:
        x0, y0, x1, y1 = fp.rect if fp.rect is not None else (0, 0, W, H)
        crop = img[y0:y1, x0:x1]
        if fp.skew is not None:
            theta = float(fp.skew) if not isinstance(fp.skew, str) else SP.find_blocks(
                img, (x0, y0, x1, y1), fp.direction, fp.polarity, fp.gap_x, fp.gap_y, "auto", fp.max_skew)["skew"]
            c, s = ops.skew_cos_sin([theta])[0]
            m, size = skew_flat_matrix(x1 - x0, y1 - y0, c, s)
            flat = warp_affine_cubic_u8(crop, m, size)
            return dict(image=flat, kind="skew", size=size, skew=theta)
        frame, kind, out = crop, "rect", {}
    h, w = frame.shape[:2]
    res = dict(out, image=np.ascontiguousarray(frame), kind=kind, size=(w, h))
    if fp.curve is None:
        return res
    blocks = []
    for b in P.find_blocks(frame, None, fp.direction, fp.polarity, fp.gap_x, fp.gap_y)["blocks"]:
        r = CB.find_lines(frame, b, polarity=fp.polarity, strips=flat_strips(fp.strips, b[2] - b[0]))
        if "error" in r:
            raise ValueError(f"block {b}: error {r['error']}")
        blocks.append((b, r["lines"]))
    res["lines"] = [q for _, ls in blocks for q in ls]
    if not any(isinstance(q, CurvedRegion) for q in res["lines"]):
        return res
    table = flat_line_table(blocks)
    if kind == "rect":
        mx, my = maps(table, w, h, "rect", (x0, y0))
    else:
        (a, b, c), (d, e, f), (g, hh, _) = _quad_homography([tuple(p) for p in q])
        mx, my = maps(table, w, h, "quad", (a, b, c, d, e, f, g, hh))
    res["image"] = remap_cubic_u8(img, mx, my)
    res["table"] = table
    return res
