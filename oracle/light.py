"""numpy twin of the even lighting of pipeline.flatten_pages (DESIGN.md section 7b, "Even lighting"): the grey closing of a page
with a k x k window cut to the page, the page divided by it as cv2.divide(F, B, scale=255) does, light ink through the
complement, the ink of a frame by steps 1-3 of "Text blocks", and oracle.flat_pages.flatten for evened pages.  Written from
the definition, not from the kernels.
TEST INFRASTRUCTURE ONLY."""
import numpy as np
from scipy import ndimage

from . import blocks as B
from . import curled_blocks as CB
from . import flat_pages as FP
from . import pages as P
from . import quad_pages as QP
from . import skewed_pages as SP
from .remap import remap_cubic_u8
from .warp_affine import warp_affine_cubic_u8


def window(w, h):
    """The default window of a w x h frame: max(3, 2 floor(min(w, h) / 40) + 1)."""
    return max(3, 2 * (min(w, h) // 40) + 1)


def _extreme_1d(a, k, axis, fn):
    """np.maximum or np.minimum over the window [i - k // 2, i + k // 2] cut to the array, along ``axis``: scipy's 1-D filter
    with the border filled by the operation's identity (0 for max, 255 for min), which no window can pick."""
    if fn is np.maximum:
        return ndimage.maximum_filter1d(a, k, axis=axis, mode="constant", cval=0)
    return ndimage.minimum_filter1d(a, k, axis=axis, mode="constant", cval=255)


def closing(page, k):
    """The grey closing of a uint8 [h, w, c] page, per channel: the min over the k x k window cut to the page of the max over
    the k x k window cut to the page."""
    d = _extreme_1d(_extreme_1d(page, k, 0, np.maximum), k, 1, np.maximum)
    return _extreme_1d(_extreme_1d(d, k, 0, np.minimum), k, 1, np.minimum)


def divide(f, b):
    """cv2.divide(f, b, scale=255) on uint8 arrays: rint(255 f / b) in fp64, half to even, 0 where b = 0, saturated."""
    f64, b64 = f.astype(np.float64), b.astype(np.float64)
    with np.errstate(divide="ignore", invalid="ignore"):
        q = np.rint(255.0 * f64 / b64)
    return np.where(b == 0, 0, np.minimum(q, 255)).astype(np.uint8)


def ink(frame, polarity="auto"):
    """"dark" or "light": the polarity given, or under "auto" the minority side of Otsu's threshold of the frame's grey value."""
    if polarity != "auto":
        return polarity
    g = B.grey(frame)
    t = B.otsu(g)
    return "dark" if 2 * int((g <= t).sum()) <= g.size else "light"


def even(page, k, polarity):
    """The evened page: divide(F, closing(F)) for dark ink, 255 - that of 255 - F for light ink."""
    if polarity == "light":
        return 255 - even(255 - page, k, "dark")
    return divide(page, closing(page, k))


def flatten(img, fp):
    """oracle.flat_pages.flatten for a FlatPage that may ask for light="even": dict(image, kind, size, quad | skew, lines,
    light_window, ink) as pipeline.flatten_pages gives it.  The corners of quad="auto" are found on the photo as it is; the
    frame (the crop, or R) is evened with the page's window and ink; the skew search, the blocks and the curled tracing run on
    the evened frame; and the flat page the photo gives with that geometry is evened alike (rect and quad pages without curl
    are the evened frame).  A page with light=None is oracle.flat_pages.flatten's."""
    from marconet_b200.pipeline import (CurvedRegion, QuadRegion, _quad_homography, flat_line_table, flat_strips,
                                        skew_flat_matrix)
    from marconet_b200 import ops
    if fp.light is None:
        return FP.flatten(img, fp)
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
        frame, kind, out = img[y0:y1, x0:x1], "rect", {}
    polarity = ink(frame, fp.polarity)
    k = fp.light_window or window(frame.shape[1], frame.shape[0])
    lit = dict(light_window=k, ink=polarity)
    seen = even(frame, k, polarity)
    if quad is None and fp.skew is not None:
        theta = float(fp.skew) if not isinstance(fp.skew, str) else SP.find_blocks(
            seen, None, fp.direction, fp.polarity, fp.gap_x, fp.gap_y, "auto", fp.max_skew)["skew"]
        c, s = ops.skew_cos_sin([theta])[0]
        m, size = skew_flat_matrix(x1 - x0, y1 - y0, c, s)
        flat = warp_affine_cubic_u8(frame, m, size)
        return dict(image=even(flat, k, polarity), kind="skew", size=size, skew=theta, **lit)
    h, w = frame.shape[:2]
    res = dict(out, image=np.ascontiguousarray(seen), kind=kind, size=(w, h), **lit)
    if fp.curve is None:
        return res
    blocks = []
    for b in P.find_blocks(seen, None, fp.direction, fp.polarity, fp.gap_x, fp.gap_y)["blocks"]:
        r = CB.find_lines(seen, b, polarity=fp.polarity, strips=flat_strips(fp.strips, b[2] - b[0]))
        if "error" in r:
            raise ValueError(f"block {b}: error {r['error']}")
        blocks.append((b, r["lines"]))
    res["lines"] = [q for _, ls in blocks for q in ls]
    if not any(isinstance(q, CurvedRegion) for q in res["lines"]):
        return res
    table = flat_line_table(blocks)
    if kind == "rect":
        mx, my = FP.maps(table, w, h, "rect", (x0, y0))
    else:
        (a, b, c), (d, e, f), (g, hh, _) = _quad_homography([tuple(p) for p in q])
        mx, my = FP.maps(table, w, h, "quad", (a, b, c, d, e, f, g, hh))
    res["image"] = even(remap_cubic_u8(img, mx, my), k, polarity)
    res["table"] = table
    return res
