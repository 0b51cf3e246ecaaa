"""numpy twin of pipeline.restore_regions for pages that hold curved regions (DESIGN.md section 7b, "Curved text regions"): each
CurvedRegion rectified by cv2.remap with its crop map (oracle.remap: OpenCV's own remap, IPP off) and its restored line put back
onto its footprint by inverting every page pixel onto T, by bisection along the curves, vectorised over pixels; fp64 elementwise
with every operation rounded on its own (numpy never contracts), through pipeline.curved_maps' column fractions and slopes --
the same doubles the kernels get.  Rectangles, oriented regions and quads are composed exactly as oracle.quad_regions composes
them.
TEST INFRASTRUCTURE ONLY."""
import numpy as np

from .oriented_regions import oriented_patch
from .quad_regions import quad_patch
from .regions import alpha, background, blend, resized_region
from .remap import remap_cubic_u8
from .warp_affine import warp_sample_u8

BISECTION_STEPS = 48


def bezier(p, t):
    """De Casteljau's point of the cubic Beziers p ([..., 4, 2], broadcast against t) at t: s = 1 - t and three levels of lerps
    fl(fl(s A) + fl(t B)) per coordinate.  Returns (x, y)."""
    p = np.asarray(p, np.float64)
    t = np.asarray(t, np.float64)
    s = 1.0 - t
    out = []
    for k in (0, 1):
        v = [p[..., j, k] for j in range(4)]
        a0, a1, a2 = s * v[0] + t * v[1], s * v[1] + t * v[2], s * v[2] + t * v[3]
        b0, b1 = s * a0 + t * a1, s * a1 + t * a2
        out.append(s * b0 + t * b1)
    return out[0], out[1]


def segments(maps):
    """fp64 [k, 4, 2] top and bottom control points of every segment."""
    k = len(maps.c) - 1
    top, bottom = np.asarray(maps.top, np.float64), np.asarray(maps.bottom, np.float64)
    idx = 3 * np.arange(k)[:, None] + np.arange(4)[None, :]
    return top[idx], bottom[idx]


def crop_map(maps):
    """fp64 (mapx, mapy) [h_r, w_r]: crop pixel (j, i) -> a = (j + 0.5)/w_r, b = (i + 0.5)/h_r, m the last segment with
    c_m <= a (at most k - 1), t = (a - c_m)/(c_{m+1} - c_m), x = fl(fl(fl(1 - b) T_m(t).x) + fl(b B_m(t).x)) - 0.5, y likewise."""
    (w_r, h_r), k = maps.size, len(maps.c) - 1
    c = np.asarray(maps.c, np.float64)
    a = (np.arange(w_r, dtype=np.float64) + 0.5) / w_r
    b = ((np.arange(h_r, dtype=np.float64) + 0.5) / h_r)[:, None]
    m = np.searchsorted(c[1:k], a, side="right")
    t = (a - c[m]) / (c[m + 1] - c[m])
    top, bot = segments(maps)
    tx, ty = bezier(top[m], t)
    bx, by = bezier(bot[m], t)
    return (1.0 - b) * tx + b * bx - 0.5, (1.0 - b) * ty + b * by - 0.5


def rectify(img, region):
    """C = cv2.remap(img, fl32(mapx), fl32(mapy), INTER_CUBIC, BORDER_REPLICATE): the curved region's rectified crop, the image
    restore_images restores."""
    from marconet_b200.pipeline import curved_maps
    mx, my = crop_map(curved_maps(region, 1))
    return remap_cubic_u8(img, mx, my)


def _side(top, bot, qx, qy, t):
    """g(t) = fl(fl(d.x (q.y - T.y)) - fl(d.y (q.x - T.x))), d = B(t) - T(t)."""
    tx, ty = bezier(top, t)
    bx, by = bezier(bot, t)
    return (bx - tx) * (qy - ty) - (by - ty) * (qx - tx)


def invert(maps, qx, qy):
    """The inverse of the band at image points (qx, qy) (fp64 arrays of one shape): (ok, m, t*, b).  The segments are tried in
    order; one whose control points' bounding box does not hold q is skipped, one whose g(0) < 0 and g(1) < 0 agree has no root,
    else 48 bisection steps mid = fl(0.5 fl(lo + hi)) (lo keeps g(0)'s sign), t* = fl(0.5 fl(lo + hi)) and
    b = fl(dot(q - T, d) / dot(d, d)) at t*; the first segment with 0 <= b <= 1 is accepted."""
    qx, qy = np.asarray(qx, np.float64).ravel(), np.asarray(qy, np.float64).ravel()
    n = qx.size
    ok = np.zeros(n, bool)
    mm, tt, bb = np.zeros(n, np.int64), np.zeros(n, np.float64), np.zeros(n, np.float64)
    tops, bots = segments(maps)
    for m, (top, bot) in enumerate(zip(tops, bots)):
        pts = np.concatenate([top, bot])
        x0, y0 = pts.min(0)
        x1, y1 = pts.max(0)
        idx = np.flatnonzero(~ok & (qx >= x0) & (qx <= x1) & (qy >= y0) & (qy <= y1))
        px, py = qx[idx], qy[idx]
        neg = _side(top, bot, px, py, np.zeros_like(px)) < 0
        root = neg != (_side(top, bot, px, py, np.ones_like(px)) < 0)
        idx, px, py, neg = idx[root], px[root], py[root], neg[root]
        lo, hi = np.zeros_like(px), np.ones_like(px)
        for _ in range(BISECTION_STEPS):
            mid = 0.5 * (lo + hi)
            keep = (_side(top, bot, px, py, mid) < 0) == neg
            lo, hi = np.where(keep, mid, lo), np.where(keep, hi, mid)
        t = 0.5 * (lo + hi)
        tx, ty = bezier(top, t)
        bx, by = bezier(bot, t)
        dx, dy, rx, ry = bx - tx, by - ty, px - tx, py - ty
        with np.errstate(divide="ignore", invalid="ignore"):
            b = (rx * dx + ry * dy) / (dx * dx + dy * dy)
        acc = (b >= 0) & (b <= 1)
        idx = idx[acc]
        ok[idx], mm[idx], tt[idx], bb[idx] = True, m, t[acc], b[acc]
    return ok, mm, tt, bb


def t_maps(maps, m, t, b, t_hw):
    """fp64 (u, v), T's pixel indices of inverted points: a = c_m + t (c_{m+1} - c_m), u = fl(a W_T) - 0.5, v = fl(b H_T) - 0.5."""
    c = np.asarray(maps.c, np.float64)
    th, tw = t_hw
    a = c[m] + t * (c[m + 1] - c[m])
    return a * float(tw) - 0.5, b * float(th) - 0.5


def t_coords(maps, m, t, b, t_hw):
    """(Xq, Yq) = rint(fl32(u) 32), rint(fl32(v) 32) of t_maps' (u, v): where cv2.remap(T[..., ::-1], fl32(u), fl32(v), ...)
    samples."""
    u, v = t_maps(maps, m, t, b, t_hw)
    f32 = np.float32
    xq = np.rint(np.multiply(u.astype(f32), f32(32), dtype=f32)).astype(np.int64)
    yq = np.rint(np.multiply(v.astype(f32), f32(32), dtype=f32)).astype(np.int64)
    return xq, yq


def curved_footprint(t_shape, region, s, page_hw, feather):
    """Where a curved region whose restored bytes have shape t_shape = (128, W_T, ...) lands on an image of page_hw = (H, W)
    output pixels at scale s: (box, xq, yq, mask, alpha) over pipeline.curved_footprint_box, with page pixel (X, Y) inverted at
    q = ((X + 0.5)/s, (Y + 0.5)/s), the footprint mask (a root accepted and -16 <= Xq < 32 W_T - 16, -16 <= Yq < 32 H_T - 16)
    and the oriented regions' feather with curved_maps' kx, ky."""
    from marconet_b200.pipeline import curved_footprint_box, curved_maps
    th, tw = t_shape[:2]
    m = curved_maps(region, s, tw, th)
    box = curved_footprint_box(region, s, page_hw)
    xs, ys = np.arange(box[0], box[2], dtype=np.float64), np.arange(box[1], box[3], dtype=np.float64)
    qx = np.broadcast_to(((xs + 0.5) / s)[None, :], (len(ys), len(xs)))
    qy = np.broadcast_to(((ys + 0.5) / s)[:, None], (len(ys), len(xs)))
    ok, mm, tt, bb = invert(m, qx, qy)
    xq, yq = t_coords(m, mm, tt, bb, (th, tw))
    xq, yq = np.where(ok, xq, 0).reshape(qx.shape), np.where(ok, yq, 0).reshape(qx.shape)
    mask = ok.reshape(qx.shape) & (xq >= -16) & (xq < 32 * tw - 16) & (yq >= -16) & (yq < 32 * th - 16)
    return box, xq, yq, mask, feather_alpha(xq, yq, (th, tw), m.kx, m.ky, feather)


def feather_alpha(xq, yq, t_hw, kx, ky, feather):
    """alpha = min(1, fl(min(fl(kx min(u, W_T - u)), fl(ky min(v, H_T - v))) / F)), u = (Xq + 16)/32, v = (Yq + 16)/32; 1 when
    F = 0 (the oriented regions' feather)."""
    th, tw = t_hw
    if feather == 0:
        return np.ones(xq.shape, np.float32)
    f32 = np.float32
    u = (xq + 16).astype(f32) / f32(32)                  # exact: both have at most 20 significant bits
    v = (yq + 16).astype(f32) / f32(32)
    du = np.multiply(f32(kx), np.minimum(u, np.subtract(f32(tw), u, dtype=f32)), dtype=f32)
    dv = np.multiply(f32(ky), np.minimum(v, np.subtract(f32(th), v, dtype=f32)), dtype=f32)
    return np.minimum(f32(1), np.divide(np.minimum(du, dv), f32(feather), dtype=f32))


def curved_patch(t, region, s, page_hw, feather):
    """curved_footprint's (box, P, alpha, mask) for the restored bytes t (cv2.imwrite order), P = remap's cubic sample of
    t[..., ::-1] at the fixed-point T coordinates."""
    box, xq, yq, mask, a = curved_footprint(t.shape, region, s, page_hw, feather)
    return box, warp_sample_u8(np.ascontiguousarray(t[..., ::-1]), xq, yq), a, mask


def compose(img, rects, srs, s, feather):
    """One image's result: img uint8 [H, W, 3], rects its regions -- (x0, y0, x1, y1) in source pixels, OrientedRegions,
    QuadRegions or CurvedRegions -- srs each region's restored bytes (restore_images' sr_u8, cv2.imwrite order) or None for a
    failed region, which keeps the background."""
    from marconet_b200.pipeline import CurvedRegion, OrientedRegion, QuadRegion
    out = background(img, s)
    for rect, t in zip(rects, srs):
        if t is None:
            continue
        if isinstance(rect, (OrientedRegion, QuadRegion, CurvedRegion)):
            patch = curved_patch if isinstance(rect, CurvedRegion) else quad_patch if isinstance(rect, QuadRegion) else \
                oriented_patch
            (x0, y0, x1, y1), p, a, mask = patch(t, rect, s, out.shape[:2], feather)
            sl = out[y0:y1, x0:x1]
            sl[mask] = blend(sl, p, a)[mask]
            continue
        x0, y0, x1, y1 = rect
        r = (s * x0, s * y0, s * x1, s * y1)
        p = resized_region(t, r[2] - r[0], r[3] - r[1])
        sl = out[r[1]:r[3], r[0]:r[2]]
        out[r[1]:r[3], r[0]:r[2]] = blend(sl, p, alpha(r, out.shape[:2], feather))
    return out
