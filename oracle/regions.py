"""numpy twin of pipeline.restore_regions' composition (DESIGN.md section 7b, "Text regions in whole images"): the cubic
background of the whole image, each region's restored line resized onto its rectangle, the feather ramp and the blend, with
every rounding spelled out as mn_resize_cubic_u8_batched and mn_composite_regions_u8 compute it.  The resizes are
oracle.image_ops.resize_cubic_u8 (OpenCV's own 8-bit INTER_CUBIC, IPP off); fx = dw/w, fy = dh/h reproduce cv2's dsize form.
TEST INFRASTRUCTURE ONLY."""
import numpy as np

from .image_ops import resize_cubic_rows, resize_cubic_u8


def background(img, s):
    """B = cv2.resize(img, (0, 0), fx=s, fy=s, interpolation=INTER_CUBIC): uint8 [s H, s W, 3]."""
    return resize_cubic_u8(img, s, s)


def resized_region(t, dw, dh):
    """P = cv2.resize(t[..., ::-1], (dw, dh), interpolation=INTER_CUBIC): a region's restored bytes (cv2.imwrite order) back in
    the caller's channel order, resized onto its dh x dw output rectangle."""
    t = np.ascontiguousarray(t[..., ::-1])
    return resize_cubic_u8(t, dw / t.shape[1], dh / t.shape[0])


def alpha(rect, page_hw, feather, box=None):
    """fp32 [Y1 - Y0, X1 - X0] feather weights of output rectangle rect = (X0, Y0, X1, Y1) on a page of page_hw = (H, W) output
    pixels: d = the distance to the nearest side that is not on the page border, alpha = min(1, fl((float)d + 0.5) / F); 1 when
    F = 0 or every side is on the border.  box: only the pixels of this part (x0, y0, x1, y1) of the rectangle."""
    x0, y0, x1, y1 = rect
    bx0, by0, bx1, by1 = rect if box is None else box
    ph, pw = page_hw
    xs = np.arange(bx0, bx1)[None, :]
    ys = np.arange(by0, by1)[:, None]
    d = np.full((by1 - by0, bx1 - bx0), np.iinfo(np.int64).max, np.int64)
    for counts, dist in ((x0 > 0, xs - x0), (x1 < pw, x1 - 1 - xs), (y0 > 0, ys - y0), (y1 < ph, y1 - 1 - ys)):
        if counts:
            d = np.minimum(d, np.broadcast_to(dist, d.shape))
    if feather == 0 or not (x0 > 0 or x1 < pw or y0 > 0 or y1 < ph):
        return np.ones(d.shape, np.float32)
    a = np.divide(np.add(d.astype(np.float32), np.float32(0.5), dtype=np.float32), np.float32(feather), dtype=np.float32)
    return np.minimum(a, np.float32(1))


def blend(out, p, a):
    """sat_u8(rint_half_even(fl(fl(a P) + fl(fl(1 - a) out)))), every fp32 operation rounded on its own."""
    a = a[..., None]
    x = np.multiply(a, p.astype(np.float32), dtype=np.float32)
    y = np.multiply(np.subtract(np.float32(1), a, dtype=np.float32), out.astype(np.float32), dtype=np.float32)
    return np.clip(np.rint(np.add(x, y, dtype=np.float32)), 0, 255).astype(np.uint8)


def compose(img, rects, srs, s, feather):
    """One image's result: img uint8 [H, W, 3], rects its regions (x0, y0, x1, y1) in source pixels, srs each region's restored
    bytes (restore_images' sr_u8, cv2.imwrite order) or None for a failed region, which keeps the background."""
    out = background(img, s)
    for (x0, y0, x1, y1), t in zip(rects, srs):
        if t is None:
            continue
        r = (s * x0, s * y0, s * x1, s * y1)
        p = resized_region(t, r[2] - r[0], r[3] - r[1])
        sl = out[r[1]:r[3], r[0]:r[2]]
        out[r[1]:r[3], r[0]:r[2]] = blend(sl, p, alpha(r, out.shape[:2], feather))
    return out


def clip_box(box, window):
    """The part of box (x0, y0, x1, y1) inside window (same form), or None when they do not meet."""
    b = (max(box[0], window[0]), max(box[1], window[1]), min(box[2], window[2]), min(box[3], window[3]))
    return b if b[0] < b[2] and b[1] < b[3] else None


def rect_patch(t, rect, s, page_hw, feather, window=None):
    """A rectangle's (box, P, alpha, mask) as compose composes it, over the part ``box`` of its output rectangle inside
    ``window`` (the whole rectangle when None; box None when they do not meet): P the rows and columns of the cubic resize of t
    (channels flipped back) onto the whole rectangle that fall in box."""
    x0, y0, x1, y1 = rect
    r = (s * x0, s * y0, s * x1, s * y1)
    box = r if window is None else clip_box(r, window)
    if box is None:
        return None, None, None, None
    tt = np.ascontiguousarray(t[..., ::-1])
    p = resize_cubic_rows(tt, (r[2] - r[0], r[3] - r[1]), np.arange(box[1], box[3]) - r[1], np.arange(box[0], box[2]) - r[0])
    return box, p, alpha(r, page_hw, feather, box), np.ones(p.shape[:2], bool)


def compose_window_with(patch, background_window, origin, page_hw, rects, srs, s, feather):
    """compose restricted to one window of the page, every coordinate the page's own: background_window uint8 [h, w, 3] holds
    the page bytes of columns origin[0] .. origin[0] + w and rows origin[1] .. origin[1] + h of a page of page_hw = (H, W) output
    pixels, and the regions are composed over it in order.  patch(t, rect, s, page_hw, feather, window) gives a region's
    (box, P, alpha, mask) inside the window (box None when it does not meet it)."""
    out = np.array(background_window, np.uint8, copy=True)
    ox, oy = origin
    window = (ox, oy, ox + out.shape[1], oy + out.shape[0])
    for rect, t in zip(rects, srs):
        if t is None:
            continue
        box, p, a, mask = patch(t, rect, s, page_hw, feather, window)
        if box is None:
            continue
        sl = out[box[1] - oy:box[3] - oy, box[0] - ox:box[2] - ox]
        sl[mask] = blend(sl, p, a)[mask]
    return out


def compose_window(background_window, origin, page_hw, rects, srs, s, feather):
    """compose over one window of the page (compose_window_with): rects (x0, y0, x1, y1) in source pixels."""
    return compose_window_with(rect_patch, background_window, origin, page_hw, rects, srs, s, feather)
