"""numpy twin of pipeline.restore_regions' composition (DESIGN.md section 7b, "Text regions in whole images"): the cubic
background of the whole image, each region's restored line resized onto its rectangle, the feather ramp and the blend, with
every rounding spelled out as mn_resize_cubic_u8_batched and mn_composite_regions_u8 compute it.  The resizes are
oracle.image_ops.resize_cubic_u8 (OpenCV's own 8-bit INTER_CUBIC, IPP off); fx = dw/w, fy = dh/h reproduce cv2's dsize form.
TEST INFRASTRUCTURE ONLY."""
import numpy as np

from .image_ops import resize_cubic_u8


def background(img, s):
    """B = cv2.resize(img, (0, 0), fx=s, fy=s, interpolation=INTER_CUBIC): uint8 [s H, s W, 3]."""
    return resize_cubic_u8(img, s, s)


def resized_region(t, dw, dh):
    """P = cv2.resize(t[..., ::-1], (dw, dh), interpolation=INTER_CUBIC): a region's restored bytes (cv2.imwrite order) back in
    the caller's channel order, resized onto its dh x dw output rectangle."""
    t = np.ascontiguousarray(t[..., ::-1])
    return resize_cubic_u8(t, dw / t.shape[1], dh / t.shape[0])


def alpha(rect, page_hw, feather):
    """fp32 [Y1 - Y0, X1 - X0] feather weights of output rectangle rect = (X0, Y0, X1, Y1) on a page of page_hw = (H, W) output
    pixels: d = the distance to the nearest side that is not on the page border, alpha = min(1, fl((float)d + 0.5) / F); 1 when
    F = 0 or every side is on the border."""
    x0, y0, x1, y1 = rect
    ph, pw = page_hw
    xs = np.arange(x0, x1)[None, :]
    ys = np.arange(y0, y1)[:, None]
    d = np.full((y1 - y0, x1 - x0), np.iinfo(np.int64).max, np.int64)
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
