"""numpy twin of pipeline.restore_regions for pages that hold oriented regions (DESIGN.md section 7b, "Oriented text regions"):
each oriented region rectified and its restored line warped back onto its footprint with oracle.warp_affine (OpenCV's own
warpAffine, IPP off) through the fp64 maps of pipeline.oriented_maps -- the same doubles the kernels get -- and feathered on
all four sides; rectangles composed exactly as oracle.regions composes them.
TEST INFRASTRUCTURE ONLY."""
import numpy as np

from .regions import alpha, background, blend, resized_region
from .warp_affine import warp_affine_cubic_u8, warp_coords, warp_sample_u8


def rectify(img, region):
    """C = cv2.warpAffine(img, M, (w_r, h_r), INTER_CUBIC | WARP_INVERSE_MAP, BORDER_REPLICATE): the oriented region's
    rectified crop, the image restore_images restores."""
    from marconet_b200.pipeline import oriented_maps
    m = oriented_maps(region, 1)
    return warp_affine_cubic_u8(img, m.matrix, m.size)


def oriented_footprint(t_shape, region, s, page_hw, feather):
    """Where an oriented region whose restored bytes have shape t_shape = (128, W_T, ...) lands on an image of page_hw = (H, W)
    output pixels at scale s: (box, xq, yq, mask, alpha) over the footprint's bounding box (X0, Y0, X1, Y1) -- cv2.warpAffine's
    fixed-point T coordinates (xq, yq) of every pixel of the box under N, the footprint mask -16 <= Xq < 32 W_T - 16,
    -16 <= Yq < 32 * 128 - 16, and alpha = min(1, fl(min(fl(kx min(u, W_T - u)), fl(ky min(v, 128 - v))) / F)) with
    u = (Xq + 16)/32, v = (Yq + 16)/32 (1 when F = 0)."""
    from marconet_b200.pipeline import footprint_box, oriented_maps
    th, tw = t_shape[:2]
    m = oriented_maps(region, s, tw)
    box = footprint_box(region, m, s, page_hw)
    xq, yq = warp_coords(m.page_map, np.arange(box[0], box[2]), np.arange(box[1], box[3]))
    mask = (xq >= -16) & (xq < 32 * tw - 16) & (yq >= -16) & (yq < 32 * th - 16)
    if feather == 0:
        return box, xq, yq, mask, np.ones(xq.shape, np.float32)
    f32 = np.float32
    u = (xq + 16).astype(f32) / f32(32)                  # exact: both have at most 20 significant bits
    v = (yq + 16).astype(f32) / f32(32)
    du = np.multiply(f32(m.kx), np.minimum(u, np.subtract(f32(tw), u, dtype=f32)), dtype=f32)
    dv = np.multiply(f32(m.ky), np.minimum(v, np.subtract(f32(th), v, dtype=f32)), dtype=f32)
    return box, xq, yq, mask, np.minimum(f32(1), np.divide(np.minimum(du, dv), f32(feather), dtype=f32))


def oriented_patch(t, region, s, page_hw, feather):
    """oriented_footprint's (box, P, alpha, mask) for the restored bytes t (cv2.imwrite order), with P = cv2.warpAffine(
    t[..., ::-1], N, (W, H), INTER_CUBIC | WARP_INVERSE_MAP, BORDER_REPLICATE) over the box."""
    box, xq, yq, mask, a = oriented_footprint(t.shape, region, s, page_hw, feather)
    return box, warp_sample_u8(np.ascontiguousarray(t[..., ::-1]), xq, yq), a, mask


def compose(img, rects, srs, s, feather):
    """One image's result: img uint8 [H, W, 3], rects its regions -- (x0, y0, x1, y1) in source pixels or
    pipeline.OrientedRegions -- srs each region's restored bytes (restore_images' sr_u8, cv2.imwrite order) or None for a failed
    region, which keeps the background."""
    from marconet_b200.pipeline import OrientedRegion
    out = background(img, s)
    for rect, t in zip(rects, srs):
        if t is None:
            continue
        if isinstance(rect, OrientedRegion):
            (x0, y0, x1, y1), p, a, mask = oriented_patch(t, rect, s, out.shape[:2], feather)
            sl = out[y0:y1, x0:x1]
            sl[mask] = blend(sl, p, a)[mask]
            continue
        x0, y0, x1, y1 = rect
        r = (s * x0, s * y0, s * x1, s * y1)
        p = resized_region(t, r[2] - r[0], r[3] - r[1])
        sl = out[r[1]:r[3], r[0]:r[2]]
        out[r[1]:r[3], r[0]:r[2]] = blend(sl, p, alpha(r, out.shape[:2], feather))
    return out
