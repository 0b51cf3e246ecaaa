"""numpy twin of pipeline.restore_regions for pages that hold perspective regions (DESIGN.md section 7b, "Perspective text
regions"): each QuadRegion rectified and its restored line warped back onto its footprint with oracle.warp_perspective (OpenCV's
own warpPerspective, IPP off) through the fp64 maps of pipeline.quad_maps -- the same doubles the kernels get -- and feathered on
all four sides with the oriented regions' formula; rectangles and oriented regions composed exactly as oracle.oriented_regions
composes them.
TEST INFRASTRUCTURE ONLY."""
import numpy as np

from .oriented_regions import oriented_patch
from .regions import alpha, background, blend, resized_region
from .warp_perspective import warp_coords, warp_perspective_cubic_u8, warp_sample_u8


def rectify(img, region):
    """C = cv2.warpPerspective(img, M, (w_r, h_r), INTER_CUBIC | WARP_INVERSE_MAP, BORDER_REPLICATE): the quad's rectified
    crop, the image restore_images restores."""
    from marconet_b200.pipeline import quad_maps
    m = quad_maps(region, 1)
    return warp_perspective_cubic_u8(img, m.matrix, m.size)


def quad_footprint(t_shape, region, s, page_hw, feather):
    """Where a quad whose restored bytes have shape t_shape = (128, W_T, ...) lands on an image of page_hw = (H, W) output pixels
    at scale s: (box, xq, yq, mask, alpha) over the footprint's bounding box, as oracle.oriented_regions.oriented_footprint
    computes them, with cv2.warpPerspective's fixed-point T coordinates under the 3 x 3 N of the whole page as the destination
    (its column blocks start from the page's column 0)."""
    from marconet_b200.pipeline import quad_footprint_box, quad_maps
    th, tw = t_shape[:2]
    m = quad_maps(region, s, tw)
    box = quad_footprint_box(m, s, page_hw)
    xq, yq = warp_coords(m.page_map, np.arange(box[0], box[2]), np.arange(box[1], box[3]), page_hw[::-1])
    mask = (xq >= -16) & (xq < 32 * tw - 16) & (yq >= -16) & (yq < 32 * th - 16)
    if feather == 0:
        return box, xq, yq, mask, np.ones(xq.shape, np.float32)
    f32 = np.float32
    u = (xq + 16).astype(f32) / f32(32)                  # exact: both have at most 20 significant bits
    v = (yq + 16).astype(f32) / f32(32)
    du = np.multiply(f32(m.kx), np.minimum(u, np.subtract(f32(tw), u, dtype=f32)), dtype=f32)
    dv = np.multiply(f32(m.ky), np.minimum(v, np.subtract(f32(th), v, dtype=f32)), dtype=f32)
    return box, xq, yq, mask, np.minimum(f32(1), np.divide(np.minimum(du, dv), f32(feather), dtype=f32))


def quad_patch(t, region, s, page_hw, feather):
    """quad_footprint's (box, P, alpha, mask) for the restored bytes t (cv2.imwrite order), with P = cv2.warpPerspective(
    t[..., ::-1], N, (W, H), INTER_CUBIC | WARP_INVERSE_MAP, BORDER_REPLICATE) over the box."""
    box, xq, yq, mask, a = quad_footprint(t.shape, region, s, page_hw, feather)
    return box, warp_sample_u8(np.ascontiguousarray(t[..., ::-1]), xq, yq), a, mask


def compose(img, rects, srs, s, feather):
    """One image's result: img uint8 [H, W, 3], rects its regions -- (x0, y0, x1, y1) in source pixels,
    pipeline.OrientedRegions or pipeline.QuadRegions -- srs each region's restored bytes (restore_images' sr_u8, cv2.imwrite
    order) or None for a failed region, which keeps the background."""
    from marconet_b200.pipeline import OrientedRegion, QuadRegion
    out = background(img, s)
    for rect, t in zip(rects, srs):
        if t is None:
            continue
        if isinstance(rect, (OrientedRegion, QuadRegion)):
            patch = quad_patch if isinstance(rect, QuadRegion) else oriented_patch
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
