"""numpy twin of pipeline.restore_regions' vertical text columns (DESIGN.md section 7b, "Vertical text columns"): the cell plan,
the layout of a column crop C into the horizontal line L, the line boxes, R, the inverse layout of the restored line T into the
column T_col, the mapping of boxes predicted on L back into C, and the composition of pages that hold columns among rectangles,
oriented regions and quads.  Written from the definition, not from pipeline.vertical_plan; the composition takes the fp64 maps
of pipeline.oriented_maps / quad_maps at T_col's size, as the kernels do.
TEST INFRASTRUCTURE ONLY."""
import math

import numpy as np

from . import warp_affine as WA
from . import warp_perspective as WP
from .oriented_regions import rectify as rectify_oriented
from .quad_regions import rectify as rectify_quad
from .regions import alpha, background, blend, resized_region


def cells(h_r, w_r, n=None, boxes=None):
    """The boundaries [c_0 = 0, ..., c_n = h_r]: from boxes (c_k = floor((y2_{k-1} + y1_k) / 2)), from n equal cells
    (c_k = (k h_r) // n), or with neither from n = clamp(round_half_even(h_r / w_r), 1, h_r)."""
    if boxes is not None:
        return [0] + [int(math.floor((boxes[k - 1][3] + boxes[k][1]) / 2)) for k in range(1, len(boxes))] + [h_r]
    if n is None:
        n = min(max(int(round(h_r / w_r)), 1), h_r)
    return [(k * h_r) // n for k in range(n + 1)]


def geometry(c):
    """(t, H_L, p) of boundaries c: t_k = c_{k+1} - c_k, H_L = max t_k, p_k = (H_L - t_k) // 2."""
    t = np.diff(np.asarray(c, np.int64))
    hl = int(t.max())
    return t, hl, (hl - t) // 2


def layout(C, c):
    """L [H_L, n w_r, 3]: L[i, k w_r + j] = C[c_k + clamp(i - p_k, 0, t_k - 1), j]."""
    t, hl, p = geometry(c)
    i = np.arange(hl)
    return np.concatenate([C[c[k] + np.clip(i - p[k], 0, t[k] - 1)] for k in range(len(t))], axis=1)


def line_boxes(c, w_r, boxes):
    """Box k of C -> [k w_r + x1, p_k + y1 - c_k, k w_r + x2, p_k + y2 - c_k] on L."""
    _, _, p = geometry(c)
    return [[k * w_r + b[0], p[k] + b[1] - c[k], k * w_r + b[2], p[k] + b[3] - c[k]] for k, b in enumerate(boxes)]


def R(y, hl):
    """round_half_even(y * (128 / H_L)), fp64."""
    return int(round(y * (128 / hl)))


def t_size(c, w_r):
    """(W_c, H_c) = (R(w_r), R(h_r))."""
    _, hl, _ = geometry(c)
    return R(w_r, hl), R(c[-1], hl)


def unlayout(T, c, w_r):
    """T_col [R(h_r), R(w_r), 3] of the restored line T [128, W_T, 3]: row i of cell k (R(c_k) <= i < R(c_{k+1})) reads T at row
    clamp(R(p_k) + i - R(c_k), R(p_k), R(p_k + t_k) - 1), column clamp(R(k w_r) + j, R(k w_r), min(R((k+1) w_r), W_T) - 1)."""
    t, hl, p = geometry(c)
    wc, hc = t_size(c, w_r)
    wt = T.shape[1]
    out = np.empty((hc, wc, 3), np.uint8)
    j = np.arange(wc)
    for k in range(len(t)):
        r0, r1 = R(c[k], hl), R(c[k + 1], hl)
        if r1 <= r0:
            continue
        lo, hi = R(p[k], hl), R(p[k] + t[k], hl) - 1
        rows = np.minimum(np.maximum(lo + np.arange(r1 - r0), lo), hi)
        clo, chi = R(k * w_r, hl), min(R((k + 1) * w_r, hl), wt) - 1
        cols = np.minimum(np.maximum(clo + j, clo), chi)
        out[r0:r1] = T[rows][:, cols]
    return out


def boxes_back(c, w_r, boxes):
    """Boxes on L -> C through the cell k that holds each box's centre: x - k w_r clipped to [0, w_r], y - p_k + c_k clipped to
    [c_k, c_{k+1}]."""
    t, _, p = geometry(c)
    out = []
    for b in boxes:
        k = int(np.clip(math.floor((b[0] + b[2]) / 2 / w_r), 0, len(t) - 1))
        cx = lambda v: min(max(v - k * w_r, 0), w_r)               # noqa: E731
        cy = lambda v: min(max(v - p[k] + c[k], c[k]), c[k + 1])   # noqa: E731
        out.append([cx(b[0]), cy(b[1]), cx(b[2]), cy(b[3])])
    return out


def crop(img, shape):
    """The column crop C of a VerticalRegion's shape: img[y0:y1, x0:x1] or the shape's rectified crop."""
    from marconet_b200.pipeline import OrientedRegion, QuadRegion
    if isinstance(shape, OrientedRegion):
        return rectify_oriented(img, shape)
    if isinstance(shape, QuadRegion):
        return rectify_quad(img, shape)
    x0, y0, x1, y1 = shape
    return np.ascontiguousarray(img[y0:y1, x0:x1])


def _warped_patch(t, region, s, page_hw, feather):
    """(box, P, alpha, mask) of an oriented region or quad whose restored bytes t have any height H_T: the composite of
    oracle.oriented_regions / oracle.quad_regions with N, kx, ky and the footprint box at (W_T, H_T) = t's size."""
    from marconet_b200.pipeline import (OrientedRegion, footprint_box, oriented_maps, quad_footprint_box, quad_maps)
    th, tw = t.shape[:2]
    if isinstance(region, OrientedRegion):
        m = oriented_maps(region, s, tw, th)
        box = footprint_box(region, m, s, page_hw, th)
        xq, yq = WA.warp_coords(m.page_map, np.arange(box[0], box[2]), np.arange(box[1], box[3]))
    else:
        m = quad_maps(region, s, tw, th)
        box = quad_footprint_box(m, s, page_hw, th)
        xq, yq = WP.warp_coords(m.page_map, np.arange(box[0], box[2]), np.arange(box[1], box[3]), page_hw[::-1])
    mask = (xq >= -16) & (xq < 32 * tw - 16) & (yq >= -16) & (yq < 32 * th - 16)
    f32 = np.float32
    if feather == 0:
        a = np.ones(xq.shape, f32)
    else:
        u = (xq + 16).astype(f32) / f32(32)
        v = (yq + 16).astype(f32) / f32(32)
        du = np.multiply(f32(m.kx), np.minimum(u, np.subtract(f32(tw), u, dtype=f32)), dtype=f32)
        dv = np.multiply(f32(m.ky), np.minimum(v, np.subtract(f32(th), v, dtype=f32)), dtype=f32)
        a = np.minimum(f32(1), np.divide(np.minimum(du, dv), f32(feather), dtype=f32))
    return box, WA.warp_sample_u8(np.ascontiguousarray(t[..., ::-1]), xq, yq), a, mask


def compose(img, regs, srs, s, feather):
    """One image's result: img uint8 [H, W, 3], regs its regions -- (x0, y0, x1, y1), pipeline.OrientedRegions, QuadRegions or
    VerticalRegions -- and srs the bytes each composes (restore_images' sr_u8, or a column's T_col; cv2.imwrite order), None
    for a failed region, which keeps the background."""
    from marconet_b200.pipeline import OrientedRegion, QuadRegion, VerticalRegion
    out = background(img, s)
    for reg, t in zip(regs, srs):
        if t is None:
            continue
        if isinstance(reg, VerticalRegion):
            reg = reg.shape
        if isinstance(reg, (OrientedRegion, QuadRegion)):
            (x0, y0, x1, y1), p, a, mask = _warped_patch(t, reg, s, out.shape[:2], feather)
            sl = out[y0:y1, x0:x1]
            sl[mask] = blend(sl, p, a)[mask]
            continue
        x0, y0, x1, y1 = reg
        r = (s * x0, s * y0, s * x1, s * y1)
        p = resized_region(t, r[2] - r[0], r[3] - r[1])
        sl = out[r[1]:r[3], r[0]:r[2]]
        out[r[1]:r[3], r[0]:r[2]] = blend(sl, p, alpha(r, out.shape[:2], feather))
    return out
