"""Generates tests/golden/vertical_regions.npz: a seeded synthetic portrait page (360 x 128) with six regions -- a rectangle column
whose characters sit at unequal pitch, a long rectangle column of 24 cells whose laid-out line is wider than the 32x512 LQ canvas,
a column tilted a few degrees (pipeline.OrientedRegion), a column seen in perspective (pipeline.QuadRegion), a one-cell column
and a horizontal rectangle line that overlaps the long column -- every column given as a pipeline.VerticalRegion with given
labels and boxes in its crop's frame.  Each oriented or quad column is rectified with live cv2 (IPP off); each column is laid out
by oracle/vertical_regions.py, its line restored on the CPU by the data flow of the reference's test_sr.py with the reference's
UNMODIFIED modules (make_golden_regions.restore_region) and put back into a column by the twin; the page is composed at s = 4,
F = 8 with live cv2 (background, cv2.resize of each rectangle's bytes, cv2.warpAffine / cv2.warpPerspective of each warped
column's T_col by N over the whole page) and the footprint, feather and blend of oracle/oriented_regions.py / quad_regions.py.
The one-cell column has one box, so its plan is the plan cells=1 gives.

Stored as tests/golden/quad_regions.npz stores its own: the page, each region's kind (0 rectangle, 1 oriented, 2 quad), whether
it is a column, its corners (tl, tr, br, bl; an oriented region's br is tr + bl - tl), the labels and boxes as restore_regions
takes them, each region's restored line T (sr{r}) and the composed page strided [::STRIDE, ::STRIDE].  The T of the lines that
fit the canvas are stored whole, so that the twin recomposes the page from them everywhere outside the long column's footprint;
the long column's T is stored strided [::WIDE_STRIDE, ::WIDE_STRIDE].  sr_strides holds each region's stride and sr_widths each
W_T.

Needs a reference checkout (MARCONET_REFERENCE=<path>):  python -m oracle.make_golden_vertical_regions
"""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OUT = os.path.join(ROOT, "tests", "golden", "vertical_regions.npz")
SCALE, FEATHER = 4, 8
STRIDE = 8
WIDE_STRIDE = 4
H, W = 360, 128
RECT, ORIENTED, QUAD = 0, 1, 2
# kind, column, tl, tr, br, bl.  Short lines keep the file small: a line restores to 128 * width / height incompressible columns.
REGIONS = [
    (RECT, True, (4, 6), (24, 6), (24, 110), (4, 110)),              # characters at unequal pitch
    (RECT, True, (30, 6), (42, 6), (42, 294), (30, 294)),            # 24 cells of 12: a 288 x 12 line, wider than the canvas
    (ORIENTED, True, None, None, None, None),                        # tilted 4 degrees
    (QUAD, True, (88, 10), (112, 14), (111, 118), (90, 113)),        # in perspective
    (RECT, True, (64, 130), (88, 130), (88, 160), (64, 160)),        # one cell
    (RECT, False, (20, 280), (100, 280), (100, 300), (20, 300)),     # a horizontal line over the long column's foot
]
TILTED = dict(cx=66.0, cy=64.0, w=18.0, h=100.0, angle=4.0)
WIDE = 1


def regions():
    from marconet_b200.pipeline import OrientedRegion, QuadRegion, VerticalRegion
    out = []
    for kind, column, tl, tr, br, bl in REGIONS:
        if kind == ORIENTED:
            shape = OrientedRegion.from_rotated(TILTED["cx"], TILTED["cy"], TILTED["w"], TILTED["h"], TILTED["angle"])
        elif kind == QUAD:
            shape = QuadRegion(tl, tr, br, bl)
        else:
            shape = (tl[0], tl[1], br[0], br[1])
        out.append(VerticalRegion(shape) if column else shape)
    return out


def corners():
    out = []
    for reg in regions():
        shape = getattr(reg, "shape", reg)
        if len(shape) == 3:
            (a, b), (c, d), (e, f) = shape
            out.append(((a, b), (c, d), (c + e - a, d + f - b), (e, f)))
        elif len(shape) == 4 and not isinstance(shape[0], (int, np.integer)):
            out.append(tuple(shape))
        else:
            x0, y0, x1, y1 = shape
            out.append(((x0, y0), (x1, y0), (x1, y1), (x0, y1)))
    return np.asarray(out, np.float64)


def _size(shape):
    from marconet_b200.pipeline import OrientedRegion, QuadRegion, oriented_maps, quad_maps
    if isinstance(shape, OrientedRegion):
        return oriented_maps(shape, 1)
    if isinstance(shape, QuadRegion):
        return quad_maps(shape, 1)
    return None


def make_page(seed=0):
    """H x W uint8 page: a smooth background with sparse speckle, and each region's text -- dark character boxes on a light band,
    drawn in its crop's frame (down the column for a column, along the line otherwise) -- pasted at the region's place
    (cv2.warpAffine / cv2.warpPerspective by M, nearest pixel; rectangles as they are).  Returns the page and each region's
    labels and boxes as restore_regions takes them (the crop's frame for a column, image coordinates for the rectangle line)."""
    import cv2
    rng = np.random.default_rng(seed)
    yy, xx = np.mgrid[0:H, 0:W]
    img = np.stack([90 + 60 * np.sin(xx / 41.0 + c) + 40 * np.cos(yy / 57.0 - c) for c in range(3)], -1).astype(np.int32)
    img[rng.random((H, W)) < 0.02] += rng.integers(-40, 41, 3)
    img = np.clip(img, 0, 255).astype(np.uint8)
    labels, boxes = [], []
    for r, reg in enumerate(regions()):
        column = REGIONS[r][1]
        shape = getattr(reg, "shape", reg)
        maps = _size(shape)
        w, h = maps.size if maps else (shape[2] - shape[0], shape[3] - shape[1])
        band = (rng.integers(180, 230, 3) + rng.integers(-15, 16, (h, w, 1))).astype(np.int32)
        bx = []
        if column:
            y = 1
            while True:                                  # the long column at a pitch of w, the others unequal
                ch = w - 2 if r == WIDE else h - 2 if r == 4 else int(rng.integers(w * 5 // 8, w * 5 // 4))
                if len(bx) == 24 or y + ch > h - 1:
                    break
                bx0, bx1 = int(rng.integers(0, 3)), w - int(rng.integers(0, 3))
                bx.append([bx0, y, bx1, y + ch])
                y += ch + (2 if r == WIDE else int(rng.integers(2, 7)))
        else:
            x = 2
            while True:
                cw = int(rng.integers(h * 5 // 8, h * 7 // 8))
                if x + cw > w - 2:
                    break
                by0, by1 = int(rng.integers(1, 4)), h - int(rng.integers(1, 4))
                bx.append([x, by0, x + cw, by1])
                x += cw + int(rng.integers(2, 5))
        for b in bx:
            mask = rng.random((b[3] - b[1], b[2] - b[0])) < 0.5
            band[b[1]:b[3], b[0]:b[2]][mask] = rng.integers(0, 80, 3)
        band = np.clip(band, 0, 255).astype(np.uint8)
        if maps is None:
            x0, y0 = shape[:2]
            img[y0:y0 + h, x0:x0 + w] = band
            if not column:
                bx = [[b[0] + x0, b[1] + y0, b[2] + x0, b[3] + y0] for b in bx]
        else:
            warp = cv2.warpAffine if maps.matrix.shape[0] == 2 else cv2.warpPerspective
            warped = warp(band, maps.matrix, (W, H), flags=cv2.INTER_NEAREST, borderMode=cv2.BORDER_CONSTANT)
            inside = warp(np.ones((h, w), np.uint8), maps.matrix, (W, H), flags=cv2.INTER_NEAREST,
                          borderMode=cv2.BORDER_CONSTANT).astype(bool)
            img[inside] = warped[inside]
        boxes.append(bx)
        labels.append(rng.integers(0, 6735, len(bx)).astype(np.int64))
    return img, labels, boxes


def main():
    import cv2
    sys.path.insert(0, ROOT)
    cv2.ipp.setUseIPP(False)
    from marconet_b200.pipeline import OrientedRegion, QuadRegion, oriented_maps, plan_regions, quad_maps
    from marconet_b200.testing import synth
    from oracle import ref_harness
    from oracle import regions as RR
    from oracle import vertical_regions as V
    from oracle import warp_affine as WA
    from oracle import warp_perspective as WP
    from oracle.make_golden_regions import restore_region
    torch.set_num_threads(os.cpu_count() or 1)
    page, labels, boxes = make_page()
    regs = regions()
    plan_regions([page.shape[:2]], [regs], [labels], [boxes], scale=SCALE, feather=FEATHER)      # every region is valid
    models = ref_harness.build_reference_models(synth.make_checkpoints(0))
    s = SCALE
    out = cv2.resize(page, (0, 0), fx=s, fy=s, interpolation=cv2.INTER_CUBIC)
    flags = cv2.INTER_CUBIC | cv2.WARP_INVERSE_MAP
    ts = []
    for r, (reg, lab, bx) in enumerate(zip(regs, labels, boxes)):
        column = REGIONS[r][1]
        shape = getattr(reg, "shape", reg)
        maps = _size(shape)
        if maps is None:
            x0, y0, x1, y1 = shape
            crop = np.ascontiguousarray(page[y0:y1, x0:x1])
        else:
            warp = cv2.warpAffine if isinstance(shape, OrientedRegion) else cv2.warpPerspective
            crop = warp(page, maps.matrix, maps.size, flags=flags, borderMode=cv2.BORDER_REPLICATE)
        if column:
            w_r = crop.shape[1]
            c = V.cells(crop.shape[0], w_r, boxes=bx)
            line = V.layout(crop, c)
            t = restore_region(models, line, (0, 0, line.shape[1], line.shape[0]), list(lab), V.line_boxes(c, w_r, bx))
            tc = V.unlayout(t, c, w_r)
        else:
            rel = bx if maps else [[b[0] - x0, b[1] - y0, b[2] - x0, b[3] - y0] for b in bx]
            t = restore_region(models, crop, (0, 0, crop.shape[1], crop.shape[0]), list(lab), rel)
            tc = t
        ts.append(t)
        src = np.ascontiguousarray(tc[..., ::-1])
        th, tw = tc.shape[:2]
        if maps is None:
            rr = (s * x0, s * y0, s * x1, s * y1)
            p = cv2.resize(src, (rr[2] - rr[0], rr[3] - rr[1]), interpolation=cv2.INTER_CUBIC)
            out[rr[1]:rr[3], rr[0]:rr[2]] = RR.blend(out[rr[1]:rr[3], rr[0]:rr[2]], p, RR.alpha(rr, out.shape[:2], FEATHER))
            continue
        if isinstance(shape, OrientedRegion):
            n = oriented_maps(shape, s, tw, th).page_map
            p = cv2.warpAffine(src, n, (s * W, s * H), flags=flags, borderMode=cv2.BORDER_REPLICATE)
            xq, yq = WA.warp_coords(n, np.arange(s * W), np.arange(s * H))
        else:
            assert isinstance(shape, QuadRegion)
            n = quad_maps(shape, s, tw, th).page_map
            p = cv2.warpPerspective(src, n, (s * W, s * H), flags=flags, borderMode=cv2.BORDER_REPLICATE)
            xq, yq = WP.warp_coords(n, np.arange(s * W), np.arange(s * H), (s * W, s * H))
        (x0, y0, x1, y1), _, a, mask = V._warped_patch(tc, shape, s, out.shape[:2], FEATHER)
        whole = (xq >= -16) & (xq < 32 * tw - 16) & (yq >= -16) & (yq < 32 * th - 16)
        assert whole.sum() == mask.sum(), "the footprint leaves its box"
        sl = out[y0:y1, x0:x1]
        sl[mask] = RR.blend(sl, p[y0:y1, x0:x1], a)[mask]
    strides = [WIDE_STRIDE if r == WIDE else 1 for r in range(len(regs))]
    box_arr = np.asarray([b + [r] for r, bx in enumerate(boxes) for b in bx], np.int64)     # x1, y1, x2, y2, region
    np.savez_compressed(OUT, image=page, kinds=np.asarray([k[0] for k in REGIONS], np.int64),
                        columns=np.asarray([k[1] for k in REGIONS], bool), corners=corners(),
                        labels=np.concatenate(labels), boxes=box_arr, scale=np.array(s), feather=np.array(FEATHER),
                        stride=np.array(STRIDE), page=np.ascontiguousarray(out[::STRIDE, ::STRIDE]),
                        sr_strides=np.asarray(strides, np.int64), sr_widths=np.asarray([t.shape[1] for t in ts], np.int64),
                        **{f"sr{r}": np.ascontiguousarray(t[::k, ::k]) for r, (t, k) in enumerate(zip(ts, strides))})
    print("wrote", OUT, page.shape, out.shape, [t.shape for t in ts], os.path.getsize(OUT))


if __name__ == "__main__":
    main()
