"""Generates tests/golden/quad_regions.npz: a seeded synthetic page (128 x 360) with six text regions -- a strongly foreshortened
line (pipeline.QuadRegion) that is wider than the 32x512 LQ canvas once rectified, a mild keystone line, an interior rectangle, a
quad overlapping it, a quad partly off the page and a quad that is exactly a parallelogram -- each quad rectified with live
cv2.warpPerspective (IPP off) through pipeline.quad_maps' M, restored on the CPU by the data flow of the reference's test_sr.py
with the reference's UNMODIFIED modules (make_golden_regions.restore_region: plan_segments' crops through the script, stitched)
and composed at s = 4, F = 8: live cv2 background, live cv2.resize of the rectangle's line and live cv2.warpPerspective of every
restored quad line by N over the whole page, oracle/warp_perspective.warp_coords' fixed-point footprint and
oracle/quad_regions.py's feather and blend.

Stored as tests/golden/oriented_regions.npz stores its own: the page, each region's kind (0 rectangle, 2 quad) and four corners
(tl, tr, br, bl), their labels and boxes as restore_regions takes them (image coordinates for the rectangle, each quad's crop
frame otherwise), each region's SR bytes and the composed page strided [::STRIDE, ::STRIDE].  The SR bytes of the regions that
fit the canvas are stored whole, so that the twin recomposes the page from them everywhere outside the wide region's footprint;
the wide region's SR bytes are stored strided [::WIDE_STRIDE, ::WIDE_STRIDE].  sr_strides holds each region's stride and
sr_widths each W_T.

Needs a reference checkout (MARCONET_REFERENCE=<path>):  python -m oracle.make_golden_quad_regions
"""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OUT = os.path.join(ROOT, "tests", "golden", "quad_regions.npz")
SCALE, FEATHER = 4, 8
STRIDE = 8
WIDE_STRIDE = 4
H, W = 128, 360
# tl, tr, br, bl.  Short lines keep the file small: a line that fits the canvas restores to 128 * w / h incompressible columns.
CORNERS = [
    ((20, 22), (300, 10), (300, 26), (20, 28)),          # foreshortened 16 / 6 at the far end: 280 x 16, wider than the canvas
    ((290, 40), (330, 38.5), (331, 62), (289, 60)),      # mild keystone
    ((30, 80), (60, 80), (60, 104), (30, 104)),          # the interior rectangle (30, 80, 60, 104)
    ((55, 90), (95, 84.5), (97, 110), (57, 113)),        # overlaps the rectangle
    ((330, 100), (375, 104), (372, 138), (328, 126)),    # partly off the right and bottom borders
    ((150, 60), (180, 54), (184, 76), (154, 82)),        # exactly a parallelogram: br = tr + bl - tl
]
RECT = 2
WIDE = 0


def regions():
    from marconet_b200.pipeline import QuadRegion
    return [(c[0][0], c[0][1], c[2][0], c[2][1]) if r == RECT else QuadRegion(*c) for r, c in enumerate(CORNERS)]


def make_page(seed=0):
    """H x W uint8 page: a smooth background with sparse speckle, and each region's line -- dark character boxes on a light band,
    drawn in its crop's frame -- pasted at the region's place (cv2.warpPerspective by M, nearest pixel; the rectangle as is).
    Returns the page and each region's labels and boxes as restore_regions takes them."""
    import cv2
    from marconet_b200.pipeline import quad_maps
    rng = np.random.default_rng(seed)
    yy, xx = np.mgrid[0:H, 0:W]
    img = np.stack([90 + 60 * np.sin(xx / 53.0 + c) + 40 * np.cos(yy / 31.0 - c) for c in range(3)], -1).astype(np.int32)
    img[rng.random((H, W)) < 0.02] += rng.integers(-40, 41, 3)
    img = np.clip(img, 0, 255).astype(np.uint8)
    labels, boxes = [], []
    for r, reg in enumerate(regions()):
        if r == RECT:
            x0, y0, x1, y1 = reg
            w, h = x1 - x0, y1 - y0
        else:
            m = quad_maps(reg, 1)
            w, h = m.size
        line = (rng.integers(180, 230, 3) + rng.integers(-15, 16, (h, w, 1))).astype(np.int32)
        bx, x = [], 2
        while True:
            cw = int(rng.integers(h * 5 // 8, h * 7 // 8))
            if x + cw > w - 2:
                break
            by0, by1 = int(rng.integers(1, 4)), h - int(rng.integers(1, 4))
            bx.append([x, by0, x + cw, by1])
            mask = rng.random((by1 - by0, cw)) < 0.5
            line[by0:by1, x:x + cw][mask] = rng.integers(0, 80, 3)
            x += cw + int(rng.integers(2, 5))
        line = np.clip(line, 0, 255).astype(np.uint8)
        if r == RECT:
            img[y0:y1, x0:x1] = line
            bx = [[b[0] + x0, b[1] + y0, b[2] + x0, b[3] + y0] for b in bx]
        else:
            warped = cv2.warpPerspective(line, m.matrix, (W, H), flags=cv2.INTER_NEAREST, borderMode=cv2.BORDER_CONSTANT)
            inside = cv2.warpPerspective(np.ones((h, w), np.uint8), m.matrix, (W, H), flags=cv2.INTER_NEAREST,
                                         borderMode=cv2.BORDER_CONSTANT).astype(bool)
            img[inside] = warped[inside]
        boxes.append(bx)
        labels.append(rng.integers(0, 6735, len(bx)).astype(np.int64))
    return img, labels, boxes


def main():
    import cv2
    sys.path.insert(0, ROOT)
    cv2.ipp.setUseIPP(False)
    from marconet_b200.pipeline import plan_regions, quad_maps
    from marconet_b200.testing import synth
    from oracle import ref_harness
    from oracle import quad_regions as R
    from oracle import regions as RR
    from oracle.warp_perspective import warp_coords
    from oracle.make_golden_regions import restore_region
    torch.set_num_threads(os.cpu_count() or 1)
    page, labels, boxes = make_page()
    regs = regions()
    plan_regions([page.shape[:2]], [regs], [labels], [boxes], scale=SCALE, feather=FEATHER)      # every region is valid
    models = ref_harness.build_reference_models(synth.make_checkpoints(0))
    s = SCALE
    out = cv2.resize(page, (0, 0), fx=s, fy=s, interpolation=cv2.INTER_CUBIC)
    flags = cv2.INTER_CUBIC | cv2.WARP_INVERSE_MAP
    srs = []
    for r, (reg, lab, bx) in enumerate(zip(regs, labels, boxes)):
        if r == RECT:
            x0, y0, x1, y1 = reg
            t = restore_region(models, page, reg, list(lab), bx)
            srs.append(t)
            rr = (s * x0, s * y0, s * x1, s * y1)
            p = cv2.resize(np.ascontiguousarray(t[..., ::-1]), (rr[2] - rr[0], rr[3] - rr[1]), interpolation=cv2.INTER_CUBIC)
            out[rr[1]:rr[3], rr[0]:rr[2]] = RR.blend(out[rr[1]:rr[3], rr[0]:rr[2]], p, RR.alpha(rr, out.shape[:2], FEATHER))
            continue
        m = quad_maps(reg, 1)
        crop = cv2.warpPerspective(page, m.matrix, m.size, flags=flags, borderMode=cv2.BORDER_REPLICATE)
        t = restore_region(models, crop, (0, 0, m.size[0], m.size[1]), list(lab), bx)
        srs.append(t)
        n = quad_maps(reg, s, t.shape[1])
        p = cv2.warpPerspective(np.ascontiguousarray(t[..., ::-1]), n.page_map, (s * W, s * H), flags=flags,
                                borderMode=cv2.BORDER_REPLICATE)
        (x0, y0, x1, y1), _, a, mask = R.quad_patch(t, reg, s, out.shape[:2], FEATHER)
        xq, yq = warp_coords(n.page_map, np.arange(s * W), np.arange(s * H), (s * W, s * H))
        whole = (xq >= -16) & (xq < 32 * t.shape[1] - 16) & (yq >= -16) & (yq < 32 * t.shape[0] - 16)
        assert whole.sum() == mask.sum(), "the footprint leaves its box"
        sl = out[y0:y1, x0:x1]
        sl[mask] = R.blend(sl, p[y0:y1, x0:x1], a)[mask]
    strides = [WIDE_STRIDE if r == WIDE else 1 for r in range(len(regs))]
    box_arr = np.asarray([b + [r] for r, bx in enumerate(boxes) for b in bx], np.int64)     # x1, y1, x2, y2, region
    kinds = np.asarray([0 if r == RECT else 2 for r in range(len(regs))], np.int64)
    np.savez_compressed(OUT, image=page, kinds=kinds, corners=np.asarray(CORNERS, np.float64), labels=np.concatenate(labels),
                        boxes=box_arr, scale=np.array(s), feather=np.array(FEATHER), stride=np.array(STRIDE),
                        page=np.ascontiguousarray(out[::STRIDE, ::STRIDE]), sr_strides=np.asarray(strides, np.int64),
                        sr_widths=np.asarray([t.shape[1] for t in srs], np.int64),
                        **{f"sr{r}": np.ascontiguousarray(t[::k, ::k]) for r, (t, k) in enumerate(zip(srs, strides))})
    print("wrote", OUT, page.shape, out.shape, [t.shape for t in srs], os.path.getsize(OUT))


if __name__ == "__main__":
    main()
