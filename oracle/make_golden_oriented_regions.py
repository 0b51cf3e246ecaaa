"""Generates tests/golden/oriented_regions.npz: a seeded synthetic page (128 x 360) with six oriented text regions
(pipeline.OrientedRegion) -- a line at -20 degrees that is wider than the 32x512 LQ canvas once rectified, a line at +7 degrees,
a line at 90 degrees, an interior axis-aligned region, a region at 35 degrees overlapping it and one at -12 degrees partly off
the page -- each rectified with live cv2.warpAffine (IPP off) through pipeline.oriented_maps' M, restored on the CPU by the data
flow of the reference's test_sr.py with the reference's UNMODIFIED modules (make_golden_regions.restore_region: plan_segments'
crops through the script, stitched) and composed at s = 4, F = 8: live cv2 background and live cv2.warpAffine of every restored
line by N over the whole page, oracle/warp_affine.warp_coords' fixed-point footprint and oracle/oriented_regions.py's feather and blend.

Stored as tests/golden/regions.npz stores its own: the page, the regions' corners, their labels and boxes (each in its crop's frame), each
region's SR bytes and the composed page strided [::STRIDE, ::STRIDE].  The SR bytes of the regions that fit the canvas are stored
whole, so that the twin recomposes the page from them everywhere outside the wide region's footprint; the wide region's SR
bytes are stored strided [::WIDE_STRIDE, ::WIDE_STRIDE].  sr_strides holds each region's stride and sr_widths each W_T.

Needs a reference checkout (MARCONET_REFERENCE=<path>):  python -m oracle.make_golden_oriented_regions
"""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OUT = os.path.join(ROOT, "tests", "golden", "oriented_regions.npz")
SCALE, FEATHER = 4, 8
STRIDE = 8
WIDE_STRIDE = 4
H, W = 128, 360
# (cx, cy, w, h, angle) for OrientedRegion.from_rotated, except the axis-aligned one, given by its corners.  Short lines keep the
# file small: a line that fits the canvas restores to 128 * w / h columns of incompressible bytes.
ROTATED = [(150, 64, 264, 16, -20), (310, 30, 33, 22, 7), (330, 85, 36, 22, 90), None, (60, 100, 30, 20, 35),
           (352, 122, 30, 20, -12)]
AXIS = ((20, 90), (56, 90), (20, 114))
WIDE = 0


def regions():
    from marconet_b200.pipeline import OrientedRegion
    return [OrientedRegion(*AXIS) if r is None else OrientedRegion.from_rotated(*r) for r in ROTATED]


def make_page(seed=0):
    """H x W uint8 page: a smooth background with sparse speckle, and each region's line -- dark character boxes on a light band,
    drawn in its crop's frame -- pasted at the region's place (cv2.warpAffine by M, nearest pixel).  Returns the page and each
    region's labels and boxes in its crop's frame."""
    import cv2
    from marconet_b200.pipeline import oriented_maps
    rng = np.random.default_rng(seed)
    yy, xx = np.mgrid[0:H, 0:W]
    img = np.stack([90 + 60 * np.sin(xx / 53.0 + c) + 40 * np.cos(yy / 31.0 - c) for c in range(3)], -1).astype(np.int32)
    img[rng.random((H, W)) < 0.02] += rng.integers(-40, 41, 3)
    img = np.clip(img, 0, 255).astype(np.uint8)
    labels, boxes = [], []
    for reg in regions():
        m = oriented_maps(reg, 1)
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
        warped = cv2.warpAffine(line, m.matrix, (W, H), flags=cv2.INTER_NEAREST, borderMode=cv2.BORDER_CONSTANT)
        inside = cv2.warpAffine(np.ones((h, w), np.uint8), m.matrix, (W, H), flags=cv2.INTER_NEAREST,
                                borderMode=cv2.BORDER_CONSTANT).astype(bool)
        img[inside] = warped[inside]
        boxes.append(bx)
        labels.append(rng.integers(0, 6735, len(bx)).astype(np.int64))
    return img, labels, boxes


def main():
    import cv2
    sys.path.insert(0, ROOT)
    cv2.ipp.setUseIPP(False)
    from marconet_b200.pipeline import oriented_maps
    from marconet_b200.testing import synth
    from oracle import ref_harness
    from oracle import oriented_regions as R
    from oracle.warp_affine import warp_coords
    from oracle.make_golden_regions import restore_region
    torch.set_num_threads(os.cpu_count() or 1)
    models = ref_harness.build_reference_models(synth.make_checkpoints(0))
    page, labels, boxes = make_page()
    regs = regions()
    s = SCALE
    out = cv2.resize(page, (0, 0), fx=s, fy=s, interpolation=cv2.INTER_CUBIC)
    flags = cv2.INTER_CUBIC | cv2.WARP_INVERSE_MAP
    srs = []
    for reg, lab, bx in zip(regs, labels, boxes):
        m = oriented_maps(reg, 1)
        crop = cv2.warpAffine(page, m.matrix, m.size, flags=flags, borderMode=cv2.BORDER_REPLICATE)
        t = restore_region(models, crop, (0, 0, m.size[0], m.size[1]), list(lab), bx)
        srs.append(t)
        n = oriented_maps(reg, s, t.shape[1])
        p = cv2.warpAffine(np.ascontiguousarray(t[..., ::-1]), n.page_map, (s * W, s * H), flags=flags,
                           borderMode=cv2.BORDER_REPLICATE)
        (x0, y0, x1, y1), _, a, mask = R.oriented_patch(t, reg, s, out.shape[:2], FEATHER)
        xq, yq = warp_coords(n.page_map, np.arange(s * W), np.arange(s * H))
        whole = (xq >= -16) & (xq < 32 * t.shape[1] - 16) & (yq >= -16) & (yq < 32 * t.shape[0] - 16)
        assert whole.sum() == mask.sum(), "the footprint leaves its box"
        sl = out[y0:y1, x0:x1]
        sl[mask] = R.blend(sl, p[y0:y1, x0:x1], a)[mask]
    strides = [WIDE_STRIDE if r == WIDE else 1 for r in range(len(regs))]
    box_arr = np.asarray([b + [r] for r, bx in enumerate(boxes) for b in bx], np.int64)     # x1, y1, x2, y2, region
    corners = np.asarray([[list(p) for p in reg] for reg in regs], np.float64)
    np.savez_compressed(OUT, image=page, corners=corners, labels=np.concatenate(labels), boxes=box_arr, scale=np.array(s),
                        feather=np.array(FEATHER), stride=np.array(STRIDE), page=np.ascontiguousarray(out[::STRIDE, ::STRIDE]),
                        sr_strides=np.asarray(strides, np.int64), sr_widths=np.asarray([t.shape[1] for t in srs], np.int64),
                        **{f"sr{r}": np.ascontiguousarray(t[::k, ::k]) for r, (t, k) in enumerate(zip(srs, strides))})
    print("wrote", OUT, page.shape, out.shape, [t.shape for t in srs], os.path.getsize(OUT))


if __name__ == "__main__":
    main()
