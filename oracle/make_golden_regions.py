"""Generates tests/golden/regions.npz: a seeded synthetic page (160 x 700) with four text regions -- a line that fits the 32x512
LQ canvas, a line wider than the canvas, a region that overlaps the first and one that touches the right and bottom borders --
each region restored on the CPU by the data flow of the reference's test_sr.py (:98-201) with the reference's UNMODIFIED modules
(oracle/ref_harness.py, synthetic checkpoints seed 0) through make_golden_wide_line.script_sr_bytes, the crops of the wide line
stitched with oracle/wide_line.stitch_sr where pipeline.plan_segments cuts it, and the page composed at s = 4, F = 8 with live
cv2 (IPP off) for both resizes plus oracle/regions.py's feather and blend.

Stored: the page, the regions with their labels and boxes (image coordinates), each region's SR bytes and the composed page
strided [::STRIDE, ::STRIDE].  The SR bytes of the regions that fit the canvas are stored whole, so that the twin recomposes the
page from them everywhere outside the wide region's rectangle (no pixel there depends on that region); the wide region's SR bytes
(over 2048 columns of incompressible bytes) are stored strided [::WIDE_STRIDE, ::WIDE_STRIDE], enough for a comparison with
restore_regions' own bytes.  sr_strides holds each region's stride.

Needs a reference checkout (MARCONET_REFERENCE=<path>):  python -m oracle.make_golden_regions
"""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OUT = os.path.join(ROOT, "tests", "golden", "regions.npz")
SCALE, FEATHER = 4, 8
STRIDE = 8
WIDE_STRIDE = 4
# (x0, y0, x1, y1): fits the canvas; wider than the canvas (LQ width 521); overlaps the first two; touches the right and bottom
# borders.  The ones that fit are short (256 SR columns each) to keep the file small.
REGIONS = [(16, 8, 96, 48), (8, 64, 464, 92), (64, 28, 144, 68), (620, 120, 700, 160)]
WIDE = 1


def make_page(seed=0, h=160, w=700):
    """h x w uint8 page: a smooth background with sparse speckle, and in each region dark character boxes on a light band."""
    rng = np.random.default_rng(seed)
    yy, xx = np.mgrid[0:h, 0:w]
    img = np.stack([90 + 60 * np.sin(xx / 53.0 + c) + 40 * np.cos(yy / 31.0 - c) for c in range(3)], -1).astype(np.int32)
    img[rng.random((h, w)) < 0.02] += rng.integers(-40, 41, 3)                         # sparse speckle
    labels, boxes = [], []
    for x0, y0, x1, y1 in REGIONS:
        rh = y1 - y0
        img[y0:y1, x0:x1] = rng.integers(180, 230, 3) + rng.integers(-15, 16, (rh, x1 - x0, 1))
        bx, x = [], x0 + 4
        while True:
            cw = int(rng.integers(rh * 5 // 8, rh * 7 // 8))
            if x + cw > x1 - 4:
                break
            by0, by1 = y0 + int(rng.integers(1, 4)), y1 - int(rng.integers(1, 4))
            bx.append([x, by0, x + cw, by1])
            mask = rng.random((by1 - by0, cw)) < 0.5
            img[by0:by1, x:x + cw][mask] = rng.integers(0, 80, 3)
            x += cw + int(rng.integers(2, 7))
        boxes.append(bx)
        labels.append(rng.integers(0, 6735, len(bx)).astype(np.int64))
    return np.clip(img, 0, 255).astype(np.uint8), labels, boxes


def restore_region(models, page, rect, labels, boxes):
    """The region's SR bytes as restore_images computes them for the crop: plan_segments' crops through the script, stitched."""
    from marconet_b200 import pipeline
    from oracle import wide_line
    from oracle.make_golden_wide_line import script_sr_bytes
    x0, y0, x1, y1 = rect
    crop = np.ascontiguousarray(page[y0:y1, x0:x1])
    h, w = crop.shape[:2]
    rel = [[b[0] - x0, b[1] - y0, b[2] - x0, b[3] - y0] for b in boxes]
    segs = pipeline.plan_segments(h, w, rel, labels=labels)
    srs = [script_sr_bytes(models, np.ascontiguousarray(crop[:, s.crop[0]:s.crop[1]]), s.boxes, labels[s.chars[0]:s.chars[1]])
           for s in segs]
    print("region", rect, "segments", [s.crop for s in segs], flush=True)
    return wide_line.stitch_sr(h, w, [s.core[0] for s in segs] + [w], [s.crop for s in segs], srs)


def main():
    import cv2
    sys.path.insert(0, ROOT)
    cv2.ipp.setUseIPP(False)
    from oracle import ref_harness, regions
    from marconet_b200.testing import synth
    torch.set_num_threads(os.cpu_count() or 1)
    models = ref_harness.build_reference_models(synth.make_checkpoints(0))
    page, labels, boxes = make_page()
    srs = [restore_region(models, page, r, l, b) for r, l, b in zip(REGIONS, labels, boxes)]
    s = SCALE
    out = cv2.resize(page, (0, 0), fx=s, fy=s, interpolation=cv2.INTER_CUBIC)
    for (x0, y0, x1, y1), t in zip(REGIONS, srs):
        rect = (s * x0, s * y0, s * x1, s * y1)
        p = cv2.resize(np.ascontiguousarray(t[..., ::-1]), (rect[2] - rect[0], rect[3] - rect[1]), interpolation=cv2.INTER_CUBIC)
        out[rect[1]:rect[3], rect[0]:rect[2]] = regions.blend(out[rect[1]:rect[3], rect[0]:rect[2]], p,
                                                              regions.alpha(rect, out.shape[:2], FEATHER))
    strides = [WIDE_STRIDE if r == WIDE else 1 for r in range(len(REGIONS))]
    box_arr = np.asarray([b + [r] for r, bx in enumerate(boxes) for b in bx], np.int64)     # x1, y1, x2, y2, region
    np.savez_compressed(OUT, image=page, regions=np.asarray(REGIONS, np.int64), labels=np.concatenate(labels), boxes=box_arr,
                        scale=np.array(s), feather=np.array(FEATHER), stride=np.array(STRIDE),
                        page=np.ascontiguousarray(out[::STRIDE, ::STRIDE]), sr_strides=np.asarray(strides, np.int64),
                        **{f"sr{r}": np.ascontiguousarray(t[::k, ::k]) for r, (t, k) in enumerate(zip(srs, strides))})
    print("wrote", OUT, page.shape, out.shape, [t.shape for t in srs], os.path.getsize(OUT))


if __name__ == "__main__":
    main()
