"""Generates tests/golden/curved_regions.npz: a seeded synthetic page (176 x 320) with seven text regions -- a seal's top arc
(pipeline.CurvedRegion.from_arc, 200 degrees, k = 3) that is wider than the 32x512 LQ canvas once rectified, a bottom arc read
left to right with the inner arc as its top, a gentle single-segment S-curve, a straight curved region over the interior
rectangle (200, 60, 236, 84), an OrientedRegion, a curved region overlapping it and a curved region partly off the page -- each
curved region rectified with live cv2.remap (IPP off) through the crop maps of oracle/curved_regions.py, restored on the CPU by
the data flow of the reference's test_sr.py with the reference's UNMODIFIED modules (make_golden_regions.restore_region) and
composed at s = 4, F = 8: live cv2 background, live cv2.remap of every restored curved line at the twin's T coordinates
(u, v) of its footprint and live cv2.warpAffine of the oriented line by N, with the twins' footprints, feathers and blend.

Stored as tests/golden/quad_regions.npz stores its own: the page, each region's kind (1 oriented, 3 curved) and points (for a
curved region its top then its bottom curve; for the oriented region tl, tr, bl), their labels and boxes in each region's crop
frame, each region's SR bytes and the composed page strided [::STRIDE, ::STRIDE].  The SR bytes of the two arcs and the S-curve
are stored strided [::WIDE_STRIDE, ::WIDE_STRIDE], the others whole, so that the twin recomposes the page from them everywhere
outside the strided regions' footprints.  sr_strides holds each region's stride, sr_widths each W_T and n_points each curve's
point count.

Needs a reference checkout (MARCONET_REFERENCE=<path>):  python -m oracle.make_golden_curved_regions
"""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OUT = os.path.join(ROOT, "tests", "golden", "curved_regions.npz")
SCALE, FEATHER = 4, 8
STRIDE = 8
WIDE_STRIDE = 4
H, W = 176, 320
ORIENTED = 4
STRIDED = (0, 1, 2)


def regions():
    from marconet_b200.pipeline import CurvedRegion, OrientedRegion
    return [
        CurvedRegion.from_arc(100, 100, 84, 72, 190, -10),                            # seal top arc: 272 x 12, wider than the canvas
        CurvedRegion.from_arc(100, 100, 48, 62, 240, 300),                            # bottom arc, inner arc on top
        CurvedRegion(((200, 20), (225, 10), (250, 34), (275, 22)), ((200, 38), (225, 28), (250, 52), (275, 40))),   # S-curve
        CurvedRegion(((200, 60), (212, 60), (224, 60), (236, 60)), ((200, 84), (212, 84), (224, 84), (236, 84))),   # straight
        OrientedRegion.from_rotated(265, 100, 34, 22, 15),
        CurvedRegion(((245, 108), (257, 103), (268, 103), (280, 108)), ((245, 130), (257, 125), (268, 125), (280, 130))),
        CurvedRegion(((295, 140), (308, 136), (321, 136), (334, 140)), ((295, 166), (308, 162), (321, 162), (334, 166))),
    ]


def points(reg):
    """The region's points as one [n, 2] list: a curved region's top then bottom curve, an oriented region's tl, tr, bl."""
    from marconet_b200.pipeline import CurvedRegion
    return [list(p) for p in (reg.top + reg.bottom if isinstance(reg, CurvedRegion) else reg)]


def make_page(seed=0):
    """H x W uint8 page: a smooth background with sparse speckle, and each region's line -- dark character boxes on a light band,
    drawn in its crop's frame -- pasted at the region's place (nearest pixel: a curved region's page pixels inverted by the twin,
    the oriented one by cv2.warpAffine with M).  Returns the page and each region's labels and boxes (crop frames)."""
    import cv2
    from marconet_b200.pipeline import CurvedRegion, curved_maps, oriented_maps
    from oracle import curved_regions as R
    rng = np.random.default_rng(seed)
    yy, xx = np.mgrid[0:H, 0:W]
    img = np.stack([90 + 60 * np.sin(xx / 53.0 + c) + 40 * np.cos(yy / 31.0 - c) for c in range(3)], -1).astype(np.int32)
    img[rng.random((H, W)) < 0.02] += rng.integers(-40, 41, 3)
    img = np.clip(img, 0, 255).astype(np.uint8)
    labels, boxes = [], []
    for reg in regions():
        m = curved_maps(reg, 1) if isinstance(reg, CurvedRegion) else oriented_maps(reg, 1)
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
        if isinstance(reg, CurvedRegion):
            qx, qy = np.meshgrid(np.arange(W) + 0.5, np.arange(H) + 0.5)
            ok, mm, tt, bb = R.invert(m, qx, qy)
            u, v = R.t_maps(m, mm, tt, bb, (h, w))
            j, i = np.floor(u + 0.5).astype(np.int64), np.floor(v + 0.5).astype(np.int64)
            inside = (ok & (j >= 0) & (j < w) & (i >= 0) & (i < h)).reshape(H, W)
            img[inside] = line[i.reshape(H, W)[inside], j.reshape(H, W)[inside]]
        else:
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
    from marconet_b200.pipeline import CurvedRegion, curved_footprint_box, curved_maps, oriented_maps, plan_regions
    from marconet_b200.testing import synth
    from oracle import ref_harness
    from oracle import curved_regions as R
    from oracle.make_golden_regions import restore_region
    torch.set_num_threads(os.cpu_count() or 1)
    page, labels, boxes = make_page()
    regs = regions()
    plan_regions([page.shape[:2]], [regs], [labels], [boxes], scale=SCALE, feather=FEATHER)      # every region is valid
    models = ref_harness.build_reference_models(synth.make_checkpoints(0))
    s = SCALE
    out = cv2.resize(page, (0, 0), fx=s, fy=s, interpolation=cv2.INTER_CUBIC)
    srs = []
    for r, (reg, lab, bx) in enumerate(zip(regs, labels, boxes)):
        if isinstance(reg, CurvedRegion):
            m = curved_maps(reg, 1)
            mx, my = R.crop_map(m)
            crop = cv2.remap(page, mx.astype(np.float32), my.astype(np.float32), cv2.INTER_CUBIC, borderMode=cv2.BORDER_REPLICATE)
        else:
            m = oriented_maps(reg, 1)
            crop = cv2.warpAffine(page, m.matrix, m.size, flags=cv2.INTER_CUBIC | cv2.WARP_INVERSE_MAP,
                                  borderMode=cv2.BORDER_REPLICATE)
        t = restore_region(models, crop, (0, 0, m.size[0], m.size[1]), list(lab), bx)
        srs.append(t)
        tb = np.ascontiguousarray(t[..., ::-1])
        if isinstance(reg, CurvedRegion):
            n = curved_maps(reg, s, t.shape[1])
            box = curved_footprint_box(reg, s, out.shape[:2])
            (x0, y0, x1, y1), _, _, mask, a = R.curved_footprint(t.shape, reg, s, out.shape[:2], FEATHER)
            assert (x0, y0, x1, y1) == box
            qx, qy = np.meshgrid((np.arange(x0, x1) + 0.5) / s, (np.arange(y0, y1) + 0.5) / s)
            ok, mm, tt, bb = R.invert(n, qx, qy)
            u, v = R.t_maps(n, mm, tt, bb, t.shape[:2])
            u, v = np.where(ok, u, 0).reshape(qx.shape), np.where(ok, v, 0).reshape(qx.shape)
            p = cv2.remap(tb, u.astype(np.float32), v.astype(np.float32), cv2.INTER_CUBIC, borderMode=cv2.BORDER_REPLICATE)
        else:
            n = oriented_maps(reg, s, t.shape[1])
            (x0, y0, x1, y1), _, a, mask = R.oriented_patch(t, reg, s, out.shape[:2], FEATHER)
            p = cv2.warpAffine(tb, n.page_map, (s * W, s * H), flags=cv2.INTER_CUBIC | cv2.WARP_INVERSE_MAP,
                               borderMode=cv2.BORDER_REPLICATE)[y0:y1, x0:x1]
        sl = out[y0:y1, x0:x1]
        sl[mask] = R.blend(sl, p, a)[mask]
    strides = [WIDE_STRIDE if r in STRIDED else 1 for r in range(len(regs))]
    box_arr = np.asarray([b + [r] for r, bx in enumerate(boxes) for b in bx], np.int64)     # x1, y1, x2, y2, region
    kinds = np.asarray([1 if r == ORIENTED else 3 for r in range(len(regs))], np.int64)
    pts = [points(reg) for reg in regs]
    np.savez_compressed(OUT, image=page, kinds=kinds, points=np.asarray([p for q in pts for p in q], np.float64),
                        n_points=np.asarray([len(q) for q in pts], np.int64), labels=np.concatenate(labels),
                        boxes=box_arr, scale=np.array(s), feather=np.array(FEATHER), stride=np.array(STRIDE),
                        page=np.ascontiguousarray(out[::STRIDE, ::STRIDE]), sr_strides=np.asarray(strides, np.int64),
                        sr_widths=np.asarray([t.shape[1] for t in srs], np.int64),
                        **{f"sr{r}": np.ascontiguousarray(t[::k, ::k]) for r, (t, k) in enumerate(zip(srs, strides))})
    print("wrote", OUT, page.shape, out.shape, [t.shape for t in srs], os.path.getsize(OUT))


if __name__ == "__main__":
    main()
