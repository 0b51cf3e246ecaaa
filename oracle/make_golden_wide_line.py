"""Generates tests/golden/wide_line.npz: a seeded synthetic text line wider than the 32x512 LQ canvas (about 1250 LQ pixels,
22 characters, one character-free gap wider than the canvas), cut into crops by marconet_b200.pipeline.plan_segments, each crop
restored on the CPU by the data flow of the reference's test_sr.py (:98-201) with the reference's UNMODIFIED modules
(oracle/ref_harness.py, synthetic checkpoints seed 0), real cv2 (IPP off, as oracle/make_golden_script.py) and torchvision's
ToTensor / Normalize, and the crops' SR bytes stitched back into one line (oracle/wide_line.stitch_sr).

A crop without characters runs the SR decoder with empty prior lists, which the reference module accepts (its per-character
loops at models/networks.py:423-448 and :457-481 are then empty).

Needs a reference checkout (MARCONET_REFERENCE=<path>):  python -m oracle.make_golden_wide_line
"""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OUT = os.path.join(ROOT, "tests", "golden", "wide_line.npz")
STRIDE = 2      # the stored SR line is subsampled [::STRIDE, ::STRIDE], like script_sr_row.npz


def make_line(seed=0, h=40):
    """h x ~1580 uint8 BGR line: 11 characters, a 900-pixel blank gap (720 LQ pixels), 11 characters; boxes in reading order."""
    rng = np.random.default_rng(seed)
    boxes, x = [], 14
    for i in range(22):
        cw = int(rng.integers(20, 31))
        boxes.append([x, int(rng.integers(2, 6)), x + cw, h - int(rng.integers(2, 6))])
        x += cw + int(rng.integers(2, 8))
        if i == 10:
            x += 900
    w = x + 14
    img = np.full((h, w, 3), rng.integers(170, 230, 3), np.int32)
    img += rng.integers(-20, 21, (h, w, 1))
    for x1, y1, x2, y2 in boxes:
        ink = rng.integers(0, 80, 3)
        mask = rng.random((y2 - y1, x2 - x1)) < 0.55
        img[y1:y2, x1:x2][mask] = ink
    labels = rng.integers(0, 6735, len(boxes))
    return np.clip(img, 0, 255).astype(np.uint8), boxes, labels.astype(np.int64)


def script_sr_bytes(models, crop, boxes, labels):
    """test_sr.py:98-201 on one crop (boxes already relative to the crop) -> the ShowSR bytes cv2.imwrite stores (:231), [128, 2048, 3]."""
    import cv2
    from torchvision import transforms
    h = crop.shape[0]
    lq = cv2.resize(crop, (0, 0), fx=32 / h, fy=32 / h, interpolation=cv2.INTER_CUBIC)
    canvas = np.zeros((32, 32 * 16, 3)).astype(lq.dtype)
    assert lq.shape[-2] <= 32 * 16, lq.shape
    canvas[:, :lq.shape[-2], :] = canvas[:, :lq.shape[-2], :] + lq
    t = transforms.Normalize((0.5, 0.5, 0.5), (0.5, 0.5, 0.5))(transforms.ToTensor()(canvas)).unsqueeze(0)
    locs = torch.zeros(1, len(boxes) * 2).float()
    lq_width = int(t.shape[-1])
    for i, (x1, _, x2, _) in enumerate(boxes):
        locs[0, 2 * i] = ((x1 + x2) / 2.0 * 32.0 / h) / lq_width
        locs[0, 2 * i + 1] = ((x2 - x1) / 2.0 * 32.0 / h) / lq_width
    with torch.no_grad():
        _, _, w = models["encoder"](t)
        p64, p32 = [], []
        if len(labels):
            lab = torch.Tensor(list(labels)).type(torch.LongTensor).unsqueeze(1)
            _, f64, f32_ = models["tspgan"](styles=w[:1].clone().repeat(lab.size(0), 1), labels=lab, noise=None)
            p64, p32 = [f64], [f32_]
        sr = models["sr"](t, p64, p32, locs)
    sr = (sr * 0.5 + 0.5).squeeze(0).permute(1, 2, 0).flip(2)
    sr = np.clip(sr.float().cpu().numpy(), 0, 1) * 255.0
    return cv2.imdecode(cv2.imencode(".png", sr)[1], cv2.IMREAD_UNCHANGED)      # the float -> uint8 conversion of cv2.imwrite


def main():
    import cv2
    sys.path.insert(0, ROOT)
    cv2.ipp.setUseIPP(False)
    from marconet_b200 import pipeline
    from marconet_b200.testing import synth
    from oracle import ref_harness, wide_line
    torch.set_num_threads(os.cpu_count() or 1)
    models = ref_harness.build_reference_models(synth.make_checkpoints(0))
    img, boxes, labels = make_line()
    h, w = img.shape[:2]
    segs = pipeline.plan_segments(h, w, boxes, labels=labels)
    srs = []
    for s in segs:
        crop = np.ascontiguousarray(img[:, s.crop[0]:s.crop[1]])
        srs.append(script_sr_bytes(models, crop, s.boxes, labels[s.chars[0]:s.chars[1]]))
        print("crop", s.crop, "chars", s.chars, flush=True)
    cuts = [s.core[0] for s in segs] + [w]
    crops = [s.crop for s in segs]
    line = wide_line.stitch_sr(h, w, cuts, crops, srs)
    np.savez_compressed(OUT, image=img, boxes=np.asarray(boxes, np.int64), labels=labels, cuts=np.asarray(cuts, np.int64),
                        crops=np.asarray(crops, np.int64), chars=np.asarray([s.chars for s in segs], np.int64),
                        sr_line=np.ascontiguousarray(line[::STRIDE, ::STRIDE]), stride=np.array(STRIDE))
    print("wrote", OUT, img.shape, "LQ width", round(w * 32 / h), "segments", len(segs), line.shape, os.path.getsize(OUT))


if __name__ == "__main__":
    main()
