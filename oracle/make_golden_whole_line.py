"""Generates tests/golden/whole_line.npz: two seeded synthetic text lines wider than the 32x512 LQ canvas, each restored with its
SR decoder run ONCE on the whole line (pipeline.restore_images(whole_lines=True); DESIGN.md section 7b) by the reference's
UNMODIFIED modules on the CPU (oracle/ref_harness.py, synthetic checkpoints seed 0), real cv2 (IPP off) and torchvision's
ToTensor / Normalize:

* the encoder runs on the crops of marconet_b200.pipeline.plan_segments, each as test_sr.py (:98-111) prepares a hand-cut crop,
  and every character takes the style w of the crop that owns it;
* TSPGAN runs once for all characters of the line;
* TSPSRNet runs on the cubic resize of the whole image to height 32, zero-filled to Wc = 4*ceil(lq_w/4) columns, with
  locs = boxes_to_locs(boxes, h, Wc); its window integers are read from the reference loop itself (make_golden2.traced_sr);
* the output is converted as test_sr.py:198-201 and kept to columns [0, min(rint(w*128/h), 4*Wc)).

Lines: make_golden_wide_line.make_line() (h = 40, about 1260 LQ pixels, a gap wider than the canvas) and a second seeded line at
a non-integer scale (h = 24, about 700 LQ pixels, 30 characters).

Needs a reference checkout (MARCONET_REFERENCE=<path>):  python -m oracle.make_golden_whole_line
"""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OUT = os.path.join(ROOT, "tests", "golden", "whole_line.npz")
STRIDE = 2              # the stored bytes are subsampled [::STRIDE, ::STRIDE], like wide_line.npz
SAMPLE = (7, 29)        # fp32 samples: sr[0, :, ::7, ::29]


def make_line2(seed=1, h=24):
    """h x ~525 uint8 BGR line of 30 characters at a non-integer LQ scale (32/24)."""
    rng = np.random.default_rng(seed)
    boxes, x = [], 6
    for _ in range(30):
        cw = int(rng.integers(11, 17))
        boxes.append([x, int(rng.integers(1, 4)), x + cw, h - int(rng.integers(1, 4))])
        x += cw + int(rng.integers(1, 6))
    w = x + 7
    img = np.full((h, w, 3), rng.integers(160, 235, 3), np.int32)
    img += rng.integers(-25, 26, (h, w, 1))
    for x1, y1, x2, y2 in boxes:
        ink = rng.integers(0, 90, 3)
        mask = rng.random((y2 - y1, x2 - x1)) < 0.5
        img[y1:y2, x1:x2][mask] = ink
    labels = rng.integers(0, 6735, len(boxes))
    return np.clip(img, 0, 255).astype(np.uint8), boxes, labels.astype(np.int64)


def script_lq(img, out_w):
    """test_sr.py:98-111 with a canvas of out_w columns: cv2's cubic resize to height 32, zero fill, ToTensor, Normalize."""
    import cv2
    from torchvision import transforms
    h = img.shape[0]
    lq = cv2.resize(img, (0, 0), fx=32 / h, fy=32 / h, interpolation=cv2.INTER_CUBIC)
    canvas = np.zeros((32, out_w, 3)).astype(lq.dtype)
    assert lq.shape[-2] <= out_w, lq.shape
    canvas[:, :lq.shape[-2], :] = canvas[:, :lq.shape[-2], :] + lq
    return transforms.Normalize((0.5, 0.5, 0.5), (0.5, 0.5, 0.5))(transforms.ToTensor()(canvas)).unsqueeze(0), lq.shape[1]


def script_bytes(sr):
    """test_sr.py:198-201 and cv2.imwrite's float -> uint8 conversion: [1, 3, 128, W] -> uint8 [128, W, 3]."""
    import cv2
    x = (sr * 0.5 + 0.5).squeeze(0).permute(1, 2, 0).flip(2)
    x = np.clip(x.float().cpu().numpy(), 0, 1) * 255.0
    return cv2.imdecode(cv2.imencode(".png", x)[1], cv2.IMREAD_UNCHANGED)


def whole_line(models, img, boxes, labels):
    from marconet_b200 import pipeline
    from oracle import whole_line as wl
    from oracle.make_golden2 import traced_sr
    h, w = img.shape[:2]
    segs = pipeline.plan_segments(h, w, boxes, labels=labels)
    owner = np.zeros(len(boxes), np.int64)
    styles = []
    with torch.no_grad():
        for k, s in enumerate(segs):
            t, _ = script_lq(np.ascontiguousarray(img[:, s.crop[0]:s.crop[1]]), 512)
            _, _, st = models["encoder"](t)
            owner[s.chars[0]:s.chars[1]] = k
            styles.append(st[:1])
        style = torch.cat([styles[k] for k in owner.tolist()], dim=0)
        lab = torch.Tensor(list(labels)).type(torch.LongTensor).unsqueeze(1)
        _, f64, f32_ = models["tspgan"](styles=style, labels=lab, noise=None)
    lq_w, wc = wl.whole_line_width(h, w)
    t, got = script_lq(img, wc)
    assert got == lq_w and lq_w > 512 and wc % 512, (lq_w, wc)
    locs = pipeline.boxes_to_locs(boxes, h, wc)
    sr, wins = traced_sr(models, t, [f64], [f32_], locs)
    out = wl.whole_line_bytes(h, w, wc, script_bytes(sr))
    return dict(segs=segs, owner=owner, wc=wc, lq_w=lq_w, windows=wins, sr=sr, out=out)


def main():
    import cv2
    sys.path.insert(0, ROOT)
    cv2.ipp.setUseIPP(False)
    from marconet_b200.testing import synth
    from oracle import ref_harness
    from oracle.make_golden_wide_line import make_line
    torch.set_num_threads(os.cpu_count() or 1)
    models = ref_harness.build_reference_models(synth.make_checkpoints(0))
    data = dict(stride=np.array(STRIDE), sample=np.asarray(SAMPLE, np.int64), lines=np.array(2))
    for i, (img, boxes, labels) in enumerate([make_line(), make_line2()]):
        r = whole_line(models, img, boxes, labels)
        sr = r["sr"][0]
        data.update({
            f"image{i}": img, f"boxes{i}": np.asarray(boxes, np.int64), f"labels{i}": labels,
            f"crops{i}": np.asarray([s.crop for s in r["segs"]], np.int64), f"chars{i}": np.asarray([s.chars for s in r["segs"]], np.int64),
            f"owner{i}": r["owner"], f"wc{i}": np.array(r["wc"]), f"lq_w{i}": np.array(r["lq_w"]),
            f"windows{i}": r["windows"],
            f"sr_samples{i}": np.ascontiguousarray(sr[:, ::SAMPLE[0], ::SAMPLE[1]].numpy()),
            f"sr_sum{i}": np.array(sr.double().sum().item()),
            f"sr_u8{i}": np.ascontiguousarray(r["out"][::STRIDE, ::STRIDE]),
        })
        print("line", i, img.shape, "lq_w", r["lq_w"], "Wc", r["wc"], "segments", len(r["segs"]), "windows", len(r["windows"]),
              "out", r["out"].shape, flush=True)
    np.savez_compressed(OUT, **data)
    print("wrote", OUT, os.path.getsize(OUT))


if __name__ == "__main__":
    main()
