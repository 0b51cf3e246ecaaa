"""Generates tests/golden/figure.npz: the four-panel figure of test_sr.py (:206-231; DESIGN.md section 7b) for

(a) the PNGs the reference's UNMODIFIED test_sr.py writes on the CPU for a directory of synthetic line images, run exactly as
    oracle/make_golden_script.py runs it (detector / OCR stand-ins of oracle/stubs, OPENCV_IPP=disabled, synthetic checkpoints
    seed 0).  The lines cover ShowLQ widths S equal to (identity prior resize), above (up-scaled strip) and below (down-scaled
    strip, non-integer scales) 128 * n.  Stored per line: the image the script used, its boxes and labels, panels 1-2 in full,
    the prior panel's every column at rows [::PRIOR_ROWS] and the SR panel subsampled [::STRIDE, ::STRIDE];

(b) one line wider than the LQ canvas (make_golden_whole_line.make_line2: 24 x ~520, 30 characters, S = 4*Wc), which the script
    skips: its prior panel computed with the reference's UNMODIFIED modules on the CPU (oracle/ref_harness.py), every character
    taking the style w of the crop of pipeline.plan_segments that owns it (as make_golden_whole_line.py), real cv2's INTER_LINEAR
    resize of the prior strip (every column, rows [::PRIOR_ROWS]), and the figure geometry.

Needs a reference checkout (MARCONET_REFERENCE=<path>):  python -m oracle.make_golden_figure
"""
import os
import subprocess
import sys
import tempfile

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF = os.environ.get("MARCONET_REFERENCE", "")
STUBS = os.path.join(ROOT, "oracle", "stubs")
OUT = os.path.join(ROOT, "tests", "golden", "figure.npz")
STRIDE = 4      # the stored SR panel of (a) is subsampled [::STRIDE, ::STRIDE] (the SR bytes are pinned by other fixtures too)
PRIOR_ROWS = 4  # the prior panels keep every column (the resize is horizontal: 128 -> 128 rows is the identity), rows [::PRIOR_ROWS]
# (h, w): S = rint(w*128/h) against the stand-in detector's 8 boxes (128 * 8 = 1024 strip columns)
LINES = [(32, 256),      # S = 1024: the identity resize of the prior strip
         (24, 300),      # S = 1600: up-scaled strip
         (40, 250),      # S = 800: down-scaled, non-integer factor
         (36, 190)]      # S = 676: down-scaled, h does not divide 128


def make_flat_line(h, w, seed):
    """Low-entropy uint8 line: a flat background and 8 flat ink blocks where the stand-in detector puts its boxes."""
    rng = np.random.default_rng(seed)
    img = np.empty((h, w, 3), np.uint8)
    img[:] = rng.integers(150, 240, 3)
    step = w / 8
    for i in range(8):
        x1, x2 = int(i * step + 0.25 * step), int((i + 1) * step - 0.25 * step)
        img[h // 5:h - h // 5, x1:x2] = rng.integers(0, 90, 3)
    return img


def script_figures():
    import cv2
    from marconet_b200.testing import synth
    sds = synth.make_checkpoints(0)
    out = {}
    with tempfile.TemporaryDirectory() as d:
        os.makedirs(os.path.join(d, "checkpoints"))
        for key, name in (("tspgan", "net_prior_generation.pth"), ("sr", "net_sr.pth"), ("encoder", "net_transformer_encoder.pth")):
            torch.save({"params": sds[key]}, os.path.join(d, "checkpoints", name))
        os.makedirs(os.path.join(d, "LQs"))
        paths = []
        for i, (h, w) in enumerate(LINES):
            paths.append(os.path.join(d, "LQs", f"line{i}.png"))
            cv2.imwrite(paths[-1], make_flat_line(h, w, 10 + i))
        env = dict(os.environ, PYTHONPATH=STUBS, OPENCV_IPP="disabled", OMP_NUM_THREADS=str(os.cpu_count() or 1))
        r = subprocess.run([sys.executable, os.path.join(REF, "test_sr.py"), "-i", "./LQs", "-o", "./out"], cwd=d, env=env,
                           capture_output=True, text=True, timeout=3600)
        assert r.returncode == 0, r.stderr[-3000:]
        pngs = sorted(os.listdir(os.path.join(d, "out")))
        assert len(pngs) == len(LINES), pngs
        # detector / OCR stand-ins, through the reference's own helper, to record what the script fed the nets
        sys.path[:0] = [STUBS, REF]
        from ultralytics import YOLO
        from modelscope.pipelines import pipeline
        from utils.yolo_ocr_xloc import get_yolo_ocr_xloc
        from utils.alphabets import alphabet
        for i, path in enumerate(paths):
            png = cv2.imread(os.path.join(d, "out", pngs[i]))
            assert pngs[i].startswith(f"line{i}_"), pngs
            rgb, boxes, chars, _ = get_yolo_ocr_xloc(path, yolo_model=YOLO(None), ocr_pipeline=pipeline(None), num_cropped_boxes=5,
                                                     expand_px=1, expand_px_for_first_last_cha=12, yolo_iou=0.1, yolo_conf=0.07)
            labels = [alphabet.find(c) for c in chars]
            assert min(labels) >= 0
            h, w = LINES[i]
            assert png.shape == (512, int(np.rint(w * 128 / h)), 3), png.shape
            out.update({f"image{i}": np.ascontiguousarray(rgb), f"boxes{i}": np.asarray(boxes, np.int64),
                        f"labels{i}": np.asarray(labels, np.int64), f"show{i}": np.ascontiguousarray(png[:256]),
                        f"sr_row{i}": np.ascontiguousarray(png[256:384][::STRIDE, ::STRIDE]),
                        f"prior_row{i}": np.ascontiguousarray(png[384::PRIOR_ROWS])})
            print("line", i, rgb.shape, "S", png.shape[1], "chars", "".join(chars), flush=True)
    return out


def wide_line_prior():
    import cv2
    from marconet_b200 import pipeline
    from marconet_b200.testing import synth
    from oracle import ref_harness
    from oracle.make_golden_whole_line import make_line2, script_lq
    cv2.ipp.setUseIPP(False)
    models = ref_harness.build_reference_models(synth.make_checkpoints(0))
    img, boxes, labels = make_line2()
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
        prior_cha, _, _ = models["tspgan"](styles=style, labels=lab, noise=None)
    S = int(np.rint(w * 128 / h))
    lq_w, wc = pipeline.whole_line_width(h, w)
    W = min(S, 4 * wc)
    assert lq_w > 512 and len(boxes) * 128 > S, (lq_w, S)          # wider than the canvas; the strip is down-scaled
    # test_sr.py:206-211 and cv2.imwrite's float -> uint8 conversion
    p = (prior_cha * 0.5 + 0.5).permute(0, 2, 3, 1).cpu().numpy()
    prior128 = p[0]
    for i in range(1, len(p)):
        prior128 = np.hstack((prior128, p[i]))
    prior = cv2.resize(prior128, (S, 128)) * 255
    row = cv2.imdecode(cv2.imencode(".png", prior)[1], cv2.IMREAD_UNCHANGED)
    print("wide line", img.shape, "S", S, "Wc", wc, "W", W, "segments", len(segs), flush=True)
    return {"wide_image": img, "wide_boxes": np.asarray(boxes, np.int64), "wide_labels": labels, "wide_owner": owner,
            "wide_crops": np.asarray([s.crop for s in segs], np.int64),
            "wide_geometry": np.array([S, W, wc, 4 * wc], np.int64), "wide_prior_row": np.ascontiguousarray(row[::PRIOR_ROWS, :W])}


def main():
    sys.path.insert(0, ROOT)
    torch.set_num_threads(os.cpu_count() or 1)
    data = dict(stride=np.array(STRIDE), prior_rows=np.array(PRIOR_ROWS), lines=np.array(len(LINES)))
    data.update(script_figures())
    data.update(wide_line_prior())
    np.savez_compressed(OUT, **data)
    print("wrote", OUT, os.path.getsize(OUT))


if __name__ == "__main__":
    main()
