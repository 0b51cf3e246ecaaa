"""Text-line images of mixed widths end to end (host uint8 in, host uint8 out, every copy inside the timed region):
pipeline.restore_images at max_lines 1, 4 and 8, against the loop a user writes today -- restore_image on each crop of the same
plan, then a device->host copy of its bytes.

    python tools/bench_images.py [--images 42] [--passes 3] [--warmup 1] [--whole-lines | --figures | --predicted]

--whole-lines compares the two ways restore_images decodes a line wider than the canvas, at max_lines 1 and 8: crop by crop
(the default) and in one piece (whole_lines=True), with the arms' passes alternated, and reports each mode's decoder SR columns
per pass (batch lines x SR canvas width, summed over the decoder calls).

--figures times test_sr.py's four-panel figure at max_lines 8: restore_images without figures, with figure=True (composed on the
device, one pinned copy back), and the host path a user has without it -- restore_images' SR bytes, then every character's prior
image copied back (fp32 [3, 128, 128]) and the figure composed with cv2 as test_sr.py:206-231 does (ShowLQ cubic resize, markers,
INTER_LINEAR prior strip, vstack).  The host arm reads priors generated once before timing (the generator's work is already
inside restore_images; only the copy back and the cv2 work are added).

--predicted times restore_images at max_lines 8 with the set's labels and boxes given against labels=None, boxes=None (the
encoder predicts both on its detection windows first, pipeline.predict_characters; skip_invalid, since the synthetic weights'
boxes need not fit a plan), and predict_characters alone, whose time over the predicted arm's is the share spent in detection.
Run it with MN_MODULE_GRAPHS=0: the synthetic weights predict 16 characters on every crop, and six recorded TSPSRNet signatures
of such batches outgrow an 80 GB card.

The image set reuses the 17 (h, w) sizes of the reference's Testsets/LQs (resized LQ widths 92 to 464 pixels, all inside the
512-pixel canvas) and adds lines 2 to 4 times wider than the canvas, which test_sr.py refuses (:107-110), with one character box
per 28 LQ pixels.  Host clock around whole passes over the set (each ends synchronised).  Prints one JSON line with the card's
name and power limit read in the same run.  Not part of the product path.
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

TESTSET_SIZES = [(22, 181), (12, 108), (17, 49), (20, 112), (17, 86), (15, 61), (14, 47), (12, 52), (49, 304), (14, 45), (14, 44),
                 (15, 55), (32, 388), (128, 1472), (128, 1268), (128, 1160), (128, 1856)]
WIDE_LINES = [(32, 1100), (40, 1536), (24, 2040), (64, 1300)]        # (h, LQ width)


def make_image_set(n, seed=0):
    """n seeded uint8 line images cycling through TESTSET_SIZES and WIDE_LINES, one character box per 28 LQ pixels."""
    rng = np.random.default_rng(seed)
    sizes = TESTSET_SIZES + [(h, round(lq_w * h / 32)) for h, lq_w in WIDE_LINES]
    images, labels, boxes = [], [], []
    for i in range(n):
        h, w = sizes[i % len(sizes)]
        pitch = 28 * h / 32
        k = max(1, int(w // pitch))
        images.append(rng.integers(0, 256, (h, w, 3), dtype=np.uint8))
        boxes.append([[int(j * pitch + 0.15 * pitch), 0, int(j * pitch + 0.85 * pitch), h] for j in range(k)])
        labels.append(rng.integers(0, 6735, k).tolist())
    return images, labels, boxes


def sr_columns(arm, images, plans):
    """SR columns the decoder computes in one pass of an arm: every crop line is a 2048-column canvas; in whole-line mode every
    batch of pipeline.pack_by_columns is (lines) x 4 x (its widest Wc)."""
    from marconet_b200 import pipeline
    if "_whole_lines" not in arm:
        return 4 * 512 * sum(len(p) for p in plans)
    m = int(arm.rsplit("_", 1)[1])
    wcs = [pipeline.whole_line_width(im.shape[0], im.shape[1])[1] for im in images]
    return sum(4 * len(b) * max(wcs[j] for j in b) for b in pipeline.pack_by_columns(wcs, m))


def host_figure(img, boxes, priors_host, sr_u8):
    """test_sr.py:98,206-231 on the host with cv2: the figure of one image from its SR bytes and its priors (fp32 numpy)."""
    import cv2
    from marconet_b200 import pipeline
    h, w = img.shape[:2]
    show_lq = cv2.resize(img, (0, 0), fx=128 / h, fy=128 / h, interpolation=cv2.INTER_CUBIC)
    wc = pipeline.whole_line_width(h, w)[1]
    top, bot = pipeline.figure_markers(pipeline.boxes_to_locs(boxes, h, wc)[0].tolist(), show_lq.shape[1], 4 * wc)
    show_locs = show_lq.copy()
    for a, b in top:
        show_locs[:64, a:b] = (255, 0, 0)
    for a, b in bot:
        show_locs[64:, a:b] = (0, 0, 255)
    strip = np.hstack(list((priors_host * 0.5 + 0.5).transpose(0, 2, 3, 1)))
    prior = cv2.resize(strip, (show_lq.shape[1], 128)) * 255
    W = sr_u8.shape[1]
    return np.vstack((show_lq[:, :W, ::-1], show_locs[:, :W, ::-1], sr_u8, np.clip(np.rint(prior[:, :W]), 0, 255).astype(np.uint8)))


def figure_arms(enc, gen, sr, images, labels, boxes, dev, max_lines=8):
    from marconet_b200 import pipeline
    n_chars = sum(len(l) for l in labels)
    with torch.no_grad():                                   # stand-in device priors, as many as the set has characters
        lab = torch.tensor([v for l in labels for v in l], dtype=torch.long).reshape(-1, 1)
        priors_dev = torch.cat([gen(styles=torch.zeros(min(256, n_chars - o), 512, device=dev), labels=lab[o:o + 256], noise=None)[0]
                                for o in range(0, n_chars, 256)])

    def host():
        res = pipeline.restore_images(enc, gen, sr, images, labels, boxes, max_lines=max_lines, to_host=True)
        pri = priors_dev.cpu().numpy()
        o = 0
        for im, l, bx, r in zip(images, labels, boxes, res):
            host_figure(im, bx, pri[o:o + len(l)], r["sr_u8"])
            o += len(l)

    return {f"restore_images_max_lines_{max_lines}": lambda: pipeline.restore_images(enc, gen, sr, images, labels, boxes,
                                                                                     max_lines=max_lines, to_host=True),
            f"restore_images_max_lines_{max_lines}_figure": lambda: pipeline.restore_images(enc, gen, sr, images, labels, boxes,
                                                                                            max_lines=max_lines, to_host=True, figure=True),
            f"restore_images_max_lines_{max_lines}_host_cv2_figure": host}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--images", type=int, default=42)
    ap.add_argument("--passes", type=int, default=3, help="timed passes over the image set per arm")
    ap.add_argument("--warmup", type=int, default=1, help="untimed passes per arm first")
    ap.add_argument("--whole-lines", action="store_true", help="crop-by-crop vs whole-line decoding of the wide lines")
    ap.add_argument("--figures", action="store_true", help="test_sr.py's figure on the device vs on the host with cv2")
    ap.add_argument("--predicted", action="store_true", help="given labels and boxes vs encoder-predicted ones")
    args = ap.parse_args()
    from marconet_b200 import pipeline
    from marconet_b200.models import networks
    from marconet_b200.testing import synth

    if not torch.cuda.is_available():
        raise SystemExit("bench_images.py: no CUDA device (the product path has no CPU fallback)")
    dev = torch.device("cuda:0")
    sds = synth.make_checkpoints(0)
    nets = {}
    for key, cls in (("tspgan", networks.TSPGAN), ("encoder", networks.TextContextEncoderV2), ("sr", networks.TSPSRNet)):
        m = cls()
        m.load_state_dict(sds[key], strict=True)
        nets[key] = m.eval().to(dev)
    enc, gen, sr = nets["encoder"], nets["tspgan"], nets["sr"]

    images, labels, boxes = make_image_set(args.images)
    plans = [pipeline.plan_segments(im.shape[0], im.shape[1], b) for im, b in zip(images, boxes)]
    crops = [(np.ascontiguousarray(im[:, s.crop[0]:s.crop[1]]), lab[s.chars[0]:s.chars[1]], s.boxes)
             for im, lab, p in zip(images, labels, plans) for s in p if s.chars[1] > s.chars[0]]
    n_chars = sum(len(l) for l in labels)

    def loop():
        for c, lab, bx in crops:
            pipeline.restore_image(enc, gen, sr, c, lab, bx)["sr_u8"].cpu()

    if args.figures:
        arms = figure_arms(enc, gen, sr, images, labels, boxes, dev)
    elif args.predicted:
        arms = {"restore_images_max_lines_8": lambda: pipeline.restore_images(enc, gen, sr, images, labels, boxes, max_lines=8, to_host=True),
                "restore_images_max_lines_8_predicted": lambda: pipeline.restore_images(enc, gen, sr, images, None, None, max_lines=8,
                                                                                         to_host=True, skip_invalid=True),
                "predict_characters_max_lines_8": lambda: pipeline.predict_characters(enc, images, max_lines=8)}
    elif args.whole_lines:
        arms = {f"restore_images{'_whole_lines' if wl else ''}_max_lines_{m}":
                (lambda m=m, wl=wl: pipeline.restore_images(enc, gen, sr, images, labels, boxes, max_lines=m, to_host=True, whole_lines=wl))
                for m in (1, 8) for wl in (False, True)}
    else:
        arms = {f"restore_images_max_lines_{m}": (lambda m=m: pipeline.restore_images(enc, gen, sr, images, labels, boxes, max_lines=m,
                                                                                      to_host=True)) for m in (1, 4, 8)}
        arms["restore_image_loop_over_crops"] = loop
    out = {}
    with torch.no_grad():
        for fn in arms.values():
            for _ in range(max(1, args.warmup)):
                fn()
        secs = dict.fromkeys(arms, 0.0)
        for _ in range(args.passes):              # arms alternated pass by pass: drift of a shared host hits all of them alike
            for name, fn in arms.items():
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                fn()
                torch.cuda.synchronize()
                secs[name] += time.perf_counter() - t0
        for name in arms:
            s = secs[name] / args.passes
            out[name] = {"s_per_pass": s, "images_per_sec": len(images) / s, "chars_per_sec": n_chars / s}
            if args.whole_lines:
                out[name]["decoder_sr_columns_per_pass"] = sr_columns(name, images, plans)
        if args.predicted:
            res = pipeline.restore_images(enc, gen, sr, images, None, None, max_lines=8, to_host=True, skip_invalid=True)
            out["restore_images_max_lines_8_predicted"].update(
                restored=sum("error" not in r for r in res), predicted_chars=sum(len(r.get("labels", [])) for r in res),
                windows=sum(len(pipeline.plan_windows(*im.shape[:2])) for im in images))
            out["detection_share"] = out["predict_characters_max_lines_8"]["s_per_pass"] / \
                out["restore_images_max_lines_8_predicted"]["s_per_pass"]
    card = {"name": torch.cuda.get_device_name(dev)}
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=10).stdout.strip()
        card["power_limit"] = q or None
    except Exception as exc:
        card["power_limit"] = f"unavailable ({type(exc).__name__})"
    print(json.dumps({"metric": "images_e2e", "images": len(images), "lines": sum(len(p) for p in plans), "crops_with_chars": len(crops),
                      "chars": n_chars, "wide_images": sum(len(p) > 1 for p in plans), "passes": args.passes,
                      "warmup_passes": max(1, args.warmup), "arms": out, "gpu": card,
                      "workload": f"{len(images)} seeded uint8 line images cycling through the 17 sizes of the reference's Testsets/LQs "
                                  f"and {len(WIDE_LINES)} lines 2-4x wider than the canvas, one character per 28 LQ pixels; "
                                  f"host numpy in, host numpy out"}), flush=True)


if __name__ == "__main__":
    main()
