"""Generates tests/golden/predict.npz: what the reference's UNMODIFIED TextContextEncoderV2 (oracle/ref_harness.py, synthetic
checkpoints seed 0) predicts on every detection window (pipeline.plan_windows) of two seeded text lines -- one that fits the
canvas at a non-integer scale (h = 27) and one about 2.7 times wider than the canvas (three windows).

Each window is cut by hand and encoded as test_sr.py:99-113 encodes a crop: real cv2 cubic resize at fx = fy = 32/h (IPP off),
zero-fill to 32x512, torchvision ToTensor / Normalize.  Stored per window: the argmax at every timestep, the top-1 minus top-2
margin, locs_lr and the labels of the reference's own clear_labels (test_w.py:34-40, imported through the harness); per image:
the image, the windows and the twin's merged labels and boxes (oracle/predict.py).  Every margin must be at least 5e-3 -- ten
times the bound the device encoder's logits are held to -- so that the device must reproduce every label.  With the synthetic
weights a 64-step margin that wide is rare (about one seed in 35 per window), so the image is built window by window: the
columns a window adds to its left neighbour's take the next seed until that window's margins are wide enough, which leaves the
windows to its left unchanged; after 150 seeds the left neighbour moves on to its next good seed.

Needs a reference checkout (MARCONET_REFERENCE=<path>):  python -m oracle.make_golden_predict
"""
import importlib
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OUT = os.path.join(ROOT, "tests", "golden", "predict.npz")
MARGIN = 5e-3
TRIES = 150
SHAPES = dict(fit=(27, 300), wide=(40, 1757))      # wide: w = W* + 2 strides, every window adds 559 new columns


def make_image(seed, h, w):
    """Seeded h x w uint8 BGR line: a light background and dark strokes in character-sized cells."""
    rng = np.random.default_rng(seed)
    img = np.full((h, w, 3), rng.integers(170, 230, 3), np.int32) + rng.integers(-20, 21, (h, w, 1))
    x = int(rng.integers(2, 10))
    while x < w - 4:
        cw = int(rng.integers(h // 2, h + 1))
        mask = rng.random((h - 6, min(cw, w - x))) < 0.5
        img[3:h - 3, x:x + cw][mask] = rng.integers(0, 80, 3)
        x += cw + int(rng.integers(2, 8))
    return np.clip(img, 0, 255).astype(np.uint8)


def encode_crop(crop):
    """test_sr.py:99-113 on a hand-cut crop -> the [1, 3, 32, 512] tensor the script feeds the encoder."""
    import cv2
    from torchvision import transforms
    h = crop.shape[0]
    lq = cv2.resize(crop, (0, 0), fx=32 / h, fy=32 / h, interpolation=cv2.INTER_CUBIC)
    canvas = np.zeros((32, 32 * 16, 3)).astype(lq.dtype)
    assert lq.shape[-2] <= 32 * 16, lq.shape
    canvas[:, :lq.shape[-2], :] = canvas[:, :lq.shape[-2], :] + lq
    return transforms.Normalize((0.5, 0.5, 0.5), (0.5, 0.5, 0.5))(transforms.ToTensor()(canvas)).unsqueeze(0)


def main():
    import cv2
    sys.path.insert(0, ROOT)
    cv2.ipp.setUseIPP(False)
    from marconet_b200.testing import synth
    from oracle import predict, ref_harness
    torch.set_num_threads(os.cpu_count() or 1)
    encoder = ref_harness.build_reference_models(synth.make_checkpoints(0))["encoder"]
    test_w = importlib.import_module("test_w")           # the reference script, on the path the harness set up
    rec = {}
    for name, (h, w) in SHAPES.items():
        wins = predict.plan_windows(h, w)
        img, seeds, outs, k = np.zeros((h, w, 3), np.uint8), [1000 * j for j in range(len(wins))], [None] * len(wins), 0
        while k < len(wins):                             # window by window: new columns [start, b) until every margin is wide enough
            (a, b), _ = wins[k]
            start = wins[k - 1][0][1] if k else 0
            for _ in range(TRIES if k else 1 << 30):
                img[:, start:b] = make_image(seeds[k], h, b - start)
                with torch.no_grad():
                    logits, locs, _ = encoder(encode_crop(np.ascontiguousarray(img[:, a:b])))
                top2 = torch.topk(logits[0], 2, dim=1).values
                margin = float((top2[:, 0] - top2[:, 1]).min())
                print(name, "window", k, "seed", seeds[k], "margin", margin, flush=True)
                if margin >= MARGIN:
                    break
                seeds[k] += 1
            if margin >= MARGIN:
                outs[k] = (logits[0], locs[0])
                k += 1
            else:                                        # this window's fixed columns leave no room: move the left one on
                seeds[k], k = 1000 * k, k - 1
                seeds[k] += 1
        with torch.no_grad():                            # the finished image: every window again, as the device reads it
            for k, ((a, b), _) in enumerate(wins):
                logits, locs, _ = encoder(encode_crop(np.ascontiguousarray(img[:, a:b])))
                assert torch.equal(logits[0], outs[k][0]) and torch.equal(locs[0], outs[k][1])
        top2 = [torch.topk(lg, 2, dim=1).values for lg, _ in outs]
        rows = []
        for k, ((a, _), (lo, hi)) in enumerate(wins):
            lg, lr = outs[k]
            rec[f"{name}_ref_labels_{k}"] = np.asarray([int(v) for v in test_w.clear_labels(lg)], np.int64)
            rows.append(predict.decode_row(lg.numpy(), lr.numpy(), a, 16.0 * h, lo, hi)[:3])
        labels, boxes = predict.merge(h, w, rows)
        rec.update({f"{name}_image": img, f"{name}_seeds": np.asarray(seeds), f"{name}_crops": np.asarray([c for c, _ in wins], np.int64),
                    f"{name}_argmax": np.stack([lg.argmax(1).numpy() for lg, _ in outs]).astype(np.int32),
                    f"{name}_margin": np.stack([(t[:, 0] - t[:, 1]).numpy() for t in top2]).astype(np.float32),
                    f"{name}_locs_lr": np.stack([lr.numpy() for _, lr in outs]).astype(np.float32),
                    f"{name}_labels": np.asarray(labels, np.int64), f"{name}_boxes": np.asarray(boxes, np.float64).reshape(-1, 4)})
        print(name, "labels", labels, flush=True)
    np.savez_compressed(OUT, **rec)
    print("wrote", OUT, os.path.getsize(OUT))


if __name__ == "__main__":
    main()
