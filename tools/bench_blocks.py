"""Text blocks (DESIGN.md section 7b, "Text blocks"): the segmentation alone and restore_regions with blocks.

    MN_MODULE_GRAPHS=0 python tools/bench_blocks.py [--pages 4] [--lines 16] [--passes 3] [--iters 200] [--scale 2] [--skew]

The pages are seeded paragraphs drawn with cv2.putText (Hershey fonts) on a light, slightly noisy background, one TextBlock
around each paragraph.  Prints one JSON line each for:
  - segmentation: ops.find_lines (mn_find_lines_u8: four launches for every block of the call) on the uploaded pages, timed with
    CUDA events over --iters calls, per call and per block;
  - restore_regions with the blocks against the same call given the found rectangles, host uint8 in and out, pages/s; the arms
    alternate pass by pass and must give the same bytes.
With --skew (DESIGN.md section 7b, "Skewed blocks") each page is rotated by a seeded angle in +-8 degrees and its block is
TextBlock(rect, skew="auto"): the first line times the angle search and the segmentation (mn_find_lines_skewed_u8, six
launches), and restore_regions with the blocks is compared against the call given the found OrientedRegions.
Every line carries the card's name and power limit, read in the same run.  Not part of the product path.
"""
import argparse
import json
import os
import subprocess
import sys
import time

os.environ.setdefault("MN_MODULE_GRAPHS", "0")

import cv2  # noqa: E402
import numpy as np  # noqa: E402
import torch  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

WORDS = "the quick brown fox jumps over a lazy dog pack my box with five dozen liquor jugs 0123456789".split()


def make_pages(n_pages, n_lines, seed=0, skew=False):
    """n_pages paragraphs of n_lines lines, 40 pixels apart: (pages, blocks, angles).  With ``skew`` each page is rotated by a
    seeded angle in +-8 degrees about its centre (the text drawn inside a margin that keeps it on the page) and its block
    searches for the angle."""
    from marconet_b200 import pipeline
    rng = np.random.default_rng(seed)
    pages, blocks, angles = [], [], []
    for _ in range(n_pages):
        m = 90 if skew else 0
        H, W = 60 + 40 * n_lines + 2 * m, 900 + 2 * m
        bg = rng.integers(215, 246, 3)
        page = np.empty((H, W, 3), np.uint8) if skew else np.clip(bg + rng.integers(-12, 13, (H, W, 1)), 0, 255).astype(np.uint8)
        if skew:
            page[:] = bg
        for k in range(n_lines):
            text = " ".join(rng.choice(WORDS, int(rng.integers(5, 10))))
            cv2.putText(page, text, (30 + m, 60 + 40 * k + m), cv2.FONT_HERSHEY_SIMPLEX, 0.9, (20, 20, 20), 2, cv2.LINE_AA)
        angle = float(rng.uniform(-8, 8)) if skew else 0.0
        if skew:                                        # rotated, then the same noise as the level pages
            rot = cv2.getRotationMatrix2D((W / 2, H / 2), angle, 1.0)
            page = cv2.warpAffine(page, rot, (W, H), flags=cv2.INTER_LINEAR, borderValue=tuple(int(v) for v in bg))
            page = np.clip(page.astype(np.int32) + rng.integers(-12, 13, (H, W, 1)), 0, 255).astype(np.uint8)
        pages.append(page)
        angles.append(angle)
        blocks.append([pipeline.TextBlock((10, 10, W - 10, H - 10), skew="auto" if skew else None)])
    return pages, blocks, angles


def _card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True,
                       text=True)
    name, _, power = q.stdout.strip().partition(", ")
    return {"gpu": name or torch.cuda.get_device_name(0), "power_limit": power or None}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--pages", type=int, default=4)
    ap.add_argument("--lines", type=int, default=16)
    ap.add_argument("--passes", type=int, default=3)
    ap.add_argument("--iters", type=int, default=200)
    ap.add_argument("--scale", type=int, default=2)
    ap.add_argument("--skew", action="store_true", help="rotated pages and TextBlock(skew='auto')")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_blocks.py needs a CUDA device")
    from marconet_b200 import _lib, ops, pipeline
    from marconet_b200.models import networks
    from marconet_b200.testing import synth
    dev = torch.device("cuda:0")
    card = _card()
    pages, blocks, angles = make_pages(args.pages, args.lines, skew=args.skew)

    dpages = [torch.from_numpy(p).to(dev) for p in pages]
    items = [(dpages[i], b.rect, False, _lib.INK_AUTO, None, None, None, b.skew, b.max_skew) for i, bl in enumerate(blocks)
             for b in bl]
    for _ in range(5):
        ops.find_lines(items)
    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0.record()
    for _ in range(args.iters):
        ops.find_lines(items)
    t1.record()
    t1.synchronize()
    ms = t0.elapsed_time(t1) / args.iters
    pixels = sum((b.rect[2] - b.rect[0]) * (b.rect[3] - b.rect[1]) for bl in blocks for b in bl)
    what = "angle search and segmentation" if args.skew else "segmentation"
    extra = dict(angles_per_block=401, true_angles=[round(a, 3) for a in angles]) if args.skew else {}
    print(json.dumps(dict(card, what=what, blocks=len(items), megapixels=pixels / 1e6, ms_per_call=round(ms, 4),
                          us_per_block=round(1000 * ms / len(items), 2), **extra)), flush=True)

    sds = synth.make_checkpoints(0)
    m = []
    for key, cls in (("encoder", networks.TextContextEncoderV2), ("tspgan", networks.TSPGAN), ("sr", networks.TSPSRNet)):
        net = cls()
        net.load_state_dict(sds[key], strict=True)
        m.append(net.eval().to(dev))
    found = pipeline.find_lines(pages, blocks)
    if args.skew:
        print(json.dumps(dict(card, what="found angles", skew=[r["skew"] for f in found for r in f],
                              lines=[len(r["lines"]) for f in found for r in f])), flush=True)
    rects = [[q for r in f for q in r["lines"]] for f in found]
    kw = dict(scale=args.scale, skip_invalid=True, to_host=True)
    given = "found lines" if args.skew else "rectangles"
    arms = {"blocks": lambda: pipeline.restore_regions(*m, pages, blocks, **kw),
            given: lambda: pipeline.restore_regions(*m, pages, rects, **kw)}
    outs = {name: fn() for name, fn in arms.items()}          # warm-up of every shape
    times = {name: [] for name in arms}
    for _ in range(args.passes):
        for name, fn in arms.items():
            torch.cuda.synchronize()
            t = time.perf_counter()
            outs[name] = fn()
            times[name].append(time.perf_counter() - t)
    for a, b in zip(outs["blocks"], outs[given]):
        assert np.array_equal(a["image"], b["image"]), "the arms differ"
    for name, ts in times.items():
        med = float(np.median(ts))
        print(json.dumps(dict(card, what=f"restore_regions with {name}", pages=len(pages), lines=sum(len(r) for r in rects),
                              scale=args.scale, pages_per_s=round(len(pages) / med, 3), seconds=[round(t, 4) for t in ts])),
              flush=True)


if __name__ == "__main__":
    main()
