"""Ruled pages (DESIGN.md section 7b, "Ruled pages"): the layout with and without rules, the rule kernels alone and
restore_regions with ruled pages.

    MN_MODULE_GRAPHS=0 python tools/bench_rules.py [--pages 4] [--passes 3] [--iters 100] [--scale 2] [--profile]

The pages are seeded 1600 x 1200 pages: a heading, a ruled table of 10 x 5 cells (one word each, 2-pixel rules) and a framed
paragraph of 8 lines, capitals drawn with cv2.putText (Hershey DUPLEX) on a light, slightly noisy background.  Prints one JSON
line each for:
  - layout: ops.find_blocks on the uploaded pages with the default rule length and without rules, timed with CUDA events over
    --iters calls per arm, the arms alternating pass by pass;
  - restore_regions with TextPage(rules="auto") against the same call given the found blocks, host uint8 in and out, pages/s;
    the arms alternate pass by pass and must give the same bytes.
With --profile, instead: torch.profiler over --iters ruled layout calls, the device time of the three rule kernels and of every
kernel of the call, per call.  Every line carries the card's name and power limit, read in the same run.  Not part of the
product path.
"""
import argparse
import json
import os
import re
import subprocess
import sys
import time

os.environ.setdefault("MN_MODULE_GRAPHS", "0")

import cv2  # noqa: E402
import numpy as np  # noqa: E402
import torch  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

WORDS = "THE QUICK BROWN FOX JUMPS OVER A LAZY DOG PACK MY BOX WITH FIVE DOZEN JUGS 0123456789".split()
FONT = cv2.FONT_HERSHEY_DUPLEX


def make_pages(n_pages, seed=0):
    """n_pages 1600 x 1200 pages: a heading, a 10 x 5 ruled table of 260 x 47 cells and a framed paragraph of 8 lines."""
    rng = np.random.default_rng(seed)
    H, W = 1200, 1600
    pages = []
    for _ in range(n_pages):
        bg = rng.integers(215, 246, 3)
        page = np.clip(bg + rng.integers(-12, 13, (H, W, 1)), 0, 255).astype(np.uint8)
        ink = (20, 20, 20)
        cv2.putText(page, "A HEADING OVER A TABLE AND A BOX", (40, 70), FONT, 1.0, ink, 2, cv2.LINE_AA)
        x0, y0, cw, ch = 40, 110, 260, 47
        for r in range(11):
            page[y0 + r * ch - 1:y0 + r * ch + 1, x0 - 1:x0 + 5 * cw + 1] = ink
        for c in range(6):
            page[y0 - 1:y0 + 10 * ch + 1, x0 + c * cw - 1:x0 + c * cw + 1] = ink
        for r in range(10):
            for c in range(5):
                cv2.putText(page, str(rng.choice(WORDS)), (x0 + c * cw + 14, y0 + r * ch + 35), FONT, 1.0, ink, 2, cv2.LINE_AA)
        fy = y0 + 10 * ch + 60
        page[fy - 1:fy + 1, 40:W - 40] = ink
        page[fy + 8 * 33 + 39:fy + 8 * 33 + 41, 40:W - 40] = ink
        page[fy:fy + 8 * 33 + 40, 39:41] = ink
        page[fy:fy + 8 * 33 + 40, W - 41:W - 39] = ink
        for k in range(8):
            t = str(rng.choice(WORDS))
            while cv2.getTextSize(t + " " + WORDS[0], FONT, 1.0, 2)[0][0] < W - 200:
                t += " " + str(rng.choice(WORDS))
            cv2.putText(page, t, (70, fy + 48 + 33 * k), FONT, 1.0, ink, 2, cv2.LINE_AA)
        pages.append(page)
    return pages


def _card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True,
                       text=True)
    name, _, power = q.stdout.strip().partition(", ")
    return {"gpu": name or torch.cuda.get_device_name(0), "power_limit": power or None}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--pages", type=int, default=4)
    ap.add_argument("--passes", type=int, default=3)
    ap.add_argument("--iters", type=int, default=100)
    ap.add_argument("--scale", type=int, default=2)
    ap.add_argument("--profile", action="store_true")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_rules.py needs a CUDA device")
    from marconet_b200 import _lib, ops, pipeline
    from marconet_b200.models import networks
    from marconet_b200.testing import synth
    dev = torch.device("cuda:0")
    card = _card()
    pages = make_pages(args.pages)
    d = [torch.from_numpy(p).to(dev) for p in pages]
    plain = [ops.PageItem(x, (0, 0, x.shape[1], x.shape[0]), False, _lib.INK_AUTO) for x in d]
    ruled = [r._replace(rule_length=ops.rule_length(x.shape[1], x.shape[0])) for r, x in zip(plain, d)]

    if args.profile:
        from torch.profiler import ProfilerActivity, profile
        for _ in range(5):
            ops.find_blocks(ruled)
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(args.iters):
                ops.find_blocks(ruled)
            torch.cuda.synchronize()
        us = {}
        for e in prof.key_averages():
            t = getattr(e, "device_time_total", None) or getattr(e, "cuda_time_total", 0)
            if t:
                us[e.key] = us.get(e.key, 0.0) + t
        rule = {k: v for k, v in us.items() if re.search(r"rule_\w+_kernel", k)}
        kernels = {k: v for k, v in us.items() if "kernel" in k}
        print(json.dumps(dict(card, what="profile", pages=len(pages), calls=args.iters,
                              rule_kernels_us_per_call={re.search(r"rule_\w+_kernel", k).group(0): round(v / args.iters, 2)
                                                        for k, v in rule.items()},
                              rule_us_per_call=round(sum(rule.values()) / args.iters, 2),
                              all_kernels_us_per_call=round(sum(kernels.values()) / args.iters, 2))), flush=True)
        return

    def events_ms(items):
        t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        t0.record()
        for _ in range(args.iters):
            ops.find_blocks(items)
        t1.record()
        t1.synchronize()
        return t0.elapsed_time(t1) / args.iters

    for items in (ruled, plain):
        for _ in range(5):
            ops.find_blocks(items)
    ms = {"rules": [], "no rules": []}
    for _ in range(args.passes):
        ms["rules"].append(events_ms(ruled))
        ms["no rules"].append(events_ms(plain))
    page = pipeline.TextPage(rules="auto")
    found = pipeline.find_blocks(pages, [[page] for _ in pages])
    plain_found = pipeline.find_blocks(pages, [[pipeline.TextPage()] for _ in pages])
    print(json.dumps(dict(card, what="layout", pages=len(pages), megapixels=sum(p.shape[0] * p.shape[1] for p in pages) / 1e6,
                          blocks=[len(f[0]["blocks"]) for f in found], blocks_without_rules=[len(f[0]["blocks"]) for f in plain_found],
                          rule_pixels=[f[0]["rule_pixels"] for f in found], rule_length=found[0][0]["rule_length"],
                          ms_per_call={k: round(float(np.median(v)), 4) for k, v in ms.items()},
                          ms_per_call_passes={k: [round(x, 4) for x in v] for k, v in ms.items()})), flush=True)

    sds = synth.make_checkpoints(0)
    m = []
    for key, cls in (("encoder", networks.TextContextEncoderV2), ("tspgan", networks.TSPGAN), ("sr", networks.TSPSRNet)):
        net = cls()
        net.load_state_dict(sds[key], strict=True)
        m.append(net.eval().to(dev))
    blocks = [f[0]["blocks"] for f in found]
    kw = dict(scale=args.scale, skip_invalid=True, to_host=True)
    arms = {"ruled pages": lambda: pipeline.restore_regions(*m, pages, [[page] for _ in pages], **kw),
            "found blocks": lambda: pipeline.restore_regions(*m, pages, blocks, **kw)}
    outs = {name: fn() for name, fn in arms.items()}          # warm-up of every shape
    times = {name: [] for name in arms}
    for _ in range(args.passes):
        for name, fn in arms.items():
            torch.cuda.synchronize()
            t = time.perf_counter()
            outs[name] = fn()
            times[name].append(time.perf_counter() - t)
    for a, b in zip(outs["ruled pages"], outs["found blocks"]):
        assert np.array_equal(a["image"], b["image"]), "the arms differ"
    n_lines = sum(len(e["lines"]) for f in outs["ruled pages"] for p in f["regions"] for e in p.get("regions", []) if "lines" in e)
    for name, ts in times.items():
        med = float(np.median(ts))
        print(json.dumps(dict(card, what=f"restore_regions with {name}", pages=len(pages), lines=n_lines, scale=args.scale,
                              pages_per_s=round(len(pages) / med, 3), seconds=[round(t, 4) for t in ts])), flush=True)


if __name__ == "__main__":
    main()
