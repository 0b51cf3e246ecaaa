"""Seal centre lines (DESIGN.md section 7b, "Seal centre lines"): the line kernel's device time, the layout with and without
seal_lines="auto", restore_regions of the pages and how many drawn centre lines it restored.

    MN_MODULE_GRAPHS=0 python tools/bench_seal_lines.py [--passes 4] [--iters 50] [--scale 2]

The pages are four seeded 1654 x 2339 pages (A4 at 200 dpi) drawn with cv2.putText: paragraphs of dark lines, a company seal
(round, a star and one centre line) and an oval invoice seal (a number line across its centre and a title line under it),
red or blue, turned by hand, drawn as the host tests draw them.  Prints one JSON line each for:
  - profile: torch.profiler over --iters layout calls with seal_lines, the device time of the line kernel per call;
  - layout: ops.find_blocks on the uploaded pages with seals and with seals and seal_lines, timed with CUDA events over --iters
    calls per arm, the median of --passes passes, the arms' order swapped pass by pass;
  - restore_regions with TextPage(seals="auto", seal_lines="auto"), host uint8 in and out, pages per second, and the drawn
    centre lines restored: a found line region whose centre lies inside a drawn line's box.
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
sys.path.insert(0, os.path.join(ROOT, "tests"))

H, W = 2339, 1654
FONT = cv2.FONT_HERSHEY_SIMPLEX
WORDS = "the of and to in is that for it as was with be by on not he this are or his from at which".split()


def make_pages(seed=0):
    """(pages, drawn line boxes per page): each drawn line's pixel box (x0, y0, x1, y1)."""
    from test_seal_lines import inner_line
    from test_seal_pages import BLUE, RED, stamp
    rng = np.random.default_rng(seed)
    pages, drawn = [], []
    for p in range(4):
        img = np.full((H, W, 3), int(rng.integers(236, 250)), np.uint8)
        for k in range(60):
            cv2.putText(img, " ".join(rng.choice(WORDS, 9)), (100, 150 + 34 * k), FONT, 1.0, (20, 20, 20), 2, cv2.LINE_AA)
        boxes = []
        for (cx, cy), oval in (((1200, 700 + 200 * p), False), ((1250, 1900), True)):
            r = int(rng.integers(170, 230))
            rx, ry = (int(r * 1.33), r) if oval else (r, r)
            colour, rot = RED if rng.integers(2) else BLUE, float(rng.uniform(-20, 20))
            stamp(img, cx, cy, rx, ry, colour, rot=rot, star=not oval)
            lines = ((0.0, 0.17, "1234567890"), (0.38, 0.15, "ABCDEF")) if oval else ((0.45, 0.17, "ABCDE"),)
            for dy, gh, text in lines:
                m = inner_line(H, W, cx, cy, text, dy * ry, gh * ry, rot)
                img[m] = colour
                ys, xs = np.nonzero(m)
                boxes.append((xs.min(), ys.min(), xs.max() + 1, ys.max() + 1))
        pages.append(img)
        drawn.append(boxes)
    return pages, drawn


def _card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True,
                       text=True)
    name, _, power = q.stdout.strip().partition(", ")
    return {"gpu": name or torch.cuda.get_device_name(0), "power_limit": power or None}


def _centre(reg):
    if len(reg) == 4:                                           # a rectangle
        return (reg[0] + reg[2]) / 2, (reg[1] + reg[3]) / 2
    (ax, ay), (bx, by), (cx, cy) = reg                       # tl, tr, bl: the centre is the middle of tr and bl
    return (bx + cx) / 2, (by + cy) / 2


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--passes", type=int, default=4)
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--scale", type=int, default=2)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_seal_lines.py needs a CUDA device")
    from marconet_b200 import _lib, ops, pipeline
    from marconet_b200.models import networks
    from marconet_b200.testing import synth
    dev = torch.device("cuda:0")
    card = _card()
    pages, drawn = make_pages()
    d = [torch.from_numpy(p).to(dev) for p in pages]
    sealed = [ops.PageItem(x, (0, 0, W, H), False, _lib.INK_AUTO, seal_size=pipeline.seal_size(W, H)) for x in d]
    lined = [r._replace(seal_lines=True) for r in sealed]

    from torch.profiler import ProfilerActivity, profile
    for _ in range(5):
        ops.find_blocks(lined)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(args.iters):
            ops.find_blocks(lined)
        torch.cuda.synchronize()
    us = 0.0
    for e in prof.key_averages():
        t = getattr(e, "device_time_total", None) or getattr(e, "cuda_time_total", 0)
        if t and "centre_lines_kernel" in e.key:
            us += t
    print(json.dumps(dict(card, what="profile", pages=len(pages), calls=args.iters,
                          centre_lines_kernel_us_per_call=round(us / args.iters, 2))), flush=True)

    def events_ms(items):
        t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        t0.record()
        for _ in range(args.iters):
            ops.find_blocks(items)
        t1.record()
        t1.synchronize()
        return t0.elapsed_time(t1) / args.iters

    for items in (lined, sealed):
        for _ in range(3):
            ops.find_blocks(items)
    ms = {"seal_lines": [], "seals": []}
    for k in range(args.passes):
        for name, items in (("seal_lines", lined), ("seals", sealed))[::1 if k % 2 == 0 else -1]:
            ms[name].append(events_ms(items))
    tps = [[pipeline.TextPage(seals="auto", seal_lines="auto")] for _ in pages]
    found = pipeline.find_blocks(pages, tps)
    print(json.dumps(dict(card, what="layout", pages=len(pages), megapixels=sum(p.shape[0] * p.shape[1] for p in pages) / 1e6,
                          seals=[len(f[0]["seals"]) for f in found],
                          lines=[sum(len(s["lines"]) for s in f[0]["seals"]) for f in found],
                          turns=[[s["turn"] for s in f[0]["seals"]] for f in found],
                          ms_per_call={k: round(float(np.median(v)), 4) for k, v in ms.items()},
                          ms_per_call_passes={k: [round(x, 4) for x in v] for k, v in ms.items()})), flush=True)

    sds = synth.make_checkpoints(0)
    m = []
    for key, cls in (("encoder", networks.TextContextEncoderV2), ("tspgan", networks.TSPGAN), ("sr", networks.TSPSRNet)):
        net = cls()
        net.load_state_dict(sds[key], strict=True)
        m.append(net.eval().to(dev))
    kw = dict(scale=args.scale, skip_invalid=True, to_host=True)
    pipeline.restore_regions(*m, pages, tps, **kw)                  # warm-up of every shape
    ts = []
    for _ in range(args.passes):
        torch.cuda.synchronize()
        t = time.perf_counter()
        out = pipeline.restore_regions(*m, pages, tps, **kw)
        ts.append(time.perf_counter() - t)
    med = float(np.median(ts))
    hit = 0
    for o, f, boxes in zip(out, found, drawn):                     # a found line region whose restored entry has no error
        regs = [ln["region"] for s in f[0]["seals"] for ln in s["lines"] if ln["region"] is not None]
        regs = [r for r, e in zip(regs, o["regions"][0].get("seal_line_regions", [])) if "error" not in e]
        for x0, y0, x1, y1 in boxes:
            hit += any(x0 <= c[0] < x1 and y0 <= c[1] < y1 for c in map(_centre, regs))
    print(json.dumps(dict(card, what="restore_regions with seal_lines pages", pages=len(pages), scale=args.scale,
                          seal_line_regions=[len(o["regions"][0].get("seal_line_regions", [])) for o in out],
                          drawn_lines=sum(len(b) for b in drawn), drawn_lines_restored=hit,
                          pages_per_second=round(len(pages) / med, 3), seconds=[round(t, 4) for t in ts])), flush=True)


if __name__ == "__main__":
    main()
