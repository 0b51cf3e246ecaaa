"""Reversed panels (DESIGN.md section 7b, "Reversed panels"): the layout with and without panels="auto", restore_regions with
panel pages, and how many drawn reversed lines are restored.

    MN_MODULE_GRAPHS=0 python tools/bench_panels.py [--passes 4] [--iters 100] [--scale 2] [--profile]

The pages are four seeded 1600 x 1200 pages drawn with cv2.putText, each a dark headline banner with one or two white lines,
two or three columns of dark lines, a rule-less table whose header row is dark cells with white words, and a dark sidebar of
white lines.  Prints one JSON line each for:
  - layout: ops.find_blocks on the uploaded pages with and without panels, timed with CUDA events over --iters calls per
    arm, the median of --passes passes, the arms' order swapped pass by pass (ABBA);
  - restore_regions with TextPage(panels="auto") against the same call given the found blocks, host uint8 in and out,
    pages/s; the arms' order is swapped pass by pass, and they must give the same bytes;
  - the drawn reversed lines restored (a restored line's centre inside the drawn line), with panels and without.
With --profile, instead: torch.profiler over --iters layout calls with panels, the device time of panel_test_kernel and
panel_paint_kernel per call.  Every line carries the card's name and power limit, read in the same run.  Not part of the
product path.
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

H, W = 1200, 1600
FONT = cv2.FONT_HERSHEY_SIMPLEX
WORDS = "the of and to in is that for it as was with be by on not he this are or his from at which".split()


def _line(rng, n):
    return " ".join(str(w) for w in rng.choice(WORDS, n))


def _put(img, s, x, y, scale, grey, thick):
    """Draws s with its baseline at y; returns the drawn line's rectangle."""
    (tw, th), base = cv2.getTextSize(s, FONT, scale, thick)
    cv2.putText(img, s, (x, y), FONT, scale, (grey,) * 3, thick, cv2.LINE_AA)
    return x, y - th, x + tw, y + base


def make_pages(seed=0):
    """Four pages: (image, [the drawn reversed lines' rectangles])."""
    rng = np.random.default_rng(seed)
    pages = []
    for p in range(4):
        img = np.full((H, W, 3), int(rng.integers(236, 250)), np.uint8)
        rev = []
        fill = lambda: int(rng.integers(15, 70))
        img[40:40 + 60 * (1 + p % 2) + 30, 40:W - 40] = fill()          # the headline banner
        for k in range(1 + p % 2):
            rev.append(_put(img, _line(rng, 5).upper(), 70, 100 + 60 * k, 1.4, 250, 3))
        n_cols = 2 + p % 2
        cw = (W - 80 - 380) // n_cols
        for c in range(n_cols):                                          # columns of dark lines
            for k in range(18):
                _put(img, _line(rng, 4), 40 + c * cw, 260 + 32 * k, 0.7, 20, 1)
        ty = 880                                                         # the table: a dark header row, rule-less body
        for c in range(4):
            x = 40 + c * 270
            img[ty:ty + 44, x:x + 260] = fill()
            rev.append(_put(img, "HEAD %d" % c, x + 20, ty + 31, 0.8, 250, 2))
            for r in range(5):
                _put(img, _line(rng, 2), x + 20, ty + 80 + 36 * r, 0.7, 20, 1)
        img[240:820, W - 360:W - 40] = fill()                           # the sidebar
        for k in range(10):
            rev.append(_put(img, _line(rng, 3), W - 340, 290 + 50 * k, 0.8, 250, 2))
        pages.append((img, rev))
    return pages


def _card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True,
                       text=True)
    name, _, power = q.stdout.strip().partition(", ")
    return {"gpu": name or torch.cuda.get_device_name(0), "power_limit": power or None}


def _restored(out, drawn):
    """The drawn lines with a restored line's centre inside them."""
    centres = []

    def walk(entries):
        for e in entries:
            if isinstance(e, dict):
                centres.extend(((q[0] + q[2]) / 2, (q[1] + q[3]) / 2) for q in e.get("lines", []) if isinstance(q, tuple))
                walk(e.get("regions", []))
    walk(out["regions"])
    return sum(any(x0 <= cx < x1 and y0 <= cy < y1 for cx, cy in centres) for x0, y0, x1, y1 in drawn)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--passes", type=int, default=4)
    ap.add_argument("--iters", type=int, default=100)
    ap.add_argument("--scale", type=int, default=2)
    ap.add_argument("--profile", action="store_true")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_panels.py needs a CUDA device")
    from marconet_b200 import _lib, ops, pipeline
    from marconet_b200.models import networks
    from marconet_b200.testing import synth
    dev = torch.device("cuda:0")
    card = _card()
    drawn = make_pages()
    pages = [p for p, _ in drawn]
    d = [torch.from_numpy(p).to(dev) for p in pages]
    plain = [ops.PageItem(x, (0, 0, x.shape[1], x.shape[0]), False, _lib.INK_AUTO) for x in d]
    panels = [r._replace(panel_size=0) for r in plain]

    if args.profile:
        from torch.profiler import ProfilerActivity, profile
        for _ in range(5):
            ops.find_blocks(panels)
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(args.iters):
                ops.find_blocks(panels)
            torch.cuda.synchronize()
        us = {}
        for e in prof.key_averages():
            t = getattr(e, "device_time_total", None) or getattr(e, "cuda_time_total", 0)
            if t:
                us[e.key] = us.get(e.key, 0.0) + t
        pick = lambda s: round(sum(v for k, v in us.items() if s in k) / args.iters, 2)
        print(json.dumps(dict(card, what="profile", pages=len(pages), calls=args.iters,
                              us_per_call=dict(panel_test_kernel=pick("panel_test_kernel"),
                                               panel_paint_kernel=pick("panel_paint_kernel"),
                                               page_size_kernel=pick("page_size_kernel"), all_kernels=pick("kernel")))),
              flush=True)
        return

    def events_ms(items):
        t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        t0.record()
        for _ in range(args.iters):
            ops.find_blocks(items)
        t1.record()
        t1.synchronize()
        return t0.elapsed_time(t1) / args.iters

    for items in (panels, plain):
        for _ in range(5):
            ops.find_blocks(items)
    ms = {"panels": [], "none": []}
    for k in range(args.passes):                         # the arms' order swapped pass by pass: ABBA ...
        for name, items in (("panels", panels), ("none", plain))[::1 if k % 2 == 0 else -1]:
            ms[name].append(events_ms(items))
    tps = [[pipeline.TextPage(panels="auto")] for _ in pages]
    found = pipeline.find_blocks(pages, tps)
    print(json.dumps(dict(card, what="layout", pages=len(pages), megapixels=sum(p.shape[0] * p.shape[1] for p in pages) / 1e6,
                          blocks=[len(f[0]["blocks"]) for f in found], panels=[len(f[0]["panels"]) for f in found],
                          light_blocks=[sum(b.polarity == "light" for b in f[0]["blocks"]) for f in found],
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
    arms = {"panel pages": lambda: pipeline.restore_regions(*m, pages, tps, **kw),
            "found blocks": lambda: pipeline.restore_regions(*m, pages, blocks, **kw)}
    outs = {name: fn() for name, fn in arms.items()}          # warm-up of every shape
    times = {name: [] for name in arms}
    for k in range(args.passes):
        for name, fn in list(arms.items())[::1 if k % 2 == 0 else -1]:
            torch.cuda.synchronize()
            t = time.perf_counter()
            outs[name] = fn()
            times[name].append(time.perf_counter() - t)
    for a, b in zip(outs["panel pages"], outs["found blocks"]):
        assert np.array_equal(a["image"], b["image"]), "the arms differ"
    n_lines = sum(len(e["lines"]) for f in outs["found blocks"] for e in f["regions"] if "lines" in e)
    for name, ts in times.items():
        med = float(np.median(ts))
        print(json.dumps(dict(card, what=f"restore_regions with {name}", pages=len(pages), lines=n_lines, scale=args.scale,
                              pages_per_s=round(len(pages) / med, 3), seconds=[round(t, 4) for t in ts])), flush=True)
    without = pipeline.restore_regions(*m, pages, [[pipeline.TextPage()] for _ in pages], **kw)
    print(json.dumps(dict(card, what="drawn reversed lines restored", pages=len(pages), drawn=[len(r) for _, r in drawn],
                          panels=[_restored(o, r) for o, (_, r) in zip(outs["panel pages"], drawn)],
                          none=[_restored(o, r) for o, (_, r) in zip(without, drawn)])), flush=True)


if __name__ == "__main__":
    main()
