"""Figures (DESIGN.md section 7b, "Figures"): the layout with and without figures, the figure kernels alone, restore_regions
with figure pages, and the restored lines that meet a drawn figure.

    MN_MODULE_GRAPHS=0 python tools/bench_figures.py [--pages 4] [--passes 3] [--iters 100] [--scale 2] [--profile]

The pages are seeded 1600 x 1200 pages: a heading over two or three columns of lines at a 33-pixel pitch (capitals drawn with
cv2.putText, Hershey DUPLEX, on a light, slightly noisy background), a smooth greyscale photo in place of some lines of one
column and a line chart (two axes and a polyline) in another.  Prints one JSON line each for:
  - layout: ops.find_blocks on the uploaded pages with and without figures, timed with CUDA events over --iters calls per
    arm, the arms alternating pass by pass;
  - restore_regions with TextPage(figures="auto") against the same call given the found blocks, host uint8 in and out,
    pages/s; the arms alternate pass by pass and must give the same bytes;
  - the restored lines whose rectangle meets a drawn photo or chart, with figures and without.
With --profile, instead: torch.profiler over --iters figure layout calls, the device time of the figure launch and of the
text-size kernel that selects the figures, per call, against the same calls without figures.  Every line carries the card's
name and power limit, read in the same run.  Not part of the product path.
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

WORDS = "THE QUICK BROWN FOX JUMPS OVER A LAZY DOG PACK MY BOX WITH FIVE DOZEN JUGS 0123456789".split()
FONT = cv2.FONT_HERSHEY_DUPLEX


def make_pages(n_pages, seed=0):
    """n_pages 1600 x 1200 pages: (image, the drawn pictures' rectangles)."""
    rng = np.random.default_rng(seed)
    H, W, pitch, top, gutter = 1200, 1600, 33, 130, 60
    ink = (20, 20, 20)
    pages = []
    for p in range(n_pages):
        page = np.clip(rng.integers(215, 246, 3) + rng.integers(-12, 13, (H, W, 1)), 0, 255).astype(np.uint8)
        cv2.putText(page, "A HEADING OVER THE COLUMNS", (40, 70), FONT, 1.0, ink, 2, cv2.LINE_AA)
        n_cols = 2 + p % 2
        cw = (W - 80 - gutter * (n_cols - 1)) // n_cols
        a, b = int(rng.integers(2, 10)), int(rng.integers(14, 22))       # the photo's lines in column 0
        c, d = int(rng.integers(4, 14)), int(rng.integers(20, 28))       # the chart's lines in the last column
        pics = []
        for col in range(n_cols):
            x0 = 40 + col * (cw + gutter)
            skip = range(a, b) if col == 0 else range(c, d) if col == n_cols - 1 else range(0)
            for k in range(30):
                if k in skip:
                    continue
                t = str(rng.choice(WORDS))
                while True:                              # the longest run of words that fits the column
                    longer = t + " " + str(rng.choice(WORDS))
                    if cv2.getTextSize(longer, FONT, 1.0, 2)[0][0] > cw:
                        break
                    t = longer
                cv2.putText(page, t, (x0, top + pitch * k), FONT, 1.0, ink, 2, cv2.LINE_AA)
            if col == 0 or col == n_cols - 1:
                y0, y1 = top + pitch * skip.start - 10, top + pitch * (skip.stop - 1)
                if col == 0:
                    f = cv2.GaussianBlur(rng.normal(0, 1, (y1 - y0, cw)), (0, 0), 12)
                    f = (f - f.min()) / (f.max() - f.min())
                    page[y0:y1, x0:x0 + cw] = (40 + 200 * f).astype(np.uint8)[..., None]
                else:
                    page[y0:y1, x0:x0 + cw] = 232
                    cv2.line(page, (x0 + 20, y0 + 10), (x0 + 20, y1 - 20), ink, 2)
                    cv2.line(page, (x0 + 20, y1 - 20), (x0 + cw - 10, y1 - 20), ink, 2)
                    pts = np.stack([np.linspace(x0 + 20, x0 + cw - 20, 12), y1 - 40 - rng.uniform(0, y1 - y0 - 100, 12)], 1)
                    cv2.polylines(page, [pts.astype(np.int32)], False, ink, 2)
                pics.append((x0, y0, x0 + cw, y1))
        pages.append((page, pics))
    return pages


def _card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True,
                       text=True)
    name, _, power = q.stdout.strip().partition(", ")
    return {"gpu": name or torch.cuda.get_device_name(0), "power_limit": power or None}


def _meets(a, b):
    return a[0] < b[2] and b[0] < a[2] and a[1] < b[3] and b[1] < a[3]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--pages", type=int, default=4)
    ap.add_argument("--passes", type=int, default=3)
    ap.add_argument("--iters", type=int, default=100)
    ap.add_argument("--scale", type=int, default=2)
    ap.add_argument("--profile", action="store_true")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_figures.py needs a CUDA device")
    from marconet_b200 import _lib, ops, pipeline
    from marconet_b200.models import networks
    from marconet_b200.testing import synth
    dev = torch.device("cuda:0")
    card = _card()
    drawn = make_pages(args.pages)
    pages = [p for p, _ in drawn]
    d = [torch.from_numpy(p).to(dev) for p in pages]
    plain = [ops.PageItem(x, (0, 0, x.shape[1], x.shape[0]), False, _lib.INK_AUTO) for x in d]
    figured = [r._replace(figure_size=0) for r in plain]

    if args.profile:
        from torch.profiler import ProfilerActivity, profile
        out = {}
        for name, items in (("figures", figured), ("no figures", plain)):
            for _ in range(5):
                ops.find_blocks(items)
            torch.cuda.synchronize()
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                for _ in range(args.iters):
                    ops.find_blocks(items)
                torch.cuda.synchronize()
            us = {}
            for e in prof.key_averages():
                t = getattr(e, "device_time_total", None) or getattr(e, "cuda_time_total", 0)
                if t:
                    us[e.key] = us.get(e.key, 0.0) + t
            pick = lambda s: round(sum(v for k, v in us.items() if s in k) / args.iters, 2)
            out[name] = dict(figure_paint_kernel=pick("figure_paint_kernel"), page_size_kernel=pick("page_size_kernel"),
                             page_blocks_kernel=pick("page_blocks_kernel"), all_kernels=pick("kernel"))
        print(json.dumps(dict(card, what="profile", pages=len(pages), calls=args.iters, us_per_call=out)), flush=True)
        return

    def events_ms(items):
        t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        t0.record()
        for _ in range(args.iters):
            ops.find_blocks(items)
        t1.record()
        t1.synchronize()
        return t0.elapsed_time(t1) / args.iters

    for items in (figured, plain):
        for _ in range(5):
            ops.find_blocks(items)
    ms = {"figures": [], "no figures": []}
    for _ in range(args.passes):
        ms["figures"].append(events_ms(figured))
        ms["no figures"].append(events_ms(plain))
    page = pipeline.TextPage(figures="auto")
    found = pipeline.find_blocks(pages, [[page] for _ in pages])
    plain_found = pipeline.find_blocks(pages, [[pipeline.TextPage()] for _ in pages])
    print(json.dumps(dict(card, what="layout", pages=len(pages), megapixels=sum(p.shape[0] * p.shape[1] for p in pages) / 1e6,
                          blocks=[len(f[0]["blocks"]) for f in found], blocks_without_figures=[len(f[0]["blocks"]) for f in plain_found],
                          figures=[len(f[0]["figures"]) for f in found], figure_size=[f[0]["figure_size"] for f in found],
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
    arms = {"figure pages": lambda: pipeline.restore_regions(*m, pages, [[page] for _ in pages], **kw),
            "found blocks": lambda: pipeline.restore_regions(*m, pages, blocks, **kw)}
    outs = {name: fn() for name, fn in arms.items()}          # warm-up of every shape
    times = {name: [] for name in arms}
    for _ in range(args.passes):
        for name, fn in arms.items():
            torch.cuda.synchronize()
            t = time.perf_counter()
            outs[name] = fn()
            times[name].append(time.perf_counter() - t)
    for a, b in zip(outs["figure pages"], outs["found blocks"]):
        assert np.array_equal(a["image"], b["image"]), "the arms differ"

    def lines_in(res):
        return [tuple(r) for f in res for p in f["regions"] for e in p.get("regions", []) if "lines" in e for r in e["lines"]]
    without = pipeline.restore_regions(*m, pages, [[pipeline.TextPage()] for _ in pages], **kw)
    n_lines = len(lines_in(outs["figure pages"]))
    for name, ts in times.items():
        med = float(np.median(ts))
        print(json.dumps(dict(card, what=f"restore_regions with {name}", pages=len(pages), lines=n_lines, scale=args.scale,
                              pages_per_s=round(len(pages) / med, 3), seconds=[round(t, 4) for t in ts])), flush=True)
    inside = {}
    for name, res in (("figures", outs["figure pages"]), ("no figures", without)):
        per = [[r for r in lines_in([f]) if any(_meets(r, pic) for pic in pics)] for f, (_, pics) in zip(res, drawn)]
        inside[name] = [len(x) for x in per]
    print(json.dumps(dict(card, what="restored lines meeting a drawn figure", pages=len(pages), lines=inside,
                          total_lines={"figures": n_lines, "no figures": len(lines_in(without))})), flush=True)


if __name__ == "__main__":
    main()
