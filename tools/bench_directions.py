"""Mixed directions (DESIGN.md section 7b, "Mixed directions"): the layout with and without block_direction="auto",
restore_regions with mixed pages, and how many drawn blocks get their drawn direction.

    MN_MODULE_GRAPHS=0 python tools/bench_directions.py [--passes 3] [--iters 100] [--scale 2] [--profile]

The pages are four seeded 1600 x 1200 pages of square pseudo-glyphs (S x S cells of seeded strokes, some split into left and
right or top and bottom parts) set on grids: two vertical pages, each a horizontal headline over blocks of vertical columns
with a horizontal caption under them, and two horizontal pages, each with columns of horizontal lines beside a vertical
sidebar.  Prints one JSON line each for:
  - layout: ops.find_blocks on the uploaded pages with and without block_direction="auto", timed with CUDA events over
    --iters calls per arm, the median of --passes passes, the arms alternating pass by pass;
  - restore_regions with TextPage(block_direction="auto") against the same call given the found blocks, host uint8 in and
    out, pages/s; the arms alternate pass by pass and must give the same bytes;
  - the drawn blocks whose found block has the drawn direction, with "auto" and without.
With --profile, instead: torch.profiler over --iters layout calls with "auto", the device time of page_direction_kernel per
call.  Every line carries the card's name and power limit, read in the same run.  Not part of the product path.
"""
import argparse
import json
import os
import subprocess
import sys
import time

os.environ.setdefault("MN_MODULE_GRAPHS", "0")

import numpy as np  # noqa: E402
import torch  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

H, W = 1200, 1600


def glyph(rng, s):
    """An s x s pseudo-glyph: stems on both sides and one or two strokes across, whole or split in two."""
    t, gap = max(2, s // 10), max(2, s // 8)

    def part(h, w):
        m = np.zeros((h, w), bool)
        m[:, :t] = m[:, w - t:] = m[:t] = True
        for y in rng.integers(t, h - t, int(rng.integers(1, 3))):
            m[y:y + t] = True
        return m
    kind, a = int(rng.integers(0, 4)), (s - gap) // 2
    m = np.zeros((s, s), bool)
    if kind == 2:
        m[:, :a], m[:, s - a:] = part(s, a), part(s, a)
    elif kind == 3:
        m[:a], m[s - a:] = part(a, s), part(a, s)
    else:
        m[:] = part(s, s)
    return m


def text(m, rng, x, y, lines, chars, vertical, s=24, track=3, lead=10):
    """Glyphs on a grid from (x, y); returns the ink rectangle."""
    x1 = y1 = 0
    for i in range(lines):
        for j in range(chars):
            gx, gy = (x + i * (s + lead), y + j * (s + track)) if vertical else (x + j * (s + track), y + i * (s + lead))
            m[gy:gy + s, gx:gx + s] |= glyph(rng, s)
            x1, y1 = max(x1, gx + s), max(y1, gy + s)
    return x, y, x1, y1


def make_pages(seed=0):
    """Four pages: (image, page direction, [(drawn rectangle, drawn direction)])."""
    rng = np.random.default_rng(seed)
    pages = []
    for p in range(4):
        m = np.zeros((H, W), bool)
        drawn = []
        if p % 2 == 0:                                   # vertical: headline, blocks of columns, caption
            drawn.append((text(m, rng, 60, 40, 1, 25, False, s=56, track=2), "horizontal"))
            x = W - 60
            for cols in (6, 5, 7, 4)[:3 + p // 2]:
                x -= cols * 24 + (cols - 1) * 10
                drawn.append((text(m, rng, x, 150, cols, 30, True), "vertical"))
                x -= 50
            drawn.append((text(m, rng, 300, 1050, 1, 40, False, s=22, track=2), "horizontal"))
            direction = "vertical"
        else:                                            # horizontal: columns of lines and a vertical sidebar
            drawn.append((text(m, rng, 60, 50, 1, 30, False, s=36, track=2), "horizontal"))
            for c in range(2 + p // 2):
                drawn.append((text(m, rng, 60 + c * 420, 150, 20, 14, False), "horizontal"))
            drawn.append((text(m, rng, W - 60 - 4 * 34 + 10, 150, 4, 36, True), "vertical"))
            direction = "horizontal"
        paper = np.clip(rng.integers(215, 246, 3) + rng.integers(-12, 13, (H, W, 1)), 0, 255).astype(np.uint8)
        pages.append((np.where(m[..., None], np.uint8(20), paper), direction, drawn))
    return pages


def _card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True,
                       text=True)
    name, _, power = q.stdout.strip().partition(", ")
    return {"gpu": name or torch.cuda.get_device_name(0), "power_limit": power or None}


def _overlap(a, b):
    return max(0, min(a[2], b[2]) - max(a[0], b[0])) * max(0, min(a[3], b[3]) - max(a[1], b[1]))


def _right(found, drawn):
    """The drawn blocks whose most overlapping found block has the drawn direction."""
    n = 0
    for rect, d in drawn:
        best = max(found, key=lambda b: _overlap(b.rect, rect), default=None)
        n += best is not None and _overlap(best.rect, rect) > 0 and best.direction == d
    return n


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--passes", type=int, default=3)
    ap.add_argument("--iters", type=int, default=100)
    ap.add_argument("--scale", type=int, default=2)
    ap.add_argument("--profile", action="store_true")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_directions.py needs a CUDA device")
    from marconet_b200 import _lib, ops, pipeline
    from marconet_b200.models import networks
    from marconet_b200.testing import synth
    dev = torch.device("cuda:0")
    card = _card()
    drawn = make_pages()
    pages = [p for p, _, _ in drawn]
    d = [torch.from_numpy(p).to(dev) for p in pages]
    plain = [ops.PageItem(x, (0, 0, x.shape[1], x.shape[0]), dr == "vertical", _lib.INK_AUTO) for x, (_, dr, _) in zip(d, drawn)]
    auto = [r._replace(directions=True) for r in plain]

    if args.profile:
        from torch.profiler import ProfilerActivity, profile
        for _ in range(5):
            ops.find_blocks(auto)
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(args.iters):
                ops.find_blocks(auto)
            torch.cuda.synchronize()
        us = {}
        for e in prof.key_averages():
            t = getattr(e, "device_time_total", None) or getattr(e, "cuda_time_total", 0)
            if t:
                us[e.key] = us.get(e.key, 0.0) + t
        pick = lambda s: round(sum(v for k, v in us.items() if s in k) / args.iters, 2)
        print(json.dumps(dict(card, what="profile", pages=len(pages), calls=args.iters,
                              us_per_call=dict(page_direction_kernel=pick("page_direction_kernel"),
                                               page_blocks_kernel=pick("page_blocks_kernel"), all_kernels=pick("kernel")))),
              flush=True)
        return

    def events_ms(items):
        t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        t0.record()
        for _ in range(args.iters):
            ops.find_blocks(items)
        t1.record()
        t1.synchronize()
        return t0.elapsed_time(t1) / args.iters

    for items in (auto, plain):
        for _ in range(5):
            ops.find_blocks(items)
    ms = {"auto": [], "none": []}
    for _ in range(args.passes):
        ms["auto"].append(events_ms(auto))
        ms["none"].append(events_ms(plain))
    tps = [[pipeline.TextPage(direction=dr, block_direction="auto")] for _, dr, _ in drawn]
    found = pipeline.find_blocks(pages, tps)
    plain_found = pipeline.find_blocks(pages, [[pipeline.TextPage(direction=dr)] for _, dr, _ in drawn])
    print(json.dumps(dict(card, what="layout", pages=len(pages), megapixels=sum(p.shape[0] * p.shape[1] for p in pages) / 1e6,
                          blocks=[len(f[0]["blocks"]) for f in found], undecided=[len(f[0]["undecided"]) for f in found],
                          ms_per_call={k: round(float(np.median(v)), 4) for k, v in ms.items()},
                          ms_per_call_passes={k: [round(x, 4) for x in v] for k, v in ms.items()})), flush=True)
    right = {"auto": [_right(f[0]["blocks"], dr) for f, (_, _, dr) in zip(found, drawn)],
             "none": [_right(f[0]["blocks"], dr) for f, (_, _, dr) in zip(plain_found, drawn)]}
    print(json.dumps(dict(card, what="drawn blocks with their drawn direction", pages=len(pages),
                          drawn=[len(dr) for _, _, dr in drawn], right=right)), flush=True)

    sds = synth.make_checkpoints(0)
    m = []
    for key, cls in (("encoder", networks.TextContextEncoderV2), ("tspgan", networks.TSPGAN), ("sr", networks.TSPSRNet)):
        net = cls()
        net.load_state_dict(sds[key], strict=True)
        m.append(net.eval().to(dev))
    blocks = [f[0]["blocks"] for f in found]
    kw = dict(scale=args.scale, skip_invalid=True, to_host=True)
    arms = {"mixed pages": lambda: pipeline.restore_regions(*m, pages, tps, **kw),
            "found blocks": lambda: pipeline.restore_regions(*m, pages, blocks, **kw)}
    outs = {name: fn() for name, fn in arms.items()}          # warm-up of every shape
    times = {name: [] for name in arms}
    for _ in range(args.passes):
        for name, fn in arms.items():
            torch.cuda.synchronize()
            t = time.perf_counter()
            outs[name] = fn()
            times[name].append(time.perf_counter() - t)
    for a, b in zip(outs["mixed pages"], outs["found blocks"]):
        assert np.array_equal(a["image"], b["image"]), "the arms differ"
    n_lines = sum(len(e["lines"]) for f in outs["found blocks"] for e in f["regions"] if "lines" in e)
    for name, ts in times.items():
        med = float(np.median(ts))
        print(json.dumps(dict(card, what=f"restore_regions with {name}", pages=len(pages), lines=n_lines, scale=args.scale,
                              pages_per_s=round(len(pages) / med, 3), seconds=[round(t, 4) for t in ts])), flush=True)


if __name__ == "__main__":
    main()
