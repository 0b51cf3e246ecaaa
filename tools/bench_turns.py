"""Page turns (DESIGN.md section 7b, "Page turns"): the layout of turned pages with turn="auto" against the plain layout of their
upright copies, and restore_regions of the turned pages against the same call given the found blocks.

    MN_MODULE_GRAPHS=0 python tools/bench_turns.py [--passes 4] [--iters 20] [--scale 2]

The pages are four seeded 1600 x 1200 pages: a cv2.putText heading over two columns of pseudo-glyph paragraphs drawn as the host
tests draw them (indented first lines, ragged right sides, short last lines), turned 0, 90, 180 and 270 degrees with np.rot90.
Prints one JSON line each for:
  - layout: pipeline.find_blocks' device path (_find_pages, the uploaded pages, its synchronisations included) with
    TextPage(turn="auto") on the turned pages and TextPage() on their upright copies, ms per call of the four pages timed with
    CUDA events over --iters calls per arm, the median of --passes passes, the arms' order swapped pass by pass; with the
    turns found and whether every page's blocks equal its upright copy's;
  - restore_regions of the turned pages with TextPage(turn="auto") and with the found blocks given, host uint8 in and out,
    pages per second (median of --passes alternated passes), and whether the two give the same bytes.
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

H, W = 1200, 1600
FONT = cv2.FONT_HERSHEY_SIMPLEX
WORDS = "the of and to in is that for it as was with be by on not he this are or his from at which".split()


def make_page(rng):
    """An upright page: a cv2.putText heading over two columns of pseudo-glyph paragraphs (tests/test_mixed_pages.py's glyphs),
    first lines indented by two glyphs, lines ragged on the right and last lines short."""
    from test_mixed_pages import INK, LEAD, S, TRACK, image, text
    m = np.zeros((H, W), bool)
    for c in range(2):
        x, y = 80 + c * 760, 150
        while y < H - 3 * (S + LEAD):
            n = int(rng.integers(3, 8))
            for k in range(n):
                if y >= H - 2 * (S + LEAD):
                    break
                indent = 2 if k == 0 else 0
                chars = int(rng.integers(6, 11)) if k == n - 1 else int(rng.integers(22, 25)) - indent
                text(m, rng, x + indent * (S + TRACK), y, 1, chars)
                y += S + LEAD
            y += S
    img = image(m)
    cv2.putText(img, "PAGE TURNS " + " ".join(rng.choice(WORDS, 3)).upper(), (80, 90), FONT, 1.6, (INK,) * 3, 3, cv2.LINE_AA)
    return img


def _card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True,
                       text=True)
    name, _, power = q.stdout.strip().partition(", ")
    return {"gpu": name or torch.cuda.get_device_name(0), "power_limit": power or None}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--passes", type=int, default=4)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--scale", type=int, default=2)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_turns.py needs a CUDA device")
    from marconet_b200 import pipeline
    from marconet_b200.models import networks
    from marconet_b200.testing import synth
    dev = torch.device("cuda:0")
    card = _card()
    rng = np.random.default_rng(0)
    upright = [make_page(rng) for _ in range(4)]
    turned = [np.ascontiguousarray(np.rot90(p, k)) for k, p in enumerate(upright)]
    du = dict(enumerate(torch.from_numpy(p).to(dev) for p in upright))
    dt = dict(enumerate(torch.from_numpy(p).to(dev) for p in turned))

    def items(imgs, pg):
        return [(k, pg, (0, 0, im.shape[1], im.shape[0])) for k, im in imgs.items()]
    arms = {"turn_auto": (dt, items(dt, pipeline.TextPage(turn="auto"))), "upright_plain": (du, items(du, pipeline.TextPage()))}

    def events_ms(imgs, its):
        t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        t0.record()
        for _ in range(args.iters):
            pipeline._find_pages(imgs, its)
        t1.record()
        t1.synchronize()
        return t0.elapsed_time(t1) / args.iters

    for imgs, its in arms.values():
        for _ in range(3):
            pipeline._find_pages(imgs, its)
    ms = {k: [] for k in arms}
    for p in range(args.passes):
        for name in list(arms)[::1 if p % 2 == 0 else -1]:
            ms[name].append(events_ms(*arms[name]))
    got = pipeline._find_pages(dt, arms["turn_auto"][1])[0]
    ref = pipeline._find_pages(du, arms["upright_plain"][1])[0]
    same = all([b.window for b in g["blocks"]] == [tuple(b.rect) for b in r["blocks"]] if g["turn"] else
               [b.rect for b in g["blocks"]] == [b.rect for b in r["blocks"]] for g, r in zip(got, ref))
    print(json.dumps(dict(card, what="layout", pages=4, size=[W, H], turns=[g["turn"] for g in got],
                          turn_votes=[list(g["turn_votes"]) for g in got], blocks=[len(g["blocks"]) for g in got],
                          blocks_equal_upright=same, ms_per_call={k: round(float(np.median(v)), 4) for k, v in ms.items()},
                          ms_per_call_passes={k: [round(x, 4) for x in v] for k, v in ms.items()})), flush=True)

    sds = synth.make_checkpoints(0)
    m = []
    for key, cls in (("encoder", networks.TextContextEncoderV2), ("tspgan", networks.TSPGAN), ("sr", networks.TSPSRNet)):
        net = cls()
        net.load_state_dict(sds[key], strict=True)
        m.append(net.eval().to(dev))
    found = pipeline.find_blocks(turned, [[pipeline.TextPage(turn="auto")] for _ in turned])
    calls = {"turn_auto": [[pipeline.TextPage(turn="auto")] for _ in turned], "found_blocks": [f[0]["blocks"] for f in found]}
    kw = dict(scale=args.scale, skip_invalid=True, to_host=True)
    outs = {k: pipeline.restore_regions(*m, turned, regs, **kw) for k, regs in calls.items()}     # warm-up of every shape
    ts = {k: [] for k in calls}
    for p in range(args.passes):
        for name in list(calls)[::1 if p % 2 == 0 else -1]:
            torch.cuda.synchronize()
            t = time.perf_counter()
            outs[name] = pipeline.restore_regions(*m, turned, calls[name], **kw)
            ts[name].append(time.perf_counter() - t)
    same = all(np.array_equal(a["image"], b["image"]) for a, b in zip(outs["turn_auto"], outs["found_blocks"]))
    print(json.dumps(dict(card, what="restore_regions", pages=4, scale=args.scale, same_bytes=same,
                          pages_per_second={k: round(4 / float(np.median(v)), 3) for k, v in ts.items()},
                          seconds={k: [round(x, 4) for x in v] for k, v in ts.items()})), flush=True)


if __name__ == "__main__":
    main()
