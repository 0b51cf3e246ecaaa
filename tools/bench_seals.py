"""Seals (DESIGN.md section 7b, "Seals"): the seal kernels' device time, the layout with and without seals="auto", and
restore_regions of seal pages.

    MN_MODULE_GRAPHS=0 python tools/bench_seals.py [--passes 4] [--iters 50] [--scale 2]

The pages are four seeded 1654 x 2339 pages (A4 at 200 dpi) drawn with cv2.putText: paragraphs of dark lines, and two
stamps each (red or blue, round or oval, one over a paragraph), drawn as the host tests draw them.  Prints one JSON line each
for:
  - profile: torch.profiler over --iters layout calls with seals, the device time of each seal kernel per call;
  - layout: ops.find_blocks on the uploaded pages with and without seals, timed with CUDA events over --iters calls per arm,
    the median of --passes passes, the arms' order swapped pass by pass;
  - restore_regions with TextPage(seals="auto"), host uint8 in and out, seconds per page.
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
KERNELS = ("seal_cells_kernel", "seal_union_kernel", "seal_box_kernel", "seal_cand_kernel", "seal_test_kernel",
           "seal_copy_kernel")


def make_pages(seed=0):
    from test_seal_pages import BLUE, RED, stamp
    rng = np.random.default_rng(seed)
    pages = []
    for p in range(4):
        img = np.full((H, W, 3), int(rng.integers(236, 250)), np.uint8)
        for k in range(60):
            cv2.putText(img, " ".join(rng.choice(WORDS, 9)), (100, 150 + 34 * k), FONT, 1.0, (20, 20, 20), 2, cv2.LINE_AA)
        for cx, cy in ((1200, 700 + 200 * p), (1250, 1900)):
            r = int(rng.integers(170, 230))
            stamp(img, cx, cy, r, int(r * rng.uniform(0.75, 1.0)), RED if rng.integers(2) else BLUE,
                  rot=float(rng.uniform(-20, 20)))
        pages.append(img)
    return pages


def _card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True,
                       text=True)
    name, _, power = q.stdout.strip().partition(", ")
    return {"gpu": name or torch.cuda.get_device_name(0), "power_limit": power or None}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--passes", type=int, default=4)
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--scale", type=int, default=2)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_seals.py needs a CUDA device")
    from marconet_b200 import _lib, ops, pipeline
    from marconet_b200.models import networks
    from marconet_b200.testing import synth
    dev = torch.device("cuda:0")
    card = _card()
    pages = make_pages()
    d = [torch.from_numpy(p).to(dev) for p in pages]
    plain = [ops.PageItem(x, (0, 0, W, H), False, _lib.INK_AUTO) for x in d]
    sealed = [r._replace(seal_size=pipeline.seal_size(W, H)) for r in plain]

    from torch.profiler import ProfilerActivity, profile
    for _ in range(5):
        ops.find_blocks(sealed)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(args.iters):
            ops.find_blocks(sealed)
        torch.cuda.synchronize()
    us = {}
    for e in prof.key_averages():
        t = getattr(e, "device_time_total", None) or getattr(e, "cuda_time_total", 0)
        if t:
            us[e.key] = us.get(e.key, 0.0) + t
    per = {k: round(sum(v for n, v in us.items() if k in n) / args.iters, 2) for k in KERNELS}
    print(json.dumps(dict(card, what="profile", pages=len(pages), calls=args.iters, us_per_call=per,
                          seal_kernels_us=round(sum(per.values()), 2))), flush=True)

    def events_ms(items):
        t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        t0.record()
        for _ in range(args.iters):
            ops.find_blocks(items)
        t1.record()
        t1.synchronize()
        return t0.elapsed_time(t1) / args.iters

    for items in (sealed, plain):
        for _ in range(3):
            ops.find_blocks(items)
    ms = {"seals": [], "none": []}
    for k in range(args.passes):
        for name, items in (("seals", sealed), ("none", plain))[::1 if k % 2 == 0 else -1]:
            ms[name].append(events_ms(items))
    tps = [[pipeline.TextPage(seals="auto")] for _ in pages]
    found = pipeline.find_blocks(pages, tps)
    print(json.dumps(dict(card, what="layout", pages=len(pages), megapixels=sum(p.shape[0] * p.shape[1] for p in pages) / 1e6,
                          seals=[len(f[0]["seals"]) for f in found], arcs=[sum(s["arc"] is not None for s in f[0]["seals"])
                                                                           for f in found],
                          blocks=[len(f[0]["blocks"]) for f in found],
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
    print(json.dumps(dict(card, what="restore_regions with seal pages", pages=len(pages), scale=args.scale,
                          seal_regions=[len(o["regions"][0].get("seal_regions", [])) for o in out],
                          seconds_per_page=round(med / len(pages), 4), seconds=[round(t, 4) for t in ts])), flush=True)


if __name__ == "__main__":
    main()
