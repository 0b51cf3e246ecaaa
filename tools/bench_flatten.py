"""Flat pages (DESIGN.md section 7b, "Flat pages"): pipeline.flatten_pages alone, and flattening before restore_regions.

    MN_MODULE_GRAPHS=0 python tools/bench_flatten.py [--pages 4] [--lines 16] [--passes 3] [--iters 200] [--scale 2]

The pages are tools/bench_blocks.py's curled pages (16 lines, rows moved down by a (x / W)^2, a seeded in +-80 pixels), and an
open-book set: the same pages warped into a darker photo by a homography that shrinks one side to 1/1.8 of the other.  Prints one
JSON line each for:
  - the field: ops.flat_remap (mn_flat_columns_batched and mn_flat_remap_u8_batched, two launches for every page of the call)
    on the found line tables: the two kernels' device time per call from torch.profiler over --iters calls (a separate pass),
    and, with CUDA events over --iters calls, the time per whole call, which also holds building the records and line tables on
    the host and their pageable upload;
  - flatten_pages(curve="auto") on the curled pages and flatten_pages(quad="auto", curve="auto") on the photos: host wall time
    around the whole call (host images in, device pages out) ending in a synchronise, median over --passes, per page;
  - restore_regions on the flat pages (flatten_pages, then TextPage()) against restore_regions on the curled pages with
    TextPage(curve="auto"), host uint8 in and out, pages/s; the arms alternate pass by pass.
Every line carries the card's name and power limit, read in the same run.  Not part of the product path.
"""
import argparse
import json
import os
import sys
import time

os.environ.setdefault("MN_MODULE_GRAPHS", "0")

import cv2  # noqa: E402
import numpy as np  # noqa: E402
import torch  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from bench_blocks import _card, make_pages  # noqa: E402


def open_books(pages, fore=1.8):
    """Each page warped into a darker photo 1.3 times its size, its right side shrunk by ``fore``."""
    out = []
    for page in pages:
        h, w = page.shape[:2]
        H, W = int(h * 1.3), int(w * 1.3)
        m = 0.12
        dst = np.float32([[W * m, H * m], [W * (1 - m), H * (0.5 - (0.5 - m) / fore)],
                          [W * (1 - m), H * (0.5 + (0.5 - m) / fore)], [W * m, H * (1 - m)]])
        hom = cv2.getPerspectiveTransform(np.float32([[0, 0], [w, 0], [w, h], [0, h]]), dst)
        photo = np.full((H, W, 3), 40, np.uint8)
        out.append(cv2.warpPerspective(page, hom, (W, H), dst=photo, flags=cv2.INTER_LINEAR, borderMode=cv2.BORDER_TRANSPARENT))
    return out


def _wall(fn, passes):
    fn()
    ts = []
    for _ in range(passes):
        torch.cuda.synchronize()
        t = time.perf_counter()
        out = fn()
        torch.cuda.synchronize()
        ts.append(time.perf_counter() - t)
    return out, ts


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--pages", type=int, default=4)
    ap.add_argument("--lines", type=int, default=16)
    ap.add_argument("--passes", type=int, default=3)
    ap.add_argument("--iters", type=int, default=200)
    ap.add_argument("--scale", type=int, default=2)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_flatten.py needs a CUDA device")
    from marconet_b200 import ops, pipeline
    from marconet_b200.models import networks
    from marconet_b200.testing import synth
    dev = torch.device("cuda:0")
    card = _card()
    pages, _, amps = make_pages(args.pages, args.lines, curve=True)
    photos = open_books(pages)
    flat_fp, book_fp = pipeline.FlatPage(curve="auto"), pipeline.FlatPage(quad="auto", curve="auto")

    res = pipeline.flatten_pages(pages, [[flat_fp]] * len(pages))
    dpages = [torch.from_numpy(p).to(dev) for p in pages]
    items = [(d, r[0]["image"].clone(), "rect", (0, 0), pipeline.flat_line_table([((0, 0, d.shape[1], d.shape[0]), r[0]["lines"])]))
             for d, r in zip(dpages, res)]
    for _ in range(5):
        ops.flat_remap(items)
    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0.record()
    for _ in range(args.iters):
        ops.flat_remap(items)
    t1.record()
    t1.synchronize()
    ms = t0.elapsed_time(t1) / args.iters
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        for _ in range(args.iters):
            ops.flat_remap(items)
        torch.cuda.synchronize()
    kernel_us = {}
    for e in prof.key_averages():
        for name in ("flat_columns_kernel", "flat_remap_kernel"):
            if name in e.key:
                t = getattr(e, "device_time_total", None)
                kernel_us[name] = kernel_us.get(name, 0.0) + (e.cuda_time_total if t is None else t)
    kernel_ms = {k: round(v / 1000 / args.iters, 4) for k, v in kernel_us.items()}
    print(json.dumps(dict(card, what="dewarp field (flat_remap)", pages=len(items),
                          megapixels=sum(p.shape[0] * p.shape[1] for p in pages) / 1e6,
                          lines=[len(r[0]["lines"]) for r in res], curl_pixels=[round(a, 1) for a in amps],
                          kernel_ms_per_call=kernel_ms, kernel_ms_per_page=round(sum(kernel_ms.values()) / len(items), 4),
                          call_ms_with_host_tables_and_upload=round(ms, 4))), flush=True)

    for name, imgs, fp in (("curled pages", pages, flat_fp), ("open-book photos", photos, book_fp)):
        out, ts = _wall(lambda: pipeline.flatten_pages(imgs, [[fp]] * len(imgs)), args.passes)
        med = float(np.median(ts))
        print(json.dumps(dict(card, what=f"flatten_pages on {name}", pages=len(imgs), sizes=[o[0]["size"] for o in out],
                              lines=[len(o[0].get("lines", [])) for o in out], ms_per_page=round(1000 * med / len(imgs), 3),
                              seconds=[round(t, 4) for t in ts])), flush=True)

    sds = synth.make_checkpoints(0)
    m = []
    for key, cls in (("encoder", networks.TextContextEncoderV2), ("tspgan", networks.TSPGAN), ("sr", networks.TSPSRNet)):
        net = cls()
        net.load_state_dict(sds[key], strict=True)
        m.append(net.eval().to(dev))
    kw = dict(scale=args.scale, skip_invalid=True, to_host=True)

    def flat_then_restore(imgs, fp):
        flat = pipeline.flatten_pages(imgs, [[fp]] * len(imgs))
        return pipeline.restore_regions(*m, [f[0]["image"] for f in flat], [[pipeline.TextPage()]] * len(imgs), **kw)
    arms = {"curled pages, TextPage(curve='auto')":
            lambda: pipeline.restore_regions(*m, pages, [[pipeline.TextPage(curve="auto")]] * len(pages), **kw),
            "flatten_pages, then TextPage()": lambda: flat_then_restore(pages, flat_fp),
            "open-book photos: flatten_pages(quad='auto'), then TextPage()": lambda: flat_then_restore(photos, book_fp)}
    outs = {name: fn() for name, fn in arms.items()}          # warm-up of every shape
    times = {name: [] for name in arms}
    for _ in range(args.passes):
        for name, fn in arms.items():
            torch.cuda.synchronize()
            t = time.perf_counter()
            outs[name] = fn()
            times[name].append(time.perf_counter() - t)
    for name, ts in times.items():
        med = float(np.median(ts))
        lines = [sum(len(b.get("lines", [])) for r in o["regions"] for b in r.get("regions", [])) for o in outs[name]]
        print(json.dumps(dict(card, what=f"restore_regions: {name}", pages=len(pages), lines=lines, scale=args.scale,
                              pages_per_s=round(len(pages) / med, 3), seconds=[round(t, 4) for t in ts])), flush=True)


if __name__ == "__main__":
    main()
