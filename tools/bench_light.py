"""Even lighting (DESIGN.md section 7b, "Even lighting"): the evening kernels alone, and flatten_pages with and without it.

    MN_MODULE_GRAPHS=0 python tools/bench_light.py [--pages 4] [--lines 16] [--passes 5] [--iters 50]

The pages are tools/bench_blocks.py's curled pages (16 lines) under a seeded shading: a linear falloff of up to 0.6 in a random
direction times a vignette of up to 0.5 around a random centre; and one 4000 x 3000 page of noisy paper under the same kind of
shading.  Prints one JSON line each for:
  - ops.even_light (mn_even_light_u8, six launches for every page of the call) on the curled pages in one call, and on the large
    page alone: the kernels' device time per call and per page from torch.profiler over --iters calls (a separate pass), and
    with CUDA events the time per whole call, which also holds building and uploading the records;
  - flatten_pages(FlatPage(curve="auto")) on the shaded pages with and without light="even": host wall time around the whole
    call (host images in, device pages out) ending in a synchronise, median over --passes, the two arms alternating.
Every line carries the card's name and power limit, read in the same run.  Not part of the product path.
"""
import argparse
import json
import os
import sys
import time

os.environ.setdefault("MN_MODULE_GRAPHS", "0")

import numpy as np  # noqa: E402
import torch  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from bench_blocks import _card, make_pages  # noqa: E402


def shaded(img, rng):
    """img under a seeded falloff times a vignette."""
    h, w = img.shape[:2]
    y, x = np.mgrid[0:h, 0:w].astype(np.float32)
    a = rng.uniform(0, 2 * np.pi)
    t = (np.cos(a) * x / w + np.sin(a) * y / h)
    t = (t - t.min()) / max(float(t.max() - t.min()), 1e-6)
    cx, cy = rng.uniform(0.2, 0.8, 2)
    f = (1 - 0.6 * t) * (1 - 0.5 * ((x / w - cx) ** 2 + (y / h - cy) ** 2))
    return np.clip(np.rint(img * f[..., None]), 0, 255).astype(np.uint8)


def large_page(rng, h=3000, w=4000):
    paper = rng.integers(200, 246, (h, w, 3), dtype=np.uint8)
    return shaded(paper, rng)


def kernel_ms(fn, iters, names):
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        for _ in range(iters):
            fn()
        torch.cuda.synchronize()
    total = 0.0
    for e in prof.key_averages():
        if any(n in e.key for n in names):
            t = getattr(e, "device_time_total", None)
            total += e.cuda_time_total if t is None else t
    return total / 1000 / iters


def event_ms(fn, iters):
    for _ in range(3):
        fn()
    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0.record()
    for _ in range(iters):
        fn()
    t1.record()
    t1.synchronize()
    return t0.elapsed_time(t1) / iters


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--pages", type=int, default=4)
    ap.add_argument("--lines", type=int, default=16)
    ap.add_argument("--passes", type=int, default=5)
    ap.add_argument("--iters", type=int, default=50)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_light.py needs a CUDA device")
    from marconet_b200 import _lib, ops, pipeline
    dev = torch.device("cuda:0")
    card = _card()
    rng = np.random.default_rng(0)
    pages = [shaded(p, rng) for p in make_pages(args.pages, args.lines, curve=True)[0]]
    big = large_page(rng)
    names = ("light_pass_kernel", "block_hist_kernel", "block_threshold_kernel")
    for what, imgs in (("curled pages", pages), ("4000x3000 page", [big])):
        dimgs = [torch.from_numpy(p).to(dev) for p in imgs]
        outs = [torch.empty_like(d) for d in dimgs]
        items = [(d, d, o, ops.light_window(d.shape[1], d.shape[0]), _lib.INK_AUTO) for d, o in zip(dimgs, outs)]
        ms = event_ms(lambda: ops.even_light(items), args.iters)
        kms = kernel_ms(lambda: ops.even_light(items), args.iters, names)
        mpix = sum(p.shape[0] * p.shape[1] for p in imgs) / 1e6
        print(json.dumps(dict(card, what=f"even_light on {what}", pages=len(imgs), megapixels=round(mpix, 3),
                              windows=[it[3] for it in items], kernel_ms_per_call=round(kms, 4),
                              kernel_ms_per_page=round(kms / len(imgs), 4), call_ms_with_records=round(ms, 4))), flush=True)

    arms = {"curve='auto'": pipeline.FlatPage(curve="auto"),
            "curve='auto', light='even'": pipeline.FlatPage(curve="auto", light="even")}
    for fp in arms.values():                                   # warm-up of every shape
        pipeline.flatten_pages(pages, [[fp]] * len(pages))
    times = {name: [] for name in arms}
    lines = {}
    for _ in range(args.passes):
        for name, fp in arms.items():
            torch.cuda.synchronize()
            t = time.perf_counter()
            out = pipeline.flatten_pages(pages, [[fp]] * len(pages))
            torch.cuda.synchronize()
            times[name].append(time.perf_counter() - t)
            lines[name] = [len(o[0].get("lines", [])) for o in out]
    for name, ts in times.items():
        med = float(np.median(ts))
        print(json.dumps(dict(card, what=f"flatten_pages, {name}", pages=len(pages), lines=lines[name],
                              ms_per_call=round(1000 * med, 3), ms_per_page=round(1000 * med / len(pages), 3),
                              seconds=[round(t, 4) for t in ts])), flush=True)


if __name__ == "__main__":
    main()
