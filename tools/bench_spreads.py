"""Book spreads (DESIGN.md section 7b, "Book spreads"): the spine search's two kernels, and flatten_pages on photographed spreads
against the same call given the two halves.

    MN_MODULE_GRAPHS=0 python tools/bench_spreads.py [--spreads 4] [--passes 5] [--iters 200] [--out FILE]

The spreads are tests/test_spread_pages.py's book_spread: two curled_page pages of 12 and 10 lines side by side (1600 x 640),
each column squeezed towards the centre row by s(x) = 1 - a (1 - |x - x_s| / 800)^p, a and p seeded per spread, and warped
into a darker 2080 x 832 photo by a homography that shrinks one side by a seeded foreshortening.  Prints (and with --out
writes) one JSON line each for:
  - the spine kernels: mn_find_page_spines_u8 (spine_cols_kernel and spine_kernel, two launches for every spread of the call)
    replayed on the work a find_page_quads call left, device time per call from CUDA events over --iters calls; the
    kernels' split from torch.profiler over --iters calls (a separate pass); and ops.find_page_quads with and without the
    spreads, CUDA events over --iters calls each, arms alternated;
  - flatten_pages(quad="auto", spread="auto", curve="auto") against flatten_pages given the two halves' quads with
    curve="auto", host images in and device pages out, host wall time ending in a synchronise, median of --passes passes with
    the arms alternated, bytes compared.
Every line carries the card's name and power limit, read in the same run.  Not part of the product path.
"""
import argparse
import json
import os
import statistics
import sys
import time

os.environ.setdefault("MN_MODULE_GRAPHS", "0")

import numpy as np  # noqa: E402
import torch  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
sys.path.insert(0, os.path.join(ROOT, "tests"))

from bench_blocks import _card  # noqa: E402
from test_spread_pages import book_spread  # noqa: E402


def _events(fn, iters):
    fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / iters


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--spreads", type=int, default=4)
    ap.add_argument("--passes", type=int, default=5)
    ap.add_argument("--iters", type=int, default=200)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_spreads.py needs a CUDA device")
    import ctypes
    from marconet_b200 import _lib, ops
    from marconet_b200.pipeline import FlatPage, QuadRegion, flatten_pages
    card = _card()
    rng = np.random.default_rng(35)
    made = [book_spread(12, 10, float(rng.uniform(0.08, 0.15)), float(rng.uniform(1.0, 3.0)), float(rng.uniform(1.2, 2.0)), 40 + 2 * k)
            for k in range(args.spreads)]
    photos = [p for p, _ in made]
    dev = [torch.from_numpy(p).cuda() for p in photos]
    lines = []

    def emit(d):
        d = dict(card, **d)
        print(json.dumps(d), flush=True)
        lines.append(d)

    items = [(d, _lib.INK_AUTO) for d in dev]
    n = len(items)
    spreads = list(range(n))
    quads, spines = ops.find_page_quads(items, spreads=spreads)
    torch.cuda.synchronize()
    rec = spines.untyped_storage().data_ptr() + n * (ctypes.sizeof(_lib.TextBlock) + ctypes.sizeof(_lib.QuadPage))
    tiles = max(-(-p.shape[1] // 32) * -(-p.shape[0] // 32) for p in photos)
    lib = _lib.load()
    stream = torch.cuda.current_stream().cuda_stream

    def spine_call():
        _lib.check(lib.mn_find_page_spines_u8(rec, n, tiles, stream), "mn_find_page_spines_u8")
    before = spines.cpu().numpy().copy()
    spine_ms = _events(spine_call, args.iters)
    assert np.array_equal(spines.cpu().numpy(), before)              # a replay writes the same records
    found = spines.cpu().numpy().view(ops.page_spine_dtype())
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(args.iters):
            spine_call()
        torch.cuda.synchronize()
    split = {e.key: round(e.device_time_total / 1000 / args.iters, 4) for e in prof.key_averages() if "spine" in e.key}
    split = {("spine_cols_kernel" if "cols" in k else "spine_kernel"): v for k, v in split.items()}
    with_ms, without_ms = [], []
    for _ in range(args.passes):
        without_ms.append(_events(lambda: ops.find_page_quads(items), args.iters // 4))
        with_ms.append(_events(lambda: ops.find_page_quads(items, spreads=spreads), args.iters // 4))
    emit(dict(what="spine kernels (mn_find_page_spines_u8)", spreads=n, sizes=[[p.shape[1], p.shape[0]] for p in photos],
              found=[bool(r["found"]) for r in found], kernel_ms_per_call=round(spine_ms, 4), kernel_split_ms=split,
              find_page_quads_ms=dict(without_spreads=round(statistics.median(without_ms), 4),
                                      with_spreads=round(statistics.median(with_ms), 4))))

    spread_pages = [[FlatPage(quad="auto", spread="auto", curve="auto")] for _ in photos]
    got = flatten_pages(photos, spread_pages, to_host=True)
    halves = [[FlatPage(quad=QuadRegion(*p["quad"]), curve="auto") for p in g[0]["pages"]] for g in got]
    want = flatten_pages(photos, halves, to_host=True)
    same = all(np.array_equal(a["image"], b["image"]) for g, w in zip(got, want) for a, b in zip(g[0]["pages"], w))

    def wall(fn):
        torch.cuda.synchronize()
        t = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        return time.perf_counter() - t
    ts, tg = [], []
    for k in range(args.passes):
        arms = [(ts, lambda: flatten_pages(photos, spread_pages)), (tg, lambda: flatten_pages(photos, halves))]
        for out, fn in (arms if k % 2 == 0 else arms[::-1]):
            out.append(wall(fn))
    emit(dict(what="flatten_pages spread='auto' vs halves given (curve='auto')", spreads=n, same_bytes=same,
              spine=[g[0]["spine"] for g in got], depth=[[round(v, 2) for v in g[0]["depth"]] for g in got],
              ms_per_spread=dict(spread_auto=round(1000 * statistics.median(ts) / n, 3),
                                 halves_given=round(1000 * statistics.median(tg) / n, 3)),
              seconds=dict(spread_auto=[round(v, 4) for v in ts], halves_given=[round(v, 4) for v in tg])))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            for d in lines:
                f.write(json.dumps(d) + "\n")


if __name__ == "__main__":
    main()
