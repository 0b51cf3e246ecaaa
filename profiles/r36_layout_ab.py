"""Layout time per call of two versions of ops.py, arms alternated in one process (r36_layout_ab.jsonl).

    python profiles/r36_layout_ab.py OLD_OPS_PY [--samples 8] [--iters 20]

OLD_OPS_PY is the other version's marconet_b200/ops.py.  The workloads are the layout-alone modes of tools/bench_pages.py
(ops.find_blocks on level and on skewed pages, ops.find_page_quads on photographed pages) and tools/bench_blocks.py
(ops.find_lines on level and skewed blocks, ops.find_lines_curved on curled blocks), on the same generated pages.  Each sample
times ``iters`` calls with CUDA events after a warm-up; the two arms alternate sample by sample.  The outputs of the two arms
are compared byte for byte.  One JSON line per workload: the card, its power limit, both arms' median and range in ms.
"""
import argparse
import ctypes
import importlib.util
import json
import os
import statistics
import sys

os.environ.setdefault("MN_MODULE_GRAPHS", "0")

import cv2  # noqa: E402
import numpy as np  # noqa: E402
import torch  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tools")]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("old")
    ap.add_argument("--samples", type=int, default=8)
    ap.add_argument("--iters", type=int, default=20)
    a = ap.parse_args()
    import bench_blocks
    import bench_pages
    from marconet_b200 import _lib
    from marconet_b200 import ops as new
    spec = importlib.util.spec_from_file_location("marconet_b200._ops_old", a.old)
    old = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(old)
    dev = torch.device("cuda:0")
    card = bench_pages._card()
    up = lambda imgs: [torch.from_numpy(p).to(dev) for p in imgs]  # noqa: E731
    A = _lib.INK_AUTO

    pages, _ = bench_pages.make_pages(4)
    rng = np.random.default_rng(1)
    tilted = [cv2.warpAffine(p, cv2.getRotationMatrix2D((p.shape[1] / 2, p.shape[0] / 2), float(t), 1.0), (p.shape[1], p.shape[0]),
                             flags=cv2.INTER_LINEAR, borderMode=cv2.BORDER_REPLICATE) for p, t in zip(pages, rng.uniform(-7.5, 7.5, 4))]
    photos, _ = bench_pages.photograph(pages)
    level_b, lb, _ = bench_blocks.make_pages(4, 16)
    skew_b, sb, _ = bench_blocks.make_pages(4, 16, skew=True)
    curl_b, cb, _ = bench_blocks.make_pages(4, 16, curve=True)
    dp, dt, dq, dl, ds, dc = (up(x) for x in (pages, tilted, photos, level_b, skew_b, curl_b))
    page_items = lambda d, skew: [(x, (0, 0, x.shape[1], x.shape[0]), False, A, None, None, skew) for x in d]  # noqa: E731
    block_items = lambda d, bl: [(d[i], b[0].rect, False, A, None, None, None, b[0].skew, b[0].max_skew)  # noqa: E731
                                 for i, b in enumerate(bl)]
    work = {
        "find_blocks level (bench_pages)": lambda m: m.find_blocks(page_items(dp, None)),
        "find_blocks skewed (bench_pages --skew)": lambda m: m.find_blocks(page_items(dt, "auto")),
        "find_page_quads (bench_pages --quad)": lambda m: m.find_page_quads([(x, A) for x in dq]),
        "find_lines level (bench_blocks)": lambda m: m.find_lines(block_items(dl, lb)),
        "find_lines skewed (bench_blocks --skew)": lambda m: m.find_lines(block_items(ds, sb)),
        "find_lines_curved (bench_blocks --curve)": lambda m: m.find_lines_curved(
            [(dc[i], b[0].rect, A, None, None, None, None) for i, b in enumerate(cb)]),
    }
    ssz, osz = ctypes.sizeof(_lib.SkewBlock), ctypes.sizeof(_lib.BlockLines)
    results = {"find_blocks skewed (bench_pages --skew)": lambda r: r[0][4 * ssz:],     # past the skew records, which hold
               "find_lines skewed (bench_blocks --skew)": lambda r: r[:4 * osz]}       # pointers into each arm's own buffer
    for name, fn in work.items():
        cut = results.get(name, lambda r: r[0] if isinstance(r, tuple) else r)
        outs = [cut(fn(m)).cpu() for m in (old, new)]
        same = bool(torch.equal(outs[0], outs[1]))
        for m in (old, new):
            for _ in range(3):
                fn(m)
        ms = {"old": [], "new": []}
        for _ in range(a.samples):
            for key, m in (("old", old), ("new", new)):
                t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                t0.record()
                for _ in range(a.iters):
                    fn(m)
                t1.record()
                t1.synchronize()
                ms[key].append(t0.elapsed_time(t1) / a.iters)
        print(json.dumps(dict(card, workload=name, same_output=same, iters=a.iters, samples=a.samples,
                              **{f"{k}_median_ms": round(statistics.median(v), 4) for k, v in ms.items()},
                              **{f"{k}_range_ms": [round(min(v), 4), round(max(v), 4)] for k, v in ms.items()})), flush=True)


if __name__ == "__main__":
    main()
