"""Text pages (DESIGN.md section 7b, "Text pages"): the layout analysis alone and restore_regions with pages.

    MN_MODULE_GRAPHS=0 python tools/bench_pages.py [--pages 4] [--passes 3] [--iters 100] [--scale 2] [--skew | --quad]

The pages are seeded 1600 x 1200 pages: a heading over two or three columns of capital-letter lines drawn with cv2.putText
(Hershey DUPLEX) on a light, slightly noisy background, one TextPage each.  Prints one JSON line each for:
  - layout: ops.find_blocks (mn_find_blocks_u8: 149 launches for every page of the call) on the uploaded pages, timed with
    CUDA events over --iters calls, per call and per page;
  - restore_regions with the pages against the same call given the found blocks, host uint8 in and out, pages/s; the arms
    alternate pass by pass and must give the same bytes.
With --skew (DESIGN.md section 7b, "Skewed pages") the pages are turned by seeded angles within +-7.5 degrees and searched with
TextPage(skew="auto"): the layout line times mn_find_blocks_skewed_u8 against the level pages in the same run, and the
restore_regions arms are the tilted pages against the call given the found lines.
With --quad (DESIGN.md section 7b, "Perspective pages") each page is photographed: warped by a seeded homography (each corner
pulled inwards by up to 10% of the page's sides) onto a canvas 120 pixels wider on every side, over a darker textured background,
and found with TextPage(quad="auto"): the layout line times the corner search (mn_find_page_quads_u8), the warp of the found
quads and the XY-cut of the rectified crops apart and together (with the host copy of the corners between them), and the
restore_regions arms are the photographed pages against the call given the found lines.
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

WORDS = "THE QUICK BROWN FOX JUMPS OVER A LAZY DOG PACK MY BOX WITH FIVE DOZEN JUGS 0123456789".split()


def make_pages(n_pages, seed=0):
    """n_pages 1600 x 1200 pages, each a heading over two or three columns of 30 lines 33 pixels apart: (pages, columns)."""
    rng = np.random.default_rng(seed)
    H, W, pitch, gutter = 1200, 1600, 33, 60
    pages, cols = [], []
    for p in range(n_pages):
        n_cols = 2 + p % 2
        cw = (W - 80 - gutter * (n_cols - 1)) // n_cols
        bg = rng.integers(215, 246, 3)
        page = np.clip(bg + rng.integers(-12, 13, (H, W, 1)), 0, 255).astype(np.uint8)
        cv2.putText(page, "A HEADING OVER THE COLUMNS", (40, 70), cv2.FONT_HERSHEY_DUPLEX, 1.0, (20, 20, 20), 2, cv2.LINE_AA)
        for c in range(n_cols):
            for k in range(30):
                t = str(rng.choice(WORDS))
                while True:
                    longer = t + " " + str(rng.choice(WORDS))
                    if cv2.getTextSize(longer, cv2.FONT_HERSHEY_DUPLEX, 1.0, 2)[0][0] > cw:
                        break
                    t = longer
                cv2.putText(page, t, (40 + c * (cw + gutter), 130 + pitch * k), cv2.FONT_HERSHEY_DUPLEX, 1.0, (20, 20, 20), 2,
                            cv2.LINE_AA)
        pages.append(page)
        cols.append(n_cols)
    return pages, cols


def photograph(pages, seed=2, margin=120):
    """The pages warped by seeded homographies over darker textured backgrounds: (images, corners tl, tr, br, bl)."""
    rng = np.random.default_rng(seed)
    out, corners = [], []
    for p in pages:
        h, w = p.shape[:2]
        a = rng.uniform(0, 0.1, 8) * np.array([w, h] * 4)
        c = np.float32([[margin + a[0], margin + a[1]], [margin + w - a[2], margin + a[3]],
                        [margin + w - a[4], margin + h - a[5]], [margin + a[6], margin + h - a[7]]])
        M = cv2.getPerspectiveTransform(np.float32([[0, 0], [w, 0], [w, h], [0, h]]) - 0.5, c - 0.5)
        size = (w + 2 * margin, h + 2 * margin)
        warped = cv2.warpPerspective(p, M, size, flags=cv2.INTER_LINEAR)
        cover = cv2.warpPerspective(np.full((h, w), 255, np.uint8), M, size, flags=cv2.INTER_NEAREST) > 0
        bg = cv2.GaussianBlur(rng.integers(80, 150, size[::-1]).astype(np.uint8), (7, 7), 0)[..., None].repeat(3, axis=2)
        out.append(np.where(cover[..., None], warped, bg))
        corners.append([[round(float(x), 2), round(float(y), 2)] for x, y in c])
    return out, corners


def _card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True,
                       text=True)
    name, _, power = q.stdout.strip().partition(", ")
    return {"gpu": name or torch.cuda.get_device_name(0), "power_limit": power or None}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--pages", type=int, default=4)
    ap.add_argument("--passes", type=int, default=3)
    ap.add_argument("--iters", type=int, default=100)
    ap.add_argument("--scale", type=int, default=2)
    ap.add_argument("--skew", action="store_true")
    ap.add_argument("--quad", action="store_true")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_pages.py needs a CUDA device")
    from marconet_b200 import _lib, ops, pipeline
    from marconet_b200.models import networks
    from marconet_b200.testing import synth
    dev = torch.device("cuda:0")
    card = _card()
    pages, cols = make_pages(args.pages)

    level = pages
    angles = [round(float(a), 2) for a in np.random.default_rng(1).uniform(-7.5, 7.5, len(pages))] if args.skew else None
    if args.skew:
        pages = [cv2.warpAffine(p, cv2.getRotationMatrix2D((p.shape[1] / 2, p.shape[0] / 2), a, 1.0), (p.shape[1], p.shape[0]),
                                flags=cv2.INTER_LINEAR, borderMode=cv2.BORDER_REPLICATE) for p, a in zip(pages, angles)]
    if args.quad:
        pages, drawn = photograph(pages)
    page = pipeline.TextPage(skew="auto") if args.skew else pipeline.TextPage(quad="auto") if args.quad else pipeline.TextPage()

    def events_ms(fn):
        for _ in range(5):
            fn()
        t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        t0.record()
        for _ in range(args.iters):
            fn()
        t1.record()
        t1.synchronize()
        return t0.elapsed_time(t1) / args.iters

    def quad_layout():
        d = dict(enumerate(torch.from_numpy(p).to(dev) for p in pages))
        items = [(i, page, (0, 0, x.shape[1], x.shape[0])) for i, x in d.items()]
        found = pipeline._page_quads(d, items)
        keys = [pipeline._quad_key(i, pg.quad) for i, pg, _ in found]
        rq = pipeline._rectify(d, keys)
        crops = [ops.PageItem(rq[k], (0, 0, rq[k].shape[1], rq[k].shape[0]), False, _lib.INK_AUTO) for k in keys]
        times = dict(search_ms=events_ms(lambda: ops.find_page_quads([(x, _lib.INK_AUTO) for x in d.values()])),
                     warp_ms=events_ms(lambda: pipeline._rectify(d, keys)), xy_cut_ms=events_ms(lambda: ops.find_blocks(crops)),
                     ms_per_call=events_ms(lambda: pipeline._find_pages(d, items)))
        return {k: round(v, 4) for k, v in times.items()}, [[list(p) for p in pg.quad] for _, pg, _ in found]

    def layout_ms(imgs, skew):
        d = [torch.from_numpy(p).to(dev) for p in imgs]
        items = [ops.PageItem(x, (0, 0, x.shape[1], x.shape[0]), False, _lib.INK_AUTO, skew=skew) for x in d]
        for _ in range(5):
            ops.find_blocks(items)
        t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        t0.record()
        for _ in range(args.iters):
            ops.find_blocks(items)
        t1.record()
        t1.synchronize()
        return t0.elapsed_time(t1) / args.iters

    extra = {}
    if args.quad:
        extra, quads = quad_layout()
        ms = extra.pop("ms_per_call")
        extra.update(drawn=drawn, found=quads)
    else:
        ms = layout_ms(pages, "auto" if args.skew else None)
    found = pipeline.find_blocks(pages, [[page] for _ in pages])
    if args.skew:
        extra = dict(angles=angles, found=[f[0]["skew"] for f in found], level_ms_per_call=round(layout_ms(level, None), 4))
    print(json.dumps(dict(card, what="layout", pages=len(pages), megapixels=sum(p.shape[0] * p.shape[1] for p in pages) / 1e6,
                          columns=cols, blocks=[len(f[0]["blocks"]) for f in found], text_size=[f[0]["text_size"] for f in found],
                          ms_per_call=round(ms, 4), ms_per_page=round(ms / len(pages), 4), **extra)), flush=True)

    sds = synth.make_checkpoints(0)
    m = []
    for key, cls in (("encoder", networks.TextContextEncoderV2), ("tspgan", networks.TSPGAN), ("sr", networks.TSPSRNet)):
        net = cls()
        net.load_state_dict(sds[key], strict=True)
        m.append(net.eval().to(dev))
    blocks = [f[0]["blocks"] for f in found]
    kw = dict(scale=args.scale, skip_invalid=True, to_host=True)
    if args.skew or args.quad:
        lines = [[q for r in f for q in r["lines"]] for f in pipeline.find_lines(pages, blocks)]
        base = ("found lines", lambda: pipeline.restore_regions(*m, pages, lines, **kw))
    else:
        base = ("found blocks", lambda: pipeline.restore_regions(*m, pages, blocks, **kw))
    arms = {"pages": lambda: pipeline.restore_regions(*m, pages, [[page] for _ in pages], **kw), base[0]: base[1]}
    outs = {name: fn() for name, fn in arms.items()}          # warm-up of every shape
    times = {name: [] for name in arms}
    for _ in range(args.passes):
        for name, fn in arms.items():
            torch.cuda.synchronize()
            t = time.perf_counter()
            outs[name] = fn()
            times[name].append(time.perf_counter() - t)
    for a, b in zip(outs["pages"], outs[base[0]]):
        assert np.array_equal(a["image"], b["image"]), "the arms differ"
    n_lines = sum(len(e["lines"]) for f in outs["pages"] for p in f["regions"] for e in p.get("regions", []) if "lines" in e)
    for name, ts in times.items():
        med = float(np.median(ts))
        print(json.dumps(dict(card, what=f"restore_regions with {name}", pages=len(pages), lines=n_lines, scale=args.scale,
                              pages_per_s=round(len(pages) / med, 3), seconds=[round(t, 4) for t in ts])), flush=True)


if __name__ == "__main__":
    main()
