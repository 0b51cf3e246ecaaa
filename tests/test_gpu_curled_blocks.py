"""Curled text blocks on the device (DESIGN.md section 7b, "Curled blocks"): mn_find_lines_curved_u8's strip profiles, runs and
link tables bit for bit against the numpy twin over one call of about 40 blocks, its constant launch count, curled blocks beside
plain, skewed and windowed ones, and pipeline.restore_regions with curled blocks and pages against the same call given the found
lines."""
import math

import cv2
import numpy as np
import pytest
import torch

from oracle import blocks as B
from oracle import curled_blocks as C

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda:0")
TEXTS = ["The quick brown fox jumps over dogs", "Sphinx of black quartz, judge my vow", "Pack my box with five dozen jugs",
         "How vexingly quick daft zebras jump"]


def _models(gpu_models):
    return gpu_models["encoder"], gpu_models["tspgan"], gpu_models["sr"]


def _page(rng, n_lines, kind, amp, light=False, noise=0, margin=60, w=560):
    """n_lines putText lines 36 pixels apart, each column moved down by d(x): "cylinder" amp (x / W)^2, "s" amp sin(2 pi x / W),
    "tilt" amp (x / W - 1/2), or level."""
    h, W = 30 + 36 * n_lines + 2 * margin + int(abs(amp)), w + 2 * margin
    bg = rng.integers(195, 256, 3)
    page = np.empty((h, W, 3), np.uint8)
    page[:] = bg
    top = margin + (int(abs(amp)) if amp < 0 else 0)
    for k in range(n_lines):
        cv2.putText(page, TEXTS[k % len(TEXTS)], (margin + 8, top + 36 + 36 * k), cv2.FONT_HERSHEY_SIMPLEX, 0.7,
                    tuple(int(v) for v in rng.integers(0, 60, 3)), 2, cv2.LINE_AA)
    x = np.arange(W, dtype=np.float64) / (W - 1)
    d = {"cylinder": amp * x ** 2, "s": amp * np.sin(2 * math.pi * x), "tilt": amp * (x - 0.5)}.get(kind, 0 * x)
    mapx = np.tile(np.arange(W, dtype=np.float32), (h, 1))
    mapy = (np.arange(h, dtype=np.float64)[:, None] - d[None, :]).astype(np.float32)
    page = cv2.remap(page, mapx, mapy, cv2.INTER_LINEAR, borderMode=cv2.BORDER_REPLICATE)
    if noise:
        page = np.clip(page.astype(np.int32) + rng.integers(-noise, noise + 1, page.shape), 0, 255).astype(np.uint8)
    return 255 - page if light else page


def _blocks(rng):
    """About 40 blocks: curled, S-curved, tilted and level pages, light on dark, noisy, crops through their pitch, given strip
    counts (one strip, 32 strips of 32 pixels), given knobs, 1 x N, N x 1, 1 x 1, uniform and random blocks, and a tall block
    of 32 strips."""
    pages = [_page(rng, 6, "cylinder", 72), _page(rng, 5, "s", -18), _page(rng, 4, "tilt", 30), _page(rng, 3, "flat", 0),
             _page(rng, 4, "cylinder", -50, light=True), _page(rng, 5, "cylinder", 40, noise=25),
             rng.integers(0, 256, (90, 300, 3), dtype=np.uint8), np.full((40, 200, 3), 131, np.uint8)]
    tall = np.full((6000, 1024, 3), 240, np.uint8)
    tall[(np.arange(6000) // 5) % 12 == 0, 40:1000] = 10
    pages.append(tall)
    items = [(i, (0, 0, pages[i].shape[1], pages[i].shape[0]), "auto", [None] * 3, None) for i in range(len(pages))]
    items += [(0, (0, 0, pages[0].shape[1], pages[0].shape[0]), "auto", [None] * 3, 1),
              (0, (0, 0, pages[0].shape[1], pages[0].shape[0]), "dark", [None] * 3, pages[0].shape[1] // 32),
              (8, (0, 0, 1024, 6000), "auto", [None] * 3, 32), (3, (5, 5, 6, 6), "auto", [None] * 3, None),
              (3, (0, 40, pages[3].shape[1], 41), "auto", [None] * 3, None),
              (3, (100, 0, 101, pages[3].shape[0]), "auto", [None] * 3, None),
              (1, (0, 0, pages[1].shape[1], pages[1].shape[0]), "auto", [2, 3, 4], 8)]
    while len(items) < 40:
        i = int(rng.integers(0, 6))
        H, W = pages[i].shape[:2]
        x0, y0 = int(rng.integers(0, W // 2)), int(rng.integers(0, H // 2))
        rect = (x0, y0, int(rng.integers(x0 + 1, W + 1)), int(rng.integers(y0 + 1, H + 1)))
        pol = ["auto", "dark", "light"][int(rng.integers(0, 3))]
        knobs = [int(rng.integers(1, 6)) if rng.random() < 0.15 else None for _ in range(3)]
        w = rect[2] - rect[0]
        strips = int(rng.integers(1, min(32, w // 32) + 1)) if w >= 64 and rng.random() < 0.3 else None
        items.append((i, rect, pol, knobs, strips))
    return pages, items


def _args(dpages, items):
    from marconet_b200 import _lib
    pol = dict(auto=_lib.INK_AUTO, dark=_lib.INK_DARK, light=_lib.INK_LIGHT)
    return [(dpages[i], rect, pol[p], *knobs, strips) for i, rect, p, knobs, strips in items]


def test_curved_tables_equal_twin():
    """Every strip profile, run table, link header and line row equals the twin's, and the lines of curve=None equal
    oracle/blocks.py's; seven launches for 40 blocks as for one."""
    from marconet_b200 import ops
    from marconet_b200.pipeline import CurvedRegion
    rng = np.random.default_rng(0)
    pages, items = _blocks(rng)
    dpages = [torch.from_numpy(p).to(DEV) for p in pages]
    args = _args(dpages, items)
    n = len(args)
    n0 = ops.LAUNCHES
    ops.find_lines_curved(args[:1])
    assert ops.LAUNCHES - n0 == 7
    n0 = ops.LAUNCHES
    buf, views = ops.find_lines_curved(args, tables=True)
    assert ops.LAUNCHES - n0 == 7
    host = buf.cpu().numpy()
    ldt, cdt = ops.block_lines_dtype(), ops.curve_lines_dtype()
    rec, cur = host[:n * ldt.itemsize].view(ldt), host[n * ldt.itemsize:].view(cdt)
    seen = set()
    for k, ((i, rect, p, knobs, strips), r, c, v) in enumerate(zip(items, rec, cur, views)):
        ref = C.find_lines(pages[i], rect, *knobs, polarity=p, strips=strips)
        d = ref["detail"]
        assert int(r["threshold"]) == ref["threshold"], k
        np.testing.assert_array_equal(v["profiles"].cpu().numpy(), d["profiles"], err_msg=str(k))
        nr = v["nruns"].cpu().numpy()
        rt = v["runs"].cpu().numpy()
        for j, runs in enumerate(d["runs"]):
            if isinstance(runs, int):
                assert nr[j] == runs, (k, j)
                continue
            assert nr[j] == len(runs), (k, j)
            assert [tuple(int(x) for x in q) for q in rt[j, :len(runs)]] == runs, (k, j)
        np.testing.assert_array_equal(c["header"], d["header"], err_msg=str(k))
        nl = int(d["header"][1])
        np.testing.assert_array_equal(c["lines"][:nl], d["table"], err_msg=str(k))
        x0, y0, x1, y1 = rect
        g = B.grey(pages[i][y0:y1, x0:x1])
        ink = (g <= ref["threshold"]) if ref["ink"] == "dark" else (g > ref["threshold"])
        try:
            plain = B.segment(ink, *knobs)
            assert int(r["n_lines"]) == len(plain), k
            assert [tuple(int(x) for x in q) for q in r["rect"][:len(plain)]] == \
                [(x0 + a, y0 + b, x0 + e, y0 + f) for b, a, f, e in plain], k
        except ValueError:
            assert int(r["n_lines"]) < 0, k
        seen.add("curved" if ref["lines"] and isinstance(ref["lines"][0], CurvedRegion) else "level" if ref["lines"] else "none")
        seen.add(f"strips{d['strips']}" if d["strips"] in (1, 32) else "strips")
        if min(x1 - x0, y1 - y0) == 1:
            seen.add("thin")
    assert {"curved", "level", "none", "strips1", "strips32", "strips", "thin"} <= seen, seen


def test_curled_blocks_beside_plain_skewed_and_windowed_blocks():
    """pipeline.find_lines: curled blocks give the twin's lines and curve; the other blocks of the same call return exactly what
    a call without curled blocks returns."""
    from marconet_b200 import pipeline
    rng = np.random.default_rng(1)
    page = _page(rng, 6, "cylinder", 72)
    H, W = page.shape[:2]
    others = [pipeline.TextBlock((0, 0, W, H)), pipeline.TextBlock((0, 0, W, H), skew="auto"),
              pipeline.TextBlock((0, 0, W, H), skew=2.0, window=(0, 0, 300, 200))]
    curled = [pipeline.TextBlock((0, 0, W, H), curve="auto"), pipeline.TextBlock((10, 5, W - 3, H - 2), curve="auto", strips=6)]
    out = pipeline.find_lines([page], [[others[0], curled[0], others[1], curled[1], others[2]]])[0]
    alone = pipeline.find_lines([page], [others])[0]
    assert [out[0], out[2], out[4]] == alone
    for got, blk in ((out[1], curled[0]), (out[3], curled[1])):
        ref = C.find_lines(page, blk.rect, strips=blk.strips)
        assert got["lines"] == ref["lines"] and got["curve"] == ref["curve"]
        assert (got["threshold"], got["ink"]) == (ref["threshold"], ref["ink"])
    assert len(out[1]["lines"]) == 6 and all(isinstance(q, pipeline.CurvedRegion) for q in out[1]["lines"])


def _same(a, b):
    if isinstance(a, dict):
        assert a.keys() == b.keys()
        for k in a:
            _same(a[k], b[k])
    elif isinstance(a, (list, tuple)):
        assert len(a) == len(b)
        for x, y in zip(a, b):
            _same(x, y)
    elif isinstance(a, (np.ndarray, torch.Tensor)):
        x = a.cpu().numpy() if isinstance(a, torch.Tensor) else a
        y = b.cpu().numpy() if isinstance(b, torch.Tensor) else b
        np.testing.assert_array_equal(x, y)
    else:
        assert a == b


@pytest.mark.parametrize("to_host", [False, True])
def test_restore_regions_curled_block_equals_the_found_lines(gpu_models, to_host):
    """A call with a curled block gives the bytes of the call given its CurvedRegion lines, beside a rectangle and an oriented
    region."""
    from marconet_b200 import pipeline
    m = _models(gpu_models)
    rng = np.random.default_rng(2)
    img = np.full((330, 620, 3), 236, np.uint8)
    page = _page(rng, 3, "cylinder", 40, margin=20, w=400)
    ph, pw = page.shape[:2]
    img[:ph, :pw] = page
    blk = pipeline.TextBlock((0, 0, pw, ph), curve="auto")
    others = [(460, 240, 600, 280), pipeline.OrientedRegion.from_rotated(150, 270, 120, 30, 8)]
    found = pipeline.find_lines([img], [[blk]])[0][0]
    assert len(found["lines"]) == 3 and all(isinstance(q, pipeline.CurvedRegion) for q in found["lines"])
    kw = dict(scale=2, feather=3, skip_invalid=True, to_host=to_host)
    a = pipeline.restore_regions(*m, [img], [[others[0], blk, others[1]]], **kw)[0]
    b = pipeline.restore_regions(*m, [img], [[others[0], *found["lines"], others[1]]], **kw)[0]
    _same(a["image"], b["image"])
    e = a["regions"]
    assert {x: e[1][x] for x in ("lines", "threshold", "ink", "curve")} == found
    _same(e[0], b["regions"][0])
    _same(e[1]["regions"], b["regions"][1:4])
    _same(e[2], b["regions"][4])


@pytest.mark.parametrize("to_host", [False, True])
def test_restore_regions_curled_page_equals_the_found_lines(gpu_models, to_host):
    """TextPage(curve="auto"): its blocks are curled blocks, and the call gives the bytes of the call given their lines."""
    from marconet_b200 import pipeline
    m = _models(gpu_models)
    rng = np.random.default_rng(4)
    page = _page(rng, 3, "cylinder", 30, margin=20, w=420)
    pg = pipeline.TextPage(curve="auto")
    blocks = pipeline.find_blocks([page], [[pg]])[0][0]["blocks"]
    assert blocks and all(b.curve == "auto" for b in blocks)
    found = pipeline.find_lines([page], [blocks])[0]
    lines = [q for f in found for q in f["lines"]]
    assert any(isinstance(q, pipeline.CurvedRegion) for q in lines)
    kw = dict(scale=2, skip_invalid=True, to_host=to_host)
    a = pipeline.restore_regions(*m, [page], [[pg]], **kw)[0]
    b = pipeline.restore_regions(*m, [page], [lines], **kw)[0]
    _same(a["image"], b["image"])
    got = [r for blk in a["regions"][0]["regions"] for r in blk["regions"]]
    _same(got, b["regions"])


def test_level_page_under_auto_gives_the_bytes_of_curve_none(gpu_models):
    from marconet_b200 import pipeline
    m = _models(gpu_models)
    rng = np.random.default_rng(3)
    page = _page(rng, 3, "flat", 0, margin=10, w=300)
    H, W = page.shape[:2]
    auto = pipeline.restore_regions(*m, [page], [[pipeline.TextBlock((0, 0, W, H), curve="auto")]], scale=2, to_host=True)[0]
    none = pipeline.restore_regions(*m, [page], [[pipeline.TextBlock((0, 0, W, H))]], scale=2, to_host=True)[0]
    _same(auto["image"], none["image"])
    assert auto["regions"][0]["lines"] == none["regions"][0]["lines"] and len(none["regions"][0]["lines"]) == 3
    _same(auto["regions"][0]["regions"], none["regions"][0]["regions"])
