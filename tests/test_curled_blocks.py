"""Curled text blocks (DESIGN.md section 7b, "Curled blocks") on the host: pages drawn with cv2.putText and bent with cv2.remap
through a known vertical displacement, the row profile's failure on them, the twin's traced lines and their CurvedRegions, the
level and tilted cases, the empty cases, the limits of the link, and every validation error of find_lines, find_blocks and
restore_regions, raised before any launch."""
import math

import cv2
import numpy as np
import pytest
import torch

from oracle import blocks as B
from oracle import curled_blocks as C

TEXTS = ["The quick brown fox jumps over dogs", "Sphinx of black quartz, judge my vow", "Pack my box with five dozen jugs",
         "How vexingly quick daft zebras jump", "Hershey fonts need no download 0123", "Bright vixens jump; dozy fowl quack"]
PITCH = 36


def curl(kind, w, amp):
    """The vertical displacement d(x) of a page w pixels wide: "cylinder", a curl toward the right side reaching ``amp`` pixels,
    or "s", a gentle S-curve of amplitude ``amp``; "tilt" is a straight slope of ``amp`` pixels over the width."""
    x = np.arange(w, dtype=np.float64)
    if kind == "cylinder":
        return amp * (x / (w - 1)) ** 2
    if kind == "s":
        return amp * np.sin(2 * math.pi * x / (w - 1))
    if kind == "tilt":
        return amp * (x / (w - 1) - 0.5)
    return np.zeros(w)


def curled_page(n_lines, kind, amp, seed, margin=110, scale=0.7, light=False):
    """A page of n_lines lines PITCH pixels apart, about 560 pixels wide, each row moved down by d(x) (curl) with cv2.remap.
    Returns the image, one boolean ink mask per line bent alike, and the block rectangle around the text."""
    rng = np.random.default_rng(seed)
    h, w = 30 + PITCH * n_lines + 2 * margin, 580 + 2 * margin
    masks = []
    for k in range(n_lines):
        m = np.zeros((h, w), np.uint8)
        cv2.putText(m, TEXTS[(k + seed) % len(TEXTS)], (margin + 8, margin + 36 + PITCH * k), cv2.FONT_HERSHEY_SIMPLEX, scale,
                    255, 2, cv2.LINE_8)
        masks.append(m)
    ink = np.zeros((h, w), np.uint8)
    for m in masks:
        ink |= m
    paper, dark = rng.integers(205, 256, 3), rng.integers(0, 50, 3)
    if light:
        paper, dark = dark, paper
    page = np.empty((h, w, 3), np.uint8)
    page[:] = paper
    page[ink > 0] = dark
    d = curl(kind, w, amp)
    mapx = np.tile(np.arange(w, dtype=np.float32), (h, 1))
    mapy = (np.arange(h, dtype=np.float64)[:, None] - d[None, :]).astype(np.float32)
    page = cv2.remap(page, mapx, mapy, cv2.INTER_LINEAR, borderMode=cv2.BORDER_REPLICATE)
    masks = [cv2.remap(m, mapx, mapy, cv2.INTER_NEAREST) > 0 for m in masks]
    rect = (margin - 20, max(0, int(margin - 20 + min(0, d.min()))), w - margin + 20,
            min(h, int(h - margin + 30 + max(0, d.max()))))
    return page, masks, rect


def _ink(page, rect):
    x0, y0, x1, y1 = rect
    g = B.grey(page[y0:y1, x0:x1])
    t = B.otsu(g)
    return (g <= t) if 2 * int((g <= t).sum()) <= g.size else (g > t)


def inside_curved(region, shape, grow=0.0):
    """Pixels of an image of ``shape`` whose centres lie in a one-segment CurvedRegion's band, by the twin's inversion: the
    column's t by bisection on the x of the mid curve (x is monotone in t here), then T(t).y - grow <= y <= B(t).y + grow."""
    from marconet_b200.pipeline import _bezier_1d
    top, bottom = region
    tx, ty = [p[0] for p in top], [p[1] for p in top]
    bx, by = [p[0] for p in bottom], [p[1] for p in bottom]
    H, W = shape
    out = np.zeros(shape, bool)
    ys = np.arange(H) + 0.5
    for x in range(W):
        xc = x + 0.5
        if not (min(tx[0], bx[0]) <= xc <= max(tx[3], bx[3])):
            continue
        lo, hi = 0.0, 1.0
        for _ in range(40):
            mid = (lo + hi) / 2
            if 0.5 * (_bezier_1d(tx, mid) + _bezier_1d(bx, mid)) < xc:
                lo = mid
            else:
                hi = mid
        t = (lo + hi) / 2
        out[:, x] = (ys >= _bezier_1d(ty, t) - grow) & (ys <= _bezier_1d(by, t) + grow)
    return out


def check_curved_lines(lines, masks, ink, rect, shape, tol=0.5):
    """Each drawn line's ink (its mask where the block's threshold finds ink) lies inside its own CurvedRegion, widened by
    ``tol`` pixels, and outside every other one, narrowed by ``tol``: every drawn line is in exactly one region."""
    x0, y0, x1, y1 = rect
    full = np.zeros(shape, bool)
    full[y0:y1, x0:x1] = ink
    bands = [inside_curved(q, shape, tol) for q in lines]
    cores = [inside_curved(q, shape, -tol) for q in lines]
    for k, m in enumerate(masks):
        mk = m & full
        assert mk.any(), k
        assert not (mk & ~bands[k]).any(), f"line {k} leaves its region ({int((mk & ~bands[k]).sum())} pixels)"
        for j in range(len(lines)):
            if j != k:
                assert not (mk & cores[j]).any(), f"line {k}'s ink is inside line {j}'s region"


CURLS = [(6, "cylinder", 2 * PITCH, 1), (8, "cylinder", -2 * PITCH, 2), (5, "cylinder", 1.5 * PITCH, 3), (7, "s", 0.5 * PITCH, 4),
         (4, "s", -0.5 * PITCH, 5)]


@pytest.mark.parametrize("n_lines,kind,amp,seed", CURLS)
def test_row_profile_merges_lines_of_a_curled_page(n_lines, kind, amp, seed):
    """The failure curve="auto" fixes: the single row profile of curve=None runs lines together on these pages."""
    page, _, rect = curled_page(n_lines, kind, amp, seed)
    assert len(B.find_lines(page, rect)["lines"]) < n_lines


@pytest.mark.parametrize("n_lines,kind,amp,seed", CURLS)
def test_twin_traces_every_line_into_its_own_region(n_lines, kind, amp, seed):
    from marconet_b200.pipeline import CurvedRegion, plan_regions
    page, masks, rect = curled_page(n_lines, kind, amp, seed)
    res = C.find_lines(page, rect)
    lines = res["lines"]
    assert len(lines) == n_lines
    assert all(isinstance(q, CurvedRegion) for q in lines)
    assert res["curve"]["strips"] == C.strip_count(rect[2] - rect[0])
    check_curved_lines(lines, masks, _ink(page, rect), rect, page.shape[:2])
    plan_regions([page.shape[:2]], [lines])                     # every traced line passes the curved rules


def test_light_on_dark_page():
    page, masks, rect = curled_page(5, "cylinder", 60, 7, light=True)
    res = C.find_lines(page, rect)
    assert res["ink"] == "light" and len(res["lines"]) == 5
    check_curved_lines(res["lines"], masks, _ink(page, rect), rect, page.shape[:2])


@pytest.mark.parametrize("n_lines,seed", [(1, 1), (4, 2), (9, 3)])
def test_level_pages_give_the_rectangles_of_curve_none(n_lines, seed):
    page, _, rect = curled_page(n_lines, "flat", 0, seed)
    res = C.find_lines(page, rect)
    assert res["lines"] == B.find_lines(page, rect)["lines"]
    assert all(isinstance(q, tuple) and len(q) == 4 and isinstance(q[0], int) for q in res["lines"])


@pytest.mark.parametrize("amp,seed", [(30, 1), (-40, 2), (22, 3)])
def test_tilted_pages_give_straight_curves(amp, seed):
    """A page tilted by a few degrees is not level (curve=None runs its lines together): its lines stay CurvedRegions, nearly
    straight ones, each holding its own line.  The edges follow each strip's ink extent, whose ascenders and descenders move it
    by a few pixels, so an edge may leave its chord by up to 4 pixels."""
    from marconet_b200.pipeline import _bezier_1d
    page, masks, rect = curled_page(6, "tilt", amp, seed)
    assert len(B.find_lines(page, rect)["lines"]) < 6
    res = C.find_lines(page, rect)
    assert len(res["lines"]) == 6
    for top, bottom in res["lines"]:
        for curve in (top, bottom):
            ys = [p[1] for p in curve]
            assert max(abs(_bezier_1d(ys, i / 32) - (ys[0] + (ys[3] - ys[0]) * i / 32)) for i in range(33)) <= 4.0
    check_curved_lines(res["lines"], masks, _ink(page, rect), rect, page.shape[:2])


@pytest.mark.parametrize("fill", [0, 255, 128])
def test_uniform_crops_have_no_lines(fill):
    img = np.full((200, 400, 3), fill, np.uint8)
    res = C.find_lines(img, (0, 0, 400, 200))
    assert res["lines"] == [] and "error" not in res
    assert int(res["detail"]["header"][1]) == 0


def test_one_pixel_crops():
    img = np.zeros((5, 5, 3), np.uint8)
    img[2, 2] = 255
    for rect in ((2, 2, 3, 3), (0, 2, 5, 3), (2, 0, 3, 5)):
        res = C.find_lines(img, rect)
        assert "error" not in res and res["detail"]["strips"] == 1


def test_lines_skip_strips():
    """A line whose words leave gaps of up to MAX_GAP strips stays one line; a gap of more starts a new one, and lines over fewer
    than a quarter of the strips are dropped."""
    w, n = 32 * 16, 16
    ink = np.zeros((60, w), bool)
    for j in range(n):
        if j not in (4, 5, 9, 10, 11):                  # skips 2 strips, then 3
            ink[20:32, 32 * j + 4:32 * j + 28] = True
    xb = C.bounds(w, n)
    prof = C.strip_profiles(ink, n)
    runs = [C.strip_runs(prof[j], xb[j + 1] - xb[j], w) for j in range(n)]
    header, table = C.link(runs, n)
    assert int(header[1]) == 2                          # strips 0-8 (one line), 12-15 (a second); neither is short
    assert [int(v) for v in table[:, 2]] == [7, 4]
    assert [(int(a), int(b)) for a, b in table[:, :2]] == [(0, 8), (12, 15)]


def test_link_tie_goes_to_the_upper_run():
    """Two runs of the next strip overlap the line's last run equally: the upper one continues it, the lower starts a line."""
    runs = [[(10, 20, 0, 31)], [(5, 15, 32, 63), (15, 25, 32, 63)]]
    header, table = C.link(runs, 2)
    assert int(header[1]) == 2
    assert [int(v) for v in table[0, 8:12]] == [10, 20, 5, 15]
    assert [int(v) for v in table[1, 8:12]] == [-1, -1, 15, 25]


def test_single_strip_block():
    page, _, rect = curled_page(3, "flat", 0, 1)
    res = C.find_lines(page, rect, strips=1)
    assert res["detail"]["strips"] == 1
    assert res["lines"] == B.find_lines(page, rect)["lines"]


def test_default_strip_count():
    assert [C.strip_count(w) for w in (1, 47, 48, 95, 96, 1000, 1536, 10000)] == [1, 1, 1, 1, 2, 20, 32, 32]
    from marconet_b200 import ops
    assert all(ops.curve_strips(w) == C.strip_count(w) for w in range(1, 4000, 37))


BAD = [
    (dict(curve="yes"), "curve must be None or 'auto'"),
    (dict(curve=True), "curve must be None or 'auto'"),
    (dict(curve="auto", strips=0), "strips must be a positive integer"),
    (dict(curve="auto", strips=2.0), "strips must be a positive integer"),
    (dict(curve="auto", strips=True), "strips must be a positive integer"),
    (dict(strips=4), "strips is given, but curve is None"),
    (dict(curve="auto", strips=33), "at most 32 strips"),
    (dict(curve="auto", strips=10), "each at least 32 pixels wide"),
    (dict(curve="auto", skew="auto"), "curve and skew are both given"),
    (dict(curve="auto", skew=2.0, window=(0, 0, 10, 10)), "curve and skew are both given"),
    (dict(curve="auto", direction="vertical"), "curved columns are not supported|curled columns are not supported"),
]


@pytest.mark.parametrize("kw,msg", BAD)
def test_find_lines_rejects_bad_curve_before_any_launch(kw, msg):
    from marconet_b200 import pipeline
    img = np.zeros((30, 300, 3), np.uint8)
    blk = pipeline.TextBlock((0, 0, 300, 30), **kw)
    with pytest.raises(ValueError, match=f"image 1, block 1: .*({msg})"):
        pipeline.find_lines([img, img], [[], [pipeline.TextBlock((0, 0, 4, 4), curve="auto"), blk]])


@pytest.mark.parametrize("kw,msg", BAD)
def test_restore_regions_rejects_bad_curve_before_any_launch(kw, msg):
    from marconet_b200 import pipeline
    img = np.zeros((30, 300, 3), np.uint8)
    blk = pipeline.TextBlock((0, 0, 300, 30), **kw)
    with pytest.raises(ValueError, match=f"image 0, region 1 \\(a text block\\): .*({msg})"):
        pipeline.restore_regions(None, None, None, [img], [[pipeline.TextBlock((0, 0, 4, 4), curve="auto"), blk]])


def test_curve_with_quad_is_rejected():
    from marconet_b200 import pipeline
    img = np.zeros((100, 300, 3), np.uint8)
    q = pipeline.QuadRegion((10, 10), (290, 12), (288, 90), (12, 88))
    blk = pipeline.TextBlock.from_quad(q, curve="auto")
    with pytest.raises(ValueError, match="image 0, block 0: curve and quad are both given"):
        pipeline.find_lines([img], [[blk]])


PAGE_BAD = [
    (dict(curve="no"), "curve must be None or 'auto'"),
    (dict(curve="auto", skew="auto"), "curve and skew are both given"),
    (dict(curve="auto", quad="auto"), "curve and quad are both given"),
    (dict(curve="auto", direction="vertical"), "curve is given for a vertical block \\(curled columns are not supported\\)"),
]


@pytest.mark.parametrize("kw,msg", PAGE_BAD)
def test_find_blocks_and_restore_regions_reject_bad_page_curve_before_any_launch(kw, msg):
    from marconet_b200 import pipeline
    img = np.zeros((60, 300, 3), np.uint8)
    pg = pipeline.TextPage(**kw)
    with pytest.raises(ValueError, match=f"image 0, page 0: {msg}"):
        pipeline.find_blocks([img], [[pg]])
    with pytest.raises(ValueError, match=f"image 0, region 0 \\(a text page\\): {msg}"):
        pipeline.restore_regions(None, None, None, [img], [[pg]])


def test_work_limit_is_checked_before_any_launch(monkeypatch):
    """The curled blocks of a call add up their work memory in order; the block that passes the limit is named.  The image is a
    broadcast view: validation reads its shape only."""
    from marconet_b200 import ops, pipeline
    img = torch.zeros(1, 1, 3, dtype=torch.uint8).expand(4000, 3200, 3)
    one = ops.curve_block_bytes(3200, 4000)
    monkeypatch.setattr(ops, "CURVE_MAX_WORK", 2 * one)
    blk = pipeline.TextBlock((0, 0, 3200, 4000), curve="auto")
    with pytest.raises(ValueError, match="image 0, block 3: the call's curled blocks up to this one need"):
        pipeline.find_lines([img], [[blk, pipeline.TextBlock((0, 0, 3200, 4000)), blk, blk]])
    with pytest.raises(ValueError, match="image 0, region 2 \\(a text block\\): the call's curled blocks"):
        pipeline.restore_regions(None, None, None, [img], [[blk, blk, blk]])
    assert one == ops.curve_block_bytes(3200, 4000, 32) and ops.curve_strips(3200) == 32


def test_curve_lines_level_rule():
    """curve_lines on a hand-made table of two lines: level when curve=None's two rectangles hold every run of their line (the
    rectangles come back as they are); curves when a run leaves its rectangle, when the counts differ or without rectangles."""
    from marconet_b200.pipeline import CurvedRegion, curve_lines
    row = np.full(C.LINE_INTS, -1, np.int64)
    row[:8] = 0, 3, 4, 5, 250, 0b1111, 0, 0
    a, b = row.copy(), row.copy()
    for j in range(4):
        a[8 + 2 * j:10 + 2 * j] = 10, 22
        b[8 + 2 * j:10 + 2 * j] = 40, 52
    rect, table = (100, 200, 356, 300), np.stack([a, b])
    level = [(102, 207, 354, 231), (102, 231, 354, 255)]
    lines, curve = curve_lines(rect, 4, table, level)
    assert lines == level and curve["strips"] == 4 and len(curve["samples"]) == 2
    for lv in (None, level[:1], [(102, 207, 354, 221), (102, 231, 354, 255)]):
        lines, _ = curve_lines(rect, 4, table, lv)
        assert len(lines) == 2 and all(isinstance(q, CurvedRegion) for q in lines)
    (top, bottom), (top2, _) = lines
    assert [p[0] for p in top] == [102.0, 186.0, 270.0, 354.0]          # span [xmin - p, xmax + 1 + p], p = (12 + 3) // 4
    assert [p[1] for p in top] == pytest.approx([207.0] * 4) and [p[1] for p in bottom] == pytest.approx([225.0] * 4)
    assert [p[1] for p in top2] == pytest.approx([237.0] * 4)
    a[8 + 2 * 3:10 + 2 * 3] = 14, 26                    # the upper line bends down toward the lower one: its pad is cut
    (top, bottom), (top2, _) = curve_lines(rect, 4, np.stack([a, b]))[0]
    assert max(p[1] for p in bottom) <= min(p[1] for p in top2) + 1e-9
