"""Skewed text blocks (DESIGN.md section 7b, "Skewed blocks") on the host: the twin's angle estimate and lines on pages drawn
with cv2.putText and rotated with cv2.warpAffine, the vertical sign convention, the level cases that must give skew=None's
rectangles, the theta = 0 frame, and every validation error of find_lines and restore_regions, raised before any launch."""
import math

import cv2
import numpy as np
import pytest
import torch

from oracle import blocks as B
from oracle import skewed_blocks as S

TEXTS = ["The quick brown fox jumps over dogs", "Sphinx of black quartz, judge my vow", "Pack my box with five dozen jugs",
         "How vexingly quick daft zebras jump", "Hershey fonts need no download 0123", "Bright vixens jump; dozy fowl quack"]


def rotated_page(n_lines, angle, seed, margin=150):
    """A page of n_lines dark lines 36 pixels apart, about 560 pixels wide, rotated by ``angle`` degrees counter-clockwise about
    its centre on a white canvas.  Returns the image and one boolean ink mask per line, rotated alike."""
    rng = np.random.default_rng(seed)
    h, w = 30 + 36 * n_lines + 2 * margin, 580 + 2 * margin
    masks = []
    for k in range(n_lines):
        m = np.zeros((h, w), np.uint8)
        cv2.putText(m, TEXTS[(k + seed) % len(TEXTS)], (margin + 8, margin + 36 + 36 * k), cv2.FONT_HERSHEY_SIMPLEX, 0.7, 255, 2,
                    cv2.LINE_8)
        masks.append(m)
    rot = cv2.getRotationMatrix2D((w / 2, h / 2), angle, 1.0)
    ink = np.zeros((h, w), np.uint8)
    for m in masks:
        ink |= m
    page = np.empty((h, w, 3), np.uint8)
    page[:] = rng.integers(205, 256, 3)
    page[ink > 0] = rng.integers(0, 50, 3)
    page = cv2.warpAffine(page, rot, (w, h), flags=cv2.INTER_LINEAR, borderValue=tuple(int(v) for v in page[0, 0]))
    return page, [cv2.warpAffine(m, rot, (w, h), flags=cv2.INTER_NEAREST) > 0 for m in masks]


def inside(q, shape, grow=0.0):
    """Pixels of an image of ``shape`` whose centres lie in the parallelogram q = (tl, tr, bl), widened by ``grow`` pixels on
    every side (narrowed for grow < 0)."""
    (tx, ty), (rx, ry), (lx, ly) = q
    ex, ey, fx, fy = rx - tx, ry - ty, lx - tx, ly - ty
    d = ex * fy - ey * fx
    ys, xs = np.mgrid[:shape[0], :shape[1]] + 0.5
    px, py = xs - tx, ys - ty
    a, b = (px * fy - py * fx) / d, (ex * py - ey * px) / d
    ga, gb = grow / math.hypot(ex, ey), grow / math.hypot(fx, fy)
    return (a >= -ga) & (a <= 1 + ga) & (b >= -gb) & (b <= 1 + gb)


def _check_lines(lines, masks, ink, shape):
    """Each line's ink (its mask where the block's threshold finds ink) lies inside its own region and outside the others'.  A
    frame bin takes the pixel centres in [k, k + 1) past the least corner's while the region's edges sit at k - 1/2 (so that
    the level frame gives the rectangles), so a centre may lie up to half a pixel beyond its line's edge: the check allows
    that half pixel, and no more."""
    for k, m in enumerate(masks):
        mk = m & ink
        assert mk.any(), k
        assert not (mk & ~inside(lines[k], shape, 0.5)).any(), f"line {k} leaves its region"
        for j, q in enumerate(lines):
            if j != k:
                assert not (mk & inside(q, shape, -0.5)).any(), f"line {k}'s ink is inside line {j}'s region"


def _ink(page):
    g = B.grey(page)
    t = B.otsu(g)
    return g <= t


CASES = [(1, 3.7), (2, -0.5), (3, 0.5), (5, -6.25), (8, 1.0), (8, -2.5), (12, 1.0), (12, 2.5), (12, -4.0), (12, 7.0),
         (12, -9.5), (6, 14.0), (4, -14.0), (10, 11.3)]


@pytest.mark.parametrize("n_lines,angle", CASES)
def test_twin_finds_the_angle_and_the_lines(n_lines, angle):
    page, masks = rotated_page(n_lines, angle, seed=n_lines)
    H, W = page.shape[:2]
    res = S.find_lines(page, (0, 0, W, H), skew="auto", max_skew=15)
    assert abs(res["skew"] - angle) <= 0.2, (res["skew"], angle)
    assert len(res["lines"]) == n_lines
    assert res["skew"] == res["detail"]["i"][res["detail"]["chosen"]] / 20
    _check_lines(res["lines"], masks, _ink(page), (H, W))


@pytest.mark.parametrize("n_lines,angle", [(3, 4.0), (8, -2.5), (12, 9.5), (5, -12.0)])
def test_vertical_blocks_use_the_same_convention(n_lines, angle):
    """Columns: the rotated page transposed.  The columns of the transposed page lean by -angle counter-clockwise on screen,
    and the block's lines are VerticalRegion-ordered corners (across, then down), right to left."""
    page, masks = rotated_page(n_lines, angle, seed=n_lines + 1)
    tp = np.ascontiguousarray(page.transpose(1, 0, 2))
    H, W = tp.shape[:2]
    res = S.find_lines(tp, (0, 0, W, H), direction="vertical", skew="auto", max_skew=15)
    assert abs(res["skew"] + angle) <= 0.2, (res["skew"], angle)
    assert len(res["lines"]) == n_lines
    hor = S.find_lines(page, (0, 0, page.shape[1], page.shape[0]), skew="auto", max_skew=15)
    assert res["skew"] == -hor["skew"] and res["detail"]["frame_lines"] == hor["detail"]["frame_lines"]
    tmasks = [m.T for m in masks][::-1]
    _check_lines(res["lines"], tmasks, _ink(tp), (H, W))
    for tl, tr, bl in res["lines"]:                   # tl -> tr across the column (right), tl -> bl down it
        assert (tr[0] - tl[0]) * (bl[1] - tl[1]) - (tr[1] - tl[1]) * (bl[0] - tl[0]) > 0
        assert abs(bl[1] - tl[1]) > abs(bl[0] - tl[0])


def test_given_angle_is_used_and_negated_for_a_vertical_block():
    page, masks = rotated_page(5, 3.0, seed=9)
    H, W = page.shape[:2]
    res = S.find_lines(page, (0, 0, W, H), skew=3.0)
    assert res["skew"] == 3.0 and res["detail"]["scores"] is None and len(res["lines"]) == 5
    _check_lines(res["lines"], masks, _ink(page), (H, W))
    tp = np.ascontiguousarray(page.transpose(1, 0, 2))
    v = S.find_lines(tp, (0, 0, H, W), direction="vertical", skew=-3.0)
    assert v["skew"] == -3.0 and v["detail"]["frame_lines"] == res["detail"]["frame_lines"]


def _level_page(n_lines, seed):
    page, _ = rotated_page(n_lines, 0.0, seed, margin=20)
    return page


@pytest.mark.parametrize("direction", ["horizontal", "vertical"])
def test_level_blocks_give_the_rectangles_of_skew_none(direction):
    """skew=0 and a level page under "auto" (chosen angle exactly 0) return skew=None's rectangles exactly."""
    page = _level_page(6, 3)
    if direction == "vertical":
        page = np.ascontiguousarray(page.transpose(1, 0, 2))
    H, W = page.shape[:2]
    rect = (5, 3, W - 4, H - 2)
    ref = B.find_lines(page, rect, direction)
    assert len(ref["lines"]) == 6
    for kw in (dict(skew=0), dict(skew=-0.0), dict(skew="auto"), dict(skew="auto", max_skew=20)):
        res = S.find_lines(page, rect, direction, **kw)
        assert res["skew"] == 0 and res["lines"] == ref["lines"], kw
        assert (res["threshold"], res["ink"]) == (ref["threshold"], ref["ink"])


def test_frame_at_zero_is_rows_and_columns():
    for h, w in ((1, 1), (7, 13), (40, 3), (32767, 9)):
        u_min, v_min, L, M = S.frame(h, w, np.array([1.0]), np.array([0.0]))
        assert (int(L[0]), int(M[0])) == (h, w)
        ys, xs = np.mgrid[:h, :w]
        u, v = S._uv(ys.astype(np.float64), xs.astype(np.float64), h, w, 1.0, 0.0)
        np.testing.assert_array_equal(np.floor(v - v_min[0]), ys)
        np.testing.assert_array_equal(np.floor(u - u_min[0]), xs)


def test_angle_table_and_frame_bounds():
    tab = S.angles("auto", 10.0)
    assert len(tab) == 401 and tab[0] == (-200, -10.0) and tab[200] == (0, 0.0) and tab[-1] == (200, 10.0)
    assert len(S.angles("auto", 0.01)) == 1 and S.angles(2.5) == [(0, 2.5)]
    from marconet_b200 import ops
    assert ops.skew_table("auto", 10.0, True) == [t for _, t in tab] and ops.skew_table(2.5, 10.0, True) == [-2.5]
    cs = ops.skew_cos_sin([t for _, t in tab])
    c, s = np.array([p[0] for p in cs]), np.array([p[1] for p in cs])
    for h, w in ((1, 1), (90, 560), (32767, 9)):
        _, _, L, M = S.frame(h, w, c, s)
        assert ops.skew_stride(w, h, False, cs) == int(L.max())
        assert ops.skew_stride(h, w, True, cs) == int(L.max())
        assert L.min() >= 1 and M.min() >= 1


def test_uniform_block_picks_zero_and_has_no_lines():
    img = np.full((60, 90, 3), 141, np.uint8)
    res = S.find_lines(img, (0, 0, 90, 60), skew="auto")
    assert res["lines"] == [] and res["skew"] == 0.0 and res["detail"]["i"][res["detail"]["chosen"]] == 0
    assert set(res["detail"]["scores"]) == {0}
    one = S.find_lines(img, (4, 5, 5, 6), direction="vertical", skew="auto", max_skew=20)
    assert one["lines"] == [] and one["skew"] == 0.0


def test_tie_rule():
    assert S.choose([-2, -1, 0, 1, 2], [5, 5, 3, 5, 5]) == 1
    assert S.choose([-2, -1, 0, 1, 2], [5, 4, 3, 4, 5]) == 0
    assert S.choose([-1, 0, 1], [0, 0, 0]) == 1


BAD = [
    (dict(skew="Auto"), "skew must be None, 'auto' or a finite angle"),
    (dict(skew=45), "skew must be None"),
    (dict(skew=-45.0), "skew must be None"),
    (dict(skew=float("nan")), "skew must be None"),
    (dict(skew=float("inf")), "skew must be None"),
    (dict(skew=True), "skew must be None"),
    (dict(skew=(1, 2)), "skew must be None"),
    (dict(skew="auto", max_skew=0), "max_skew must be a number of degrees in \\(0, 20\\]"),
    (dict(skew="auto", max_skew=20.5), "max_skew must be"),
    (dict(skew="auto", max_skew=float("nan")), "max_skew must be"),
    (dict(skew="auto", max_skew="5"), "max_skew must be"),
    (dict(skew=None, max_skew=5), "max_skew is given, but skew is None"),
    (dict(skew=3.0, max_skew=15), "max_skew is given, but skew is 3.0"),
]


@pytest.mark.parametrize("kw,msg", BAD)
def test_find_lines_rejects_bad_skew_before_any_launch(kw, msg):
    from marconet_b200 import pipeline
    img = np.zeros((30, 40, 3), np.uint8)
    blk = pipeline.TextBlock((0, 0, 40, 30), **kw)
    with pytest.raises(ValueError, match=f"image 1, block 1: .*{msg}"):
        pipeline.find_lines([img, img], [[], [pipeline.TextBlock((0, 0, 4, 4), skew="auto"), blk]])


@pytest.mark.parametrize("kw,msg", BAD)
def test_restore_regions_rejects_bad_skew_before_any_launch(kw, msg):
    from marconet_b200 import pipeline
    img = np.zeros((30, 40, 3), np.uint8)
    blk = pipeline.TextBlock((0, 0, 40, 30), **kw)
    with pytest.raises(ValueError, match=f"image 0, region 1 \\(a text block\\): .*{msg}"):
        pipeline.restore_regions(None, None, None, [img], [[pipeline.TextBlock((0, 0, 4, 4), skew=2), blk]])


def test_profile_limit_is_checked_before_any_launch():
    """A 20000 x 20000 block searched over +-20 degrees needs 801 x about 25630 profile bins, over the stated limit; +-10 degrees
    fits.  The image is a broadcast view: validation reads its shape only."""
    from marconet_b200 import ops, pipeline
    img = torch.zeros(1, 1, 3, dtype=torch.uint8).expand(20000, 20000, 3)
    blk = pipeline.TextBlock((0, 0, 20000, 20000), skew="auto", max_skew=20)
    with pytest.raises(ValueError, match="image 0, block 0: the angle search needs 801 angles x 2563\\d bins"):
        pipeline.find_lines([img], [[blk]])
    with pytest.raises(ValueError, match="image 0, region 0 \\(a text block\\): the angle search needs"):
        pipeline.restore_regions(None, None, None, [img], [[blk]])
    cs = ops.skew_cos_sin(ops.skew_table("auto", 10.0, False))
    assert len(cs) * ops.skew_stride(20000, 20000, False, cs) <= ops.SKEW_MAX_PROFILE
    assert math.isclose(ops.skew_stride(20000, 20000, False, ops.skew_cos_sin([20.0])),
                        20000 * (math.sin(math.radians(20)) + math.cos(math.radians(20))), abs_tol=2)


def test_skew_lines_equal_the_twins_corners():
    """pipeline.skew_lines converts frame lines exactly as the twin does, horizontal and vertical."""
    from marconet_b200 import pipeline
    page, _ = rotated_page(4, -5.5, seed=4)
    H, W = page.shape[:2]
    for direction, img in (("horizontal", page), ("vertical", np.ascontiguousarray(page.transpose(1, 0, 2)))):
        rect = (3, 2, img.shape[1] - 1, img.shape[0] - 5)
        res = S.find_lines(img, rect, direction, skew="auto")
        d = res["detail"]
        p = d["chosen"]
        lines = pipeline.skew_lines(rect, direction == "vertical", float(d["c"][p]), float(d["s"][p]), d["frame"][0],
                                    d["frame"][1], d["frame_lines"])
        if direction == "vertical":
            assert [tuple(q.shape) for q in lines] == [tuple(q) for q in res["lines"]]
        else:
            assert [tuple(q) for q in lines] == [tuple(q) for q in res["lines"]]
        assert len(lines) == 4
