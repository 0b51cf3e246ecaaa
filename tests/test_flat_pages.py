"""Flat pages (DESIGN.md section 7b, "Flat pages") on the host: the numpy twin against live OpenCV on its own maps, curled pages
(cylinders and S-curves, flat and photographed as an open book at an angle) whose lines come back level after flattening, the
dewarp field's edge cases against hand-computed values, and every refusal of flatten_pages, raised before any launch."""

import cv2
import numpy as np
import pytest

from marconet_b200 import ops
from marconet_b200.pipeline import (CurvedRegion, FlatPage, QuadRegion, TextBlock, TextPage, find_blocks, find_lines,
                                    flat_line_table, flatten_pages, quad_maps, skew_flat_matrix)
from oracle import curled_blocks as CB
from oracle import flat_pages as F
from oracle import pages as P
from oracle import quad_pages as QP

from test_curled_blocks import PITCH, curled_page

cv2.ipp.setUseIPP(False)


def mid_spread(q):
    """How far a traced line's mid curve moves across its span (0 for a rectangle): the spread of its control values, which
    bounds the curve's."""
    if not isinstance(q, CurvedRegion):
        return 0.0
    mu = [0.5 * (t[1] + b[1]) for t, b in zip(q.top, q.bottom)]
    return max(mu) - min(mu)


def level_after(flat, polarity="auto"):
    """Every line of every block of the flat page, traced with curve="auto" by the twin."""
    out = []
    for b in P.find_blocks(flat, None, "horizontal", polarity)["blocks"]:
        r = CB.find_lines(flat, b, polarity=polarity)
        assert "error" not in r
        out += r["lines"]
    return out


def test_twin_remap_equals_cv2_on_its_own_maps():
    page, _, _ = curled_page(6, "cylinder", 30, 1)
    res = F.flatten(page, FlatPage(curve="auto"))
    assert "table" in res
    h, w = page.shape[:2]
    mx, my = F.maps(res["table"], w, h, "rect", (0, 0))
    want = cv2.remap(page, mx.astype(np.float32), my.astype(np.float32), cv2.INTER_CUBIC, borderMode=cv2.BORDER_REPLICATE)
    np.testing.assert_array_equal(res["image"], want)


@pytest.mark.parametrize("theta", [3.5, -7.25, 0.0])
def test_twin_skew_equals_cv2_warp_affine(theta):
    page, _, _ = curled_page(4, "flat", 0, 2)
    rect = (30, 20, page.shape[1] - 40, page.shape[0] - 10)
    res = F.flatten(page, FlatPage(rect, skew=theta))
    c, s = ops.skew_cos_sin([theta])[0]
    m, size = skew_flat_matrix(rect[2] - rect[0], rect[3] - rect[1], c, s)
    crop = np.ascontiguousarray(page[rect[1]:rect[3], rect[0]:rect[2]])
    want = cv2.warpAffine(crop, np.array(m, np.float64), size, flags=cv2.INTER_CUBIC | cv2.WARP_INVERSE_MAP,
                          borderMode=cv2.BORDER_REPLICATE)
    assert res["size"] == size and res["skew"] == theta
    np.testing.assert_array_equal(res["image"], want)
    if theta == 0.0:
        np.testing.assert_array_equal(res["image"], crop)


def test_twin_quad_equals_rectify_and_rect_is_the_crop():
    page, _, _ = curled_page(3, "flat", 0, 3)
    q = QuadRegion((40.0, 30.0), (600.0, 50.0), (590.0, 300.0), (30.0, 280.0))
    res = F.flatten(page, FlatPage(quad=q))
    np.testing.assert_array_equal(res["image"], QP.rectify(page, q))
    assert res["size"] == quad_maps(q, 1).size
    np.testing.assert_array_equal(F.flatten(page, FlatPage((5, 6, 70, 90)))["image"], page[6:90, 5:70])


# S-curves stop at half a pitch, short of the +-2 pitches the cylinders reach: at a full pitch or more the curled-block
# tracer's single cubic per edge does not follow one period of a sine, and the field can only straighten the lines it is given.
@pytest.mark.parametrize("kind,amp", [("cylinder", PITCH), ("cylinder", 2 * PITCH), ("cylinder", -2 * PITCH), ("s", PITCH // 2),
                                      ("s", -PITCH // 2)])
def test_flattened_curled_pages_have_level_lines(kind, amp):
    page, _, _ = curled_page(8, kind, amp, 5)
    before = F.flatten(page, FlatPage(curve="auto"))
    assert max(mid_spread(q) for q in before["lines"]) > abs(amp) / 3
    lines = level_after(before["image"])
    assert len(lines) >= 8
    assert max(mid_spread(q) for q in lines) <= 2.0


def open_book(kind, amp, seed, fore):
    """A curled page warped into a darker photo by a homography that shrinks its right side by ``fore``."""
    page, _, _ = curled_page(8, kind, amp, seed)
    h, w = page.shape[:2]
    H, W = int(h * 1.3), int(w * 1.3)
    m = 0.12
    dst = np.float32([[W * m, H * m], [W * (1 - m), H * (0.5 - (0.5 - m) / fore)], [W * (1 - m), H * (0.5 + (0.5 - m) / fore)],
                      [W * m, H * (1 - m)]])
    hom = cv2.getPerspectiveTransform(np.float32([[0, 0], [w, 0], [w, h], [0, h]]), dst)
    photo = np.full((H, W, 3), 40, np.uint8)
    return cv2.warpPerspective(page, hom, (W, H), dst=photo, flags=cv2.INTER_LINEAR, borderMode=cv2.BORDER_TRANSPARENT)


@pytest.mark.parametrize("kind,amp,fore", [("cylinder", 2 * PITCH, 2.0), ("cylinder", -PITCH, 1.5), ("s", PITCH // 2, 2.0)])
def test_open_book_at_an_angle_flattens_level(kind, amp, fore):
    photo = open_book(kind, amp, 7, fore)
    res = F.flatten(photo, FlatPage(quad="auto", curve="auto"))
    assert res["kind"] == "quad" and "table" in res
    lines = level_after(res["image"])
    assert len(lines) >= 8
    assert max(mid_spread(q) for q in lines) <= 2.0


def _table(*lines):
    """A line table from (xs, xe, mu, block x0, block x1) rows, mu four values, in the given order."""
    rows = [(xs, xe, *mu, sum(mu) / 4, bx0, bx1) for xs, xe, mu, bx0, bx1 in lines]
    return np.array(sorted(rows, key=lambda r: r[6]), np.float64)


def test_field_without_lines_is_the_identity():
    src = F.field(np.zeros((0, 9)), 5, 4)
    np.testing.assert_array_equal(src, np.repeat((np.arange(4) + 0.5)[:, None], 5, axis=1))


def test_field_on_covered_columns_and_margins():
    # one level line at 10 and one at 30 bent by +4 at its right end (linear mu), block [2, 6) of an 8-column frame
    t = _table((2.0, 6.0, (10.0, 10.0, 10.0, 10.0), 2, 6), (2.0, 6.0, (30.0, 32.0, 34.0, 36.0), 2, 6))
    src = F.field(t, 8, 40)
    Y1 = 33.0
    for x in range(2, 6):
        m1 = 30.0 + 6.0 * ((x + 0.5 - 2.0) / 4.0)
        for y in (0, 5, 15, 25, 35, 39):
            yc = y + 0.5
            if yc < 10:
                want = yc
            elif yc >= Y1:
                want = yc + (m1 - Y1)
            else:
                want = 10 + (yc - 10) * (m1 - 10) / (Y1 - 10)
            assert src[y, x] == pytest.approx(want, abs=1e-12)
    np.testing.assert_array_equal(src[:, 0], src[:, 2])          # the left margin: column 2's displacement
    np.testing.assert_array_equal(src[:, 7], src[:, 5])          # the right margin: column 5's


def test_field_gutter_between_side_by_side_blocks():
    # block A [0, 4): one line with mu = (10, 12, 14, 16) over [0, 4], Y = 13; at column 3 (xc = 3.5, t = 0.875) m = 15.25, so
    # d_l = 2.25.  Block B [8, 12): mu = (30, 29, 28, 27) over [8, 12], Y = 28.5; at column 8 (xc = 8.5, t = 0.125) m = 29.625,
    # so d_r = 1.125.  A one-line column moves every row by its d; gutter column x takes 2.25 + (x - 3)(1.125 - 2.25) / 5.
    t = _table((0.0, 4.0, (10.0, 12.0, 14.0, 16.0), 0, 4), (8.0, 12.0, (30.0, 29.0, 28.0, 27.0), 8, 12))
    src = F.field(t, 12, 30)
    yc = np.arange(30) + 0.5
    np.testing.assert_array_equal(src[:, 3], yc + 2.25)
    np.testing.assert_array_equal(src[:, 8], yc + 1.125)
    for x, d in ((4, 2.025), (5, 1.8), (6, 1.575), (7, 1.35)):
        np.testing.assert_allclose(src[:, x], yc + d, rtol=0, atol=1e-12)
    for x, m in ((0, 10.75), (1, 12.25), (2, 13.75), (9, 28.875), (10, 28.125), (11, 27.375)):
        np.testing.assert_array_equal(src[:, x] - yc, m - (13.0 if x < 4 else 28.5))


def test_field_tied_anchors():
    # two lines with the same anchor Y = 20 in one column (side by side in the table): the last with Y <= yc decides
    t = _table((0.0, 4.0, (18.0, 18.0, 22.0, 22.0), 0, 4), (0.0, 4.0, (22.0, 22.0, 18.0, 18.0), 0, 4),
               (0.0, 4.0, (40.0,) * 4, 0, 4))
    assert t[0, 6] == t[1, 6] == 20.0
    src = F.field(t, 4, 50)
    cover, M = F.column_values(t, 4)
    for x in range(4):
        for y in (5, 19, 20, 30, 45):
            yc = y + 0.5
            if yc < 20:
                want = yc + (M[0, x] - 20)
            elif yc >= 40:
                want = yc + (M[2, x] - 40)
            else:
                want = M[1, x] + (yc - 20) * (M[2, x] - M[1, x]) / 20
            assert src[y, x] == want


def test_line_table_order_and_values():
    c1 = CurvedRegion(((10.0, 5.0), (20.0, 6.0), (30.0, 7.0), (40.0, 8.0)), ((10.0, 15.0), (20.0, 16.0), (30.0, 17.0), (40.0, 18.0)))
    t = flat_line_table([((0, 0, 50, 60), [(2, 30, 48, 40), c1])])
    np.testing.assert_array_equal(t[0], [10.0, 40.0, 10.0, 11.0, 12.0, 13.0, 11.5, 0.0, 50.0])
    np.testing.assert_array_equal(t[1], [2.0, 48.0, 35.0, 35.0, 35.0, 35.0, 35.0, 0.0, 50.0])


def test_level_page_under_auto_gives_the_bytes_of_no_curve():
    page, _, _ = curled_page(4, "flat", 0, 9)
    a, b = F.flatten(page, FlatPage(curve="auto")), F.flatten(page, FlatPage())
    assert "table" not in a and all(not isinstance(q, CurvedRegion) for q in a["lines"])
    np.testing.assert_array_equal(a["image"], b["image"])


BAD = [
    (FlatPage(curve="auto", skew=3.0), "curve and skew"),
    (FlatPage(curve="auto", skew="auto"), "curve and skew"),
    (FlatPage(curve="auto", direction="vertical"), "vertical"),
    (FlatPage(quad=QuadRegion((1.0, 1.0), (50.0, 1.0), (50.0, 40.0), (1.0, 40.0)), skew=2.0), "skew and quad"),
    (FlatPage(quad="auto", skew="auto"), "skew and quad"),
    (FlatPage(strips=4), "strips"),
    (FlatPage(curve="auto", strips=0), "strips"),
    (FlatPage(curve="maybe"), "curve"),
    (FlatPage((0, 0, 500, 10)), "outside"),
    (FlatPage(rect=(1, 2, 3)), "integer rectangle"),
    (FlatPage(skew=50.0), "skew"),
]


@pytest.mark.parametrize("fp,what", BAD)
def test_refusals_before_any_launch(fp, what):
    img = np.zeros((60, 80, 3), np.uint8)
    n = ops.LAUNCHES
    with pytest.raises(ValueError, match=f"image 1, page 1: .*{what}"):
        flatten_pages([img, img], [[], [FlatPage(), fp]])
    assert ops.LAUNCHES == n


def test_frame_side_and_work_refusals():
    wide = np.zeros((1000, 32767, 3), np.uint8)
    n = ops.LAUNCHES
    with pytest.raises(ValueError, match="image 0, page 0: .*frame reaches 3278"):
        flatten_pages([wide], [[FlatPage(skew=2.0)]])
    with pytest.raises(ValueError, match="image 0, page 0: .*frame reaches"):
        flatten_pages([wide], [[FlatPage(skew="auto", max_skew=2.0)]])
    tall = np.zeros((40000, 1000, 3), np.uint8)
    with pytest.raises(ValueError, match="image 0, page 0: a curled page is resampled from the whole 1000x40000 image"):
        flatten_pages([tall], [[FlatPage((0, 0, 1000, 1000), curve="auto")]])
    big = np.zeros((16000, 16000, 3), np.uint8)
    with pytest.raises(ValueError, match="image 0, page 2: the call's flat pages .*work memory"):
        flatten_pages([big], [[FlatPage()] * 3])
    assert ops.LAUNCHES == n
    with pytest.raises(ValueError, match="expected a FlatPage"):
        flatten_pages([wide], [[TextPage()]])


def test_text_page_and_block_still_refuse_curve_with_quad():
    img = np.zeros((60, 80, 3), np.uint8)
    q = QuadRegion((1.0, 1.0), (50.0, 1.0), (50.0, 40.0), (1.0, 40.0))
    with pytest.raises(ValueError, match="curve and quad"):
        find_blocks([img], [[TextPage(quad=q, curve="auto")]])
    with pytest.raises(ValueError, match="curve and quad"):
        find_lines([img], [[TextBlock.from_quad(q, curve="auto")]])


def test_column_cap_is_refused_before_the_launch():
    import torch
    lines = np.array([(0.0, 4.0, *(10.0 * k,) * 4, 10.0 * k, 0.0, 4.0) for k in range(ops.FLAT_MAX_COLUMN_LINES + 1)])
    assert ops.flat_column_lines(lines[:-1], 4) == ops.FLAT_MAX_COLUMN_LINES
    img = torch.zeros(8, 8, 3, dtype=torch.uint8)
    n = ops.LAUNCHES
    with pytest.raises(ValueError, match=f"flat_remap: page 0: a column meets {ops.FLAT_MAX_COLUMN_LINES + 1} lines"):
        ops.flat_remap([(img, img[:4, :4], "rect", (0, 0), lines)])
    assert ops.LAUNCHES == n
