"""Book spreads (DESIGN.md section 7b, "Book spreads") on the host: the numpy twin's spine on hand-made masks (exact points, ties,
the ends of the search range, the depth test at its limit), on generated spreads of two curled pages photographed at an angle
(spine within tolerance, level lines after flattening each half, each half's lines, the reading order), and every refusal of
FlatPage(spread=...), raised before any launch."""
import math

import cv2
import numpy as np
import pytest

from marconet_b200 import ops
from marconet_b200.pipeline import CurvedRegion, FlatPage, QuadRegion, flatten_pages
from oracle import quad_pages as QP
from oracle import spread_pages as SP

from test_curled_blocks import curled_page
from test_flat_pages import level_after, mid_spread

cv2.ipp.setUseIPP(False)


def book_spread(n, m, a, p, fore, seed, light=False):
    """An open book: a page of n lines and one of m lines (test_curled_blocks.curled_page, level) side by side, each column x
    scaled vertically about the centre row by s(x) = 1 - a (1 - |x - x_s| / half)^p, x_s the spine, which cuts a notch of a h / 2
    into the top and the bottom edge and bows the lines towards the spine; then warped into a darker photo by a homography
    that shrinks the right side by ``fore``, as test_flat_pages.open_book.  Returns the photo and the true spine points
    (x, y) at the top and bottom of the paper."""
    pages = [curled_page(k, "flat", 0, seed + j, light=light)[0] for j, k in enumerate((n, m))]
    h = max(pg.shape[0] for pg in pages)
    pages = [np.concatenate([pg, np.repeat(pg[-1:], h - pg.shape[0], axis=0)]) for pg in pages]
    book = np.hstack(pages)
    half = pages[0].shape[1]
    w = 2 * half
    cy = h / 2
    xc = np.arange(w, dtype=np.float64) + 0.5
    s = 1 - a * (1 - np.abs(xc - half) / half) ** p
    yc = np.arange(h, dtype=np.float64)[:, None] + 0.5
    mapy = (cy + (yc - cy) / s[None, :] - 0.5).astype(np.float32)
    mapx = np.repeat((xc - 0.5)[None, :].astype(np.float32), h, axis=0)
    bg = 255 - 40 if light else 40
    book = cv2.remap(book, mapx, mapy, cv2.INTER_LINEAR, borderMode=cv2.BORDER_CONSTANT, borderValue=(bg, bg, bg))
    H, W = int(h * 1.3), int(w * 1.3)
    mg = 0.12
    dst = np.float32([[W * mg, H * mg], [W * (1 - mg), H * (0.5 - (0.5 - mg) / fore)], [W * (1 - mg), H * (0.5 + (0.5 - mg) / fore)],
                      [W * mg, H * (1 - mg)]])
    hom = cv2.getPerspectiveTransform(np.float32([[0, 0], [w, 0], [w, h], [0, h]]), dst)
    photo = np.full((H, W, 3), bg, np.uint8)
    photo = cv2.warpPerspective(book, hom, (W, H), dst=photo, flags=cv2.INTER_LINEAR, borderMode=cv2.BORDER_TRANSPARENT)
    ends = cv2.perspectiveTransform(np.float64([[[half, cy - (1 - a) * cy], [half, cy + (1 - a) * cy]]]), hom)[0]
    return photo, [tuple(float(v) for v in e) for e in ends]


def notched(w, h, top=(), bottom=(), pad=6):
    """A w x h rectangle of paper (True) at (pad, pad) in a mask with ``pad`` columns and rows around it, with notches cut into its
    top and bottom edges: each (c, d, k) a V of depth d at column c whose flanks fall by k rows per column (k = 0: a slot one
    column wide).  Columns in rectangle coordinates."""
    mask = np.zeros((h + 2 * pad, w + 2 * pad), bool)
    mask[pad:pad + h, pad:pad + w] = True
    x = np.arange(w)
    for edge, notches in ((0, top), (1, bottom)):
        cut = np.zeros(w, np.int64)
        for c, d, k in notches:
            depth = np.where(x == c, d, 0) if k == 0 else np.maximum(0, d - k * np.abs(x - c))
            cut = np.maximum(cut, depth)
        for xx in range(w):
            if cut[xx]:
                if edge == 0:
                    mask[pad:pad + cut[xx], pad + xx] = False
                else:
                    mask[pad + h - cut[xx]:pad + h, pad + xx] = False
    return mask


def flat_notch(mask, edge, c0, c1, d, pad=6):
    """``mask`` with a notch of depth d over rectangle columns [c0, c1) cut into its top (edge 0) or bottom (edge 1) edge."""
    mask = mask.copy()
    h = mask.shape[0] - 2 * pad
    if edge == 0:
        mask[pad:pad + d, pad + c0:pad + c1] = False
    else:
        mask[pad + h - d:pad + h, pad + c0:pad + c1] = False
    return mask


def text_rows(lines):
    """The number of text rows among traced lines (rectangles or CurvedRegions): their row spans merged where they overlap,
    since the page's blocks may cut one row into words."""
    spans = sorted((min(p[1] for p in q.top), max(p[1] for p in q.bottom)) if isinstance(q, CurvedRegion) else (q[1], q[3])
                   for q in lines)
    rows, end = 0, -math.inf
    for y0, y1 in spans:
        if y0 >= end:
            rows += 1
        end = max(end, y1) if y0 < end else y1
    return rows


def rect_quad(w, h, pad=6):
    return [(pad, pad), (pad + w, pad), (pad + w, pad + h), (pad, pad + h)]


def mask_image(mask):
    """The mask as a photo: paper 230, the rest 20."""
    return np.repeat(np.where(mask, 230, 20).astype(np.uint8)[:, :, None], 3, axis=2)


def test_column_extents_and_corners_of_a_notched_rectangle():
    mask = notched(120, 60, top=[(60, 8, 1)], bottom=[(50, 5, 2)])
    t, b = SP.column_extents(mask)
    assert t[0] == -1 and b[0] == -1 and t[6] == 6 and b[6] == 66
    assert t[6 + 60] == 6 + 8 and t[6 + 61] == 6 + 7 and b[6 + 50] == 66 - 5 and b[6 + 51] == 66 - 3
    res = QP.find_corners(mask_image(mask))
    assert [tuple(p) for p in res["quad"]] == rect_quad(120, 60)


@pytest.mark.parametrize("w,h,ct,dt,cb,db", [(120, 60, 60, 8, 50, 5), (400, 200, 150, 30, 250, 12), (64, 40, 16, 3, 48, 2)])
def test_exact_spine_points(w, h, ct, dt, cb, db):
    mask = notched(w, h, top=[(ct, dt, 1)], bottom=[(cb, db, 1)])
    sp = SP.spine(mask, rect_quad(w, h))
    assert sp["st"] == (6 + ct, 6 + dt) and sp["sb"] == (6 + cb, 6 + h - db)
    assert sp["D"] == w * dt and sp["E"] == w * db
    assert sp["found"] == (dt >= max(2, w / 100) and db >= max(2, w / 100))
    assert SP.find_spine(mask_image(mask))["spine"] == sp


def test_ties_go_to_the_smallest_column():
    mask = flat_notch(flat_notch(notched(200, 80), 0, 90, 97, 9), 1, 70, 130, 4)
    sp = SP.spine(mask, rect_quad(200, 80))
    assert sp["st"] == (6 + 90, 6 + 9) and sp["sb"] == (6 + 70, 6 + 80 - 4) and sp["found"]


def test_range_ends_and_a_deeper_notch_outside_them():
    # w = 202: the middle half is 4 x >= 202 and 4 (202 - x) >= 202, columns 51 .. 151 of the rectangle
    w, h = 202, 90
    lo, hi = 51, 151
    assert 4 * lo >= w > 4 * (lo - 1) and 4 * (w - hi) >= w > 4 * (w - hi - 1)
    for out, at in ((lo - 1, lo), (hi + 1, hi)):
        mask = notched(w, h, top=[(out, 40, 0), (at, 20, 0), (100, 10, 1)], bottom=[(out, 30, 0), (101, 6, 1)])
        sp = SP.spine(mask, rect_quad(w, h))
        assert sp["st"] == (6 + at, 6 + 20) and sp["sb"] == (6 + 101, 6 + h - 6) and sp["found"]
    mask = notched(w, h, top=[(lo - 1, 40, 0), (100, 10, 1)], bottom=[(hi + 1, 30, 0), (101, 6, 1)])
    sp = SP.spine(mask, rect_quad(w, h))
    assert sp["st"] == (6 + 100, 16) and sp["sb"] == (6 + 101, 6 + h - 6)


@pytest.mark.parametrize("w,need", [(150, 2), (199, 2), (200, 2), (500, 5), (1000, 10), (1234, 13)])
def test_depth_limit(w, need):
    """max(2, L / 100): d = need is accepted and need - 1 refused, on the top and on the bottom edge."""
    assert need == max(2, math.ceil(w / 100))
    quad = rect_quad(w, 60)
    for dt, db, ok in ((need, need, True), (need - 1, need, False), (need, need - 1, False)):
        mask = notched(w, 60, top=[(w // 2, dt, 1)], bottom=[(w // 2 + 3, db, 1)])
        sp = SP.spine(mask, quad)
        assert sp["D"] == w * dt and sp["E"] == w * db and sp["found"] == ok, (dt, db)


def test_no_notch_and_degenerate_edges():
    sp = SP.spine(notched(300, 100), rect_quad(300, 100))
    assert not sp["found"] and sp["D"] == 0 and sp["E"] == 0 and sp["st"] == (6 + 75, 6)
    assert SP.deep_enough(2 * 150, (0, 0), (150, 0)) and not SP.deep_enough(2 * 150 - 1, (0, 0), (150, 0))
    assert not SP.deep_enough(0, (0, 0), (0, 0))


SPREADS = [(8, 6, 0.10, 1.0, 1.5, 1), (6, 8, 0.12, 2.0, 1.8, 2), (7, 5, 0.08, 3.0, 1.3, 3), (5, 7, 0.15, 1.5, 2.0, 4)]


@pytest.mark.parametrize("n,m,a,p,fore,seed", SPREADS)
def test_twin_finds_the_spine_of_a_generated_spread(n, m, a, p, fore, seed):
    photo, (top, bot) = book_spread(n, m, a, p, fore, seed)
    res = SP.find_spine(photo)
    sp = res["spine"]
    tol = max(3, photo.shape[1] / 100)
    assert sp["found"]
    assert abs(sp["st"][0] - top[0]) <= tol and abs(sp["sb"][0] - bot[0]) <= tol, (sp, top, bot)
    assert abs(sp["st"][1] - top[1]) <= tol and abs(sp["sb"][1] - bot[1]) <= tol, (sp, top, bot)


@pytest.mark.parametrize("n,m,a,p,fore,seed", SPREADS[:3])
def test_each_half_flattens_level_with_its_own_lines(n, m, a, p, fore, seed):
    photo, _ = book_spread(n, m, a, p, fore, seed)
    res = SP.flatten(photo, FlatPage(quad="auto", spread="auto", curve="auto"))
    assert res["kind"] == "spread" and [pg["side"] for pg in res["pages"]] == ["left", "right"]
    for pg, k in zip(res["pages"], (n, m)):
        assert pg["kind"] == "quad"
        lines = level_after(pg["image"])
        assert text_rows(lines) == k
        assert max(mid_spread(q) for q in lines) <= 2.0
    left, right = (pg["quad"] for pg in res["pages"])
    assert left[1] == right[0] and left[2] == right[3]            # the halves meet at the spine
    assert left[0] == res["quad"][0] and right[1] == res["quad"][1] and right[2] == res["quad"][2] and left[3] == res["quad"][3]
    assert res["spine"] == (tuple(int(v) for v in left[1]), tuple(int(v) for v in left[2]))


def test_vertical_spreads_are_read_right_to_left():
    photo, _ = book_spread(6, 4, 0.12, 1.0, 1.5, 5)
    h = SP.flatten(photo, FlatPage(quad="auto", spread="auto"))
    v = SP.flatten(photo, FlatPage(quad="auto", spread="auto", direction="vertical"))
    assert [pg["side"] for pg in v["pages"]] == ["right", "left"]
    for a, b in zip(h["pages"], v["pages"][::-1]):
        np.testing.assert_array_equal(a["image"], b["image"])
        assert a["quad"] == b["quad"]
    assert h["spine"] == v["spine"] and h["depth"] == v["depth"]


def test_a_photo_without_a_notch_is_no_spread():
    photo, _ = book_spread(6, 6, 0.0, 1.0, 1.5, 6)
    assert not SP.find_spine(photo)["spine"]["found"]
    with pytest.raises(ValueError, match="no spread found"):
        SP.flatten(photo, FlatPage(quad="auto", spread="auto"))


Q = QuadRegion((1.0, 1.0), (50.0, 1.0), (50.0, 40.0), (1.0, 40.0))
BAD = [
    (FlatPage(quad="auto", spread="yes"), "spread must be None or 'auto'"),
    (FlatPage(quad="auto", spread=True), "spread must be None or 'auto'"),
    (FlatPage(spread="auto"), "spread='auto' needs quad='auto'"),
    (FlatPage(quad=Q, spread="auto"), "spread='auto' needs quad='auto'"),
    (FlatPage((0, 0, 40, 30), quad="auto", spread="auto"), "spread and rect"),
    (FlatPage(quad="auto", skew=2.0, spread="auto"), "spread and skew"),
    (FlatPage(quad="auto", skew="auto", spread="auto"), "spread and skew"),
    (FlatPage(quad="auto", spread="auto", curve="auto", direction="vertical"), "curve is given for a vertical page"),
    (FlatPage(quad="auto", spread="auto", light="dim"), "light must be"),
]


@pytest.mark.parametrize("fp,what", BAD)
def test_refusals_before_any_launch(fp, what):
    img = np.zeros((60, 80, 3), np.uint8)
    n = ops.LAUNCHES
    with pytest.raises(ValueError, match=f"image 1, page 1: .*{what}"):
        flatten_pages([img, img], [[], [FlatPage(), fp]])
    assert ops.LAUNCHES == n


def test_spine_memory_is_counted_in_the_work_limit():
    assert ops.spine_page_bytes(32767) >= 8 * 32767
    w = 32767
    # sized so that the corner search of the image fits the page search's limit only without the spine's columns
    base = ops.quad_page_bytes(w, 1)
    per_row = ops.quad_page_bytes(w, 2) - base
    rows = (ops.PAGE_MAX_WORK - base) // per_row + 1
    while ops.quad_page_bytes(w, rows) > ops.PAGE_MAX_WORK:
        rows -= 1
    assert ops.quad_page_bytes(w, rows) + ops.spine_page_bytes(w) > ops.PAGE_MAX_WORK
    img = np.zeros((rows, w, 3), np.uint8)
    n = ops.LAUNCHES
    with pytest.raises(ValueError, match="work memory"):
        flatten_pages([img], [[FlatPage(quad="auto", spread="auto")]])
    assert ops.LAUNCHES == n
