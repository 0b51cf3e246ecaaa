"""Perspective pages and blocks (DESIGN.md section 7b, "Perspective pages") on the host: the twin on photographed `putText` pages
of a heading over columns, the reduction of a rectangle quad to the level page and block, every validation error of
find_blocks, find_lines and restore_regions (raised before anything reaches a device), and the build of the new kernels."""
import os
import re
import subprocess

import cv2
import numpy as np
import pytest

from marconet_b200 import ops, pipeline
from oracle import blocks as B
from oracle import pages as P
from oracle import quad_pages as Q
from oracle.quad_regions import rectify

from test_skewed_pages import drawn_page


def photo(widths, n_lines, corners, seed, misalign=False, vertical=False, light=False):
    """A drawn page (test_skewed_pages.drawn_page, level) warped by cv2.warpPerspective so that its corners land on ``corners``
    (tl, tr, br, bl in continuous image coordinates), over a background 90-130 grey levels darker with noise, on a canvas 220
    pixels wider and taller than the corners' box.  ``light`` inverts the page and the background (light ink on a dark page,
    over a lighter background).  Returns the image and the warped ink masks, as drawn_page's."""
    rng = np.random.default_rng(seed)
    flat, masks = drawn_page(widths, n_lines, 0.0, seed, misalign, vertical)
    h, w = flat.shape[:2]
    c = np.float32(corners)
    Wc, Hc = int(c[:, 0].max()) + 110, int(c[:, 1].max()) + 110
    src = np.float32([[0, 0], [w, 0], [w, h], [0, h]]) - 0.5
    M = cv2.getPerspectiveTransform(src, c - 0.5)
    page = cv2.warpPerspective(flat, M, (Wc, Hc), flags=cv2.INTER_LINEAR)
    cover = cv2.warpPerspective(np.full((h, w), 255, np.uint8), M, (Wc, Hc), flags=cv2.INTER_NEAREST) > 0
    bg = cv2.GaussianBlur(rng.integers(100, 140, (Hc, Wc)).astype(np.uint8), (5, 5), 0)[..., None].repeat(3, axis=2)
    img = np.where(cover[..., None], page, bg).astype(np.int16) + rng.integers(-6, 7, (Hc, Wc, 1))
    img = np.clip(img, 0, 255).astype(np.uint8)
    if light:
        img = 255 - img
    warp = lambda m: cv2.warpPerspective(m.astype(np.uint8), M, (Wc, Hc), flags=cv2.INTER_NEAREST) > 0
    return img, [warp(masks[0])] + [[warp(m) for m in col] for col in masks[1:]]


def inside(quad, shape, grow):
    """Pixels whose centre lies inside the convex quad tl, tr, br, bl (clockwise on screen) grown by ``grow`` pixels."""
    ys, xs = np.mgrid[0:shape[0], 0:shape[1]] + 0.5
    out = np.ones(shape, bool)
    for k in range(4):
        (ax, ay), (bx, by) = quad[k], quad[(k + 1) % 4]
        n = np.hypot(bx - ax, by - ay)
        out &= ((bx - ax) * (ys - ay) - (by - ay) * (xs - ax)) / n >= -grow
    return out


def corners_of(w, h, x0, y0, pull):
    """The corners of a w x h page placed at (x0, y0) and foreshortened: ``pull`` (dx_top, dx_bottom, dy_left, dy_right) moves
    the top corners inwards by dx_top each, and so on."""
    t, b, l, r = pull
    return [(x0 + t, y0 + l), (x0 + w - t, y0 + r), (x0 + w - b, y0 + h - r), (x0 + b, y0 + h - l)]


def _check_photo(img, masks, corners, vertical, polarity="auto"):
    direction = "vertical" if vertical else "horizontal"
    H, W = img.shape[:2]
    found = Q.find_corners(img, polarity)
    assert found["quad"] is not None
    for (fx, fy), (cx, cy) in zip(found["quad"], corners):
        assert abs(fx - cx) <= 2 and abs(fy - cy) <= 2, (found["quad"], corners)
    quad = Q.accepted(found, img.shape)
    assert quad is not None
    r = Q.find_blocks(img, quad, direction, polarity)
    assert len(r["blocks"]) == len(masks), r["blocks"]
    groups = [[masks[0]]] + masks[1:]
    for g, win in enumerate(r["blocks"]):               # the heading (title column) first, then the columns in reading order
        member = inside(Q.line_quad(quad, r["size"], win), (H, W), 0.5)
        for other, grp in enumerate(groups):
            got = [bool((m & member).any()) for m in grp]
            assert all(got) if other == g else not any(got), (win, g, other)
        lines = Q.find_lines(img, quad, win, direction, polarity=polarity)["lines"]
        assert len(lines) == len(groups[g]), (g, len(lines), len(groups[g]))
        for k, m in enumerate(groups[g]):
            assert not (m & ~inside(lines[k], (H, W), 0.5)).any(), (g, k)
            for k2 in range(len(lines)):
                if k2 != k:
                    assert not (m & inside(lines[k2], (H, W), -0.5)).any(), (g, k, k2)
    return found, r


PULLS = [(0, 0, 0, 0), (60, 0, 0, 0), (0, 90, 0, 0), (0, 0, 0, 80), (40, 0, 30, 0), (0, 60, 0, 40)]


@pytest.mark.parametrize("pull", PULLS)
@pytest.mark.parametrize("widths,misalign", [((300, 300), False), ((260, 320, 240), True)])
def test_drawn_photographed_pages(pull, widths, misalign):
    flat, _ = drawn_page(widths, 8, 0.0, 0, misalign)
    h, w = flat.shape[:2]
    corners = corners_of(w, h, 110, 110, pull)
    img, masks = photo(widths, 8, corners, seed=sum(pull) + len(widths), misalign=misalign)
    _check_photo(img, masks, corners, vertical=False)


@pytest.mark.parametrize("pull", [(0, 0, 0, 0), (50, 0, 0, 0), (0, 0, 0, 70)])
def test_drawn_photographed_vertical_pages(pull):
    flat, _ = drawn_page((300, 300), 8, 0.0, 7, vertical=True)
    h, w = flat.shape[:2]
    corners = corners_of(w, h, 110, 110, pull)
    img, masks = photo((300, 300), 8, corners, seed=7, vertical=True)
    _check_photo(img, masks, corners, vertical=True)


def test_light_on_dark_photographed_page():
    flat, _ = drawn_page((300, 300), 6, 0.0, 3)
    h, w = flat.shape[:2]
    corners = corners_of(w, h, 110, 110, (40, 0, 0, 30))
    img, masks = photo((300, 300), 6, corners, seed=3, light=True)
    _check_photo(img, masks, corners, vertical=False, polarity="light")


def test_foreshortening_of_two():
    """The far side half as long as the near one."""
    flat, _ = drawn_page((300, 300), 8, 0.0, 5)
    h, w = flat.shape[:2]
    corners = corners_of(w, h, 110, 110, (w // 4, 0, 0, 0))
    assert corners[1][0] - corners[0][0] == pytest.approx(w / 2, abs=1)
    img, masks = photo((300, 300), 8, corners, seed=5)
    _check_photo(img, masks, corners, vertical=False)


def test_hull_and_quad_by_hand():
    mask = np.zeros((6, 8), bool)
    mask[1:5, 2:7] = True
    mask[0, 3] = True                                   # a bump on the top row
    label, size, members = Q.page_component(mask)
    assert (label, size) == (3, 21)
    hull = Q.monotone_chain(Q.row_points(members))
    assert sorted(hull) == sorted([(3, 0), (4, 0), (7, 1), (7, 5), (2, 5), (2, 1)])
    area2, idx = Q.largest_quad(hull)
    assert area2 == 41                                  # the bump's left corner beats the 5 x 4 rectangle's 40
    assert Q.order_corners(hull, idx) == [(3, 0), (7, 1), (7, 5), (2, 5)]


def test_tie_rule_of_the_component():
    mask = np.zeros((4, 9), bool)
    mask[:, 0:3] = True
    mask[:, 6:9] = True
    assert Q.page_component(mask)[:2] == (0, 12)        # equal sizes: the smaller label
    assert Q.page_component(np.zeros((3, 3), bool))[0] == -1


def test_frame_filling_page_is_the_image():
    img = np.full((40, 60, 3), 230, np.uint8)
    img[10:14, 10:50] = 20
    r = Q.find_corners(img)
    assert r["quad"] == [(0, 0), (60, 0), (60, 40), (0, 40)]
    assert Q.accepted(r, img.shape) == pipeline.QuadRegion((0.0, 0.0), (60.0, 0.0), (60.0, 40.0), (0.0, 40.0))
    small = np.full((40, 60, 3), 20, np.uint8)
    small[5:15, 5:25] = 230                             # a page of a twelfth of the image
    assert Q.find_corners(small)["quad"] is not None and Q.accepted(Q.find_corners(small), small.shape) is None


def test_rectangle_quad_reduces_to_the_level_page_and_block():
    img, _ = drawn_page((300, 300), 6, 0.0, 11)
    H, W = img.shape[:2]
    x0, y0, x1, y1 = 13, 7, W - 9, H - 4
    quad = pipeline.QuadRegion((x0, y0), (x1, y0), (x1, y1), (x0, y1))
    R = rectify(img, quad)
    assert np.array_equal(R, img[y0:y1, x0:x1])
    r = Q.find_blocks(img, quad)
    level = P.find_blocks(img, (x0, y0, x1, y1))
    assert r["size"] == (x1 - x0, y1 - y0)
    assert [(a + x0, b + y0, c + x0, d + y0) for a, b, c, d in r["blocks"]] == level["blocks"]
    for win, blk in zip(r["blocks"], level["blocks"]):
        got = Q.find_lines(img, quad, win)
        want = B.find_lines(img, blk)
        assert len(got["lines"]) == len(want["lines"]) > 0
        for q, (a, b, c, d) in zip(got["lines"], want["lines"]):
            assert np.allclose(q, [(a, b), (c, b), (c, d), (a, d)], rtol=0, atol=1e-9)
    # the pipeline's mapping is the twin's
    rect = r["blocks"][0]
    want = Q.line_quad(quad, r["size"], rect)
    assert tuple(pipeline._line_quad(quad, r["size"], rect)) == want


def test_from_quad_box():
    q = pipeline.QuadRegion((10.5, 3.2), (50.0, 2.0), (49.1, 30.9), (-1.0, 28.0))
    blk = pipeline.TextBlock.from_quad(q, direction="vertical")
    assert blk.rect == (0, 2, 50, 31) and blk.quad == q and blk.direction == "vertical"
    assert pipeline.TextBlock.from_quad(q, (20, 40)).rect == (0, 2, 40, 20)
    assert pipeline._check_block(pipeline.TextBlock.from_quad(q, (40, 60)), 40, 60, "b") == (0, 2, 50, 31)


QUAD = pipeline.QuadRegion((20.0, 10.0), (180.0, 20.0), (170.0, 150.0), (30.0, 140.0))


def test_validation_errors_name_the_region():
    H, W = 200, 240
    cp = lambda pg: pipeline._check_page(pg, H, W, "image 3, region 1 (a text page)")
    cb = lambda blk: pipeline._check_block(blk, H, W, "image 3, region 2 (a text block)")
    with pytest.raises(ValueError, match=r"image 3, region 1 \(a text page\): rect and quad are both given"):
        cp(pipeline.TextPage((0, 0, 10, 10), quad=QUAD))
    with pytest.raises(ValueError, match=r"image 3, region 1 \(a text page\): skew and quad are both given"):
        cp(pipeline.TextPage(quad=QUAD, skew=2.0))
    with pytest.raises(ValueError, match=r"image 3, region 1 \(a text page\): skew and quad are both given"):
        cp(pipeline.TextPage(quad="auto", skew="auto"))
    with pytest.raises(ValueError, match=r"image 3, region 2 \(a text block\): skew and quad are both given"):
        cb(pipeline.TextBlock.from_quad(QUAD, skew=1.0))
    with pytest.raises(ValueError, match=r"image 3, region 1 \(a text page\): quad must be a QuadRegion"):
        cp(pipeline.TextPage(quad="corners"))
    with pytest.raises(ValueError, match=r"image 3, region 1 \(a text page\): the quad is not strictly convex"):
        cp(pipeline.TextPage(quad=pipeline.QuadRegion(QUAD.tl, QUAD.bl, QUAD.br, QUAD.tr)))
    with pytest.raises(ValueError, match=r"image 3, region 2 \(a text block\): the quad is not strictly convex"):
        cb(pipeline.TextBlock.from_quad(pipeline.QuadRegion(QUAD.tl, QUAD.bl, QUAD.br, QUAD.tr)))
    with pytest.raises(ValueError, match=r"image 3, region 2 \(a text block\): rectangle .* is not the quad's pixel box"):
        cb(pipeline.TextBlock((0, 0, 100, 100), quad=QUAD))
    w_r, h_r = pipeline.quad_maps(QUAD, 1).size
    cb(pipeline.TextBlock.from_quad(QUAD, window=(0, 0, w_r, h_r)))
    with pytest.raises(ValueError, match=r"image 3, region 2 \(a text block\): window .* outside the .* rectified crop"):
        cb(pipeline.TextBlock.from_quad(QUAD, window=(0, 0, w_r + 1, h_r)))
    with pytest.raises(ValueError, match=r"image 3, region 2 \(a text block\): a window is four integers"):
        cb(pipeline.TextBlock.from_quad(QUAD, window=(0, 0, 1.5, 2)))


def test_rectified_side_over_32767():
    n = 30000
    over = pipeline.QuadRegion((0.0, 0.0), (float(n), 14000.0), (float(n), 14100.0), (0.0, 100.0))
    assert pipeline.quad_maps(over, 1).size[0] > 32767
    with pytest.raises(ValueError, match=r"image 0, region 0 \(a text page\): crop .* exceeds 32767"):
        pipeline._check_page(pipeline.TextPage(quad=over), n, n, "image 0, region 0 (a text page)")
    with pytest.raises(ValueError, match=r"image 0, region 1 \(a text block\): crop .* exceeds 32767"):
        pipeline._check_block(pipeline.TextBlock.from_quad(over, (n, n)), n, n, "image 0, region 1 (a text block)")


def test_work_limit_counts_the_rectified_crop(monkeypatch):
    w_r, h_r = pipeline.quad_maps(QUAD, 1).size
    need = pipeline._page_bytes(pipeline.TextPage(quad=QUAD), (0, 0, 240, 200), False)
    assert need == 3 * w_r * h_r + ops.page_bytes(w_r, h_r)
    monkeypatch.setattr(ops, "PAGE_MAX_WORK", need - 1)
    with pytest.raises(ValueError, match=r"image 0, region 0 \(a text page\): the page needs more than .* bytes"):
        pipeline._check_page(pipeline.TextPage(quad=QUAD), 200, 240, "image 0, region 0 (a text page)")
    monkeypatch.setattr(ops, "PAGE_MAX_WORK", ops.quad_page_bytes(240, 200) - 1)
    with pytest.raises(ValueError, match="bytes of work memory"):
        pipeline._check_page(pipeline.TextPage(quad="auto"), 200, 240, "p")


def _no_launch(monkeypatch):
    def boom(*a, **k):
        raise AssertionError("a launch was reached")
    for f in ("find_page_quads", "find_blocks", "find_lines", "warp_perspective"):
        monkeypatch.setattr(ops, f, boom)
    monkeypatch.setattr(pipeline, "_device_images", boom)


def test_public_calls_raise_before_any_launch(monkeypatch):
    _no_launch(monkeypatch)
    img = np.zeros((200, 240, 3), np.uint8)
    with pytest.raises(ValueError, match=r"image 0, page 1: rect and quad are both given"):
        pipeline.find_blocks([img], [[pipeline.TextPage(quad="auto"), pipeline.TextPage((0, 0, 5, 5), quad=QUAD)]])
    with pytest.raises(ValueError, match=r"image 0, block 0: window"):
        pipeline.find_lines([img], [[pipeline.TextBlock.from_quad(QUAD, window=(0, 0, 999, 5))]])
    with pytest.raises(ValueError, match=r"image 0, region 1 \(a text page\): skew and quad"):
        pipeline.restore_regions(None, None, None, [img], [[(0, 0, 4, 4), pipeline.TextPage(quad=QUAD, skew=1.0)]])
    with pytest.raises(ValueError, match=r"image 0, region 0 \(a text block\): the quad is not strictly convex"):
        pipeline.restore_regions(None, None, None, [img], [[pipeline.TextBlock.from_quad(QUAD[::-1])]])


def test_quad_region_as_rect_still_raises():
    with pytest.raises(ValueError, match="a text block is an integer rectangle"):
        pipeline._check_block(pipeline.TextBlock(QUAD), 200, 240, "b")
    with pytest.raises(ValueError, match="a text page is None or an integer rectangle"):
        pipeline._check_page(pipeline.TextPage(QUAD), 200, 240, "p")


def test_new_kernels_build_without_spills(tmp_path):
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    if not os.path.exists(nvcc):
        pytest.skip("nvcc not found")
    src = os.path.join(os.path.dirname(ops.__file__), "csrc", "block_ops.cu")
    r = subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-Xcompiler", "-fPIC",
                        "-DMN_BUILD", "-Xptxas", "-v", "-c", src, "-o", str(tmp_path / "b.o")], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    for kernel in ("quad_label_local_kernel", "quad_label_border_kernel", "quad_label_count_kernel", "quad_pick_kernel",
                   "quad_rows_kernel", "quad_hull_kernel"):
        props = re.search(rf"Function properties for \S*{kernel}\S*\n(.*)\n", r.stderr)
        assert props, kernel
        assert "0 bytes spill stores, 0 bytes spill loads" in props.group(1), props.group(1)
