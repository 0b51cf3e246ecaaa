"""Text blocks split into lines (DESIGN.md section 7b, "Text blocks") on the host: the twin's Otsu threshold against cv2, its
lines on pages drawn with cv2.putText, polarity and the vertical transpose, and every validation error of find_lines and
restore_regions, raised before anything reaches a device."""
import cv2
import numpy as np
import pytest

from oracle import blocks as B

TEXTS = ["The quick brown fox", "jumps over 12 lazy dogs", "Hershey fonts, no download", "pack my box: 5 dozen jugs",
         "Sphinx of black quartz"]


def _page(n_lines, rng, fonts=(cv2.FONT_HERSHEY_SIMPLEX, cv2.FONT_HERSHEY_DUPLEX, cv2.FONT_HERSHEY_COMPLEX)):
    """A white-ish page with n_lines lines of dark text 36 pixels apart, strokes 2 pixels wide; returns the page and one ink
    mask per line."""
    h, w = 30 + 36 * n_lines, 360
    bg, fg = rng.integers(200, 256, 3), rng.integers(0, 60, 3)
    page = np.empty((h, w, 3), np.uint8)
    page[:] = bg
    masks = []
    for k in range(n_lines):
        m = np.zeros((h, w), np.uint8)
        cv2.putText(m, TEXTS[k % len(TEXTS)], (8 + 4 * k, 36 + 36 * k), fonts[k % len(fonts)], 0.7, 255, 2, cv2.LINE_8)
        masks.append(m > 0)
        page[m > 0] = fg
    return page, masks


def _otsu_cases():
    rng = np.random.default_rng(0)
    for k in range(2100):
        kind = k % 7
        if kind == 0:
            g = rng.integers(0, 256, (int(rng.integers(1, 60)), int(rng.integers(1, 60))), dtype=np.uint8)
        elif kind == 1:
            g = np.full((int(rng.integers(1, 40)), int(rng.integers(1, 40))), rng.integers(0, 256), np.uint8)
        elif kind == 2:
            a, b = rng.integers(0, 256, 2)
            g = np.where(rng.random((int(rng.integers(1, 50)), int(rng.integers(1, 50)))) < rng.random(), a, b).astype(np.uint8)
        elif kind == 3:
            s = (int(rng.integers(2, 70)), int(rng.integers(2, 70)))
            g = np.where(rng.random(s) < rng.random(), rng.normal(rng.integers(0, 120), 20, s),
                         rng.normal(rng.integers(130, 256), 25, s)).clip(0, 255).astype(np.uint8)
        elif kind == 4:
            g = rng.integers(0, 256, (1, 1), dtype=np.uint8)
        elif kind == 5:
            g = rng.integers(0, 256, (1, int(rng.integers(1, 400))), dtype=np.uint8)
        else:
            g = rng.integers(0, 256, (int(rng.integers(1, 400)), 1), dtype=np.uint8)
        yield g


def test_otsu_equals_cv2():
    """Random, uniform, two-valued, bimodal, 1x1, 1xN and Nx1 images: the twin's t is cv2's, on 2100 images."""
    n = 0
    for g in _otsu_cases():
        assert B.otsu(g) == cv2.threshold(g, 0, 255, cv2.THRESH_BINARY | cv2.THRESH_OTSU)[0], g
        n += 1
    assert n >= 2000


def test_grey_is_channel_order_free():
    rng = np.random.default_rng(1)
    img = rng.integers(0, 256, (20, 30, 3), dtype=np.uint8)
    for perm in ([2, 1, 0], [1, 2, 0], [0, 2, 1]):
        np.testing.assert_array_equal(B.grey(img), B.grey(img[..., perm]))


@pytest.mark.parametrize("n_lines", [1, 2, 5])
def test_lines_of_a_drawn_page(n_lines):
    """Each found rectangle holds all of its line's ink and none of another line's; the rectangles are disjoint."""
    rng = np.random.default_rng(n_lines)
    page, masks = _page(n_lines, rng)
    H, W = page.shape[:2]
    res = B.find_lines(page, (0, 0, W, H))
    assert res["ink"] == "dark" and len(res["lines"]) == n_lines
    for k, (x0, y0, x1, y1) in enumerate(res["lines"]):
        inside = np.zeros((H, W), bool)
        inside[y0:y1, x0:x1] = True
        assert not (masks[k] & ~inside).any(), f"line {k} leaves its rectangle"
        for j in range(n_lines):
            if j != k:
                assert not (masks[j] & inside).any(), f"line {j}'s ink is inside line {k}'s rectangle"
        for j, (a0, b0, a1, b1) in enumerate(res["lines"][:k]):
            assert max(x0, a0) >= min(x1, a1) or max(y0, b0) >= min(y1, b1), f"lines {j} and {k} overlap"


def test_block_inside_a_page_and_light_on_dark():
    rng = np.random.default_rng(7)
    page, _ = _page(4, rng)
    big = np.full((page.shape[0] + 50, page.shape[1] + 70, 3), 128, np.uint8)
    big[20:20 + page.shape[0], 30:30 + page.shape[1]] = page
    rect = (30, 20, 30 + page.shape[1], 20 + page.shape[0])
    dark = B.find_lines(big, rect)
    light = B.find_lines(255 - big, rect)
    assert dark["ink"] == "dark" and light["ink"] == "light"
    assert dark["lines"] == light["lines"] and len(dark["lines"]) == 4
    assert B.find_lines(big, rect, polarity="dark")["lines"] == dark["lines"]
    assert all(rect[0] <= x0 < x1 <= rect[2] and rect[1] <= y0 < y1 <= rect[3] for x0, y0, x1, y1 in dark["lines"])


def test_vertical_block_is_the_transposed_block():
    """Columns of the transposed page: the horizontal lines transposed, right to left."""
    rng = np.random.default_rng(3)
    page, _ = _page(3, rng)
    H, W = page.shape[:2]
    hor = B.find_lines(page, (0, 0, W, H))
    ver = B.find_lines(np.ascontiguousarray(page.transpose(1, 0, 2)), (0, 0, H, W), direction="vertical")
    assert ver["threshold"] == hor["threshold"] and ver["ink"] == hor["ink"]
    assert ver["lines"] == [(y0, x0, y1, x1) for x0, y0, x1, y1 in hor["lines"]][::-1]


def test_uniform_block_has_no_lines():
    img = np.full((40, 50, 3), 77, np.uint8)
    assert B.find_lines(img, (0, 0, 50, 40)) == dict(lines=[], threshold=0, ink="dark")
    assert B.find_lines(img, (3, 4, 5, 6), polarity="dark")["lines"] == []


def test_knobs_and_the_line_limit():
    rng = np.random.default_rng(5)
    page, _ = _page(3, rng)
    H, W = page.shape[:2]
    assert len(B.find_lines(page, (0, 0, W, H), gap=100)["lines"]) == 1
    assert B.find_lines(page, (0, 0, W, H), min_height=100)["lines"] == []
    assert B.find_lines(page, (0, 0, W, H), min_ink=10 ** 6)["lines"] == []
    stripes = np.full((6 * 300, 20, 3), 255, np.uint8)
    stripes[np.arange(6 * 300) % 6 < 3] = 0
    with pytest.raises(ValueError, match="300 lines exceed"):
        B.find_lines(stripes, (0, 0, 20, 6 * 300))
    assert len(B.find_lines(stripes[:6 * 256], (0, 0, 20, 6 * 256))["lines"]) == 256


BAD = [
    (dict(rect=(0, 0, 0, 5)), "is empty or outside"),
    (dict(rect=(0, 0, 41, 5)), "is empty or outside"),
    (dict(rect=(-1, 0, 4, 5)), "is empty or outside"),
    (dict(rect=(0.5, 0, 4, 5)), "integer rectangle"),
    (dict(rect="abcd"), "integer rectangle"),
    (dict(direction="diagonal"), "direction must be"),
    (dict(polarity="grey"), "polarity must be"),
    (dict(min_ink=0), "min_ink must be a positive integer"),
    (dict(gap=-2), "gap must be a positive integer"),
    (dict(min_height=2.0), "min_height must be a positive integer"),
    (dict(min_ink=True), "min_ink must be a positive integer"),
]


@pytest.mark.parametrize("kw,msg", BAD)
def test_find_lines_rejects_before_any_launch(kw, msg):
    from marconet_b200 import pipeline
    img = np.zeros((30, 40, 3), np.uint8)
    blk = pipeline.TextBlock(**dict(dict(rect=(0, 0, 40, 30)), **kw))
    with pytest.raises(ValueError, match=f"image 1, block 1: .*{msg}"):
        pipeline.find_lines([img, img], [[], [pipeline.TextBlock((0, 0, 4, 4)), blk]])


def test_find_lines_rejects_other_shapes():
    from marconet_b200 import pipeline
    img = np.zeros((30, 40, 3), np.uint8)
    for shape in (pipeline.OrientedRegion.from_rotated(20, 15, 20, 8, 10), pipeline.QuadRegion((1, 1), (20, 1), (20, 9), (1, 9)),
                  pipeline.VerticalRegion((0, 0, 5, 20))):
        with pytest.raises(ValueError, match="image 0, block 0: a text block is an integer rectangle.*not supported"):
            pipeline.find_lines([img], [[pipeline.TextBlock(shape)]])
    with pytest.raises(ValueError, match="image 0, block 0: expected a TextBlock"):
        pipeline.find_lines([img], [[(0, 0, 4, 4)]])
    big = np.zeros((1, 32768, 3), np.uint8)
    with pytest.raises(ValueError, match="exceeds 32767 pixels"):
        pipeline.find_lines([big], [[pipeline.TextBlock((0, 0, 32768, 1))]])
    assert pipeline.find_lines([img], [[]]) == [[]]


@pytest.mark.parametrize("kw,msg", BAD)
def test_restore_regions_rejects_blocks_before_any_launch(kw, msg):
    """The encoder is never touched: every error is raised before the call reaches a device."""
    from marconet_b200 import pipeline
    img = np.zeros((30, 40, 3), np.uint8)
    blk = pipeline.TextBlock(**dict(dict(rect=(0, 0, 40, 30)), **kw))
    with pytest.raises(ValueError, match=f"image 0, region 1 \\(a text block\\): .*{msg}"):
        pipeline.restore_regions(None, None, None, [img], [[(0, 0, 4, 4), blk]])


def test_restore_regions_rejects_labels_for_blocks_and_bad_regions_beside_them():
    from marconet_b200 import pipeline
    img = np.zeros((30, 40, 3), np.uint8)
    blk = pipeline.TextBlock((0, 0, 40, 30))
    with pytest.raises(ValueError, match="region 0 \\(a text block\\): labels or boxes are given"):
        pipeline.restore_regions(None, None, None, [img], [[blk]], labels=[[[1, 2]]])
    with pytest.raises(ValueError, match="region 0 \\(a text block\\): labels or boxes are given"):
        pipeline.restore_regions(None, None, None, [img], [[blk]], labels=[[None]], boxes=[[[[0, 0, 1, 1]]]])
    with pytest.raises(ValueError, match="image 0, region 1: rectangle \\(0, 0, 50, 5\\) is empty or outside"):
        pipeline.restore_regions(None, None, None, [img], [[blk, (0, 0, 50, 5)]])
    with pytest.raises(ValueError, match="region 0 \\(a text block\\): a text block is an integer rectangle"):
        pipeline.restore_regions(None, None, None, [img], [[pipeline.TextBlock(pipeline.CurvedRegion.from_arc(20, 15, 5, 12, 200, 340))]])
