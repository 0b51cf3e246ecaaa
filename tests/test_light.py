"""Even lighting (DESIGN.md section 7b, "Even lighting") on the host: the kernels' fp32 divide against live cv2.divide on every
pair, the numpy twin against live OpenCV closing and divide for both polarities and edge sizes, the default window, every
refusal of flatten_pages, and shaded curled pages (flat, and photographed as an open book) that lose or split lines until
they are evened."""

import cv2
import numpy as np
import pytest

from marconet_b200 import ops
from marconet_b200.pipeline import FlatPage, QuadRegion, flatten_pages
from oracle import curled_blocks as CB
from oracle import light as L
from oracle import pages as P

from test_curled_blocks import PITCH, curled_page
from test_flat_pages import level_after, mid_spread, open_book

cv2.ipp.setUseIPP(False)


def shade(img, kind):
    """img times a smooth shading field: "gradient", 1 - 0.65 x / w, or "vignette", 1 - 0.7 r^2 with r the distance of
    (x / w, y / h) from (0.3, 0.3)."""
    h, w = img.shape[:2]
    y, x = np.mgrid[0:h, 0:w].astype(np.float64)
    f = 1 - 0.65 * x / w if kind == "gradient" else 1 - 0.7 * ((x / w - 0.3) ** 2 + (y / h - 0.3) ** 2)
    return np.rint(img * f[..., None]).astype(np.uint8)


def rows(lines):
    """The number of text rows among traced lines (a row's pieces share its height)."""
    ys = sorted(0.5 * (q[1] + q[3]) if not hasattr(q, "top") else 0.25 * sum(t[1] + b[1] for t, b in zip(q.top, q.bottom)) / 2
                for q in lines)
    return 1 + sum(1 for a, b in zip(ys, ys[1:]) if b - a > PITCH / 2)


def test_fp32_divide_equals_cv2_on_every_pair():
    f, b = np.meshgrid(np.arange(256, dtype=np.uint8), np.arange(256, dtype=np.uint8), indexing="ij")
    with np.errstate(divide="ignore", invalid="ignore"):
        q = np.rint(np.float32(255) * f.astype(np.float32) / b.astype(np.float32))
    kernel = np.where(b == 0, 0, np.minimum(q, 255)).astype(np.uint8)
    want = cv2.divide(f, b, scale=255)
    np.testing.assert_array_equal(kernel, want)
    np.testing.assert_array_equal(L.divide(f, b), want)


@pytest.mark.parametrize("h,w", [(1, 1), (1, 37), (41, 1), (17, 23), (64, 9)])
@pytest.mark.parametrize("k", [3, 5, 101, 32767])
def test_twin_equals_cv2_closing_and_divide(h, w, k):
    rng = np.random.default_rng(h * 1000 + w + k)
    page = rng.integers(0, 256, (h, w, 3), dtype=np.uint8)
    kern = np.ones((k, k), np.uint8)
    dark = cv2.divide(page, cv2.morphologyEx(page, cv2.MORPH_CLOSE, kern), scale=255)
    light = 255 - cv2.divide(255 - page, 255 - cv2.morphologyEx(page, cv2.MORPH_OPEN, kern), scale=255)
    np.testing.assert_array_equal(L.even(page, k, "dark"), dark.reshape(page.shape))
    np.testing.assert_array_equal(L.even(page, k, "light"), light.reshape(page.shape))


def test_default_window():
    assert ops.light_window(800, 538) == L.window(800, 538) == 27
    assert [ops.light_window(w, h) for w, h in [(1, 1), (79, 500), (80, 80), (119, 4000), (4000, 3000), (32767, 32767)]] == \
        [3, 3, 5, 5, 151, 1639]
    page, _, _ = curled_page(8, "cylinder", PITCH, 11)
    res = L.flatten(page, FlatPage(light="even"))
    assert res["light_window"] == 27 and res["ink"] == "dark"
    assert L.flatten(page, FlatPage((10, 20, 90, 300), light="even", light_window=5))["light_window"] == 5


@pytest.mark.parametrize("fp,what", [
    (FlatPage(light="on"), "light must be None or 'even'"),
    (FlatPage(light=True), "light must be None or 'even'"),
    (FlatPage(light_window=5), "light_window is given, but light is None"),
    (FlatPage(light="even", light_window=4), "light_window must be an odd integer"),
    (FlatPage(light="even", light_window=1), "light_window must be an odd integer"),
    (FlatPage(light="even", light_window=32769), "light_window must be an odd integer"),
    (FlatPage(light="even", light_window=True), "light_window must be an odd integer"),
    (FlatPage(light="even", light_window=5.0), "light_window must be an odd integer"),
])
def test_refusals_name_the_image_and_page(fp, what):
    img = np.full((40, 50, 3), 200, np.uint8)
    with pytest.raises(ValueError, match=f"image 1, page 1: {what}"):
        flatten_pages([img, img], [[], [FlatPage(), fp]])


def test_light_pages_count_their_work_memory():
    from marconet_b200 import pipeline
    plain = pipeline._flat_bytes(FlatPage(), (100, 50), (100, 50))
    lit = pipeline._flat_bytes(FlatPage(light="even"), (100, 50), (100, 50))
    assert plain == 3 * 100 * 50 and lit == plain + ops.even_light_bytes(100, 50, (100, 50))


@pytest.mark.parametrize("kind", ["gradient", "vignette"])
def test_shading_breaks_the_page_and_evening_restores_it(kind):
    page, _, _ = curled_page(8, "cylinder", PITCH, 11)
    shaded = shade(page, kind)
    blocks = P.find_blocks(shaded, None, "horizontal", "auto")["blocks"]
    found = [len(CB.find_lines(shaded, b)["lines"]) for b in blocks]
    assert found != [8]                                     # the precondition: unevened, the page loses or splits lines
    evened = L.even(shaded, 27, "dark")
    blocks = P.find_blocks(evened, None, "horizontal", "auto")["blocks"]
    assert [len(CB.find_lines(evened, b)["lines"]) for b in blocks] == [8]
    res = L.flatten(shaded, FlatPage(curve="auto", light="even"))
    assert res["light_window"] == 27 and res["ink"] == "dark" and "table" in res
    lines = level_after(res["image"])
    assert rows(lines) == 8
    assert max(mid_spread(q) for q in lines) <= 2.0


# Under the 0.65 gradient the table and the shaded half outnumber the paper, so "auto" takes the paper for ink; the caller
# passes polarity="dark" (DESIGN.md 7b, "Even lighting").
@pytest.mark.parametrize("kind,polarity", [("gradient", "dark"), ("vignette", "auto")])
def test_shaded_open_book_flattens_level(kind, polarity):
    photo = shade(open_book("cylinder", PITCH, 11, 1.5), kind)
    before = level_after(L.flatten(photo, FlatPage(quad="auto", curve="auto", polarity=polarity))["image"])
    res = L.flatten(photo, FlatPage(quad="auto", curve="auto", light="even", polarity=polarity))
    assert res["kind"] == "quad" and res["ink"] == "dark" and "table" in res
    lines = level_after(res["image"])
    assert rows(before) < 8 or len(before) > len(lines)     # the precondition: unevened, lines are lost or split
    assert rows(lines) == 8
    assert max(mid_spread(q) for q in lines) <= 2.0


def test_light_and_dark_ink_are_complements():
    page, _, _ = curled_page(4, "flat", 0, 3, light=True)
    shaded = shade(page, "vignette")
    res = L.flatten(shaded, FlatPage(light="even"))
    assert res["ink"] == "light"
    np.testing.assert_array_equal(res["image"], 255 - L.even(255 - shaded, res["light_window"], "dark"))
    q = QuadRegion((10.0, 10.0), (300.0, 12.0), (298.0, 150.0), (12.0, 148.0))
    assert L.flatten(shaded, FlatPage(quad=q, light="even", polarity="light"))["ink"] == "light"
