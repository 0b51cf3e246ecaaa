"""Figures (DESIGN.md section 7b, "Figures") on the host: the twin on drawn pages with photos, charts, framed and dark pictures,
wrapped text and a large headline; its invariance on pages without a piece of the figure size, the exact threshold, symmetry,
polarity, ruled and photographed pages; every validation error of find_blocks and restore_regions (raised before anything
reaches a device); and the build of the kernels."""
import os
import re
import subprocess

import cv2
import numpy as np
import pytest

from marconet_b200 import ops, pipeline
from oracle import blocks as B
from oracle import figure_pages as FP
from oracle import pages as P
from oracle import quad_pages as Q
from oracle import ruled_pages as RP

from test_ruled_pages import _photo, framed_page, newspaper_page, table, table_page

FONT = cv2.FONT_HERSHEY_DUPLEX
WORDS = "THE QUICK BROWN FOX JUMPS OVER A LAZY DOG PACK MY BOX WITH FIVE DOZEN JUGS 0123456789".split()
H, W, PITCH, TOP = 1200, 1600, 33, 130


def _paper(rng, shape):
    return np.clip(rng.integers(215, 246, 3) + rng.integers(-12, 13, shape + (1,)), 0, 255).astype(np.uint8)


def _lines(page, rng, x, width, ys):
    """Lines of words fitting ``width`` at baselines ys, from x."""
    for y in ys:
        t = str(rng.choice(WORDS))
        while True:
            longer = t + " " + str(rng.choice(WORDS))
            if cv2.getTextSize(longer, FONT, 1.0, 2)[0][0] > width:
                break
            t = longer
        cv2.putText(page, t, (x, y), FONT, 1.0, (20,) * 3, 2, cv2.LINE_AA)


def smooth_photo(rng, h, w, lo=40, hi=240):
    """A smooth greyscale photo: blurred noise stretched to [lo, hi]."""
    f = cv2.GaussianBlur(rng.normal(0, 1, (h, w)), (0, 0), 12)
    f = (f - f.min()) / (f.max() - f.min())
    return (lo + (hi - lo) * f).astype(np.uint8)[..., None].repeat(3, axis=2)


def blotch_photo(rng, h, w, sigma=3):
    """A two-tone photo of blotches about 2 sigma across, half of them dark: its ink runs are short."""
    f = cv2.GaussianBlur(rng.normal(0, 1, (h, w)), (0, 0), sigma)
    return np.where(f > 0, 60, 200).astype(np.uint8)[..., None].repeat(3, axis=2)


def chart(rng, h, w):
    """A line chart on paper: two axes and a polyline of 12 points starting on the vertical axis."""
    c = np.full((h, w, 3), 232, np.uint8)
    cv2.line(c, (20, 10), (20, h - 20), (20,) * 3, 2)
    cv2.line(c, (20, h - 20), (w - 10, h - 20), (20,) * 3, 2)
    pts = np.stack([np.linspace(20, w - 20, 12), h - 40 - rng.uniform(0, h - 100, 12)], 1).astype(np.int32)
    cv2.polylines(c, [pts], False, (20,) * 3, 2)
    return c


def column_page(picture="photo", seed=0):
    """The page of the issue: a heading over two columns of up to 30 lines; the picture replaces lines 12-24 of the left column.
    (image, the picture's rectangle)."""
    rng = np.random.default_rng(seed)
    cw = (W - 80 - 60) // 2
    page = _paper(rng, (H, W))
    cv2.putText(page, "A HEADING OVER THE COLUMNS", (40, 70), FONT, 1.0, (20,) * 3, 2, cv2.LINE_AA)
    _lines(page, rng, 40, cw, [TOP + PITCH * k for k in list(range(12)) + list(range(25, 30))])
    _lines(page, rng, 40 + cw + 60, cw, [TOP + PITCH * k for k in range(30)])
    y0, y1, x0, x1 = TOP + PITCH * 12 - 10, TOP + PITCH * 24, 40, 40 + cw
    if picture == "photo":
        page[y0:y1, x0:x1] = smooth_photo(rng, y1 - y0, x1 - x0)
    elif picture == "chart":
        page[y0:y1, x0:x1] = chart(rng, y1 - y0, x1 - x0)
    elif picture == "dark":
        page[y0:y1, x0:x1] = smooth_photo(rng, y1 - y0, x1 - x0, 5, 90)
    return page, (x0, y0, x1, y1)


def framed_photo_page(seed=4):
    """A paragraph of 5 lines, a light photo inside a 3-pixel frame, and a paragraph of 4 lines on an 800-pixel page: a frame
    side is thin, but the two sides of a row reach the page width's 1 / 128.  (image, the frame's rectangle)."""
    rng = np.random.default_rng(seed)
    page = _paper(rng, (700, 800))
    _lines(page, rng, 40, 720, [60 + PITCH * k for k in range(5)])
    x0, y0, x1, y1 = 40, 240, 760, 500
    page[y0:y1, x0:x1] = smooth_photo(rng, y1 - y0, x1 - x0, 150, 250)
    page[y0:y0 + 3, x0:x1] = page[y1 - 3:y1, x0:x1] = page[y0:y1, x0:x0 + 3] = page[y0:y1, x1 - 3:x1] = 20
    _lines(page, rng, 40, 720, [550 + PITCH * k for k in range(4)])
    return page, (x0, y0, x1, y1)


def wide_photo_page(seed=5):
    """A paragraph of 8 lines, a photo across the page's full width, and a paragraph of 6 lines."""
    rng = np.random.default_rng(seed)
    page = _paper(rng, (900, 1200))
    _lines(page, rng, 40, 1100, [60 + PITCH * k for k in range(8)])
    page[340:640, 0:1200] = smooth_photo(rng, 300, 1200)
    _lines(page, rng, 40, 1100, [690 + PITCH * k for k in range(6)])
    return page, (0, 340, 1200, 640)


def wrapped_page(seed=6):
    """A photo over half the page's width in its top left corner, 8 lines wrapped beside it 20 pixels to its right, and a
    paragraph of 6 lines across the page under both: (image, photo rectangle)."""
    rng = np.random.default_rng(seed)
    page = _paper(rng, (740, 1100))
    page[40:300, 40:640] = smooth_photo(rng, 260, 600, 20, 160)
    _lines(page, rng, 660, 400, [60 + PITCH * k for k in range(8)])
    _lines(page, rng, 40, 1020, [350 + PITCH * k for k in range(6)])
    return page, (40, 40, 640, 300)


def headline_page(seed=7):
    """A headline whose capitals are drawn about 4 S high (scale 4.4, stroke 8) over a paragraph of 10 lines."""
    rng = np.random.default_rng(seed)
    page = _paper(rng, (560, 1100))
    cv2.putText(page, "MOW", (40, 130), FONT, 4.4, (20,) * 3, 8, cv2.LINE_AA)
    _lines(page, rng, 40, 1020, [190 + PITCH * k for k in range(10)])
    return page


def _ink(img):
    g = B.grey(img)
    t = B.otsu(g)
    return g <= t if 2 * int((g <= t).sum()) <= g.size else g > t


def _meets(a, b):
    return a[0] < b[2] and b[0] < a[2] and a[1] < b[3] and b[1] < a[3]


def _n_lines(img, blocks, direction="horizontal"):
    return [len(B.find_lines(img, b, direction)["lines"]) for b in blocks]


def _inside(inner, outer):
    return outer[0] <= inner[0] and outer[1] <= inner[1] and inner[2] <= outer[2] and inner[3] <= outer[3]


def _no_block_meets(res):
    assert not any(_meets(b, f) for b in res["blocks"] for f in res["figures"]), res


# ---- invariance ----

def _random_page(rng):
    h, w = int(rng.integers(20, 300)), int(rng.integers(20, 500))
    ink = rng.random((h, w)) < rng.choice([0.005, 0.03])
    return np.where(ink[..., None], 20, 235).astype(np.uint8).repeat(3, axis=2)


def test_pages_without_a_figure_piece_are_unchanged():
    """On drawn, random and ruled pages without a piece of at least f, the dict, blocks and S are those of figures=None, with
    figures=[]."""
    rng = np.random.default_rng(0)
    pages = [(table_page(4, 3)[0], dict(rules=True)), (framed_page(5)[0], dict(rules=True)),
             (newspaper_page()[0], dict(rules=True)), (column_page(None)[0], {}), (headline_page(), dict(figure_size=500))]
    pages += [(_random_page(rng), dict(rect=None)) for _ in range(12)]
    seen = 0
    for img, kw in pages:
        res = FP.find_blocks(img, **kw)
        if kw == dict(rect=None) and res["figures"]:     # specks dense enough to make a piece of f: not this test's page
            continue
        plain = (RP.find_blocks(img, rule_length=kw.get("rule_length")) if kw.get("rules")
                 else P.find_blocks(img, kw.get("rect")))
        assert res["figures"] == [] and res["figure_size"] == (kw.get("figure_size") or 3 * plain["text_size"])
        assert {k: v for k, v in res.items() if k not in ("figures", "figure_size")} == plain
        seen += len(plain["blocks"]) > 0
    assert seen >= 10


def test_page_without_text_size_has_no_figures():
    img = np.full((40, 50, 3), 235, np.uint8)
    img[10, 10] = 20
    res = FP.find_blocks(img)
    assert res["figure_size"] == 0 and res["figures"] == [] and res["blocks"] == [] and res["text_size"] == 0


# ---- named pages ----

def test_photo_page():
    """Without figures the photo and the 5 lines under it are one block of one "line"; with them the photo is one figure and
    the page gives the heading and blocks of 12, 5 and 30 lines."""
    img, photo = column_page("photo")
    plain = P.find_blocks(img)
    assert len(plain["blocks"]) == 4 and any(_meets(b, photo) and _n_lines(img, [b]) == [1] for b in plain["blocks"])
    res = FP.find_blocks(img)
    assert res["text_size"] == 24 and res["figure_size"] == 72
    assert len(res["figures"]) == 1 and _inside(res["figures"][0], photo)
    assert _n_lines(img, res["blocks"]) == [1, 12, 5, 30]
    _no_block_meets(res)


def test_chart():
    img, box = column_page("chart")
    res = FP.find_blocks(img)
    assert len(res["figures"]) == 1 and _inside(res["figures"][0], box)
    assert _n_lines(img, res["blocks"]) == [1, 12, 5, 30]
    _no_block_meets(res)


def test_light_photo_in_a_thin_frame():
    img, box = framed_photo_page()
    res = FP.find_blocks(img)
    assert res["figures"] == [box]
    assert _n_lines(img, res["blocks"]) == [5, 4]
    _no_block_meets(res)


def test_dark_photo_is_rejected_without_figures_and_a_figure_with_them():
    img, box = column_page("dark")
    plain = P.find_blocks(img)
    assert any(_inside(box, r) for r in plain["rejected"])         # the photo and the lines under it: over half ink
    res = FP.find_blocks(img)
    assert res["figures"] == [box] and box not in res["rejected"]
    assert _n_lines(img, res["blocks"]) == [1, 12, 5, 30]
    _no_block_meets(res)


def test_photo_across_the_page_between_two_paragraphs():
    img, box = wide_photo_page()
    res = FP.find_blocks(img)
    assert len(res["figures"]) == 1 and _inside(res["figures"][0], box)
    assert _n_lines(img, res["blocks"]) == [8, 6]
    _no_block_meets(res)


def test_text_wrapped_beside_a_figure_keeps_its_lines():
    """The figure is wider than half the page, yet the rows beside it stay non-white: the 8 wrapped lines and the 6 lines
    under them are all found."""
    img, box = wrapped_page()
    plain = P.find_blocks(img)
    res = FP.find_blocks(img)
    assert res["figures"] == [box]
    assert sum(_n_lines(img, res["blocks"])) == 14 and sum(_n_lines(img, plain["blocks"])) < 14
    _no_block_meets(res)


def lone_photo(seed=8):
    """A 480 x 300 photo alone on a 900 x 600 page."""
    rng = np.random.default_rng(seed)
    img = np.full((600, 900, 3), 235, np.uint8)
    img[50:350, 60:540] = smooth_photo(rng, 300, 480)
    return img


def test_photo_alone_with_a_figure_size():
    img = lone_photo()
    res = FP.find_blocks(img, figure_size=100)
    assert res["figure_size"] == 100 and len(res["figures"]) == 1 and _inside(res["figures"][0], (60, 50, 540, 350))
    assert res["blocks"] == []


def test_headline_at_four_text_sizes_becomes_a_figure():
    """A known effect of the default f = 3 S: glyphs of a headline drawn at 4 S are pieces of at least f, so they are figures
    and leave the text; the paragraph keeps its 10 lines."""
    img = headline_page()
    res = FP.find_blocks(img)
    assert res["text_size"] == 24 and len(res["figures"]) >= 1
    assert all(f[3] <= 150 for f in res["figures"])
    assert _n_lines(img, res["blocks"])[-1] == 10


# ---- threshold, symmetry, polarity ----

def threshold_page():
    """Two solid pieces, 50 x 40 and 70 x 30, beside a column of 3-pixel dashes."""
    ink = np.zeros((120, 200), bool)
    ink[20:60, 30:80] = True                            # 40 x 50
    ink[80:110, 120:190] = True                         # 30 x 70
    for y in range(5, 115, 12):
        ink[y:y + 3, 100:105] = True
    return np.where(ink[..., None], 20, 235).astype(np.uint8).repeat(3, axis=2)


def test_exact_threshold():
    """A piece whose shorter side is exactly f is a figure; f - 1 is not."""
    img = threshold_page()
    assert FP.find_blocks(img, figure_size=30)["figures"] == [(30, 20, 80, 60), (120, 80, 190, 110)]
    assert FP.find_blocks(img, figure_size=31)["figures"] == [(30, 20, 80, 60)]
    assert FP.find_blocks(img, figure_size=40)["figures"] == [(30, 20, 80, 60)]
    assert FP.find_blocks(img, figure_size=41)["figures"] == []


def test_transposed_page_gives_transposed_figures_and_blocks():
    img, _ = column_page("photo")
    t = np.ascontiguousarray(img.transpose(1, 0, 2)[:, ::-1])
    hor, ver = FP.find_blocks(img), FP.find_blocks(t, direction="vertical")
    tr = lambda r: [(H - y1, x0, H - y0, x1) for x0, y0, x1, y1 in r]
    assert ver["figures"] == tr(hor["figures"]) and ver["blocks"] == tr(hor["blocks"])


def test_light_on_dark_gives_the_same_result():
    img, _ = column_page("photo")
    res, inv = FP.find_blocks(img), FP.find_blocks(255 - img)
    assert inv["ink"] == "light" and res["ink"] == "dark"
    assert {k: v for k, v in inv.items() if k not in ("ink", "threshold")} == \
        {k: v for k, v in res.items() if k not in ("ink", "threshold")}


# ---- rules and perspective ----

def table_beside_photo(seed=9):
    """A 4 x 2 ruled table beside a photo: (image, photo rectangle, the cells' masks).  Its rules are 190 pixels or longer and
    the photo's ink runs shorter than 150: runs of a photo at least the rule length are rules too."""
    rng = np.random.default_rng(seed)
    shape = (24 + 47 * 4 + 40, 48 + 2 * 168 + 60 + 300)
    rules = np.zeros(shape, bool)
    masks = table(shape, rules, rng, 24, 24, 4, 2)
    ink = rules | np.any(masks, axis=0)
    img = np.where(ink[..., None], 20, 235).astype(np.uint8).repeat(3, axis=2)
    x0 = 24 + 2 * 168 + 60
    img[24:24 + 188, x0:x0 + 300] = blotch_photo(rng, 188, 300)
    return img, (x0, 24, x0 + 300, 24 + 188), masks


def test_ruled_table_beside_a_photo():
    img, box, masks = table_beside_photo()
    res = FP.find_blocks(img, rules=True, rule_length=150)
    assert len(res["figures"]) == 1 and _inside(res["figures"][0], box)
    assert len(res["blocks"]) == len(masks) == 8 and _n_lines(img, res["blocks"]) == [1] * 8
    _no_block_meets(res)


def photographed_photo_page():
    """The photo page at 800 x 600 warped by cv2.warpPerspective over a darker noisy background."""
    img, _ = column_page("photo")
    small = cv2.resize(img, (800, 600), interpolation=cv2.INTER_AREA)
    h, w = small.shape[:2]
    return _photo(small, [(112, 118), (112 + w - 10, 110), (112 + w, 112 + h), (106, 116 + h - 6)], 10)


def test_photographed_photo_page_under_quad_auto():
    photo = photographed_photo_page()
    quad = Q.accepted(Q.find_corners(photo), photo.shape)
    assert quad is not None
    res = FP.find_quad_blocks(photo, quad)
    assert res["size"][0] > 700 and len(res["figures"]) == 1
    fx0, fy0, fx1, fy1 = res["figures"][0]
    assert fx1 - fx0 > 300 and fy1 - fy0 > 150 and fx1 <= res["size"][0] and fy1 <= res["size"][1]
    _no_block_meets(res)


# ---- validation, work and build ----

def _no_launch(monkeypatch):
    def boom(*a, **k):
        raise AssertionError("a launch was reached")
    for f in ("find_page_quads", "find_blocks", "find_lines", "warp_perspective"):
        monkeypatch.setattr(ops, f, boom)
    monkeypatch.setattr(pipeline, "_device_images", boom)


@pytest.mark.parametrize("page, match", [
    (pipeline.TextPage(figures="on"), "figures must be None or 'auto', got 'on'"),
    (pipeline.TextPage(figures=True), "figures must be None or 'auto', got True"),
    (pipeline.TextPage(figures="auto", figure_size=1), r"figure_size must be an integer in \[2, 32767\], got 1"),
    (pipeline.TextPage(figures="auto", figure_size=32768), r"figure_size must be an integer in \[2, 32767\], got 32768"),
    (pipeline.TextPage(figures="auto", figure_size=40.0), r"figure_size must be an integer in \[2, 32767\], got 40.0"),
    (pipeline.TextPage(figures="auto", figure_size=True), r"figure_size must be an integer in \[2, 32767\], got True"),
    (pipeline.TextPage(figure_size=40), "figure_size is given, but figures is None"),
    (pipeline.TextPage(figures="auto", skew="auto"), "figures and skew are both given"),
    (pipeline.TextPage(figures="auto", skew=2.0), "figures and skew are both given"),
    (pipeline.TextPage(figures="auto", curve="auto"), "figures and curve are both given"),
])
def test_validation_errors_raise_before_any_launch(monkeypatch, page, match):
    _no_launch(monkeypatch)
    img = np.zeros((200, 240, 3), np.uint8)
    with pytest.raises(ValueError, match=r"image 0, page 1: " + match):
        pipeline.find_blocks([img], [[pipeline.TextPage(figures="auto"), page]])
    with pytest.raises(ValueError, match=r"image 0, region 1 \(a text page\): " + match):
        pipeline.restore_regions(None, None, None, [img], [[(0, 0, 4, 4), page]])


def test_work_memory_counts_the_figure_plane_and_table(monkeypatch):
    _no_launch(monkeypatch)
    pg = pipeline.TextPage(figures="auto")
    assert ops.figure_page_bytes(70, 40) == 4 * 40 * 3 + 12 * 1024
    assert pipeline._page_bytes(pg, (0, 0, 70, 40), False) == ops.page_bytes(70, 40) + ops.figure_page_bytes(70, 40)
    both = pg._replace(rules="auto")
    assert pipeline._page_bytes(both, (0, 0, 70, 40), False) == \
        ops.page_bytes(70, 40) + ops.rule_page_bytes(70, 40) + ops.figure_page_bytes(70, 40)
    quad = pipeline.QuadRegion((10.0, 12.0), (200.0, 8.0), (210.0, 180.0), (6.0, 170.0))
    w_r, h_r = pipeline.quad_maps(quad, 1).size
    assert pipeline._page_bytes(pg._replace(quad=quad), (0, 0, 240, 200), False) == \
        3 * w_r * h_r + ops.page_bytes(w_r, h_r) + ops.figure_page_bytes(w_r, h_r)
    monkeypatch.setattr(ops, "PAGE_MAX_WORK", ops.page_bytes(240, 200) + ops.figure_page_bytes(240, 200) - 1)
    pipeline._check_page(pipeline.TextPage(), 200, 240, "p")
    with pytest.raises(ValueError, match=r"image 0, page 0: the page needs more than .* bytes of work memory"):
        pipeline.find_blocks([np.zeros((200, 240, 3), np.uint8)], [[pg]])
    monkeypatch.setattr(ops, "PAGE_MAX_WORK", 2 * ops.page_bytes(240, 200) + ops.figure_page_bytes(240, 200) - 1)
    with pytest.raises(ValueError, match=r"the call's 2 text pages need more than"):
        pipeline.find_blocks([np.zeros((200, 240, 3), np.uint8)], [[pg, pipeline.TextPage()]])


def test_ops_refuses_a_bad_figure_size():
    import torch
    img = torch.zeros((8, 8, 3), dtype=torch.uint8)
    for bad, skew in ((1, None), (32768, None), (True, None), (-1, None), (40, 2.0), (0, 2.0)):
        with pytest.raises(ValueError, match="find_blocks: page 0: figure_size"):
            ops.find_blocks([ops.PageItem(img, (0, 0, 8, 8), False, 0, skew=skew, figure_size=bad)])


def test_kernels_build_without_spills(tmp_path):
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    if not os.path.exists(nvcc):
        pytest.skip("nvcc not found")
    src = os.path.join(os.path.dirname(ops.__file__), "csrc", "block_ops.cu")
    r = subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-Xcompiler", "-fPIC",
                        "-DMN_BUILD", "-Xptxas", "-v", "-c", src, "-o", str(tmp_path / "b.o")], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    for kernel in ("figure_paint_kernel", "page_size_kernel", "page_blocks_kernel", "rule_transpose_kernel"):
        props = re.search(rf"Function properties for \S*{kernel}\S*\n(.*)\n", r.stderr)
        assert props, kernel
        assert "0 bytes spill stores, 0 bytes spill loads" in props.group(1), props.group(1)
