"""Ruled pages (DESIGN.md section 7b, "Ruled pages") on the host: the twin's rule pixels against live OpenCV morphology, its
blocks on drawn tables, framed paragraphs, newspaper pages, vertical, light-on-dark and photographed tables, the rule-index edge,
every validation error of find_blocks and restore_regions (raised before anything reaches a device), and the build of the
kernels."""
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
from oracle import ruled_pages as RP
from oracle.quad_regions import rectify

FONT = cv2.FONT_HERSHEY_DUPLEX
WORDS = "THE QUICK BROWN FOX JUMPS OVER A LAZY DOG PACK MY BOX WITH FIVE DOZEN JUGS".split()


def _img(ink, light=False):
    """A uint8 page of the boolean mask: ink 20 on 235, or the inverse."""
    img = np.where(ink[..., None], 20, 235).astype(np.uint8).repeat(3, axis=2)
    return 255 - img if light else img


def _text(shape, s, x, y):
    """The ink mask of the capitals ``s`` drawn at baseline (x, y) as test_pages.py draws them (DUPLEX, scale 1, thickness 2)."""
    m = np.zeros(shape, np.uint8)
    cv2.putText(m, s, (x, y), FONT, 1.0, 255, 2, cv2.LINE_8)
    return m > 0


def _line_of(rng, width):
    """Words of WORDS that fit in ``width`` pixels."""
    t = str(rng.choice(WORDS))
    while True:
        longer = t + " " + str(rng.choice(WORDS))
        if cv2.getTextSize(longer, FONT, 1.0, 2)[0][0] > width:
            return t
        t = longer


def _grid(rules, x0, y0, xs, ys, t=2):
    """2-pixel rules of a table at (x0, y0) whose column and row edges are x0 + xs[k] and y0 + ys[k]."""
    for y in ys:
        rules[y0 + y - t // 2:y0 + y - t // 2 + t, x0 + xs[0] - 1:x0 + xs[-1] + 1] = True
    for x in xs:
        rules[y0 + ys[0] - 1:y0 + ys[-1] + 1, x0 + x - t // 2:x0 + x - t // 2 + t] = True


def table(shape, rules, rng, x0, y0, n_rows, n_cols, cw=168, ch=47):
    """A ruled table of n_rows x n_cols cells of cw x ch at (x0, y0), each holding one short word: the cells' ink masks in
    reading order."""
    _grid(rules, x0, y0, [c * cw for c in range(n_cols + 1)], [r * ch for r in range(n_rows + 1)])
    return [_text(shape, str(rng.choice(WORDS))[:5], x0 + c * cw + 14, y0 + r * ch + 35)
            for r in range(n_rows) for c in range(n_cols)]


def table_page(n_rows=4, n_cols=3, seed=0, heading=True):
    """A heading over an n_rows x n_cols ruled table: (image, masks), masks the heading's (when drawn) then the cells'."""
    rng = np.random.default_rng(seed)
    top = 70 if heading else 24
    shape = (top + 47 * n_rows + 24, 48 + 168 * n_cols)
    rules = np.zeros(shape, bool)
    masks = [_text(shape, "HEADING OF THE TABLE", 24, 42)] if heading else []
    masks += table(shape, rules, rng, 24, top, n_rows, n_cols)
    return _img(rules | np.any(masks, axis=0)), masks


def framed_page(n_lines=5, seed=1):
    """A paragraph of n_lines inside a 2-pixel frame: (image, mask of the text)."""
    rng = np.random.default_rng(seed)
    shape = (60 + 33 * n_lines + 40, 560)
    rules = np.zeros(shape, bool)
    _grid(rules, 20, 20, [0, 520], [0, 33 * n_lines + 40])
    text = np.any([_text(shape, _line_of(rng, 470), 40, 72 + 33 * k) for k in range(n_lines)], axis=0)
    return _img(rules | text), text


def table_beside_column(seed=2):
    """A 3 x 2 table beside a free column of 6 lines 60 pixels to its right: (image, the cells' masks then the column's)."""
    rng = np.random.default_rng(seed)
    shape = (24 + 47 * 3 + 60, 48 + 2 * 168 + 60 + 300)
    rules = np.zeros(shape, bool)
    masks = table(shape, rules, rng, 24, 24, 3, 2)
    masks.append(np.any([_text(shape, _line_of(rng, 300), 24 + 2 * 168 + 60, 50 + 33 * k) for k in range(6)], axis=0))
    return _img(rules | np.any(masks, axis=0)), masks


def newspaper_page(seed=3):
    """A masthead over a rule, then two columns 16 pixels apart with a column rule in the gutter, each with two articles split
    after different lines by an article rule 10 pixels below the last line of the first: without the rules no white run is
    wide enough to cut.  (image, masks in reading order: masthead, then each column's articles)."""
    rng = np.random.default_rng(seed)
    cw, gutter, pitch = 300, 16, 33
    shape = (300, 40 + 2 * cw + gutter)
    rules = np.zeros(shape, bool)
    masks = [_text(shape, "THE DAILY JUGS", 20, 40)]
    rules[54:56, 20:shape[1] - 20] = True
    x_rule = 20 + cw + gutter // 2
    rules[60:shape[0] - 10, x_rule - 1:x_rule + 1] = True
    for c, split in enumerate((3, 2)):
        x = 20 + c * (cw + gutter)
        ys = [90 + pitch * k + (10 if k >= split else 0) for k in range(6)]
        rules[ys[split - 1] + 10:ys[split - 1] + 12, x:x + cw - 6] = True
        for part in (ys[:split], ys[split:]):
            masks.append(np.any([_text(shape, _line_of(rng, cw - 10), x, y) for y in part], axis=0))
    return _img(rules | np.any(masks, axis=0)), masks


def _inside(rect, shape):
    m = np.zeros(shape, bool)
    m[rect[1]:rect[3], rect[0]:rect[2]] = True
    return m


def _check_cells(img, res, masks, rule):
    """One block per mask in reading order, each holding its mask, no U pixel and exactly one line, unless a mask is a
    paragraph (then its block's lines are counted by the caller)."""
    assert len(res["blocks"]) == len(masks), res["blocks"]
    for blk, m in zip(res["blocks"], masks):
        assert not (m & ~_inside(blk, m.shape)).any(), blk
        assert not (rule & _inside(blk, rule.shape)).any(), blk


def _ink(img):
    g = B.grey(img)
    t = B.otsu(g)
    return g <= t if 2 * int((g <= t).sum()) <= g.size else g > t


# ---- U against OpenCV ----

def _cv_rules(ink, l):
    a = l // 2
    m = ink.astype(np.uint8)
    kw = dict(borderType=cv2.BORDER_CONSTANT, borderValue=0)
    h = cv2.dilate(cv2.erode(m, np.ones((1, l), np.uint8), anchor=(a, 0), **kw), np.ones((1, l), np.uint8), anchor=(l - 1 - a, 0), **kw)
    v = cv2.dilate(cv2.erode(m, np.ones((l, 1), np.uint8), anchor=(0, a), **kw), np.ones((l, 1), np.uint8), anchor=(0, l - 1 - a), **kw)
    return (h | v) > 0


@pytest.fixture
def no_ipp():
    before = cv2.ipp.useIPP()
    cv2.ipp.setUseIPP(False)
    yield
    cv2.ipp.setUseIPP(before)


def test_rule_pixels_equal_opencv_opening(no_ipp):
    """U is the OR of the openings of the ink by a 1 x l and an l x 1 segment (erode at anchor l // 2, dilate at l - 1 - l // 2,
    outside is paper), for odd and even l, on random and banded masks, masks whose ink touches every border, 1 x 1, 1 x N and
    N x 1 masks, and runs of exactly l and l - 1."""
    rng = np.random.default_rng(0)
    masks = [rng.random((37, 53)) < p for p in (0.3, 0.7, 0.95)]
    masks += [np.ones((40, 45), bool), np.ones((1, 1), bool), np.zeros((1, 1), bool), rng.random((1, 70)) < 0.9,
              rng.random((70, 1)) < 0.9]
    band = rng.random((60, 80)) < 0.5
    band[:, :3] = band[:, -3:] = band[:3] = band[-3:] = True
    masks.append(band)
    for l in range(2, 34):
        exact = np.zeros((3, l + 3), bool)
        exact[0, 1:1 + l] = exact[2, 2:1 + l] = True          # a run of l and one of l - 1
        for m in masks + [exact, exact.T]:
            np.testing.assert_array_equal(RP.rule_pixels(m, l), _cv_rules(m, l), err_msg=f"l={l}, shape={m.shape}")
        u = RP.rule_pixels(exact, l)
        assert u[0].sum() == l and u[2].sum() == 0 and (RP.rule_pixels(exact.T, l) == u.T).all()


# ---- known answers ----

def test_heading_over_a_ruled_table():
    """Without rules the table is one leaf, one "line"; with them the heading and each of the 12 cells is a block of one line."""
    img, masks = table_page(4, 3)
    plain = P.find_blocks(img)
    assert len(plain["blocks"]) == 2 and len(B.find_lines(img, plain["blocks"][1])["lines"]) == 1
    res = RP.find_blocks(img)
    rule = RP.rule_pixels(_ink(img), res["rule_length"])
    assert res["rule_length"] == 32 and res["rule_pixels"] == int(rule.sum()) > 0 and res["rejected"] == []
    _check_cells(img, res, masks, rule)
    assert all(len(B.find_lines(img, b)["lines"]) == 1 for b in res["blocks"])


def test_framed_paragraph_gives_its_lines():
    img, text = framed_page(5)
    plain = P.find_blocks(img)
    assert len(plain["blocks"]) == 1 and len(B.find_lines(img, plain["blocks"][0])["lines"]) == 1
    res = RP.find_blocks(img)
    assert len(res["blocks"]) == 1 and res["text_size"] == 24
    blk = res["blocks"][0]
    assert not (text & ~_inside(blk, text.shape)).any()
    assert not (RP.rule_pixels(_ink(img), 32) & _inside(blk, text.shape)).any()
    assert len(B.find_lines(img, blk)["lines"]) == 5


def test_table_beside_a_free_column():
    """The table's vertical rules are over half the page's height, so the page's first column attempt cuts at them: the cells
    read column by column, then the free column, a block of its 6 lines."""
    img, masks = table_beside_column()
    res = RP.find_blocks(img)
    _check_cells(img, res, [masks[k] for k in (0, 2, 4, 1, 3, 5, 6)], RP.rule_pixels(_ink(img), res["rule_length"]))
    assert [len(B.find_lines(img, b)["lines"]) for b in res["blocks"]] == [1] * 6 + [6]


def test_newspaper_rules_cut_columns_and_articles():
    img, masks = newspaper_page()
    assert len(P.find_blocks(img)["blocks"]) == 2
    res = RP.find_blocks(img)
    _check_cells(img, res, masks, RP.rule_pixels(_ink(img), res["rule_length"]))
    assert [len(B.find_lines(img, b)["lines"]) for b in res["blocks"]] == [1, 3, 3, 2, 4]


def test_vertical_table_reads_right_to_left():
    """The table page transposed and mirrored (the heading becomes the rightmost column) as a vertical page: the horizontal
    page's blocks mapped through the same transform, in the same order."""
    img, _ = table_page(4, 3)
    H = img.shape[0]
    t = np.ascontiguousarray(img.transpose(1, 0, 2)[:, ::-1])
    hor, ver = RP.find_blocks(img), RP.find_blocks(t, direction="vertical")
    assert len(ver["blocks"]) == 13
    assert ver["blocks"] == [(H - y1, x0, H - y0, x1) for x0, y0, x1, y1 in hor["blocks"]]
    assert all(len(B.find_lines(t, b, "vertical")["lines"]) == 1 for b in ver["blocks"])


def test_light_on_dark_table():
    img, _ = table_page(4, 3)
    res, inv = RP.find_blocks(img), RP.find_blocks(255 - img)
    assert inv["ink"] == "light" and inv["blocks"] == res["blocks"] and inv["rule_pixels"] == res["rule_pixels"]


def test_rule_index_at_exactly_half_the_extent():
    """A row whose U pixels are exactly half the node's width is a rule index and cuts however short its white run; one U pixel
    fewer leaves it white by its count alone, and the run of one is under the gap."""
    for run, leaves in ((20, 2), (19, 1)):
        ink = np.zeros((21, 40), bool)
        ink[2:9, 2:38:3] = ink[12:19, 2:38:3] = True
        ink[10, 0:run] = True
        rule = RP.rule_pixels(ink, 10)
        assert rule[10].sum() == run and rule.sum() == run
        assert len(RP.xy_cut(ink & ~rule, rule, False, 100, 100)) == leaves


def _photo(flat, corners, seed):
    """``flat`` warped by cv2.warpPerspective so that its corners land on ``corners`` over a darker noisy background."""
    rng = np.random.default_rng(seed)
    h, w = flat.shape[:2]
    c = np.float32(corners)
    Wc, Hc = int(c[:, 0].max()) + 110, int(c[:, 1].max()) + 110
    M = cv2.getPerspectiveTransform(np.float32([[0, 0], [w, 0], [w, h], [0, h]]) - 0.5, c - 0.5)
    page = cv2.warpPerspective(flat, M, (Wc, Hc), flags=cv2.INTER_LINEAR)
    cover = cv2.warpPerspective(np.full((h, w), 255, np.uint8), M, (Wc, Hc), flags=cv2.INTER_NEAREST) > 0
    bg = cv2.GaussianBlur(rng.integers(100, 140, (Hc, Wc)).astype(np.uint8), (5, 5), 0)[..., None].repeat(3, axis=2)
    img = np.where(cover[..., None], page, bg).astype(np.int16) + rng.integers(-6, 7, (Hc, Wc, 1))
    return np.clip(img, 0, 255).astype(np.uint8)


def photographed_table(seed=4):
    flat, _ = table_page(4, 3, seed=seed)
    h, w = flat.shape[:2]
    return _photo(flat, [(112, 118), (112 + w - 10, 110), (112 + w, 112 + h), (106, 116 + h - 6)], seed)


def test_photographed_table_under_quad_auto():
    img = photographed_table()
    quad = Q.accepted(Q.find_corners(img), img.shape)
    assert quad is not None
    res = RP.find_quad_blocks(img, quad)
    R = rectify(img, quad)
    assert res["size"] == (R.shape[1], R.shape[0]) and res["rule_length"] == RP.default_rule_length(*res["size"])
    assert len(res["blocks"]) == 13
    assert all(len(B.find_lines(R, b)["lines"]) == 1 for b in res["blocks"])


# ---- validation, work and build ----

def _no_launch(monkeypatch):
    def boom(*a, **k):
        raise AssertionError("a launch was reached")
    for f in ("find_page_quads", "find_blocks", "find_lines", "warp_perspective"):
        monkeypatch.setattr(ops, f, boom)
    monkeypatch.setattr(pipeline, "_device_images", boom)


@pytest.mark.parametrize("page, match", [
    (pipeline.TextPage(rules="on"), "rules must be None or 'auto', got 'on'"),
    (pipeline.TextPage(rules=True), "rules must be None or 'auto', got True"),
    (pipeline.TextPage(rules="auto", rule_length=1), r"rule_length must be an integer in \[2, 32767\], got 1"),
    (pipeline.TextPage(rules="auto", rule_length=32768), r"rule_length must be an integer in \[2, 32767\], got 32768"),
    (pipeline.TextPage(rules="auto", rule_length=40.0), r"rule_length must be an integer in \[2, 32767\], got 40.0"),
    (pipeline.TextPage(rules="auto", rule_length=True), r"rule_length must be an integer in \[2, 32767\], got True"),
    (pipeline.TextPage(rule_length=40), "rule_length is given, but rules is None"),
    (pipeline.TextPage(rules="auto", skew="auto"), "rules and skew are both given"),
    (pipeline.TextPage(rules="auto", skew=2.0), "rules and skew are both given"),
    (pipeline.TextPage(rules="auto", curve="auto"), "rules and curve are both given"),
])
def test_validation_errors_raise_before_any_launch(monkeypatch, page, match):
    _no_launch(monkeypatch)
    img = np.zeros((200, 240, 3), np.uint8)
    with pytest.raises(ValueError, match=r"image 0, page 1: " + match):
        pipeline.find_blocks([img], [[pipeline.TextPage(rules="auto"), page]])
    with pytest.raises(ValueError, match=r"image 0, region 1 \(a text page\): " + match):
        pipeline.restore_regions(None, None, None, [img], [[(0, 0, 4, 4), page]])


def test_work_memory_counts_the_rule_planes(monkeypatch):
    _no_launch(monkeypatch)
    pg = pipeline.TextPage(rules="auto")
    assert ops.rule_page_bytes(70, 40) == 4 * (40 * 3 + 70 * 2)
    assert pipeline._page_bytes(pg, (0, 0, 70, 40), False) == ops.page_bytes(70, 40) + ops.rule_page_bytes(70, 40)
    quad = pipeline.QuadRegion((10.0, 12.0), (200.0, 8.0), (210.0, 180.0), (6.0, 170.0))
    w_r, h_r = pipeline.quad_maps(quad, 1).size
    assert pipeline._page_bytes(pg._replace(quad=quad), (0, 0, 240, 200), False) == \
        3 * w_r * h_r + ops.page_bytes(w_r, h_r) + ops.rule_page_bytes(w_r, h_r)
    monkeypatch.setattr(ops, "PAGE_MAX_WORK", ops.page_bytes(240, 200) + ops.rule_page_bytes(240, 200) - 1)
    pipeline._check_page(pipeline.TextPage(), 200, 240, "p")
    with pytest.raises(ValueError, match=r"image 0, page 0: the page needs more than .* bytes of work memory"):
        pipeline.find_blocks([np.zeros((200, 240, 3), np.uint8)], [[pg]])


def test_ops_refuses_a_bad_rule_length():
    import torch
    img = torch.zeros((8, 8, 3), dtype=torch.uint8)
    for bad, skew in ((1, None), (32768, None), (True, None), (40, 2.0)):
        with pytest.raises(ValueError, match="find_blocks: page 0: rule_length"):
            ops.find_blocks([ops.PageItem(img, (0, 0, 8, 8), False, 0, skew=skew, rule_length=bad)])


def test_kernels_build_without_spills(tmp_path):
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    if not os.path.exists(nvcc):
        pytest.skip("nvcc not found")
    src = os.path.join(os.path.dirname(ops.__file__), "csrc", "block_ops.cu")
    r = subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-Xcompiler", "-fPIC",
                        "-DMN_BUILD", "-Xptxas", "-v", "-c", src, "-o", str(tmp_path / "b.o")], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    for kernel in ("rule_transpose_kernel", "rule_runs_kernel", "rule_merge_kernel", "page_count_kernel", "page_emit_kernel",
                   "page_blocks_kernel"):
        props = re.search(rf"Function properties for \S*{kernel}\S*\n(.*)\n", r.stderr)
        assert props, kernel
        assert "0 bytes spill stores, 0 bytes spill loads" in props.group(1), props.group(1)
