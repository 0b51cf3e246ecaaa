"""Reversed panels (DESIGN.md section 7b, "Reversed panels") on the host: the twin on drawn pages with light text on dark fills (a
headline banner, a ruled table with a shaded header row, a dark sidebar beside two columns with and without a dark photo, a
rounded button), its pinned limits (a bold glyph, a gradient bar), its exact thresholds, its invariants under transposition,
polarity and perspective, pages without panels; every validation error of find_blocks and restore_regions (raised before
anything reaches a device); the work memory; the constants; and the build of the kernels."""
import os
import re
import subprocess

import cv2
import numpy as np
import pytest

from marconet_b200 import _lib, ops, pipeline
from oracle import blocks as B
from oracle import figure_pages as FP
from oracle import pages as P
from oracle import panel_pages as PP
from oracle import quad_pages as Q
from oracle import ruled_pages as RP

from test_ruled_pages import _photo

PAPER, INK, FILL = 245, 20, 40
FONT = cv2.FONT_HERSHEY_SIMPLEX


def _put(img, s, xy, scale=0.8, grey=INK, thick=1):
    cv2.putText(img, s, xy, FONT, scale, (grey, grey, grey), thick, cv2.LINE_AA)


def banner_page():
    """An 800 x 600 page: a 741 x 91 dark banner with two white lines over six dark lines of text.  (image, banner rectangle)."""
    img = np.full((600, 800, 3), PAPER, np.uint8)
    for k in range(6):
        _put(img, "the quick brown fox jumps %d" % k, (40, 220 + 34 * k))
    cv2.rectangle(img, (30, 60), (770, 150), (60, 40, 30), -1)
    _put(img, "REVERSED HEADLINE TEXT", (60, 100), 0.9, 250, 2)
    _put(img, "a second reversed line", (60, 135), 0.8, 250, 2)
    return img, (30, 60, 771, 151)


def shaded_table(n_rows=4, n_cols=3):
    """A ruled table whose header cells are filled dark with a white word each, a 2-pixel white margin inside each cell's
    rules.  (image, header cell fills, body cells)."""
    cw, ch, x0, y0 = 180, 44, 30, 30
    img = np.full((y0 + ch * n_rows + 40, x0 + cw * n_cols + 40, 3), PAPER, np.uint8)
    heads, cells = [], []
    for r in range(n_rows):
        for c in range(n_cols):
            x, y = x0 + c * cw, y0 + r * ch
            if r == 0:
                img[y + 3:y + ch - 2, x + 3:x + cw - 2] = FILL
                heads.append((x + 3, y + 3, x + cw - 2, y + ch - 2))
                _put(img, "Head %d" % c, (x + 20, y + 30), 0.8, 250, 2)
            else:
                _put(img, "cell %d%d" % (r, c), (x + 20, y + 30))
                cells.append((x, y, x + cw, y + ch))
    for r in range(n_rows + 1):
        img[y0 + r * ch, x0:x0 + cw * n_cols + 1] = INK
    for c in range(n_cols + 1):
        img[y0:y0 + ch * n_rows + 1, x0 + c * cw] = INK
    return img, heads, cells


def blurred_photo(rng, h, w, lo=10, hi=120):
    """A dark photo: blurred noise spread over [lo, hi], so its greys are not flat."""
    z = cv2.GaussianBlur(rng.random((h, w)).astype(np.float32), (0, 0), 3)
    z = (z - z.min()) / (z.max() - z.min() + 1e-9)
    return (lo + (hi - lo) * z).astype(np.uint8)[..., None].repeat(3, axis=2)


def sidebar_page(photo=False, seed=3):
    """Two columns of dark lines and, at the right, a dark sidebar of 5 white lines; with ``photo`` a blurred-noise dark photo
    under the columns.  (image, sidebar rectangle, photo rectangle or None)."""
    rng = np.random.default_rng(seed)
    img = np.full((620, 1000, 3), PAPER, np.uint8)
    for col, x in enumerate((30, 330)):
        for k in range(8):
            _put(img, "column %d line %d text" % (col, k), (x, 60 + 30 * k), 0.7)
    side = (660, 40, 960, 330)
    img[side[1]:side[3], side[0]:side[2]] = FILL
    for k in range(5):
        _put(img, "sidebar line %d" % k, (680, 90 + 50 * k), 0.8, 250, 2)
    box = None
    if photo:
        box = (40, 330, 600, 580)
        img[box[1]:box[3], box[0]:box[2]] = blurred_photo(rng, box[3] - box[1], box[2] - box[0])
    return img, side, box


def button_page():
    """Two lines of text and a dark rounded-corner button with a white label."""
    img = np.full((300, 600, 3), PAPER, np.uint8)
    _put(img, "press the button below to go on", (30, 50))
    _put(img, "or read the small print here", (30, 85))
    cv2.rectangle(img, (160, 140), (440, 220), (FILL,) * 3, -1)
    for x, y in ((160, 140), (428, 140), (160, 208), (428, 208)):      # cut the corners round: paper, then a disc of fill
        img[y:y + 13, x:x + 13] = PAPER
    for cx, cy in ((172, 152), (428, 152), (172, 208), (428, 208)):
        cv2.circle(img, (cx, cy), 12, (FILL,) * 3, -1)
    _put(img, "CONTINUE", (220, 192), 1.0, 250, 2)
    return img, (160, 140, 441, 221)


def bold_glyph_page(glyph="I"):
    """Text lines and one bold glyph over 4 S high that passes as a panel."""
    img = np.full((300, 600, 3), PAPER, np.uint8)
    for k in range(4):
        _put(img, "small words on a line %d" % k, (30, 40 + 30 * k), 0.7)
    _put(img, glyph, (400, 260), 3.0, INK, 24)
    return img


def gradient_page():
    """Text lines and a bar filled with a horizontal gradient from 0 to 90 holding a white line."""
    img = np.full((300, 700, 3), PAPER, np.uint8)
    for k in range(3):
        _put(img, "plain text line number %d" % k, (30, 40 + 30 * k), 0.7)
    img[150:230, 20:680] = np.linspace(0, 90, 660).astype(np.uint8)[None, :, None]
    _put(img, "TEXT ON A GRADIENT BAR", (60, 200), 1.0, 250, 2)
    return img


def _inside(r, box):
    return box[0] <= r[0] and box[1] <= r[1] and r[2] <= box[2] and r[3] <= box[3]


def _light(res):
    return [b for b, p in zip(res["blocks"], res["polarities"]) if p == "light"]


def _lines(img, blocks, polarity):
    """The text lines the blocks hold together: find_lines' line rows of every block, in page rows, merged where they
    overlap (the words of one line are blocks of their own)."""
    rows = sorted((b[1] + y0, b[1] + y1) for b in blocks for _, y0, _, y1 in B.find_lines(img, b, polarity=polarity)["lines"])
    merged = []
    for y0, y1 in rows:
        if merged and y0 < merged[-1][1]:
            merged[-1][1] = max(merged[-1][1], y1)
        else:
            merged.append([y0, y1])
    return len(merged)


# ---- drawn pages ----

def test_banner_is_one_panel_of_light_blocks():
    img, banner = banner_page()
    res, plain = PP.find_blocks(img), P.find_blocks(img)
    assert plain["rejected"] == [banner]                # today: the banner is one rejected leaf
    assert res["panels"] == [banner] and res["panel_size"] == res["text_size"] == plain["text_size"]
    light = _light(res)
    assert light and all(_inside(b, banner) for b in light)
    assert _lines(img, light, "light") == 2
    assert [b for b, p in zip(res["blocks"], res["polarities"]) if p != "light"] == plain["blocks"]
    assert set(res["polarities"]) == {"light", "auto"} and all(_inside(r, banner) for r in res["rejected"])


def test_shaded_header_cells_are_light_one_line_blocks():
    img, heads, cells = shaded_table()
    res = PP.find_blocks(img, rules=True, rule_length=200)
    assert res["panels"] == heads
    light = _light(res)
    assert len(light) == len(heads) and all(_inside(b, h) for b, h in zip(light, heads))
    assert [len(B.find_lines(img, b, polarity="light")["lines"]) for b in light] == [1] * len(heads)
    dark = [b for b, p in zip(res["blocks"], res["polarities"]) if p != "light"]
    assert all(any(_inside(b, c) for c in cells) for b in dark)
    assert all(any(_inside(b, c) for b in dark) for c in cells)
    assert res["rule_pixels"] == RP.find_blocks(img, rule_length=200)["rule_pixels"]


@pytest.mark.parametrize("figures", [False, True])
def test_sidebar_lines_with_and_without_figures(figures):
    img, side, _ = sidebar_page()
    res = PP.find_blocks(img, figures=figures)
    assert res["panels"] == [(side[0], side[1], side[2], side[3])]
    light = _light(res)
    assert _lines(img, light, "light") == 5 and all(_inside(b, side) for b in light)
    if figures:
        assert res["figures"] == []


def test_dark_photo_stays_a_figure_and_is_no_panel():
    img, side, box = sidebar_page(photo=True)
    res = PP.find_blocks(img, figures=True)
    assert res["panels"] == [side]
    assert len(res["figures"]) == 1 and _inside(res["figures"][0], box) and _inside(box, res["figures"][0])
    assert sorted(FP.find_blocks(img)["figures"]) == sorted([side] + res["figures"])
    plain = PP.find_blocks(img)
    assert plain["panels"] == [side] and any(_inside(r, box) for r in plain["rejected"])
    assert _lines(img, _light(res), "light") == 5


def test_rounded_button_adds_its_label_and_no_corner():
    img, button = button_page()
    res = PP.find_blocks(img)
    assert res["panels"] == [button]
    light = _light(res)
    assert len(light) == 1 and _lines(img, light, "light") == 1
    x0, y0, x1, y1 = light[0]
    assert x0 > button[0] + 20 and x1 < button[2] - 20     # the label's block, no corner piece


def test_bold_glyph_panel_adds_no_block():
    """Pinned: a bold glyph over 4 S high is over half ink and flat, so it is a panel (today a rejected leaf); the paper
    around its stroke is solid in J and gives no block."""
    img = bold_glyph_page("I")
    res, plain = PP.find_blocks(img), P.find_blocks(img)
    assert len(res["panels"]) == 1 and res["panels"] == plain["rejected"]
    (gx0, gy0, gx1, gy1), = res["panels"]
    assert max(gx1 - gx0, gy1 - gy0) >= 4 * res["text_size"]
    assert _light(res) == [] and res["blocks"] == plain["blocks"]


def test_bold_ring_glyph_panel_adds_its_counter():
    """Pinned as a limit: the counter and the paper corners of a bold 'O' that passes as a panel are one leaf of J under half
    ink, so they add one light block inside the glyph."""
    img = bold_glyph_page("O")
    res, plain = PP.find_blocks(img), P.find_blocks(img)
    assert len(res["panels"]) == 1 and res["panels"] == plain["rejected"]
    light = _light(res)
    assert len(light) == 1 and _inside(light[0], res["panels"][0])
    assert [b for b in res["blocks"] if b not in light] == plain["blocks"]


def test_gradient_bar_is_not_a_panel():
    """Pinned as a limit: a gradient fill fails the flat test, and its text stays lost."""
    img = gradient_page()
    res = PP.find_blocks(img)
    assert res["panels"] == [] and _light(res) == []


# ---- exact thresholds ----

def _patch_page(patch):
    """Lines of text and the h x w grey ``patch`` (all of it ink) at (400, 60)."""
    img = np.full((200, 600, 3), PAPER, np.uint8)
    for k in range(3):
        _put(img, "text line %d" % k, (30, 40 + 30 * k), 0.7)
    h, w = patch.shape
    img[60:60 + h, 400:400 + w] = patch[..., None]
    return img, (400, 60, 400 + w, 60 + h)


def half_flat_patch(more):
    """A 20 x 20 patch, all ink: 200 pixels at the mode 30 and 200 spread over 60..99 (5 each), a flat count of exactly half;
    with ``more`` one of the spread pixels is at 30 too."""
    patch = np.full(400, 30, np.uint8)
    patch[200:] = np.repeat(np.arange(60, 100), 5)
    if more:
        patch[399] = 30
    return patch.reshape(20, 20)


def tied_mode_patch(near):
    """A 20 x 20 patch, all ink, whose greys 50 and 70 tie at 150 pixels each, so its mode is 50: the other 100 pixels at 30
    (a flat count of 150, under half), or with ``near`` at 45 (250, over half)."""
    patch = np.full(400, 50, np.uint8)
    patch[:150] = 70
    patch[150:250] = 45 if near else 30
    return patch.reshape(20, 20)


def threshold_pages():
    """[(image, panel_size, its panels)] at each exact threshold: the flat count at half and half + 1, the tied mode, and the
    shorter side at p and p - 1."""
    out = []
    for patch, p, panel in ((half_flat_patch(False), 20, False), (half_flat_patch(True), 20, True),
                            (tied_mode_patch(False), 20, False), (tied_mode_patch(True), 20, True),
                            (np.full((20, 30), FILL, np.uint8), 20, True), (np.full((20, 30), FILL, np.uint8), 21, False)):
        img, box = _patch_page(patch)
        out.append((img, p, [box] if panel else []))
    return out


def test_flat_count_of_exactly_half_is_not_a_panel():
    img, box = _patch_page(half_flat_patch(False))
    assert PP.find_blocks(img, panel_size=20)["panels"] == []
    img, box = _patch_page(half_flat_patch(True))         # one more pixel within 8 of the mode
    assert PP.find_blocks(img, panel_size=20)["panels"] == [box]


def test_mode_ties_go_to_the_smaller_grey():
    img, _ = _patch_page(tied_mode_patch(False))
    assert PP.find_blocks(img, panel_size=20)["panels"] == []
    img, box = _patch_page(tied_mode_patch(True))         # mode 50 (its tie with 70 goes to 50): flat 250
    assert PP.find_blocks(img, panel_size=20)["panels"] == [box]


def test_shorter_side_p_is_a_panel_and_p_minus_1_is_not():
    img, box = _patch_page(np.full((20, 30), FILL, np.uint8))
    assert PP.find_blocks(img, panel_size=20)["panels"] == [box]
    assert PP.find_blocks(img, panel_size=21)["panels"] == []


def test_threshold_pages_are_the_pinned_cases():
    for img, p, panels in threshold_pages():
        assert PP.find_blocks(img, panel_size=p)["panels"] == panels


# ---- equivalences ----

def _tr(H):
    return lambda rs: [(H - y1, x0, H - y0, x1) for x0, y0, x1, y1 in rs]


@pytest.mark.parametrize("make, kw", [(lambda: banner_page()[0], {}), (lambda: sidebar_page()[0], {}),
                                      (lambda: shaded_table()[0], dict(rules=True, rule_length=200))])
def test_transposed_page_gives_the_transposed_result(make, kw):
    img = make()
    t = np.ascontiguousarray(img.transpose(1, 0, 2)[:, ::-1])
    hor, ver = PP.find_blocks(img, **kw), PP.find_blocks(t, direction="vertical", **kw)
    tr = _tr(img.shape[0])
    assert ver["panels"] == tr(hor["panels"])
    assert sorted(zip(ver["blocks"], ver["polarities"])) == sorted(zip(tr(hor["blocks"]), hor["polarities"]))


def test_light_page_with_a_light_panel_gives_the_mirrored_result():
    img, _ = banner_page()
    res, inv = PP.find_blocks(img), PP.find_blocks(255 - img)
    assert inv["ink"] == "light" and res["ink"] == "dark"
    assert inv["polarities"] == [{"light": "dark"}.get(p, p) for p in res["polarities"]]
    assert {k: v for k, v in inv.items() if k not in ("ink", "threshold", "polarities")} == \
        {k: v for k, v in res.items() if k not in ("ink", "threshold", "polarities")}


def vertical_sidebar_page():
    """A horizontal page of dark lines with a dark panel holding a vertical sidebar: 3 columns of white square glyphs."""
    from test_mixed_pages import text
    rng = np.random.default_rng(5)
    img = np.full((520, 900, 3), PAPER, np.uint8)
    for k in range(10):
        _put(img, "a horizontal line of text %d" % k, (30, 50 + 40 * k), 0.8)
    m = np.zeros(img.shape[:2], bool)
    text(m, rng, 640, 60, 3, 12, vertical=True)
    img[30:470, 610:780] = FILL
    img[m] = 250
    return img, (610, 30, 780, 470)


def test_block_direction_finds_a_vertical_sidebar_inside_a_panel():
    img, panel = vertical_sidebar_page()
    res = PP.find_blocks(img, block_direction=True)
    assert res["panels"] == [panel]
    inside = [(b, d) for b, d, p in zip(res["blocks"], res["directions"], res["polarities"]) if p == "light"]
    assert len(inside) == 1 and inside[0][1] == "vertical"
    assert len(B.find_lines(img, inside[0][0], "vertical", polarity="light")["lines"]) == 3


def photographed_banner():
    img, _ = banner_page()
    h, w = img.shape[:2]
    return _photo(img, [(112, 118), (112 + w - 10, 110), (112 + w, 112 + h), (106, 116 + h - 6)], 10)


def test_photographed_banner_under_quad_auto():
    photo = photographed_banner()
    quad = Q.accepted(Q.find_corners(photo), photo.shape)
    assert quad is not None
    res = PP.find_quad_blocks(photo, quad)
    w_r, h_r = res["size"]
    assert len(res["panels"]) == 1
    x0, y0, x1, y1 = res["panels"][0]
    assert x1 - x0 > 0.85 * w_r and 60 < y1 - y0 < 120 and x1 <= w_r and y1 <= h_r
    light = _light(res)
    assert light and all(_inside(b, res["panels"][0]) for b in light)


@pytest.mark.parametrize("kw", [{}, dict(rules=True), dict(figures=True), dict(block_direction=True)])
def test_pages_without_panels_equal_panels_none(kw):
    from test_figure_pages import column_page
    img, _ = column_page("photo") if kw.get("figures") else (banner_page()[0][150:], None)
    res = PP.find_blocks(img, **kw)
    assert res["panels"] == [] and set(res["polarities"]) <= {"auto"}
    if kw.get("figures"):
        ref = FP.find_blocks(img)
    elif kw.get("rules"):
        ref = RP.find_blocks(img)
    elif kw.get("block_direction"):
        from oracle import mixed_pages as MP
        ref = MP.find_blocks(img)
    else:
        ref = P.find_blocks(img)
    assert {k: v for k, v in res.items() if k not in ("panel_size", "panels", "polarities")} == ref


# ---- validation, work and build ----

def _no_launch(monkeypatch):
    def boom(*a, **k):
        raise AssertionError("a launch was reached")
    for f in ("find_page_quads", "find_blocks", "find_lines", "warp_perspective"):
        monkeypatch.setattr(ops, f, boom)
    monkeypatch.setattr(pipeline, "_device_images", boom)


@pytest.mark.parametrize("page, match", [
    (pipeline.TextPage(panels="on"), "panels must be None or 'auto', got 'on'"),
    (pipeline.TextPage(panels=True), "panels must be None or 'auto', got True"),
    (pipeline.TextPage(panels="auto", panel_size=1), r"panel_size must be an integer in \[2, 32767\], got 1"),
    (pipeline.TextPage(panels="auto", panel_size=32768), r"panel_size must be an integer in \[2, 32767\], got 32768"),
    (pipeline.TextPage(panels="auto", panel_size=20.0), r"panel_size must be an integer in \[2, 32767\], got 20.0"),
    (pipeline.TextPage(panels="auto", panel_size=True), r"panel_size must be an integer in \[2, 32767\], got True"),
    (pipeline.TextPage(panel_size=20), "panel_size is given, but panels is None"),
    (pipeline.TextPage(panels="auto", skew="auto"), "panels and skew are both given"),
    (pipeline.TextPage(panels="auto", skew=2.0), "panels and skew are both given"),
    (pipeline.TextPage(panels="auto", curve="auto"), "panels and curve are both given"),
])
def test_validation_errors_raise_before_any_launch(monkeypatch, page, match):
    _no_launch(monkeypatch)
    img = np.zeros((200, 240, 3), np.uint8)
    with pytest.raises(ValueError, match=r"image 0, page 1: " + match):
        pipeline.find_blocks([img], [[pipeline.TextPage(panels="auto"), page]])
    with pytest.raises(ValueError, match=r"image 0, region 1 \(a text page\): " + match):
        pipeline.restore_regions(None, None, None, [img], [[(0, 0, 4, 4), page]])


def test_work_memory_counts_the_outline_plane_and_table(monkeypatch):
    _no_launch(monkeypatch)
    pg = pipeline.TextPage(panels="auto")
    assert ops.panel_page_bytes(70, 40, False) == 4 * 40 * 3 + 12 * 1024
    assert ops.panel_page_bytes(70, 40, True) == 12 * 1024
    assert pipeline._page_bytes(pg, (0, 0, 70, 40), False) == ops.page_bytes(70, 40) + ops.panel_page_bytes(70, 40, False)
    both = pg._replace(rules="auto", figures="auto")
    assert pipeline._page_bytes(both, (0, 0, 70, 40), False) == ops.page_bytes(70, 40) + ops.rule_page_bytes(70, 40) + \
        ops.figure_page_bytes(70, 40) + ops.panel_page_bytes(70, 40, True)
    quad = pipeline.QuadRegion((10.0, 12.0), (200.0, 8.0), (210.0, 180.0), (6.0, 170.0))
    w_r, h_r = pipeline.quad_maps(quad, 1).size
    assert pipeline._page_bytes(pg._replace(quad=quad), (0, 0, 240, 200), False) == \
        3 * w_r * h_r + ops.page_bytes(w_r, h_r) + ops.panel_page_bytes(w_r, h_r, False)
    monkeypatch.setattr(ops, "PAGE_MAX_WORK", ops.page_bytes(240, 200) + ops.panel_page_bytes(240, 200, False) - 1)
    pipeline._check_page(pipeline.TextPage(), 200, 240, "p")
    with pytest.raises(ValueError, match=r"image 0, page 0: the page needs more than .* bytes of work memory"):
        pipeline.find_blocks([np.zeros((200, 240, 3), np.uint8)], [[pg]])
    monkeypatch.setattr(ops, "PAGE_MAX_WORK", 2 * ops.page_bytes(240, 200) + ops.panel_page_bytes(240, 200, False) - 1)
    with pytest.raises(ValueError, match=r"the call's 2 text pages need more than"):
        pipeline.find_blocks([np.zeros((200, 240, 3), np.uint8)], [[pg, pipeline.TextPage()]])


def test_ops_refuses_a_bad_panel_size():
    import torch
    img = torch.zeros((8, 8, 3), dtype=torch.uint8)
    for bad, skew in ((1, None), (32768, None), (True, None), (-1, None), (40, 2.0), (0, 2.0)):
        with pytest.raises(ValueError, match="find_blocks: page 0: panel_size"):
            ops.find_blocks([ops.PageItem(img, (0, 0, 8, 8), False, 0, skew=skew, panel_size=bad)])


def test_constants_match_the_header():
    hdr = open(os.path.join(os.path.dirname(ops.__file__), "..", "include", "marconet_b200.h")).read()
    for name, value in (("MN_PAGE_PANELS", _lib.PAGE_PANELS), ("MN_PAGE_MAX_PANELS", _lib.PAGE_MAX_PANELS),
                        ("MN_PAGE_ERR_PANELS", _lib.PAGE_ERR_PANELS)):
        assert re.search(rf"#define {name} {value}\b", hdr), name
    assert (_lib.PAGE_PANELS, _lib.PAGE_MAX_PANELS, _lib.PAGE_ERR_PANELS) == (8, 1024, 4) == (8, PP.MAX_PANELS, 4)
    assert _lib.PAGE_PANELS not in (_lib.PAGE_RULES, _lib.PAGE_FIGURES, _lib.PAGE_DIRECTIONS)
    fields = [f for f, _ in _lib.PageResult._fields_]
    assert fields[-3:] == ["panel_size", "n_panels", "pad"] and _lib.PageResult.panel_size.offset == 44
    assert [f for f, _ in _lib.TextPage._fields_][-5:] == ["pans", "panel_size", "prows", "pdone", "pad3"]
    assert _lib.TextPage.pans.offset == _lib.TextPage.frows.offset + 4


def test_kernels_build_without_spills(tmp_path):
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    if not os.path.exists(nvcc):
        pytest.skip("nvcc not found")
    src = os.path.join(os.path.dirname(ops.__file__), "csrc", "block_ops.cu")
    r = subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-Xcompiler", "-fPIC",
                        "-DMN_BUILD", "-Xptxas", "-v", "-c", src, "-o", str(tmp_path / "b.o")], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    for kernel in ("panel_test_kernel", "panel_paint_kernel", "page_size_kernel", "figure_paint_kernel", "page_blocks_kernel"):
        props = re.search(rf"Function properties for \S*{kernel}\S*\n(.*)\n", r.stderr)
        assert props, kernel
        assert "0 bytes spill stores, 0 bytes spill loads" in props.group(1), props.group(1)
