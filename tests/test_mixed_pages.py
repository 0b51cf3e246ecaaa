"""Mixed directions (DESIGN.md section 7b, "Mixed directions") on the host: the twin on drawn pages of square pseudo-glyphs (a
vertical newspaper page with a horizontal headline and caption, a magazine page with a vertical sidebar, grid paragraphs,
single lines and columns, a ruled table, a page with a photo and a photographed page), its ties, its invariants under
transposition, polarity and pages of one direction; every validation error of find_blocks and restore_regions (raised before
anything reaches a device); the unchanged work memory; the constants; and the build of the kernel."""
import os
import re
import subprocess

import cv2
import numpy as np
import pytest

from marconet_b200 import _lib, ops, pipeline
from oracle import blocks as B
from oracle import mixed_pages as MP
from oracle import pages as P
from oracle import quad_pages as Q

from test_figure_pages import smooth_photo
from test_ruled_pages import _photo

INK, PAPER = 20, 235
S, TRACK, LEAD = 24, 3, 10                              # glyph size, tracking (between characters), leading (between lines)


def glyph(rng, s, kind=None):
    """An s x s pseudo-glyph: stems on both sides and a few seeded strokes across, whole or (kind "lr" / "tb") split into left
    and right or top and bottom parts, as many hanzi are."""
    kind = kind or str(rng.choice(["whole", "whole", "lr", "tb"]))
    t, gap = max(2, s // 10), max(2, s // 8)

    def part(h, w):
        m = np.zeros((h, w), bool)
        m[:, :t] = m[:, w - t:] = m[:t] = True
        for y in rng.integers(t, h - t, int(rng.integers(1, 3))):
            m[y:y + t] = True
        if w > 4 * t and rng.random() < 0.5:
            a = int(rng.integers(0, h // 2))
            m[a:a + int(rng.integers(h // 3, h - a + 1)), w // 2 - t // 2:w // 2 - t // 2 + t] = True
        return m

    m = np.zeros((s, s), bool)
    if kind == "lr":
        a = (s - gap) // 2
        m[:, :a], m[:, s - a:] = part(s, a), part(s, a)
    elif kind == "tb":
        a = (s - gap) // 2
        m[:a], m[s - a:] = part(a, s), part(a, s)
    else:
        m[:] = part(s, s)
    return m


def text(mask, rng, x, y, lines, chars, vertical=False, s=S, track=TRACK, lead=LEAD, kind=None, last=None):
    """Glyphs set on a grid into ``mask`` from (x, y): ``lines`` lines (columns when vertical) of ``chars`` characters (the last
    one of ``last``), ``track`` between characters and ``lead`` between lines.  Returns the ink rectangle (x0, y0, x1, y1)."""
    x1 = y1 = 0
    for i in range(lines):
        for j in range(last if last is not None and i == lines - 1 else chars):
            gx, gy = (x + i * (s + lead), y + j * (s + track)) if vertical else (x + j * (s + track), y + i * (s + lead))
            mask[gy:gy + s, gx:gx + s] |= glyph(rng, s, kind)
            x1, y1 = max(x1, gx + s), max(y1, gy + s)
    return x, y, x1, y1


def image(mask):
    return np.where(mask[..., None], INK, PAPER).astype(np.uint8).repeat(3, axis=2)


def newspaper_page(seed=0, photo=False):
    """A vertical newspaper page: a horizontal headline, three blocks of vertical columns (4, 3 and 5 columns) and a horizontal
    caption; with ``photo``, a photo at the left of the blocks.  (image, [(rect, direction, lines)] as drawn, in reading
    order)."""
    rng = np.random.default_rng(seed)
    m = np.zeros((760, 1000), bool)
    drawn = [(text(m, rng, 40, 30, 1, 25, s=36, track=2), "horizontal", 1)]
    x = 960
    for cols in (4, 3, 5):
        w = cols * S + (cols - 1) * LEAD
        x -= w
        drawn.append((text(m, rng, x, 120, cols, 16, vertical=True), "vertical", cols))
        x -= 44
    if photo:
        m[120:520, 40:x - 4] = False
    drawn.append((text(m, rng, 200, 620, 1, 22, s=22, track=2), "horizontal", 1))
    img = image(m)
    if photo:
        img[150:500, 60:x - 20] = smooth_photo(rng, 350, x - 80, 10, 120)
    return img, drawn


def magazine_page(seed=1):
    """A horizontal magazine page: two columns of horizontal lines and a vertical sidebar of three columns."""
    rng = np.random.default_rng(seed)
    m = np.zeros((480, 1000), bool)
    drawn = [(text(m, rng, 40, 40, 9, 12, last=7), "horizontal", 9),
             (text(m, rng, 40 + 12 * (S + TRACK) + 40, 40, 7, 12), "horizontal", 7)]
    drawn.append((text(m, rng, 40 + 24 * (S + TRACK) + 80, 40, 3, 14, vertical=True), "vertical", 3))
    return image(m), drawn


def blocks_of(res):
    """A twin result's blocks as [(rect, direction)]."""
    return list(zip(res["blocks"], res["directions"]))


def _inside(rect, blk):
    return blk[0] <= rect[0] and blk[1] <= rect[1] and rect[2] <= blk[2] and rect[3] <= blk[3]


def _holds_drawn(res, img, drawn):
    """Every drawn piece is one block of its drawn direction, in reading order, whose find_lines gives its drawn lines."""
    assert len(res["blocks"]) == len(drawn), (res["blocks"], drawn)
    for (blk, d), (rect, dd, n) in zip(blocks_of(res), drawn):
        assert _inside(rect, blk) and d == dd, (blk, d, rect, dd)
        assert len(B.find_lines(img, blk, d)["lines"]) == n, (blk, d, n)


# ---- drawn pages ----

def test_newspaper_page():
    img, drawn = newspaper_page()
    res = MP.find_blocks(img, direction="vertical")
    _holds_drawn(res, img, drawn)
    assert res["undecided"] == []
    plain = P.find_blocks(img, direction="vertical")
    assert res["blocks"] == plain["blocks"]                  # the same cut; without "auto" every block is vertical


def test_magazine_page():
    img, drawn = magazine_page()
    res = MP.find_blocks(img)
    _holds_drawn(res, img, drawn)
    assert res["undecided"] == [] and res["blocks"] == P.find_blocks(img)["blocks"]


@pytest.mark.parametrize("direction", ["horizontal", "vertical"])
@pytest.mark.parametrize("vertical", [False, True])
def test_grid_paragraphs(direction, vertical):
    """A paragraph of 5 lines (columns) of 12 characters, leading over tracking, is one block of its direction under either
    page direction."""
    rng = np.random.default_rng(2)
    m = np.zeros((460, 460), bool)
    rect = text(m, rng, 30, 30, 5, 12, vertical=vertical, track=2, lead=9)
    res = MP.find_blocks(image(m), direction=direction)
    assert len(res["blocks"]) == 1 and _inside(rect, res["blocks"][0])
    assert res["directions"] == ["vertical" if vertical else "horizontal"] and res["undecided"] == []


def _single(draw, h=200, w=700, seed=3):
    rng = np.random.default_rng(seed)
    m = np.zeros((h, w), bool)
    draw(m, rng)
    return image(m)


def _latin(text_, w=700):
    img = np.full((80, w, 3), PAPER, np.uint8)
    cv2.putText(img, text_, (10, 55), cv2.FONT_HERSHEY_DUPLEX, 1.0, (INK,) * 3, 2, cv2.LINE_AA)
    return img


def _t(img):
    """The transposed page, read as a vertical page: the columns of ``img`` become its rows, right to left."""
    return np.ascontiguousarray(img.transpose(1, 0, 2)[:, ::-1])


def _untransposed(img):
    """The page whose _t is ``img``."""
    return np.ascontiguousarray(img[:, ::-1].transpose(1, 0, 2))


SINGLE = {
    "touching line": (lambda: _single(lambda m, r: (text(m, r, 20, 30, 1, 20, track=0, kind="whole"),
                                                    text(m, r, 20, 100, 2, 20))), "horizontal", 2),
    "single column": (lambda: _single(lambda m, r: text(m, r, 40, 20, 1, 12, vertical=True), h=400, w=120), "vertical", 1),
    "unaligned columns": (lambda: _single(lambda m, r: [text(m, r, 20 + k * (S + LEAD), 20 + 9 * k, 1, 10, vertical=True)
                                                        for k in range(3)], h=340, w=160), "vertical", 1),
    "latin line": (lambda: _latin("THE QUICK BROWN FOX JUMPS"), "horizontal", 1),
    "latin transposed": (lambda: _t(_latin("THE QUICK BROWN FOX JUMPS")), "vertical", 1),
}


@pytest.mark.parametrize("direction", ["horizontal", "vertical"])
@pytest.mark.parametrize("case", sorted(SINGLE))
def test_single_band_cases(case, direction):
    """One block of its drawn direction under the page direction that keeps it whole; under the other one the cut may split
    it (a Latin line at its word gaps), and every piece still has the drawn direction."""
    draw, want, n = SINGLE[case]
    res = MP.find_blocks(draw(), direction=direction)
    assert res["directions"] == [want] * len(res["blocks"]) and res["undecided"] == [], res
    assert len(res["blocks"]) == n or direction != want and len(res["blocks"]) >= n


def _frames(boxes, h, w):
    """1-pixel rectangle outlines (x0, y0, x1, y1)."""
    m = np.zeros((h, w), bool)
    for x0, y0, x1, y1 in boxes:
        m[y0:y1, [x0, x1 - 1]] = True
        m[[y0, y1 - 1], x0:x1] = True
    return image(m)


TIES = {
    "rule 1: a square piece": lambda: _frames([(30, 30, 70, 70)], 100, 100),
    "rule 2: h = 2 b_c": lambda: _frames([(30, 30, 50, 70), (60, 30, 80, 70)], 100, 110),
    "rule 3: w = 2 b_r": lambda: _t(_frames([(30, 30, 50, 70), (60, 30, 80, 70)], 100, 110)),
    "rule 4: a 2 x 2 grid": lambda: _frames([(30, 30, 50, 50), (56, 30, 76, 50), (30, 56, 50, 76), (56, 56, 76, 76)], 110, 110),
    "equal leading and tracking": lambda: _single(lambda m, r: text(m, r, 20, 20, 4, 9, kind="whole", track=5, lead=5),
                                                  h=160, w=280),
}


@pytest.mark.parametrize("direction", ["horizontal", "vertical"])
@pytest.mark.parametrize("case", sorted(TIES))
def test_ties_are_undecided(case, direction):
    res = MP.find_blocks(TIES[case](), direction=direction)
    assert len(res["blocks"]) == 1 and res["undecided"] == [0] and res["directions"] == [direction], res


def test_rule_4_uses_mean_gaps():
    """Two lines of 20 characters with leading 6 and tracking 4 are horizontal: the mean gap between row bands exceeds the mean
    gap between column bands, however long the lines are."""
    img = _single(lambda m, r: text(m, r, 20, 20, 2, 20, kind="whole", track=4, lead=6), h=120, w=640)
    (rb, cb) = MP.leaf_bands(*(lambda ink: (ink, np.zeros_like(ink)))(B.grey(img) <= B.otsu(B.grey(img))),
                             (20, 20, 20 + 20 * 28 - 4, 20 + 54))
    assert rb == (2, S, 6) and cb == (20, S, 19 * 4)
    assert MP.find_blocks(img, direction="vertical")["directions"] == ["horizontal"]


def test_single_glyph_is_undecided():
    """A lone glyph is a solid square piece (rule 1's tie): it takes the page's direction."""
    for d in ("horizontal", "vertical"):
        res = MP.find_blocks(_single(lambda m, r: text(m, r, 30, 30, 1, 1, kind="whole"), h=90, w=90), direction=d)
        assert res["directions"] == [d] and res["undecided"] == [0]


def ruled_table(seed=4):
    """A 2 x 3 table drawn with rules, its cells holding a horizontal line or a vertical column of glyphs."""
    rng = np.random.default_rng(seed)
    m = np.zeros((460, 520), bool)
    drawn = []
    for r in range(2):
        for c in range(3):
            x, y = 20 + 160 * c, 20 + 210 * r
            if (r + c) % 2 == 0:
                drawn.append((text(m, rng, x + 12, y + 90, 1, 6, s=20, track=3), "horizontal", 1))
            else:
                drawn.append((text(m, rng, x + 70, y + 20, 1, 7, vertical=True, s=20, track=3), "vertical", 1))
    img = image(m)
    for r in range(3):
        cv2.line(img, (20, 20 + 210 * r), (500, 20 + 210 * r), (INK,) * 3, 2)
    for c in range(4):
        cv2.line(img, (20 + 160 * c, 20), (20 + 160 * c, 440), (INK,) * 3, 2)
    return img, drawn


def test_ruled_table_with_cells_of_both_directions():
    img, drawn = ruled_table()
    res = MP.find_blocks(img, rules=True)
    _holds_drawn(res, img, drawn)
    assert res["rule_pixels"] > 0 and res["undecided"] == []


def test_newspaper_page_with_a_photo():
    img, drawn = newspaper_page(photo=True)
    res = MP.find_blocks(img, direction="vertical", figures=True)
    assert len(res["figures"]) == 1
    _holds_drawn(res, img, drawn)


def photographed_newspaper():
    img, _ = newspaper_page()
    h, w = img.shape[:2]
    return _photo(img, [(112, 118), (112 + w - 10, 110), (112 + w, 112 + h), (106, 116 + h - 6)], 5)


def test_photographed_newspaper_under_quad_auto():
    photo = photographed_newspaper()
    quad = Q.accepted(Q.find_corners(photo), photo.shape)
    assert quad is not None
    res = MP.find_quad_blocks(photo, quad, direction="vertical")
    assert res["directions"] == ["horizontal", "vertical", "vertical", "vertical", "horizontal"] and res["undecided"] == []


# ---- invariants ----

def _transposed(rect, h):
    """A rectangle of an h-row page on its transposed page (_t)."""
    x0, y0, x1, y1 = rect
    return h - y1, x0, h - y0, x1


@pytest.mark.parametrize("make, direction", [(newspaper_page, "vertical"), (magazine_page, "horizontal")])
def test_transposed_page_swaps_directions(make, direction):
    img, _ = make()
    img = _untransposed(img) if direction == "vertical" else img    # a horizontal page whose _t is the drawn vertical one
    a = MP.find_blocks(img)
    b = MP.find_blocks(_t(img), direction="vertical")
    swap = {"horizontal": "vertical", "vertical": "horizontal"}
    assert b["blocks"] == [_transposed(r, img.shape[0]) for r in a["blocks"]]
    assert b["directions"] == [swap[d] for d in a["directions"]] and b["undecided"] == a["undecided"]


def test_light_on_dark_gives_the_same_result():
    img, _ = newspaper_page()
    a, b = MP.find_blocks(img, direction="vertical"), MP.find_blocks(255 - img, direction="vertical")
    assert {k: v for k, v in a.items() if k != "ink"} == {k: v for k, v in b.items() if k != "ink"}


def test_pages_of_one_direction_give_the_plain_result():
    rng = np.random.default_rng(6)
    m = np.zeros((500, 900), bool)
    text(m, rng, 30, 30, 6, 14)
    text(m, rng, 30 + 14 * (S + TRACK) + 40, 30, 8, 14)
    img = image(m)
    res = MP.find_blocks(img)
    assert res["directions"] == ["horizontal"] * 2 and res["undecided"] == []
    assert {k: v for k, v in res.items() if k not in ("block_direction", "undecided", "directions")} == P.find_blocks(img)


def random_mixed(rng):
    """A seeded random page of glyph grids of either direction, with random sizes, gaps, crop and page direction: (image, the
    twin's keyword arguments)."""
    h, w = int(rng.integers(160, 520)), int(rng.integers(200, 900))
    m = np.zeros((h, w), bool)
    for _ in range(int(rng.integers(1, 6))):
        s = int(rng.integers(12, 30))
        vertical = bool(rng.random() < 0.5)
        lines, chars = int(rng.integers(1, 5)), int(rng.integers(1, 12))
        track, lead = int(rng.integers(0, s // 3 + 1)), int(rng.integers(0, s))
        x, y = int(rng.integers(0, w - s)), int(rng.integers(0, h - s))
        sub = np.zeros((h + 40 * s, w + 40 * s), bool)
        text(sub, rng, x, y, lines, chars, vertical, s, track, lead)
        m |= sub[:h, :w]
    if rng.random() < 0.3:
        m |= rng.random((h, w)) < 0.002
    kw = dict(direction="vertical") if rng.random() < 0.5 else {}
    if rng.random() < 0.3:
        kw["rect"] = (int(rng.integers(0, w // 4)), int(rng.integers(0, h // 4)), w - int(rng.integers(0, w // 4)), h)
    return image(m), kw


def test_random_pages_give_every_kept_leaf_one_direction():
    rng = np.random.default_rng(7)
    seen = set()
    for _ in range(20):
        img, kw = random_mixed(rng)
        res = MP.find_blocks(img, **kw)
        assert len(res["directions"]) == len(res["blocks"])
        assert all(d in ("horizontal", "vertical") for d in res["directions"])
        page = kw.get("direction", "horizontal")
        assert all(res["directions"][k] == page for k in res["undecided"])
        plain = P.find_blocks(img, **kw)
        assert res["blocks"] == plain["blocks"] and res["rejected"] == plain["rejected"]
        seen |= set(res["directions"])
    assert seen == {"horizontal", "vertical"}


# ---- validation, work, constants and build ----

def _no_launch(monkeypatch):
    def boom(*a, **k):
        raise AssertionError("a launch was reached")
    for f in ("find_page_quads", "find_blocks", "find_lines", "warp_perspective"):
        monkeypatch.setattr(ops, f, boom)
    monkeypatch.setattr(pipeline, "_device_images", boom)


@pytest.mark.parametrize("page, match", [
    (pipeline.TextPage(block_direction="on"), "block_direction must be None or 'auto', got 'on'"),
    (pipeline.TextPage(block_direction=True), "block_direction must be None or 'auto', got True"),
    (pipeline.TextPage(block_direction="horizontal"), "block_direction must be None or 'auto', got 'horizontal'"),
    (pipeline.TextPage(block_direction="auto", skew="auto"), "block_direction and skew are both given"),
    (pipeline.TextPage(block_direction="auto", skew=2.0), "block_direction and skew are both given"),
    (pipeline.TextPage(block_direction="auto", curve="auto"), "block_direction and curve are both given"),
])
def test_validation_errors_raise_before_any_launch(monkeypatch, page, match):
    _no_launch(monkeypatch)
    img = np.zeros((200, 240, 3), np.uint8)
    with pytest.raises(ValueError, match=r"image 0, page 1: " + match):
        pipeline.find_blocks([img], [[pipeline.TextPage(block_direction="auto"), page]])
    with pytest.raises(ValueError, match=r"image 0, region 1 \(a text page\): " + match):
        pipeline.restore_regions(None, None, None, [img], [[(0, 0, 4, 4), page]])


def test_ops_refuses_bad_directions():
    import torch
    img = torch.zeros((8, 8, 3), dtype=torch.uint8)
    for bad, skew in ((1, None), ("auto", None), (True, 2.0)):
        with pytest.raises(ValueError, match="find_blocks: page 0: directions"):
            ops.find_blocks([ops.PageItem(img, (0, 0, 8, 8), False, 0, skew=skew, directions=bad)])


def test_work_memory_is_unchanged():
    pg = pipeline.TextPage(block_direction="auto")
    for rect in ((0, 0, 70, 40), (3, 5, 1203, 805)):
        for extra in ({}, dict(rules="auto"), dict(figures="auto"), dict(rules="auto", figures="auto")):
            assert pipeline._page_bytes(pg._replace(**extra), rect, False) == \
                pipeline._page_bytes(pipeline.TextPage(**extra), rect, False)
    quad = pipeline.QuadRegion((10.0, 12.0), (200.0, 8.0), (210.0, 180.0), (6.0, 170.0))
    assert pipeline._page_bytes(pg._replace(quad=quad), (0, 0, 240, 200), False) == \
        pipeline._page_bytes(pipeline.TextPage(quad=quad), (0, 0, 240, 200), False)


def test_header_and_ctypes_constants():
    here = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    with open(os.path.join(here, "include", "marconet_b200.h")) as f:
        header = f.read()
    for name, value in (("MN_PAGE_DIRECTIONS", _lib.PAGE_DIRECTIONS), ("MN_PAGE_VERTICAL", _lib.PAGE_VERTICAL),
                        ("MN_PAGE_UNDECIDED", _lib.PAGE_UNDECIDED)):
        assert re.search(rf"#define {name} (\d+)", header).group(1) == str(value)
    assert (_lib.PAGE_DIRECTIONS, _lib.PAGE_VERTICAL, _lib.PAGE_UNDECIDED) == (4, 16, 32)
    bits = (_lib.PAGE_RULES, _lib.PAGE_FIGURES, _lib.PAGE_DIRECTIONS)
    assert sum(bits) == 7 and not (_lib.PAGE_VERTICAL | _lib.PAGE_UNDECIDED) & (1 | 2 | 4 | _lib.PAGE_REJECTED)
    fields = dict((f[0], f[1]) for f in _lib.TextPage._fields_)
    assert "dirs" in fields and _lib.TextPage.dirs.offset == _lib.TextPage.rule_length.offset + 4


def test_kernel_builds_without_spills(tmp_path):
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    if not os.path.exists(nvcc):
        pytest.skip("nvcc not found")
    src = os.path.join(os.path.dirname(ops.__file__), "csrc", "block_ops.cu")
    r = subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-Xcompiler", "-fPIC",
                        "-DMN_BUILD", "-Xptxas", "-v", "-c", src, "-o", str(tmp_path / "b.o")], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    props = re.search(r"Function properties for \S*page_direction_kernel\S*\n(.*)\n.*Used (\d+) registers", r.stderr)
    assert props, r.stderr[-2000:]
    assert "0 bytes spill stores, 0 bytes spill loads" in props.group(1), props.group(1)
