"""Page turns (DESIGN.md section 7b, "Page turns") on the host: turn_quad's corners and their rectified crops against np.rot90,
the twin's turn on drawn pages at every quarter turn, every row of the vote table, its ties, every validation error of
find_blocks, restore_regions and flatten_pages (raised before anything reaches a device), the work memory, the constants and
the build of the kernel."""
import os
import re
import subprocess

import cv2
import numpy as np
import pytest

from marconet_b200 import _lib, ops, pipeline
from oracle import pages as P
from oracle import turn_pages as T
from oracle.quad_regions import rectify

from test_mixed_pages import INK, PAPER, S, TRACK, LEAD, image, magazine_page, text

TP, FP = pipeline.TextPage, pipeline.FlatPage


# ---- drawn pages ----

def paragraphs(seed=20):
    """Two paragraphs of pseudo-glyph lines, each with a 2-glyph indent and a short last line."""
    rng = np.random.default_rng(seed)
    m = np.zeros((420, 560), bool)
    y = 30
    for lines, last in ((5, 6), (4, 9)):
        text(m, rng, 30 + 2 * (S + TRACK), y, 1, 16)
        text(m, rng, 30, y + S + LEAD, lines - 1, 18, last=last)
        y += lines * (S + LEAD) + 30
    return image(m)


def heading_columns(seed=21):
    """A ragged-right cv2.putText heading over two columns of ragged lines."""
    rng = np.random.default_rng(seed)
    m = np.zeros((460, 760), bool)
    for c in range(2):
        x = 30 + c * 370
        for i, n in enumerate(rng.integers(6, 13, 9)):
            text(m, rng, x, 90 + i * (S + LEAD), 1, int(n))
    img = image(m)
    cv2.putText(img, "TURNED PAGES", (30, 55), cv2.FONT_HERSHEY_DUPLEX, 1.2, (INK,) * 3, 2, cv2.LINE_AA)
    return img


def newspaper(seed=22):
    """A vertical newspaper page: a horizontal headline over blocks of vertical columns of uneven length (top aligned)."""
    rng = np.random.default_rng(seed)
    m = np.zeros((640, 760), bool)
    text(m, rng, 40, 30, 1, 18, s=34, track=2)
    x = 720
    for cols in (4, 5):
        for c in range(cols):
            x -= S
            text(m, rng, x, 110, 1, int(rng.integers(8, 18)), vertical=True)
            x -= LEAD
        x -= 40
    return image(m)


PAGES = {"paragraphs": (paragraphs, "horizontal"), "heading": (heading_columns, "horizontal"),
         "newspaper": (newspaper, "vertical"), "magazine": (lambda: magazine_page()[0], "horizontal")}


def turned(img, k):
    return np.ascontiguousarray(np.rot90(img, k))


@pytest.mark.parametrize("k", range(4))
@pytest.mark.parametrize("name", sorted(PAGES))
def test_drawn_pages_find_their_turn(name, k):
    make, d = PAGES[name]
    up = make()
    img = turned(up, k)
    v = T.votes(img, direction=d)
    assert v["turn"] == 90 * k and v["votes"][k] > 0, v["votes"]
    H, W = img.shape[:2]
    R = T.upright(img, (0, 0, W, H), v["turn"])
    assert np.array_equal(R, up)
    assert P.find_blocks(R, direction=d)["blocks"] == P.find_blocks(up, direction=d)["blocks"]


# ---- turn_quad ----

@pytest.mark.parametrize("h, w", [(1, 9), (9, 1), (7, 10), (8, 11), (12, 12)])
def test_turn_quad_rectifies_to_rot90(h, w):
    rng = np.random.default_rng(h * 31 + w)
    img = rng.integers(0, 256, (h + 6, w + 8, 3), dtype=np.uint8)
    rect = (3, 2, 3 + w, 2 + h)
    crop = img[2:2 + h, 3:3 + w]
    for k, t in enumerate(pipeline.TURNS):
        q = pipeline.turn_quad(rect, t)
        assert tuple(q) == tuple(T.turn_quad(rect, k))
        assert np.array_equal(rectify(img, q), np.rot90(crop, -k))


def test_turn_quad_corners():
    x0, y0, x1, y1 = 2, 3, 50, 40
    want = {0: ((x0, y0), (x1, y0), (x1, y1), (x0, y1)), 90: ((x0, y1), (x0, y0), (x1, y0), (x1, y1)),
            180: ((x1, y1), (x0, y1), (x0, y0), (x1, y0)), 270: ((x1, y0), (x1, y1), (x0, y1), (x0, y0))}
    for t, q in want.items():
        assert tuple(pipeline.turn_quad((x0, y0, x1, y1), t)) == tuple((float(a), float(b)) for a, b in q)
    quad = pipeline.QuadRegion((10.5, 12.0), (200.0, 8.0), (210.0, 180.0), (6.0, 170.0))
    assert pipeline.turn_quad(quad, 90) == (quad.bl, quad.tl, quad.tr, quad.br)
    assert pipeline.turn_quad(quad, 270) == (quad.tr, quad.br, quad.bl, quad.tl)
    with pytest.raises(ValueError):
        pipeline.turn_quad((0, 0, 4, 4), 45)


# ---- the vote ----

def test_hand_made_leaf_statistics():
    """Three lines starting at columns 2, 0 and 0 and ending at 9, 7 and 4: E_lo = 2, E_hi = 0 + 2 + 5."""
    ink = np.zeros((12, 12), bool)
    for y, (a, b) in zip((1, 5, 9), ((2, 9), (0, 7), (0, 4))):
        ink[y:y + 2, a:b + 1] = True
    assert T.leaf_stats(ink, np.zeros_like(ink), (0, 0, 12, 12), False) == (3, 2, 7)
    assert T.leaf_stats(ink.T, np.zeros_like(ink), (0, 0, 12, 12), True) == (3, 2, 7)


def test_every_row_of_the_vote_table():
    """pipeline's table equals the twin's, and each row is the one rot90 gives: an upright leaf has D > 0."""
    assert pipeline._TURN_VOTE == T.VOTE
    lines = paragraphs()
    for page_v in (False, True):
        up = lines if not page_v else np.ascontiguousarray(np.rot90(lines, -1))    # a vertical page: columns top down
        for k in range(4):
            v = T.votes(turned(up, k), direction="vertical" if page_v else "horizontal")
            assert v["turn"] == 90 * k, (page_v, k, v["votes"])
            leaf_v = (k % 2 == 1) != page_v
            D = [e_hi - e_lo for _, e_lo, e_hi in v["stats"]]
            assert all(d == ("vertical" if leaf_v else "horizontal") for d in v["directions"])
            assert sum(abs(d) for d in D) == v["votes"][k] and pipeline._TURN_VOTE[(page_v, leaf_v, D[0] > 0)] == 90 * k


def _blank(h=120, w=200):
    return np.full((h, w, 3), PAPER, np.uint8)


def test_ties_and_pages_without_votes():
    assert pipeline.page_turn((0, 0, 0, 0)) == 0 and pipeline.page_turn((0, 5, 5, 0)) == 90
    assert pipeline.page_turn((3, 0, 0, 3)) == 0
    assert T.votes(_blank())["votes"] == (0, 0, 0, 0)
    rng = np.random.default_rng(3)
    m = np.zeros((80, 500), bool)
    text(m, rng, 20, 20, 1, 14)
    one = T.votes(image(m))
    assert one["votes"] == (0, 0, 0, 0) and one["turn"] == 0
    m = np.zeros((300, 600), bool)
    for i, n in enumerate((8, 14, 6, 12)):                  # centred lines: E_lo = E_hi
        text(m, rng, 300 - (n * (S + TRACK) - TRACK) // 2, 20 + i * (S + LEAD), 1, n, kind="whole")
    c = T.votes(image(m))
    assert c["votes"] == (0, 0, 0, 0) and c["turn"] == 0


# ---- results, validation, work, constants and build ----

def _no_launch(monkeypatch):
    def boom(*a, **k):
        raise AssertionError("a launch was reached")
    for f in ("find_page_quads", "find_blocks", "find_lines", "warp_perspective", "warp_affine", "even_light"):
        monkeypatch.setattr(ops, f, boom)
    monkeypatch.setattr(pipeline, "_device_images", boom)


BAD = [(TP(turn=True), "turn must be None, 0, 90, 180, 270 or 'auto', got True"),
       (TP(turn="90"), "turn must be None, 0, 90, 180, 270 or 'auto', got '90'"),
       (TP(turn=-90), r"turn .*, got -90"), (TP(turn=360), r"turn .*, got 360"), (TP(turn=45), r"turn .*, got 45"),
       (TP(turn=90.0), r"turn .*, got 90.0"),
       (TP(turn="auto", skew="auto"), "turn and skew are both given"),
       (TP(turn=90, skew=2.0), "turn and skew are both given"),
       (TP(turn=90, curve="auto"), "turn and curve are both given"),
       (TP(turn="auto", seals="auto"), "turn and seals are both given")]


@pytest.mark.parametrize("page, match", BAD)
def test_validation_errors_raise_before_any_launch(monkeypatch, page, match):
    _no_launch(monkeypatch)
    img = np.zeros((200, 240, 3), np.uint8)
    with pytest.raises(ValueError, match=r"image 0, page 1: " + match):
        pipeline.find_blocks([img], [[TP(turn="auto"), page]])
    with pytest.raises(ValueError, match=r"image 0, region 1 \(a text page\): " + match):
        pipeline.restore_regions(None, None, None, [img], [[(0, 0, 4, 4), page]])


@pytest.mark.parametrize("page, match", [(FP(turn=True), r"turn .*, got True"), (FP(turn=45), r"turn .*, got 45"),
                                         (FP(turn="auto", skew="auto"), "turn and skew are both given"),
                                         (FP(turn=90, curve="auto"), "turn and curve are both given"),
                                         (FP(quad="auto", spread="auto", turn="auto"), "turn and spread are both given")])
def test_flat_validation_errors_raise_before_any_launch(monkeypatch, page, match):
    _no_launch(monkeypatch)
    img = np.zeros((200, 240, 3), np.uint8)
    with pytest.raises(ValueError, match=r"image 0, page 1: " + match):
        pipeline.flatten_pages([img], [[FP(turn="auto"), page]])


def test_work_memory_limit_is_checked_before_any_launch(monkeypatch):
    _no_launch(monkeypatch)
    H = W = 20000                                           # the turned second pass's R passes the limit
    with pytest.raises(ValueError, match="work memory"):
        pipeline._check_page(TP(turn="auto"), H, W, "image 0, page 0")
    assert pipeline._check_page(TP(), H, W, "p") == (0, 0, W, H)


def test_work_memory():
    rect = (3, 5, 1203, 805)
    w, h = 1200, 800
    plain = pipeline._page_bytes(TP(), rect, False)
    table = ops.page_bytes(w, h, turns=True) - ops.page_bytes(w, h)
    assert table == ctypes_size() * ops.page_cap(w, h) + 16
    assert pipeline._page_bytes(TP(turn="auto"), rect, False) == plain + table + 3 * w * h
    q = pipeline.turn_quad(rect, 90)
    assert pipeline._page_bytes(TP(turn=90), rect, False) == pipeline._page_bytes(TP(quad=q), pipeline._quad_box(q), False)
    assert pipeline._page_bytes(TP(turn=0), rect, False) == plain


def ctypes_size():
    import ctypes
    return ctypes.sizeof(_lib.PageTurn)


def test_header_and_ctypes_constants():
    here = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    with open(os.path.join(here, "include", "marconet_b200.h")) as f:
        header = f.read()
    for name, value in (("MN_PAGE_TURNS", _lib.PAGE_TURNS), ("MN_PAGE_DIRS_TURN", _lib.PAGE_DIRS_TURN)):
        assert re.search(rf"#define {name} (\d+)", header).group(1) == str(value)
    assert _lib.PAGE_TURNS not in (_lib.PAGE_RULES, _lib.PAGE_FIGURES, _lib.PAGE_DIRECTIONS, _lib.PAGE_PANELS)
    assert ctypes_size() == 24 and ops.page_turn_dtype().itemsize == 24
    assert re.search(r"int32_t n_bands, pad;\s*int64_t e_lo, e_hi;\s*\} mn_page_turn;", header)


def test_kernel_builds_without_spills(tmp_path):
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    if not os.path.exists(nvcc):
        pytest.skip("nvcc not found")
    src = os.path.join(os.path.dirname(ops.__file__), "csrc", "block_ops.cu")
    r = subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-Xcompiler", "-fPIC",
                        "-DMN_BUILD", "-Xptxas", "-v", "-c", src, "-o", str(tmp_path / "b.o")], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    props = re.search(r"Function properties for \S*page_turn_kernel\S*\n(.*)\n.*Used (\d+) registers", r.stderr)
    assert props, r.stderr[-2000:]
    assert "0 bytes spill stores, 0 bytes spill loads" in props.group(1), props.group(1)
