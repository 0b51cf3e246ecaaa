"""Seals on the host (DESIGN.md section 7b, "Seals"): the numpy twin on drawn round and oval stamps (red and blue, rotated by
hand, stamped over black paragraphs), the thresholds of every constant on both sides, the layout copy's effect on the page
twin, CurvedRegion.from_arc's ovals, every refusal before any launch, the work memory, the constants against the header and
the new kernels' spills."""
import math
import os
import re
import subprocess

import cv2
import numpy as np
import pytest

from marconet_b200 import _lib, ops, pipeline
from oracle import pages as P
from oracle import seal_pages as S

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PAPER, INK = 245, 20
RED, BLUE = (200, 40, 40), (40, 60, 190)
FONT = cv2.FONT_HERSHEY_SIMPLEX


def seal_masks(h, w, cx, cy, rx, ry, rot=0.0, text=(200.0, -20.0), glyphs="ABCDEFGHIJ", star=True):
    """Boolean masks (ring, glyphs, star) of a stamp drawn on an h x w canvas: an ellipse ring of semi-axes (rx, ry), one
    rotated putText glyph per letter along its upper arc from angle text[0] to text[1] (degrees, reading clockwise, heads
    outward) at 0.72 of the radius, all turned by ``rot`` degrees, and a five-point star at its centre."""
    ring = np.zeros((h, w), np.uint8)
    t = max(2, min(rx, ry) // 18)
    cv2.ellipse(ring, (cx, cy), (rx - t // 2, ry - t // 2), 0, 0, 360, 255, t)
    gl = np.zeros((h, w), np.uint8)
    g = max(10, int(min(rx, ry) * 0.28))
    for j, ch in enumerate(glyphs):
        a = text[0] + (text[1] - text[0]) * (j + 0.5) / len(glyphs) + rot
        patch = np.zeros((2 * g, 2 * g), np.uint8)
        scale = cv2.getFontScaleFromHeight(FONT, g, 2)
        (tw, th), _ = cv2.getTextSize(ch, FONT, scale, 2)
        cv2.putText(patch, ch, (g - tw // 2, g + th // 2), FONT, scale, 255, 2)
        m = cv2.getRotationMatrix2D((g, g), a - 90, 1.0)
        patch = cv2.warpAffine(patch, m, (2 * g, 2 * g))
        px = int(round(cx + 0.70 * rx * math.cos(math.radians(a))))
        py = int(round(cy - 0.70 * ry * math.sin(math.radians(a))))
        y0, x0 = py - g, px - g
        gl[y0:y0 + 2 * g, x0:x0 + 2 * g] |= patch
    st = np.zeros((h, w), np.uint8)
    if star:
        r = 0.22 * min(rx, ry)
        pts = [(cx + (r if k % 2 == 0 else r / 2.5) * math.cos(math.radians(90 + 36 * k + rot)),
                cy - (r if k % 2 == 0 else r / 2.5) * math.sin(math.radians(90 + 36 * k + rot))) for k in range(10)]
        cv2.fillPoly(st, [np.round(np.array(pts)).astype(np.int32)], 255)
    return ring > 127, gl > 127, st > 127


def stamp(img, cx, cy, rx, ry, colour=RED, **kw):
    """Draws a stamp onto img; returns (box, ring, glyphs) in image pixels."""
    ring, gl, st = seal_masks(img.shape[0], img.shape[1], cx, cy, rx, ry, **kw)
    allm = ring | gl | st
    img[allm] = colour
    ys, xs = np.nonzero(allm)
    return (int(xs.min()), int(ys.min()), int(xs.max()) + 1, int(ys.max()) + 1), ring, gl


def paragraph(img, x, y, n, width=40, scale=0.7):
    for k in range(n):
        cv2.putText(img, ("the quick brown fox %d " % k * 3)[:width], (x, y + 30 * k), FONT, scale, (INK,) * 3, 1, cv2.LINE_AA)


def contract_page(h=700, w=900, rx=110, ry=110, colour=RED, over=True, rot=0.0):
    """A page of three paragraphs and a stamp, over the second one (``over``) or in the empty bottom right corner."""
    img = np.full((h, w, 3), PAPER, np.uint8)
    paragraph(img, 40, 60, 5)
    paragraph(img, 40, 300, 5)
    cx, cy = (260, 360) if over else (w - rx - 30, h - ry - 20)
    box, ring, gl = stamp(img, cx, cy, rx, ry, colour, rot=rot)
    return img, box, gl


def _angles(mask, box):
    """Parametric angles (degrees in [0, 360)) of the mask's pixels in the box's ellipse frame."""
    X, Y, A, B = S.ellipse_coords(box)
    ys, xs = np.nonzero(mask[box[1]:box[3], box[0]:box[2]])
    return np.degrees(np.arctan2(-Y[ys, 0] * A, X[0, xs] * B)) % 360


# ---- the twin on drawn stamps ----

@pytest.mark.parametrize("rx, ry, colour, rot", [(110, 110, RED, 0.0), (110, 110, BLUE, 20.0), (110, 110, RED, -20.0),
                                                 (130, 95, RED, 0.0), (130, 95, BLUE, 15.0), (95, 125, RED, -10.0)])
def test_drawn_seals_give_their_box_arc_and_band(rx, ry, colour, rot):
    img, box, gl = contract_page(rx=rx, ry=ry, colour=colour, rot=rot)
    t, boxes = S.page_seals(img)
    assert boxes == [box]
    s = next(s for s in t["seals"] if s["found"])
    assert s["ring"] >= S.RING_SECTORS and s["why"] == 0
    A, B = box[2] - box[0], box[3] - box[1]
    X, Y, _, _ = S.ellipse_coords(box)
    ys, xs = np.nonzero(gl[box[1]:box[3], box[0]:box[2]])
    rho = np.sqrt((X[0, xs] / A) ** 2 + (Y[ys, 0] / B) ** 2)
    assert s["k_bottom"] / 32 <= rho.min() + 1 / 32 and (s["k_top"] + 1) / 32 >= rho.max() - 1 / 32
    start, end = 5 * s["g0"], 5 * s["g0"] - 5 * (72 - s["n_gap"])
    r = (start - _angles(gl, box) + 5) % 360 - 5           # clockwise from start: the text lies in [0, start - end]
    assert -5 <= r.min() <= 5 and abs(r.max() - (start - end)) <= 5


def test_page_whose_text_misses_the_seal_keeps_its_blocks():
    img, box, _ = contract_page(over=False)
    plain = np.full_like(img, PAPER)
    paragraph(plain, 40, 60, 5)
    paragraph(plain, 40, 300, 5)
    t, boxes = S.page_seals(img)
    assert boxes == [box]
    assert P.find_blocks(S.layout_image(img, (0, 0, img.shape[1], img.shape[0]), boxes))["blocks"] == \
        P.find_blocks(plain)["blocks"]


def test_paragraph_under_a_stamp_keeps_its_line_count():
    from oracle import blocks as BL
    img, box, _ = contract_page(over=True)
    plain = np.full_like(img, PAPER)
    paragraph(plain, 40, 300, 5)
    rect = (30, 270, 700, 450)
    _, boxes = S.page_seals(img)
    assert boxes == [box]
    copy = S.layout_image(img, (0, 0, img.shape[1], img.shape[0]), boxes)
    assert not (S.seal_mask(copy[box[1]:box[3], box[0]:box[2]]) & S.seal_mask(img[box[1]:box[3], box[0]:box[2]])).any()
    assert len(BL.find_lines(plain, rect)["lines"]) == 5
    assert len(BL.find_lines(copy, rect)["lines"]) == 5
    assert len(BL.find_lines(img, rect)["lines"]) != 5          # the stamp's own ink cuts the profile without the copy


def test_red_headline_is_no_seal_and_stays_ink():
    img = np.full((1654, 1169, 3), PAPER, np.uint8)      # A4 at 141 dpi: the default seal size is 97 pixels
    cv2.putText(img, "PURCHASE CONTRACT", (60, 120), FONT, 2.4, RED, 6)
    paragraph(img, 40, 220, 4)
    t, boxes = S.page_seals(img)
    assert boxes == [] and t["n_seals"] == 0
    assert (S.layout_image(img, (0, 0, 1169, 1654), boxes) == img).all()


def test_ring_without_text_and_text_all_around():
    img = np.full((400, 400, 3), PAPER, np.uint8)
    stamp(img, 200, 200, 120, 120, glyphs="", star=True)
    t, boxes = S.page_seals(img)
    s = next(s for s in t["seals"] if s["found"])
    assert s["why"] == S.NO_BAND and s["k_top"] == -1
    img = np.full((400, 400, 3), PAPER, np.uint8)
    stamp(img, 200, 200, 120, 120, glyphs="ABCDEFGHIJKLMNOPQRSTUVWX", text=(90.0, -262.0))
    s = next(s for s in S.page_seals(img)[0]["seals"] if s["found"])
    assert s["k_top"] >= 0 and s["why"] == S.NO_GAP


def test_grey_stamp_of_chroma_63_is_not_found_and_64_is():
    for c, n in ((63, 0), (64, 1)):
        img = np.full((400, 400, 3), PAPER, np.uint8)
        stamp(img, 200, 200, 120, 120, colour=(120 + c, 120, 120))
        assert len(S.page_seals(img)[1]) == n


def test_channel_order_does_not_matter():
    img, box, _ = contract_page(rx=130, ry=100, colour=BLUE, rot=10.0)
    t = S.page_seals(img)
    for perm in ((2, 1, 0), (1, 2, 0)):
        assert S.page_seals(np.ascontiguousarray(img[..., perm])) == t


# ---- thresholds ----

def _cells_img(n_px):
    img = np.full((8, 8, 3), PAPER, np.uint8)
    for k in range(n_px):
        img[k, k] = RED
    return img


def test_cell_threshold():
    assert S.candidates(_cells_img(2), 1)[0] == 1 and S.candidates(_cells_img(1), 1)[0] == 0


@pytest.mark.parametrize("A, B, ok", [(60, 40, True), (61, 40, False), (40, 60, True), (40, 61, False)])
def test_ratio_threshold(A, B, ok):
    img = np.full((80, 80, 3), PAPER, np.uint8)
    img[5:5 + B, 5:5 + A] = RED
    assert S.candidates(img, 24)[0] == int(ok)


def test_size_threshold():
    img = np.full((80, 80, 3), PAPER, np.uint8)
    img[5:45, 5:45] = RED
    assert S.candidates(img, 40)[0] == 1 and S.candidates(img, 41)[0] == 0
    for side, n in ((4096, 1), (4097, 0)):             # a square outline of side MAX_SIDE and MAX_SIDE + 1
        img = np.full((4100, 4100, 3), PAPER, np.uint8)
        img[:side, :2] = img[:side, side - 2:side] = img[:2, :side] = img[side - 2:side, :side] = RED
        assert S.candidates(img, 8) [0] == n and S.MAX_SIDE == 4096


def test_radial_bin_is_exact_at_its_edges():
    A = B = np.int64(64)
    for k in (10, 26, 32, 33):                      # X = k A / 32 on the axis: rho = k / 32 exactly
        X = np.int64(k * 2)
        assert int(S.radial_bin(X, np.int64(0), A, B)) == k
        assert int(S.radial_bin(X - 1, np.int64(0), A, B)) == k - 1


def test_sector_boundaries_follow_the_table():
    for j in range(72):
        d = S.DIRS[j % 36] * (1 if j < 36 else -1)
        assert int(S.sector(d[0], d[1])) == j
        assert int(S.sector(d[0] + d[1] // 1000, d[1] - d[0] // 1000)) == (j - 1) % 72     # just clockwise of d_j
    assert int(S.sector(0, 0)) == 0 and int(S.sector(-5, 0)) == 36 and int(S.sector(0, -5)) == 54


BOX = (0, 0, 200, 200, 0)


def _painted(*layers):
    """A 200 x 200 crop whose pixels of radial bins ks and sectors secs, for each (ks, secs) of ``layers``, are seal red (the
    box of the whole crop is the candidate BOX)."""
    X, Y, A, B = S.ellipse_coords(BOX)
    k, sec = np.broadcast_arrays(S.radial_bin(X, Y, A, B), S.sector(X * B, -Y * A))
    img = np.full((200, 200, 3), PAPER, np.uint8)
    for ks, secs in layers:
        img[np.isin(k, list(ks)) & np.isin(sec, list(secs))] = RED
    return img


RING = (range(30, 32), range(72))


def test_ring_sector_threshold():
    for n, found in ((S.RING_SECTORS - 1, 0), (S.RING_SECTORS, 1)):
        r = S.seal_record(_painted((range(30, 32), range(n))), BOX)
        assert (r["ring"], r["found"]) == (n, found)


def test_gap_and_text_thresholds():
    band = range(20, 25)
    for n_text, why in ((71, S.NO_GAP), (70, 0), (S.MIN_TEXT - 1, S.SHORT), (S.MIN_TEXT, 0)):
        r = S.seal_record(_painted(RING, (band, range(n_text))), BOX)
        assert (r["k_bottom"], r["k_top"], r["n_gap"], r["why"]) == (20, 24, 72 - n_text, why)
    r = S.seal_record(_painted(RING), BOX)
    assert (r["found"], r["why"], r["k_top"]) == (1, S.NO_BAND, -1)


def test_ring_band_and_arc_thresholds():
    area = np.full(S.BINS, 3200, np.int64)
    ink = np.zeros(S.BINS, np.int64)
    ink[30:33] = 800                                 # 4 ink == area: the ring
    ink[20:25] = 100                                 # 32 ink == area: the band
    assert S.band(ink, area) == (20, 24)
    ink2 = ink.copy()
    ink2[20:25] = 99                                 # 32 ink < area: no band
    assert S.band(ink2, area) is None
    ink3 = ink.copy()
    ink3[30:33] = 799                                # no ring run
    assert S.band(ink3, area) is None
    ink4 = ink.copy()
    ink4[8:25] = 100                                 # the band stops at k = 10
    ink4[25] = 0
    assert S.band(ink4, area) == (10, 24)
    sec = np.zeros(72, np.int64)
    sec[10] = 500
    sec[30] = 1                                      # band ink 501: 720 * 1 = max(720, 501), not empty
    assert S.arc_gap(sec) == (31, 51)
    sec[30] = 0
    assert S.arc_gap(sec) == (11, 71)
    sec[:] = 0
    sec[10:20] = 100
    sec[30] = 2                                      # band ink 1002: 720 * 2 >= 1002, not empty
    assert S.arc_gap(sec) == (31, 51)
    sec[30] = 1                                      # band ink 1001: 720 * 1 < 1001, empty
    assert S.arc_gap(sec) == (20, 62)
    sec = np.zeros(72, np.int64)
    sec[:71] = 5
    assert S.arc_gap(sec) == (71, 1)
    sec = np.zeros(72, np.int64)
    sec[:9] = 5
    assert S.arc_gap(sec) == (9, 63)


def test_arc_gap_ties_go_to_the_smallest_start():
    sec = np.ones(72, np.int64) * 10
    sec[5:10] = 0
    sec[40:45] = 0
    assert S.arc_gap(sec) == (5, 5)


# ---- from_arc ----

def test_from_arc_pair_equals_scalar_and_ovals_lie_on_their_ellipse():
    a = pipeline.CurvedRegion.from_arc(100.0, 80.0, 50.0, 30.0, 200.0, -20.0)
    b = pipeline.CurvedRegion.from_arc(100.0, 80.0, (50.0, 50.0), (30.0, 30.0), 200.0, -20.0)
    assert a == b
    c = pipeline.CurvedRegion.from_arc(100.0, 80.0, (60.0, 40.0), (30.0, 20.0), 200.0, -20.0)
    for curve, (rx, ry) in ((c.top, (60.0, 40.0)), (c.bottom, (30.0, 20.0))):
        for x, y in curve[::3]:
            assert abs(((x - 100) / rx) ** 2 + ((y - 80) / ry) ** 2 - 1) < 1e-12


def _entries(img, seal_size=None):
    """pipeline._seal_entries of the twin's seal table of a whole image."""
    t = S.find_seals(img, seal_size or S.default_seal_size(img.shape[1], img.shape[0]))
    tab = np.zeros((), ops.seal_table_dtype())
    tab["n_cand"], tab["n_seals"] = t["n_cand"], t["n_seals"]
    for j, r in enumerate(t["seals"]):
        for f, v in r.items():
            tab["seal"][j][f] = v
    return pipeline._seal_entries(tab, 0, 0, img.shape[:2])


@pytest.mark.parametrize("rx, ry, rot, text", [(130, 95, 0.0, (200.0, -20.0)), (130, 100, 0.0, (210.0, -30.0)),
                                               (95, 130, 20.0, (200.0, -20.0)), (130, 95, -20.0, (240.0, -60.0)),
                                               (120, 120, 0.0, (225.0, -45.0)), (135, 90, 10.0, (250.0, -70.0))])
def test_found_arcs_pass_the_curved_planner(rx, ry, rot, text):
    img = np.full((700, 900, 3), PAPER, np.uint8)
    paragraph(img, 40, 60, 5)
    stamp(img, 450, 360, rx, ry, RED, rot=rot, text=text, glyphs="ABCDEFGHIJKLMN")
    (e,) = _entries(img)
    assert e["arc"] is not None and "why" not in e
    start, end = e["arc"]
    for scale in (1, 2, 4):
        pipeline.plan_regions([img.shape[:2]], [[e["region"]]], None, None, scale)
    assert len(e["region"].top) == 3 * pipeline.arc_segments((e["box"][2] - e["box"][0]) / 2, (e["box"][3] - e["box"][1]) / 2,
                                                             start, end) + 1


def test_arc_segments_keep_every_ruling_turn_under_90_degrees():
    assert pipeline.arc_segments(100, 100, 160, 0) == 2 and pipeline.arc_segments(100, 100, 180, 0) == 3
    assert pipeline.arc_segments(100, 100, 225, -45) == 4                # 3 segments of exactly 90 degrees on a circle
    assert pipeline.arc_segments(130, 95, 200, -20) == 4                 # 3 segments turn by 90.8 degrees on this oval
    for rx, ry in ((130, 95), (120, 90), (150, 100), (100, 150), (100, 100)):        # 4:3, 3:2 both ways, a circle
        for span in range(45, 320, 5):
            for start in range(0, 360, 15):
                k = pipeline.arc_segments(rx, ry, start, start - span)
                reg = pipeline.CurvedRegion.from_arc(500.0, 500.0, (0.9 * rx, 0.9 * ry), (0.6 * rx, 0.6 * ry), start, start - span,
                                                     segments=k)
                pipeline._plan_curved(reg, 1000, 1000, 1, "arc")
    with pytest.raises(ValueError, match=r"segments must be an integer in \[3, 8\], got 2"):
        pipeline.CurvedRegion.from_arc(0.0, 0.0, 2.0, 1.0, 200, -20, segments=2)


# ---- validation, work and build ----

def _no_launch(monkeypatch):
    def boom(*a, **k):
        raise AssertionError("a launch was reached")
    for f in ("find_page_quads", "find_blocks", "find_lines", "warp_perspective"):
        monkeypatch.setattr(ops, f, boom)
    monkeypatch.setattr(pipeline, "_device_images", boom)


@pytest.mark.parametrize("page, match", [
    (pipeline.TextPage(seals="on"), "seals must be None or 'auto', got 'on'"),
    (pipeline.TextPage(seals="auto", seal_size=7), r"seal_size must be an integer in \[8, 4096\], got 7"),
    (pipeline.TextPage(seals="auto", seal_size=4097), r"seal_size must be an integer in \[8, 4096\], got 4097"),
    (pipeline.TextPage(seals="auto", seal_size=20.0), r"seal_size must be an integer in \[8, 4096\], got 20.0"),
    (pipeline.TextPage(seals="auto", seal_size=True), r"seal_size must be an integer in \[8, 4096\], got True"),
    (pipeline.TextPage(seal_size=20), "seal_size is given, but seals is None"),
    (pipeline.TextPage(seals="auto", skew="auto"), "seals and skew are both given .* flatten_pages"),
    (pipeline.TextPage(seals="auto", curve="auto"), "seals and curve are both given .* flatten_pages"),
    (pipeline.TextPage(seals="auto", quad="auto"), "seals and quad are both given .* flatten_pages"),
    (pipeline.TextPage(seals="auto", polarity="light"), "seals are asked for on a page of polarity 'light'"),
])
def test_page_refusals_before_any_launch(monkeypatch, page, match):
    _no_launch(monkeypatch)
    img = np.zeros((200, 240, 3), np.uint8)
    with pytest.raises(ValueError, match=r"image 0, page 1: " + match):
        pipeline.find_blocks([img], [[pipeline.TextPage(seals="auto"), page]])
    with pytest.raises(ValueError, match=r"image 0, region 1 \(a text page\): " + match):
        pipeline.restore_regions(None, None, None, [img], [[pipeline.TextPage(seals="auto"), page]])


@pytest.mark.parametrize("blk, match", [
    (pipeline.TextBlock((0, 0, 100, 100), seals=((0, 0, 0, 10),)), "is empty, outside"),
    (pipeline.TextBlock((0, 0, 100, 100), seals=((0, 0, 10, 201),)), "is empty, outside"),
    (pipeline.TextBlock((0, 0, 100, 100), seals=((0, 0, 10.0, 10),)), "integer boxes"),
    (pipeline.TextBlock((0, 0, 100, 100), seals=((0, 0, 10),)), "integer boxes"),
    (pipeline.TextBlock((0, 0, 100, 100), seals=((0, 0, 10, 10),) * 65), "65 seals exceed the 64"),
    (pipeline.TextBlock((0, 0, 100, 100), seals=((0, 0, 10, 10),), skew=2.0), "seals and skew are both given"),
    (pipeline.TextBlock((0, 0, 100, 100), seals=((0, 0, 10, 10),), curve="auto"), "seals and curve are both given"),
    (pipeline.TextBlock((0, 0, 100, 100), seals=((0, 0, 10, 10),), polarity="light"), "polarity 'light'"),
])
def test_block_refusals_before_any_launch(monkeypatch, blk, match):
    _no_launch(monkeypatch)
    img = np.zeros((200, 240, 3), np.uint8)
    with pytest.raises(ValueError, match=r"image 0, block 0: .*" + match):
        pipeline.find_lines([img], [[blk]])


def test_a_wide_seal_box_is_refused():
    img = np.zeros((10, 5000, 3), np.uint8)
    with pytest.raises(ValueError, match="side over 4096"):
        pipeline.find_lines([img], [[pipeline.TextBlock((0, 0, 100, 10), seals=((0, 0, 4097, 10),))]])


def test_ops_refuses_a_bad_seal_size():
    with pytest.raises(ValueError, match=r"seal_size 7 is not an integer in \[8, 4096\]"):
        ops._check_page_options(ops.PageItem(None, None, False, 0, seal_size=7), "p")
    with pytest.raises(ValueError, match="seal_size 24 is not"):
        ops._check_page_options(ops.PageItem(None, None, False, 0, skew="auto", seal_size=24), "p")


def test_work_memory_counts_the_copy_and_the_cells(monkeypatch):
    w, h = 240, 200
    assert ops.page_bytes(w, h, seals=True) - ops.page_bytes(w, h) == ops.seal_bytes(w, h)
    cells = 60 * 50
    assert ops.seal_bytes(w, h) >= 3 * w * h + 20 * cells + ctypes_size("SealTable")
    _no_launch(monkeypatch)
    img = np.zeros((h, w, 3), np.uint8)
    monkeypatch.setattr(ops, "PAGE_MAX_WORK", ops.page_bytes(w, h, seals=True) - 1)
    with pytest.raises(ValueError, match="work memory"):
        pipeline.find_blocks([img], [[pipeline.TextPage(seals="auto")]])
    pipeline._check_page(pipeline.TextPage(), h, w, "page")           # the same page without seals fits


def ctypes_size(name):
    import ctypes
    return ctypes.sizeof(getattr(_lib, name))


def test_constants_match_the_header():
    src = open(os.path.join(ROOT, "include", "marconet_b200.h")).read()

    def define(name):
        return int(re.search(r"#define %s (-?\d+)" % name, src).group(1))
    for name, value in (("MN_PAGE_SEALS", _lib.PAGE_SEALS), ("MN_PAGE_MAX_SEALS", _lib.PAGE_MAX_SEALS),
                        ("MN_SEAL_ERR_SEALS", _lib.SEAL_ERR_SEALS), ("MN_SEAL_NO_BAND", S.NO_BAND),
                        ("MN_SEAL_NO_GAP", S.NO_GAP), ("MN_SEAL_SHORT", S.SHORT), ("MN_SEAL_CHROMA", S.CHROMA),
                        ("MN_SEAL_CELL", S.CELL), ("MN_SEAL_CELL_MIN", S.CELL_MIN), ("MN_SEAL_MAX_SIDE", S.MAX_SIDE),
                        ("MN_SEAL_BINS", S.BINS), ("MN_SEAL_SECTORS", S.SECTORS), ("MN_SEAL_RING_K", S.RING_K),
                        ("MN_SEAL_RING_SECTORS", S.RING_SECTORS), ("MN_SEAL_RING_DENSITY", S.RING_DENSITY),
                        ("MN_SEAL_BAND_DENSITY", S.BAND_DENSITY), ("MN_SEAL_BAND_MIN_K", S.BAND_MIN_K),
                        ("MN_SEAL_EMPTY_DIV", S.EMPTY_DIV), ("MN_SEAL_MIN_GAP", S.MIN_GAP), ("MN_SEAL_MIN_TEXT", S.MIN_TEXT)):
        assert define(name) == value, name
    assert _lib.PAGE_SEALS not in (_lib.PAGE_RULES, _lib.PAGE_FIGURES, _lib.PAGE_DIRECTIONS, _lib.PAGE_PANELS)
    dirs = re.search(r"#define MN_SEAL_DIRS \{(.*?)\}\}", src, re.S).group(1).replace("\\", "")
    pairs = [tuple(int(v) for v in p.split(",")) for p in re.findall(r"\{?(-?\d+, -?\d+)", dirs)]
    assert pairs == [tuple(int(v) for v in d) for d in S.DIRS]
    assert ops.seal_table_dtype().itemsize == ctypes_size("SealTable") == 16 + 64 * 64


def test_seal_kernels_do_not_spill(tmp_path):
    nvcc = "/usr/local/cuda/bin/nvcc" if os.path.isfile("/usr/local/cuda/bin/nvcc") else "nvcc"
    try:
        out = subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-Xcompiler", "-fPIC",
                              "-DMN_BUILD", "-I", os.path.join(ROOT, "include"), "-Xptxas", "-v", "-c",
                              os.path.join(ROOT, "marconet_b200", "csrc", "block_ops.cu"), "-o", str(tmp_path / "b.o")],
                             capture_output=True, text=True, timeout=600)
    except FileNotFoundError:
        pytest.skip("nvcc is not installed")
    assert out.returncode == 0, out.stdout + out.stderr
    text = out.stdout + out.stderr
    seen = 0
    for m in re.finditer(r"Function properties for (\S+)\n\s+(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes "
                         r"spill loads", text):
        if "seal_" in m.group(1):
            seen += 1
            assert m.group(3) == m.group(4) == "0", m.group(1)
    assert seen == 6


def test_sealed_blocks_count_their_copies_before_any_launch(monkeypatch):
    _no_launch(monkeypatch)
    img = np.zeros((200, 240, 3), np.uint8)
    blk = pipeline.TextBlock((0, 0, 240, 200), seals=((10, 10, 60, 60),))
    assert ops.seal_block_bytes(240, 200) >= 3 * 240 * 200 + ctypes_size("SealTable")
    monkeypatch.setattr(ops, "PAGE_MAX_WORK", 2 * ops.seal_block_bytes(240, 200) - 1)
    with pytest.raises(ValueError, match=r"image 0, block 1: the call's sealed blocks up to this one need \d+ bytes of layout "
                                         r"copies, over the \d+ a call may use"):
        pipeline.find_lines([img], [[blk, blk, pipeline.TextBlock((0, 0, 240, 200))]])
    with pytest.raises(ValueError, match=r"image 0, region 1 \(a text block\): the call's sealed blocks"):
        pipeline.restore_regions(None, None, None, [img], [[blk, blk]])


def test_ops_refuses_a_sealed_skewed_block():
    import torch
    img = torch.zeros((20, 20, 3), dtype=torch.uint8)
    with pytest.raises(ValueError, match="a sealed block is level"):
        ops.find_lines([(img, (0, 0, 20, 20), False, 0, None, None, None, 2.0, 10.0, [(0, 0, 10, 10)])])
