"""Seal centre lines on the host (DESIGN.md section 7b, "Seal centre lines"): the numpy twin on drawn company, invoice and
receipt stamps (red and blue, turned by hand), every constant on both sides of its threshold, the planner on the found line
regions, every refusal before any launch, the work memory, the constants against the header and the new kernel's spills."""
import math
import os
import re
import subprocess

import cv2
import numpy as np
import pytest

from marconet_b200 import _lib, ops, pipeline
from oracle import seal_lines as L
from oracle import seal_pages as S

from test_seal_pages import BLUE, FONT, PAPER, RED, _angles, _painted, paragraph, stamp

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def inner_line(h, w, cx, cy, text, dy, gh, rot=0.0):
    """Boolean mask of one putText line of glyph height gh centred dy pixels below (cx, cy), turned by ``rot`` degrees
    counter-clockwise on screen about (cx, cy)."""
    m = np.zeros((h, w), np.uint8)
    scale = cv2.getFontScaleFromHeight(FONT, int(gh), 2)
    (tw, th), _ = cv2.getTextSize(text, FONT, scale, 2)
    cv2.putText(m, text, (int(cx - tw / 2), int(cy + dy + th / 2)), FONT, scale, 255, 2)
    if rot:
        m = cv2.warpAffine(m, cv2.getRotationMatrix2D((cx, cy), rot, 1.0), (w, h))
    return m > 127


def seal_page(rx=110, ry=110, rot=0.0, colour=RED, lines=(("ABCDE", 0.45, 0.17),), star=True, glyphs="ABCDEFGHIJ",
              h=700, w=900, cx=450, cy=360):
    """A page with a paragraph and a stamp with centre ``lines`` (text, centre below the stamp's centre and glyph height, both
    in units of min(rx, ry)).  (image, seal box, arc glyph mask, [line masks])."""
    img = np.full((h, w, 3), PAPER, np.uint8)
    paragraph(img, 40, 60, 5)
    box, _, gl = stamp(img, cx, cy, rx, ry, colour, rot=rot, star=star, glyphs=glyphs)
    r, masks = min(rx, ry), []
    for text, dy, gh in lines:
        masks.append(inner_line(h, w, cx, cy, text, dy * r, gh * r, rot))
        img[masks[-1]] = colour
    return img, box, gl, masks


DRAWN = {
    "company": dict(),
    "company, blue, turned 20": dict(colour=BLUE, rot=20.0),
    "company, turned -20": dict(rot=-20.0),
    "company, blue, turned -20": dict(colour=BLUE, rot=-20.0),
    "company, turned 20": dict(rot=20.0),
    "two lines under the star": dict(lines=(("ABCDE", 0.28, 0.12), ("FGHIJK", 0.48, 0.12))),
    "oval invoice seal": dict(rx=140, ry=105, star=False, lines=(("1234567890", 0.0, 0.17), ("ABCDEF", 0.38, 0.15))),
    "oval invoice seal, blue, turned 10": dict(rx=140, ry=105, star=False, colour=BLUE, rot=10.0,
                                              lines=(("1234567890", 0.0, 0.17), ("ABCDEF", 0.38, 0.15))),
    "receipt ring": dict(star=False, glyphs="", lines=(("ABCD", 0.0, 0.2),)),
    "no inner text": dict(lines=()),
}


def _lines_of(img):
    """(seal table, line record) of the twin for the page's one seal."""
    t, recs = L.page_lines(img)
    (j,) = [j for j, s in enumerate(t["seals"]) if s["found"]]
    return t["seals"][j], recs[j]


@pytest.mark.parametrize("name", list(DRAWN))
def test_drawn_centre_lines_turns_and_arcs(name):
    kw = DRAWN[name]
    img, box, gl, masks = seal_page(**kw)
    s, r = _lines_of(img)
    assert (s["x0"], s["y0"], s["x1"], s["y1"]) == box
    assert r["n_found"] == r["n_lines"] == len(masks)
    if kw.get("glyphs", "x") == "":                              # a ring with no arc text: no band, no turn
        assert (r["why"], r["turn"], r["k_top"]) == (S.NO_BAND, 0, -1)
    else:
        assert r["why"] == 0 and abs(2.5 * r["turn"] - kw.get("rot", 0.0)) <= 2.5
        # the arc lies within one sector of the drawn arc glyphs, and a pixel at their radius (under a degree)
        start, end = 5 * r["g0"], 5 * r["g0"] - 5 * (72 - r["n_gap"])
        a = (start - _angles(gl, box) + 10) % 360 - 10
        assert -6 <= a.min() <= 6 and abs(a.max() - (start - end)) <= 6
    u, v = L.stamp_frame(box, r["turn"])
    u, v = np.broadcast_arrays(u, v)
    for m, (u0, v0, u1, v1) in zip(masks, r["boxes"]):
        sel = m[box[1]:box[3], box[0]:box[2]]
        assert u0 - 2 <= u[sel].min() and u[sel].max() < u1 + 2 and v0 - 2 <= v[sel].min() and v[sel].max() < v1 + 2
        if r["k_bottom"] >= 0:                                   # the arc's band and sectors stay clear of the centre line
            X, Y, A, B = S.ellipse_coords(box)
            k, sec = np.broadcast_arrays(S.radial_bin(X, Y, A, B), S.sector(X * B, -Y * A))
            low = sel & (k >= r["k_bottom"])
            assert ((sec[low] - r["g0"]) % 72 < r["n_gap"]).all() and k[sel].max() < r["k_top"] - L.HEAD_BINS + 1


def test_the_inner_line_no_longer_pulls_the_band_and_gap():
    """Without the centre-line definition the band runs into the inner line and its ink fills the gap; with it, the band and
    gap are those of the same stamp without the line."""
    bare = _lines_of(seal_page(lines=())[0])
    for rot in (0.0, 15.0):
        s, r = _lines_of(seal_page(rot=rot)[0])
        assert s["k_bottom"] < bare[0]["k_bottom"] and s["n_gap"] < 10
        assert (r["k_bottom"], r["k_top"], r["n_gap"]) == (bare[1]["k_bottom"], bare[1]["k_top"], bare[1]["n_gap"])
        assert r["n_gap"] >= 28


def _entries(img):
    """pipeline._seal_entries of the twin's seal and line tables of a whole image."""
    t, recs = L.page_lines(img)
    tab = np.zeros((), ops.seal_table_dtype())
    tab["n_cand"], tab["n_seals"] = t["n_cand"], t["n_seals"]
    for j, r in enumerate(t["seals"]):
        for f, v in r.items():
            tab["seal"][j][f] = v
    return pipeline._seal_entries(tab, 0, 0, img.shape[:2], line_table(recs))


def line_table(recs):
    """The mn_seal_line_table of twin line records (None: a zero record)."""
    ltab = np.zeros((), ops.seal_line_table_dtype())
    for j, r in enumerate(recs):
        if r is None:
            continue
        for f in L.FIELDS:
            ltab["seal"][j][f] = r[f]
        for m, b in enumerate(r["boxes"]):
            ltab["seal"][j]["box"][m] = b
    return ltab


@pytest.mark.parametrize("name", list(DRAWN))
def test_found_line_regions_pass_the_planner(name):
    img, box, _, masks = seal_page(**DRAWN[name])
    (e,) = _entries(img)
    assert len(e["lines"]) == len(masks) and all(ln["region"] is not None for ln in e["lines"])
    assert e["turn"] == 2.5 * round(e["turn"] / 2.5)
    for ln in e["lines"]:
        assert isinstance(ln["region"], tuple if e["turn"] == 0 else pipeline.OrientedRegion)
        for scale in (1, 2, 4):
            pipeline.plan_regions([img.shape[:2]], [[ln["region"]]], None, None, scale)
    if masks and e["turn"] == 0:                                 # the rectangle holds the drawn line
        ys, xs = np.nonzero(masks[-1])
        x0, y0, x1, y1 = e["lines"][-1]["region"]
        assert x0 <= xs.min() and xs.max() < x1 and y0 <= ys.min() and ys.max() < y1


def test_line_region_of_a_turned_seal_is_its_box_turned_about_the_centre():
    e = pipeline._seal_line(100.0, 80.0, (-30, 10, 30, 24), 90.0, (400, 400))
    tl, tr, bl = e["region"]
    np.testing.assert_allclose([tl, tr, bl], [(110.0, 110.0), (110.0, 50.0), (124.0, 110.0)], atol=1e-9)
    e = pipeline._seal_line(100.5, 80.0, (-30, 10, 30, 24), 0.0, (400, 400))
    assert e["region"] == (70, 90, 131, 104)
    e = pipeline._seal_line(10.0, 10.0, (-30, 10, 30, 24), 0.0, (400, 400))
    assert e["region"] is None and "rejected" in e["why"]


# ---- thresholds ----

def _rows(*runs):
    """A row map of runs (v0, v1, u0, u1): every row of [v0, v1] with ink from u0 to u1."""
    return {v: (u0, u1) for v0, v1, u0, u1 in runs for v in range(v0, v1 + 1)}


def test_line_gap_threshold():
    A = B = 200                                                   # min_h = max(4, 400 // 64) = 6
    gap = L.LINE_GAP
    assert L.lines_of(_rows((0, 4, -30, 30), (5 + gap - 1, 12, -30, 30)), A, B, 20)[0] == 1      # a gap of LINE_GAP - 1 rows
    assert L.lines_of(_rows((0, 6, -30, 30), (7 + gap, 14 + gap, -30, 30)), A, B, 20)[0] == 2    # a gap of LINE_GAP rows


def test_line_height_threshold():
    for A, B, h in ((200, 200, 6), (100, 100, L.LINE_MIN_H), (640, 640, 20)):
        assert max(L.LINE_MIN_H, (A + B) // L.LINE_H_DIV) == h
        assert L.lines_of(_rows((0, h - 1, -40, 40)), A, B, 31)[0] == 1
        assert L.lines_of(_rows((0, h - 2, -40, 40)), A, B, 31)[0] == 0


def test_line_ratio_threshold():
    h = 10
    assert L.lines_of(_rows((0, h - 1, 0, L.LINE_RATIO * h - 1)), 200, 200, 31)[0] == 1            # w = 2 h
    assert L.lines_of(_rows((0, h - 1, 0, L.LINE_RATIO * h - 2)), 200, 200, 31)[0] == 0            # w = 2 h - 1


def test_line_padding_and_clip():
    assert L.lines_of(_rows((0, 9, -20, 20)), 200, 200, 31)[1] == [(-22, -2, 23, 12)]             # p = LINE_PAD
    assert L.lines_of(_rows((0, 23, -60, 60)), 200, 200, 31)[1] == [(-63, -3, 64, 27)]            # p = 24 // LINE_PAD_DIV
    assert L.lines_of(_rows((0, 23, -60, 60)), 200, 200, 10)[1] == [(-32, -3, 32, 27)]            # R = 10 * 200 // 64


def test_max_lines_keeps_the_first_and_counts_all():
    runs = [(20 * j, 20 * j + 9, -30, 30) for j in range(L.MAX_LINES + 1)]
    n, boxes = L.lines_of(_rows(*runs), 200, 200, 31)
    assert (n, len(boxes)) == (L.MAX_LINES + 1, L.MAX_LINES) and boxes[0][1] == -2
    n, boxes = L.lines_of(_rows(*runs[:L.MAX_LINES]), 200, 200, 31)
    assert (n, len(boxes)) == (L.MAX_LINES, L.MAX_LINES)


def test_turn_table_and_quarter_turns():
    for t in range(-71, 73):
        c, s = L.turn_dir(t)
        assert abs(c - 2 ** 20 * math.cos(math.radians(2.5 * t))) <= 0.5 and abs(s - 2 ** 20 * math.sin(math.radians(2.5 * t))) <= 0.5
    assert L.turn_dir(36) == (0, 2 ** 20) and L.turn_dir(72) == (-2 ** 20, 0) and L.turn_dir(-36) == (0, -2 ** 20)


def test_head_bins_gap_and_turn():
    """The head gap reads only the band's outer HEAD_BINS bins: ink one bin below them does not fill the gap."""
    band, gap = range(20, 25), range(36, 66)                     # a gap of 30 sectors centred on 255 degrees
    text = [s for s in range(72) if s not in gap]
    r = S.seal_record(_painted(((30, 31), range(72)), (band, text), ((24 - L.HEAD_BINS,), range(72))), BOX)
    assert (r["k_bottom"], r["k_top"], r["n_gap"]) == (20, 24, 0)
    ink, area = S.histograms(_painted(((30, 31), range(72)), (band, text), ((24 - L.HEAD_BINS,), range(72))), BOX)
    assert L.head(ink, 24) == (36, 30, 0, 2 * 36 + 30 - 108)
    ink, _ = S.histograms(_painted(((30, 31), range(72)), (band, text), ((24 - L.HEAD_BINS + 1,), range(72))), BOX)
    assert L.head(ink, 24)[1] == 0                               # the same ink one bin outward fills it
    assert L.head(ink, 24)[2:] == (S.NO_GAP, 0)


def test_turn_normalisation():
    for g0, n, t in ((0, 36, 72), (36, 36, 0), (54, 36, 36), (1, 36, -70), (71, 36, 70), (37, 36, 2), (18, 36, -36)):
        ink = np.zeros((S.BINS, 72), np.int64)
        ink[20:24] = 10
        ink[20:24, (g0 + np.arange(n)) % 72] = 0
        assert L.head(ink, 23) == (g0, n, 0, t)


def test_head_min_k_threshold():
    """A band whose outer bin is under HEAD_MIN_K (central text taken for arc text) is no arc band: no turn, no arc."""
    for k_top, has in ((L.HEAD_MIN_K - 1, False), (L.HEAD_MIN_K, True)):
        img = _painted(((30, 31), range(72)), (range(k_top - 3, k_top + 1), range(0, 40)))
        r = S.seal_record(img, BOX)
        assert r["k_top"] == k_top
        rec = L.line_record(img, r)
        assert (rec["k_top"] == k_top, rec["why"] == S.NO_BAND) == (has, not has)


def test_gap_margin_threshold():
    """Ink below the arc band joins the interior inside the head gap less GAP_MARGIN sectors at each end."""
    arc = range(0, 40)                                          # the gap is [40, 72)
    for sec, inside in ((40 + L.GAP_MARGIN - 1, False), (40 + L.GAP_MARGIN, True), (71 - L.GAP_MARGIN, True),
                        (72 - L.GAP_MARGIN, False)):
        img = _painted(((30, 31), range(72)), (range(20, 25), arc), ((20,), (sec,)))
        r = L.line_record(img, S.seal_record(img, BOX))
        assert (r["g0"], r["n_gap"], r["k_in"], r["k_gap"]) == (40, 32, 20, 21)
        X, Y, A, B = S.ellipse_coords(BOX)
        k, s = np.broadcast_arrays(S.radial_bin(X, Y, A, B), S.sector(X * B, -Y * A))
        assert ((k == 20) & (s == sec)).any()
        rows = r["n_found"]                                     # too few pixels for a line: check the mask itself
        m = S.seal_mask(img) & ((k < r["k_in"]) | ((k < r["k_gap"]) & ((s - r["g0"] - L.GAP_MARGIN) % 72 <
                                                                          r["n_gap"] - 2 * L.GAP_MARGIN)))
        assert m[k == 20].any() == inside and rows == 0


BOX = (0, 0, 200, 200, 0)


def test_arc_band_density_threshold():
    area = np.full(S.BINS, 7200, np.int64)
    ink = np.zeros((S.BINS, 72), np.int64)
    g0, n = 40, 30                                              # 42 arc sectors
    arc = [(g0 + n + j) % 72 for j in range(72 - n)]
    ink[24, arc] = 10
    ink[23, arc[:30]] = 5                                       # 32 * 72 * 150 = 7200 * 48 < 7200 * 42 * ... see below
    # bin 23: 32 * 72 * ink' >= area * 42  <=>  ink' >= 131.25: 132 passes, 131 does not
    ink[23] = 0
    ink[23, arc[0]] = 132
    assert L.arc_bottom(ink, area, 24, g0, n) == 23
    ink[23, arc[0]] = 131
    assert L.arc_bottom(ink, area, 24, g0, n) == 24
    ink[23, g0] = 10 ** 6                                       # gap sectors do not count
    assert L.arc_bottom(ink, area, 24, g0, n) == 24
    ink[S.BAND_MIN_K:24, arc[0]] = 10 ** 6                      # the walk stops at BAND_MIN_K
    assert L.arc_bottom(ink, area, 24, g0, n) == S.BAND_MIN_K


def test_ring_without_band_reads_inside_the_ring_edge():
    img, box, _, masks = seal_page(**DRAWN["receipt ring"])
    s, r = _lines_of(img)
    ink, area = S.histograms(img, box)
    assert r["k_in"] == r["k_gap"] == L.walk_gap_top(ink.sum(axis=1), area) and r["k_in"] >= 26


# ---- validation, work and build ----

def _no_launch(monkeypatch):
    def boom(*a, **k):
        raise AssertionError("a launch was reached")
    for f in ("find_page_quads", "find_blocks", "find_lines", "warp_perspective"):
        monkeypatch.setattr(ops, f, boom)
    monkeypatch.setattr(pipeline, "_device_images", boom)


@pytest.mark.parametrize("page, match", [
    (pipeline.TextPage(seals="auto", seal_lines="on"), "seal_lines must be None or 'auto', got 'on'"),
    (pipeline.TextPage(seals="auto", seal_lines=True), "seal_lines must be None or 'auto', got True"),
    (pipeline.TextPage(seal_lines="auto"), "seal_lines is given, but seals is None"),
    (pipeline.TextPage(seal_lines="auto", rules="auto"), "seal_lines is given, but seals is None"),
])
def test_page_refusals_before_any_launch(monkeypatch, page, match):
    _no_launch(monkeypatch)
    img = np.zeros((200, 240, 3), np.uint8)
    with pytest.raises(ValueError, match=r"image 0, page 1: " + match):
        pipeline.find_blocks([img], [[pipeline.TextPage(seals="auto", seal_lines="auto"), page]])
    with pytest.raises(ValueError, match=r"image 0, region 1 \(a text page\): " + match):
        pipeline.restore_regions(None, None, None, [img], [[pipeline.TextPage(seals="auto", seal_lines="auto"), page]])


def test_ops_refuses_lines_without_seals():
    for v in (True, 1, None):
        with pytest.raises(ValueError, match="seal_lines .* is not False, or True on a page with a seal_size"):
            ops._check_page_options(ops.PageItem(None, None, False, 0, seal_lines=v), "p")
    ops._check_page_options(ops.PageItem(None, None, False, 0, seal_size=24, seal_lines=True), "p")


def test_work_memory_counts_the_line_table(monkeypatch):
    w, h = 240, 200
    assert ops.page_bytes(w, h, seals=True, seal_lines=True) - ops.page_bytes(w, h, seals=True) == ops.seal_line_bytes()
    assert ops.seal_line_bytes() >= ctypes_size("SealLineTable") + ctypes_size("CentrePage")
    _no_launch(monkeypatch)
    img = np.zeros((h, w, 3), np.uint8)
    monkeypatch.setattr(ops, "PAGE_MAX_WORK", ops.page_bytes(w, h, seals=True, seal_lines=True) - 1)
    with pytest.raises(ValueError, match="work memory"):
        pipeline.find_blocks([img], [[pipeline.TextPage(seals="auto", seal_lines="auto")]])
    pipeline._check_page_work([(0, pipeline.TextPage(seals="auto"), (0, 0, w, h))])     # the page without lines fits


def ctypes_size(name):
    import ctypes
    return ctypes.sizeof(getattr(_lib, name))


def test_constants_match_the_header():
    src = open(os.path.join(ROOT, "include", "marconet_b200.h")).read()

    def define(name):
        return int(re.search(r"#define %s (-?\d+)" % name, src).group(1))
    for name, value in (("MN_SEAL_HEAD_BINS", L.HEAD_BINS), ("MN_SEAL_HEAD_MIN_K", L.HEAD_MIN_K),
                        ("MN_SEAL_GAP_MARGIN", L.GAP_MARGIN), ("MN_SEAL_LINE_GAP", L.LINE_GAP), ("MN_SEAL_LINE_MIN_H", L.LINE_MIN_H),
                        ("MN_SEAL_LINE_H_DIV", L.LINE_H_DIV), ("MN_SEAL_LINE_RATIO", L.LINE_RATIO),
                        ("MN_SEAL_LINE_PAD", L.LINE_PAD), ("MN_SEAL_LINE_PAD_DIV", L.LINE_PAD_DIV),
                        ("MN_SEAL_MAX_LINES", L.MAX_LINES), ("MN_SEAL_MAX_LINES", _lib.SEAL_MAX_LINES),
                        ("MN_SEAL_TURN_STEPS", L.TURN_STEPS)):
        assert define(name) == value, name
    turns = re.search(r"#define MN_SEAL_TURNS \{(.*?)\}\}", src, re.S).group(1).replace("\\", "")
    pairs = [tuple(int(v) for v in p.split(",")) for p in re.findall(r"\{?(-?\d+, -?\d+)", turns)]
    assert pairs == [tuple(int(v) for v in d) for d in L.TURNS]
    assert ops.seal_line_table_dtype().itemsize == ctypes_size("SealLineTable") == 64 * (12 + 4 * 4) * 4
    assert [f for f, _ in _lib.SealLines._fields_[:10]] == list(L.FIELDS)


def test_centre_line_kernel_does_not_spill(tmp_path):
    nvcc = "/usr/local/cuda/bin/nvcc" if os.path.isfile("/usr/local/cuda/bin/nvcc") else "nvcc"
    try:
        out = subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-Xcompiler", "-fPIC",
                              "-DMN_BUILD", "-I", os.path.join(ROOT, "include"), "-Xptxas", "-v", "-c",
                              os.path.join(ROOT, "marconet_b200", "csrc", "block_ops.cu"), "-o", str(tmp_path / "b.o")],
                             capture_output=True, text=True, timeout=600)
    except FileNotFoundError:
        pytest.skip("nvcc is not installed")
    assert out.returncode == 0, out.stdout + out.stderr
    m = re.search(r"Function properties for \S*centre_lines_kernel\S*\n\s+(\d+) bytes stack frame, (\d+) bytes spill stores, "
                  r"(\d+) bytes spill loads", out.stdout + out.stderr)
    assert m and m.group(2) == m.group(3) == "0"
