"""Vertical text columns on the CPU (DESIGN.md section 7b, "Vertical text columns"): the numpy twin's layout and inverse layout
by hand, pipeline.vertical_plan in its three modes against the twin and every rejection of plan_regions, R against the stitch,
the one-cell reduction, the page maps at t_height = 128, the golden page, and the record layout and register report of the two
gathers."""
import ctypes
import math
import os
import re

import numpy as np
import pytest

from oracle import vertical_regions as V

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "vertical_regions.npz")


def _pixels(a):
    """An int array [h, w] as uint8 [h, w, 3] pixels (v, v + 1, v + 2)."""
    a = np.asarray(a, np.uint8)
    return np.stack([a, a + 1, a + 2], -1)


def test_layout_by_hand():
    """A 2-wide, 5-row column cut at [0, 2, 5]: cells of 2 and 3 rows, H_L = 3, p = (0, 0); the short cell repeats its last row."""
    C = _pixels([[10, 11], [20, 21], [30, 31], [40, 41], [50, 51]])
    want = _pixels([[10, 11, 30, 31], [20, 21, 40, 41], [20, 21, 50, 51]])
    np.testing.assert_array_equal(V.layout(C, [0, 2, 5]), want)
    # cells of 1 and 4 rows: H_L = 4, p = (1, 0): the one-row cell is centred, padded with its own row above and below
    want = _pixels([[10, 11, 20, 21], [10, 11, 30, 31], [10, 11, 40, 41], [10, 11, 50, 51]])
    np.testing.assert_array_equal(V.layout(C, [0, 1, 5]), want)
    assert V.line_boxes([0, 1, 5], 2, [[0, 0, 2, 1], [0, 2, 1, 4]]) == [[0, 1, 2, 2], [2, 1, 3, 3]]


def test_unlayout_by_hand():
    """H_L = 64 (R doubles), w_r = 2, cells [0, 64, 128]: T_col [256, 4] takes T's columns [0, 4) for cell 0's rows and [4, 8)
    for cell 1's, row i of a cell from T row i; a T narrower than R(n w_r) clamps the last cell to its own last column."""
    T = _pixels(np.arange(128)[:, None] + 0 * np.arange(8)[None, :])
    T[..., 0] = np.arange(8)[None, :]
    tc = V.unlayout(T, [0, 64, 128], 2)
    assert tc.shape == (256, 4, 3)
    np.testing.assert_array_equal(tc[:128, :, 0], np.tile(np.arange(4), (128, 1)))
    np.testing.assert_array_equal(tc[128:, :, 0], np.tile(np.arange(4, 8), (128, 1)))
    np.testing.assert_array_equal(tc[:128, 0, 1], np.arange(128) + 1)
    np.testing.assert_array_equal(tc[128:, 0, 1], np.arange(128) + 1)
    tc = V.unlayout(T[:, :6], [0, 64, 128], 2)
    np.testing.assert_array_equal(tc[128:, :, 0], np.tile([4, 5, 5, 5], (128, 1)))
    # unequal cells 16 and 48 rows, H_L = 48: cell 0 (p = 16) reads T rows [R(16), R(32)) = [43, 85)
    tc = V.unlayout(_pixels(np.tile(np.arange(128)[:, None], (1, 6))), [0, 16, 64], 2)
    assert tc.shape == (171, 5, 3)
    np.testing.assert_array_equal(tc[:43, 0, 0], np.arange(43, 86).clip(max=84))
    np.testing.assert_array_equal(tc[43:, 0, 0], np.arange(128))


def test_boxes_back_by_hand():
    c = [0, 1, 5]
    assert V.boxes_back(c, 2, V.line_boxes(c, 2, [[0, 0, 2, 1], [0, 2, 1, 4]])) == [[0, 0, 2, 1], [0, 2, 1, 4]]
    assert V.boxes_back(c, 2, [[-1, -3, 1.5, 9]]) == [[0, 0, 1.5, 1]]           # clipped to its cell
    assert V.boxes_back(c, 2, [[1, 0, 4, 2]]) == [[0, 1, 2, 3]]                 # centre 2.5: cell 1


def _random_boxes(rng, w, h):
    y, out = int(rng.integers(0, 3)), []
    while True:
        ch = int(rng.integers(max(1, w // 2), 2 * w))
        if y + ch > h:
            return out
        out.append([float(rng.integers(0, 2)), float(y), float(w - rng.integers(0, 2)), float(y + ch)])
        y += ch + int(rng.integers(1, 6))


def test_vertical_plan_matches_twin():
    from marconet_b200.pipeline import layout_cells, unlayout_cells, vertical_plan, vertical_r
    rng = np.random.default_rng(1)
    for _ in range(200):
        w, h = int(rng.integers(4, 40)), int(rng.integers(1, 400))
        mode = rng.integers(0, 3)
        boxes = _random_boxes(rng, w, h) if mode == 0 else None
        if mode == 0 and len(boxes) < 1:
            continue
        n = int(rng.integers(1, min(h, 12) + 1)) if mode == 1 else None
        vp = vertical_plan(w, h, cells=n, boxes=boxes)
        c = V.cells(h, w, n, boxes)
        t, hl, p = V.geometry(c)
        assert vp.cells == c and vp.heights == t.tolist() and vp.line_height == hl and vp.pads == p.tolist()
        assert vp.t_size == V.t_size(c, w)
        assert vp.boxes == (None if boxes is None else V.line_boxes(c, w, boxes))
        assert layout_cells(vp) == list(zip(c[:-1], p.tolist(), t.tolist()))
        wt = vertical_r(len(t) * w, hl) - int(rng.integers(0, 3))
        tab = unlayout_cells(vp, wt)
        assert [r[0] for r in tab] == [V.R(v, hl) for v in c[:-1]] and tab[-1][4] == min(V.R(len(t) * w, hl), wt)
        if mode == 2:
            assert len(t) == min(max(round(h / w), 1), h)


def test_cell_modes_by_hand():
    from marconet_b200.pipeline import vertical_plan
    assert vertical_plan(20, 100).cells == [0, 20, 40, 60, 80, 100]
    assert vertical_plan(20, 50).cells == [0, 25, 50]                            # round_half_even(2.5) = 2
    assert vertical_plan(20, 70).cells == [0, 17, 35, 52, 70]                    # round_half_even(3.5) = 4
    assert vertical_plan(40, 10).cells == [0, 10]                                # at least one cell
    assert vertical_plan(20, 100, cells=3).cells == [0, 33, 66, 100]
    vp = vertical_plan(20, 100, boxes=[[0, 2, 20, 18], [1, 25, 19, 40], [0, 50, 20, 95]])
    assert vp.cells == [0, 21, 45, 100] and vp.line_height == 55 and vp.pads == [17, 15, 0]
    assert vp.t_size == (round(20 * 128 / 55), round(100 * 128 / 55))


def test_r_is_the_stitch():
    """R(w_r) with one cell is the sr_u8 width restore_images gives the crop, over a sweep of sizes (the whole-width box)."""
    from marconet_b200.pipeline import plan_batches, plan_segments, vertical_plan
    for h in (1, 2, 3, 7, 12, 31, 32, 33, 64, 97, 128, 300):
        for w in (1, 2, 5, 9, 17, 40, 111, 255, 513, 999):
            if w * 128 / h > 32767:
                continue
            boxes = [[float(x), 0.0, float(min(w, x + h)), float(h)] for x in range(0, w, h)]
            segs = plan_segments(h, w, boxes, labels=[1] * len(boxes))
            out_w, _ = plan_batches([(h, w)], [[1] * len(boxes)], [boxes], [segs], 8)
            assert vertical_plan(w, h, cells=1).t_size == (out_w[0], 128), (h, w)


def test_one_cell_is_the_identity():
    rng = np.random.default_rng(2)
    for h, w in ((1, 1), (5, 3), (32, 200), (37, 11), (300, 20)):
        C = rng.integers(0, 256, (h, w, 3), dtype=np.uint8)
        np.testing.assert_array_equal(V.layout(C, [0, h]), C)
        wt = round(w * 128 / h)
        T = rng.integers(0, 256, (128, wt, 3), dtype=np.uint8)
        np.testing.assert_array_equal(V.unlayout(T, [0, h], w), T)


def test_page_maps_default_height_is_128():
    """t_height = 128 gives the maps and boxes the functions gave before it existed, bit for bit."""
    from marconet_b200.pipeline import (OrientedRegion, QuadRegion, footprint_box, oriented_maps, quad_footprint_box,
                                        quad_maps)
    rng = np.random.default_rng(3)
    for _ in range(50):
        o = OrientedRegion.from_rotated(*rng.uniform(20, 200, 2), rng.uniform(5, 300), rng.uniform(3, 40), rng.uniform(-180, 180))
        q = QuadRegion(o.tl, o.tr, (o.tr[0] + o.bl[0] - o.tl[0] + rng.uniform(-1, 1), o.tr[1] + o.bl[1] - o.tl[1]), o.bl)
        for s in (1, 4):
            for wt in (None, 77):
                a, b = oriented_maps(o, s, wt), oriented_maps(o, s, wt, 128)
                assert a.matrix.tobytes() == b.matrix.tobytes() and a.page_map.tobytes() == b.page_map.tobytes()
                assert (a.kx, a.ky, a.size, a.t_width) == (b.kx, b.ky, b.size, b.t_width)
                assert footprint_box(o, a, s, (900, 900)) == footprint_box(o, b, s, (900, 900), 128)
                a, b = quad_maps(q, s, wt), quad_maps(q, s, wt, 128)
                assert a.matrix.tobytes() == b.matrix.tobytes() and a.page_map.tobytes() == b.page_map.tobytes()
                assert (a.kx, a.ky, a.size, a.t_width, a.homography) == (b.kx, b.ky, b.size, b.t_width, b.homography)
                assert quad_footprint_box(a, s, (900, 900)) == quad_footprint_box(b, s, (900, 900), 128)
    # the row of N and ky follow t_height: a T twice as tall maps the same page point twice as far down
    m1, m2 = oriented_maps(o, 2, 50, 128), oriented_maps(o, 2, 50, 256)
    np.testing.assert_allclose(m2.page_map[1, :2], 2 * m1.page_map[1, :2], rtol=1e-12)
    assert m2.page_map[1, 2] + 0.5 == pytest.approx(2 * (m1.page_map[1, 2] + 0.5), rel=1e-12)
    assert m2.ky == pytest.approx(m1.ky / 2, rel=1e-6) and m2.kx == m1.kx


def _golden():
    from marconet_b200.pipeline import OrientedRegion, QuadRegion, VerticalRegion
    g = np.load(GOLDEN)
    regs = []
    for k, col, c in zip(g["kinds"].tolist(), g["columns"].tolist(), g["corners"].tolist()):
        shape = (OrientedRegion(tuple(c[0]), tuple(c[1]), tuple(c[3])) if k == 1 else QuadRegion(*map(tuple, c)) if k == 2 else
                 (int(c[0][0]), int(c[0][1]), int(c[2][0]), int(c[2][1])))
        regs.append(VerticalRegion(shape) if col else shape)
    labels, boxes = [[] for _ in regs], [[] for _ in regs]
    for lab, (x1, y1, x2, y2, r) in zip(g["labels"].tolist(), g["boxes"].tolist()):
        labels[r].append(lab)
        boxes[r].append([x1, y1, x2, y2])
    return g, regs, labels, boxes


def golden_columns(g, regs, boxes):
    """Each region's T_col from its stored T (None for the strided one), and its plan."""
    from marconet_b200 import pipeline
    plan = pipeline.plan_regions([g["image"].shape[:2]], [regs], [[[0] * len(b) for b in boxes]], [boxes], scale=int(g["scale"]),
                                 feather=int(g["feather"]))
    out = []
    for r, p in enumerate(plan):
        t = g[f"sr{r}"] if int(g["sr_strides"][r]) == 1 else None
        out.append(t if t is None or p.vertical is None else V.unlayout(t, p.vertical.cells, p.vertical.size[0]))
    return out, plan


def test_twin_reproduces_golden_page():
    """Every stored page pixel outside the long column's box (whose T is stored strided) is the twin's composition of the other
    regions' stored lines, put back into their columns."""
    g, regs, _, boxes = _golden()
    st, s = int(g["stride"]), int(g["scale"])
    tcs, plan = golden_columns(g, regs, boxes)
    full = V.compose(g["image"], regs, tcs, s, int(g["feather"]))
    keep = np.ones(full.shape[:2], bool)
    for r in np.flatnonzero(g["sr_strides"] != 1):
        x0, y0, x1, y1 = plan[r].out
        keep[y0:y1, x0:x1] = False
    keep = keep[::st, ::st]
    assert keep.mean() > 0.8
    np.testing.assert_array_equal(full[::st, ::st][keep], g["page"][keep])
    assert not np.array_equal(g["page"], V.background(g["image"], s)[::st, ::st])


def test_plan_golden_columns():
    from marconet_b200 import pipeline
    g, regs, labels, boxes = _golden()
    plan = pipeline.plan_regions([g["image"].shape[:2]], [regs], [labels], [boxes], scale=4, feather=8)
    for p, reg, bx in zip(plan, regs, boxes):
        if not isinstance(reg, pipeline.VerticalRegion):
            assert p.vertical is None
            continue
        c = V.cells(p.vertical.size[1], p.vertical.size[0], boxes=bx)
        assert p.vertical.cells == c and p.boxes == V.line_boxes(c, p.vertical.size[0], bx) and p.labels == labels[regs.index(reg)]
    assert len(plan[1].vertical.heights) == 24 and round(plan[1].vertical.line_height and 288 * 32 / 12) > 512
    assert plan[5].overlaps == [1] and len(plan[4].vertical.heights) == 1
    assert plan[2].oriented is not None and plan[3].quad is not None


@pytest.mark.parametrize("reg,kw,match", [
    (("V", (0, 0, 4, 40), 0), {}, r"image 0, region 0: cells must be an integer in \[1, 40\]"),
    (("V", (0, 0, 4, 40), 41), {}, r"image 0, region 0: cells must be an integer in \[1, 40\]"),
    (("V", (0, 0, 4, 40), 2.0), {}, r"image 0, region 0: cells must be an integer"),
    (("V", (0, 0, 4, 40), True), {}, r"image 0, region 0: cells must be an integer"),
    (("V", (0, 0, 4, 40), 2), dict(labels=[[[1]]], boxes=[[[[0, 0, 4, 4]]]]), "image 0, region 0: cells and boxes are both given"),
    (("V", (0, 0, 4, 40), None), dict(labels=[[[1, 2]]], boxes=[[[[0, 0, 4, 4]]]]), "image 0, region 0: 2 labels for 1 boxes"),
    (("V", (0, 0, 4, 40), None), dict(labels=[[None]], boxes=[[[[0, 0, 4, 4]]]]), "image 0, region 0: boxes without labels"),
    (("V", (0, 0, 4, 40), None), dict(labels=[[[1]]], boxes=[[[[0, 0, 5, 4]]]]),
     r"image 0, region 0, character 0: box .* is outside the column crop \[0, 4\] x \[0, 40\]"),
    (("V", (0, 0, 4, 40), None), dict(labels=[[[1]]], boxes=[[[[0, 30, 4, 41]]]]), r"image 0, region 0, character 0: .* outside"),
    (("V", (0, 0, 4, 40), None), dict(labels=[[[1, 2]]], boxes=[[[[0, 20, 4, 29], [0, 0, 4, 9]]]]),
     r"image 0, region 0, character 1: the box's centre 4.5 lies above the previous character's 24.5"),
    (("V", (0, 0, 4, 40), None), dict(labels=[[[1, 2, 3]]], boxes=[[[[0, 0, 4, 30], [0, 10, 4, 20], [0, 20, 4, 21]]]]),
     r"image 0, region 0, character 2: the cell boundary 20 .* is not strictly inside \(20, 40\)"),
    (("V", (0, 0, 4, 40), None), dict(labels=[[[1, 2]]], boxes=[[[[0, 0, 4, 0], [0, 0, 4, 1]]]]),
     r"image 0, region 0, character 1: .* boundary 0 .* is not strictly inside \(0, 40\)"),
    (("V", (0, 0, 4, 40), None), dict(labels=[[[1, 2]]], boxes=[[[[0, 30, 4, 40], [0, 40, 4, 40]]]]),
     r"image 0, region 0, character 1: .* boundary 40 .* is not strictly inside \(0, 40\)"),
    (("V", ("V", (0, 0, 4, 40), None), None), {}, "image 0, region 0: the shape of a VerticalRegion is itself a VerticalRegion"),
    (("V", (0, 0, 4, 41), None), {}, r"image 0, region 0: rectangle \(0, 0, 4, 41\) is empty or outside the 10x40 image"),
    (("V", ((0, 0), (math.nan, 0), (0, 5)), None), {}, "image 0, region 0: corners .* are not finite"),
    (("V", ((1, 1), (9, 1), (1, 6), (9, 6)), None), {}, "image 0, region 0: the quad is not strictly convex"),
    (("V", (0, 0, 2000, 2), 2), dict(shape=(4, 2000)), r"image 0, region 0: line width 4000, restored column .* exceeds 32767"),
    (("V", (0, 0, 300, 1), None), dict(shape=(4, 400)), r"image 0, region 0: line width 300, restored column 38400x128 .* exceeds"),
])
def test_plan_rejects_column(reg, kw, match):
    from marconet_b200 import pipeline

    def build(v):
        if isinstance(v, tuple) and v and v[0] == "V":
            return pipeline.VerticalRegion(build(v[1]), v[2])
        if isinstance(v, tuple) and len(v) == 3:
            return pipeline.OrientedRegion(*v)
        if isinstance(v, tuple) and len(v) == 4 and isinstance(v[0], tuple):
            return pipeline.QuadRegion(*v)
        return v
    args = dict(regions=[[build(reg)]], labels=None, boxes=None, scale=4, feather=None)
    args.update(kw)
    shape = args.pop("shape", (40, 10))
    with pytest.raises(ValueError, match=match):
        pipeline.plan_regions([shape], **args)


def test_plan_rejects_column_naming_the_region():
    from marconet_b200 import pipeline
    with pytest.raises(ValueError, match="image 1, region 2: cells must be"):
        pipeline.plan_regions([(40, 10), (40, 10)], [[(0, 0, 4, 4)], [(0, 0, 2, 2), pipeline.VerticalRegion((0, 0, 4, 40)),
                                                                         pipeline.VerticalRegion((0, 0, 4, 40), cells=-1)]])


def test_column_footprint_uses_the_column_size():
    from marconet_b200 import pipeline
    o = pipeline.OrientedRegion.from_rotated(30, 50, 12, 80, 5)
    p = pipeline.plan_regions([(100, 60)], [[pipeline.VerticalRegion(o, cells=4)]], scale=2)[0]
    wc, hc = p.vertical.t_size
    m = pipeline.oriented_maps(o, 2, wc, hc)
    assert p.out == pipeline.footprint_box(o, m, 2, (200, 120), hc) and (wc, hc) == (77, 512)
    assert np.array_equal(p.matrix, pipeline.oriented_maps(o, 1).matrix)


def _fields(header, name):
    body = re.search(r"typedef struct \{([^{}]*)\}\s*" + name + ";", header).group(1)
    body = re.sub(r"/\*.*?\*/", "", body, flags=re.S)
    names = []
    for decl in body.split(";"):
        parts = [re.sub(r"\[\d+\]$", "", p.strip()) for p in decl.strip().split(",") if p.strip()]
        names += [re.findall(r"[A-Za-z_0-9]+$", p)[0] for p in parts]
    return names


def test_vertical_record_matches_header():
    from marconet_b200 import _lib
    header = open(os.path.join(ROOT, "include", "marconet_b200.h")).read()
    assert _fields(header, "mn_vertical_column") == [f[0] for f in _lib.VerticalColumn._fields_]
    assert ctypes.sizeof(_lib.VerticalColumn) == 56
    assert (_lib.VerticalColumn.cells.offset, _lib.VerticalColumn.dh.offset, _lib.VerticalColumn.w.offset) == (32, 40, 52)
    for name in ("mn_vertical_layout_u8_batched", "mn_vertical_unlayout_u8_batched"):
        assert re.search(r"int " + name + r"\(const mn_vertical_column\* columns, int n, long long max_pixels, void\* stream\);",
                         header)


def test_vertical_kernels_build_without_spills(tmp_path):
    import subprocess
    from marconet_b200 import build
    src = os.path.join(ROOT, "marconet_b200", "csrc", "image_ops.cu")
    r = subprocess.run([build.nvcc_path(), "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-DMN_BUILD", "-Xptxas", "-v",
                        "-cubin", src, "-o", str(tmp_path / "image_ops.cubin")], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-2000:]
    for kernel in ("vertical_gather_kernelILb0E", "vertical_gather_kernelILb1E"):
        props = re.search(kernel + r"[^\n]*\n[^\n]*Function properties for [^\n]*" + kernel + r"[^\n]*\n([^\n]*)", r.stderr)
        assert props, f"no ptxas report for {kernel}"
        assert "0 bytes spill stores, 0 bytes spill loads" in props.group(1), props.group(1)
