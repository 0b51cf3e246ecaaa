"""Curved text regions on the CPU (DESIGN.md section 7b, "Curved text regions"): the numpy twin of cv2.remap against live cv2
(IPP off), CurvedRegion.from_arc, the twin's inverse, pipeline.curved_maps by hand, plan_regions' validation of CurvedRegions,
the golden page, and the layout and register report of the two kernels."""
import ctypes
import math
import os
import re

import numpy as np
import pytest

from oracle import curved_regions as R
from oracle import remap as RM

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "curved_regions.npz")


@pytest.fixture
def cv2_no_ipp():
    cv2 = pytest.importorskip("cv2")
    was = cv2.ipp.useIPP()
    cv2.ipp.setUseIPP(False)
    yield cv2
    cv2.ipp.setUseIPP(was)


def _straight(x0, y0, x1, y1):
    from marconet_b200.pipeline import CurvedRegion
    w = x1 - x0
    return CurvedRegion(((x0, y0), (x0 + w / 3, y0), (x0 + 2 * w / 3, y0), (x1, y0)),
                        ((x0, y1), (x0 + w / 3, y1), (x0 + 2 * w / 3, y1), (x1, y1)))


@pytest.mark.parametrize("cn", [1, 3, 4])
def test_remap_twin_equals_cv2(cv2_no_ipp, cn):
    rng = np.random.default_rng(cn)
    src = rng.integers(0, 256, (41, 67, cn), dtype=np.uint8)
    mx = rng.uniform(-6, 73, (90, 110)).astype(np.float32)
    my = rng.uniform(-6, 47, (90, 110)).astype(np.float32)
    mx[:30] = np.round(mx[:30] * 64) / 64                # exact multiples of 1/64: the half-way ties of rint(map * 32)
    my[:30] = np.round(my[:30] * 64) / 64
    mx[30:40], my[30:40] = mx[30:40] + 300, my[30:40] - 200            # far outside: replicated borders
    out = cv2_no_ipp.remap(src, mx, my, cv2_no_ipp.INTER_CUBIC, borderMode=cv2_no_ipp.BORDER_REPLICATE)
    np.testing.assert_array_equal(RM.remap_cubic_u8(src, mx, my), out.reshape(90, 110, cn))
    xq, _ = RM.remap_coords(mx[:30], my[:30])
    assert ((mx[:30] * 64) % 2 == 1).any() and (xq % 1 == 0).all()


def test_from_arc_lies_on_the_circle():
    from marconet_b200.pipeline import CurvedRegion, bezier_point
    for cx, cy, rt, rb, a0, a1 in ((100, 100, 84, 72, 190, -10), (0, 0, 10, 20, 240, 300), (5, -3, 300, 280, 170, 10),
                                   (1, 2, 7, 5, -100, 259)):
        reg = CurvedRegion.from_arc(cx, cy, rt, rb, a0, a1)
        k = math.ceil(abs(a1 - a0) / 90)
        assert len(reg.top) == len(reg.bottom) == 3 * k + 1
        for curve, r in ((reg.top, rt), (reg.bottom, rb)):
            assert curve[0] == pytest.approx((cx + r * math.cos(math.radians(a0)), cy - r * math.sin(math.radians(a0))), abs=1e-9)
            assert curve[-1] == pytest.approx((cx + r * math.cos(math.radians(a1)), cy - r * math.sin(math.radians(a1))), abs=1e-9)
            for m in range(k):
                for i in range(33):
                    x, y = bezier_point(curve[3 * m:3 * m + 4], i / 32)
                    assert abs(math.hypot(x - cx, y - cy) - r) <= 1e-3 * r
    top = CurvedRegion.from_arc(0, 0, 10, 8, 150, 30).top
    assert top[0][0] < top[-1][0] and min(p[1] for p in top) < top[0][1]          # left to right over the top
    with pytest.raises(ValueError, match="0 < |span| < 360"):
        CurvedRegion.from_arc(0, 0, 10, 8, 10, 370)


def test_twin_inverse_returns_crop_coordinates():
    from marconet_b200.pipeline import CurvedRegion, curved_maps
    for reg in (CurvedRegion.from_arc(100, 100, 84, 72, 190, -10), CurvedRegion.from_arc(50, 50, 30, 44, 200, 340),
                CurvedRegion(((200, 20), (225, 10), (250, 34), (275, 22)), ((200, 38), (225, 28), (250, 52), (275, 40)))):
        m = curved_maps(reg, 1)
        mx, my = R.crop_map(m)
        ok, mm, t, b = R.invert(m, mx + 0.5, my + 0.5)
        c = np.asarray(m.c)
        (w_r, h_r) = m.size
        a_want = np.broadcast_to((np.arange(w_r) + 0.5) / w_r, mx.shape).ravel()
        b_want = np.broadcast_to(((np.arange(h_r) + 0.5) / h_r)[:, None], mx.shape).ravel()
        assert ok.all()
        assert np.abs(c[mm] + t * (c[mm + 1] - c[mm]) - a_want).max() < 1e-9
        assert np.abs(b - b_want).max() < 1e-9


def test_curved_maps_by_hand():
    from marconet_b200.pipeline import CurvedRegion, curved_maps
    m = curved_maps(_straight(13, 9, 77, 41), 4)
    assert m.size == (64, 32) and m.c == (0.0, 1.0) and m.t_width == 256 and m.kx == 1.0 and m.ky == 1.0
    assert m.lengths == (64.0,) and set(m.rulings) == {32.0}
    # two straight segments of 30 and 10 pixels, 10 high: c = (0, 3/4, 1), W_T = 512, s = 2: kx = 2 * 40 / 512, ky = 2 * 10 / 128
    reg = CurvedRegion(((0, 0), (10, 0), (20, 0), (30, 0), (30 + 10 / 3, 0), (30 + 20 / 3, 0), (40, 0)),
                       ((0, 10), (10, 10), (20, 10), (30, 10), (30 + 10 / 3, 10), (30 + 20 / 3, 10), (40, 10)))
    m = curved_maps(reg, 2)
    assert m.size == (40, 10) and m.t_width == 512
    assert m.c[0] == 0 and m.c[1] == pytest.approx(0.75, abs=1e-14) and m.c[2] == 1
    assert m.kx == pytest.approx(0.15625, rel=1e-7) and m.ky == 0.15625
    assert curved_maps(reg, 2, 300).kx == float(np.float32(2 * sum(m.lengths) / 300))
    # a ruling growing from 10 to 20: h_r = 20, h = the mean of the 33 samples
    reg = CurvedRegion(((0, 0), (10, 0), (20, 0), (30, 0)), ((0, 10), (10, 40 / 3), (20, 50 / 3), (30, 20)))
    m = curved_maps(reg, 1)
    assert m.size[1] == 20 and m.ky == pytest.approx(15 / 128, rel=1e-6)


def test_rectangle_reduction_is_exact(cv2_no_ipp):
    from marconet_b200.pipeline import curved_maps
    from oracle import regions as RR
    rng = np.random.default_rng(3)
    img = rng.integers(0, 256, (60, 100, 3), dtype=np.uint8)
    for x0, y0, x1, y1 in ((13, 9, 77, 41), (1, 1, 99, 59), (40, 20, 41, 45)):
        mx, my = R.crop_map(curved_maps(_straight(x0, y0, x1, y1), 1))
        assert np.array_equal(mx.astype(np.float32), np.broadcast_to(np.arange(x0, x1, dtype=np.float32), mx.shape))
        np.testing.assert_array_equal(R.rectify(img, _straight(x0, y0, x1, y1)), img[y0:y1, x0:x1])
        out = cv2_no_ipp.remap(img, mx.astype(np.float32), my.astype(np.float32), cv2_no_ipp.INTER_CUBIC,
                               borderMode=cv2_no_ipp.BORDER_REPLICATE)
        np.testing.assert_array_equal(out, img[y0:y1, x0:x1])
    t = rng.integers(0, 256, (128, 256, 3), dtype=np.uint8)
    for f in (0, 3, 8):                                  # h = 32, s = 4: the page of the rectangle call
        np.testing.assert_array_equal(R.compose(img, [_straight(13, 9, 77, 41)], [t], 4, f),
                                      RR.compose(img, [(13, 9, 77, 41)], [t], 4, f))


def test_curved_compose_equals_cv2_remap(cv2_no_ipp):
    """The twin's patch is cv2.remap of T at the twin's (u, v), blended where the footprint holds."""
    from marconet_b200.pipeline import CurvedRegion, curved_maps
    rng = np.random.default_rng(5)
    reg = CurvedRegion.from_arc(40, 40, 30, 20, 200, 340)
    t = rng.integers(0, 256, (128, 700, 3), dtype=np.uint8)
    s = 3
    box, p, a, mask = R.curved_patch(t, reg, s, (3 * 80, 3 * 80), 5)
    m = curved_maps(reg, s, 700)
    qx, qy = np.meshgrid((np.arange(box[0], box[2]) + 0.5) / s, (np.arange(box[1], box[3]) + 0.5) / s)
    ok, mm, tt, bb = R.invert(m, qx, qy)
    u, v = R.t_maps(m, mm, tt, bb, t.shape[:2])
    ref = cv2_no_ipp.remap(np.ascontiguousarray(t[..., ::-1]), np.where(ok, u, 0).reshape(qx.shape).astype(np.float32),
                           np.where(ok, v, 0).reshape(qx.shape).astype(np.float32), cv2_no_ipp.INTER_CUBIC,
                           borderMode=cv2_no_ipp.BORDER_REPLICATE)
    assert mask.mean() > 0.2
    np.testing.assert_array_equal(p[mask], ref[mask])


def _golden():
    from marconet_b200.pipeline import CurvedRegion, OrientedRegion
    g = np.load(GOLDEN)
    pts, regs, o = g["points"].tolist(), [], 0
    for kind, n in zip(g["kinds"].tolist(), g["n_points"].tolist()):
        p = [tuple(v) for v in pts[o:o + n]]
        regs.append(CurvedRegion(tuple(p[:n // 2]), tuple(p[n // 2:])) if kind == 3 else OrientedRegion(*p))
        o += n
    labels, boxes = [[] for _ in regs], [[] for _ in regs]
    for lab, (x1, y1, x2, y2, r) in zip(g["labels"].tolist(), g["boxes"].tolist()):
        labels[r].append(lab)
        boxes[r].append([x1, y1, x2, y2])
    return g, regs, labels, boxes


def test_twin_reproduces_golden_page():
    """Every stored page pixel outside the strided regions' footprints (no pixel outside them depends on their bytes) is the
    twin's composition of the other regions' stored bytes."""
    g, regs, _, _ = _golden()
    st, s = int(g["stride"]), int(g["scale"])
    whole = g["sr_strides"] == 1
    assert os.path.getsize(GOLDEN) < 620_000 and whole.sum() == len(regs) - 3
    srs = [g[f"sr{r}"] if whole[r] else None for r in range(len(regs))]
    full = R.compose(g["image"], regs, srs, s, int(g["feather"]))
    keep = np.ones(full.shape[:2], bool)
    for r in np.flatnonzero(~whole):
        (x0, y0, x1, y1), _, _, mask, _ = R.curved_footprint((128, int(g["sr_widths"][r])), regs[r], s, full.shape[:2], 8)
        keep[y0:y1, x0:x1] &= ~mask
    keep = keep[::st, ::st]
    assert keep.mean() > 0.7
    np.testing.assert_array_equal(full[::st, ::st][keep], g["page"][keep])
    assert not np.array_equal(g["page"], R.background(g["image"], s)[::st, ::st])


def test_plan_curved_regions():
    from marconet_b200 import pipeline
    g, regs, labels, boxes = _golden()
    plan = pipeline.plan_regions([g["image"].shape[:2]], [regs], [labels], [boxes], scale=4, feather=8)
    for p, reg, bx in zip(plan, regs, boxes):
        assert p.boxes == [[float(v) for v in b] for b in bx]
        if not isinstance(reg, pipeline.CurvedRegion):
            assert p.curved is None and p.oriented is not None
            continue
        assert p.curved == reg and p.oriented is None and p.quad is None and p.matrix is None
        assert p.size == pipeline.curved_maps(reg, 4).size
        assert p.out == pipeline.curved_footprint_box(reg, 4, (4 * 176, 4 * 320))
    assert plan[5].overlaps == [4]                          # the curved region over the oriented one
    assert plan[0].size[0] > 16 * plan[0].size[1]          # the seal's arc is wider than the canvas
    assert plan[6].out[2] == 4 * 320                        # partly off the page


LONG = (((0, 0), (6000, 0), (12000, 0), (20000, 0)), ((0, 100), (6000, 100), (12000, 100), (20000, 100)))


def _arc1(span):
    """One Bezier segment of an annulus (radii 20 and 30 about (50, 50)) over ``span`` degrees from 270 - span/2, read
    counter-clockwise with the inner arc on top."""
    h = 4 / 3 * math.tan(math.radians(span) / 4)
    a0, a1 = math.radians(270 - span / 2), math.radians(270 + span / 2)

    def seg(r):
        p0 = (50 + r * math.cos(a0), 50 - r * math.sin(a0))
        p3 = (50 + r * math.cos(a1), 50 - r * math.sin(a1))
        return (p0, (p0[0] - h * r * math.sin(a0), p0[1] - h * r * math.cos(a0)),
                (p3[0] + h * r * math.sin(a1), p3[1] + h * r * math.cos(a1)), p3)
    return seg(20), seg(30)


@pytest.mark.parametrize("reg,kw,match", [
    ((((0, 0), (1, 0), (2, 0), (math.nan, 0)), ((0, 5), (1, 5), (2, 5), (3, 5))), {}, "region 0: the control points are not"),
    ((((0, 0), (1, 0), (2, 0)), ((0, 5), (1, 5), (2, 5))), {}, "region 0: the curves have 3 and 3 points; both need 3k"),
    ((((0, 0), (1, 0), (2, 0), (3, 0)), ((0, 5), (1, 5), (1.5, 5), (2, 5), (2.5, 5), (3, 5), (3.5, 5))), {},
     "region 0: the curves have 4 and 7 points"),
    ((tuple((v, 0) for v in range(28)), tuple((v, 5) for v in range(28))), {}, r"region 0: the curves have 28 and 28 .* k <= 8"),
    ((((1, 1), (2, 1), (3, 1), (4, 1)), ((1, 1.2), (2, 1.2), (3, 1.2), (4, 1.2))), {}, "region 0: the band is 0.2 pixels high"),
    ((((1, 1), (5, 1), (6, 1), (7, 1), (7.2, 1), (7.4, 1), (7.6, 1)), ((1, 6), (5, 6), (6, 6), (7, 6), (7.2, 6), (7.4, 6), (7.6, 6))),
     {}, r"region 0: segment 1's mid curve is 0.6 pixels long, below h_r / 8 = 0.625"),
    ((((1, 6), (3, 6), (6, 6), (9, 6)), ((1, 1), (3, 1), (6, 1), (9, 1))), {}, "region 0: the band folds or runs against its"),
    ((((9, 1), (6, 1), (3, 1), (1, 1)), ((9, 6), (6, 6), (3, 6), (1, 6))), {}, "region 0: the band folds or runs against its"),
    ((((1, 1), (9, 6), (1, 6), (9, 1)), ((1, 3), (9, 8), (1, 8), (9, 3))), dict(shape=(20, 20)), "region 0: the band folds"),
    (_arc1(120), dict(shape=(100, 100)), r"region 0: the ruling B - T turns by 120 degrees within segment 0"),
    ((((0, 0), (10, 0), (20, 0), (30, 0)), ((0, 20), (10, 14), (20, 8), (30, 4))), dict(shape=(30, 40)),
     "region 0: the longest ruling 20 is more than 4 times the shortest 4"),
    ((((20, 1), (30, 1), (40, 1), (50, 1)), ((20, 6), (30, 6), (40, 6), (50, 6))), {}, r"mid point \(35, 3.5\) is outside the 10x8"),
    ((((0, 0), (30, 0), (60, 0), (90, 0)), ((0, 30), (30, 30), (60, 30), (90, 30))), dict(shape=(40000, 100)),
     "region 0: crop 90x30, restored width 384 or image 100x40000 exceeds 32767"),
    ((((0, 0), (100, 0), (200, 0), (300, 0)), ((0, 1), (100, 1), (200, 1), (300, 1))), dict(shape=(8, 400)),
     "region 0: crop 300x1, restored width 38400 .* exceeds"),
    (LONG, dict(shape=(200, 32767)), r"region 0: the crop map reaches 19998.9 pixels, beyond OpenCV's int16 remap coordinates"),
    ((((0, 0), (3, 0), (6, 0), (9, 0)), ((0, 5), (3, 5), (6, 5), (9, 5))), dict(labels=[[[1]]], boxes=[[[[1, 0, 9.5, 5]]]]),
     r"image 0, region 0, character 0: .* \[0, 9\]"),
    ((((0, 0), (3, 0), (6, 0), (9, 0)), ((0, 5), (3, 5), (6, 5), (9, 5))), dict(labels=[[[1, 2]]], boxes=[[[[1, 0, 3, 5]]]]),
     "image 0, region 0: 2 labels for 1 boxes"),
    ((((0, 0), (3, 0), (6, 0), (9, 0)), ((0, 5), (3, 5), (6, 5), (9, 5))), dict(labels=[[None]], boxes=[[[[1, 0, 3, 5]]]]),
     "image 0, region 0: boxes without labels"),
    (("ab", "cd"), {}, "image 0, region 0: expected two curves"),
])
def test_plan_rejects_curved(reg, kw, match):
    from marconet_b200 import pipeline
    args = dict(regions=[[pipeline.CurvedRegion(*reg)]], labels=None, boxes=None, scale=4, feather=None)
    args.update(kw)
    shape = args.pop("shape", (8, 10))
    with pytest.raises(ValueError, match=match):
        pipeline.plan_regions([shape], **args)


def test_plan_accepts_the_long_band_inside_the_int16_range():
    from marconet_b200 import pipeline
    top, bottom = ([(x * 0.8, y) for x, y in c] for c in LONG)
    plan = pipeline.plan_regions([(200, 32767)], [[pipeline.CurvedRegion(top, bottom)]], scale=1)
    assert plan[0].size == (16000, 100)


def test_vertical_region_on_a_curve_is_refused():
    from marconet_b200 import pipeline
    with pytest.raises(ValueError, match="image 0, region 1: the shape of a VerticalRegion is a CurvedRegion"):
        pipeline.plan_regions([(40, 40)], [[(0, 0, 5, 5), pipeline.VerticalRegion(_straight(5, 1, 15, 35))]])


def _fields(header, name):
    body = re.search(r"typedef struct \{([^{}]*)\}\s*" + name + ";", header).group(1)
    body = re.sub(r"/\*.*?\*/", "", body, flags=re.S)
    names = []
    for decl in body.split(";"):
        parts = [re.sub(r"\[\d+\]$", "", p.strip()) for p in decl.strip().split(",") if p.strip()]
        names += [re.findall(r"[A-Za-z_0-9]+$", p)[0] for p in parts]
    return names


@pytest.mark.parametrize("c_name,py_name,size", [("mn_remap_curved_image", "RemapCurvedImage", 64),
                                                 ("mn_region_curved", "RegionCurved", 184)])
def test_curved_structs_match_header(c_name, py_name, size):
    from marconet_b200 import _lib
    header = open(os.path.join(ROOT, "include", "marconet_b200.h")).read()
    cls = getattr(_lib, py_name)
    assert _fields(header, c_name) == [f[0] for f in cls._fields_]
    assert ctypes.sizeof(cls) == size
    assert re.search(r"#define MN_REGION_CURVED 3\s", header) and _lib.REGION_CURVED == 3
    if py_name == "RegionCurved":
        assert (cls.q.offset, cls.curve.offset, cls.n_seg.offset) == (0, 168, 176)
    else:
        assert (cls.curve.offset, cls.n_seg.offset) == (48, 56)


def test_curved_kernels_build_without_spills(tmp_path):
    import subprocess
    from marconet_b200 import build
    src = os.path.join(ROOT, "marconet_b200", "csrc", "image_ops.cu")
    r = subprocess.run([build.nvcc_path(), "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-DMN_BUILD", "-Xptxas", "-v",
                        "-cubin", src, "-o", str(tmp_path / "image_ops.cubin")], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-2000:]
    for kernel in ("remap_curved_batched_kernel", "composite_regions_curved_kernel"):
        props = re.search(kernel + r"[^\n]*\n[^\n]*Function properties for [^\n]*" + kernel + r"[^\n]*\n([^\n]*)", r.stderr)
        assert props, f"no ptxas report for {kernel}"
        assert "0 bytes spill stores, 0 bytes spill loads" in props.group(1), props.group(1)
