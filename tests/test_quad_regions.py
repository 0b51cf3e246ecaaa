"""Perspective text regions on the CPU (DESIGN.md section 7b, "Perspective text regions"): the numpy twin of cv2.warpPerspective
against live cv2 (IPP off), pipeline.quad_maps by hand and against oriented_maps, the footprint box, plan_regions' validation of
QuadRegions, the golden page, and the layout and register report of the two kernels."""
import ctypes
import math
import os
import re

import numpy as np
import pytest

from oracle import quad_regions as R
from oracle import warp_perspective as P

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "quad_regions.npz")


@pytest.fixture
def cv2_no_ipp():
    cv2 = pytest.importorskip("cv2")
    was = cv2.ipp.useIPP()
    cv2.ipp.setUseIPP(False)
    yield cv2
    cv2.ipp.setUseIPP(was)


def _cv2_warp(cv2, src, m, dsize):
    out = cv2.warpPerspective(src, np.asarray(m, np.float64), dsize, flags=cv2.INTER_CUBIC | cv2.WARP_INVERSE_MAP,
                              borderMode=cv2.BORDER_REPLICATE)
    return out.reshape(dsize[1], dsize[0], src.shape[2])


def _random_homography(rng):
    a = math.radians(rng.uniform(-180, 180))
    sx, sy = rng.uniform(0.25, 4.0, 2)
    rot = np.array([[math.cos(a), -math.sin(a)], [math.sin(a), math.cos(a)]])
    lin = rot @ np.diag([sx, sy]) @ np.array([[1, rng.uniform(-0.6, 0.6)], [0, 1]])
    m = np.vstack([np.hstack([lin, rng.uniform(-40, 90, (2, 1))]), [0, 0, 1]])
    m[2, :2] = rng.uniform(-0.004, 0.004, 2)
    return m


def warp_cases():
    rng = np.random.default_rng(12)
    cases = []
    for k in range(12):                                  # rotations, scales 0.25 to 4, shears and a perspective row
        src = rng.integers(0, 256, (57, 91, 3), dtype=np.uint8)
        cases.append((f"random{k}", src, _random_homography(rng), (120, 80)))
    persp = [[0.41, 0.13, -3.0], [0.2, 0.7, -0.4], [0.003, -0.002, 1.1]]
    cases.append(("1x1", rng.integers(0, 256, (1, 1, 3), dtype=np.uint8), [[0.3, 0.1, -2.0], [0.2, 0.7, 1.0], [0.01, 0, 1]], (9, 7)))
    cases.append(("1xN", rng.integers(0, 256, (1, 23, 3), dtype=np.uint8), persp, (40, 7)))
    cases.append(("Nx1", rng.integers(0, 256, (23, 1, 3), dtype=np.uint8), persp, (7, 40)))
    cases.append(("outside", rng.integers(0, 256, (20, 30, 3), dtype=np.uint8),
                  [[0.9, 0.3, -60.0], [-0.3, 0.9, 45.0], [0.002, 0.001, 0.9]], (90, 70)))
    cases.append(("zoom32", rng.integers(0, 256, (6, 7, 3), dtype=np.uint8), [[1 / 32, 0, 1.3], [0, 1 / 32, 2.1], [0, 0, 1]], (96, 96)))
    cases.append(("wide", rng.integers(0, 256, (40, 300, 3), dtype=np.uint8),
                  [[0.25, 0.02, 3.0], [0.001, 0.9, 1.0], [2e-4, 0.0, 1.0]], (1500, 30)))
    cases.append(("cn1", rng.integers(0, 256, (31, 45, 1), dtype=np.uint8), _random_homography(rng), (50, 33)))
    return cases


@pytest.mark.parametrize("name,src,m,dsize", warp_cases(), ids=[c[0] for c in warp_cases()])
def test_warp_twin_equals_cv2(cv2_no_ipp, name, src, m, dsize):
    np.testing.assert_array_equal(P.warp_perspective_cubic_u8(src, m, dsize), _cv2_warp(cv2_no_ipp, src, m, dsize))


def test_zoom_case_hits_every_fraction_pair():
    xq, yq = P.warp_coords([[1 / 32, 0, 1.3], [0, 1 / 32, 2.1], [0, 0, 1]], np.arange(96), np.arange(96), (96, 96))
    assert len(set(((yq & 31) * 32 + (xq & 31)).ravel().tolist())) == 1024


def test_integer_translation_is_a_copy(cv2_no_ipp):
    rng = np.random.default_rng(2)
    src = rng.integers(0, 256, (30, 40, 3), dtype=np.uint8)
    m = [[1, 0, 7], [0, 1, 5], [0, 0, 1]]
    np.testing.assert_array_equal(P.warp_perspective_cubic_u8(src, m, (20, 12)), src[5:17, 7:27])
    np.testing.assert_array_equal(_cv2_warp(cv2_no_ipp, src, m, (20, 12)), src[5:17, 7:27])


def test_quad_maps_by_hand():
    """tl (0, 0), tr (4, 0), br (3, 2), bl (1, 2): g = 0, h = 1, H = [[4, 2, 0], [0, 4, 0], [0, 1, 1]]."""
    from marconet_b200.pipeline import QuadRegion, quad_maps
    m = quad_maps(QuadRegion((0, 0), (4, 0), (3, 2), (1, 2)), 1)
    assert m.homography == ((4, 2, 0), (0, 4, 0), (0, 1, 1))
    assert m.size == (4, 2) and m.t_width == 256
    assert m.matrix.tolist() == [[1, 0.75, 0.375], [0, 1.75, 0.375], [0, 0.5, 1.25]]
    # crop pixel (0, 0) is (u, v) = (1/8, 1/4): image point (1/1.25, 1/1.25), pixel indices (0.3, 0.3)
    x, y, w = m.matrix @ [0, 0, 1]
    assert (x / w, y / w) == pytest.approx((0.3, 0.3), abs=1e-15)
    assert m.kx == float(np.float32(6 / (math.sqrt(5) * 256))) and m.ky == 1 / 64
    # N inverts H: the page pixel of image point (3, 2) (br) at s = 2 lands on T's far corner (W_T - 0.5, 127.5)
    m2 = quad_maps(QuadRegion((0, 0), (4, 0), (3, 2), (1, 2)), 2)
    u, v, w = m2.page_map @ [2 * 3 - 0.5, 2 * 2 - 0.5, 1]
    assert (u / w, v / w) == pytest.approx((255.5, 127.5), abs=1e-12)
    c = m2.page_map @ [2 * 2 - 0.5, 2 * (4 / 3) - 0.5, 1]              # the footprint centre H(0.5, 0.5) = (2, 4/3)
    assert c[2] == pytest.approx(1, abs=1e-15)


def test_integer_rectangles_are_exact(cv2_no_ipp):
    from marconet_b200.pipeline import QuadRegion, quad_maps
    rng = np.random.default_rng(3)
    img = rng.integers(0, 256, (50, 80, 3), dtype=np.uint8)
    for x0, y0, x1, y1 in ((0, 0, 80, 50), (7, 3, 61, 35), (79, 49, 80, 50), (12, 20, 13, 45)):
        q = QuadRegion((x0, y0), (x1, y0), (x1, y1), (x0, y1))
        m = quad_maps(q, 1)
        assert m.matrix.tolist() == [[1, 0, x0], [0, 1, y0], [0, 0, 1]] and m.size == (x1 - x0, y1 - y0)
        np.testing.assert_array_equal(R.rectify(img, q), img[y0:y1, x0:x1])
        np.testing.assert_array_equal(_cv2_warp(cv2_no_ipp, img, m.matrix, m.size), img[y0:y1, x0:x1])
    for x0, y0, x1, y1 in ((13, 9, 77, 41), (0, 0, 5, 32), (100, 7, 1000, 39)):           # h = 32, s = 4
        m = quad_maps(QuadRegion((x0, y0), (x1, y0), (x1, y1), (x0, y1)), 4)
        assert m.page_map.tolist() == [[1, 0, -4 * x0], [0, 1, -4 * y0], [0, 0, 1]]
        assert m.t_width == 4 * (x1 - x0) and m.kx == m.ky == 1.0


def test_parallelograms_agree_with_oriented_maps():
    from marconet_b200.pipeline import OrientedRegion, QuadRegion, oriented_maps, quad_maps
    rng = np.random.default_rng(4)
    for _ in range(100):
        o = OrientedRegion.from_rotated(*rng.uniform(20, 200, 2), rng.uniform(5, 300), rng.uniform(3, 40), rng.uniform(-180, 180))
        (tlx, tly), (trx, try_), (blx, bly) = o
        q = QuadRegion(o.tl, o.tr, (trx + blx - tlx, try_ + bly - tly), o.bl)
        for s in (1, 3, 4):
            a, b = oriented_maps(o, s), quad_maps(q, s)
            assert a.size == b.size and a.t_width == b.t_width
            np.testing.assert_allclose(b.matrix[:2], a.matrix, rtol=0, atol=1e-12)
            np.testing.assert_allclose(b.matrix[2], [0, 0, 1], rtol=0, atol=1e-12)
            np.testing.assert_allclose(b.page_map[:2], a.page_map, rtol=1e-12, atol=1e-12)
            np.testing.assert_allclose(b.page_map[2], [0, 0, 1], rtol=0, atol=1e-12)
            assert b.kx == pytest.approx(a.kx, rel=1e-6) and b.ky == pytest.approx(a.ky, rel=1e-6)


def _random_quad(rng, H, W):
    """A valid QuadRegion of an H x W image: a rotated trapezoid whose far side is up to 3 times shorter."""
    from marconet_b200 import pipeline
    while True:
        L, w = rng.uniform(4, 30), rng.uniform(10, W * 0.8)
        R_ = L / rng.uniform(1, 3)
        pts = np.array([[0, -L / 2], [w, -R_ / 2], [w, R_ / 2], [0, L / 2]])
        if rng.random() < 0.5:
            pts = pts[[0, 1, 2, 3]] * [-1, 1]
            pts = pts[[1, 0, 3, 2]]
        a = rng.uniform(-math.pi, math.pi)
        rot = np.array([[math.cos(a), -math.sin(a)], [math.sin(a), math.cos(a)]])
        q = pipeline.QuadRegion(*map(tuple, pts @ rot.T + [rng.uniform(0, W), rng.uniform(0, H)]))
        try:
            pipeline.plan_regions([(H, W)], [[q]], scale=1)
            return q
        except ValueError:
            continue


def test_footprint_box_holds_the_footprint():
    """The box holds every pixel that cv2's fixed-point coordinates over the whole page mark inside the footprint."""
    from marconet_b200.pipeline import quad_footprint_box, quad_maps
    rng = np.random.default_rng(6)
    for k in range(12):
        q = _random_quad(rng, 40, 70)
        for s in (1, 2, 4):
            m = quad_maps(q, s, int(rng.integers(1, 3)) + quad_maps(q, s).t_width)
            x0, y0, x1, y1 = quad_footprint_box(m, s, (40 * s, 70 * s))
            xq, yq = P.warp_coords(m.page_map, np.arange(70 * s), np.arange(40 * s), (70 * s, 40 * s))
            inside = (xq >= -16) & (xq < 32 * m.t_width - 16) & (yq >= -16) & (yq < 32 * 128 - 16)
            assert inside[y0:y1, x0:x1].sum() == inside.sum() > 0, (k, s)


def test_quad_compose_equals_cv2_warp(cv2_no_ipp):
    """Inside the footprint the twin's P is cv2.warpPerspective of the whole page by N; outside it the page keeps its
    background."""
    from marconet_b200.pipeline import QuadRegion, quad_maps
    rng = np.random.default_rng(5)
    img = rng.integers(0, 256, (40, 70, 3), dtype=np.uint8)
    reg = QuadRegion((12, 10), (60, 6), (61, 30), (10, 26))
    for s in (1, 3):
        m = quad_maps(reg, s)
        t = rng.integers(0, 256, (128, m.t_width, 3), dtype=np.uint8)
        full = _cv2_warp(cv2_no_ipp, np.ascontiguousarray(t[..., ::-1]), m.page_map, (70 * s, 40 * s))
        (x0, y0, x1, y1), p, a, mask = R.quad_patch(t, reg, s, (40 * s, 70 * s), 0)
        np.testing.assert_array_equal(p, full[y0:y1, x0:x1])
        assert mask.any() and not (mask[0].any() or mask[-1].any() or mask[:, 0].any() or mask[:, -1].any())
        out = R.compose(img, [reg], [t], s, 0)
        bg = R.background(img, s)
        sl = np.zeros(bg.shape[:2], bool)
        sl[y0:y1, x0:x1] = mask
        np.testing.assert_array_equal(out[sl], full[sl])
        np.testing.assert_array_equal(out[~sl], bg[~sl])


def test_reduction_to_a_rectangle():
    """h = 32, s = 4: an interior integer rectangle given as a QuadRegion composes exactly as the rectangle."""
    from marconet_b200.pipeline import QuadRegion
    rng = np.random.default_rng(4)
    img = rng.integers(0, 256, (60, 100, 3), dtype=np.uint8)
    reg = QuadRegion((13, 9), (77, 9), (77, 41), (13, 41))
    t = rng.integers(0, 256, (128, 256, 3), dtype=np.uint8)
    for f in (0, 3, 8):
        np.testing.assert_array_equal(R.compose(img, [reg], [t], 4, f), R.compose(img, [(13, 9, 77, 41)], [t], 4, f))


def _golden():
    from marconet_b200.pipeline import QuadRegion
    g = np.load(GOLDEN)
    regs = [QuadRegion(*map(tuple, c)) if k == 2 else (int(c[0][0]), int(c[0][1]), int(c[2][0]), int(c[2][1]))
            for k, c in zip(g["kinds"].tolist(), g["corners"].tolist())]
    labels, boxes = [[] for _ in regs], [[] for _ in regs]
    for lab, (x1, y1, x2, y2, r) in zip(g["labels"].tolist(), g["boxes"].tolist()):
        labels[r].append(lab)
        boxes[r].append([x1, y1, x2, y2])
    return g, regs, labels, boxes


def test_twin_reproduces_golden_page():
    """Every stored page pixel outside the wide region's footprint (whose SR bytes are stored strided; no pixel outside it
    depends on them) is the twin's composition of the other regions' stored bytes."""
    from marconet_b200.pipeline import quad_footprint_box, quad_maps
    g, regs, _, _ = _golden()
    st, s = int(g["stride"]), int(g["scale"])
    whole = g["sr_strides"] == 1
    assert whole.sum() == len(regs) - 1
    srs = [g[f"sr{r}"] if whole[r] else None for r in range(len(regs))]
    full = R.compose(g["image"], regs, srs, s, int(g["feather"]))
    keep = np.ones(full.shape[:2], bool)
    for r in np.flatnonzero(~whole):
        m = quad_maps(regs[r], s, int(g["sr_widths"][r]))
        x0, y0, x1, y1 = quad_footprint_box(m, s, full.shape[:2])
        xq, yq = P.warp_coords(m.page_map, np.arange(x0, x1), np.arange(y0, y1), full.shape[1::-1])
        keep[y0:y1, x0:x1] &= ~((xq >= -16) & (xq < 32 * int(g["sr_widths"][r]) - 16) & (yq >= -16) & (yq < 32 * 128 - 16))
    keep = keep[::st, ::st]
    assert keep.mean() > 0.8
    np.testing.assert_array_equal(full[::st, ::st][keep], g["page"][keep])
    assert not np.array_equal(g["page"], R.background(g["image"], s)[::st, ::st])


def test_plan_quad_regions():
    from marconet_b200 import pipeline
    g, regs, labels, boxes = _golden()
    plan = pipeline.plan_regions([g["image"].shape[:2]], [regs], [labels], [boxes], scale=4, feather=8)
    for p, reg, bx in zip(plan, regs, boxes):
        if not isinstance(reg, pipeline.QuadRegion):
            assert p.quad is None and p.oriented is None and p.out == tuple(4 * v for v in reg)
            continue
        assert p.quad == reg and p.oriented is None and p.boxes == [[float(v) for v in b] for b in bx]
        m = pipeline.quad_maps(reg, 4)
        assert p.size == m.size and np.array_equal(p.matrix, m.matrix)
        assert p.out == pipeline.quad_footprint_box(m, 4, (4 * 128, 4 * 360))
    assert plan[3].overlaps == [2]                          # the quad over the rectangle
    assert plan[0].size == (280, 16)


BEHIND = ((33.97973038638403, 16.57158735391618), (19.529221952984074, 21.495003526899268), (6.111386821220968, 15.637427820988794),
          (-0.10234046845014433, 1.6930090820900228))         # the far side short and turned: the box reaches N's vanishing line


@pytest.mark.parametrize("reg,kw,match", [
    (((0, 0), (math.nan, 0), (5, 5), (0, 5)), {}, "image 0, region 0: corners .* are not finite"),
    (((1, 1), (1.9, 1), (1.9, 6), (1, 6)), {}, r"image 0, region 0: sides \[0.9, "),
    (((1, 6), (9, 6), (9, 1), (1, 1)), {}, "image 0, region 0: the quad is not strictly convex in reading order .* at tl"),
    (((1, 1), (9, 1), (1, 6), (9, 6)), {}, "image 0, region 0: the quad is not strictly convex in reading order .* at br"),
    (((1, 1), (9, 1), (13, 3), (5, 3)), {}, r"image 0, region 0: the interior angle at tl is outside \[30, 150\] degrees"),
    (((1, 3.5), (9, 0.5), (9, 7.5), (1, 4.5)), {}, "image 0, region 0: the foreshortening 7 exceeds 4"),
    (((20, 1), (40, 1), (40, 6), (20, 6)), {}, r"image 0, region 0: the centre \(30, 3.5\) is outside the 10x8 image"),
    (((0, 0), (40000, 0), (40000, 5), (0, 5)), dict(shape=(8, 40000)), "image 0, region 0: crop 40000x5, .* exceeds 32767"),
    (((0, 0), (300, 0), (300, 1), (0, 1)), dict(shape=(8, 400)), "image 0, region 0: crop 300x1, restored width 38400 .* exceeds"),
    (((0, 0), (30, 0), (30, 10), (0, 10)), dict(shape=(40000, 40)), "image 0, region 0: .* image 40x40000 exceeds 32767"),
    (BEHIND, dict(shape=(70, 70)), "image 0, region 0: the page map's denominator is not positive over the footprint box"),
    (((0, 0), (9, 0), (9, 5), (0, 5)), dict(labels=[[[1]]], boxes=[[[[1, 0, 9.5, 5]]]]), r"image 0, region 0, character 0: .* \[0, 9\]"),
    (((0, 0), (9, 0), (9, 5), (0, 5)), dict(labels=[[[1, 2]]], boxes=[[[[1, 0, 3, 5]]]]), "image 0, region 0: 2 labels for 1 boxes"),
    (((0, 0), (9, 0), (9, 5), (0, 5)), dict(labels=[[None]], boxes=[[[[1, 0, 3, 5]]]]), "image 0, region 0: boxes without labels"),
    (("a", "b", "c", "d"), {}, "image 0, region 0: expected four"),
])
def test_plan_rejects_quad(reg, kw, match):
    from marconet_b200 import pipeline
    args = dict(regions=[[pipeline.QuadRegion(*reg)]], labels=None, boxes=None, scale=4, feather=None)
    args.update(kw)
    shape = args.pop("shape", (8, 10))
    with pytest.raises(ValueError, match=match):
        pipeline.plan_regions([shape], **args)


NEAR = ((33.97973038638403, 16.57158735391618), (20.54469098811772, 21.93830803108284), (5.095917786087324, 15.194123316805221),
        (-0.10234046845014433, 1.6930090820900228))         # BEHIND's far side widened until a box corner sits just inside the
#                                                             vanishing line: a positive denominator near 0, coordinates past 2^30


def test_plan_rejects_quad_fixed_point_overflow():
    from marconet_b200 import pipeline
    good = pipeline.QuadRegion((1, 1), (9, 1), (9, 6), (1, 6))
    with pytest.raises(ValueError, match="image 1, region 2: the quad is not strictly convex"):
        pipeline.plan_regions([(8, 10), (8, 10)], [[good], [good, (0, 0, 2, 2), pipeline.QuadRegion((1, 6), (9, 6), (9, 1), (1, 1))]])
    with pytest.raises(ValueError, match="image 0, region 0: the map onto its .* exceeds OpenCV's 32-bit fixed-point"):
        pipeline.plan_regions([(70, 70)], [[pipeline.QuadRegion(*NEAR)]], scale=1)


def _fields(header, name):
    body = re.search(r"typedef struct \{([^{}]*)\}\s*" + name + ";", header).group(1)
    body = re.sub(r"/\*.*?\*/", "", body, flags=re.S)
    names = []
    for decl in body.split(";"):
        parts = [re.sub(r"\[\d+\]$", "", p.strip()) for p in decl.strip().split(",") if p.strip()]
        names += [re.findall(r"[A-Za-z_0-9]+$", p)[0] for p in parts]
    return names


@pytest.mark.parametrize("c_name,py_name,size", [("mn_warp_perspective_image", "WarpPerspectiveImage", 120),
                                                 ("mn_region_quad", "RegionQuad", 168)])
def test_quad_structs_match_header(c_name, py_name, size):
    from marconet_b200 import _lib
    header = open(os.path.join(ROOT, "include", "marconet_b200.h")).read()
    cls = getattr(_lib, py_name)
    assert _fields(header, c_name) == [f[0] for f in cls._fields_]
    assert ctypes.sizeof(cls) == size
    assert re.search(r"#define MN_REGION_PERSPECTIVE 2\s", header) and _lib.REGION_PERSPECTIVE == 2
    assert cls.m.offset == 48 if py_name == "WarpPerspectiveImage" else (cls.r.offset, cls.kind.offset, cls.n.offset) == (0, 80, 96)


def test_quad_kernels_build_without_spills(tmp_path):
    import subprocess
    from marconet_b200 import build
    src = os.path.join(ROOT, "marconet_b200", "csrc", "image_ops.cu")
    r = subprocess.run([build.nvcc_path(), "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-DMN_BUILD", "-Xptxas", "-v",
                        "-cubin", src, "-o", str(tmp_path / "image_ops.cubin")], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-2000:]
    for kernel in ("warp_perspective_batched_kernel", "composite_regions_quad_kernel"):
        props = re.search(kernel + r"[^\n]*\n[^\n]*Function properties for [^\n]*" + kernel + r"[^\n]*\n([^\n]*)", r.stderr)
        assert props, f"no ptxas report for {kernel}"
        assert "0 bytes spill stores, 0 bytes spill loads" in props.group(1), props.group(1)
