"""Oriented text regions on the CPU (DESIGN.md section 7b, "Oriented text regions"): the numpy twin of cv2.warpAffine against live
cv2 (IPP off), pipeline.oriented_maps and OrientedRegion.from_rotated by hand, the golden page, plan_regions' validation of
oriented regions, and the layout and register report of the two kernels."""
import ctypes
import math
import os
import re

import numpy as np
import pytest

from oracle import warp_affine as I
from oracle import oriented_regions as R

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "oriented_regions.npz")


@pytest.fixture
def cv2_no_ipp():
    cv2 = pytest.importorskip("cv2")
    was = cv2.ipp.useIPP()
    cv2.ipp.setUseIPP(False)
    yield cv2
    cv2.ipp.setUseIPP(was)


def _cv2_warp(cv2, src, m, dsize):
    return cv2.warpAffine(src, np.asarray(m, np.float64), dsize, flags=cv2.INTER_CUBIC | cv2.WARP_INVERSE_MAP,
                          borderMode=cv2.BORDER_REPLICATE)


def _random_matrix(rng, max_scale=4.0):
    a = math.radians(rng.uniform(-180, 180))
    sx, sy = rng.uniform(0.25, max_scale, 2)
    rot = np.array([[math.cos(a), -math.sin(a)], [math.sin(a), math.cos(a)]])
    lin = rot @ np.diag([sx, sy]) @ np.array([[1, rng.uniform(-0.6, 0.6)], [0, 1]])
    return np.hstack([lin, rng.uniform(-40, 90, (2, 1))])


def warp_cases():
    rng = np.random.default_rng(11)
    cases = []
    for k in range(12):                                  # rotations over +-180 degrees, scales 0.25 to 4, shears
        src = rng.integers(0, 256, (57, 91, 3), dtype=np.uint8)
        cases.append((f"random{k}", src, _random_matrix(rng), (120, 80)))
    cases.append(("1x1", rng.integers(0, 256, (1, 1, 3), dtype=np.uint8), [[0.3, 0.1, -2.0], [0.2, 0.7, 1.0]], (9, 7)))
    cases.append(("1xN", rng.integers(0, 256, (1, 23, 3), dtype=np.uint8), [[0.41, 0.13, -3.0], [0.2, 0.7, -0.4]], (40, 7)))
    cases.append(("Nx1", rng.integers(0, 256, (23, 1, 3), dtype=np.uint8), [[0.41, 0.13, -3.0], [0.2, 0.7, -0.4]], (7, 40)))
    cases.append(("outside", rng.integers(0, 256, (20, 30, 3), dtype=np.uint8), [[0.9, 0.3, -60.0], [-0.3, 0.9, 45.0]], (90, 70)))
    cases.append(("zoom32", rng.integers(0, 256, (6, 7, 3), dtype=np.uint8), [[1 / 32, 0, 1.3], [0, 1 / 32, 2.1]], (96, 96)))
    return cases


@pytest.mark.parametrize("name,src,m,dsize", warp_cases(), ids=[c[0] for c in warp_cases()])
def test_warp_twin_equals_cv2(cv2_no_ipp, name, src, m, dsize):
    np.testing.assert_array_equal(I.warp_affine_cubic_u8(src, m, dsize), _cv2_warp(cv2_no_ipp, src, m, dsize))


def test_zoom_case_hits_every_fraction_pair():
    xq, yq = I.warp_coords([[1 / 32, 0, 1.3], [0, 1 / 32, 2.1]], np.arange(96), np.arange(96))
    assert len(set(((yq & 31) * 32 + (xq & 31)).ravel().tolist())) == 1024


def test_warp_taps_sum_to_one():
    tab = I.warp_taps()
    assert tab.shape == (32, 32, 4, 4)
    np.testing.assert_array_equal(tab.sum(axis=(2, 3)), 32768)
    assert tab[0, 0, 1, 1] == 32767 and tab[0, 0, 2, 2] == 1         # int16 saturation, then the fix-up at taps (2, 2)


def test_axis_aligned_maps_are_exact(cv2_no_ipp):
    from marconet_b200.pipeline import OrientedRegion, oriented_maps
    rng = np.random.default_rng(3)
    img = rng.integers(0, 256, (50, 80, 3), dtype=np.uint8)
    for x0, y0, x1, y1 in ((0, 0, 80, 50), (7, 3, 61, 35), (79, 49, 80, 50), (12, 20, 13, 45)):
        m = oriented_maps(OrientedRegion((x0, y0), (x1, y0), (x0, y1)), 1)
        assert m.matrix.tolist() == [[1, 0, x0], [0, 1, y0]] and m.size == (x1 - x0, y1 - y0)
        np.testing.assert_array_equal(R.rectify(img, OrientedRegion((x0, y0), (x1, y0), (x0, y1))), img[y0:y1, x0:x1])
        np.testing.assert_array_equal(_cv2_warp(cv2_no_ipp, img, m.matrix, m.size), img[y0:y1, x0:x1])


def test_reduction_to_a_rectangle():
    """h = 32, s = 4: N is an integer translation, kx = ky = 1, and the page is the rectangle's, bit for bit."""
    from marconet_b200.pipeline import OrientedRegion, oriented_maps
    rng = np.random.default_rng(4)
    img = rng.integers(0, 256, (60, 100, 3), dtype=np.uint8)
    reg = OrientedRegion((13, 9), (77, 9), (13, 41))
    m = oriented_maps(reg, 4)
    assert m.t_width == 256 and m.kx == m.ky == 1.0
    assert m.page_map.tolist() == [[1, 0, -52], [0, 1, -36]]
    t = rng.integers(0, 256, (128, 256, 3), dtype=np.uint8)
    for f in (0, 3, 8):
        np.testing.assert_array_equal(R.compose(img, [reg], [t], 4, f), R.compose(img, [(13, 9, 77, 41)], [t], 4, f))


def test_from_rotated_corners():
    from marconet_b200.pipeline import OrientedRegion
    assert OrientedRegion.from_rotated(10, 20, 8, 4, 0) == ((6, 18), (14, 18), (6, 22))
    r = OrientedRegion.from_rotated(10, 20, 8, 4, 90)            # e = (0, -8), f = (4, 0), tl = c - e/2 - f/2 = (8, 24)
    np.testing.assert_allclose(np.array(r), [[8, 24], [8, 16], [12, 24]], atol=1e-12)
    r = OrientedRegion.from_rotated(10, 20, 8, 4, 30)            # e = 8 (cos 30, -sin 30), f = 4 (sin 30, cos 30)
    c, s = math.sqrt(3) / 2, 0.5
    tl = (10 - 4 * c - 2 * s, 20 + 4 * s - 2 * c)
    np.testing.assert_allclose(np.array(r), [tl, (tl[0] + 8 * c, tl[1] - 8 * s), (tl[0] + 4 * s, tl[1] + 4 * c)], atol=1e-12)
    r = OrientedRegion.from_rotated(0.5, 0.5, 3, 2, -180)        # upside down: reads right to left
    np.testing.assert_allclose(np.array(r), [[2, 1.5], [-1, 1.5], [2, -0.5]], atol=1e-12)


def test_oriented_compose_equals_cv2_warp(cv2_no_ipp):
    """Inside the footprint the twin's P is cv2.warpAffine of the whole page by N; outside it the page keeps its background."""
    from marconet_b200.pipeline import OrientedRegion, oriented_maps
    rng = np.random.default_rng(5)
    img = rng.integers(0, 256, (40, 70, 3), dtype=np.uint8)
    reg = OrientedRegion.from_rotated(35, 20, 40, 14, 23)
    for s in (1, 3):
        m = oriented_maps(reg, s)
        t = rng.integers(0, 256, (128, m.t_width, 3), dtype=np.uint8)
        full = _cv2_warp(cv2_no_ipp, np.ascontiguousarray(t[..., ::-1]), oriented_maps(reg, s, t.shape[1]).page_map, (70 * s, 40 * s))
        (x0, y0, x1, y1), p, a, mask = R.oriented_patch(t, reg, s, (40 * s, 70 * s), 0)
        np.testing.assert_array_equal(p, full[y0:y1, x0:x1])
        assert mask.any() and not (mask[0].any() or mask[-1].any() or mask[:, 0].any() or mask[:, -1].any())
        out = R.compose(img, [reg], [t], s, 0)
        bg = R.background(img, s)
        sl = np.zeros(bg.shape[:2], bool)
        sl[y0:y1, x0:x1] = mask
        np.testing.assert_array_equal(out[sl], full[sl])
        np.testing.assert_array_equal(out[~sl], bg[~sl])


def _golden():
    from marconet_b200.pipeline import OrientedRegion
    g = np.load(GOLDEN)
    regs = [OrientedRegion(*map(tuple, c)) for c in g["corners"].tolist()]
    labels, boxes = [[] for _ in regs], [[] for _ in regs]
    for lab, (x1, y1, x2, y2, r) in zip(g["labels"].tolist(), g["boxes"].tolist()):
        labels[r].append(lab)
        boxes[r].append([x1, y1, x2, y2])
    return g, regs, labels, boxes


def test_twin_reproduces_golden_page():
    """Every stored page pixel outside the wide region's footprint (whose SR bytes are stored strided; no pixel outside it
    depends on them) is the twin's composition of the other regions' stored bytes."""
    from marconet_b200.pipeline import footprint_box, oriented_maps
    g, regs, _, _ = _golden()
    st, s = int(g["stride"]), int(g["scale"])
    whole = g["sr_strides"] == 1
    assert whole.sum() == len(regs) - 1
    srs = [g[f"sr{r}"] if whole[r] else None for r in range(len(regs))]
    full = R.compose(g["image"], regs, srs, s, int(g["feather"]))
    keep = np.ones(full.shape[:2], bool)
    for r in np.flatnonzero(~whole):
        m = oriented_maps(regs[r], s, int(g["sr_widths"][r]))
        x0, y0, x1, y1 = footprint_box(regs[r], m, s, full.shape[:2])
        xq, yq = I.warp_coords(m.page_map, np.arange(x0, x1), np.arange(y0, y1))
        keep[y0:y1, x0:x1] &= ~((xq >= -16) & (xq < 32 * int(g["sr_widths"][r]) - 16) & (yq >= -16) & (yq < 32 * 128 - 16))
    keep = keep[::st, ::st]
    assert keep.mean() > 0.8
    np.testing.assert_array_equal(full[::st, ::st][keep], g["page"][keep])
    assert not np.array_equal(g["page"], R.background(g["image"], s)[::st, ::st])


def test_plan_oriented_regions():
    from marconet_b200 import pipeline
    g, regs, labels, boxes = _golden()
    plan = pipeline.plan_regions([g["image"].shape[:2]], [regs + [(0, 0, 10, 10)]], [labels + [None]], [boxes + [None]],
                                 scale=4, feather=8)
    for p, reg, bx in zip(plan, regs, boxes):
        assert p.oriented == reg and p.boxes == [[float(v) for v in b] for b in bx]          # boxes stay in the crop's frame
        m = pipeline.oriented_maps(reg, 4)
        assert p.size == m.size and np.array_equal(p.matrix, m.matrix)
        assert p.out == pipeline.footprint_box(reg, m, 4, (4 * 128, 4 * 360))
    assert plan[-1].oriented is None and plan[-1].out == (0, 0, 40, 40) and plan[-1].overlaps == []
    assert plan[4].overlaps == [0, 3]                       # footprint boxes meet: the region at 35 degrees and the axis-aligned one
    assert plan[0].size == (264, 16)


@pytest.mark.parametrize("reg,kw,match", [
    (((0, 0), (math.nan, 0), (0, 5)), {}, "image 0, region 0: corners .* are not finite"),
    (((1, 1), (1.9, 1), (1, 6)), {}, r"image 0, region 0: sides \|e\| = 0.9"),
    (((1, 1), (9, 1), (1, 1.5)), {}, r"image 0, region 0: sides"),
    (((1, 6), (9, 6), (1, 1)), {}, "image 0, region 0: the region is mirrored"),
    (((1, 1), (9, 1), (9.5, 2)), {}, "image 0, region 0: the region is sheared"),
    (((20, 1), (40, 1), (20, 6)), {}, r"image 0, region 0: the centre \(30, 3.5\) is outside the 10x8 image"),
    (((0, 0), (40000, 0), (0, 5)), dict(shape=(8, 40000)), "image 0, region 0: crop 40000x5, .* exceeds 32767"),
    (((0, 0), (300, 0), (0, 1)), dict(shape=(8, 400)), "image 0, region 0: crop 300x1, restored width 38400 .* exceeds 32767"),
    (((0, 0), (30, 0), (0, 10)), dict(shape=(40000, 40)), "image 0, region 0: .* image 40x40000 exceeds 32767"),
    (((0, 0), (9, 0), (0, 5)), dict(labels=[[[1]]], boxes=[[[[1, 0, 9.5, 5]]]]), r"image 0, region 0, character 0: .* \[0, 9\]"),
    (((0, 0), (9, 0), (0, 5)), dict(labels=[[[1, 2]]], boxes=[[[[1, 0, 3, 5]]]]), "image 0, region 0: 2 labels for 1 boxes"),
    (((0, 0), (9, 0), (0, 5)), dict(labels=[[None]], boxes=[[[[1, 0, 3, 5]]]]), "image 0, region 0: boxes without labels"),
    (("a", "b", "c"), {}, "image 0, region 0: expected three"),
])
def test_plan_rejects_oriented(reg, kw, match):
    from marconet_b200 import pipeline
    args = dict(regions=[[pipeline.OrientedRegion(*reg)]], labels=None, boxes=None, scale=4, feather=None)
    args.update(kw)
    shape = args.pop("shape", (8, 10))
    with pytest.raises(ValueError, match=match):
        pipeline.plan_regions([shape], **args)


def test_plan_rejects_names_the_image_and_region():
    from marconet_b200 import pipeline
    good = pipeline.OrientedRegion((1, 1), (9, 1), (1, 6))
    with pytest.raises(ValueError, match="image 1, region 2: the region is mirrored"):
        pipeline.plan_regions([(8, 10), (8, 10)], [[good], [good, (0, 0, 2, 2), pipeline.OrientedRegion((1, 6), (9, 6), (1, 1))]])
    with pytest.raises(ValueError, match="image 0, region 0: the map onto its .* exceeds OpenCV's 32-bit fixed-point"):
        pipeline.plan_regions([(4000, 32000)], [[pipeline.OrientedRegion((31990, 10), (31999, 10), (31990, 11))]], scale=1)


def _fields(header, name):
    body = re.search(r"typedef struct \{([^{}]*)\}\s*" + name + ";", header).group(1)
    body = re.sub(r"/\*.*?\*/", "", body, flags=re.S)
    names = []
    for decl in body.split(";"):
        parts = [re.sub(r"\[\d+\]$", "", p.strip()) for p in decl.strip().split(",") if p.strip()]
        names += [re.findall(r"[A-Za-z_0-9]+$", p)[0] for p in parts]
    return names


@pytest.mark.parametrize("c_name,py_name,size", [("mn_warp_image", "WarpImage", 96), ("mn_region_affine", "RegionAffine", 144)])
def test_oriented_structs_match_header(c_name, py_name, size):
    from marconet_b200 import _lib
    header = open(os.path.join(ROOT, "include", "marconet_b200.h")).read()
    cls = getattr(_lib, py_name)
    assert _fields(header, c_name) == [f[0] for f in cls._fields_]
    assert ctypes.sizeof(cls) == size
    assert re.search(r"#define MN_REGION_RECT 0\s+#define MN_REGION_AFFINE 1", header)
    assert (_lib.REGION_RECT, _lib.REGION_AFFINE) == (0, 1)
    if py_name == "RegionAffine":
        assert _lib.RegionAffine.r.offset == 0 and _lib.RegionAffine.n.offset == 96


def test_oriented_kernels_build_without_spills(tmp_path):
    import subprocess
    from marconet_b200 import build
    src = os.path.join(ROOT, "marconet_b200", "csrc", "image_ops.cu")
    r = subprocess.run([build.nvcc_path(), "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-DMN_BUILD", "-Xptxas", "-v",
                        "-cubin", src, "-o", str(tmp_path / "image_ops.cubin")], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-2000:]
    for kernel in ("warp_affine_batched_kernel", "composite_regions_affine_kernel"):
        props = re.search(kernel + r"[^\n]*\n[^\n]*Function properties for [^\n]*" + kernel + r"[^\n]*\n([^\n]*)", r.stderr)
        assert props, f"no ptxas report for {kernel}"
        assert "0 bytes spill stores, 0 bytes spill loads" in props.group(1), props.group(1)
