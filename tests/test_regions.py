"""Text regions in whole images on the CPU (DESIGN.md section 7b): the numpy twin of restore_regions' composition against live cv2
(IPP off) and hand-worked feather weights, the golden page, pipeline.plan_regions' validation and overlap lists, and the layout of
the two kernels' descriptor records."""
import ctypes
import os
import re

import numpy as np
import pytest

from oracle import regions as R

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "regions.npz")


@pytest.fixture
def cv2_no_ipp():
    cv2 = pytest.importorskip("cv2")
    was = cv2.ipp.useIPP()
    cv2.ipp.setUseIPP(False)
    yield cv2
    cv2.ipp.setUseIPP(was)


@pytest.mark.parametrize("s", range(1, 9))
def test_background_equals_cv2(cv2_no_ipp, s):
    rng = np.random.default_rng(s)
    for h, w in ((7, 13), (1, 9), (11, 1), (3, 40)):
        img = rng.integers(0, 256, (h, w, 3), dtype=np.uint8)
        ref = cv2_no_ipp.resize(img, (0, 0), fx=s, fy=s, interpolation=cv2_no_ipp.INTER_CUBIC)
        np.testing.assert_array_equal(R.background(img, s), ref)


@pytest.mark.parametrize("th,tw,dh,dw", [(128, 300, 64, 150), (128, 517, 48, 193), (128, 77, 12, 7), (128, 40, 4, 160),
                                         (128, 64, 1, 9), (128, 64, 9, 1), (128, 1, 40, 3), (1, 30, 4, 120), (128, 90, 512, 360)])
def test_region_resize_equals_cv2(cv2_no_ipp, th, tw, dh, dw):
    t = np.random.default_rng(th * tw + dh).integers(0, 256, (th, tw, 3), dtype=np.uint8)
    ref = cv2_no_ipp.resize(np.ascontiguousarray(t[..., ::-1]), (dw, dh), interpolation=cv2_no_ipp.INTER_CUBIC)
    np.testing.assert_array_equal(R.resized_region(t, dw, dh), ref)


def test_alpha_hand_worked():
    a = R.alpha((10, 10, 30, 30), (40, 40), 4)                       # every side counts
    assert a.dtype == np.float32
    np.testing.assert_array_equal(a[10, :5], np.float32([0.125, 0.375, 0.625, 0.875, 1]))
    np.testing.assert_array_equal(a[:5, 10], np.float32([0.125, 0.375, 0.625, 0.875, 1]))
    assert a[0, 0] == a[19, 19] == a[0, 19] == np.float32(0.125)
    assert a[10, 19] == np.float32(0.125) and a[10, 18] == np.float32(0.375)
    np.testing.assert_array_equal(R.alpha((10, 10, 30, 30), (40, 40), 0), 1)
    np.testing.assert_array_equal(R.alpha((0, 0, 40, 40), (40, 40), 8), 1)   # the whole page: no side counts
    b = R.alpha((0, 10, 20, 30), (40, 40), 4)                        # the left side lies on the border: no ramp there
    assert b[10, 0] == 1 and b[0, 0] == np.float32(0.125) and b[10, 19] == np.float32(0.125)
    c = R.alpha((10, 10, 20, 30), (40, 40), 3)                       # fl((float)d + 0.5) / F with one fp32 division
    assert c[10, 1] == np.float32(np.float32(1.5) / np.float32(3))
    assert R.alpha((5, 5, 9, 9), (20, 20), 1000)[1, 1] == np.float32(np.float32(1.5) / np.float32(1000))


def test_blend_rounds_each_operation():
    out = np.array([[[200, 10, 0]]], np.uint8)
    p = np.array([[[0, 255, 255]]], np.uint8)
    a = np.float32([[0.5]])
    np.testing.assert_array_equal(R.blend(out, p, a), [[[100, 132, 128]]])       # 132.5 and 127.5 round half to even
    np.testing.assert_array_equal(R.blend(out, p, np.float32([[1]])), p)
    np.testing.assert_array_equal(R.blend(out, p, np.float32([[0]])), out)


def test_hard_paste_and_chained_overlaps():
    rng = np.random.default_rng(5)
    img = rng.integers(0, 256, (24, 40, 3), dtype=np.uint8)
    ts = [rng.integers(0, 256, (128, 64 + 16 * k, 3), dtype=np.uint8) for k in range(3)]
    rects = [(2, 2, 20, 14), (10, 6, 30, 20), (16, 0, 40, 10)]       # a chain of three; the last touches the top and right
    s, f = 2, 5
    out = R.compose(img, rects[:1], ts[:1], s, 0)
    np.testing.assert_array_equal(out[4:28, 4:40], R.resized_region(ts[0], 36, 24))
    want = R.background(img, s)
    for (x0, y0, x1, y1), t in zip(rects, ts):
        r = (s * x0, s * y0, s * x1, s * y1)
        sl = want[r[1]:r[3], r[0]:r[2]]
        sl[...] = R.blend(sl, R.resized_region(t, r[2] - r[0], r[3] - r[1]), R.alpha(r, want.shape[:2], f))
    np.testing.assert_array_equal(R.compose(img, rects, ts, s, f), want)
    assert not np.array_equal(R.compose(img, rects[::-1], ts[::-1], s, f), want)     # the order matters
    np.testing.assert_array_equal(R.compose(img, rects, [ts[0], None, ts[2]], s, f),
                                  R.compose(img, rects[::2], ts[::2], s, f))           # a failed region keeps the background


def test_twin_reproduces_golden_page():
    """Every stored page pixel outside the wide region's rectangle (whose SR bytes are stored strided; no pixel outside it
    depends on them) is the twin's composition of the other regions' stored bytes."""
    g = np.load(GOLDEN)
    st, s = int(g["stride"]), int(g["scale"])
    rects = [tuple(r) for r in g["regions"].tolist()]
    whole = g["sr_strides"] == 1
    assert whole.sum() == 3
    srs = [g[f"sr{r}"] if whole[r] else None for r in range(len(rects))]
    page = R.compose(g["image"], rects, srs, s, int(g["feather"]))[::st, ::st]
    ys, xs = np.mgrid[0:page.shape[0], 0:page.shape[1]] * st
    outside = np.ones(page.shape[:2], bool)
    for (x0, y0, x1, y1), w in zip(rects, whole):
        inside = (xs >= s * x0) & (xs < s * x1) & (ys >= s * y0) & (ys < s * y1)
        if w:
            assert inside.sum() >= 40                     # each stored region is sampled
        else:
            outside &= ~inside
    np.testing.assert_array_equal(page[outside], g["page"][outside])


def _golden_args(g):
    rects = [tuple(r) for r in g["regions"].tolist()]
    labels = [[] for _ in rects]
    boxes = [[] for _ in rects]
    for lab, (x1, y1, x2, y2, r) in zip(g["labels"].tolist(), g["boxes"].tolist()):
        labels[r].append(lab)
        boxes[r].append([x1, y1, x2, y2])
    return rects, labels, boxes


def test_plan_regions_overlaps_and_crops():
    from marconet_b200 import pipeline
    g = np.load(GOLDEN)
    rects, labels, boxes = _golden_args(g)
    plan = pipeline.plan_regions([(160, 700), (30, 50)], [rects, [(0, 0, 50, 30), (10, 10, 20, 20), (30, 0, 50, 30)]],
                                 [labels, None], [boxes, None], scale=4, feather=8)
    assert [(p.image, p.region) for p in plan] == [(0, 0), (0, 1), (0, 2), (0, 3), (1, 0), (1, 1), (1, 2)]
    assert [p.overlaps for p in plan] == [[], [], [0, 1], [], [], [4], [4]]
    assert plan[2].out == (4 * 64, 4 * 28, 4 * 144, 4 * 68)
    x0, y0 = rects[1][:2]
    assert plan[1].boxes == [[b[0] - x0, b[1] - y0, b[2] - x0, b[3] - y0] for b in boxes[1]]
    assert plan[1].labels == labels[1]
    assert plan[4].labels is None and plan[4].boxes is None
    assert pipeline.region_chains(plan, list(range(7))) == [[0, 2], [1, 2], [0, 1, 2], [3], [4, 5, 6], [4, 5], [4, 6]]
    assert pipeline.region_chains(plan, [0, 2, 5, 6]) == [[0, 1], [0, 1], [2], [3]]       # left-out regions leave the chains
    touching = pipeline.plan_regions([(10, 10)], [[(0, 0, 5, 5), (5, 0, 10, 5)]])          # sharing an edge is no overlap
    assert touching[1].overlaps == []


@pytest.mark.parametrize("kw,match", [
    (dict(regions=[[(0, 0, 0, 5)]]), "image 0, region 0: rectangle"),
    (dict(regions=[[(0, 0, 5, 5), (3, 4, 11, 6)]]), "image 0, region 1: rectangle .* outside the 10x8 image"),
    (dict(regions=[[(0, 0, 5, 5)], [(0, -1, 3, 3)]]), "image 1, region 0: rectangle"),
    (dict(regions=[[(0, 0, 5.5, 5)]]), "image 0, region 0: expected an integer rectangle"),
    (dict(labels=[[[1, 2]]], boxes=[[[[0, 0, 2, 5]]]]), "image 0, region 0: 2 labels for 1 boxes"),
    (dict(labels=[[None]], boxes=[[[[0, 0, 2, 5]]]]), "image 0, region 0: boxes without labels"),
    (dict(regions=[[(2, 0, 6, 5)]], labels=[[[1]]], boxes=[[[[1, 0, 4, 5]]]]), r"image 0, region 0, character 0: .* columns \[2, 6\]"),
    (dict(regions=[[(2, 0, 6, 5)]], labels=[[[1]]], boxes=[[[[3, 0, 7, 5]]]]), r"image 0, region 0, character 0"),
    (dict(scale=0), "scale must be an integer in"),
    (dict(scale=9), "scale must be an integer in"),
    (dict(scale=2.0), "scale must be an integer in"),
    (dict(feather=-1), "feather must be an integer"),
    (dict(labels=[[None, None]]), r"image 0: labels \(one entry per region\): 2 entries for 1"),
    (dict(boxes=[None, None]), r"boxes \(one list per image\): 2 entries for 1"),
])
def test_plan_regions_rejects(kw, match):
    from marconet_b200 import pipeline
    args = dict(regions=[[(0, 0, 5, 5)]], labels=None, boxes=None, scale=4, feather=None)
    args.update(kw)
    shapes = [(8, 10)] * len(args["regions"])
    with pytest.raises(ValueError, match=match):
        pipeline.plan_regions(shapes, **args)


def _fields(header, name):
    body = re.search(r"typedef struct \{([^{}]*)\}\s*" + name + ";", header).group(1)
    body = re.sub(r"/\*.*?\*/", "", body, flags=re.S)
    names = []
    for decl in body.split(";"):
        parts = [p.strip() for p in decl.strip().split(",") if p.strip()]
        names += [re.findall(r"[A-Za-z_0-9]+$", p)[0] for p in parts]
    return names


@pytest.mark.parametrize("c_name,py_name,size", [("mn_resize_image", "ResizeImage", 64), ("mn_region", "Region", 80)])
def test_region_structs_match_header(c_name, py_name, size):
    from marconet_b200 import _lib
    header = open(os.path.join(ROOT, "include", "marconet_b200.h")).read()
    cls = getattr(_lib, py_name)
    assert _fields(header, c_name) == [f[0] for f in cls._fields_]
    assert ctypes.sizeof(cls) == size


def test_region_kernels_build_without_spills(tmp_path):
    import subprocess
    from marconet_b200 import build
    src = os.path.join(ROOT, "marconet_b200", "csrc", "image_ops.cu")
    r = subprocess.run([build.nvcc_path(), "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-DMN_BUILD", "-Xptxas", "-v",
                        "-cubin", src, "-o", str(tmp_path / "image_ops.cubin")], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-2000:]
    for kernel in ("resize_cubic_batched_kernel", "composite_regions_kernel"):
        props = re.search(kernel + r"[^\n]*\n[^\n]*Function properties for [^\n]*" + kernel + r"[^\n]*\n([^\n]*)", r.stderr)
        assert props, f"no ptxas report for {kernel}"
        assert "0 bytes spill stores, 0 bytes spill loads" in props.group(1), props.group(1)
