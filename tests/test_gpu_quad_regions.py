"""Perspective text regions on the device (DESIGN.md section 7b, "Perspective text regions"): the rectify and mixed composite
kernels bit for bit against the numpy twin, and pipeline.restore_regions with QuadRegions against tests/golden/quad_regions.npz,
the rectangle call, restore_images on cv2-rectified crops and its launch counts."""
import math
import os

import numpy as np
import pytest
import torch

from oracle import quad_regions as R
from oracle import warp_perspective as P

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "quad_regions.npz")
DEV = torch.device("cuda:0")


@pytest.fixture
def cv2_no_ipp():
    import cv2
    was = cv2.ipp.useIPP()
    cv2.ipp.setUseIPP(False)
    yield cv2
    cv2.ipp.setUseIPP(was)


def _models(gpu_models):
    return gpu_models["encoder"], gpu_models["tspgan"], gpu_models["sr"]


def _np(t):
    return t.cpu().numpy() if isinstance(t, torch.Tensor) else t


def _quad(rng, H, W, max_len=None):
    """A valid QuadRegion of an H x W image: a rotated trapezoid whose far side is up to 3 times shorter, or its mirror."""
    from marconet_b200 import pipeline
    while True:
        L, w = rng.uniform(3, 24), rng.uniform(4, max_len or W * 0.8)
        r = L / rng.uniform(1, 3)
        pts = np.array([[0, -L / 2], [w, -r / 2], [w, r / 2], [0, L / 2]])
        if rng.random() < 0.5:
            pts = np.array([[0, -r / 2], [w, -L / 2], [w, L / 2], [0, r / 2]])
        a = rng.uniform(-math.pi, math.pi)
        rot = np.array([[math.cos(a), -math.sin(a)], [math.sin(a), math.cos(a)]])
        pts = pts - pts.mean(0)
        q = pipeline.QuadRegion(*map(tuple, pts @ rot.T + [rng.uniform(0, W), rng.uniform(0, H)]))
        try:
            pipeline.plan_regions([(H, W)], [[q]], scale=1)
            return q
        except ValueError:
            continue


@pytest.mark.parametrize("cn", [1, 3, 4])
def test_rectify_kernel_equals_twin(cn):
    from marconet_b200 import ops, pipeline
    rng = np.random.default_rng(cn)
    pages = [rng.integers(0, 256, (57, 91, cn), dtype=np.uint8), rng.integers(0, 256, (1, 1, cn), dtype=np.uint8),
             rng.integers(0, 256, (1, 23, cn), dtype=np.uint8), rng.integers(0, 256, (40, 300, cn), dtype=np.uint8)]
    cases = []
    for k in range(8):                                   # the rectified crops of random quads
        q = _quad(rng, 57, 91)
        m = pipeline.quad_maps(q, 1)
        cases.append((0, m.matrix, m.size))
    persp = [[0.41, 0.13, -3.0], [0.2, 0.7, -0.4], [0.003, -0.002, 1.1]]
    cases += [(1, [[0.3, 0.1, -2.0], [0.2, 0.7, 1.0], [0.01, 0, 1]], (9, 7)), (2, persp, (40, 7)),
              (0, [[0.9, 0.3, -60.0], [-0.3, 0.9, 45.0], [0.002, 0.001, 0.9]], (90, 70)),         # mostly outside the source
              (0, [[1 / 32, 0, 1.3], [0, 1 / 32, 2.1], [0, 0, 1]], (96, 96)),                     # every fraction pair
              (3, [[0.25, 0.02, 3.0], [0.001, 0.9, 1.0], [2e-4, 0.0, 1.0]], (1500, 30))]          # wider than 1024 columns
    dsrc = [torch.from_numpy(s).to(DEV) for s in pages]
    wide = torch.zeros((57, 100, cn), dtype=torch.uint8, device=DEV)                    # a source read through a wider pitch
    wide[:, 4:95] = dsrc[0]
    items, refs = [], []
    for k, (si, m, (dw, dh)) in enumerate(cases):
        src = wide[:, 4:95] if k == 1 else dsrc[si]
        items.append((src, torch.empty((dh, dw, cn), dtype=torch.uint8, device=DEV), m))
        refs.append(P.warp_perspective_cubic_u8(pages[si], m, (dw, dh)))
    n0 = ops.LAUNCHES
    ops.warp_perspective(items)
    assert ops.LAUNCHES - n0 == 1
    for k, ((_, dst, _), ref) in enumerate(zip(items, refs)):
        np.testing.assert_array_equal(_np(dst), ref, err_msg=f"item {k}")


def _mixed_page(rng, H, W):
    """Rectangles, oriented regions and quads of an H x W image, overlapping, some touching or leaving the page."""
    from marconet_b200.pipeline import OrientedRegion, QuadRegion
    regs = [(0, 0, W // 2, H // 3), (W // 4, H // 5, W - 3, H // 2)]
    for _ in range(3):
        cx, cy = rng.uniform(0, W), rng.uniform(0, H)
        regs.append(OrientedRegion.from_rotated(cx, cy, rng.uniform(4, W * 0.8), rng.uniform(3, 20), rng.uniform(-180, 180)))
    regs += [_quad(rng, H, W) for _ in range(4)]
    regs.append(QuadRegion((3, 4), (3 + W // 3, 4), (3 + W // 3, 12), (3, 12)))     # axis-aligned
    regs.append(QuadRegion((5, 5), (W // 2, 9), (W // 2 + 4, 19), (9, 15)))          # exactly a parallelogram
    regs.append((W - 9, H - 7, W, H))
    order = rng.permutation(len(regs))
    return [regs[i] for i in order]


def _maps(p, s, width):
    from marconet_b200 import pipeline
    if p.quad is not None:
        return pipeline.quad_maps(p.quad, s, width)
    return pipeline.oriented_maps(p.oriented, s, width) if p.oriented is not None else None


@pytest.mark.parametrize("s", [1, 2, 4, 8])
@pytest.mark.parametrize("feather", [0, 3, 8])
def test_composite_quad_kernel_equals_twin(s, feather):
    from marconet_b200 import ops, pipeline
    rng = np.random.default_rng(10 * s + feather)
    shapes = [(40, 70), (23, 51)]
    imgs = [rng.integers(0, 256, (h, w, 3), dtype=np.uint8) for h, w in shapes]
    regs = [_mixed_page(rng, h, w) for h, w in shapes]
    plan = pipeline.plan_regions(shapes, regs, scale=s, feather=feather)
    ts = []
    for p in plan:
        warped = p.quad is not None or p.oriented is not None
        wd = _maps(p, s, None).t_width if warped else int(rng.integers(1, 300))
        ts.append(rng.integers(0, 256, (128, wd + (p.region % 3 == 1 and warped), 3), dtype=np.uint8))
    pages = [torch.from_numpy(R.background(im, s)).to(DEV) for im in imgs]
    ok = [k for k in range(len(plan)) if k % 7 != 5]    # some regions left out, as failed ones are
    items = []
    for k, c in zip(ok, pipeline.region_chains(plan, ok)):
        p, t = plan[k], torch.from_numpy(ts[k]).to(DEV)
        m = _maps(p, s, t.shape[1])
        items.append((pages[p.image], t, p.out, c, m and (m.page_map, m.kx, m.ky)))
    n0 = ops.LAUNCHES
    ops.composite_regions_quad(items, feather)
    assert ops.LAUNCHES - n0 == 1
    for i, im in enumerate(imgs):
        srs = [ts[k] if k in ok else None for k, p in enumerate(plan) if p.image == i]
        np.testing.assert_array_equal(_np(pages[i]), R.compose(im, regs[i], srs, s, feather), err_msg=f"image {i}")


def test_composite_quad_without_quads_equals_composite_affine():
    from marconet_b200 import ops, pipeline
    from marconet_b200.pipeline import OrientedRegion
    rng = np.random.default_rng(3)
    shapes, s, feather = [(24, 40), (17, 61)], 3, 5
    regs = [[(0, 0, 40, 24), OrientedRegion.from_rotated(20, 12, 30, 8, 20), (10, 6, 30, 20), (16, 0, 40, 10)],
            [(1, 4, 59, 5), OrientedRegion.from_rotated(30, 9, 40, 10, -160), (20, 3, 61, 17), (0, 0, 9, 9)]]
    plan = pipeline.plan_regions(shapes, regs, scale=s, feather=feather)
    ts = [torch.from_numpy(rng.integers(0, 256, (128, int(rng.integers(1, 300)), 3), dtype=np.uint8)).to(DEV) for _ in plan]
    bg = [torch.from_numpy(rng.integers(0, 256, (s * h, s * w, 3), dtype=np.uint8)).to(DEV) for h, w in shapes]
    ok = list(range(len(plan)))
    outs = []
    for fn in (ops.composite_regions_affine, ops.composite_regions_quad):
        pages = [b.clone() for b in bg]
        items = []
        for k, c in zip(ok, pipeline.region_chains(plan, ok)):
            m = _maps(plan[k], s, ts[k].shape[1])
            items.append((pages[plan[k].image], ts[k], plan[k].out, c, m and (m.page_map, m.kx, m.ky)))
        fn(items, feather)
        outs.append([_np(p) for p in pages])
    for a, b in zip(*outs):
        np.testing.assert_array_equal(a, b)


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


@pytest.mark.parametrize("to_host", [False, True])
def test_restore_regions_quad_golden(gpu_models, to_host):
    from marconet_b200 import pipeline
    g, regs, labels, boxes = _golden()
    s, f = int(g["scale"]), int(g["feather"])
    out = pipeline.restore_regions(*_models(gpu_models), [g["image"]], [regs], [labels], [boxes], scale=s, feather=f,
                                   to_host=to_host)
    assert len(out) == 1 and len(out[0]["regions"]) == len(regs)
    page = _np(out[0]["image"])
    srs = []
    for r, e in enumerate(out[0]["regions"]):
        t = _np(e["sr_u8"])
        assert isinstance(e["sr_u8"], np.ndarray) == to_host
        k = int(g["sr_strides"][r])
        assert t.shape == (128, int(g["sr_widths"][r]), 3), r
        d = np.abs(t[::k, ::k].astype(np.int16) - g[f"sr{r}"].astype(np.int16)).max()
        assert d <= 1, (r, d)
        assert e["labels"] == labels[r] and e["boxes"] == boxes[r]
        if isinstance(regs[r], pipeline.QuadRegion):
            m = pipeline.quad_maps(regs[r], 1)
            assert e["size"] == m.size and np.array_equal(e["matrix"], m.matrix)
        else:
            assert "matrix" not in e
        srs.append(t)
    np.testing.assert_array_equal(page, R.compose(g["image"], regs, srs, s, f))
    d = np.abs(page[::int(g["stride"]), ::int(g["stride"])].astype(np.int16) - g["page"].astype(np.int16)).max()
    assert d <= 2, d                                    # a one-level SR difference can reach two through the cubic's lobes
    assert len(out[0]["regions"][0]["segments"]) == 2                      # the region wider than the canvas is cut


def test_reduction_to_the_rectangle_call(gpu_models):
    """An interior rectangle given as a QuadRegion at h = 32, s = 4 gives the rectangle call's page and sr_u8 bit for bit."""
    from marconet_b200 import pipeline
    g, _, _, _ = _golden()
    img = np.ascontiguousarray(g["image"][:80, :200])
    m = _models(gpu_models)
    x0, y0, x1, y1 = 20, 30, 140, 62
    labels = [5, 17, 900, 31]
    boxes = [[x0 + 4 + 28 * k, y0 + 2, x0 + 28 + 28 * k, y1 - 2] for k in range(4)]
    rel = [[b[0] - x0, b[1] - y0, b[2] - x0, b[3] - y0] for b in boxes]
    a = pipeline.restore_regions(*m, [img], [[(x0, y0, x1, y1)]], [[labels]], [[boxes]], scale=4, feather=8, to_host=True)[0]
    b = pipeline.restore_regions(*m, [img], [[pipeline.QuadRegion((x0, y0), (x1, y0), (x1, y1), (x0, y1))]], [[labels]], [[rel]],
                                 scale=4, feather=8, to_host=True)[0]
    np.testing.assert_array_equal(a["image"], b["image"])
    np.testing.assert_array_equal(a["regions"][0]["sr_u8"], b["regions"][0]["sr_u8"])
    assert b["regions"][0]["matrix"].tolist() == [[1, 0, x0], [0, 1, y0], [0, 0, 1]] and b["regions"][0]["boxes"] == rel


def test_one_quad_is_restore_images_on_the_cv2_crop(gpu_models, cv2_no_ipp):
    from marconet_b200 import pipeline
    g, regs, labels, boxes = _golden()
    m = _models(gpu_models)
    for r in (1, 3):
        qm = pipeline.quad_maps(regs[r], 1)
        crop = cv2_no_ipp.warpPerspective(g["image"], qm.matrix, qm.size, flags=cv2_no_ipp.INTER_CUBIC | cv2_no_ipp.WARP_INVERSE_MAP,
                                          borderMode=cv2_no_ipp.BORDER_REPLICATE)
        ref = pipeline.restore_images(*m, [crop], [labels[r]], [boxes[r]], to_host=True)[0]
        out = pipeline.restore_regions(*m, [g["image"]], [[regs[r]]], [[labels[r]]], [[boxes[r]]], to_host=True)[0]["regions"][0]
        np.testing.assert_array_equal(out["sr_u8"], ref["sr_u8"])
        pred_ref = pipeline.restore_images(*m, [crop], skip_invalid=True, to_host=True)[0]
        pred = pipeline.restore_regions(*m, [g["image"]], [[regs[r]]], skip_invalid=True, to_host=True)[0]["regions"][0]
        assert ("error" in pred) == ("error" in pred_ref)
        if "error" not in pred:
            assert pred["labels"] == pred_ref["labels"] and pred["boxes"] == pred_ref["boxes"]
            np.testing.assert_array_equal(pred["sr_u8"], pred_ref["sr_u8"])


def test_skip_invalid_keeps_background_in_the_footprint(gpu_models):
    from marconet_b200 import pipeline
    g, regs, labels, boxes = _golden()
    m = _models(gpu_models)
    labels, boxes = list(labels), list(boxes)
    labels[5], boxes[5] = [], []                        # no characters: restore_images rejects the region
    with pytest.raises(ValueError, match="no character labels"):
        pipeline.restore_regions(*m, [g["image"]], [regs], [labels], [boxes])
    out = pipeline.restore_regions(*m, [g["image"]], [regs], [labels], [boxes], scale=2, feather=3, skip_invalid=True,
                                   to_host=True)[0]
    assert "error" in out["regions"][5] and "matrix" not in out["regions"][5]
    srs = [None if "error" in e else e["sr_u8"] for e in out["regions"]]
    want = R.compose(g["image"], regs, srs, 2, 3)
    np.testing.assert_array_equal(out["image"], want)
    plan = pipeline.plan_regions([g["image"].shape[:2]], [regs], scale=2)
    x0, y0, x1, y1 = plan[5].out
    assert not any(5 in p.overlaps for p in plan) and plan[5].overlaps == []
    bg = R.background(g["image"], 2)
    np.testing.assert_array_equal(want[y0:y1, x0:x1], bg[y0:y1, x0:x1])   # region 5's box meets no other region


def test_quad_launches_and_one_sync(gpu_models, monkeypatch):
    """A call adds one rectify launch per warped region kind, the background and one composite launch to restore_images' own;
    with to_host one synchronisation more.  A call without quads issues exactly the launches it issued before."""
    from marconet_b200 import ops, pipeline
    from marconet_b200.pipeline import OrientedRegion
    g, regs, labels, boxes = _golden()
    m = _models(gpu_models)
    calls = []
    for name in ("warp_affine", "warp_perspective", "resize_cubic", "composite_regions", "composite_regions_affine",
                 "composite_regions_quad"):
        real = getattr(ops, name)
        monkeypatch.setattr(ops, name, lambda *a, _n=name, _f=real: (calls.append(_n), _f(*a))[1])
    oriented = OrientedRegion.from_rotated(200, 100, 40, 16, 12)
    both = regs + [oriented]
    lab2, box2 = labels + [[3, 4]], boxes + [[[2, 1, 18, 15], [20, 1, 38, 15]]]
    crops = [torch.from_numpy(R.rectify(g["image"], r) if isinstance(r, pipeline.QuadRegion) else
                              np.ascontiguousarray(g["image"][r[1]:r[3], r[0]:r[2]])).to(DEV) for r in regs]
    pipeline.restore_regions(*m, [g["image"]], [both], [lab2], [box2])           # warm up
    rel = [bx if isinstance(r, pipeline.QuadRegion) else [[b[0] - r[0], b[1] - r[1], b[2] - r[0], b[3] - r[1]] for b in bx]
           for r, bx in zip(regs, boxes)]
    n0 = ops.LAUNCHES
    pipeline.restore_images(*m, crops, labels, rel)
    n_images = ops.LAUNCHES - n0
    syncs = []
    real_sync = torch.cuda.Stream.synchronize
    monkeypatch.setattr(torch.cuda.Stream, "synchronize", lambda self: (syncs.append(1), real_sync(self))[1])
    calls.clear()
    n0 = ops.LAUNCHES
    pipeline.restore_regions(*m, [g["image"]], [regs], [labels], [boxes])
    n_regions, s_dev = ops.LAUNCHES - n0, len(syncs)
    assert calls == ["warp_perspective", "resize_cubic", "composite_regions_quad"]
    assert n_regions == n_images + 3
    pipeline.restore_regions(*m, [g["image"]], [regs], [labels], [boxes], to_host=True)
    assert len(syncs) - s_dev == s_dev + 1
    calls.clear()
    pipeline.restore_regions(*m, [g["image"]], [both], [lab2], [box2])
    assert calls == ["warp_affine", "warp_perspective", "resize_cubic", "composite_regions_quad"]
    calls.clear()
    pipeline.restore_regions(*m, [g["image"]], [[oriented, (0, 0, 60, 30)]], [[[3, 4], [7]]],
                             [[[[2, 1, 18, 15], [20, 1, 38, 15]], [[2, 0, 50, 30]]]])
    assert calls == ["warp_affine", "resize_cubic", "composite_regions_affine"]
    calls.clear()
    pipeline.restore_regions(*m, [g["image"]], [[(0, 0, 60, 30)]], [[[7]]], [[[[2, 0, 50, 30]]]])
    assert calls == ["resize_cubic", "composite_regions"]
