"""Curved text regions on the device (DESIGN.md section 7b, "Curved text regions"): the rectify and mixed composite kernels bit
for bit against the numpy twin, and pipeline.restore_regions with CurvedRegions against tests/golden/curved_regions.npz, the
rectangle call, restore_images on cv2-remapped crops and its launch counts."""
import math
import os

import numpy as np
import pytest
import torch

from oracle import curved_regions as R
from oracle import remap as RM

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "curved_regions.npz")
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


def _curved(rng, H, W):
    """A valid CurvedRegion of an H x W image: an arc of 20 to 300 degrees read either way, or a wavy line of 1 to 3 segments,
    turned by a random angle."""
    from marconet_b200 import pipeline
    while True:
        if rng.random() < 0.5:
            r = rng.uniform(8, 0.6 * max(H, W))
            h = rng.uniform(3, min(20, 0.6 * r))
            span = rng.uniform(20, 300) * rng.choice([-1, 1])
            inner_top = span > 0                          # counter-clockwise reading keeps the inner arc on top
            start = rng.uniform(-180, 180)
            reg = pipeline.CurvedRegion.from_arc(rng.uniform(0, W), rng.uniform(0, H), r - h if inner_top else r,
                                                 r if inner_top else r - h, start, start + span)
        else:
            k = int(rng.integers(1, 4))
            L, h = rng.uniform(6, 0.8 * W), rng.uniform(3, 20)
            xs = np.linspace(0, L, 3 * k + 1)
            ys = rng.uniform(-0.15, 0.15, 3 * k + 1) * L / k
            a = rng.uniform(-math.pi, math.pi)
            rot = np.array([[math.cos(a), -math.sin(a)], [math.sin(a), math.cos(a)]])
            top = np.stack([xs, ys], 1)
            bottom = top + [0, h]
            c = np.array([rng.uniform(0, W), rng.uniform(0, H)]) - (top.mean(0) + [0, h / 2]) @ rot.T
            reg = pipeline.CurvedRegion(tuple(map(tuple, top @ rot.T + c)), tuple(map(tuple, bottom @ rot.T + c)))
        try:
            pipeline.plan_regions([(H, W)], [[reg]], scale=1)
            return reg
        except ValueError:
            continue


@pytest.mark.parametrize("cn", [1, 3, 4])
def test_rectify_kernel_equals_twin(cn):
    from marconet_b200 import ops, pipeline
    rng = np.random.default_rng(cn)
    pages = [rng.integers(0, 256, (57, 91, cn), dtype=np.uint8), rng.integers(0, 256, (1, 1, cn), dtype=np.uint8),
             rng.integers(0, 256, (1, 23, cn), dtype=np.uint8), rng.integers(0, 256, (40, 300, cn), dtype=np.uint8)]
    cases = [(0, _curved(rng, 57, 91)) for _ in range(8)]
    cases += [(1, pipeline.CurvedRegion(((-2, -1), (0, -1.5), (1, 3), (4, 2)), ((-2, 3), (0, 2.5), (1, 7), (4, 6)))),
              (2, pipeline.CurvedRegion.from_arc(11, 0.5, 4, 9, 200, 340)),
              (3, pipeline.CurvedRegion.from_arc(150, 612, 600, 585, 150, 30))]          # a line wider than 1024 columns
    dsrc = [torch.from_numpy(s).to(DEV) for s in pages]
    wide = torch.zeros((57, 100, cn), dtype=torch.uint8, device=DEV)                    # a source read through a wider pitch
    wide[:, 4:95] = dsrc[0]
    items, refs = [], []
    for k, (si, reg) in enumerate(cases):
        m = pipeline.curved_maps(reg, 1)
        src = wide[:, 4:95] if k == 1 else dsrc[si]
        items.append((src, torch.empty((m.size[1], m.size[0], cn), dtype=torch.uint8, device=DEV), m.curve(1)))
        refs.append(RM.remap_cubic_u8(pages[si], *R.crop_map(m)))
    assert max(r.shape[1] for r in refs) > 1024
    n0 = ops.LAUNCHES
    ops.remap_curved(items)
    assert ops.LAUNCHES - n0 == 1
    for k, ((_, dst, _), ref) in enumerate(zip(items, refs)):
        np.testing.assert_array_equal(_np(dst), ref, err_msg=f"item {k}")


def _mixed_page(rng, H, W):
    """Rectangles, oriented regions, quads and curved regions of an H x W image, overlapping, some touching or leaving the page."""
    from marconet_b200.pipeline import CurvedRegion, OrientedRegion, QuadRegion
    regs = [(0, 0, W // 2, H // 3), (W // 4, H // 5, W - 3, H // 2)]
    for _ in range(2):
        cx, cy = rng.uniform(0, W), rng.uniform(0, H)
        regs.append(OrientedRegion.from_rotated(cx, cy, rng.uniform(4, W * 0.8), rng.uniform(3, 20), rng.uniform(-180, 180)))
    regs.append(QuadRegion((5, 5), (W // 2, 9), (W // 2 + 4, 19), (9, 15)))
    regs.append(QuadRegion((W - 30, 4), (W - 2, 8), (W - 3, 20), (W - 29, 24)))
    regs += [_curved(rng, H, W) for _ in range(4)]
    y0, y1 = H // 2, H // 2 + 6
    regs.append(CurvedRegion(((3, y0), (3 + W / 9, y0), (3 + 2 * W / 9, y0), (3 + W / 3, y0)),
                             ((3, y1), (3 + W / 9, y1), (3 + 2 * W / 9, y1), (3 + W / 3, y1))))      # straight
    regs.append((W - 9, H - 7, W, H))
    order = rng.permutation(len(regs))
    return [regs[i] for i in order]


def _maps(p, s, width):
    from marconet_b200 import pipeline
    if p.curved is not None:
        return pipeline.curved_maps(p.curved, s, width)
    if p.quad is not None:
        return pipeline.quad_maps(p.quad, s, width)
    return pipeline.oriented_maps(p.oriented, s, width) if p.oriented is not None else None


def _entry(m, s):
    from marconet_b200 import pipeline
    if m is None:
        return None
    return (m.curve(s) if isinstance(m, pipeline.CurvedMaps) else m.page_map, m.kx, m.ky)


@pytest.mark.parametrize("s", [1, 2, 4, 8])
@pytest.mark.parametrize("feather", [0, 3, 8])
def test_composite_curved_kernel_equals_twin(s, feather):
    from marconet_b200 import ops, pipeline
    rng = np.random.default_rng(10 * s + feather)
    shapes = [(40, 70), (23, 51)]
    imgs = [rng.integers(0, 256, (h, w, 3), dtype=np.uint8) for h, w in shapes]
    regs = [_mixed_page(rng, h, w) for h, w in shapes]
    plan = pipeline.plan_regions(shapes, regs, scale=s, feather=feather)
    ts = []
    for p in plan:
        warped = p.quad is not None or p.oriented is not None or p.curved is not None
        wd = _maps(p, s, None).t_width if warped else int(rng.integers(1, 300))
        ts.append(rng.integers(0, 256, (128, wd + (p.region % 3 == 1 and warped), 3), dtype=np.uint8))
    pages = [torch.from_numpy(R.background(im, s)).to(DEV) for im in imgs]
    ok = [k for k in range(len(plan)) if k % 7 != 5]    # some regions left out, as failed ones are
    items = []
    for k, c in zip(ok, pipeline.region_chains(plan, ok)):
        p, t = plan[k], torch.from_numpy(ts[k]).to(DEV)
        items.append((pages[p.image], t, p.out, c, _entry(_maps(p, s, t.shape[1]), s)))
    n0 = ops.LAUNCHES
    ops.composite_regions_curved(items, feather)
    assert ops.LAUNCHES - n0 == 1
    for i, im in enumerate(imgs):
        srs = [ts[k] if k in ok else None for k, p in enumerate(plan) if p.image == i]
        want = R.compose(im, regs[i], srs, s, feather)
        assert not np.array_equal(want, R.background(im, s))
        np.testing.assert_array_equal(_np(pages[i]), want, err_msg=f"image {i}")


def test_composite_curved_without_curves_equals_composite_quad():
    from marconet_b200 import ops, pipeline
    from marconet_b200.pipeline import OrientedRegion, QuadRegion
    rng = np.random.default_rng(3)
    shapes, s, feather = [(24, 40), (17, 61)], 3, 5
    regs = [[(0, 0, 40, 24), OrientedRegion.from_rotated(20, 12, 30, 8, 20), (10, 6, 30, 20),
             QuadRegion((5, 5), (30, 7), (31, 19), (6, 16))],
            [(1, 4, 59, 5), OrientedRegion.from_rotated(30, 9, 40, 10, -160), (20, 3, 61, 17), (0, 0, 9, 9)]]
    plan = pipeline.plan_regions(shapes, regs, scale=s, feather=feather)
    ts = [torch.from_numpy(rng.integers(0, 256, (128, int(rng.integers(1, 300)), 3), dtype=np.uint8)).to(DEV) for _ in plan]
    bg = [torch.from_numpy(rng.integers(0, 256, (s * h, s * w, 3), dtype=np.uint8)).to(DEV) for h, w in shapes]
    ok = list(range(len(plan)))
    outs = []
    for fn in (ops.composite_regions_quad, ops.composite_regions_curved):
        pages = [b.clone() for b in bg]
        items = []
        for k, c in zip(ok, pipeline.region_chains(plan, ok)):
            items.append((pages[plan[k].image], ts[k], plan[k].out, c, _entry(_maps(plan[k], s, ts[k].shape[1]), s)))
        fn(items, feather)
        outs.append([_np(p) for p in pages])
    for a, b in zip(*outs):
        np.testing.assert_array_equal(a, b)


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


@pytest.mark.parametrize("to_host", [False, True])
def test_restore_regions_curved_golden(gpu_models, to_host):
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
        if isinstance(regs[r], pipeline.CurvedRegion):
            assert e["size"] == pipeline.curved_maps(regs[r], 1).size and "matrix" not in e
        srs.append(t)
    np.testing.assert_array_equal(page, R.compose(g["image"], regs, srs, s, f))
    d = np.abs(page[::int(g["stride"]), ::int(g["stride"])].astype(np.int16) - g["page"].astype(np.int16)).max()
    assert d <= 2, d                                    # a one-level SR difference can reach two through the cubic's lobes
    assert len(out[0]["regions"][0]["segments"]) == 2                      # the seal's arc is wider than the canvas


def test_reduction_to_the_rectangle_call(gpu_models):
    """A straight CurvedRegion over an interior rectangle at h = 32, s = 4 gives the rectangle call's page and sr_u8 bit for
    bit."""
    from marconet_b200 import pipeline
    g, _, _, _ = _golden()
    img = np.ascontiguousarray(g["image"][:80, :200])
    m = _models(gpu_models)
    x0, y0, x1, y1 = 20, 30, 140, 62
    w = x1 - x0
    labels = [5, 17, 900, 31]
    boxes = [[x0 + 4 + 28 * k, y0 + 2, x0 + 28 + 28 * k, y1 - 2] for k in range(4)]
    rel = [[b[0] - x0, b[1] - y0, b[2] - x0, b[3] - y0] for b in boxes]
    reg = pipeline.CurvedRegion(((x0, y0), (x0 + w / 3, y0), (x0 + 2 * w / 3, y0), (x1, y0)),
                                ((x0, y1), (x0 + w / 3, y1), (x0 + 2 * w / 3, y1), (x1, y1)))
    a = pipeline.restore_regions(*m, [img], [[(x0, y0, x1, y1)]], [[labels]], [[boxes]], scale=4, feather=8, to_host=True)[0]
    b = pipeline.restore_regions(*m, [img], [[reg]], [[labels]], [[rel]], scale=4, feather=8, to_host=True)[0]
    np.testing.assert_array_equal(a["image"], b["image"])
    np.testing.assert_array_equal(a["regions"][0]["sr_u8"], b["regions"][0]["sr_u8"])
    assert b["regions"][0]["size"] == (w, y1 - y0) and b["regions"][0]["boxes"] == rel


def test_one_curved_region_is_restore_images_on_the_cv2_crop(gpu_models, cv2_no_ipp):
    from marconet_b200 import pipeline
    g, regs, labels, boxes = _golden()
    m = _models(gpu_models)
    for r in (1, 5):
        mx, my = R.crop_map(pipeline.curved_maps(regs[r], 1))
        crop = cv2_no_ipp.remap(g["image"], mx.astype(np.float32), my.astype(np.float32), cv2_no_ipp.INTER_CUBIC,
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
    labels[1], boxes[1] = [], []                        # no characters: restore_images rejects the bottom arc
    with pytest.raises(ValueError, match="no character labels"):
        pipeline.restore_regions(*m, [g["image"]], [regs], [labels], [boxes])
    out = pipeline.restore_regions(*m, [g["image"]], [regs], [labels], [boxes], scale=2, feather=3, skip_invalid=True,
                                   to_host=True)[0]
    assert "error" in out["regions"][1] and "size" not in out["regions"][1]
    srs = [None if "error" in e else e["sr_u8"] for e in out["regions"]]
    want = R.compose(g["image"], regs, srs, 2, 3)
    np.testing.assert_array_equal(out["image"], want)
    plan = pipeline.plan_regions([g["image"].shape[:2]], [regs], scale=2)
    x0, y0, x1, y1 = plan[1].out
    bg = R.background(g["image"], 2)
    others = np.zeros(bg.shape[:2], bool)
    for k, p in enumerate(plan):
        if k != 1:
            others[p.out[1]:p.out[3], p.out[0]:p.out[2]] = True
    free = ~others[y0:y1, x0:x1]
    assert free.mean() > 0.5
    np.testing.assert_array_equal(want[y0:y1, x0:x1][free], bg[y0:y1, x0:x1][free])


def test_curved_launches_and_one_sync(gpu_models, monkeypatch):
    """A call adds one rectify launch per warped region kind, the background and one composite launch to restore_images' own;
    with to_host one synchronisation more.  A call without curved regions issues exactly the launches it issued before."""
    from marconet_b200 import ops, pipeline
    from marconet_b200.pipeline import OrientedRegion, QuadRegion
    g, regs, labels, boxes = _golden()
    m = _models(gpu_models)
    calls = []
    for name in ("warp_affine", "warp_perspective", "remap_curved", "resize_cubic", "composite_regions",
                 "composite_regions_affine", "composite_regions_quad", "composite_regions_curved"):
        real = getattr(ops, name)
        monkeypatch.setattr(ops, name, lambda *a, _n=name, _f=real: (calls.append(_n), _f(*a))[1])
    curved = [r for r in regs if isinstance(r, pipeline.CurvedRegion)]
    clab = [l for r, l in zip(regs, labels) if isinstance(r, pipeline.CurvedRegion)]
    cbox = [b for r, b in zip(regs, boxes) if isinstance(r, pipeline.CurvedRegion)]
    quad = QuadRegion((150, 140), (190, 138), (191, 162), (149, 160))
    crops = [torch.from_numpy(R.rectify(g["image"], r)).to(DEV) for r in curved]
    pipeline.restore_regions(*m, [g["image"]], [regs + [quad]], [labels + [[3]]], [boxes + [[[2, 1, 18, 15]]]])    # warm up
    pipeline.restore_regions(*m, [g["image"]], [curved], [clab], [cbox])
    pipeline.restore_images(*m, crops, clab, cbox)
    n0 = ops.LAUNCHES
    pipeline.restore_images(*m, crops, clab, cbox)
    n_images = ops.LAUNCHES - n0
    syncs = []
    real_sync = torch.cuda.Stream.synchronize
    monkeypatch.setattr(torch.cuda.Stream, "synchronize", lambda self: (syncs.append(1), real_sync(self))[1])
    calls.clear()
    n0 = ops.LAUNCHES
    pipeline.restore_regions(*m, [g["image"]], [curved], [clab], [cbox])
    n_regions, s_dev = ops.LAUNCHES - n0, len(syncs)
    assert calls == ["remap_curved", "resize_cubic", "composite_regions_curved"]
    assert n_regions == n_images + 3
    pipeline.restore_regions(*m, [g["image"]], [curved], [clab], [cbox], to_host=True)
    assert len(syncs) - s_dev == s_dev + 1
    calls.clear()
    pipeline.restore_regions(*m, [g["image"]], [regs + [quad]], [labels + [[3]]], [boxes + [[[2, 1, 18, 15]]]])
    assert calls == ["warp_affine", "warp_perspective", "remap_curved", "resize_cubic", "composite_regions_curved"]
    calls.clear()
    oriented = OrientedRegion.from_rotated(200, 100, 40, 16, 12)
    pipeline.restore_regions(*m, [g["image"]], [[oriented, quad]], [[[3, 4], [3]]],
                             [[[[2, 1, 18, 15], [20, 1, 38, 15]], [[2, 1, 18, 15]]]])
    assert calls == ["warp_affine", "warp_perspective", "resize_cubic", "composite_regions_quad"]
    calls.clear()
    pipeline.restore_regions(*m, [g["image"]], [[(0, 0, 60, 30)]], [[[7]]], [[[[2, 0, 50, 30]]]])
    assert calls == ["resize_cubic", "composite_regions"]
