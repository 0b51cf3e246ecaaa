"""Vertical text columns on the device (DESIGN.md section 7b, "Vertical text columns"): the layout and inverse-layout gathers bit
for bit against the numpy twin, and pipeline.restore_regions with VerticalRegions against tests/golden/vertical_regions.npz, the
one-cell reduction, the predicted path, skip_invalid, its launch counts and a call that mixes every region kind."""
import os

import numpy as np
import pytest
import torch

from oracle import vertical_regions as V

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "vertical_regions.npz")
DEV = torch.device("cuda:0")


def _models(gpu_models):
    return gpu_models["encoder"], gpu_models["tspgan"], gpu_models["sr"]


def _np(t):
    return t.cpu().numpy() if isinstance(t, torch.Tensor) else t


def _random_plan(rng, w, h):
    from marconet_b200.pipeline import vertical_plan
    mode = rng.integers(0, 3)
    if mode == 0:
        y, boxes = 0, []
        while True:
            ch = int(rng.integers(1, 2 * w + 2))
            if y + ch > h:
                break
            boxes.append([0, y, w, y + ch])
            y += ch + int(rng.integers(0, 4))
        if len(boxes) > 1:
            return vertical_plan(w, h, boxes=boxes)
    return vertical_plan(w, h, cells=int(rng.integers(1, min(h, 30) + 1)) if mode == 1 else None)


def test_gathers_equal_twin():
    """Random cell plans (boxes, n cells, the default), C read through a page's pitch, T through a wider buffer's pitch, a T
    narrower than R(n w_r): one launch each, every byte the twin's."""
    from marconet_b200 import ops, pipeline
    rng = np.random.default_rng(0)
    page = torch.from_numpy(rng.integers(0, 256, (400, 300, 3), dtype=np.uint8)).to(DEV)
    cols, plans = [], []
    for k in range(24):
        w, h = int(rng.integers(1, 40)), int(rng.integers(1, 390))
        if k == 0:
            w, h = 1, 1
        x0, y0 = int(rng.integers(0, 300 - w)), int(rng.integers(0, 400 - h))
        cols.append(page[y0:y0 + h, x0:x0 + w])
        plans.append(_random_plan(rng, w, h))
    lines = [torch.empty((vp.line_height, len(vp.heights) * vp.size[0], 3), dtype=torch.uint8, device=DEV) for vp in plans]
    n0 = ops.LAUNCHES
    ops.vertical_layout([(c, line, pipeline.layout_cells(vp)) for c, line, vp in zip(cols, lines, plans)])
    assert ops.LAUNCHES - n0 == 1
    for k, (c, line, vp) in enumerate(zip(cols, lines, plans)):
        np.testing.assert_array_equal(_np(line), V.layout(_np(c), vp.cells), err_msg=f"column {k}")
    ts, outs = [], []
    for vp in plans:
        wt = pipeline.vertical_r(len(vp.heights) * vp.size[0], vp.line_height)
        wt = max(1, wt - int(rng.integers(0, 3)))
        buf = torch.from_numpy(rng.integers(0, 256, (128, wt + 5, 3), dtype=np.uint8)).to(DEV)
        ts.append(buf[:, 2:2 + wt])
        outs.append(torch.empty((vp.t_size[1], vp.t_size[0], 3), dtype=torch.uint8, device=DEV))
    n0 = ops.LAUNCHES
    ops.vertical_unlayout([(t, o, pipeline.unlayout_cells(vp, t.shape[1])) for t, o, vp in zip(ts, outs, plans)])
    assert ops.LAUNCHES - n0 == 1
    for k, (t, o, vp) in enumerate(zip(ts, outs, plans)):
        np.testing.assert_array_equal(_np(o), V.unlayout(_np(t), vp.cells, vp.size[0]), err_msg=f"column {k}")


def test_gathers_reject_tables_that_read_outside():
    from marconet_b200 import ops
    c = torch.zeros((10, 4, 3), dtype=torch.uint8, device=DEV)
    with pytest.raises(ValueError, match="column 0: its cell table reads outside the 10x4 source"):
        ops.vertical_layout([(c, torch.empty((6, 8, 3), dtype=torch.uint8, device=DEV), [(0, 0, 5), (5, 0, 6)])])
    t = torch.zeros((128, 20, 3), dtype=torch.uint8, device=DEV)
    with pytest.raises(ValueError, match="column 0: its cell table reads outside the 128x20 source"):
        ops.vertical_unlayout([(t, torch.empty((10, 4, 3), dtype=torch.uint8, device=DEV), [(0, 0, 128, 0, 21)])])


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


@pytest.mark.parametrize("to_host", [False, True])
def test_restore_regions_vertical_golden(gpu_models, to_host):
    from marconet_b200 import pipeline
    g, regs, labels, boxes = _golden()
    s, f = int(g["scale"]), int(g["feather"])
    out = pipeline.restore_regions(*_models(gpu_models), [g["image"]], [regs], [labels], [boxes], scale=s, feather=f,
                                   to_host=to_host)
    assert len(out) == 1 and len(out[0]["regions"]) == len(regs)
    plan = pipeline.plan_regions([g["image"].shape[:2]], [regs], [labels], [boxes], scale=s, feather=f)
    page = _np(out[0]["image"])
    srs = []
    for r, (e, p) in enumerate(zip(out[0]["regions"], plan)):
        assert isinstance(e["sr_u8"], np.ndarray) == to_host
        t = _np(e.get("line_u8", e["sr_u8"]))
        k = int(g["sr_strides"][r])
        assert t.shape == (128, int(g["sr_widths"][r]), 3), r
        d = np.abs(t[::k, ::k].astype(np.int16) - g[f"sr{r}"].astype(np.int16)).max()
        assert d <= 1, (r, d)
        assert e["labels"] == labels[r] and e["boxes"] == boxes[r]
        if p.vertical is not None:
            tc = _np(e["sr_u8"])
            assert tc.shape == (p.vertical.t_size[1], p.vertical.t_size[0], 3) and e["cells"] == p.vertical.cells
            np.testing.assert_array_equal(tc, V.unlayout(t, p.vertical.cells, p.vertical.size[0]))
            assert isinstance(e["line_u8"], np.ndarray) == to_host
        else:
            assert "line_u8" not in e and "cells" not in e
        assert ("matrix" in e) == (p.oriented is not None or p.quad is not None)
        srs.append(_np(e["sr_u8"]))
    np.testing.assert_array_equal(page, V.compose(g["image"], regs, srs, s, f))
    d = np.abs(page[::int(g["stride"]), ::int(g["stride"])].astype(np.int16) - g["page"].astype(np.int16)).max()
    assert d <= 2, d                                    # a one-level SR difference can reach two through the cubic's lobes
    assert len(out[0]["regions"][1]["segments"]) == 2                      # the long column's line is wider than the canvas


def _shapes(g):
    """A horizontal rectangle line, an oriented one and a quad of the golden page."""
    from marconet_b200.pipeline import OrientedRegion, QuadRegion
    return [(20, 280, 100, 300), OrientedRegion.from_rotated(64, 318, 90, 18, 3),
            QuadRegion((14, 334), (112, 330), (113, 352), (15, 354))]


def test_one_cell_reduces_to_the_shape(gpu_models):
    """VerticalRegion(shape, cells=1) composes exactly the page and bytes ``shape`` composes alone, for every shape kind, with
    predicted labels and with given labels paired with predicted boxes."""
    from marconet_b200 import pipeline
    g, _, _, _ = _golden()
    m = _models(gpu_models)
    kw = dict(scale=4, feather=8, skip_invalid=True, to_host=True)
    for shape in _shapes(g):
        for lab in (None, [7, 8]):
            a = pipeline.restore_regions(*m, [g["image"]], [[shape]], [[lab]], **kw)[0]
            b = pipeline.restore_regions(*m, [g["image"]], [[pipeline.VerticalRegion(shape, cells=1)]], [[lab]], **kw)[0]
            np.testing.assert_array_equal(a["image"], b["image"])
            ea, eb = a["regions"][0], b["regions"][0]
            assert ("error" in ea) == ("error" in eb)
            if "error" not in ea:
                np.testing.assert_array_equal(ea["sr_u8"], eb["sr_u8"])
                np.testing.assert_array_equal(eb["line_u8"], eb["sr_u8"])
                x0, y0 = shape[:2] if type(shape) is tuple else (0, 0)            # a column's boxes are in its crop's frame
                assert ea["labels"] == eb["labels"] and len(eb["cells"]) == 2
                assert ea["boxes"] == [[b[0] + x0, b[1] + y0, b[2] + x0, b[3] + y0] for b in eb["boxes"]]


def test_predicted_column_is_the_device_sequence(gpu_models):
    """Labels and boxes None: restore_images' prediction on the twin's L, the twin's inverse layout and the rectangle composite."""
    from marconet_b200 import pipeline
    g, regs, _, _ = _golden()
    m = _models(gpu_models)
    for reg in (regs[0], pipeline.VerticalRegion(regs[0].shape, cells=4), regs[1]):
        x0, y0, x1, y1 = reg.shape
        vp = pipeline.plan_regions([g["image"].shape[:2]], [[reg]])[0].vertical
        line = V.layout(np.ascontiguousarray(g["image"][y0:y1, x0:x1]), vp.cells)
        ref = pipeline.restore_images(*m, [line], skip_invalid=True, to_host=True)[0]
        out = pipeline.restore_regions(*m, [g["image"]], [[reg]], scale=3, feather=5, skip_invalid=True, to_host=True)[0]
        e = out["regions"][0]
        assert ("error" in e) == ("error" in ref)
        if "error" in e:
            np.testing.assert_array_equal(out["image"], V.background(g["image"], 3))
            continue
        np.testing.assert_array_equal(e["line_u8"], ref["sr_u8"])
        tc = V.unlayout(ref["sr_u8"], vp.cells, vp.size[0])
        np.testing.assert_array_equal(e["sr_u8"], tc)
        assert e["labels"] == ref["labels"] and e["boxes"] == V.boxes_back(vp.cells, vp.size[0], ref["boxes"])
        np.testing.assert_array_equal(out["image"], V.compose(g["image"], [reg], [tc], 3, 5))


def test_skip_invalid_keeps_background_in_the_footprint(gpu_models):
    from marconet_b200 import pipeline
    g, regs, labels, boxes = _golden()
    m = _models(gpu_models)
    labels, boxes = list(labels), list(boxes)
    labels[2], boxes[2] = [], []                        # the tilted column has no characters: restore_images rejects it
    with pytest.raises(ValueError, match="no character labels"):
        pipeline.restore_regions(*m, [g["image"]], [regs], [labels], [boxes])
    out = pipeline.restore_regions(*m, [g["image"]], [regs], [labels], [boxes], scale=2, feather=3, skip_invalid=True,
                                   to_host=True)[0]
    e = out["regions"][2]
    assert "error" in e and "line_u8" not in e and "matrix" not in e
    srs = [None if "error" in e else e["sr_u8"] for e in out["regions"]]
    want = V.compose(g["image"], regs, srs, 2, 3)
    np.testing.assert_array_equal(out["image"], want)
    plan = pipeline.plan_regions([g["image"].shape[:2]], [regs], scale=2)
    x0, y0, x1, y1 = plan[2].out
    assert not any(2 in p.overlaps for p in plan) and plan[2].overlaps == []
    bg = V.background(g["image"], 2)
    np.testing.assert_array_equal(want[y0:y1, x0:x1], bg[y0:y1, x0:x1])


def test_vertical_launches_and_one_sync(gpu_models, monkeypatch):
    """A call with columns adds one layout launch before restore_images and one unlayout launch after it to the launches the
    shapes need; with to_host one synchronisation more.  A call without columns issues exactly its old launches."""
    from marconet_b200 import ops, pipeline
    g, regs, labels, boxes = _golden()
    m = _models(gpu_models)
    monkeypatch.setattr(ops, "MODULE_GRAPHS", False)    # a replayed module graph launches its kernels without counting them
    calls = []
    for name in ("warp_affine", "warp_perspective", "vertical_layout", "vertical_unlayout", "resize_cubic", "composite_regions",
                 "composite_regions_affine", "composite_regions_quad"):
        real = getattr(ops, name)
        monkeypatch.setattr(ops, name, lambda *a, _n=name, _f=real: (calls.append(_n), _f(*a))[1])
    plan = pipeline.plan_regions([g["image"].shape[:2]], [regs], [labels], [boxes])
    pipeline.restore_regions(*m, [g["image"]], [regs], [labels], [boxes])              # warm up
    lines, rel = [], []
    for reg, p, bx in zip(regs, plan, boxes):
        shape = getattr(reg, "shape", reg)
        crop = V.crop(g["image"], shape)
        lines.append(torch.from_numpy(V.layout(crop, p.vertical.cells) if p.vertical else crop).to(DEV))
        rel.append(p.boxes)
    n0 = ops.LAUNCHES
    pipeline.restore_images(*m, lines, labels, rel)
    n_images = ops.LAUNCHES - n0
    syncs = []
    real_sync = torch.cuda.Stream.synchronize
    monkeypatch.setattr(torch.cuda.Stream, "synchronize", lambda self: (syncs.append(1), real_sync(self))[1])
    calls.clear()
    n0 = ops.LAUNCHES
    pipeline.restore_regions(*m, [g["image"]], [regs], [labels], [boxes])
    n_regions, s_dev = ops.LAUNCHES - n0, len(syncs)
    assert calls == ["warp_affine", "warp_perspective", "vertical_layout", "vertical_unlayout", "resize_cubic",
                     "composite_regions_quad"]
    assert n_regions == n_images + 6
    pipeline.restore_regions(*m, [g["image"]], [regs], [labels], [boxes], to_host=True)
    assert len(syncs) - s_dev == s_dev + 1
    calls.clear()
    pipeline.restore_regions(*m, [g["image"]], [[regs[0], regs[5]]], [[labels[0], labels[5]]], [[boxes[0], boxes[5]]])
    assert calls == ["vertical_layout", "vertical_unlayout", "resize_cubic", "composite_regions"]
    calls.clear()
    pipeline.restore_regions(*m, [g["image"]], [[regs[5]]], [[labels[5]]], [[boxes[5]]])
    assert calls == ["resize_cubic", "composite_regions"]
    calls.clear()
    quad = _shapes(g)[2]
    pipeline.restore_regions(*m, [g["image"]], [[regs[5], quad]], [[labels[5], [3, 4]]],
                             [[boxes[5], [[2, 1, 40, 17], [44, 1, 86, 17]]]])
    assert calls == ["warp_perspective", "resize_cubic", "composite_regions_quad"]


def test_one_call_mixes_every_kind(gpu_models):
    """Columns of all three shapes with horizontal rectangles, oriented regions and quads, overlapping, on two images."""
    from marconet_b200 import pipeline
    g, regs, labels, boxes = _golden()
    m = _models(gpu_models)
    extra = _shapes(g)
    lab2, box2 = [[3, 4], [5, 6], [7, 8]], [[[2, 0, 40, 20], [44, 0, 78, 20]], [[2, 1, 40, 17], [44, 1, 86, 17]],
                                            [[2, 1, 40, 20], [44, 1, 90, 20]]]
    regs2 = [extra[1], regs[2], extra[2], regs[3], regs[0], extra[0]]
    labels2 = [lab2[1], labels[2], lab2[2], labels[3], labels[0], lab2[0]]
    boxes2 = [box2[1], boxes[2], box2[2], boxes[3], boxes[0], [[b[0] + 20, b[1] + 280, b[2] + 20, b[3] + 280] for b in box2[0]]]
    img2 = np.ascontiguousarray(g["image"][::-1])
    out = pipeline.restore_regions(*m, [g["image"], img2], [regs, regs2], [labels, labels2], [boxes, boxes2], scale=3,
                                   feather=4, to_host=True)
    for o, im, rr in zip(out, [g["image"], img2], [regs, regs2]):
        srs = [e["sr_u8"] for e in o["regions"]]
        np.testing.assert_array_equal(o["image"], V.compose(im, rr, srs, 3, 4))
    # alone, the first image's lines form other batches: its restored bytes may move by one level, its page is the same function
    a = pipeline.restore_regions(*m, [g["image"]], [regs], [labels], [boxes], scale=3, feather=4, to_host=True)[0]
    for ea, eb in zip(a["regions"], out[0]["regions"]):
        assert np.abs(ea["sr_u8"].astype(np.int16) - eb["sr_u8"].astype(np.int16)).max() <= 1
    np.testing.assert_array_equal(a["image"], V.compose(g["image"], regs, [e["sr_u8"] for e in a["regions"]], 3, 4))
