"""Text regions in whole images on the device (DESIGN.md section 7b): the background and composite kernels bit for bit against
live cv2 (IPP off) and the numpy twin, and pipeline.restore_regions against tests/golden/regions.npz, restore_images and itself."""
import os

import numpy as np
import pytest
import torch

from oracle import regions as R

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "regions.npz")
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


def test_background_kernel_equals_cv2(cv2_no_ipp):
    from marconet_b200 import ops
    rng = np.random.default_rng(0)
    shapes = [(7, 13), (1, 9), (11, 1), (33, 70), (1, 1), (100, 300), (48, 37), (160, 700)]
    items, refs = [], []
    for k, (h, w) in enumerate(shapes):
        s = k % 8 + 1
        img = rng.integers(0, 256, (h, w, 3), dtype=np.uint8)
        if k == 3:                                       # read through a pitch wider than its rows
            wide = torch.from_numpy(rng.integers(0, 256, (h, w + 17, 3), dtype=np.uint8)).to(DEV)
            wide[:, 5:5 + w] = torch.from_numpy(img).to(DEV)
            src = wide[:, 5:5 + w]
            assert src.stride(0) == 3 * (w + 17)
        else:
            src = torch.from_numpy(img).to(DEV)
        items.append((src, torch.empty((s * h, s * w, 3), dtype=torch.uint8, device=DEV)))
        refs.append(cv2_no_ipp.resize(img, (0, 0), fx=s, fy=s, interpolation=cv2_no_ipp.INTER_CUBIC))
    n0 = ops.LAUNCHES
    ops.resize_cubic(items)
    assert ops.LAUNCHES - n0 == 1
    for k, ((_, dst), ref) in enumerate(zip(items, refs)):
        np.testing.assert_array_equal(_np(dst), ref, err_msg=f"image {k}")


def _random_regions(rng, H, W, n):
    rects = [(0, 0, W, H), (W - 1, H - 1, W, H), (3, 2, 4, 9), (1, 4, W - 2, 5)]       # whole page, 1x1 corner, 1-wide, 1-high
    x0, y0 = W // 4, H // 4
    rects += [(x0, y0, x0 + W // 3, y0 + H // 3), (x0 + 3, y0 + 2, x0 + W // 2, y0 + H // 2),
              (x0 + 5, y0 + 4, W, H)]                    # a chain of three overlaps, the last touching the right and bottom
    while len(rects) < n:
        a, b = sorted(rng.integers(0, W + 1, 2))
        c, d = sorted(rng.integers(0, H + 1, 2))
        if a < b and c < d:
            rects.append((int(a), int(c), int(b), int(d)))
    order = rng.permutation(len(rects))
    return [rects[i] for i in order]


@pytest.mark.parametrize("feather", [0, 1, 8, 1000])
def test_composite_kernel_equals_twin(feather):
    from marconet_b200 import ops, pipeline
    rng = np.random.default_rng(feather)
    shapes = [(24, 40), (17, 61), (9, 9)]
    s = 3
    imgs = [rng.integers(0, 256, (h, w, 3), dtype=np.uint8) for h, w in shapes]
    rects = [_random_regions(rng, h, w, 14) for h, w in shapes]
    ts = [[rng.integers(0, 256, (int(rng.choice([128, 1, 37])), int(rng.integers(1, 300)), 3), dtype=np.uint8) for _ in rr]
          for rr in rects]
    plan = pipeline.plan_regions(shapes, rects, scale=s, feather=feather)
    pages = [torch.from_numpy(R.background(im, s)).to(DEV) for im in imgs]
    dts = []
    for k, p in enumerate(plan):
        t = ts[p.image][p.region]
        if k % 2:                                        # restored bytes read through a pitch wider than their rows
            buf = torch.zeros((t.shape[0], t.shape[1] + 9, 3), dtype=torch.uint8, device=DEV)
            buf[:, 2:2 + t.shape[1]] = torch.from_numpy(t).to(DEV)
            dts.append(buf[:, 2:2 + t.shape[1]])
        else:
            dts.append(torch.from_numpy(t).to(DEV))
    ok = [k for k in range(len(plan)) if k % 5 != 4]    # some regions left out, as failed ones are
    n0 = ops.LAUNCHES
    ops.composite_regions([(pages[plan[k].image], dts[k], plan[k].out, c) for k, c in zip(ok, pipeline.region_chains(plan, ok))],
                          feather)
    assert ops.LAUNCHES - n0 == 1
    for i, im in enumerate(imgs):
        srs = [ts[i][p.region] if k in ok else None for k, p in enumerate(plan) if p.image == i]
        want = R.compose(im, rects[i], srs, s, feather)
        np.testing.assert_array_equal(_np(pages[i]), want, err_msg=f"image {i}")


def _golden():
    g = np.load(GOLDEN)
    rects = [tuple(r) for r in g["regions"].tolist()]
    labels, boxes = [[] for _ in rects], [[] for _ in rects]
    for lab, (x1, y1, x2, y2, r) in zip(g["labels"].tolist(), g["boxes"].tolist()):
        labels[r].append(lab)
        boxes[r].append([x1, y1, x2, y2])
    return g, rects, labels, boxes


@pytest.mark.parametrize("to_host", [False, True])
def test_restore_regions_golden(gpu_models, to_host):
    from marconet_b200 import pipeline
    g, rects, labels, boxes = _golden()
    s, f = int(g["scale"]), int(g["feather"])
    out = pipeline.restore_regions(*_models(gpu_models), [g["image"]], [rects], [labels], [boxes], scale=s, feather=f,
                                   to_host=to_host)
    assert len(out) == 1 and len(out[0]["regions"]) == 4
    page = _np(out[0]["image"])
    assert page.shape == (s * 160, s * 700, 3)
    srs = []
    for r, e in enumerate(out[0]["regions"]):
        t = _np(e["sr_u8"])
        assert isinstance(e["sr_u8"], np.ndarray) == to_host
        k = int(g["sr_strides"][r])                         # the wide region's reference bytes are stored strided
        ref = g[f"sr{r}"]
        assert t[::k, ::k].shape == ref.shape and t.shape[0] == 128, r
        d = np.abs(t[::k, ::k].astype(np.int16) - ref.astype(np.int16)).max()
        assert d <= 1, (r, d)
        assert e["labels"] == labels[r] and e["boxes"] == boxes[r]
        srs.append(t)
    np.testing.assert_array_equal(page, R.compose(g["image"], rects, srs, s, f))
    assert len(out[0]["regions"][1]["segments"]) == 2                      # the region wider than the canvas is cut


def test_one_region_is_restore_images(gpu_models):
    from marconet_b200 import pipeline
    g, rects, labels, boxes = _golden()
    x0, y0, x1, y1 = rects[2]
    img = np.ascontiguousarray(g["image"][y0:y0 + 32, x0:x1])                # a 32-row image
    bx = [[b[0] - x0, 0, b[2] - x0, 32] for b in boxes[2]]
    m = _models(gpu_models)
    ref = pipeline.restore_images(*m, [img], [labels[2]], [bx], to_host=True)[0]["sr_u8"]
    out = pipeline.restore_regions(*m, [img], [[(0, 0, img.shape[1], 32)]], [[labels[2]]], [[bx]], scale=4, feather=0,
                                   to_host=True)[0]
    assert out["image"].shape == ref.shape
    np.testing.assert_array_equal(out["image"], ref[..., ::-1])
    np.testing.assert_array_equal(out["regions"][0]["sr_u8"], ref)


def test_given_labels_equal_restore_images_on_crops(gpu_models):
    """Same crops, same order, same max_lines: the same batches, so the same bytes."""
    from marconet_b200 import pipeline
    g, rects, labels, boxes = _golden()
    m = _models(gpu_models)
    crops = [np.ascontiguousarray(g["image"][y0:y1, x0:x1]) for x0, y0, x1, y1 in rects]
    rel = [[[b[0] - x0, b[1] - y0, b[2] - x0, b[3] - y0] for b in bx] for (x0, y0, _, _), bx in zip(rects, boxes)]
    for max_lines in (1, 8):
        ref = pipeline.restore_images(*m, crops, labels, rel, max_lines=max_lines, to_host=True)
        out = pipeline.restore_regions(*m, [g["image"]], [rects], [labels], [boxes], max_lines=max_lines, to_host=True)[0]
        for r, (a, b) in enumerate(zip(out["regions"], ref)):
            np.testing.assert_array_equal(a["sr_u8"], b["sr_u8"], err_msg=f"max_lines {max_lines}, region {r}")
            assert a["segments"] == b["segments"]


def test_predicted_regions_equal_restore_images(gpu_models):
    from marconet_b200 import pipeline
    g, rects, _, _ = _golden()
    m = _models(gpu_models)
    img2 = np.random.default_rng(7).integers(0, 256, (50, 90, 3), dtype=np.uint8)
    rects2 = [(0, 0, 90, 24), (10, 20, 80, 50)]
    crops = [np.ascontiguousarray(g["image"][y0:y1, x0:x1]) for x0, y0, x1, y1 in rects] + \
        [np.ascontiguousarray(img2[y0:y1, x0:x1]) for x0, y0, x1, y1 in rects2]
    ref = pipeline.restore_images(*m, crops, skip_invalid=True, to_host=True)
    out = pipeline.restore_regions(*m, [g["image"], img2], [rects, rects2], skip_invalid=True, to_host=True)
    entries = out[0]["regions"] + out[1]["regions"]
    n_ok = 0
    for k, (a, b, (x0, y0, _, _)) in enumerate(zip(entries, ref, rects + rects2)):
        assert ("error" in a) == ("error" in b), (k, a.get("error"), b.get("error"))
        if "error" in a:
            continue
        n_ok += 1
        assert a["labels"] == b["labels"]
        assert a["boxes"] == [[q[0] + x0, q[1] + y0, q[2] + x0, q[3] + y0] for q in b["boxes"]]
        np.testing.assert_array_equal(a["sr_u8"], b["sr_u8"], err_msg=f"region {k}")
    assert n_ok >= 3
    for i, (im, rr, ents) in enumerate(((g["image"], rects, out[0]["regions"]), (img2, rects2, out[1]["regions"]))):
        srs = [None if "error" in e else e["sr_u8"] for e in ents]
        np.testing.assert_array_equal(out[i]["image"], R.compose(im, rr, srs, 4, 8))


def test_skip_invalid_keeps_background(gpu_models):
    from marconet_b200 import pipeline
    g, rects, labels, boxes = _golden()
    m = _models(gpu_models)
    labels, boxes = list(labels), list(boxes)
    labels[3], boxes[3] = [], []                        # no characters: restore_images rejects the region
    with pytest.raises(ValueError, match="no character labels"):
        pipeline.restore_regions(*m, [g["image"]], [rects], [labels], [boxes])
    dev = pipeline.restore_regions(*m, [g["image"]], [rects], [labels], [boxes], scale=2, feather=3, skip_invalid=True)[0]
    host = pipeline.restore_regions(*m, [g["image"]], [rects], [labels], [boxes], scale=2, feather=3, skip_invalid=True,
                                    to_host=True)[0]
    assert "error" in dev["regions"][3] and "error" in host["regions"][3]
    srs = [_np(e["sr_u8"]) for e in dev["regions"][:3]] + [None]
    want = R.compose(g["image"], rects, srs, 2, 3)
    np.testing.assert_array_equal(_np(dev["image"]), want)
    np.testing.assert_array_equal(host["image"], want)
    x0, y0, x1, y1 = rects[3]
    np.testing.assert_array_equal(want[2 * y0:2 * y1, 2 * x0:2 * x1], R.background(g["image"], 2)[2 * y0:2 * y1, 2 * x0:2 * x1])
    for a, b in zip(dev["regions"][:3], host["regions"][:3]):
        np.testing.assert_array_equal(_np(a["sr_u8"]), b["sr_u8"])


def test_restore_regions_launches_and_one_sync(gpu_models, monkeypatch):
    """One background and one composite launch on top of restore_images' own; with to_host one synchronisation more."""
    from marconet_b200 import ops, pipeline
    g, rects, labels, boxes = _golden()
    m = _models(gpu_models)
    pipeline.restore_regions(*m, [g["image"]], [rects], [labels], [boxes])            # warm up
    n0 = ops.LAUNCHES
    pipeline.restore_images(*m, [torch.from_numpy(np.ascontiguousarray(g["image"][y0:y1, x0:x1])).to(DEV)
                                 for x0, y0, x1, y1 in rects], labels,
                            [[[b[0] - r[0], b[1] - r[1], b[2] - r[0], b[3] - r[1]] for b in bx] for r, bx in zip(rects, boxes)])
    n_images = ops.LAUNCHES - n0
    syncs = []
    real_sync = torch.cuda.Stream.synchronize
    monkeypatch.setattr(torch.cuda.Stream, "synchronize", lambda self: (syncs.append(1), real_sync(self))[1])
    n0 = ops.LAUNCHES
    pipeline.restore_regions(*m, [g["image"]], [rects], [labels], [boxes])
    n_regions, s_dev = ops.LAUNCHES - n0, len(syncs)
    pipeline.restore_regions(*m, [g["image"]], [rects], [labels], [boxes], to_host=True)
    monkeypatch.undo()
    assert n_regions == n_images + 2
    assert len(syncs) - s_dev == s_dev + 1
