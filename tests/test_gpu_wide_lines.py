"""Batched restoration of text-line images of any width (pipeline.restore_images) and its two kernels
(mn_preprocess_lq_u8_batched, mn_postprocess_sr_u8_pieces) against the oracle restatements (oracle/image_ops.py, oracle/wide_line.py), restore_image
and the stitched output of the reference modules on each crop (tests/golden/wide_line.npz)."""
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def _img(h, w, seed):
    rng = np.random.default_rng(seed)
    if seed % 3 == 2:
        return (rng.integers(0, 2, (h, w, 3)) * 255).astype(np.uint8)
    return rng.integers(0, 256, (h, w, 3), dtype=np.uint8)


def _random_crops(n_images=8, seed=0):
    """(images, crops): random images of heights 4..200, several crops each, touching both image edges, 1-pixel-wide crops."""
    rng = np.random.default_rng(seed)
    images, crops = [], []
    for i in range(n_images):
        h = int(rng.integers(4, 201)) if i > 1 else (4, 200)[i]
        max_cols = int(511.5 * h / 32)
        w = int(rng.integers(2, 3 * max_cols + 3))
        images.append(_img(h, w, seed * 100 + i))
        spans = [(0, min(w, int(rng.integers(1, max_cols + 1)))), (max(0, w - int(rng.integers(1, max_cols + 1))), w)]
        a = int(rng.integers(0, w))
        spans.append((a, min(w, a + int(rng.integers(1, max_cols + 1)))))
        if h <= 64:                     # a 1-pixel crop resizes to round(32/h) >= 1 columns only up to h = 64
            spans += [(0, 1), (w - 1, w), (w // 2, w // 2 + 1)]
        crops += [(i, x0, x1) for x0, x1 in spans]
    return images, crops


def test_crop_kernel_bit_exact_against_the_oracle_on_each_contiguous_crop():
    from marconet_b200 import ops
    from oracle import wide_line
    dev = torch.device("cuda:0")
    images, crops = _random_crops()
    assert len(crops) >= 20
    # image 3 is read through a row pitch wider than its own rows (a column slice of a wider buffer)
    dimg = [torch.from_numpy(im).to(dev) for im in images]
    wide = torch.zeros((images[3].shape[0], images[3].shape[1] + 37, 3), dtype=torch.uint8, device=dev)
    wide[:, 11:11 + images[3].shape[1]] = dimg[3]
    dimg[3] = wide[:, 11:11 + images[3].shape[1]]
    l0 = ops.LAUNCHES
    lq, widths = ops.preprocess_lq_crops([(dimg[i], a, b) for i, a, b in crops])
    assert ops.LAUNCHES == l0 + 1 and tuple(lq.shape) == (len(crops), 3, 32, 512)
    got = lq.cpu().numpy()
    for k, (i, a, b) in enumerate(crops):
        ref, ref_w = wide_line.preprocess_lq_crop(images[i], a, b)
        assert widths[k] == ref_w and np.array_equal(got[k], ref[0]), (k, images[i].shape, a, b)
        single, _ = ops.preprocess_lq(dimg[i][:, a:b].contiguous())
        assert torch.equal(single[0], lq[k])


def test_crop_kernel_matches_live_cv2_when_ipp_is_off():
    cv2 = pytest.importorskip("cv2")
    from marconet_b200 import ops
    dev = torch.device("cuda:0")
    images, crops = _random_crops(seed=1)
    dimg = [torch.from_numpy(im).to(dev) for im in images]
    lq, widths = ops.preprocess_lq_crops([(dimg[i], a, b) for i, a, b in crops])
    got = lq.cpu().numpy()
    was = cv2.ipp.useIPP()
    cv2.ipp.setUseIPP(False)
    try:
        for k, (i, a, b) in enumerate(crops):
            h = images[i].shape[0]
            ref = cv2.resize(np.ascontiguousarray(images[i][:, a:b]), (0, 0), fx=32 / h, fy=32 / h, interpolation=cv2.INTER_CUBIC)
            assert widths[k] == ref.shape[1]
            u8 = np.rint((got[k][:, :, :widths[k]].transpose(1, 2, 0) * 0.5 + 0.5) * 255).astype(np.uint8)
            assert np.array_equal(u8, ref), (k, h, a, b)
    finally:
        cv2.ipp.setUseIPP(was)


def test_crop_kernel_rejects_crops_that_do_not_fit():
    from marconet_b200 import ops
    dev = torch.device("cuda:0")
    img = torch.from_numpy(_img(32, 700, 0)).to(dev)
    with pytest.raises(ValueError, match="does not fit"):
        ops.preprocess_lq_crops([(img, 0, 100), (img, 100, 700)])
    with pytest.raises(ValueError, match="not a non-empty range"):
        ops.preprocess_lq_crops([(img, 50, 50)])


def test_stitch_kernel_bit_exact_against_the_numpy_twin():
    from marconet_b200 import ops
    from oracle import image_ops
    dev = torch.device("cuda:0")
    g = torch.Generator().manual_seed(5)
    sr = torch.rand(3, 3, 128, 2048, generator=g) * 2.6 - 1.3
    sr_dev = sr.to(dev).contiguous(memory_format=torch.channels_last)     # what TSPSRNet returns
    ref_lines = image_ops.postprocess_sr(sr.numpy())
    outs = [torch.full((128, 3000, 3), 7, dtype=torch.uint8, device=dev), torch.full((128, 900, 3), 7, dtype=torch.uint8, device=dev)]
    spec = [(0, 0, 0, 0, 1800), (1, 64, 0, 1800, 1200), (2, 0, 1, 0, 1), (2, 1, 1, 1, 600), (0, 2047, 1, 601, 1), (1, 3, 1, 650, 250)]
    l0 = ops.LAUNCHES
    ops.postprocess_sr_pieces(sr_dev, [(line, src, outs[d][:, x0:x0 + wd]) for line, src, d, x0, wd in spec])
    assert ops.LAUNCHES == l0 + 1
    want = [np.full((128, 3000, 3), 7, np.uint8), np.full((128, 900, 3), 7, np.uint8)]
    for line, src, d, x0, wd in spec:
        want[d][:, x0:x0 + wd] = ref_lines[line][:, src:src + wd]
    for d in range(2):
        assert np.array_equal(outs[d].cpu().numpy(), want[d]), d
    with pytest.raises(ValueError, match="outside"):
        ops.postprocess_sr_pieces(sr_dev, [(0, 2000, outs[0][:, :100])])


def _script_image():
    g = np.load(os.path.join(GOLDEN, "script_sr_row.npz"))
    return np.ascontiguousarray(g["image_rgb"]), g["labels"].tolist(), g["boxes"].tolist()


def _e2e_image():                     # the image of test_gpu_image.py::test_restore_image_end_to_end
    return _img(40, 500, 11), [5, 17, 300, 4242], [[20 + 110 * i, 4, 100 + 110 * i, 36] for i in range(4)]


def _wide_image():
    g = np.load(os.path.join(GOLDEN, "wide_line.npz"))
    return g["image"], g["labels"].tolist(), g["boxes"].tolist()


def _run(gm, images, **kw):
    from marconet_b200 import pipeline
    return pipeline.restore_images(gm["encoder"], gm["tspgan"], gm["sr"], [i[0] for i in images], [i[1] for i in images],
                                   [i[2] for i in images], **kw)


def test_single_image_equals_restore_image_bit_for_bit(gpu_models):
    from marconet_b200 import pipeline
    gm = gpu_models
    for img, labels, boxes in (_e2e_image(), _script_image()):
        ref = pipeline.restore_image(gm["encoder"], gm["tspgan"], gm["sr"], img, labels, boxes)["sr_u8"]
        for src in (img, torch.from_numpy(img), torch.from_numpy(img).cuda()):
            res = _run(gm, [(src, labels, boxes)])[0]
            assert len(res["segments"]) == 1 and res["sr_u8"].is_cuda
            assert torch.equal(res["sr_u8"], ref)
        host = _run(gm, [(img, labels, boxes)], to_host=True)[0]["sr_u8"]
        assert isinstance(host, np.ndarray) and np.array_equal(host, ref.cpu().numpy())


def _per_crop_reference(gm, img, labels, boxes, segments):
    """restore_image on every crop that owns characters, written to the columns restore_images gives it; mask of those columns."""
    from marconet_b200 import ops, pipeline
    h, w = img.shape[:2]
    width, pieces = pipeline.stitch_pieces(h, w, segments)
    out = np.zeros((128, width, 3), np.uint8)
    mask = np.zeros(width, bool)
    for k, o0, src, wd in pieces:
        s = segments[k]
        if s.chars[0] == s.chars[1]:
            continue
        crop = np.ascontiguousarray(img[:, s.crop[0]:s.crop[1]])
        r = pipeline.restore_image(gm["encoder"], gm["tspgan"], gm["sr"], crop, labels[s.chars[0]:s.chars[1]], s.boxes)["sr"]
        out[:, o0:o0 + wd] = ops.postprocess_sr(r)[0, :, src:src + wd].cpu().numpy()
        mask[o0:o0 + wd] = True
    return out, mask


def test_mixed_batch_matches_restore_image_on_each_crop(gpu_models):
    gm = gpu_models
    images = [_e2e_image(), _script_image(), _wide_image()]
    runs = {ml: _run(gm, images, max_lines=ml) for ml in (1, 8)}
    identical = all(torch.equal(a["sr_u8"], b["sr_u8"]) for a, b in zip(runs[1], runs[8]))
    print(f"\nrestore_images max_lines=1 vs 8 bit-identical: {identical}")
    assert [len(r["segments"]) for r in runs[8]] == [1, 1, 4]
    for k, (img, labels, boxes) in enumerate(images):
        ref, mask = _per_crop_reference(gm, img, labels, boxes, runs[8][k]["segments"])
        h, w = img.shape[:2]
        assert mask.mean() > 0.8
        for ml, res in runs.items():
            got = res[k]["sr_u8"].cpu().numpy()
            assert got.shape == ref.shape == (128, min(round(w * 128 / h), 2048) if len(res[k]["segments"]) == 1 else round(w * 128 / h), 3)
            diff = np.abs(got[:, mask].astype(int) - ref[:, mask].astype(int))
            assert diff.max() <= 1 and (diff != 0).mean() < 0.15, (k, ml, int(diff.max()), float((diff != 0).mean()))


def test_wide_line_matches_the_reference_modules_crop_by_crop(gpu_models):
    """Against tests/golden/wide_line.npz (the reference modules on each crop, test_sr.py's data flow, stitched): within one grey
    level where the nets' <= 1e-3 error crosses a rounding boundary, like the script-PNG tests."""
    g = np.load(os.path.join(GOLDEN, "wide_line.npz"))
    res = _run(gpu_models, [_wide_image()], to_host=True)[0]
    assert [s.core[0] for s in res["segments"]] + [g["image"].shape[1]] == g["cuts"].tolist()
    stride = int(g["stride"])
    got = res["sr_u8"][::stride, ::stride]
    assert got.shape == g["sr_line"].shape
    diff = np.abs(got.astype(int) - g["sr_line"].astype(int))
    assert diff.max() <= 1 and (diff != 0).mean() < 0.15, (int(diff.max()), float((diff != 0).mean()))


def test_invalid_images_fail_before_any_launch_or_are_skipped(gpu_models):
    from marconet_b200 import ops
    gm = gpu_models
    good = _e2e_image()
    bad_label = (good[0], [5, 17, 6736, 1], good[2])
    too_wide = (_img(32, 2000, 3), [1, 2], [[0, 0, 20, 32], [100, 0, 700, 32]])
    l0 = ops.LAUNCHES
    with pytest.raises(IndexError, match="image 1, character 2"):
        _run(gm, [good, bad_label])
    with pytest.raises(ValueError, match="image 1, character 1"):
        _run(gm, [good, too_wide])
    assert ops.LAUNCHES == l0
    res = _run(gm, [bad_label, good, too_wide], skip_invalid=True)
    assert "IndexError" in res[0]["error"] and "ValueError" in res[2]["error"]
    assert torch.equal(res[1]["sr_u8"], _run(gm, [good])[0]["sr_u8"])
