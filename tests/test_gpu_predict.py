"""Predicted characters on the device (mn_decode_predictions, pipeline.predict_characters, restore_images / restore_image without
a detector; DESIGN.md section 7b) against the numpy twin (oracle/predict.py), tests/golden/predict.npz (the reference encoder)
and the given-labels-and-boxes path."""
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "predict.npz")
PLANTED = [(32, 400, 0), (32, 3000, 1), (64, 9000, 2), (16, 513, 3), (32, 11000, 4), (27, 350, 5)]


def _models(gpu_models):
    return gpu_models["encoder"], gpu_models["tspgan"], gpu_models["sr"]


def test_kernel_equals_twin_bit_for_bit():
    """One launch over every window row of six planted lines (ties, NaNs, repeats, blank rows, > 16 characters, r < l, boxes
    beyond the image, centres on core boundaries): labels, counts and fp64 x1 / x2 equal the twin's bits; the labels also equal
    decode_labels on CUDA and on CPU for every row without multiple NaNs in a timestep."""
    from marconet_b200 import ops, pipeline
    from oracle import predict
    dev = torch.device("cuda:0")
    logits, locs, wins = [], [], []
    for h, w, seed in PLANTED:
        lg, lr = predict.planted_image(seed, h, w)
        logits.append(lg)
        locs.append(lr)
        wins += [(a, 16.0 * h, lo, hi) for (a, _), (lo, hi) in predict.plan_windows(h, w)]
    logits, locs = np.concatenate(logits), np.concatenate(locs)
    assert len(wins) > 30
    with torch.cuda.device(dev):
        table, out = ops.prediction_table(wins, dev)
        lg_d = torch.from_numpy(logits).to(dev)
        ops.decode_predictions(lg_d, torch.from_numpy(locs).to(dev), table, 0)
        rec = out.cpu().numpy().view(ops.pred_dtype())
    multi_nan = 0
    for r, (a, s, lo, hi) in enumerate(wins):
        labs, x1, x2, n_dec = predict.decode_row(logits[r], locs[r], a, s, lo, hi)
        n = int(rec[r]["n_kept"])
        assert (n, int(rec[r]["n_decoded"])) == (len(labs), n_dec), r
        assert rec[r]["label"][:n].tolist() == labs and (rec[r]["label"][n:] == -1).all(), r
        assert rec[r]["x1"][:n].tobytes() == np.asarray(x1, np.float64).tobytes(), r
        assert rec[r]["x2"][:n].tobytes() == np.asarray(x2, np.float64).tobytes(), r
        if (np.isnan(logits[r]).sum(axis=1) > 1).any():
            multi_nan += 1
            continue
        ref = predict.restate.clear_labels(torch.from_numpy(logits[r]))[:16]
        assert pipeline.decode_labels(lg_d[r])[:16] == ref == pipeline.decode_labels(torch.from_numpy(logits[r]))[:16], r
    assert multi_nan >= 1


def test_device_encoder_and_predict_characters_match_golden(gpu_models):
    """The fixture's windows: the device encoder's argmax equals the reference's at every timestep and locs_lr is within 1e-3;
    predict_characters returns the fixture's merged labels exactly and its boxes within 1e-3 * 16h source columns."""
    from marconet_b200 import ops, pipeline
    g = np.load(GOLDEN)
    enc = gpu_models["encoder"]
    dev = torch.device("cuda:0")
    for name in ("fit", "wide"):
        img = g[f"{name}_image"]
        h = img.shape[0]
        d = torch.from_numpy(img).to(dev)
        lq, _ = ops.preprocess_lq_crops([(d, int(a), int(b)) for a, b in g[f"{name}_crops"]])
        logits, locs_lr, _ = enc(lq)
        assert np.array_equal(logits.argmax(-1).cpu().numpy(), g[f"{name}_argmax"]), name
        assert np.abs(locs_lr.cpu().numpy() - g[f"{name}_locs_lr"]).max() <= 1e-3, name
        for ml in (1, 8):
            pred = pipeline.predict_characters(enc, [img], max_lines=ml)[0]
            assert pred["labels"] == g[f"{name}_labels"].tolist(), name
            assert np.abs(np.asarray(pred["boxes"], np.float64).reshape(-1, 4) - g[f"{name}_boxes"]).max() <= 1e-3 * 16 * h


class PlantedEncoder(torch.nn.Module):
    """The real encoder with chosen logits and (left, right) boxes for the first rows it encodes (the real style w always)."""

    def __init__(self, enc, logits, locs):
        super().__init__()
        self.enc, self.logits, self.locs, self.used = enc, logits, locs, 0

    def forward(self, lq):
        lg, lr, w = self.enc(lq)
        b, r0 = lq.shape[0], self.used
        if r0 < self.logits.shape[0]:
            lg, lr = self.logits[r0:r0 + b].to(lq.device), self.locs[r0:r0 + b].to(lq.device)
            self.used += b
        return lg, lr, w


def _planted_line(h, w, seed):
    """Characters every 36 source columns (widths 16 to 28, integer columns) and the encoder outputs that predict them on each
    detection window: one CTC step per character between blanks, boxes exact in fp32 (h = 32: 16h = 512)."""
    from marconet_b200 import pipeline
    rng = np.random.default_rng(seed)
    chars, x = [], 6
    while x + 30 < w:
        cw = int(rng.integers(16, 29))
        chars.append((int(rng.integers(0, 6735)), x, x + cw))
        x += 36
    wins = pipeline.plan_windows(h, w)
    logits = torch.zeros(len(wins), 64, 6736)
    logits[:, :, 6735] = 1.0
    locs = torch.rand(len(wins), 32, generator=torch.Generator().manual_seed(seed))
    for k, win in enumerate(wins):
        a, b = win.crop
        inside = [c for c in chars if a <= c[1] and c[2] <= b][:16]
        for j, (lab, x1, x2) in enumerate(inside):
            logits[k, 4 * j, lab] = 5.0
            locs[k, 2 * j], locs[k, 2 * j + 1] = (x1 - a) / (16.0 * h), (x2 - a) / (16.0 * h)
    return chars, logits, locs


@pytest.mark.parametrize("w", [400, 2300])
def test_planted_encoder_predictions_restore_end_to_end(gpu_models, w):
    """A line that fits and a six-window line: characters in window overlaps are seen by both windows and owned by one;
    predict_characters returns the planted labels and boxes exactly; restore_images restores the line without errors in both
    modes at max_lines 1 and 8, with those labels and boxes."""
    from marconet_b200 import pipeline
    enc, tsp, sr = _models(gpu_models)
    h = 32
    chars, logits, locs = _planted_line(h, w, seed=w)
    img = np.random.default_rng(w).integers(0, 256, (h, w, 3), dtype=np.uint8)
    pred = pipeline.predict_characters(PlantedEncoder(enc, logits, locs), [img])[0]
    assert len(pred["windows"]) == len(pipeline.plan_windows(h, w)) and (len(pred["windows"]) == 1) == (w == 400)
    if w != 400:
        seen_twice = [c for c in chars if sum(win.crop[0] <= c[1] and c[2] <= win.crop[1] for win in pred["windows"]) > 1]
        assert len(seen_twice) >= 4
    assert pred["labels"] == [c[0] for c in chars]
    assert pred["boxes"] == [[float(x1), 0, float(x2), h] for _, x1, x2 in chars]
    for whole in (False, True):
        for ml in (1, 8):
            res = pipeline.restore_images(PlantedEncoder(enc, logits, locs), tsp, sr, [img], max_lines=ml, whole_lines=whole)[0]
            assert "error" not in res, res
            assert res["labels"] == pred["labels"] and res["boxes"] == pred["boxes"]
            assert res["sr_u8"].shape == (128, round(w * 128 / h), 3)


def _image_set():
    g = np.load(GOLDEN)
    rng = np.random.default_rng(3)
    return [g["fit_image"], g["wide_image"], rng.integers(0, 256, (24, 200, 3), dtype=np.uint8),
            rng.integers(0, 256, (40, 1900, 3), dtype=np.uint8), g["fit_image"][:, :60].copy()]


@pytest.mark.parametrize("whole_lines", [False, True])
def test_predicted_restore_equals_given_restore(gpu_models, whole_lines):
    """restore_images(images, None, None) gives the bytes (and figures, and error entries under skip_invalid) of
    restore_images(images, pred.labels, pred.boxes), with figure on and off and with to_host; restore_image likewise."""
    from marconet_b200 import pipeline
    m = _models(gpu_models)
    images = _image_set()
    preds = pipeline.predict_characters(m[0], images)
    labels, boxes = [p["labels"] for p in preds], [p["boxes"] for p in preds]
    n_ok = 0
    for figure in (False, True):
        for to_host in (False, True):
            kw = dict(whole_lines=whole_lines, figure=figure, to_host=to_host, skip_invalid=True)
            a = pipeline.restore_images(*m, images, **kw)
            b = pipeline.restore_images(*m, images, labels, boxes, **kw)
            for i, (ra, rb) in enumerate(zip(a, b)):
                assert ("error" in ra) == ("error" in rb), (i, ra.get("error"), rb.get("error"))
                if "error" in ra:
                    continue
                n_ok += 1
                assert ra["labels"] == labels[i] and ra["boxes"] == boxes[i]
                for key in ("sr_u8", "figure") if figure else ("sr_u8",):
                    x, y = ra[key], rb[key]
                    x, y = (x, y) if to_host else (x.cpu().numpy(), y.cpu().numpy())
                    assert np.array_equal(x, y), (i, key)
    assert n_ok >= 8
    one = pipeline.restore_image(*m, images[0], figure=True)
    ref = pipeline.restore_image(*m, images[0], preds[0]["labels"], preds[0]["boxes"], figure=True)
    assert one["labels"] == preds[0]["labels"] and torch.equal(one["figure"], ref["figure"])


def test_fit_line_boxes_match_encoder_pairs(gpu_models):
    """On a line that fits, boxes_to_locs(pred.boxes, h, 512) equals the encoder's converted (centre, half-width) pairs within
    1 fp32 ulp for every box the clamp left alone."""
    from marconet_b200 import ops, pipeline
    enc = gpu_models["encoder"]
    g = np.load(GOLDEN)
    img = g["fit_image"]
    h, w = img.shape[:2]
    pred = pipeline.predict_characters(enc, [img])[0]
    lq, _ = ops.preprocess_lq_crops([(torch.from_numpy(img).cuda(), 0, w)])
    logits, locs_lr, _ = enc(lq)
    n = len(pipeline.decode_labels(logits[0])[:16])
    conv = pipeline.lr_to_center_halfwidth(locs_lr.cpu())[0]
    checked = 0
    for j in range(n):
        c, hw = conv[2 * j].item(), conv[2 * j + 1].item()
        x1, x2 = (c - hw) * 16.0 * h, (c + hw) * 16.0 * h
        if not (0 <= x1 <= x2 <= w) or [x1, 0, x2, h] not in pred["boxes"]:
            continue
        got = pipeline.boxes_to_locs([[x1, 0, x2, h]], h, 512)[0]
        want = torch.tensor([c, hw], dtype=torch.float32)
        ulp = torch.abs(torch.nextafter(want, torch.full_like(want, float("inf"))) - want)
        assert (torch.abs(got - want) <= ulp).all(), (j, got, want)
        checked += 1
    assert checked >= 1


def test_manual_labels_and_invalid_pairings(gpu_models):
    """Given labels pair with predicted boxes (the reference README's -m mode); a count mismatch raises or becomes an error
    entry; boxes without labels raise; restore_image refuses to predict on a line wider than the canvas."""
    from marconet_b200 import pipeline
    m = _models(gpu_models)
    images = _image_set()
    pred = pipeline.predict_characters(m[0], images[:1])[0]
    n = len(pred["labels"])
    manual = list(range(100, 100 + n))
    res = pipeline.restore_images(*m, images[:1], [manual], None)[0]
    ref = pipeline.restore_images(*m, images[:1], [manual], [pred["boxes"]])[0]
    assert res["labels"] == manual and res["boxes"] == pred["boxes"] and torch.equal(res["sr_u8"], ref["sr_u8"])
    one = pipeline.restore_image(*m, images[0], manual)
    assert one["labels"] == manual
    with pytest.raises(ValueError, match="image 0"):
        pipeline.restore_images(*m, images[:1], [manual + [5]], None)
    out = pipeline.restore_images(*m, images[:2], [manual + [5], None], None, skip_invalid=True)
    assert "error" in out[0] and "labels given" in out[0]["error"]
    with pytest.raises(ValueError):
        pipeline.restore_images(*m, images[:1], None, [pred["boxes"]])
    with pytest.raises(ValueError):
        pipeline.restore_image(*m, images[0], None, pred["boxes"])
    with pytest.raises(ValueError, match="restore_images"):
        pipeline.restore_image(*m, images[1])


def test_stage_launches_and_given_path_untouched(gpu_models, monkeypatch):
    """The stage adds, per detection batch, one crop launch, the encoder's launches and one decode launch, and synchronises
    once; a call with labels and boxes given never enters it."""
    from marconet_b200 import ops, pipeline
    m = _models(gpu_models)
    enc = m[0]
    images = _image_set()
    n_rows = sum(len(pipeline.plan_windows(*im.shape[:2])) for im in images)
    pipeline.predict_characters(enc, images)                       # warm-up: every batch shape recorded
    sizes = [min(8, n_rows - r0) for r0 in range(0, n_rows, 8)]
    per_enc = {}
    for b in set(sizes):
        lq = torch.zeros(b, 3, 32, 512, device="cuda")
        l0 = ops.LAUNCHES
        enc(lq)
        per_enc[b] = ops.LAUNCHES - l0
    syncs = []
    real_sync = torch.cuda.Stream.synchronize
    monkeypatch.setattr(torch.cuda.Stream, "synchronize", lambda self: (syncs.append(1), real_sync(self))[1])
    l0 = ops.LAUNCHES
    pipeline.predict_characters(enc, images)
    assert ops.LAUNCHES - l0 == sum(2 + per_enc[b] for b in sizes)
    assert len(syncs) == 1
    monkeypatch.undo()
    preds = pipeline.predict_characters(enc, images[:1])

    def refuse(*a, **k):
        raise AssertionError("the prediction stage ran")
    monkeypatch.setattr(pipeline, "_predict", refuse)
    pipeline.restore_images(*m, images[:1], [preds[0]["labels"]], [preds[0]["boxes"]])
