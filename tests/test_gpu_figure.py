"""test_sr.py's four-panel figure composed on the device (mn_figure_u8, restore_image / restore_images(figure=True); DESIGN.md
section 7b) against the numpy twins of oracle/figure.py and tests/golden/figure.npz (oracle/make_golden_figure.py)."""
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "figure.npz")


@pytest.fixture(scope="module")
def golden():
    return np.load(GOLDEN)


def _fixture_lines(g):
    return [(g[f"image{i}"], g[f"labels{i}"].tolist(), g[f"boxes{i}"].tolist()) for i in range(int(g["lines"]))]


def test_kernel_panels_bit_identical_to_twin(golden):
    """One launch over a batch that mixes the identity / up / down prior resizes, a line wider than the canvas, heights 9 to 40,
    a one-character image and a figure cropped below S: panels 1, 2 and 4 equal the twin; the SR rows are not touched."""
    from marconet_b200 import ops, pipeline
    from oracle import figure
    dev = torch.device("cuda:0")
    rng = np.random.default_rng(7)
    cases = [(img, boxes) for img, _, boxes in _fixture_lines(golden)]
    cases.append((golden["wide_image"], golden["wide_boxes"].tolist()))
    cases.append((rng.integers(0, 256, (9, 33, 3), dtype=np.uint8), [[2, 0, 30, 9]]))          # one character
    cases.append((rng.integers(0, 256, (20, 700, 3), dtype=np.uint8), [[-5, 0, 12, 20], [40, 0, 41, 20], [690, 0, 700, 20]]))
    items, refs, figs = [], [], []
    for k, (img, boxes) in enumerate(cases):
        h, w = img.shape[:2]
        S, wc = figure.show_width(h, w), figure.canvas_width(h, w)
        W = S if k != 5 else S - 37                                        # one figure cropped below S, as a 2048 clamp does
        n = len(boxes)
        pri = rng.uniform(-1.05, 1.05, (n, 3, 128, 128)).astype(np.float32)
        pri_d = torch.from_numpy(pri).to(dev).contiguous(memory_format=torch.channels_last)      # the generator's layout
        fig = torch.full((512, W, 3), 77, dtype=torch.uint8, device=dev)
        top, bot = pipeline.figure_markers(pipeline.boxes_to_locs(boxes, h, wc)[0].tolist(), S, 4 * wc)
        items.append((torch.from_numpy(img).to(dev), fig, top, bot, list(pri_d)))
        sr_u8 = np.full((128, W, 3), 77, np.uint8)
        refs.append(figure.figure_bytes(img, boxes, pri, sr_u8))
        figs.append(fig)
    before = ops.LAUNCHES
    ops.figure_panels(items)
    assert ops.LAUNCHES == before + 1
    for k, (fig, ref) in enumerate(zip(figs, refs)):
        got = fig.cpu().numpy()
        assert got.shape == ref.shape
        for r0, name in ((0, "ShowLQ"), (128, "ShowLocs"), (256, "SR rows"), (384, "prior")):
            d = got[r0:r0 + 128] != ref[r0:r0 + 128]
            assert not d.any(), (k, name, int(d.sum()))


def _models(gpu_models):
    return gpu_models["encoder"], gpu_models["tspgan"], gpu_models["sr"]


def test_restore_image_figure_vs_script_png(gpu_models, golden):
    """restore_image(figure=True) on the script's own inputs: ShowLQ and ShowLocs equal the PNG test_sr.py wrote; ShowSR and the
    prior panel (which go through the nets) are within one grey level; sr_u8 is figure[256:384] with figure=False's bytes."""
    from marconet_b200 import pipeline
    stride, rows = int(golden["stride"]), int(golden["prior_rows"])
    for i, (img, labels, boxes) in enumerate(_fixture_lines(golden)):
        res = pipeline.restore_image(*_models(gpu_models), img, labels, boxes, figure=True)
        plain = pipeline.restore_image(*_models(gpu_models), img, labels, boxes)
        fig = res["figure"].cpu().numpy()
        assert fig.shape == (512, golden[f"show{i}"].shape[1], 3)
        assert res["sr_u8"].data_ptr() == res["figure"][256:384].data_ptr()
        assert np.array_equal(res["sr_u8"].cpu().numpy(), plain["sr_u8"].cpu().numpy())
        assert np.array_equal(fig[:256], golden[f"show{i}"]), (i, int((fig[:256] != golden[f"show{i}"]).sum()))
        for got, ref in ((fig[256:384][::stride, ::stride], golden[f"sr_row{i}"]), (fig[384::rows], golden[f"prior_row{i}"])):
            diff = np.abs(got.astype(int) - ref.astype(int))
            assert diff.max() <= 1 and (diff != 0).mean() < 0.15, (i, int(diff.max()), float((diff != 0).mean()))


@pytest.mark.parametrize("whole_lines", [False, True])
@pytest.mark.parametrize("max_lines", [1, 8])
def test_restore_images_figure(gpu_models, golden, whole_lines, max_lines, monkeypatch):
    """restore_images(figure=True), seven short lines then the wide line of fixture (b), so that its two crops straddle two
    batches at max_lines 1 and 8 in the default mode: figure[256:384] is sr_u8 and equals figure=False's bytes; short lines'
    ShowLQ / ShowLocs equal the script's PNG; the wide line's prior panel is within one grey level of the fixture; at most one
    more launch (mn_figure_u8) per batch; to_host returns the same bytes with sr_u8 a view of figure; error entries have no figure."""
    from marconet_b200 import ops, pipeline
    short = _fixture_lines(golden)
    order = [0, 1, 2, 3, 0, 1, 2]
    images = [short[k][0] for k in order] + [golden["wide_image"]]
    labels = [short[k][1] for k in order] + [golden["wide_labels"].tolist()]
    boxes = [short[k][2] for k in order] + [golden["wide_boxes"].tolist()]
    kw = dict(max_lines=max_lines, whole_lines=whole_lines)
    m = _models(gpu_models)
    plain = pipeline.restore_images(*m, images, labels, boxes, **kw)
    if not whole_lines:
        assert len(plain[-1]["segments"]) == 2
    # the figure's launches, counted where they are issued (the modules' own counts change once their CUDA graphs are recorded)
    calls, figure_panels = [], ops.figure_panels

    def counted(items):
        n = ops.LAUNCHES
        figure_panels(items)
        calls.append(ops.LAUNCHES - n)
    monkeypatch.setattr(ops, "figure_panels", counted)
    res = pipeline.restore_images(*m, images, labels, boxes, figure=True, **kw)
    monkeypatch.setattr(ops, "figure_panels", figure_panels)
    if whole_lines:
        h_w = [im.shape[:2] for im in images]
        n_batches = len(pipeline.pack_by_columns([pipeline.whole_line_width(h, w)[1] for h, w in h_w], max_lines))
    else:
        n_lines = sum(len(r["segments"]) for r in plain)
        n_batches = -(-n_lines // max_lines)
    assert 1 <= len(calls) <= n_batches and calls == [1] * len(calls), (calls, n_batches)
    for j, (r, p) in enumerate(zip(res, plain)):
        fig = r["figure"]
        assert fig.shape[0] == 512 and fig.shape[1] == r["sr_u8"].shape[1] == p["sr_u8"].shape[1]
        assert r["sr_u8"].data_ptr() == fig[256:384].data_ptr()
        assert np.array_equal(r["sr_u8"].cpu().numpy(), p["sr_u8"].cpu().numpy()), j
    for j, k in enumerate(order):
        got = res[j]["figure"][:256].cpu().numpy()
        assert np.array_equal(got, golden[f"show{k}"]), (j, int((got != golden[f"show{k}"]).sum()))
    ref = golden["wide_prior_row"]
    S, W, wc, _ = golden["wide_geometry"].tolist()
    got = res[-1]["figure"][384::int(golden["prior_rows"])].cpu().numpy()
    assert got.shape == ref.shape == (128 // int(golden["prior_rows"]), W, 3)
    diff = np.abs(got.astype(int) - ref.astype(int))
    assert diff.max() <= 1 and (diff != 0).mean() < 0.15, (int(diff.max()), float((diff != 0).mean()))

    args = ([images[0], images[0], images[-1]], [labels[0], [], labels[-1]], [boxes[0], [], boxes[-1]])
    on_dev = pipeline.restore_images(*m, *args, figure=True, skip_invalid=True, **kw)
    host = pipeline.restore_images(*m, *args, figure=True, to_host=True, skip_invalid=True, **kw)
    assert "error" in host[1] and "figure" not in host[1] and "figure" not in on_dev[1]
    for j in (0, 2):
        assert isinstance(host[j]["figure"], np.ndarray) and np.shares_memory(host[j]["sr_u8"], host[j]["figure"])
        assert np.array_equal(host[j]["sr_u8"], host[j]["figure"][256:384])
        assert np.array_equal(host[j]["figure"], on_dev[j]["figure"].cpu().numpy()), j
