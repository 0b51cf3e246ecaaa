"""test_sr.py's four-panel figure (DESIGN.md section 7b) on the CPU: the numpy twins of oracle/figure.py against live cv2 and
against the script's own statements, the oracle against tests/golden/figure.npz, and the ABI of the figure kernel."""
import ctypes
import os
import re

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "figure.npz")


@pytest.fixture(scope="module")
def cv2_no_ipp():
    cv2 = pytest.importorskip("cv2")
    was = cv2.ipp.useIPP()
    cv2.ipp.setUseIPP(False)
    yield cv2
    cv2.ipp.setUseIPP(was)


def test_linear_twin_equals_cv2_on_prior_strips(cv2_no_ipp):
    """cv2.resize(strip, (S, 128)) (INTER_LINEAR, float32) bit for bit: 1 to 70 characters, targets of 1 column, the identity,
    integer factors both ways, non-integer scales and up to 8960 columns."""
    from oracle import figure
    rng = np.random.default_rng(0)
    cases = [(1, 1), (1, 3), (1, 128), (1, 256), (2, 2752), (3, 95), (4, 128), (8, 128), (8, 256), (8, 512), (8, 1024), (8, 1600),
             (8, 800), (8, 676), (16, 1023), (22, 4000), (30, 2752), (30, 3840), (70, 2499), (70, 8960), (70, 1)]
    for n, dw in cases:
        src = rng.uniform(0, 1, (128, 128 * n, 3)).astype(np.float32)
        ref = cv2_no_ipp.resize(src, (dw, 128))
        got = figure.resize_linear_f32(src, dw)
        assert got.dtype == np.float32 and np.array_equal(got, ref), (n, dw, int((got != ref).sum()))


def test_cubic_twin_at_128_rows_equals_cv2(cv2_no_ipp):
    from oracle.image_ops import resize_cubic_u8
    rng = np.random.default_rng(1)
    for h, w in [(32, 256), (40, 1562), (24, 516), (48, 400), (9, 33), (131, 97), (17, 301)]:
        img = rng.integers(0, 256, (h, w, 3), dtype=np.uint8)
        ref = cv2_no_ipp.resize(img, (0, 0), fx=128 / h, fy=128 / h, interpolation=cv2_no_ipp.INTER_CUBIC)
        assert np.array_equal(resize_cubic_u8(img, 128 / h, 128 / h), ref), (h, w)


def _script_show_locs(ShowLQ, preds_locs, n, img_max_width):
    """test_sr.py:214-230, statement for statement (pre_text replaced by its length)."""
    ShowLocs = ShowLQ.copy()
    Locs = preds_locs.clone()
    pad = 2
    padr = 1
    for c in range(n):
        l = c * 2
        center, width = int(Locs[0][l].item()*img_max_width), int(Locs[0][l+1].item()*img_max_width)
        x = center - width
        y = center + width
        ShowLocs[:64, max(0, x-pad):min(x+pad, img_max_width), 0] = ShowLocs[:64, max(0, x-pad):min(x+pad, img_max_width), 0]*0 + 255
        ShowLocs[64:, max(0, y-padr):min(y+padr, img_max_width), 0] = ShowLocs[64:, max(0, y-padr):min(y+padr, img_max_width), 0]*0
        ShowLocs[:64, max(0, x-pad):min(x+pad, img_max_width), 1] = ShowLocs[:64, max(0, x-pad):min(x+pad, img_max_width), 1]*0
        ShowLocs[64:, max(0, y-padr):min(y+padr, img_max_width), 1] = ShowLocs[64:, max(0, y-padr):min(y+padr, img_max_width), 1]*0
        ShowLocs[:64, max(0, x-pad):min(x+pad, img_max_width), 2] = ShowLocs[:64, max(0, x-pad):min(x+pad, img_max_width), 2]*0
        ShowLocs[64:, max(0, y-padr):min(y+padr, img_max_width), 2] = ShowLocs[64:, max(0, y-padr):min(y+padr, img_max_width), 2]*0 + 255
    return ShowLocs


def _random_boxes(rng, h, w):
    n = int(rng.integers(1, 40))
    boxes = []
    for _ in range(n):
        kind = rng.integers(0, 6)
        if kind == 0:
            x1, x2 = 0, int(rng.integers(0, w + 1))                          # touches the left edge
        elif kind == 1:
            x1, x2 = int(rng.integers(0, w + 1)), w                          # touches the right edge
        elif kind == 2:
            x1 = int(rng.integers(0, w)); x2 = x1 + 1                        # 1-px box
        elif kind == 3:
            x1 = int(rng.integers(-3 * h, 0)); x2 = x1 + int(rng.integers(0, 2 * h))     # outside the image: negative stops
        elif kind == 4:
            x1 = int(rng.integers(w, 2 * w + 1)); x2 = x1 + int(rng.integers(0, h))       # beyond the right edge
        else:
            x1 = int(rng.integers(0, w)); x2 = min(w, x1 + int(rng.integers(0, 3 * h)))  # ordinary, often overlapping
        boxes.append([x1, 0, max(x1, x2), h])
    return boxes


def test_marker_intervals_equal_the_script_statements():
    """pipeline.figure_markers (product) and oracle.figure.marker_intervals (twin), painted, equal test_sr.py's own statements on
    a numpy array; lines that fit the canvas (M = 2048) and wider ones (M = 4*Wc, S > M for very short rows too)."""
    import torch
    from marconet_b200 import pipeline
    from oracle import figure
    rng = np.random.default_rng(2)
    for t in range(400):
        h = int(rng.integers(8, 80))
        w = int(rng.integers(h // 2 + 1, 40 * h))
        S, wc = figure.show_width(h, w), figure.canvas_width(h, w)
        M = 4 * wc if t % 5 else int(rng.integers(16, 600))                # and arbitrary M, down to M < S
        boxes = _random_boxes(rng, h, w)
        locs = pipeline.boxes_to_locs(boxes, h, wc)
        assert np.array_equal(locs[0].numpy(), figure.locs_f32(boxes, h, wc))
        base = rng.integers(0, 256, (128, S, 3), dtype=np.uint8)
        ref = _script_show_locs(base, locs, len(boxes), M)
        twin = figure.marker_intervals(locs[0].numpy(), S, M)
        prod = pipeline.figure_markers(locs[0].tolist(), S, M)
        assert prod == twin
        assert np.array_equal(figure.show_locs(base, *twin), ref), (h, w, M, boxes)
        assert all(0 <= a < b <= S for a, b in twin[0] + twin[1])


def test_oracle_reproduces_the_figure_fixture(checkpoints):
    """oracle/restate.py nets + oracle/figure.py twins reproduce every byte of tests/golden/figure.npz: (a) the PNGs the
    UNMODIFIED test_sr.py wrote, (b) the prior panel of a line wider than the canvas."""
    import torch
    from marconet_b200 import pipeline
    from oracle import figure, image_ops, restate
    g = np.load(GOLDEN)
    stride, rows = int(g["stride"]), int(g["prior_rows"])
    for i in range(int(g["lines"])):
        img, boxes, labels = g[f"image{i}"], g[f"boxes{i}"].tolist(), g[f"labels{i}"]
        h = img.shape[0]
        lq, _ = image_ops.preprocess_lq(img)
        lq_t = torch.from_numpy(lq)
        _, _, w = restate.encoder_forward(checkpoints["encoder"], lq_t)
        lab = torch.from_numpy(labels).reshape(-1, 1)
        prior, f64, f32_ = restate.tspgan_forward(checkpoints["tspgan"], w[:1].repeat(lab.shape[0], 1), lab)
        sr = restate.tspsr_forward(checkpoints["sr"], lq_t, [f64], [f32_], pipeline.boxes_to_locs(boxes, h, 512))
        S = figure.show_width(h, img.shape[1])
        fig = figure.figure_bytes(img, boxes, prior.numpy(), image_ops.postprocess_sr(sr.numpy())[0, :, :S])
        assert fig.shape == (512, S, 3)
        assert np.array_equal(fig[:256], g[f"show{i}"]), (i, int((fig[:256] != g[f"show{i}"]).sum()))
        assert np.array_equal(fig[256:384][::stride, ::stride], g[f"sr_row{i}"]), i
        assert np.array_equal(fig[384::rows], g[f"prior_row{i}"]), (i, int((fig[384::rows] != g[f"prior_row{i}"]).sum()))
    img, labels, owner = g["wide_image"], g["wide_labels"], g["wide_owner"]
    S, W, wc, M = g["wide_geometry"].tolist()
    styles = []
    for a, b in g["wide_crops"].tolist():
        lq, _ = image_ops.preprocess_lq(np.ascontiguousarray(img[:, a:b]))
        styles.append(restate.encoder_forward(checkpoints["encoder"], torch.from_numpy(lq))[2][:1])
    style = torch.cat([styles[k] for k in owner.tolist()], dim=0)
    prior, _, _ = restate.tspgan_forward(checkpoints["tspgan"], style, torch.from_numpy(labels).reshape(-1, 1))
    assert (S, W, wc) == (figure.show_width(*img.shape[:2]), W, figure.canvas_width(*img.shape[:2]))
    assert np.array_equal(figure.prior_panel(prior.numpy(), S)[::rows, :W], g["wide_prior_row"])


def _fields(header, name):
    body = re.search(r"typedef struct \{([^{}]*)\}\s*" + name + ";", header).group(1)
    body = re.sub(r"/\*.*?\*/", "", body, flags=re.S)
    names = []
    for decl in body.split(";"):
        parts = [p.strip() for p in decl.strip().split(",") if p.strip()]
        names += [re.findall(r"[A-Za-z_0-9]+$", p)[0] for p in parts]
    return names


@pytest.mark.parametrize("c_name,py_name,size,offsets", [
    ("mn_figure_image", "FigureImage", 80, dict(img=0, row_pitch=8, fig=16, fig_pitch=24, marks=32, priors=40, h=48, n_chars=72)),
    ("mn_figure_prior", "FigurePrior", 32, dict(img=0, stride_c=8, stride_h=16, stride_w=24))])
def test_figure_descriptors_match_header(c_name, py_name, size, offsets):
    from marconet_b200 import _lib
    header = open(os.path.join(ROOT, "include", "marconet_b200.h")).read()
    cls = getattr(_lib, py_name)
    assert _fields(header, c_name) == [f[0] for f in cls._fields_]
    assert ctypes.sizeof(cls) == size
    for name, off in offsets.items():
        assert getattr(cls, name).offset == off, name
    assert "int mn_figure_u8(const mn_figure_image* images, int n_images, int max_width, void* stream);" in header
    assert "mn_figure_u8" in _lib.SYMBOLS


def test_figure_kernel_builds_without_spills(tmp_path):
    import subprocess
    from marconet_b200 import build
    src = os.path.join(ROOT, "marconet_b200", "csrc", "image_ops.cu")
    r = subprocess.run([build.nvcc_path(), "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-DMN_BUILD", "-Xptxas", "-v",
                        "-cubin", src, "-o", str(tmp_path / "image_ops.cubin")], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-2000:]
    props = re.search(r"figure_kernel[^\n]*\n[^\n]*Function properties for [^\n]*figure_kernel[^\n]*\n([^\n]*)", r.stderr)
    assert props, "no ptxas report for figure_kernel"
    assert "0 bytes spill stores, 0 bytes spill loads" in props.group(1), props.group(1)
