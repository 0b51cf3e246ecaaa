"""Predicted characters without a GPU: the detection windows (pipeline.plan_windows), the host merge against the numpy twin
(oracle/predict.py) on planted encoder outputs, the twin against tests/golden/predict.npz (the reference encoder and the
reference's own clear_labels), and the new kernel's ABI and register use."""
import ctypes
import math
import os
import re
import subprocess

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "predict.npz")


def _sizes():
    rng = np.random.default_rng(7)
    out = [(1, 1), (1, 15), (1, 16), (1, 17), (1, 400), (32, 512), (32, 513), (32, 6000), (40, 2000), (3, 95), (7, 2300)]
    for _ in range(300):
        h = int(rng.integers(1, 200))
        out.append((h, int(rng.integers(1, 25 * 16 * h))))
    return out


@pytest.mark.parametrize("overlap", [0, 64, 256])
def test_plan_windows_cover_fit_and_overlap(overlap):
    from marconet_b200 import ops, pipeline
    from oracle import predict
    counts = set()
    for h, w in _sizes():
        wins = pipeline.plan_windows(h, w, overlap=overlap)
        assert [(tuple(x.crop), tuple(x.core)) for x in wins] == predict.plan_windows(h, w, overlap=overlap), (h, w)
        counts.add(len(wins))
        if ops.round_half_even(w * (32 / h)) <= 512:
            assert [tuple(x) for x in wins] == [((0, w), (-math.inf, math.inf))]
            continue
        v = math.ceil(overlap * h / 32)
        assert wins[0].crop[0] == 0 and wins[-1].crop[1] == w
        assert wins[0].core[0] == -math.inf and wins[-1].core[1] == math.inf
        for k, x in enumerate(wins):
            a, b = x.crop
            assert 0 <= a < b <= w
            assert 1 <= ops.round_half_even((b - a) * (32 / h)) <= 512 and ops.round_half_even(h * (32 / h)) == 32
            if k + 1 < len(wins):
                nxt = wins[k + 1]
                assert b - nxt.crop[0] >= v and nxt.crop[0] > a, (h, w, k)
                assert x.core[1] == nxt.core[0]
                assert nxt.crop[0] <= x.core[1] <= b, (h, w, k)
    assert 1 in counts and max(counts) > 20


@pytest.mark.parametrize("overlap", [-1, 257, 1000])
def test_plan_windows_rejects_overlap_outside_range(overlap):
    from marconet_b200 import pipeline
    with pytest.raises(ValueError):
        pipeline.plan_windows(32, 2000, overlap=overlap)


@pytest.mark.parametrize("h,w,seed", [(32, 400, 0), (32, 3000, 1), (64, 9000, 2), (16, 513, 3), (32, 11000, 4)])
def test_host_merge_equals_oracle_on_planted_outputs(h, w, seed):
    from marconet_b200 import pipeline
    from oracle import predict
    logits, locs = predict.planted_image(seed, h, w)
    labels, boxes, rows = predict.predict(h, w, logits, locs)
    wins = pipeline.plan_windows(h, w)
    got = pipeline.merge_predictions(h, w, wins, [r[:3] for r in rows])
    assert got == (labels, boxes)
    for k in range(len(wins)):                            # the decode is test_w.py's (pipeline.decode_labels) capped at 16
        assert rows[k][3] == len(pipeline.decode_labels(torch.from_numpy(logits[k]))[:16])
    centres = [(b[0] + b[2]) / 2.0 for b in boxes]
    assert centres == sorted(centres)
    assert all(0 <= b[0] <= b[2] <= w and b[1] == 0 and b[3] == h for b in boxes)
    if len(wins) > 1:                                      # planted centres on every core boundary: owned by the right window
        def on(j, x):
            return sum(1 for x1, x2 in zip(rows[j][1], rows[j][2]) if (x1 + x2) * 0.5 == x)
        assert sum(on(j, wins[j].core[0]) for j in range(len(wins))) >= 1
        assert sum(on(j, wins[j].core[1]) for j in range(len(wins))) == 0


def test_oracle_reproduces_golden_predictions():
    from oracle import predict, restate
    g = np.load(GOLDEN)
    for name in ("fit", "wide"):
        img = g[f"{name}_image"]
        h, w = img.shape[:2]
        wins = predict.plan_windows(h, w)
        assert np.array_equal(g[f"{name}_crops"], np.asarray([c for c, _ in wins]))
        argmax, locs = g[f"{name}_argmax"], g[f"{name}_locs_lr"]
        assert g[f"{name}_margin"].min() >= 5e-3
        rows = []
        for k, ((a, _), (lo, hi)) in enumerate(wins):
            onehot = np.zeros((argmax.shape[1], 6736), np.float32)    # a logits row whose argmax is the reference's
            onehot[np.arange(argmax.shape[1]), argmax[k]] = 1.0
            r = predict.decode_row(onehot, locs[k], a, 16.0 * h, lo, hi)
            ref = g[f"{name}_ref_labels_{k}"].tolist()
            assert restate.clear_labels(torch.from_numpy(onehot)) == ref and r[3] == len(ref[:16])
            rows.append(r[:3])
        labels, boxes = predict.merge(h, w, rows)
        assert labels == g[f"{name}_labels"].tolist()
        assert np.array_equal(np.asarray(boxes, np.float64).reshape(-1, 4), g[f"{name}_boxes"])


def _fields(header, name):
    body = re.search(r"typedef struct \{([^{}]*)\}\s*" + name + ";", header).group(1)
    body = re.sub(r"/\*.*?\*/", "", body, flags=re.S)
    names = []
    for decl in body.split(";"):
        parts = [p.strip() for p in decl.strip().split(",") if p.strip()]
        names += [re.findall(r"([A-Za-z_0-9]+)(?:\[[A-Z_0-9]+\])?$", p)[0] for p in parts]
    return names


@pytest.mark.parametrize("c_name,py_name,size", [("mn_char_pred", "CharPred", 328), ("mn_pred_row", "PredRow", 40)])
def test_prediction_structs_match_header(c_name, py_name, size):
    from marconet_b200 import _lib, ops
    header = open(os.path.join(ROOT, "include", "marconet_b200.h")).read()
    cls = getattr(_lib, py_name)
    assert _fields(header, c_name) == [f[0] for f in cls._fields_]
    assert ctypes.sizeof(cls) == size
    assert int(re.search(r"#define MN_PRED_SLOTS (\d+)", header).group(1)) == _lib.PRED_SLOTS
    if py_name == "CharPred":
        dt = ops.pred_dtype()
        assert dt.itemsize == size and [dt.fields[f[0]][1] for f in cls._fields_] == [getattr(cls, f[0]).offset for f in cls._fields_]


def test_decode_kernel_builds_without_spills(tmp_path):
    from marconet_b200 import build
    src = os.path.join(ROOT, "marconet_b200", "csrc", "predict_ops.cu")
    r = subprocess.run([build.nvcc_path(), "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-DMN_BUILD", "-Xptxas", "-v",
                        "-cubin", src, "-o", str(tmp_path / "predict_ops.cubin")], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-2000:]
    kernel = "decode_predictions_kernel"
    props = re.search(kernel + r"[^\n]*\n[^\n]*Function properties for [^\n]*" + kernel + r"[^\n]*\n([^\n]*)", r.stderr)
    assert props, f"no ptxas report for {kernel}"
    assert "0 bytes spill stores, 0 bytes spill loads" in props.group(1), props.group(1)
