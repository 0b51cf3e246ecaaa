"""Font-style interpolation on the host (pipeline.interpolate_styles; DESIGN.md section 7b): the numpy twin (oracle/styles.py)
against torch and tests/golden/style_wide.npz, the C records against the header, the sweep plan and argument validation."""
import ctypes
import os
import re

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")
SCRIPT_SCALES = [i / 10 for i in range(11)]


def test_twin_lerp_equals_torch_bit_for_bit():
    """fl(fl(w1*s32) + fl(w2*t32)) equals torch's fp32 ``w1 * s + w2 * (1 - s)`` (test_w.py:107) on random rows, for the 11
    scales of the script and 50 random ones."""
    from oracle import styles
    g = torch.Generator().manual_seed(0)
    w1, w2 = torch.randn(64, 512, generator=g) * 3, torch.randn(64, 512, generator=g) * 3
    rng = np.random.default_rng(0)
    for s in SCRIPT_SCALES + [float(v) for v in rng.uniform(-2, 3, 50)]:
        ref = (w1 * s + w2 * (1 - s)).numpy()
        assert styles.lerp(w1.numpy(), w2.numpy(), s).tobytes() == ref.tobytes(), s


def _header_fields(name):
    header = open(os.path.join(ROOT, "include", "marconet_b200.h")).read()
    body = re.sub(r"/\*.*?\*/", "", header.split(f"}} {name};")[0].rsplit("typedef struct {", 1)[1], flags=re.S)
    names = []
    for decl in filter(None, (d.strip() for d in body.split(";"))):
        parts = [p.strip() for p in decl.split(",")]
        names += [re.findall(r"([A-Za-z_0-9]+)(?:\[[A-Z_0-9]+\])?$", p)[0] for p in parts]
    return names


def test_record_layouts_match_the_header():
    from marconet_b200 import _lib, ops
    for name, cls, size in (("mn_label_row", _lib.LabelRow, 4 + 4 * 64), ("mn_lerp_row", _lib.LerpRow, 16),
                            ("mn_prior_tile", _lib.PriorTile, 16)):
        assert _header_fields(name) == [f[0] for f in cls._fields_], name
        assert ctypes.sizeof(cls) == size, name
    assert ops.label_dtype().itemsize == ctypes.sizeof(_lib.LabelRow)
    assert "#define MN_LABEL_SLOTS 64" in open(os.path.join(ROOT, "include", "marconet_b200.h")).read()
    rec = np.frombuffer(ops.lerp_rows([(2, 5, 0.3), (0, 1, 1.0)], 6), dtype=np.dtype([("w1", "<i4"), ("w2", "<i4"), ("s", "<f4"),
                                                                                       ("t", "<f4")]))
    assert rec.tolist() == [(2, 5, np.float32(0.3), np.float32(1 - 0.3)), (0, 1, 1.0, 0.0)]
    with pytest.raises(ValueError):
        ops.lerp_rows([(6, 0, 0.5)], 6)
    with pytest.raises(ValueError):
        ops.lerp_rows([(0, 0, float("nan"))], 6)


@pytest.mark.parametrize("max_chars", [1, 7, 128])
def test_sweep_rows_order_and_chunking(max_chars):
    """Rows in (pair, scale, character) order, each character with its own style row and label and its pair's donor; pairs left
    out contribute nothing; chunks are consecutive, at most max_chars long, and cover every row once."""
    from marconet_b200 import pipeline
    rng = np.random.default_rng(max_chars)
    chars, donors = [], []
    for p in range(6):
        if p == 2:
            chars.append(None)
            donors.append(None)
            continue
        n = int(rng.integers(1, 40))
        chars.append([(int(rng.integers(0, 9)), int(rng.integers(0, 6735))) for _ in range(n)])
        donors.append(10 + p)
    n_scales = 5
    rows, chunks = pipeline.plan_sweep(chars, donors, n_scales, max_chars)
    want = [(p, k, c, w1, donors[p], lab) for p in range(6) if chars[p] for k in range(n_scales) for c, (w1, lab) in enumerate(chars[p])]
    assert [tuple(r) for r in rows] == want
    assert chunks[0][0] == 0 and chunks[-1][1] == len(rows)
    assert all(a[1] == b[0] for a, b in zip(chunks, chunks[1:]))
    assert all(0 < r1 - r0 <= max_chars for r0, r1 in chunks)
    assert len(chunks) == -(-len(rows) // max_chars)


class _CpuEncoder(torch.nn.Module):
    def __init__(self):
        super().__init__()
        self.p = torch.nn.Parameter(torch.zeros(1))

    def forward(self, lq):
        raise AssertionError("the encoder ran")


def test_validation_errors_with_and_without_skip_invalid():
    """Bad arguments raise before any launch; an invalid pair (malformed image, donor wider than the canvas) raises a ValueError
    naming it, or becomes an error entry with skip_invalid."""
    from marconet_b200 import pipeline
    enc = _CpuEncoder()
    ok = np.zeros((32, 200, 3), np.uint8)
    for kw, msg in ((dict(max_lines=0), "max_lines"), (dict(max_chars=0), "max_chars"), (dict(overlap=-1), "overlap"),
                    (dict(overlap=257), "overlap"), (dict(scales=()), "scales"), (dict(scales=(0.5, float("nan"))), "scales"),
                    (dict(scales=(0.5, float("inf"))), "scales"), (dict(scales=(True,)), "scales"), (dict(scales=("0.5",)), "scales")):
        with pytest.raises(ValueError, match=msg):
            pipeline.interpolate_styles(enc, None, [(ok, ok)], **kw)
    bad = [
        ((ok, np.zeros((32, 600, 3), np.uint8)), "donor's LQ width 600"),
        ((ok, np.zeros((10, 161, 3), np.uint8)), "donor's LQ width 515"),
        ((np.zeros((32, 200), np.uint8), ok), "content is not"),
        ((ok, np.zeros((32, 200, 3), np.float32)), "donor is not"),
        ((ok, np.zeros((0, 200, 3), np.uint8)), "donor is not"),
        ((ok, "image"), "donor is not"),
        ((ok,), "pair"),
        (ok, "pair"),
    ]
    for pair, msg in bad:
        with pytest.raises(ValueError, match=f"pair 1.*{msg}" if msg != "pair" else "pair 1"):
            pipeline.interpolate_styles(enc, None, [(ok, ok), pair])
    out = pipeline.interpolate_styles(enc, None, [p for p, _ in bad], skip_invalid=True)
    assert len(out) == len(bad)
    for i, (r, (_, msg)) in enumerate(zip(out, bad)):
        assert set(r) == {"error"} and r["error"].startswith(f"ValueError: pair {i}") and msg.split(".")[0] in r["error"], r
    assert pipeline.interpolate_styles(enc, None, []) == []


def test_twin_reproduces_the_wide_fixture():
    """style_wide.npz (the reference modules on a three-window content line): the twin's lerp of the stored w rows gives the
    reference's styles bit for bit, its strip of the stored prior samples gives the stored PNG samples, and the merged labels and
    windows are oracle/predict.py's on predict.npz."""
    from oracle import predict, styles
    g = np.load(os.path.join(GOLDEN, "style_wide.npz"))
    p = np.load(os.path.join(GOLDEN, "predict.npz"))
    w_rows, k_win = g["w_rows"], g["w_rows"].shape[0] - 1
    assert g["labels"].tolist() == p["wide_labels"].tolist() and len(g["labels"]) == 48
    for si, s in enumerate(g["scales"].tolist()):
        for k in range(k_win):
            assert styles.lerp(w_rows[k], w_rows[-1], s).tobytes() == g["styles"][si, k].tobytes(), (s, k)
        ry, rx = int(g["py"]) // int(g["sy"]), int(g["px"]) // int(g["sx"])
        assert np.array_equal(styles.strip(g["priors"][si]), g["strips"][si][::ry, ::rx]), s
    h, w = p["wide_image"].shape[:2]
    wins = predict.plan_windows(h, w)
    rows = [predict.decode_row(_onehot(p["wide_argmax"][k]), p["wide_locs_lr"][k], a, 16.0 * h, lo, hi)[:3]
            for k, ((a, _), (lo, hi)) in enumerate(wins)]
    labels, owners = styles.merge_with_windows(h, w, rows)
    assert labels == g["labels"].tolist() and [list(o) for o in owners] == g["owners"].tolist()
    assert [k for k, _ in owners] == sorted(k for k, _ in owners)


def _onehot(argmax, c=6736):
    lg = np.zeros((len(argmax), c), np.float32)
    lg[np.arange(len(argmax)), argmax] = 1.0
    return lg
