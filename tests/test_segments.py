"""Segment planner of pipeline.restore_images (pipeline.plan_segments / stitch_pieces): invariants on random box sets, the
single-segment rule, the errors, and the plan and bytes of tests/golden/wide_line.npz (oracle/make_golden_wide_line.py)."""
import math
import os

import numpy as np
import pytest

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "wide_line.npz")


def _random_line(rng):
    """A random line in reading order: widths / gaps drawn in LQ pixels, some gaps negative (overlapping boxes), some wider
    than the canvas."""
    h = int(rng.integers(4, 201))
    s = h / 32
    n = int(rng.integers(0, 60))
    boxes, x = [], float(rng.integers(0, 40)) * s
    for _ in range(n):
        cw = float(rng.uniform(0, 60)) * s
        if rng.random() < 0.05:
            cw = 0.0
        boxes.append([round(x, 2), 0, round(x + cw, 2), h])
        g = rng.choice([rng.uniform(-8, 0), rng.uniform(0, 20), rng.uniform(400, 900)], p=[0.1, 0.85, 0.05])
        x = max(x + cw + float(g) * s, x + cw / 2 + 0.01)          # keeps the centres increasing
    w = max(1, int(math.ceil(x + float(rng.integers(0, 40)) * s)))
    boxes = [b for b in boxes if b[2] <= w]
    return h, w, boxes


def _check_plan(h, w, boxes, segs, context=16):
    from marconet_b200 import pipeline
    fits = round(w * (32 / h)) <= 512
    assert (len(segs) == 1) == fits
    cuts = [s.core[0] for s in segs] + [segs[-1].core[1]]
    assert cuts[0] == 0 and cuts[-1] == w and all(a < b for a, b in zip(cuts, cuts[1:]))
    assert all(s.core == (cuts[k], cuts[k + 1]) for k, s in enumerate(segs))
    spans = [(math.floor(b[0]), math.ceil(b[2])) for b in boxes]
    for c in cuts:
        assert not any(s < c < e for s, e in spans), (c, [sp for sp in spans if sp[0] < c < sp[1]])
    m = -(-context * h // 32)
    if fits:
        assert segs[0].crop == (0, w) and segs[0].chars == (0, len(boxes))
    else:
        for s in segs:
            assert s.crop == (max(0, s.core[0] - m), min(w, s.core[1] + m))
            assert (s.crop[1] - s.crop[0]) * 32 / h <= 511.5
            assert round((s.crop[1] - s.crop[0]) * (32 / h)) <= 512
    # ownership: consecutive ranges covering every character, each inside its segment's core
    assert segs[0].chars[0] == 0 and segs[-1].chars[1] == len(boxes)
    assert all(a.chars[1] == b.chars[0] for a, b in zip(segs, segs[1:]))
    for s in segs:
        for j in range(*s.chars):
            sp = spans[j]
            assert sp[0] == sp[1] or s.core[0] <= sp[0] and sp[1] <= s.core[1], (j, sp, s.core)
        assert [[b[0] - s.crop[0], b[1], b[2] - s.crop[0], b[3]] for b in boxes[s.chars[0]:s.chars[1]]] == s.boxes
    # stitch: the pieces tile the output and read inside the 2048-column SR output
    width, pieces = pipeline.stitch_pieces(h, w, segs)
    assert width == (min(round(w * (128 / h)), 2048) if fits else round(w * (128 / h)))
    x = 0
    for k, o0, src, wd in pieces:
        assert o0 == x and wd > 0 and 0 <= src and src + wd <= 2048, (k, o0, src, wd)
        x += wd
    assert x == width


def test_planner_invariants_on_random_box_sets():
    from marconet_b200 import pipeline
    rng = np.random.default_rng(2024)
    done = multi = empty = 0
    while done < 1200:
        h, w, boxes = _random_line(rng)
        try:
            segs = pipeline.plan_segments(h, w, boxes)
        except ValueError as e:
            assert "wider than the" in str(e), e
            continue
        _check_plan(h, w, boxes, segs)
        done += 1
        multi += len(segs) > 1
        empty += any(s.chars[0] == s.chars[1] for s in segs) and len(segs) > 1
    assert multi > 300 and empty > 20, (multi, empty)


def test_single_segment_for_every_image_that_fits():
    from marconet_b200 import pipeline
    for h in (1, 7, 12, 17, 22, 32, 40, 49, 128, 200):
        w_max = max(w for w in range(1, 40 * h) if round(w * (32 / h)) <= 512)
        for w in sorted({1, w_max // 2, w_max}):
            boxes = [[0, 0, w / 2, h], [w / 2, 0, w, h]]
            segs = pipeline.plan_segments(h, w, boxes)
            assert segs == [pipeline.Segment((0, w), (0, w), (0, 2), [list(b) for b in boxes])]
        assert len(pipeline.plan_segments(h, w_max + 1, [])) > 1


def test_planner_errors_name_the_image_and_character():
    from marconet_b200 import pipeline
    with pytest.raises(ValueError, match=r"line 3, character 1: .* wider than the 512-pixel"):
        pipeline.plan_segments(32, 2000, [[0, 0, 20, 32], [100, 0, 620, 32]], name="line 3")
    with pytest.raises(ValueError, match=r"characters 1 to 2 \(overlapping"):
        pipeline.plan_segments(32, 2000, [[0, 0, 20, 32], [100, 0, 400, 32], [390, 0, 620, 32]])
    with pytest.raises(ValueError, match=r"image, character 2: box centre .* reading order"):
        pipeline.plan_segments(32, 300, [[0, 0, 20, 32], [30, 0, 50, 32], [10, 0, 20, 32]])
    with pytest.raises(ValueError, match=r"3 labels for 2 boxes"):
        pipeline.plan_segments(32, 300, [[0, 0, 20, 32], [30, 0, 50, 32]], labels=[1, 2, 3])
    for bad in ([-1, 0, 20, 32], [280, 0, 301, 32], [50, 0, 40, 32]):
        with pytest.raises(ValueError, match=r"character 1: box .* outside the image"):
            pipeline.plan_segments(32, 300, [[0, 0, 20, 32], bad])


def test_wide_line_plan_is_reproduced():
    from marconet_b200 import pipeline
    g = np.load(GOLDEN)
    img, boxes = g["image"], g["boxes"].tolist()
    segs = pipeline.plan_segments(img.shape[0], img.shape[1], boxes, labels=g["labels"].tolist())
    assert [s.core[0] for s in segs] + [img.shape[1]] == g["cuts"].tolist()
    assert [list(s.crop) for s in segs] == g["crops"].tolist()
    assert [list(s.chars) for s in segs] == g["chars"].tolist()
    lq_w = round(img.shape[1] * 32 / img.shape[0])
    assert 1100 <= lq_w <= 1300 and 20 <= len(boxes) <= 24
    assert any(a == b for a, b in g["chars"].tolist()), "the fixture pins a segment without characters"
    _check_plan(img.shape[0], img.shape[1], boxes, segs)


def test_oracle_reproduces_the_wide_line_fixture(checkpoints):
    """Crop by crop through the oracle (oracle/wide_line, oracle/image_ops, oracle/restate) and the numpy stitch: byte for byte the stitched SR
    bytes of the reference modules running test_sr.py's data flow on each crop (oracle/make_golden_wide_line.py)."""
    import torch
    from marconet_b200 import pipeline
    from oracle import image_ops, restate, wide_line
    g = np.load(GOLDEN)
    img, boxes, labels, stride = g["image"], g["boxes"].tolist(), g["labels"], int(g["stride"])
    h, w = img.shape[:2]
    srs = []
    for (a, b), (i0, i1) in zip(g["crops"].tolist(), g["chars"].tolist()):
        lq, _ = wide_line.preprocess_lq_crop(img, a, b)
        lq_t = torch.from_numpy(lq)
        _, _, st = restate.encoder_forward(checkpoints["encoder"], lq_t)
        p64, p32 = [], []
        if i1 > i0:
            shifted = [[x1 - a, y1, x2 - a, y2] for x1, y1, x2, y2 in boxes[i0:i1]]
            locs = pipeline.boxes_to_locs(shifted, h, 512)
            lab = torch.from_numpy(labels[i0:i1]).reshape(-1, 1)
            _, f64, f32_ = restate.tspgan_forward(checkpoints["tspgan"], st[:1].repeat(i1 - i0, 1), lab)
            p64, p32 = [f64], [f32_]
        else:
            locs = torch.zeros(1, 0)
        sr = restate.tspsr_forward(checkpoints["sr"], lq_t, p64, p32, locs)
        srs.append(image_ops.postprocess_sr(sr.numpy())[0])
    line = wide_line.stitch_sr(h, w, g["cuts"].tolist(), g["crops"].tolist(), srs)
    assert np.array_equal(line[::stride, ::stride], g["sr_line"])
