"""Batch planner of pipeline.restore_images (pipeline.plan_batches), on the host: which lines share a batch, in which order, the
characters, styles, locs, stitch pieces and figures of each batch, in crop mode and with whole_lines."""
import numpy as np
import pytest
import torch

SIZES = [(22, 181), (12, 108), (17, 49), (20, 112), (17, 86), (15, 61), (14, 47), (12, 52), (49, 304), (14, 45), (14, 44),
         (15, 55), (32, 388), (128, 1472), (128, 1268), (128, 1160), (128, 1856),
         (32, 1100), (40, 1920), (24, 1530), (64, 2600)]             # the last four: 2-4 canvases wide


def _image_set(n, seed):
    """(shapes, labels, boxes, plans) of n lines cycling through SIZES, one box per 28 LQ pixels; every 5th line has a gap wider
    than the canvas after its first box (crops without characters) and every 7th is left out (an invalid entry)."""
    from marconet_b200 import pipeline
    rng = np.random.default_rng(seed)
    shapes, labels, boxes, plans = [], [], [], []
    for i in range(n):
        h, w = SIZES[(i + seed) % len(SIZES)]
        pitch = 28 * h / 32
        k = max(1, int(w // pitch))
        xs = [j * pitch for j in range(k)]
        if i % 5 == 4:
            gap = 1200 * h / 32
            xs = xs[:1] + [x + gap for x in xs[1:]]
            w = int(xs[-1] + pitch) + 1
        bx = [[int(x + 0.15 * pitch), 0, int(x + 0.85 * pitch), h] for x in xs]
        shapes.append((h, w))
        labels.append(rng.integers(0, 6735, k).tolist())
        boxes.append(bx)
        plans.append(None if i % 7 == 6 else pipeline.plan_segments(h, w, bx))
    return shapes, labels, boxes, plans


def _lines(shapes, plans, whole_lines):
    """Expected decoder lines in order: (image, x0, x1, width, its segments)."""
    from marconet_b200 import pipeline
    out = []
    for i, segs in enumerate(plans):
        if segs is None:
            continue
        wc = pipeline.whole_line_width(*shapes[i])[1]
        if whole_lines and wc > 512:
            out.append((i, 0, shapes[i][1], wc, segs))
        else:
            out += [(i, *s.crop, 512, [s]) for s in segs]
    return out


@pytest.mark.parametrize("whole_lines", [False, True])
@pytest.mark.parametrize("max_lines", [1, 3, 8])
@pytest.mark.parametrize("seed", [0, 1])
def test_plan_batches(seed, max_lines, whole_lines):
    from marconet_b200 import ops, pipeline
    shapes, labels, boxes, plans = _image_set(42, seed)
    out_w, batches = pipeline.plan_batches(shapes, labels, boxes, plans, max_lines, whole_lines)
    lines = _lines(shapes, plans, whole_lines)
    valid = [i for i, p in enumerate(plans) if p is not None]
    assert any(len(plans[i]) > 1 for i in valid) and any(s.chars[0] == s.chars[1] for i in valid for s in plans[i])

    # which lines share a batch, in which order
    if whole_lines:
        groups = pipeline.pack_by_columns([pipeline.whole_line_width(*shapes[i])[1] for i in valid], max_lines)
    else:
        groups = [list(range(b0, min(b0 + max_lines, len(lines)))) for b0 in range(0, len(lines), max_lines)]
    assert len(batches) == len(groups)
    for bt, g in zip(batches, groups):
        assert bt.lines == [lines[j][:3] for j in g] and bt.widths == [lines[j][3] for j in g]
        assert bt.crops == [(lines[j][0], *s.crop) for j in g for s in lines[j][4]]
        assert bt.reuse == all(w == 512 for w in bt.widths)
        if not whole_lines:
            assert bt.reuse

    # output widths
    for i in valid:
        h, w = shapes[i]
        wc = pipeline.whole_line_width(h, w)[1]
        want = pipeline.stitch_pieces(h, w, plans[i])[0] if not (whole_lines and wc > 512) else \
            min(ops.round_half_even(w * 128 / h), 4 * wc)
        assert out_w[i] == want
    assert list(out_w) == valid

    # every character once, in label order, styled by the crop whose segment owns it; locs of each line
    nxt = dict.fromkeys(valid, 0)
    cover = {i: np.zeros(out_w[i], int) for i in valid}
    last, done = {}, {}
    for b_idx, bt in enumerate(batches):
        assert len(bt.counts) == len(bt.lines) and sum(bt.counts) == len(bt.labels) == len(bt.owner)
        assert bt.locs.dtype == torch.float32 and tuple(bt.locs.shape) == (len(bt.lines), 2 * max(1, max(bt.counts)))
        j = 0
        for b, ((i, x0, x1), width, n) in enumerate(zip(bt.lines, bt.widths, bt.counts)):
            last[i] = b_idx
            chars = range(nxt[i], nxt[i] + n)
            nxt[i] += n
            assert bt.labels[j:j + n] == labels[i][chars.start:chars.stop]
            for c in chars:
                seg = next(s for s in plans[i] if s.chars[0] <= c < s.chars[1])
                assert bt.crops[bt.owner[j]] == (i, *seg.crop), (i, c)
                j += 1
            h = shapes[i][0]
            ref = torch.zeros(bt.locs.shape[1])
            if n:
                line_boxes = [[bx[0] - x0, bx[1], bx[2] - x0, bx[3]] for bx in boxes[i][chars.start:chars.stop]]
                ref[:2 * n] = pipeline.boxes_to_locs(line_boxes, h, width)[0]
            assert torch.equal(bt.locs[b], ref), (b_idx, b)
        for line, src, i, o0, width in bt.pieces:
            assert bt.lines[line][0] == i and 0 <= src and src + width <= 4 * bt.widths[line] and width > 0
            cover[i][o0:o0 + width] += 1
        for i in bt.done:
            assert i not in done
            done[i] = b_idx
    assert nxt == {i: len(labels[i]) for i in valid}
    for i in valid:
        assert (cover[i] == 1).all(), i
    assert done == last
    for b_idx, bt in enumerate(batches):      # figure items in the order the images first appear in the batch
        assert bt.done == [i for i in dict.fromkeys(i for i, _, _ in bt.lines) if last[i] == b_idx]
