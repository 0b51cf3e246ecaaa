"""numpy twin of the predicted-characters stage (DESIGN.md section 7b, "Predicted characters"): the detection windows
(pipeline.plan_windows), the per-window decode of mn_decode_predictions (labels from restate.clear_labels, the reference's
test_w.py:34-40; the fp32 centre / half-width of tspgan_model.py:331-337; the fp64 box arithmetic as Python floats, which are
IEEE doubles with every operation rounded on its own) with the core test, and the merge of one image's windows.
TEST INFRASTRUCTURE ONLY."""
import math

import numpy as np
import torch

from . import restate

SLOTS = 16


def plan_windows(h, w, canvas=512, overlap=64):
    """[(crop (a, b), core (lo, hi))] of an h x w line."""
    lq_w = int(round(w * (32 / h)))         # cv2's dsize for fx = 32/h
    if lq_w <= canvas:
        return [((0, w), (-math.inf, math.inf))]
    wmax = (2 * canvas - 1) * h // 64
    v = math.ceil(overlap * h / 32)
    s = wmax - v
    k = 1 + math.ceil((w - wmax) / s)
    crops = [(j * s, j * s + wmax) for j in range(k - 1)] + [(w - wmax, w)]
    bounds = [-math.inf] + [math.floor((crops[j + 1][0] + crops[j][1]) / 2) for j in range(k - 1)] + [math.inf]
    return [(crops[j], (bounds[j], bounds[j + 1])) for j in range(k)]


def decode_row(logits, locs_lr, a, scale, lo, hi):
    """One window row: logits fp32 [T, C], locs_lr fp32 [32] -> (labels, x1s, x2s, n_decoded), the characters kept by the core."""
    labels = restate.clear_labels(torch.from_numpy(np.ascontiguousarray(logits, np.float32)))[:SLOTS]
    lr = np.asarray(locs_lr, np.float32)
    out = ([], [], [])
    for j, lab in enumerate(labels):
        l, r = lr[2 * j], lr[2 * j + 1]
        c, hw = np.float32((r + l) / np.float32(2)), np.float32((r - l) / np.float32(2))
        x1 = float(a) + (float(c) - float(hw)) * float(scale)
        x2 = float(a) + (float(c) + float(hw)) * float(scale)
        ctr = (x1 + x2) * 0.5
        if lo <= ctr < hi:
            for o, v in zip(out, (int(lab), x1, x2)):
                o.append(v)
    return out + (len(labels),)


def merge(h, w, rows):
    """rows: per window, (labels, x1s, x2s) -> (labels, boxes [lo, 0, hi, h]): window order, clamped, stable-sorted by centre."""
    pairs = []
    for labs, x1s, x2s in rows:
        for lab, x1, x2 in zip(labs, x1s, x2s):
            lo = min(max(min(x1, x2), 0.0), float(w))
            hi = min(max(max(x1, x2), 0.0), float(w))
            pairs.append((lab, [lo, 0, hi, h]))
    order = sorted(range(len(pairs)), key=lambda k: ((pairs[k][1][0] + pairs[k][1][2]) / 2.0, k))
    return [pairs[k][0] for k in order], [pairs[k][1] for k in order]


def predict(h, w, logits, locs_lr, overlap=64):
    """One image: logits [K, T, C] and locs_lr [K, 32] of its K windows -> (labels, boxes, decoded rows)."""
    rows = []
    for k, ((a, _), (lo, hi)) in enumerate(plan_windows(h, w, overlap=overlap)):
        rows.append(decode_row(logits[k], locs_lr[k], a, 16.0 * h, lo, hi))
    labels, boxes = merge(h, w, [r[:3] for r in rows])
    return labels, boxes, rows


def planted_image(seed, h, w, T=64, C=6736, blank=6735, overlap=64):
    """Seeded encoder outputs for every window of an h x w line with the cases the decode must get right planted in:
    ties at the maximum, single and multiple NaNs, repeats with and without blanks between them, all-blank rows, more than
    16 decoded characters, r < l boxes, boxes beyond the image and box centres exactly on a core boundary (h a power of two
    keeps that arithmetic exact).  Returns (logits fp32 [K, T, C], locs_lr fp32 [K, 32])."""
    rng = np.random.default_rng(seed)
    wins = plan_windows(h, w, overlap=overlap)
    k = len(wins)
    logits = rng.standard_normal((k, T, C), dtype=np.float32)
    locs = rng.random((k, 2 * SLOTS), dtype=np.float32)
    for r in range(k):
        kind = (seed + r) % 5
        if kind == 0:                                   # all blank
            seq = np.full(T, blank)
        elif kind == 1:                                 # distinct labels: more than 16 decoded
            seq = rng.integers(0, blank, T)
        else:                                           # runs of repeats, blanks in some gaps
            seq = np.repeat(rng.integers(0, 40, T // 2), 2)[:T]
            seq[rng.random(T) < 0.3] = blank
        logits[r, np.arange(T), seq] += 8.0
        for t in rng.choice(T, 4, replace=False):       # ties at the maximum
            j = int(rng.integers(0, C))
            logits[r, t, j] = logits[r, t].max()
        if kind >= 3:
            t = int(rng.integers(0, T))
            logits[r, t, int(rng.integers(0, C))] = np.nan
            if kind == 4:                               # two NaNs in one timestep: the first wins
                logits[r, t, int(rng.integers(0, C))] = np.nan
        locs[r, 0:4] = [0.6, 0.4, -0.3, -0.1]           # r < l; beyond the left edge
        locs[r, 4:6] = [1.2, 1.5]                       # beyond the right edge
    for j in range(k - 1):                              # a centre exactly on each core boundary, in both windows
        bnd = wins[j][1][1]
        for r in (j, j + 1):
            c = np.float32((bnd - wins[r][0][0]) / (16.0 * h))
            assert float(wins[r][0][0]) + float(c) * 16.0 * h == bnd
            locs[r, 6:8] = c
    return logits, locs
