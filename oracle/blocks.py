"""numpy twin of pipeline.find_lines (DESIGN.md section 7b, "Text blocks"): the grey value, OpenCV's Otsu threshold of an 8-bit
image, the ink polarity, the row profile and its line runs, and the line rectangles of a text block.  Written from the
definition, not from the kernels.
TEST INFRASTRUCTURE ONLY."""
import numpy as np

FLT_EPSILON = 1.1920928955078125e-07
MAX_LINES = 256


def grey(crop):
    """g = (c0 + c1 + c2 + 1) // 3 of a uint8 [h, w, 3] crop, as int64."""
    c = crop.astype(np.int64)
    return (c[..., 0] + c[..., 1] + c[..., 2] + 1) // 3


def otsu(g):
    """cv2.threshold(g, 0, 255, THRESH_BINARY | THRESH_OTSU)[0] for 8-bit values g: OpenCV's fp64 loop over the 256-bin
    histogram, every operation rounded on its own.  Returns an int."""
    return otsu_hist(np.bincount(np.asarray(g, np.int64).reshape(-1), minlength=256))


def otsu_hist(hist):
    """OpenCV's Otsu loop on a 256-bin histogram of pixel counts (any integer sequence): the threshold of the pixels it counts."""
    h = [int(v) for v in hist]
    scale = 1.0 / float(sum(h))
    mu = 0.0
    for i in range(256):
        mu += float(i) * float(h[i])
    mu *= scale
    mu1 = q1 = max_sigma = 0.0
    t = 0
    for i in range(256):
        p_i = float(h[i]) * scale
        mu1 *= q1
        q1 += p_i
        q2 = 1.0 - q1
        if min(q1, q2) < FLT_EPSILON or max(q1, q2) > 1.0 - FLT_EPSILON:
            continue
        mu1 = (mu1 + float(i) * p_i) / q1
        mu2 = (mu - q1 * mu1) / q2
        sigma = q1 * q2 * (mu1 - mu2) * (mu1 - mu2)
        if sigma > max_sigma:
            max_sigma, t = sigma, i
    return t


def _lower_median(v):
    return sorted(v)[(len(v) - 1) // 2]


def segment(ink, min_ink=None, gap=None, min_height=None):
    """Steps 4 to 9 on a boolean [h, w] ink mask: the lines' (y0, x0, y1, x1) in the mask's frame, top to bottom.  Raises
    ValueError for more than MAX_LINES lines."""
    h, w = ink.shape
    r = ink.sum(axis=1)
    m = min_ink if min_ink is not None else max(1, w // 128)
    text = r >= m
    runs, y = [], 0
    while y < h:
        if text[y]:
            a = y
            while y < h and text[y]:
                y += 1
            runs.append([a, y])
        else:
            y += 1
    if not runs:
        return []
    g = gap if gap is not None else max(1, _lower_median([b - a for a, b in runs]) // 4)
    merged = [runs[0]]
    for a, b in runs[1:]:
        if a - merged[-1][1] <= g:
            merged[-1][1] = b
        else:
            merged.append([a, b])
    mh = min_height if min_height is not None else max(2, _lower_median([b - a for a, b in merged]) // 3)
    kept = [(a, b) for a, b in merged if b - a >= mh]
    if len(kept) > MAX_LINES:
        raise ValueError(f"{len(kept)} lines exceed the {MAX_LINES} a block may hold")
    out = []
    for k, (a, b) in enumerate(kept):
        p = (b - a + 3) // 4
        lo = (kept[k - 1][1] + a) // 2 if k > 0 else 0
        hi = (b + kept[k + 1][0]) // 2 if k + 1 < len(kept) else h
        cols = np.nonzero(ink[a:b].any(axis=0))[0]
        out.append((max(a - p, lo), max(0, int(cols[0]) - p), min(b + p, hi), min(w, int(cols[-1]) + 1 + p)))
    return out


def find_lines(img, rect, direction="horizontal", min_ink=None, gap=None, min_height=None, polarity="auto"):
    """The text block ``rect`` = (X0, Y0, X1, Y1) of the uint8 [H, W, 3] image ``img`` -> dict(lines, threshold, ink): lines the
    integer rectangles (x0, y0, x1, y1) in image coordinates in reading order (top to bottom; right to left for a vertical
    block), ink "dark" or "light".  A vertical block is the horizontal computation on the transposed crop."""
    x0, y0, x1, y1 = rect
    g = grey(img[y0:y1, x0:x1])
    t = otsu(g)
    if polarity == "auto":
        polarity = "dark" if 2 * int((g <= t).sum()) <= g.size else "light"
    ink = g <= t if polarity == "dark" else g > t
    if direction == "horizontal":
        lines = [(x0 + a, y0 + b, x0 + c, y0 + d) for b, a, d, c in segment(ink, min_ink, gap, min_height)]
    else:
        lines = [(x0 + b, y0 + a, x0 + d, y0 + c) for b, a, d, c in segment(ink.T, min_ink, gap, min_height)][::-1]
    return dict(lines=lines, threshold=t, ink=polarity)
