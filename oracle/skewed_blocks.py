"""numpy twin of pipeline.find_lines for skewed text blocks (DESIGN.md section 7b, "Skewed blocks"): the angle table, the
rotated frame, the per-angle profiles and their scores, the chosen angle, the lines in the chosen frame and their corners in
the image.  Vectorised numpy fp64, every operation rounded on its own; written from the definition, not from the kernels.
Steps 1 to 3 (grey value, Otsu's threshold, polarity) are oracle/blocks.py's.
TEST INFRASTRUCTURE ONLY."""
import math

import numpy as np

from . import blocks as B


def angles(skew, max_skew=10.0):
    """(i, theta_i) of the search: i / 20 degrees for |i| <= round(20 max_skew) with skew "auto"; a given angle is the one
    entry (0, skew)."""
    if isinstance(skew, str):
        n = round(20 * max_skew)
        return [(i, i / 20) for i in range(-n, n + 1)]
    return [(0, float(skew))]


def frame(h, w, c, s):
    """(u_min, v_min, L, M) of an h x w crop for arrays c, s: the least u and v of the four corner pixel centres, L = floor(v_max
    - v_min) + 1, M = floor(u_max - u_min) + 1."""
    xs, ys = (0 + 0.5 - w / 2, w - 1 + 0.5 - w / 2), (0 + 0.5 - h / 2, h - 1 + 0.5 - h / 2)
    u = np.stack([x * c - y * s for x in xs for y in ys])
    v = np.stack([x * s + y * c for x in xs for y in ys])
    u_min, v_min = u.min(axis=0), v.min(axis=0)
    return (u_min, v_min, (np.floor(v.max(axis=0) - v_min) + 1).astype(np.int64),
            (np.floor(u.max(axis=0) - u_min) + 1).astype(np.int64))


def _uv(ys, xs, h, w, c, s):
    X, Y = xs + 0.5 - w / 2, ys + 0.5 - h / 2
    return X * c - Y * s, X * s + Y * c


def profiles(ink, c, s):
    """r_i[k] of a boolean [h, w] ink mask for each (c_i, s_i): a list of int64 arrays of L_i bins."""
    h, w = ink.shape
    ys, xs = np.nonzero(ink)
    ys, xs = ys.astype(np.float64), xs.astype(np.float64)
    _, v_min, L, _ = frame(h, w, c, s)
    out = []
    for i in range(len(c)):
        _, v = _uv(ys, xs, h, w, c[i], s[i])
        k = np.clip(np.floor(v - v_min[i]), 0, L[i] - 1).astype(np.int64)
        out.append(np.bincount(k, minlength=int(L[i])).astype(np.int64))
    return out


def score(r):
    """S = sum_k (r[k+1] - r[k])^2 in int64."""
    d = np.diff(r.astype(np.int64))
    return int((d * d).sum())


def choose(idx, scores):
    """The position of the largest score; ties to the least |i|, then the least i."""
    return max(range(len(idx)), key=lambda p: (scores[p], -abs(idx[p]), -idx[p]))


def _segment(r, lo, hi, L, M, min_ink, gap, min_height):
    """Steps 4 to 9 on a frame profile: r[k] the ink count of bin k, lo / hi its least and largest ink index j (ignored where r
    is 0).  Returns the lines (c0, l0, c1, l1) in frame indices, top to bottom."""
    m = min_ink if min_ink is not None else max(1, M // 128)
    text = r >= m
    runs, k = [], 0
    while k < L:
        if text[k]:
            a = k
            while k < L and text[k]:
                k += 1
            runs.append([a, k])
        else:
            k += 1
    if not runs:
        return []
    g = gap if gap is not None else max(1, B._lower_median([b - a for a, b in runs]) // 4)
    merged = [runs[0]]
    for a, b in runs[1:]:
        if a - merged[-1][1] <= g:
            merged[-1][1] = b
        else:
            merged.append([a, b])
    mh = min_height if min_height is not None else max(2, B._lower_median([b - a for a, b in merged]) // 3)
    kept = [(a, b) for a, b in merged if b - a >= mh]
    if len(kept) > B.MAX_LINES:
        raise ValueError(f"{len(kept)} lines exceed the {B.MAX_LINES} a block may hold")
    out = []
    for k, (a, b) in enumerate(kept):
        p = (b - a + 3) // 4
        l0 = max(a - p, (kept[k - 1][1] + a) // 2 if k > 0 else 0)
        l1 = min(b + p, (b + kept[k + 1][0]) // 2 if k + 1 < len(kept) else L)
        has = r[a:b] > 0
        jmin, jmax = int(lo[a:b][has].min()), int(hi[a:b][has].max())
        out.append((max(0, jmin - p), l0, min(M, jmax + 1 + p), l1))
    return out


def corners(line, c, s, u_min, v_min, O):
    """Frame line (c0, l0, c1, l1) -> its (tl, tr, bl) in the crop's frame coordinates around O: a = u_min - 0.5 + c,
    b = v_min - 0.5 + l, e = (c, -s), f = (s, c), p = O + a e + b f, in fp64."""
    c0, l0, c1, l1 = (int(v) for v in line)
    c, s, u_min, v_min = float(c), float(s), float(u_min), float(v_min)
    ex, ey, fx, fy = c, -s, s, c
    a0, a1 = u_min - 0.5 + c0, u_min - 0.5 + c1
    b0, b1 = v_min - 0.5 + l0, v_min - 0.5 + l1
    ox, oy = O
    return ((ox + a0 * ex + b0 * fx, oy + a0 * ey + b0 * fy), (ox + a1 * ex + b0 * fx, oy + a1 * ey + b0 * fy),
            (ox + a0 * ex + b1 * fx, oy + a0 * ey + b1 * fy))


def find_lines(img, rect, direction="horizontal", min_ink=None, gap=None, min_height=None, polarity="auto", skew="auto",
               max_skew=10.0):
    """The skewed text block ``rect`` of ``img`` -> dict(lines, threshold, ink, skew, detail).  lines: (tl, tr, bl) corner
    triples in image coordinates in reading order (for a vertical block already in VerticalRegion order: tl -> tr across the
    column, tl -> bl down it), or blocks.find_lines' integer rectangles when the chosen entry's s is 0.  skew: the angle used,
    counter-clockwise on screen.  detail: the table's i, c, s, the scores (None for a one-entry table), the chosen position, the
    chosen frame (u_min, v_min, L, M) and the frame lines (c0, l0, c1, l1).  A vertical block is the computation on the
    transposed crop, its frame angle the negated skew."""
    x0, y0, x1, y1 = rect
    g = B.grey(img[y0:y1, x0:x1])
    t = B.otsu(g)
    if polarity == "auto":
        polarity = "dark" if 2 * int((g <= t).sum()) <= g.size else "light"
    ink = g <= t if polarity == "dark" else g > t
    vertical = direction == "vertical"
    if vertical:
        ink = ink.T
    tab = angles(skew, max_skew)
    idx = [i for i, _ in tab]
    deg = [(-th if vertical and not isinstance(skew, str) else th) for _, th in tab]
    c = np.array([math.cos(math.radians(d)) for d in deg], np.float64)
    s = np.array([math.sin(math.radians(d)) for d in deg], np.float64)
    h, w = ink.shape
    if len(tab) > 1:
        scores = [score(r) for r in profiles(ink, c, s)]
        p = choose(idx, scores)
    else:
        scores, p = None, 0
    u_min, v_min, L, M = (a[0] for a in frame(h, w, c[p:p + 1], s[p:p + 1]))
    ys, xs = np.nonzero(ink)
    u, v = _uv(ys.astype(np.float64), xs.astype(np.float64), h, w, c[p], s[p])
    k = np.clip(np.floor(v - v_min), 0, L - 1).astype(np.int64)
    j = np.clip(np.floor(u - u_min), 0, M - 1).astype(np.int64)
    r = np.bincount(k, minlength=int(L))
    lo = np.full(int(L), np.iinfo(np.int64).max)
    hi = np.full(int(L), -1)
    np.minimum.at(lo, k, j)
    np.maximum.at(hi, k, j)
    frame_lines = _segment(r, lo, hi, int(L), int(M), min_ink, gap, min_height)
    angle = deg[p] if not vertical else 0.0 - deg[p]
    if not isinstance(skew, str):
        angle = float(skew)
    if s[p] == 0:
        if vertical:
            lines = [(x0 + l0, y0 + c0, x0 + l1, y0 + c1) for c0, l0, c1, l1 in frame_lines][::-1]
        else:
            lines = [(x0 + c0, y0 + l0, x0 + c1, y0 + l1) for c0, l0, c1, l1 in frame_lines]
    elif vertical:
        O = (y0 + (y1 - y0) / 2, x0 + (x1 - x0) / 2)
        lines = []
        for q in frame_lines:
            tl, tr, bl = corners(q, c[p], s[p], u_min, v_min, O)
            lines.append((tl[::-1], bl[::-1], tr[::-1]))
        lines = lines[::-1]
    else:
        O = (x0 + (x1 - x0) / 2, y0 + (y1 - y0) / 2)
        lines = [corners(q, c[p], s[p], u_min, v_min, O) for q in frame_lines]
    detail = dict(i=idx, c=c, s=s, scores=scores, chosen=p, frame=(float(u_min), float(v_min), int(L), int(M)),
                  frame_lines=frame_lines)
    return dict(lines=lines, threshold=t, ink=polarity, skew=angle, detail=detail)
