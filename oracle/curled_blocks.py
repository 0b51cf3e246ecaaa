"""numpy twin of pipeline.find_lines for curled text blocks (DESIGN.md section 7b, "Curled blocks"): the strips, their row
profiles and runs, the left-to-right link of the runs into lines, and the lines as CurvedRegions.  Integer arithmetic up to the
link table; the fit is pipeline.curve_lines, shared with the pipeline as skew_lines is.  Steps 1 to 3 (grey value, Otsu's
threshold, polarity) and the level lines are oracle/blocks.py's.  Written from the definition, not from the kernels.
TEST INFRASTRUCTURE ONLY."""
import numpy as np

from . import blocks as B

MAX_STRIPS = 32
MIN_STRIP = 32          # pixels of a strip, when there is more than one
MAX_GAP = 2             # strips a line may skip
RUN_CAP = 256           # kept runs of one strip
LINE_INTS = 8 + 2 * MAX_STRIPS
OK, ERR_RUNS, ERR_LINES = 0, 1, 2


def strip_count(w, strips=None):
    """n_s: ``strips``, or clamp(w // 48, 1, 32)."""
    return int(strips) if strips is not None else min(MAX_STRIPS, max(1, w // 48))


def bounds(w, n):
    """The strip boundaries x_j = j w // n, j = 0 .. n."""
    return [j * w // n for j in range(n + 1)]


def strip_profiles(ink, n):
    """int64 [n, 3, h] of a boolean [h, w] ink mask: per strip j and row y, the ink count over [x_j, x_{j+1}), w - (its least ink
    column) and its largest ink column + 1 (both 0 where the row has no ink in the strip), columns counted in the crop."""
    h, w = ink.shape
    xb = bounds(w, n)
    out = np.zeros((n, 3, h), np.int64)
    for j in range(n):
        sub = ink[:, xb[j]:xb[j + 1]]
        cnt = sub.sum(axis=1)
        has = cnt > 0
        first = xb[j] + np.argmax(sub, axis=1)
        last = xb[j + 1] - 1 - np.argmax(sub[:, ::-1], axis=1)
        out[j, 0] = cnt
        out[j, 1] = np.where(has, w - first, 0)
        out[j, 2] = np.where(has, last + 1, 0)
    return out


def strip_runs(prof, M, w, min_ink=None, gap=None, min_height=None):
    """Steps 4 to 7 of "Text blocks" on one strip's profile prof [3, h] (strip_profiles' layout), M the strip's width: the kept
    runs (a, b, least ink column, largest ink column) top to bottom, or minus their number when it exceeds RUN_CAP."""
    r, lo, hi = prof
    h = len(r)
    m = min_ink if min_ink is not None else max(1, M // 128)
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
    g = gap if gap is not None else max(1, B._lower_median([b - a for a, b in runs]) // 4)
    merged = [runs[0]]
    for a, b in runs[1:]:
        if a - merged[-1][1] <= g:
            merged[-1][1] = b
        else:
            merged.append([a, b])
    mh = min_height if min_height is not None else max(2, B._lower_median([b - a for a, b in merged]) // 3)
    kept = [(a, b) for a, b in merged if b - a >= mh]
    if len(kept) > RUN_CAP:
        return -len(kept)
    return [(a, b, w - int(lo[a:b].max()), int(hi[a:b].max()) - 1) for a, b in kept]


def _overlap(p, q):
    return min(p[1], q[1]) - max(p[0], q[0])


def link(runs, n):
    """Step 4 on the kept runs of every strip: (header, table).  header = [status, n_lines, median, strip, count, 0, 0, 0]:
    status OK, ERR_RUNS (strip ``strip`` has ``count`` runs, over RUN_CAP) or ERR_LINES (``count`` lines, over 256).  table:
    int64 [n_lines, LINE_INTS], one row per line top to bottom: first strip, last strip, runs, least and largest ink column, the
    sample mask (bit j: strip j's run is a sample; an int32 word), 0, 0, then (a_j, b_j) per strip j < MAX_STRIPS, (-1, -1)
    where the line has no run."""
    header = np.zeros(8, np.int64)
    for j, rj in enumerate(runs):
        if isinstance(rj, int):
            header[[0, 3, 4]] = ERR_RUNS, j, -rj
            return header, np.zeros((0, LINE_INTS), np.int64)
    lines = []                                          # per line: id, {strip: run}, last strip
    for j in range(n):
        act = [L for L in lines if j - L[2] <= MAX_GAP + 1]
        R = runs[j]
        best_line = []
        for r in R:                                     # each run's line: the largest overlap, ties to the upper last run
            best, bo = None, 0
            for L in act:
                last = L[1][L[2]]
                o = _overlap(last, r)
                if o > bo or (o == bo and o > 0 and (last[0], L[0]) < (best[1][best[2]][0], best[0])):
                    best, bo = L, o
            best_line.append(best)
        best_run = {}
        for L in act:                                   # each line's run: the largest overlap, ties to the upper run
            last = L[1][L[2]]
            bk, bo = None, 0
            for k, r in enumerate(R):
                o = _overlap(last, r)
                if o > bo:
                    bk, bo = k, o
            best_run[L[0]] = bk
        fresh = []
        for k, r in enumerate(R):
            L = best_line[k]
            if L is not None and best_run[L[0]] == k:
                L[1][j] = r
                L[2] = j
            else:
                fresh.append([len(lines) + len(fresh), {j: r}, j])
        lines += fresh
    need = (n + 3) // 4
    kept = sorted((L for L in lines if len(L[1]) >= need), key=lambda L: (L[1][min(L[1])][0], L[0]))
    if len(kept) > 256:
        header[[0, 4]] = ERR_LINES, len(kept)
        return header, np.zeros((0, LINE_INTS), np.int64)
    heights = [r[1] - r[0] for L in kept for r in L[1].values()]
    med = B._lower_median(heights) if heights else 0
    table = np.zeros((len(kept), LINE_INTS), np.int64)
    for k, L in enumerate(kept):
        js = sorted(L[1])
        mask = sum(1 << j for j in js if 2 * (L[1][j][1] - L[1][j][0]) <= 3 * med)
        mask -= (1 << 32) if mask >> 31 else 0              # an int32 word: bit 31 is its sign
        table[k, :8] = js[0], js[-1], len(js), min(L[1][j][2] for j in js), max(L[1][j][3] for j in js), mask, 0, 0
        table[k, 8:] = -1
        for j in js:
            table[k, 8 + 2 * j:10 + 2 * j] = L[1][j][:2]
    header[1], header[2] = len(kept), med
    return header, table


def find_lines(img, rect, min_ink=None, gap=None, min_height=None, polarity="auto", strips=None):
    """The curled text block ``rect`` of ``img`` -> dict(lines, threshold, ink, curve[, error]) as pipeline.find_lines gives it
    for TextBlock(rect, curve="auto"), and ``detail``: the strip count, profiles, runs, link header and table.  ``error`` (and
    no lines) for a block over a limit."""
    from marconet_b200.pipeline import curve_lines
    x0, y0, x1, y1 = rect
    g = B.grey(img[y0:y1, x0:x1])
    t = B.otsu(g)
    if polarity == "auto":
        polarity = "dark" if 2 * int((g <= t).sum()) <= g.size else "light"
    ink = g <= t if polarity == "dark" else g > t
    h, w = ink.shape
    n = strip_count(w, strips)
    xb = bounds(w, n)
    prof = strip_profiles(ink, n)
    runs = [strip_runs(prof[j], xb[j + 1] - xb[j], w, min_ink, gap, min_height) for j in range(n)]
    header, table = link(runs, n)
    detail = dict(strips=n, profiles=prof, runs=runs, header=header, table=table)
    res = dict(threshold=t, ink=polarity, detail=detail)
    if header[0] != OK:
        return dict(res, lines=[], error=int(header[0]))
    try:
        level = [(x0 + a, y0 + b, x0 + c, y0 + d) for b, a, d, c in B.segment(ink, min_ink, gap, min_height)]
    except ValueError:                                  # over 256 lines: never level
        level = None
    lines, curve = curve_lines(rect, n, table, level)
    return dict(res, lines=lines, curve=curve)
