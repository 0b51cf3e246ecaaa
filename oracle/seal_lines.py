"""Numpy twin of the seal centre-line search (DESIGN.md section 7b, "Seal centre lines"), written from the definition, exact in
integers so that the device's line tables equal it bit for bit.  Layered on oracle.seal_pages, whose results it leaves as they
are: it reads a seal table and the crop it was found on.  Test infrastructure only."""
import math

import numpy as np

from oracle import seal_pages as S

HEAD_BINS, HEAD_MIN_K, GAP_MARGIN, LINE_GAP, LINE_MIN_H, LINE_H_DIV, LINE_RATIO = 4, 16, 2, 3, 4, 64, 2
LINE_PAD, LINE_PAD_DIV, MAX_LINES, TURN_STEPS = 2, 8, 4, 144
# (round(2^20 cos 2.5 j), round(2^20 sin 2.5 j)) for j < 36: a quarter turn, the other three by symmetry
TURNS = np.array([(round(2 ** 20 * math.cos(math.radians(2.5 * j))), round(2 ** 20 * math.sin(math.radians(2.5 * j))))
                  for j in range(TURN_STEPS // 4)], np.int64)
FIELDS = ("turn", "g0", "n_gap", "k_bottom", "k_top", "why", "k_in", "k_gap", "n_found", "n_lines")


def turn_dir(t):
    """(c, s) ~ 2^20 (cos, sin) of the turn t (2.5-degree steps), from TURNS and quarter turns only."""
    j = t % TURN_STEPS
    c, s = (int(v) for v in TURNS[j % (TURN_STEPS // 4)])
    for _ in range(j // (TURN_STEPS // 4)):
        c, s = -s, c
    return c, s


def walk_gap_top(ink_k, area):
    """The first bin inside the ring's edge of seal_pages.band's walk (the bin after the ring run and its edge)."""
    k = S.BINS - 1
    while k >= 0 and S.RING_DENSITY * ink_k[k] < area[k]:
        k -= 1
    while k >= 0 and S.RING_DENSITY * ink_k[k] >= area[k]:
        k -= 1
    while k >= 0 and S.BAND_DENSITY * ink_k[k] >= area[k]:
        k -= 1
    return k


def head(ink, k_top):
    """(g0, n, why, turn) of a band whose outer bin is k_top: the gap of the band's outer HEAD_BINS bins by arc_gap, why as
    seal_record's, and the turn 2 g0 + n - 108 in (-72, 72] (0 unless why is 0)."""
    g0, n = S.arc_gap(ink[k_top - HEAD_BINS + 1:k_top + 1].sum(axis=0))
    why = S.NO_GAP if n < S.MIN_GAP else S.SHORT if S.SECTORS - n < S.MIN_TEXT else 0
    t = (2 * g0 + n - 108) % TURN_STEPS
    t = t - TURN_STEPS if t > TURN_STEPS // 2 else t
    return g0, n, why, t if why == 0 else 0


def arc_bottom(ink, area, k_top, g0, n):
    """The last bin of the walk inward from k_top over bins dense on the arc sectors (all but the gap [g0, g0 + n)):
    32 * 72 * ink'_k >= area_k * (72 - n), down to BAND_MIN_K; k_top itself is always in the band."""
    arc = np.ones(S.SECTORS, bool)
    arc[(g0 + np.arange(n)) % S.SECTORS] = False
    ink_a = ink[:, arc].sum(axis=1)
    k = k_top
    while k - 1 >= S.BAND_MIN_K and S.BAND_DENSITY * S.SECTORS * int(ink_a[k - 1]) >= int(area[k - 1]) * (S.SECTORS - n):
        k -= 1
    return k


def stamp_frame(box, t):
    """(u, v) int64 grids: each pixel's doubled ellipse coordinates turned by -t (2.5-degree steps), floored to pixels."""
    X, Y, _, _ = S.ellipse_coords(box)
    c, s = turn_dir(t)
    return (X * c - Y * s) >> 21, (X * s + Y * c) >> 21


def lines_of(rows_u, A, B, k_out):
    """(n_found, boxes) of an interior's rows: rows_u maps row v to the (min u, max u) of its ink.  Runs of ink rows with gaps of
    under LINE_GAP rows are candidates; a candidate h rows high and w wide is a line when h >= max(LINE_MIN_H, (A + B) //
    LINE_H_DIV) and w >= LINE_RATIO h.  Its box (u0, v0, u1, v1), end exclusive, is padded by max(LINE_PAD, h // LINE_PAD_DIV)
    and clipped to [-R - 1, R + 1], R = k_out max(A, B) // 64; the first MAX_LINES from the top are kept."""
    runs, cur, last = [], None, None
    for v in sorted(rows_u):
        lo, hi = rows_u[v]
        if cur is not None and v - last - 1 < LINE_GAP:
            cur = [min(cur[0], lo), cur[1], max(cur[2], hi), v]
        else:
            if cur is not None:
                runs.append(cur)
            cur = [lo, v, hi, v]
        last = v
    if cur is not None:
        runs.append(cur)
    min_h, R = max(LINE_MIN_H, (A + B) // LINE_H_DIV), k_out * max(A, B) // 64
    boxes = []
    for u0, v0, u1, v1 in runs:
        h, w = v1 - v0 + 1, u1 - u0 + 1
        if h < min_h or w < LINE_RATIO * h:
            continue
        p = max(LINE_PAD, h // LINE_PAD_DIV)
        boxes.append((max(u0 - p, -R - 1), max(v0 - p, -R - 1), min(u1 + 1 + p, R + 1), min(v1 + 1 + p, R + 1)))
    return len(boxes), boxes[:MAX_LINES]


def line_record(crop, s):
    """The mn_seal_lines fields of a found seal record ``s`` of seal_pages.seal_record on ``crop``, as a dict."""
    box = (s["x0"], s["y0"], s["x1"], s["y1"])
    ink, area = S.histograms(crop, box)
    k_in = max(walk_gap_top(ink.sum(axis=1), area), 0)
    r = dict(turn=0, g0=-1, n_gap=-1, k_bottom=-1, k_top=-1, why=S.NO_BAND, k_in=k_in, k_gap=k_in, n_found=0, n_lines=0,
             boxes=[])
    if s["k_top"] >= HEAD_MIN_K:
        k_top = s["k_top"]
        g0, n, why, t = head(ink, k_top)
        kb = arc_bottom(ink, area, k_top, g0, n)
        r.update(turn=t, g0=g0, n_gap=n, k_bottom=kb, k_top=k_top, why=why, k_in=kb, k_gap=max(kb, k_top - HEAD_BINS + 1))
    X, Y, A, B = S.ellipse_coords(box)
    k = S.radial_bin(X, Y, A, B)
    in_gap = (S.sector(X * B, -Y * A) - r["g0"] - GAP_MARGIN) % S.SECTORS < r["n_gap"] - 2 * GAP_MARGIN
    m = S.seal_mask(crop[box[1]:box[3], box[0]:box[2]]) & ((k < r["k_in"]) | ((k < r["k_gap"]) & in_gap))
    u, v = np.broadcast_arrays(*stamp_frame(box, r["turn"]))
    u, v = u[m], v[m]
    rows = {}
    if len(v):
        order = np.argsort(v, kind="stable")
        u, v = u[order], v[order]
        vs, first = np.unique(v, return_index=True)
        for j, vv in enumerate(vs):
            seg = u[first[j]:first[j + 1] if j + 1 < len(vs) else len(u)]
            rows[int(vv)] = (int(seg.min()), int(seg.max()))
    r["n_found"], r["boxes"] = lines_of(rows, int(A), int(B), r["k_gap"])
    r["n_lines"] = len(r["boxes"])
    return r


def find_lines(crop, table):
    """The line records of a page's seal table (seal_pages.find_seals' dict): one per candidate slot, None for a slot that is
    no seal (and for every slot of a table with an error)."""
    if table["error"]:
        return [None] * len(table["seals"])
    return [line_record(crop, s) if s["found"] else None for s in table["seals"]]


def page_lines(img, rect=None, seal_size=None):
    """(seal table, line records) of a page crop, as seal_pages.page_seals finds them."""
    H, W = img.shape[:2]
    x0, y0, x1, y1 = rect or (0, 0, W, H)
    crop = img[y0:y1, x0:x1]
    t = S.find_seals(crop, seal_size or S.default_seal_size(x1 - x0, y1 - y0))
    return t, find_lines(crop, t)
