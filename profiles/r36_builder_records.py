"""Record-equivalence check of ops.py's batched call builders against another version of ops.py (r36_builder_records.jsonl).

    python profiles/r36_builder_records.py OLD_OPS_PY [--out FILE]

OLD_OPS_PY is the other version's marconet_b200/ops.py (for example ``git show <parent>:marconet_b200/ops.py``).  Both versions
are driven with the same seeded calls while _lib.load() returns a recorder, so no kernel runs.  For every C-entry call the
recorder keeps the scalar arguments and every buffer the builder allocated (its length and its bytes, read back when the entry
is called, with every pointer into one of those buffers rewritten as (buffer, offset)); pointers into the items are the same
tensors in both versions and are kept as they are.  Allocations are filled with 0xA5 first, so the bytes a builder does not
upload show.  A call also records its return value (tensors as buffer, offset, shape, strides and dtype), the launch count it
adds and, for a refused call, its exception type and text.  One JSON line per builder: calls compared, calls that reached a C
entry, refused calls and mismatches, and apart from them the two differences the packer made on purpose: figure_panels'
dense-pixel refusals now carry _dense_u8's text (message_changes), and composite_regions_curved no longer allocates the 4 or 8
bytes that aligned its curve tables' address by hand, never uploaded nor read (slack_dropped).  Runs on the GPU, or on the CPU
for the builders that do not insist on CUDA tensors.
"""
import argparse
import ctypes
import hashlib
import importlib.util
import json
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from marconet_b200 import _lib  # noqa: E402
from marconet_b200 import ops as new_ops  # noqa: E402

CUDA = torch.cuda.is_available()
DEV = torch.device("cuda", torch.cuda.current_device()) if CUDA else torch.device("cpu")
STATE = dict(allocs=None, calls=None)
SENTINEL = 0xA5


def _register(t, fill):
    if STATE["allocs"] is not None:
        if fill:
            t.reshape(-1).view(torch.uint8).fill_(SENTINEL)
        STATE["allocs"].append(t)
    return t


class _Torch:
    """The torch module as the builders see it, with empty / zeros registering their allocations."""

    def __getattr__(self, k):
        return getattr(torch, k)

    def empty(self, *a, **k):
        return _register(torch.empty(*a, **k), True)

    def zeros(self, *a, **k):
        return _register(torch.zeros(*a, **k), False)


def _where(v):
    for i, t in enumerate(STATE["allocs"]):
        base = t.data_ptr()
        if base <= v <= base + t.numel() * t.element_size():
            return i, v - base
    return None


def _scalar(a):
    if isinstance(a, ctypes.c_void_p):
        a = a.value or 0
    if isinstance(a, bool) or a is None:
        return a
    if isinstance(a, int):
        w = _where(a) if a > 4096 else None
        return ["buf", *w] if w else a
    if isinstance(a, float):
        return repr(a)
    return repr(a)


def _snapshot():
    out = []
    ranges = [(t.data_ptr(), t.numel() * t.element_size()) for t in STATE["allocs"]]
    for t in STATE["allocs"]:
        raw = t.reshape(-1).view(torch.uint8).cpu().numpy()
        n8 = len(raw) // 8 * 8
        u = raw[:n8].view(np.uint64).copy()
        for i, (base, n) in enumerate(ranges):
            m = (u >= np.uint64(base)) & (u <= np.uint64(base + n))
            u[m] = (np.uint64(1) << np.uint64(63)) | (np.uint64(i) << np.uint64(40)) | (u[m] - np.uint64(base))
        data = u.tobytes() + raw[n8:].tobytes()
        out.append([len(raw), hashlib.sha1(data).hexdigest(), data if len(data) <= 1 << 24 else None])
    return out


class _Recorder:
    def __getattr__(self, name):
        def entry(*args):
            STATE["calls"].append([name, [_scalar(a) for a in args], _snapshot()])
            return 0
        return entry


def _describe(r):
    if isinstance(r, torch.Tensor):
        return ["tensor", _where(r.data_ptr()), list(r.shape), list(r.stride()), str(r.dtype)]
    if isinstance(r, (list, tuple)):
        return [_describe(x) for x in r]
    if isinstance(r, dict):
        return {k: _describe(v) for k, v in sorted(r.items())}
    return r


def _own(mod, a):
    """``a`` with the CurveTables made of ``mod``'s class, which its builders test for."""
    if isinstance(a, new_ops.CurveTable):
        return mod.CurveTable(*a)
    if isinstance(a, (list, tuple)) and not hasattr(a, "_fields"):
        return type(a)(_own(mod, x) for x in a)
    return a


def run(mod, fn, args, kwargs):
    args = _own(mod, args)
    STATE["allocs"], STATE["calls"] = [], []
    before = mod.LAUNCHES
    try:
        ret = ["ok", _describe(getattr(mod, fn)(*args, **kwargs))]
    except Exception as e:      # a refused call: its type and text are what is compared
        ret = ["raised", type(e).__name__, str(e)]
    rec = dict(ret=ret, calls=STATE["calls"], launches=mod.LAUNCHES - before)
    if ret[0] == "ok":          # a refused call may have allocated before its refusal; nothing of it reached a C entry
        rec["lengths"] = [t.numel() * t.element_size() for t in STATE["allocs"]]
        rec["returned"] = [h for _, h, _ in _snapshot()]
    STATE["allocs"] = STATE["calls"] = None
    return rec


def _key(rec):
    return json.dumps(rec, sort_keys=True, default=lambda b: None)


def _slack_only(old, new):
    """True when the two calls differ only in bytes at the end of the old buffer that were never uploaded: the 4 or 8 bytes
    composite_regions_curved used to allocate for aligning its curve tables' address by hand."""
    if len(old["calls"]) != 1 or len(new["calls"]) != 1 or len(old["lengths"]) != 1:
        return False
    (o_name, o_args, [(o_len, _, o_data)]), (n_name, n_args, [(n_len, _, n_data)]) = old["calls"][0], new["calls"][0]
    return (o_name == n_name and o_args == n_args and 0 < o_len - n_len <= 8 and o_data[:n_len] == n_data
            and set(o_data[n_len:]) == {SENTINEL} and old["ret"] == new["ret"] and old["launches"] == new["launches"])


def load_old(path):
    spec = importlib.util.spec_from_file_location("marconet_b200._ops_old", path)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


# ---- the seeded calls ------------------------------------------------------------------------------------------------------
def _img(rng, h, w, c=3, pitch=0):
    t = torch.from_numpy(rng.integers(0, 256, (h, w + pitch, c), dtype=np.uint8)).to(DEV)
    return t[:, :w] if pitch else t


def _curve(x0, y0, x1, y1, h, k, scale=1.0):
    xs, ys = np.linspace(x0, x1, 3 * k + 1), np.linspace(y0, y1, 3 * k + 1)
    return new_ops.CurveTable(scale, tuple(np.linspace(0, 1, k + 1)), tuple((float(x), float(y)) for x, y in zip(xs, ys)),
                              tuple((float(x), float(y) + h) for x, y in zip(xs, ys)))


def cases(rng):
    """(builder, function name, args, kwargs) of every call compared."""
    out = []
    add = lambda b, fn, *a, **k: out.append((b, fn, a, k))  # noqa: E731
    tiny = _img(rng, 4, 4)

    # images and regions
    for n in (1, 2, 7):
        for cn in (1, 3, 4):
            items = [(_img(rng, 20 + 3 * i, 30 + 5 * i, cn, pitch=i % 2), _img(rng, 11 + i, 17 + 2 * i, cn)) for i in range(n)]
            add("resize_cubic", "resize_cubic", items)
            add("warp", "warp_affine", [(s, d, [[1, 0.1, 2], [0.05, 1, 3]]) for s, d in items])
            add("warp", "warp_perspective", [(s, d, [[1, 0.1, 2], [0.05, 1, 3], [0.001, 0, 1]]) for s, d in items])
            add("remap_curved", "remap_curved", [(s, d, _curve(1, 2, 15, 5, 8, 1 + i % 3)) for i, (s, d) in enumerate(items)])
    add("resize_cubic", "resize_cubic", [])
    add("resize_cubic", "resize_cubic", [(tiny, tiny)] * 65536)
    add("resize_cubic", "resize_cubic", [(_img(rng, 4, 4, 5), _img(rng, 4, 4, 5))])
    add("resize_cubic", "resize_cubic", [(tiny, _img(rng, 4, 4, 1))])
    tall = torch.zeros((32768, 1, 3), dtype=torch.uint8, device=DEV)
    add("warp", "warp_affine", [(tall, tiny, [[1, 0, 0], [0, 1, 0]])])
    add("warp", "warp_perspective", [(tall, tiny, [[1, 0, 0], [0, 1, 0], [0, 0, 1]])])
    add("warp", "warp_affine", [(tiny, tiny, [[1, 0, 0]])])
    add("warp", "warp_affine", [])
    add("remap_curved", "remap_curved", [(tall, tiny, _curve(0, 0, 3, 0, 3, 1))])
    add("remap_curved", "remap_curved", [(tiny, tiny, new_ops.CurveTable(1.0, (0.0, 1.0), ((0, 0),), ((0, 1),)))])
    add("remap_curved", "remap_curved", [])
    add("remap_curved", "remap_curved", [(_img(rng, 4, 4, 0), tiny, _curve(0, 0, 3, 0, 3, 1))])

    page, page2 = _img(rng, 120, 160, pitch=8), _img(rng, 90, 100)
    srs = [_img(rng, 16 + i, 40 + 3 * i) for i in range(6)]
    rects = [(0, 0, 40, 30), (30, 20, 90, 60), (100, 50, 160, 120), (5, 70, 60, 119)]
    chains = [[0, 1], [0, 1], [2], [3]]
    base = [(page, srs[i], rects[i], chains[i]) for i in range(4)] + [(page2, srs[4], (10, 10, 50, 50), [4])]
    aff = ([[0.9, 0.1, 1.0], [-0.1, 0.9, 2.0]], 1.5, 2.0)
    per = ([[0.9, 0.1, 1.0], [-0.1, 0.9, 2.0], [0.001, 0.0, 1.0]], 1.5, 2.0)
    cur = (_curve(10, 10, 50, 14, 20, 2, 2.0), 1.0, 1.0)
    for feather in (0, 3):
        add("composite_regions", "composite_regions", base, feather)
        add("composite_regions", "composite_regions", [(page, srs[0], rects[0], [0])], feather)
        add("composite_regions_affine", "composite_regions_affine", [r + (m,) for r, m in zip(base, (None, aff, None, aff, None))], feather)
        add("composite_regions_quad", "composite_regions_quad", [r + (m,) for r, m in zip(base, (per, aff, None, per, None))], feather)
        add("composite_regions_curved", "composite_regions_curved",
            [r + (m,) for r, m in zip(base, (per, cur, None, aff, cur))], feather)
        add("composite_regions_curved", "composite_regions_curved", [r + (m,) for r, m in zip(base, (per, None, aff, None, None))],
            feather)
        add("composite_regions_curved", "composite_regions_curved", [(page2, srs[4], (10, 10, 50, 50), [0], cur)], feather)
    for fn in ("composite_regions", "composite_regions_affine", "composite_regions_quad", "composite_regions_curved"):
        add(fn, fn, [], 0)
        add(fn, fn, [(tiny, tiny, (0, 0, 1, 1), [0], None)] * 65536, 0)
        add(fn, fn, [(tiny, tiny, (0, 0, 1, 1), [0], None)], -1)
        add(fn, fn, [(tiny, tiny, (0, 0, 5, 1), [0], None)], 0)
        add(fn, fn, [(tiny, tiny, (0, 0, 1, 1), [1], None)], 0)
    add("composite_regions_curved", "composite_regions_curved", [(tiny, tiny, (0, 0, 1, 1), [0], (_curve(0, 0, 3, 0, 3, 1, 0.5), 1, 1))], 0)
    add("composite_regions_affine", "composite_regions_affine", [(tiny, tiny, (0, 0, 1, 1), [0], ([[1, 0, 0]], 1, 1))], 0)

    # figure, predictions, pre- and postprocessing
    fig_items = []
    for i in range(4):
        img = _img(rng, 32 + 4 * i, 90 + 20 * i, pitch=i % 2)
        S = new_ops.round_half_even(img.shape[1] * (128 / img.shape[0]))
        fig = _img(rng, 512, S - i)
        priors = [torch.rand((3, 128, 128), device=DEV) for _ in range(1 + i % 3)]
        fig_items.append((img, fig, [(0, 5), (7, 20)][:i % 3], [(1, S)], priors))
    add("figure_panels", "figure_panels", fig_items)
    add("figure_panels", "figure_panels", fig_items[2:3])
    add("figure_panels", "figure_panels", [fig_items[0][:4] + ([],)])
    add("figure_panels", "figure_panels", [])
    add("figure_panels", "figure_panels", [(fig_items[0][0], fig_items[0][1][:, :, :2], [], [], fig_items[0][4])])
    add("figure_panels", "figure_panels", [(fig_items[0][0], fig_items[0][1], [(3, 3)], [], fig_items[0][4])])
    wins = [(float(i), 512.0 + i, float(-i), float(100 + i)) for i in range(9)]
    add("prediction_table", "prediction_table", wins, DEV)
    add("prediction_table", "prediction_table", wins[:1], DEV)
    add("prediction_table", "prediction_table", [], DEV)
    if CUDA:
        crops = [(_img(rng, 32, 200, c, pitch=4), 3, 150) for c in (3, 3, 3)] + [(_img(rng, 40, 300), 0, 300)]
        add("preprocess_lq_crops", "preprocess_lq_crops", crops)
        add("preprocess_lq_crops", "preprocess_lq_crops", [(_img(rng, 32, 100, 1), 0, 100)])
        add("preprocess_lq_crops", "preprocess_lq_crops", [])
        add("preprocess_lq_crops", "preprocess_lq_crops", [crops[0], (_img(rng, 32, 100, 1), 0, 100)])
        add("preprocess_lq_crops", "preprocess_lq_crops", [(crops[0][0], 5, 5)])
        sr = torch.rand((3, 3, 128, 256), device=DEV).to(memory_format=torch.channels_last)
        dst = torch.zeros((128, 600, 3), dtype=torch.uint8, device=DEV)
        add("postprocess_sr_pieces", "postprocess_sr_pieces", sr, [(0, 0, dst[:, 0:100]), (2, 50, dst[:, 100:300]), (1, 10, dst[:, 400:401])])
        add("postprocess_sr_pieces", "postprocess_sr_pieces", sr, [(0, 0, dst[:, :256])])
        add("postprocess_sr_pieces", "postprocess_sr_pieces", sr, [])
        add("postprocess_sr_pieces", "postprocess_sr_pieces", sr, [(3, 0, dst[:, :10])])

    # vertical columns
    cols = []
    for i in range(5):
        src, n = _img(rng, 200, 24, pitch=i % 2), 1 + i
        cells = [(10 * k, 2 * k, 8 + k) for k in range(n)]
        cols.append((src, _img(rng, 30, n * (20 + i)), cells))
    add("vertical_layout", "vertical_layout", cols)
    add("vertical_layout", "vertical_layout", cols[:1])
    add("vertical_layout", "vertical_layout", [])
    add("vertical_layout", "vertical_layout", [(cols[0][0], cols[0][1], [(195, 0, 10)])])
    un = []
    for i in range(4):
        src = _img(rng, 128, 300, pitch=i % 2)
        cells = [(10 * k, 5 * k, 5 * k + 40, 60 * k, 60 * k + 60) for k in range(1 + i)]
        un.append((src, _img(rng, 100, 50 + i), cells))
    add("vertical_unlayout", "vertical_unlayout", un)
    add("vertical_unlayout", "vertical_unlayout", [])
    add("vertical_unlayout", "vertical_unlayout", [(un[0][0], un[0][1], [(1, 0, 10, 0, 10)])])

    # flat pages and lighting
    def lines(dw, n, seed):
        r = np.random.default_rng(seed)
        t = r.normal(size=(n, 9)) * 10
        a = r.integers(0, dw - 1, n)
        t[:, 7], t[:, 8] = a, np.minimum(dw, a + r.integers(1, dw, n))
        return t
    flats = []
    for i in range(5):
        src, dst = _img(rng, 80 + i, 120, 3, pitch=i % 2), _img(rng, 60, 90 + 7 * i, 3)
        m = (3, 4) if i % 2 else tuple(float(v) for v in rng.normal(size=8))
        flats.append((src, dst, "rect" if i % 2 else "quad", m, lines(dst.shape[1], i * 3, i)))
    for tables in (False, True):
        add("flat_remap", "flat_remap", flats, tables=tables)
        add("flat_remap", "flat_remap", flats[1:2], tables=tables)
        add("flat_remap", "flat_remap", [f[:4] + (np.zeros((0, 9)),) for f in flats[:3]], tables=tables)
    for cn in (1, 4):
        add("flat_remap", "flat_remap", [(_img(rng, 40, 50, cn), _img(rng, 30, 33, cn), "rect", (1, 2), lines(33, 4, 9))])
    add("flat_remap", "flat_remap", [])
    add("flat_remap", "flat_remap", [flats[0][:2] + ("quad", (1, 2), flats[0][4])])
    add("flat_remap", "flat_remap", [flats[1][:4] + (np.array([[0] * 7 + [5, 3]], float),)])
    add("flat_remap", "flat_remap", [flats[1][:4] + (lines(90, 257, 3) * 0 + np.array([0] * 7 + [0, 90.0]),)])
    ev, inks = [], torch.zeros((6, 4), dtype=torch.int32, device=DEV).unbind(0)
    for i in range(5):
        src = _img(rng, 40 + 3 * i, 50 + 5 * i, pitch=i % 2)
        dst = src if i == 2 else _img(rng, *src.shape)
        ev.append((_img(rng, 70 + i, 66), src, dst, 3 + 2 * i, i % 3))
    add("even_light", "even_light", ev)
    add("even_light", "even_light", ev[:1])
    add("even_light", "even_light", ev, inks=list(inks[:5]))
    add("even_light", "even_light", ev[3:], inks=list(inks[:2]))
    add("even_light", "even_light", [])
    add("even_light", "even_light", ev, inks=list(inks[:4]))
    add("even_light", "even_light", [ev[0][:3] + (4, 0)])
    add("even_light", "even_light", [ev[0][:4] + (7,)])
    add("even_light", "even_light", [ev[0]], inks=[torch.zeros(5, dtype=torch.int32, device=DEV)])

    # text layout
    A = _lib.INK_AUTO
    blk = [(_img(rng, 300, 400, pitch=5), (10 + 7 * i, 20 + 3 * i, 200 + 20 * i, 150 + 30 * i), i % 2 == 1, i % 3,
            None if i % 2 else 3, None, 5 if i == 2 else None) for i in range(5)]
    add("find_lines", "find_lines", blk)
    add("find_lines", "find_lines", blk[:1], scores=True)
    for sk in ("auto", 2.5, -7.0):
        add("find_lines", "find_lines", [b + ((sk, 10.0) if i % 2 == 0 else (None,)) for i, b in enumerate(blk)], scores=True)
        add("find_lines", "find_lines", [blk[1] + (sk, 10.0 if sk != "auto" else 4.0)], scores=True)
    add("find_lines", "find_lines", [])
    add("find_lines", "find_lines", [blk[0][:1] + ((0, 0, 500, 10),) + blk[0][2:]])
    add("find_lines", "find_lines", [blk[0] + (50.0,)])
    add("find_lines", "find_lines", [blk[0] + (2.0, 5.0)])
    win = []
    for i, b in enumerate(blk):
        x0, y0, x1, y1 = b[1]
        ang = [3.0, -4.5, 10.0, 0.5, -1.0][i]
        (c, s), = new_ops.skew_cos_sin(new_ops.skew_table(ang, 10.0, b[2]))
        _, _, L, M = (float(a[0]) for a in new_ops.skew_frames(x1 - x0, y1 - y0, b[2], [(c, s)]))
        win.append(b + (ang, (2 + i, 1 + i, int(M) - 3, int(L) // 2 + i)))
    add("find_lines_window", "find_lines_window", win)
    add("find_lines_window", "find_lines_window", win[2:3])
    add("find_lines_window", "find_lines_window", [])
    add("find_lines_window", "find_lines_window", [win[0][:7] + ("auto", (0, 0, 5, 5))])
    add("find_lines_window", "find_lines_window", [win[0][:8] + ((0, 0, 10 ** 6, 5),)])
    curled = [(_img(rng, 300, 500, pitch=3), (5 + i, 7, 480 - 30 * i, 200 + 20 * i), i % 3, None, 2 if i == 1 else None, None,
               [None, 1, 4, 10][i]) for i in range(4)]
    for tables in (False, True):
        add("find_lines_curved", "find_lines_curved", curled, tables=tables)
        add("find_lines_curved", "find_lines_curved", curled[2:3], tables=tables)
    add("find_lines_curved", "find_lines_curved", [])
    add("find_lines_curved", "find_lines_curved", [curled[0][:6] + (40,)])
    add("find_lines_curved", "find_lines_curved", [curled[0][:6] + (0,)])

    pimg = [_img(rng, 260, 340, pitch=i % 2 * 6) for i in range(3)]
    PI = new_ops.PageItem
    for mask in range(16):
        opts = dict(rule_length=40 if mask & 1 else None, figure_size=0 if mask & 2 else None, directions=bool(mask & 4),
                    panel_size=12 if mask & 8 else None)
        pages = [PI(pimg[i], (5 * i, 3 * i, 300 - 20 * i, 250 - 10 * i), i == 1, i % 3, gap_x=None if i else 4,
                    **(opts if i != 2 else {})) for i in range(3)]
        add("find_blocks", "find_blocks", pages)
        add("find_blocks", "find_blocks", pages[:1], scores=True)
    for sk in ("auto", 3.0):
        pages = [PI(pimg[i], (5 * i, 3 * i, 300 - 20 * i, 250 - 10 * i), i == 1, i % 3, skew=sk if i != 1 else None,
                    max_skew=10.0 if sk != "auto" else 6.0) for i in range(3)]
        add("find_blocks", "find_blocks", pages, scores=True)
        add("find_blocks", "find_blocks", [tuple(p[:8]) for p in pages])
        add("find_blocks", "find_blocks", pages[2:])
    add("find_blocks", "find_blocks", [(pimg[0], (0, 0, 100, 100), False, A)])
    add("find_blocks", "find_blocks", [])
    add("find_blocks", "find_blocks", [PI(pimg[0], (0, 0, 100, 100), False, A, skew=2.0, rule_length=40)])
    add("find_blocks", "find_blocks", [PI(pimg[0], (0, 0, 100, 100), False, A, figure_size=1)])
    add("find_blocks", "find_blocks", [PI(pimg[0], (0, 0, 100, 100), False, A, directions=3)])
    add("find_blocks", "find_blocks", [PI(pimg[0], (0, 0, 100, 100), False, 7)])
    qimg = [_img(rng, 120 + 10 * i, 150 + 20 * i, pitch=i % 2) for i in range(4)]
    qpages = [(q, i % 3) for i, q in enumerate(qimg)]
    for spreads in ((), (0,), (3, 1), (0, 1, 2, 3)):
        add("find_page_quads", "find_page_quads", qpages, spreads=spreads)
        add("find_page_quads", "find_page_quads", qpages, hulls=True, labels=True, spreads=spreads)
    add("find_page_quads", "find_page_quads", qpages[1:2], spreads=(0,))
    add("find_page_quads", "find_page_quads", qpages[1:2], hulls=True)
    add("find_page_quads", "find_page_quads", [])
    add("find_page_quads", "find_page_quads", qpages, spreads=(4,))
    add("find_page_quads", "find_page_quads", qpages, spreads=(1, 1))
    add("find_page_quads", "find_page_quads", [(qimg[0], 5)])
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("old")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    old = load_old(a.old)
    mods = (old, new_ops)
    _lib.load = lambda: _Recorder()
    for m in mods:
        m.torch = _Torch()
        if not CUDA:
            m._stream = lambda: ctypes.c_void_p(0)
    if hasattr(old, "_table"):          # the old version's tables are uploaded by .to(device), which the proxy does not see
        orig = old._table
        old._table = lambda *a: _register(orig(*a), False)
    stats, lines = {}, []
    for builder, fn, args, kw in cases(np.random.default_rng(36)):
        got = [run(m, fn, args, kw) for m in mods]
        s = stats.setdefault(builder, dict(builder=builder, compared=0, reached=0, refused=0, mismatches=0, message_changes=0))
        s["compared"] += 1
        s["reached"] += bool(got[1]["calls"])
        s["refused"] += got[1]["ret"][0] == "raised"
        if fn == "figure_panels" and all(g["ret"][0] == "raised" for g in got) and got[0]["ret"][1] == got[1]["ret"][1] and \
                "must be a uint8 [., ., 3] tensor with dense pixels on" in got[0]["ret"][2] and \
                "must be a non-empty uint8 [h, w, 3] tensor with dense pixels on" in got[1]["ret"][2]:
            s["message_changes"] += 1          # the inline dense-pixel check became _dense_u8's, with its text
            continue
        if fn == "composite_regions_curved" and _slack_only(*got):
            s["slack_dropped"] = s.get("slack_dropped", 0) + 1
            continue
        if _key(got[0]) != _key(got[1]):
            s["mismatches"] += 1
            print(f"MISMATCH {builder} {fn}: old {_key(got[0])[:600]}\n  new {_key(got[1])[:600]}", file=sys.stderr)
    dev = torch.cuda.get_device_name() if CUDA else "cpu"
    for s in stats.values():
        lines.append(json.dumps(dict(s, device=dev)))
    text = "\n".join(lines) + "\n"
    print(text, end="")
    if a.out:
        with open(a.out, "w") as f:
            f.write(text)
    return 1 if any(s["mismatches"] for s in stats.values()) else 0


if __name__ == "__main__":
    sys.exit(main())
