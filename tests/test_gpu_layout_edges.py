"""The text-layout kernels at the edges of their contracts, bit for bit against the numpy twins on the inputs that
test_layout_edges.py builds and proves to reach those edges: tables filled exactly to their limits and one past them, the run
scratch at full capacity, 32767-pixel blocks and pages, exact skew ties, quad ties, union-find components built against the
tile grid, the link at its design bound and 65535 items in one call.

Each case is tagged with the features it reaches; the last test asserts that every REQUIRED feature was seen and every negative
control failed, and prints the kernel x feature table.  Large cases free their buffers before the next one and are skipped only
when torch.cuda.mem_get_info shows too little free memory."""
import collections

import numpy as np
import pytest
import torch

from oracle import blocks as B
from oracle import curled_blocks as C
from oracle import pages as P
from oracle import quad_pages as Q
from oracle import skewed_blocks as SB
from oracle import skewed_pages as SP
from test_layout_edges import (alternating_block, big_page_lines, bit31_block, chevron_block, choose_greater, component_images,
                               curve_lines_block, curve_runs_block, lattice_page, largest_quad_last, lines_block,
                               link_bound_block, min_index_labels, plus_grid, staircase_page, tie_hull_images,
                               uneven_strips_block, _rgb)

pytestmark = pytest.mark.gpu

SEEN = collections.defaultdict(collections.Counter)        # kernel -> feature -> cases
CONTROLS = {}                                               # control -> failed as it must
REQUIRED = {
    "find_lines": {"256 lines", "257 lines", "run scratch full, odd L", "run scratch full, even L", "32767-wide horizontal",
                   "32767-tall vertical", "65535 blocks", "32767 x 32767", "page > 2^31 bytes"},
    "find_lines_skewed": {"chevron tie", "largest search", "search one bin over", "page > 2^31 bytes"},
    "find_lines_window": {"frame corners", "whole frame", "empty pixel set", "44.9 degrees", "page > 2^31 bytes"},
    "find_blocks": {"page > 2^31 bytes", "65536 nodes", "65792 nodes", "host bound attained", "open at level 24", "1024 blocks", "1025 blocks",
                    "32767-wide level", "32767-wide vertical", "65535 pages"},
    "find_blocks_skewed": {"frame side 32767", "frame side 32768"},
    "find_page_quads": {"labels", "serpentine", "spiral", "comb", "diagonal contacts", "borders", "widths", "quad ties",
                        "65535 images"},
    "find_lines_curved": {"page > 2^31 bytes", "256 runs", "257 runs", "256 lines", "257 lines", "768 open + 256 runs", "strip 31 sample bit",
                          "uneven strips", "32 strips on 32767", "just under CURVE_MAX_WORK", "one block over"},
}
GIB = 1 << 30


def _dev():
    return torch.device("cuda:0")


def _need(nbytes):
    free = torch.cuda.mem_get_info(_dev())[0]
    if free < nbytes + GIB:
        pytest.skip(f"needs {nbytes + GIB} free bytes of device memory, {free} free")


def _up(img):
    return torch.from_numpy(np.ascontiguousarray(img)).to(_dev())


# ---- text blocks ---------------------------------------------------------------------------------------------------------
def _lines_call(items):
    """ops.find_lines over items (img, vertical, knobs) (each block its whole image); per item the device record and the twin's
    dict or error, the twin memoized by crop content."""
    from marconet_b200 import _lib, ops
    dimgs = {}
    args = []
    for img, v, knobs in items:
        if id(img) not in dimgs:
            dimgs[id(img)] = _up(img)
        d = dimgs[id(img)]
        args.append((d, (0, 0, img.shape[1], img.shape[0]), v, _lib.INK_AUTO, *knobs))
    rec = ops.find_lines(args).cpu().numpy().view(ops.block_lines_dtype())
    memo, out = {}, []
    for (img, v, knobs), r in zip(items, rec):
        key = (img.tobytes(), img.shape, v, tuple(knobs))
        if key not in memo:
            try:
                memo[key] = B.find_lines(img, (0, 0, img.shape[1], img.shape[0]), "vertical" if v else "horizontal", *knobs)
            except ValueError as e:
                memo[key] = dict(error=str(e))
        out.append((r, memo[key]))
    return out


def _same_lines(r, ref, what):
    from marconet_b200 import _lib
    n = int(r["n_lines"])
    if "error" in ref:
        assert n < 0 and f"{-n} lines exceed" in ref["error"], (what, n, ref)
        return n
    assert int(r["threshold"]) == ref["threshold"], what
    assert ("dark" if r["ink"] == _lib.INK_DARK else "light") == ref["ink"], what
    assert [tuple(int(x) for x in q) for q in r["rect"][:n]] == ref["lines"], (what, n, len(ref["lines"]))
    return n


def test_find_lines_at_the_line_limit():
    b256, b257 = lines_block(256), lines_block(257)
    out = _lines_call([(b256, False, [None] * 3), (b257, False, [None] * 3),
                       (np.ascontiguousarray(b256.transpose(1, 0, 2)), True, [None] * 3)])
    assert _same_lines(*out[0], "256") == 256
    assert _same_lines(*out[1], "257") == -257
    assert _same_lines(*out[2], "256 vertical") == 256
    with pytest.MonkeyPatch.context() as mp:
        mp.setattr(B, "MAX_LINES", 255)
        try:
            B.find_lines(b256, (0, 0, b256.shape[1], b256.shape[0]))
            CONTROLS["line limit written as >= 256"] = False
        except ValueError:
            CONTROLS["line limit written as >= 256"] = int(out[0][0]["n_lines"]) == 256
    SEEN["find_lines"].update({"256 lines": 1, "257 lines": 1})


def test_find_lines_run_scratch_and_32767_sides():
    """The run scratch of (L + 2) / 2 pairs filled to (L + 1) / 2 runs at L = 32767 and 32766, then a small block whose scratch
    lies right after theirs; a 32767-wide horizontal and a 32767-tall vertical block."""
    wide = lines_block(4, w=32767)
    tall = np.ascontiguousarray(lines_block(5, w=32767).transpose(1, 0, 2))
    small = lines_block(7)
    items = [(alternating_block(32767), False, [None] * 3), (alternating_block(32766), False, [None] * 3),
             (np.ascontiguousarray(alternating_block(32767).transpose(1, 0, 2)), True, [None] * 3),
             (small, False, [None] * 3), (wide, False, [None] * 3), (tall, True, [None] * 3), (small, False, [None] * 3)]
    out = _lines_call(items)
    for k, (r, ref) in enumerate(out):
        _same_lines(r, ref, k)
    assert int(out[3][0]["n_lines"]) == 7 and int(out[4][0]["n_lines"]) == 4 and int(out[5][0]["n_lines"]) == 5
    assert max(int(q[2]) for q in out[4][0]["rect"][:4]) == 32767 - 4 + 1      # the ink's extent to the last columns
    SEEN["find_lines"].update({"run scratch full, odd L": 1, "run scratch full, even L": 1, "32767-wide horizontal": 1,
                               "32767-tall vertical": 1})


def test_find_lines_65535_blocks():
    rng = np.random.default_rng(21)
    imgs = [lines_block(int(n), w=int(w)) for n, w in zip(rng.integers(0, 12, 13), rng.integers(9, 80, 13))]
    imgs += [_rgb(rng.random((int(h), int(w))) < 0.3) for h, w in zip(rng.integers(1, 40, 6), rng.integers(1, 40, 6))]
    items = [(imgs[k % len(imgs)], bool(k % 7 == 3), [None] * 3) for k in range(65535)]
    out = _lines_call(items)
    for k, (r, ref) in enumerate(out):
        _same_lines(r, ref, k)
    SEEN["find_lines"]["65535 blocks"] += 1


def test_32767_square_block_and_far_corner_crops_past_2_31_bytes():
    """A 32767 x 32767 block on a device-built page (2^20 tiles, about 2^29.6 pixels in the paper's bin) against the banded
    reference; then level, vertical, skewed, windowed and curled blocks and a page in the far corner of that page, past 2^31
    bytes, read through a view whose row guard bytes are ink: reading one would change a histogram."""
    from marconet_b200 import _lib, ops, pipeline
    H = W = 32767
    _need(H * (3 * W + 16) + (1 << 28))
    buf = torch.zeros((H, 3 * W + 16), dtype=torch.uint8, device=_dev())
    page = buf[:, :3 * W].view(H, W, 3)
    page.fill_(240)
    for a, b in big_page_lines(H, W):
        page[a:b, 100:W - 100] = 10
    X, Y = W - 1200, H - 700                           # the far corner: its first row starts past 2^31 bytes
    assert Y * buf.stride(0) > 2 ** 31
    corner = np.full((700, 1200, 3), 240, np.uint8)
    corner[649:, 900:] = lines_block(8, w=300)
    corner[300:500, 700:739] = lines_block(6, w=200).transpose(1, 0, 2)
    corner[441:, :358] = plus_grid(1024)
    page[Y:, X:] = torch.from_numpy(corner).to(_dev())

    def shift(lines, dx, dy):
        return [(a + dx, b + dy, c + dx, d + dy) for a, b, c, d in lines]

    rec = ops.find_lines([(page, (0, 0, W, H), False, _lib.INK_AUTO, None, None, None)]).cpu().numpy()
    ref = SB.find_lines_banded(lambda a, b: page[a:b].cpu().numpy(), H, W, rows=1024)
    assert _same_lines(rec.view(ops.block_lines_dtype())[0], ref, "32767 square") >= len(big_page_lines(H, W))
    SEEN["find_lines"]["32767 x 32767"] += 1

    A, V, G = (900, 649, 1200, 700), (700, 300, 739, 500), (0, 441, 358, 700)     # in the corner
    absl = [(X + a, Y + b, X + c, Y + d) for a, b, c, d in (A, V, G)]
    rec = ops.find_lines([(page, absl[0], False, _lib.INK_AUTO, None, None, None),
                          (page, absl[1], True, _lib.INK_AUTO, None, None, None)]).cpu().numpy().view(ops.block_lines_dtype())
    for r, rect, v in zip(rec, (A, V), (False, True)):
        want = B.find_lines(corner, rect, "vertical" if v else "horizontal")
        assert _same_lines(r, dict(want, lines=shift(want["lines"], X, Y)), (rect, v)) > 0
    SEEN["find_lines"]["page > 2^31 bytes"] += 1

    buf2, scores = ops.find_lines([(page, absl[0], False, _lib.INK_AUTO, None, None, None, 3.0, 10.0)], scores=True)
    host = buf2.cpu().numpy()
    osz = ops.block_lines_dtype().itemsize
    _same_skew(host[:osz].view(ops.block_lines_dtype())[0], host[osz:].view(ops.skew_block_dtype())[0], scores[0],
               SB.find_lines(corner, A, skew=3.0))
    SEEN["find_lines_skewed"]["page > 2^31 bytes"] += 1

    _, _, L, M = ops.skew_frames(300, 51, False, ops.skew_cos_sin([3.0]))
    win = (2, 1, int(M[0]) - 1, int(L[0]))
    r = ops.find_lines_window([(page, absl[0], False, _lib.INK_AUTO, None, None, None, 3.0, win)]).cpu().numpy()
    r = r.view(ops.block_lines_dtype())[0]
    want = SP.find_lines(corner, A, win, 3.0)
    n = int(r["n_lines"])
    assert n > 0 and int(r["threshold"]) == want["threshold"]
    assert [tuple(int(x) for x in q) for q in r["rect"][:n]] == want["detail"]["frame_lines"]
    SEEN["find_lines_window"]["page > 2^31 bytes"] += 1

    got = pipeline._find_blocks({0: page}, [(0, pipeline.TextPage(absl[2]), absl[2])])[0]
    want = P.find_blocks(corner, G)
    want = dict(want, blocks=shift(want["blocks"], X, Y), rejected=shift(want["rejected"], X, Y))
    assert _same_page(got, want, "corner page") == "ok" and len(got["blocks"]) == 1024
    SEEN["find_blocks"]["page > 2^31 bytes"] += 1

    cbuf, views = ops.find_lines_curved([(page, absl[0], _lib.INK_AUTO, None, None, None, 4)], tables=True)
    host = cbuf.cpu().numpy()
    cur = host[osz:].view(ops.curve_lines_dtype())[0]
    want = C.find_lines(corner, A, strips=4)["detail"]
    np.testing.assert_array_equal(views[0]["profiles"].cpu().numpy(), want["profiles"])
    np.testing.assert_array_equal(cur["header"], want["header"])
    np.testing.assert_array_equal(cur["lines"][:int(want["header"][1])], want["table"])
    assert int(want["header"][1]) == 8
    SEEN["find_lines_curved"]["page > 2^31 bytes"] += 1

    assert bool((buf[:, 3 * W:] == 0).all().item())
    del buf, page
    torch.cuda.empty_cache()


# ---- skewed blocks and windows -------------------------------------------------------------------------------------------
def _skew_call(img, skew, max_skew=10.0):
    from marconet_b200 import _lib, ops
    args = [(_up(img), (0, 0, img.shape[1], img.shape[0]), False, _lib.INK_AUTO, None, None, None, skew, max_skew)]
    buf, scores = ops.find_lines(args, scores=True)
    host = buf.cpu().numpy()
    osz = ops.block_lines_dtype().itemsize
    return host[:osz].view(ops.block_lines_dtype())[0], host[osz:].view(ops.skew_block_dtype())[0], scores[0]


def _same_skew(r, s, scores, ref):
    d = ref["detail"]
    assert int(s["chosen"]) == d["chosen"] and int(s["n_ang"]) == len(d["i"])
    assert (float(s["u_min"]), float(s["v_min"]), int(s["L"]), int(s["M"])) == d["frame"]
    if d["scores"] is not None:
        assert scores.cpu().tolist() == d["scores"]
    n = int(r["n_lines"])
    got = [tuple(int(x) for x in q) for q in r["rect"][:n]]
    assert got == (d["frame_lines"] if s["s"] != 0 else ref["lines"])


def test_skew_chevron_tie():
    """Every +-theta pair of the 801-angle search ties exactly; the least index wins, and the greater index must fail."""
    img = chevron_block()
    r, s, scores = _skew_call(img, "auto", 20.0)
    ref = SB.find_lines(img, (0, 0, img.shape[1], img.shape[0]), skew="auto", max_skew=20.0)
    _same_skew(r, s, scores, ref)
    d = ref["detail"]
    assert d["scores"][d["chosen"]] == d["scores"][800 - d["chosen"]] and d["chosen"] != 400
    CONTROLS["skew tie to the greater index"] = choose_greater(d["i"], d["scores"]) != int(s["chosen"])
    SEEN["find_lines_skewed"]["chevron tie"] += 1


def test_skew_search_at_the_profile_limit():
    """The tallest crop whose 801 angle profiles fit SKEW_MAX_PROFILE runs; one row more is refused before any launch."""
    from marconet_b200 import _lib, ops
    cs = ops.skew_cos_sin(ops.skew_table("auto", 20.0, False))
    w = 16
    h = ops.SKEW_MAX_PROFILE // 801
    while 801 * ops.skew_stride(w, h, False, cs) > ops.SKEW_MAX_PROFILE:
        h -= 1
    assert 801 * ops.skew_stride(w, h + 1, False, cs) > ops.SKEW_MAX_PROFILE
    img = np.full((h + 1, w, 3), 240, np.uint8)
    img[np.arange(h + 1) % 100 < 5, 3:13] = 10
    r, s, scores = _skew_call(img[:h], "auto", 20.0)
    _same_skew(r, s, scores, SB.find_lines(img[:h], (0, 0, w, h), skew="auto", max_skew=20.0))
    SEEN["find_lines_skewed"]["largest search"] += 1
    n0 = ops.LAUNCHES
    with pytest.raises(ValueError, match="profile values a skewed block may use"):
        ops.find_lines([(_up(img), (0, 0, w, h + 1), False, _lib.INK_AUTO, None, None, None, "auto", 20.0)])
    assert ops.LAUNCHES == n0
    SEEN["find_lines_skewed"]["search one bin over"] += 1


def test_windows_at_the_frame_corners_at_44_9_degrees():
    """Windows of one cell at each frame corner (whose pixel sets may be empty), the whole frame and a band, on a 32767-pixel
    crop at 44.9 degrees."""
    from marconet_b200 import _lib, ops
    rng = np.random.default_rng(23)
    h, w = 24, 32767
    img = _rgb(rng.random((h, w)) < 0.2)
    d = _up(img)
    _, _, L, M = ops.skew_frames(w, h, False, ops.skew_cos_sin([44.9]))
    L, M = int(L[0]), int(M[0])
    wins = [(0, 0, 1, 1), (M - 1, 0, M, 1), (0, L - 1, 1, L), (M - 1, L - 1, M, L), (0, 0, M, L), (M // 3, 0, M // 3 + 40, L)]
    args = [(d, (0, 0, w, h), False, _lib.INK_AUTO, None, None, None, 44.9, win) for win in wins]
    rec = ops.find_lines_window(args).cpu().numpy().view(ops.block_lines_dtype())
    empty = 0
    for win, r in zip(wins, rec):
        ref = SP.find_lines(img, (0, 0, w, h), win, 44.9)
        assert int(r["threshold"]) == ref["threshold"] and \
            ("dark" if r["ink"] == _lib.INK_DARK else "light") == ref["ink"], win
        n = int(r["n_lines"])
        assert [tuple(int(x) for x in q) for q in r["rect"][:n]] == ref["detail"]["frame_lines"], win
        empty += not SP.members(h, w, False, 44.9, win).any()
    assert empty >= 1
    SEEN["find_lines_window"].update({"frame corners": 1, "whole frame": 1, "empty pixel set": 1, "44.9 degrees": 1})


# ---- text pages ----------------------------------------------------------------------------------------------------------
def _pages_call(items):
    """pipeline._find_blocks over items (img, vertical, gaps, skew) (each page its whole image) -> per item (device, twin), the
    twin's error as dict(error)."""
    from marconet_b200 import pipeline
    dimgs = {}
    args = []
    for img, v, gaps, skew in items:
        if id(img) not in dimgs:
            dimgs[id(img)] = (len(dimgs), _up(img))
        args.append((dimgs[id(img)][0], pipeline.TextPage(None, "vertical" if v else "horizontal", "auto", *gaps, skew=skew),
                     (0, 0, img.shape[1], img.shape[0])))
    got = pipeline._find_blocks({i: d for i, d in dimgs.values()}, args)
    out = []
    for (img, v, gaps, skew), g in zip(items, got):
        try:
            if skew is None:
                ref = P.find_blocks(img, None, "vertical" if v else "horizontal", "auto", *gaps)
            else:
                ref = SP.find_blocks(img, None, "vertical" if v else "horizontal", "auto", *gaps, skew=skew)
        except ValueError as e:
            ref = dict(error=str(e))
        out.append((g, ref))
    return out


def _same_page(got, ref, what):
    if "error" in ref:
        assert isinstance(got, str) and ("nodes" in got) == ("nodes" in ref["error"]), (what, got, ref)
        assert ref["error"].split()[0] == got.split()[0], (what, got, ref)
        return "error"
    assert not isinstance(got, str), (what, got)
    det = ref.get("detail")
    if det is not None and det.get("frame") is not None:
        assert [b.window for b in got["blocks"]] == ref["blocks"], what
    else:
        assert [tuple(b.rect) for b in got["blocks"]] == ref["blocks"], what
    for key in ("rejected", "threshold", "ink", "text_size", "gap_x", "gap_y"):
        assert got[key] == ref[key], (what, key, got[key], ref[key])
    return "ok"


def test_pages_at_the_node_level_and_block_limits():
    """The 511 x 511 lattice (65536 nodes in a level) is accepted and 511 x 513 (65792) refused; a 31 x 31 lattice attains the
    host bound (h + 1) (w + 1) / 4; the staircase is still open at level 24; 1024 blocks are accepted and 1025 refused."""
    lat, lat_over, lat_small = lattice_page(256, 256), lattice_page(256, 257), lattice_page(16, 16)
    stair = staircase_page(30)
    g1 = (1, 1)
    items = [(lat, False, (None, None), None), (lat_over, False, (None, None), None), (lat_small, False, g1, None),
             (stair, False, g1, None), (stair, True, g1, None), (plus_grid(1024), False, (None, None), None),
             (plus_grid(1025), False, (None, None), None)]
    out = _pages_call(items)
    states = [_same_page(g, r, k) for k, (g, r) in enumerate(out)]
    assert states == ["ok", "error", "ok", "ok", "ok", "ok", "error"], states
    assert "65536 nodes" in out[1][0] and "1025 blocks" in out[6][0]
    assert len(out[5][0]["blocks"]) == 1024
    from marconet_b200 import ops
    assert ops.page_cap(31, 31) == 256 == len(P.xy_cut(B.grey(lat_small) < 128, False, 1, 1))
    with pytest.MonkeyPatch.context() as mp:
        mp.setattr(P, "MAX_NODES", 65535)
        try:
            P.find_blocks(lat)
            CONTROLS["node limit written as >="] = False
        except ValueError:
            CONTROLS["node limit written as >="] = not isinstance(out[0][0], str)
        mp.setattr(P, "MAX_NODES", 65536)
        mp.setattr(P, "LEVELS", 23)
        ref23 = P.find_blocks(stair, None, "horizontal", "auto", 1, 1)
        CONTROLS["23 levels"] = (ref23["rejected"], [tuple(b) for b in ref23["blocks"]]) != \
            (out[3][0]["rejected"], [tuple(b.rect) for b in out[3][0]["blocks"]])
    SEEN["find_blocks"].update({"65536 nodes": 1, "65792 nodes": 1, "host bound attained": 1, "open at level 24": 1,
                                "1024 blocks": 1, "1025 blocks": 1})


def _wide_page(w=32767):
    """A 40-row page of words of five plus signs (one column apart) 40 columns apart, the last word ending at column w - 1."""
    m = np.zeros((40, w), bool)
    x = w - 29
    while x >= 0:
        for k in range(5):
            for y in (4, 22):
                m[y + 2, x + 6 * k:x + 6 * k + 5] = True
                m[y:y + 5, x + 6 * k + 2] = True
        x -= 69
    return _rgb(m)


def test_pages_32767_wide_and_skewed_frame_sides():
    """32767-wide level and vertical pages (kChunk column chunks, the last kSpanWords word, int16 x1 = 32767); a skewed page
    whose frame side is exactly 32767, and one whose side is 32768, refused before any launch."""
    from marconet_b200 import _lib, ops
    page = _wide_page()
    cs = ops.skew_cos_sin([2.0])
    w, h = 400, 32767
    while max(ops.skew_page_frame(w + 1, h, False, cs)[:2]) <= 32767:
        w += 1
    assert max(ops.skew_page_frame(w, h, False, cs)[:2]) == 32767
    assert max(ops.skew_page_frame(w + 1, h, False, cs)[:2]) == 32768
    m = np.zeros((h, w + 1), bool)                     # paragraphs of ten 3-row lines, 12 rows apart, 60 rows between them
    y = np.arange(h)
    m[((y % 180) < 120) & ((y % 12) < 3), 3:w - 3] = True
    tall = _rgb(m)
    tilt = np.ascontiguousarray(tall[:, :w])
    out = _pages_call([(page, False, (None, None), None), (page, True, (None, None), None), (tilt, False, (None, None), 2.0)])
    for k, (g, r) in enumerate(out):
        assert _same_page(g, r, k) == "ok"
    assert max(b.rect[2] for b in out[0][0]["blocks"]) == 32767
    SEEN["find_blocks"].update({"32767-wide level": 1, "32767-wide vertical": 1})
    SEEN["find_blocks_skewed"]["frame side 32767"] += 1
    n0 = ops.LAUNCHES
    with pytest.raises(ValueError, match="a frame side of 32768 exceeds 32767"):
        ops.find_blocks([ops.PageItem(_up(tall), (0, 0, w + 1, h), False, _lib.INK_AUTO, skew=2.0)])
    assert ops.LAUNCHES == n0
    SEEN["find_blocks_skewed"]["frame side 32768"] += 1


def test_find_blocks_65535_pages():
    from marconet_b200 import ops, pipeline
    rng = np.random.default_rng(25)
    imgs = [plus_grid(1024)[:11, :28], lattice_page(3, 4), staircase_page(2), _rgb(rng.random((12, 17)) < 0.1),
            _rgb(np.zeros((3, 3), bool))]
    items = [(imgs[k % len(imgs)], bool(k % 3 == 1)) for k in range(65535)]
    assert sum(ops.page_bytes(im.shape[1], im.shape[0]) for im, _ in items) <= ops.PAGE_MAX_WORK
    dimgs = [_up(im) for im in imgs]
    args = [(k % len(imgs), pipeline.TextPage(None, "vertical" if v else "horizontal"), (0, 0, im.shape[1], im.shape[0]))
            for k, (im, v) in enumerate(items)]
    got = pipeline._find_blocks(dict(enumerate(dimgs)), args)
    memo = {}
    for k, ((im, v), g) in enumerate(zip(items, got)):
        key = (k % len(imgs), v)
        if key not in memo:
            memo[key] = P.find_blocks(im, None, "vertical" if v else "horizontal")
        _same_page(g, memo[key], k)
    SEEN["find_blocks"]["65535 pages"] += 1


# ---- perspective pages ---------------------------------------------------------------------------------------------------
def test_quad_labels_of_adversarial_components_and_tie_hulls():
    """Every pixel's compressed label is the smallest raster index of its 4-connected component and every root holds its
    component's size; the page, hull and largest quad are the brute force's, ties to the smallest (i, a, j, b)."""
    from marconet_b200 import _lib, ops
    comps, ties = component_images(), tie_hull_images()
    names = list(comps) + list(ties)
    imgs = [comps[k] for k in comps] + [ties[k] for k in ties]
    res, hulls, labels = ops.find_page_quads([(_up(im), _lib.INK_AUTO) for im in imgs], hulls=True, labels=True)
    res = res.cpu().numpy().view(ops.page_quad_dtype())
    for name, img, r, hull, (lab, cnt) in zip(names, imgs, res, hulls, labels):
        mask, t = Q.paper(img)
        want_lab, want_cnt = min_index_labels(mask)
        got_lab = lab.cpu().numpy()
        assert np.array_equal(got_lab, want_lab), name
        assert np.array_equal(cnt.cpu().numpy(), want_cnt), name
        ref = Q.find_corners(img)
        assert (int(r["threshold"]), int(r["label"]), int(r["size"])) == (ref["threshold"], ref["label"], ref["size"]), name
        n = int(r["n_hull"])
        assert [tuple(p) for p in hull.cpu().numpy()[:n]] == [tuple(p) for p in ref["hull"]], name
        assert int(r["area2"]) == ref["area2"] and tuple(int(v) for v in r["idx"]) == ref["idx"], name
        assert [tuple(int(v) for v in r["quad"][2 * m:2 * m + 2]) for m in range(4)] == [tuple(p) for p in ref["quad"]], name
        if name == "diagonal":
            eight, _ = min_index_labels(mask, np.ones((3, 3), int))
            CONTROLS["8-connected labels"] = not np.array_equal(got_lab, eight)
        if name in ties:
            last = largest_quad_last(ref["hull"])
            CONTROLS.setdefault("quad search keeping the last maximal tuple", True)
            CONTROLS["quad search keeping the last maximal tuple"] &= last[1] != tuple(int(v) for v in r["idx"])
            SEEN["find_page_quads"]["quad ties"] += 1
        else:
            SEEN["find_page_quads"][{"diagonal": "diagonal contacts"}.get(name, "widths" if name.startswith("width") else name)] += 1
    SEEN["find_page_quads"]["labels"] += 1


def test_find_page_quads_65535_images():
    from marconet_b200 import _lib, ops
    rng = np.random.default_rng(27)
    imgs = [_rgb(rng.random((int(h), int(w))) < 0.5, fg=240, bg=10) for h, w in zip(rng.integers(1, 20, 11),
                                                                                    rng.integers(1, 20, 11))]
    dimgs = [_up(im) for im in imgs]
    res = ops.find_page_quads([(dimgs[k % len(imgs)], _lib.INK_AUTO) for k in range(65535)]).cpu().numpy()
    res = res.view(ops.page_quad_dtype())
    refs = [Q.find_corners(im) for im in imgs]
    for k, r in enumerate(res):
        ref = refs[k % len(imgs)]
        assert (int(r["label"]), int(r["size"]), int(r["area2"])) == (ref["label"], ref["size"], ref["area2"]), k
        if ref["idx"] is not None:
            assert tuple(int(v) for v in r["idx"]) == ref["idx"], k
    SEEN["find_page_quads"]["65535 images"] += 1


# ---- curled blocks -------------------------------------------------------------------------------------------------------
def _curve_call(items):
    """ops.find_lines_curved over items (img, strips) (each block its whole image), every table compared with the twin's."""
    from marconet_b200 import _lib, ops
    dimgs = {}
    args = []
    for img, strips in items:
        if id(img) not in dimgs:
            dimgs[id(img)] = _up(img)
        d = dimgs[id(img)]
        args.append((d, (0, 0, img.shape[1], img.shape[0]), _lib.INK_AUTO, None, None, None, strips))
    n = len(args)
    buf, views = ops.find_lines_curved(args, tables=True)
    host = buf.cpu().numpy()
    ldt, cdt = ops.block_lines_dtype(), ops.curve_lines_dtype()
    rec, cur = host[:n * ldt.itemsize].view(ldt), host[n * ldt.itemsize:].view(cdt)
    memo, refs = {}, []
    for k, ((img, strips), r, c, v) in enumerate(zip(items, rec, cur, views)):
        key = (id(img), strips)
        if key not in memo:
            memo[key] = C.find_lines(img, (0, 0, img.shape[1], img.shape[0]), strips=strips)
        ref = memo[key]
        d = ref["detail"]
        assert int(r["threshold"]) == ref["threshold"], k
        np.testing.assert_array_equal(v["profiles"].cpu().numpy(), d["profiles"], err_msg=str(k))
        nr, rt = v["nruns"].cpu().numpy(), v["runs"].cpu().numpy()
        for j, runs in enumerate(d["runs"]):
            if isinstance(runs, int):
                assert nr[j] == runs, (k, j)
            else:
                assert nr[j] == len(runs) and [tuple(int(x) for x in q) for q in rt[j, :len(runs)]] == runs, (k, j)
        np.testing.assert_array_equal(c["header"], d["header"], err_msg=str(k))
        np.testing.assert_array_equal(c["lines"][:int(d["header"][1])], d["table"], err_msg=str(k))
        refs.append((c, ref))
    return refs


def test_curled_blocks_at_their_limits():
    wide = lines_block(4, w=32767, t=6, gap=10)
    items = [(curve_runs_block(256), 1), (curve_runs_block(257), 1), (curve_lines_block(256), 2), (curve_lines_block(257), 2),
             (link_bound_block(), 5), (bit31_block(), 32), (uneven_strips_block(np.random.default_rng(3)), 5), (wide, 32)]
    out = _curve_call(items)
    hd = [c["header"] for c, _ in out]
    assert hd[0][0] == C.OK and hd[0][1] == 256
    assert list(hd[1][[0, 3, 4]]) == [C.ERR_RUNS, 0, 257]
    assert hd[2][0] == C.OK and hd[2][1] == 256
    assert list(hd[3][[0, 4]]) == [C.ERR_LINES, 257]
    assert hd[4][0] == C.OK and hd[4][1] == 256
    assert (out[5][0]["lines"][:6, 5] == -1).all()
    assert hd[6][0] == C.OK and hd[6][1] >= 5
    assert hd[7][0] == C.OK and hd[7][1] == 4
    SEEN["find_lines_curved"].update({"256 runs": 1, "257 runs": 1, "256 lines": 1, "257 lines": 1, "768 open + 256 runs": 1,
                                      "uneven strips": 1, "32 strips on 32767": 1})


def test_strip_31_sample_bit_through_curve_lines():
    from marconet_b200 import pipeline
    img = bit31_block()
    blk = pipeline.TextBlock((0, 0, img.shape[1], img.shape[0]), curve="auto", strips=32)
    got = pipeline.find_lines([img], [[blk]])[0][0]
    ref = C.find_lines(img, blk.rect, strips=32)
    assert got["lines"] == ref["lines"] and got["curve"] == ref["curve"]
    assert (ref["detail"]["table"][:, 5] == -1).all()
    SEEN["find_lines_curved"]["strip 31 sample bit"] += 1


def test_curled_blocks_at_the_work_limit():
    """As many 4096-row blocks of 32 strips as CURVE_MAX_WORK holds run and equal the twin; one block more is refused before
    any launch."""
    from marconet_b200 import _lib, ops
    h, w = 4096, 1024
    per = ops.curve_block_bytes(w, h, 32)
    k = ops.CURVE_MAX_WORK // per
    assert k * per <= ops.CURVE_MAX_WORK < (k + 1) * per
    _need(ops.CURVE_MAX_WORK + 3 * h * w)
    img = np.full((h, w, 3), 240, np.uint8)
    img[:200] = lines_block(12, w=w, t=6, gap=10)[:200]
    d = _up(img)
    arg = (d, (0, 0, w, h), _lib.INK_AUTO, None, None, None, 32)
    buf = ops.find_lines_curved([arg] * k).cpu().numpy()
    ldt, cdt = ops.block_lines_dtype(), ops.curve_lines_dtype()
    cur = buf[k * ldt.itemsize:].view(cdt)
    ref = C.find_lines(img, (0, 0, w, h), strips=32)["detail"]
    nl = int(ref["header"][1])
    assert ref["header"][0] == C.OK and nl >= 6
    for c in cur:
        np.testing.assert_array_equal(c["header"], ref["header"])
        np.testing.assert_array_equal(c["lines"][:nl], ref["table"])
    SEEN["find_lines_curved"]["just under CURVE_MAX_WORK"] += 1
    del buf, cur
    n0 = ops.LAUNCHES
    with pytest.raises(ValueError, match=f"block {k}: the blocks up to this one need"):
        ops.find_lines_curved([arg] * (k + 1))
    assert ops.LAUNCHES == n0
    SEEN["find_lines_curved"]["one block over"] += 1
    del d
    torch.cuda.empty_cache()


# ---- coverage ------------------------------------------------------------------------------------------------------------
def test_coverage_and_negative_controls():
    feats = sorted({f for v in SEEN.values() for f in v} | {f for v in REQUIRED.values() for f in v})
    print("\nkernel x feature: cases")
    for k in REQUIRED:
        print(f"  {k:18s} " + "  ".join(f"{f}={SEEN[k][f]}" for f in feats if f in REQUIRED[k] or SEEN[k][f]))
    print("negative controls (failed as they must):", CONTROLS)
    for k, want in REQUIRED.items():
        assert want <= {f for f, n in SEEN[k].items() if n}, (k, want - set(SEEN[k]))
    assert set(CONTROLS) == {"line limit written as >= 256", "8-connected labels", "quad search keeping the last maximal tuple",
                             "skew tie to the greater index", "23 levels", "node limit written as >="}, CONTROLS
    assert all(CONTROLS.values()), CONTROLS
