"""The page options' kernels at the edges of their contracts, on the host: seeded generators for every input that
test_gpu_option_edges.py gives the device, each shown in the numpy twins (oracle/ruled_pages.py, figure_pages.py,
mixed_pages.py, panel_pages.py, light.py, flat_pages.py) to reach the edge it is tagged with.  The cases too large for a twin
in the device test are checked here against either a closed form (the all-ink page, the page of 1024 full-height figures) or a
windowed reference (a crop rectangle in a page's far corner, the evening of a crop with a margin of 2 (k // 2)), both proved
equal to the whole-page twin at moderate sizes."""
import numpy as np
import pytest

from oracle import blocks as B
from oracle import figure_pages as FP
from oracle import flat_pages as F
from oracle import light as L
from oracle import mixed_pages as MP
from oracle import panel_pages as PP
from oracle import ruled_pages as RP

from test_layout_edges import _rgb

PAPER = 240


def _grey_img(g):
    """A uint8 [h, w, 3] image of the grey values g (every channel g, so B.grey gives g back)."""
    return np.repeat(np.asarray(g, np.uint8)[..., None], 3, axis=2)


# ---- rules ---------------------------------------------------------------------------------------------------------------
def straddle_runs(l, w):
    """(first bit, length) of the runs straddle_mask draws along a line of w >= 2049 bits for rule length l: a run of l and one
    of l - 1 whose first bit is 1023, the same pair whose last bit is 1024 ceil(l / 1024), a pair whose first bit is 2047
    (when w allows), and a run over bits [1000, 2100) that spans the whole iteration of words 32 .. 63 with no zero."""
    e = 1024 * -(-l // 1024)
    out = [(1023, l), (1023, l - 1), (e + 1 - l, l), (e + 2 - l, l - 1)]
    if 2047 + l <= w:
        out += [(2047, l), (2047, l - 1)]
    return out + [(1000, max(1100, l))]


def straddle_mask(l, w, h=33):
    """A boolean [h, w] page whose odd rows 1, 3, .. hold straddle_runs(l, w), one run each, and a dot row at the bottom."""
    m = np.zeros((h, w), bool)
    for k, (a, n) in enumerate(straddle_runs(l, w)):
        m[1 + 2 * k, max(0, a):a + n] = True
    m[h - 1, ::3] = True
    return m


def straddle_pages():
    """(name, image, rule length): straddle pages along rows and (transposed) along columns, with w and h both = 1 (mod 32) and
    both = 0 (mod 32), and rule lengths 2, 40 and 1500 (a run of 1500 from bit 1023 crosses bits 1024 and 2048)."""
    out = []
    for l in (2, 40, 1500):
        for w, h in ((3073, 33), (3072, 32)):
            m = straddle_mask(l, w, h)
            out.append((f"rows l={l} {w}x{h}", _rgb(m), l))
            out.append((f"columns l={l} {h}x{w}", _rgb(np.ascontiguousarray(m.T)), l))
    return out


def line_pages():
    """(name, image, rule length): a 1 x 5000 page and a 5000 x 1 page with runs of 40 and 39 straddling bits 1024 and 2048,
    and a 3 x 32767 page of a run of 32767, one of 32766 and a dotted row under rule length 32767."""
    m = np.zeros(5000, bool)
    m[1000:1040] = m[2030:2069] = m[3000:3003] = True
    n = np.zeros((3, 32767), bool)
    n[0] = True
    n[1, 1:] = True
    n[2, ::3] = True
    return [("1 x 5000", _rgb(m[None, :]), 40), ("5000 x 1", _rgb(m[:, None]), 40), ("3 x 32767", _rgb(n), 32767)]


def test_straddle_runs_reach_the_iteration_boundaries():
    """Each run of l crosses a multiple of 1024 and is in U; the same run one pixel shorter is not; the run over [1000, 2100)
    covers words 32 .. 63 whole; the same holds along the columns of the transposed pages."""
    for name, img, l in straddle_pages():
        cols = name.startswith("columns")
        ink = B.grey(img) <= B.otsu(B.grey(img))
        if cols:
            ink = ink.T
        U = RP.rule_pixels(ink, l)
        w = ink.shape[1]
        assert (w % 32) in (0, 1) and (ink.shape[0] % 32) == (w % 32)
        for k, (a, n) in enumerate(straddle_runs(l, w)):
            row = U[1 + 2 * k]
            assert ink[1 + 2 * k].sum() == n
            assert row.sum() == (n if n >= l else 0), (name, a, n)
            assert a // 1024 != (a + n - 1) // 1024 or n < 2, (name, a, n)        # it straddles bit 1024 k
        assert U[1 + 2 * len(straddle_runs(l, w)) - 2, 1024:2048].all()            # a whole iteration with no zero
        assert not U[-1].any() or l <= 1
        want = RP.find_blocks(img, polarity="dark", rule_length=l)
        assert want["rule_pixels"] == int(U.sum()) > 0


def test_line_pages_are_ruled_as_the_twin_says():
    for name, img, l in line_pages():
        res = RP.find_blocks(img, polarity="dark", rule_length=l)
        assert res["rule_pixels"] == (40 if l == 40 else 32767), name
    # one pixel more rule length takes the run of 40 out of U: the control's comparison fails
    assert RP.find_blocks(line_pages()[0][1], polarity="dark", rule_length=41)["rule_pixels"] == 0


def all_ink_expected(n, **opts):
    """The closed form of the twin on the all-ink n x n page (grey 0, polarity dark) with the options of
    panel_pages.find_blocks: rules with rule length 2 or n take every pixel into U and leave no leaf; without rules, the one
    leaf is the whole page, S = n, and it is a panel (panels), else a figure (figure size n), and nothing is left for pass 2."""
    out = dict(blocks=[], rejected=[], threshold=0, ink="dark", text_size=0, gap_x=0, gap_y=0)
    if opts.get("rules"):
        out.update(rule_length=opts["rule_length"], rule_pixels=n * n)
    if opts.get("figures"):
        out.update(figure_size=0, figures=[])
    if opts.get("block_direction"):
        out.update(block_direction="auto", undecided=[], directions=[])
    out.update(panel_size=0, panels=[], polarities=[])
    if opts.get("rules"):
        return out
    out.update(text_size=n, gap_x=n, gap_y=max(1, n // 2), panel_size=n, panels=[(0, 0, n, n)])
    if opts.get("figures"):
        out.update(figure_size=opts.get("figure_size") or 3 * n)
    return out


def all_ink_figure_expected(n):
    """The closed form of the figure twin (no panels) on the all-ink n x n page with figure size n: the page is its figure."""
    return dict(blocks=[], rejected=[], threshold=0, ink="dark", text_size=n, gap_x=n, gap_y=max(1, n // 2), figure_size=n,
                figures=[(0, 0, n, n)])


ALL_INK_OPTIONS = [dict(rules=True, rule_length=2), dict(rules=True, rule_length="n", figures=True, figure_size="n",
                                                           block_direction=True),
                   dict(), dict(figures=True, figure_size="n")]


def _opts(o, n):
    return {k: n if v == "n" else v for k, v in o.items()}


@pytest.mark.parametrize("n", [2, 33, 97])
def test_all_ink_closed_form_equals_the_twin(n):
    img = np.zeros((n, n, 3), np.uint8)
    assert B.otsu(B.grey(img)) == 0
    for o in ALL_INK_OPTIONS:
        o = _opts(o, n)
        got = PP.find_blocks(img, polarity="dark", **o)
        assert got == all_ink_expected(n, **o), o
    assert FP.find_blocks(img, polarity="dark", figure_size=n) == all_ink_figure_expected(n)
    r = RP.find_blocks(img, polarity="dark", rule_length=2)
    assert r["rule_pixels"] == n * n and r["blocks"] == []


def figure_columns(H, n=1024):
    """n figures of 2 x H pixels, one column apart: with figure size 2 every column is a figure, and the figure rows painted
    (frows) are n H, the most n figures of a page H tall can have."""
    m = np.zeros((H, 3 * n - 1), bool)
    for k in range(n):
        m[:, 3 * k:3 * k + 2] = True
    return _rgb(m)


def figure_columns_expected(H, n=1024):
    return dict(blocks=[], rejected=[], threshold=10, ink="dark", text_size=H, gap_x=H, gap_y=max(1, H // 2),
                figure_size=2, figures=[(3 * k, 0, 3 * k + 2, H) for k in range(n)])


@pytest.mark.parametrize("H", [3, 40, 129])
def test_figure_columns_closed_form(H):
    img = figure_columns(H, 64)
    got = FP.find_blocks(img, polarity="dark", figure_size=2)
    assert got == figure_columns_expected(H, 64)
    assert sum(y1 - y0 for _, y0, _, y1 in got["figures"]) == 64 * H


def figure_word_rects(w):
    return [(4, 30), (31, 60), (64, 96)] + [(x, x + 32) for x in range(128, w - 100, 64)] + [(w - 45, w)]


def figure_word_page(w=32767):
    """A 60 x w page: small plus signs (S = 5), solid figures [4, 30) and [31, 60) sharing bitmap word 0, [64, 96) exactly
    word 2, one word each at 128 + 64 j (enough ink that their rows stay non-white on a 32767-wide page) and one ending at
    x = w in the page's last word.  With figure size 20 the solids are the figures; with 2, every piece of at least 2 x 2 is."""
    m = np.zeros((60, w), bool)
    for x0, x1 in figure_word_rects(w):
        m[2:30, x0:x1] = True
    for x in range(4, w - 60, 9):
        m[44, x:x + 5] = True
        m[42:47, x + 2] = True
    return _rgb(m)


def test_figure_word_page_reaches_its_words():
    img = figure_word_page(400)
    got = FP.find_blocks(img, polarity="dark", figure_size=20)
    assert got["figures"] == [(a, 2, b, 30) for a, b in figure_word_rects(400)]
    assert got["figures"][:3] == [(4, 2, 30, 30), (31, 2, 60, 30), (64, 2, 96, 30)] and got["figures"][-1][2] == 400
    assert got["text_size"] == 5 and got["blocks"]
    assert 29 // 32 == 31 // 32 and (64 // 32, 95 // 32) == (2, 2)
    small = FP.find_blocks(img, polarity="dark", figure_size=2)
    assert len(small["figures"]) > 4 and small["figure_size"] == 2


# ---- panels --------------------------------------------------------------------------------------------------------------
def _plus(g, x, y, n, v):
    g[y + n // 2, x:x + n] = v
    g[y:y + n, x + n // 2] = v


def panel_word_page():
    """A 140 x 260 page of 15-pixel plus signs (S = 15): dark panels [4, 30) and [31, 60) sharing bitmap word 0, each with a
    white plus sign 2 pixels from its outline, a 2-pixel-wide panel at [70, 72) and a 2-row panel at rows [80, 82).  Panel
    size 2."""
    g = np.full((140, 260), PAPER, np.int64)
    g[4:40, 4:30] = g[4:40, 31:60] = 30
    _plus(g, 7, 7, 15, PAPER)
    _plus(g, 34, 20, 15, PAPER)
    g[4:40, 70:72] = 30
    g[80:82, 100:140] = 30
    for x in range(4, 240, 20):
        _plus(g, x, 110, 15, 30)
    return _grey_img(g)


def test_panel_word_page():
    img = panel_word_page()
    got = PP.find_blocks(img, panel_size=2)
    assert {(4, 4, 30, 40), (31, 4, 60, 40), (70, 4, 72, 40), (100, 80, 140, 82)} <= set(got["panels"]), got["panels"]
    assert "light" in got["polarities"] and 29 // 32 == 31 // 32


def panel_rule_page():
    """A 100 x 600 page: a 60 x 200 dark panel at (200, 20) with a white mark at its column 60 on rows 45 .. 55; a horizontal
    rule from x = 10 into the panel at row 50, whose run goes on to the mark, so its last 60 U pixels lie inside the panel
    (rule length 250, above the panel's sides).  The panel stays one leaf."""
    g = np.full((100, 600), PAPER, np.int64)
    g[20:80, 200:400] = 30
    g[45:56, 260] = PAPER
    g[50, 10:200] = 30
    for x in range(20, 580, 9):
        g[92, x:x + 5] = 30
        g[90:95, x + 2] = 30
    return _grey_img(g)


def test_panel_rule_page_has_rule_pixels_inside_its_panel():
    img = panel_rule_page()
    got = PP.find_blocks(img, rules=True, rule_length=250, panel_size=20)
    assert got["panels"] == [(200, 20, 400, 80)]
    I = B.grey(img) <= got["threshold"]
    U = RP.rule_pixels(I, 250)
    assert U[50, 10:260].all() and not U[50, 260:].any() and U[21:79, 201:399].sum() == 59


def flat_panel(counts, h=20, base=None, shuffle=False):
    """A grey leaf of h x w (w = sum(counts) / h) filled in raster order with counts[g] pixels of each grey g, on a page of
    paper 240 with plus signs to give S; returns the page and the leaf's rectangle."""
    vals = np.concatenate([np.full(c, g, np.int64) for g, c in counts.items()])
    w = len(vals) // h
    assert w * h == len(vals)
    if shuffle:
        vals = np.random.default_rng(7).permutation(vals)
    g = np.full((h + 40, w + 40), PAPER, np.int64) if base is None else base
    g[10:10 + h, 10:10 + w] = vals.reshape(h, w)
    for x in range(10, w + 30, 9):
        g[h + 30, x:x + 5] = 20
        g[h + 28:h + 33, x + 2] = 20
    return _grey_img(g), (10, 10, 10 + w, 10 + h)


def flat_pages():
    """(name, page, leaf, panel?) pairs pinning the panel test: the flat radius (m + 8 counts and m + 9 does not, the same for
    m - 8 / m - 9), the mode at grey 0 and at grey 255 (a light-ink page), a tied mode that goes to the smaller grey, and a
    leaf of exactly half ink against half + 1."""
    A = 400                                              # 20 x 20 leaves; a flat count of 201 is a panel, 200 is not
    out = []
    for d, want in ((8, True), (9, False), (-8, True), (-9, False)):
        out.append((f"m{d:+d}", *flat_panel({60: 198, 60 + d: 3, 20: 40, 25: 40, 30: 40, 35: 39, 95: 40}), want))
    out.append(("mode 0", *flat_panel({0: 190, 8: 11, 20: 80, 30: 80, 9: 39}), True))
    out.append(("mode 0, 9 out", *flat_panel({0: 190, 9: 11, 20: 80, 30: 80, 40: 39}), False))
    dark = np.full((60, 60), 15, np.int64)               # light ink on dark paper: grey 255 fills are ink
    out.append(("mode 255", *flat_panel({255: 190, 247: 11, 200: 80, 190: 80, 180: 39}, base=dark.copy()), True))
    out.append(("mode 255, 246 out", *flat_panel({255: 190, 246: 11, 200: 80, 190: 80, 180: 39}, base=dark.copy()), False))
    out.append(("tie to the smaller", *flat_panel({40: 150, 200: 150, 45: 100}, shuffle=True), True))
    assert A == 400
    return out


def half_ink_pages():
    """A 20 x 20 checkerboard of greys 100 (ink) and 108 (not) on paper 108 with dark plus signs: exactly half ink, no panel;
    with one more ink pixel, a panel (flat: both greys are within 8 of the mode)."""
    out = []
    for extra, want in ((0, False), (1, True)):
        g = np.full((60, 60), 108, np.int64)
        y, x = np.mgrid[0:20, 0:20]
        g[10:30, 10:30] = np.where((x + y) % 2 == 0, 100, 108)
        if extra:
            g[10, 11] = 100
        for c in range(10, 50, 9):
            g[50, c:c + 5] = 100
            g[48:53, c + 2] = 100
        out.append((f"half + {extra}", _grey_img(g), (10, 10, 30, 30), want))
    return out


def _mode_to_larger(g, leaf):
    x0, y0, x1, y1 = leaf
    hist = np.bincount(g[y0:y1, x0:x1].reshape(-1), minlength=256)
    m = 255 - int(np.argmax(hist[::-1]))
    return 2 * int(hist[max(0, m - PP.FLAT):m + PP.FLAT + 1].sum()) > (y1 - y0) * (x1 - x0)


def test_flat_pages_flip_on_one_pixel():
    for name, img, leaf, want in flat_pages() + half_ink_pages():
        got = PP.find_blocks(img, panel_size=20)
        assert (leaf in [(a - 0, b, c, d) for a, b, c, d in got["panels"]]) == want, (name, got["panels"])
        g = B.grey(img)
        if name.startswith("m+9") or name.startswith("m-9"):
            assert PP.flat.__defaults__ is None
            hist = np.bincount(g[10:30, 10:30].reshape(-1), minlength=256)
            assert 2 * int(hist[60 - 9:60 + 10].sum()) > 400          # a radius of 9 would make it a panel
        if name == "tie to the smaller":
            assert PP.flat(g, leaf) and not _mode_to_larger(g, leaf)


def test_panel_outline_stops_growth():
    """On the panel word page, a block inside a panel stops growing at the outline: growth without the outline differs."""
    img = panel_word_page()
    got = PP.find_blocks(img, panel_size=2)
    assert _outline_control(img, got) is True


def _outline_control(img, got):
    """Whether growing the panel page's blocks with its rules alone (the panels' outlines left out of the layout) changes a
    block the twin gives: the twin's blocks depend on the outline."""
    g = B.grey(img)
    I = g <= got["threshold"] if got["ink"] == "dark" else g > got["threshold"]
    q = (min(got["gap_x"], got["gap_y"]) - 1) // 2
    for (x0, y0, x1, y1), pol in zip(got["blocks"], got["polarities"]):
        if pol == "auto":
            continue
        inner = [p for p in got["panels"] if p[0] <= x0 and p[1] <= y0 and x1 <= p[2] and y1 <= p[3]][0]
        J = ~I
        sub = J[inner[1] + 1:inner[3] - 1, inner[0] + 1:inner[2] - 1]
        ys, xs = np.nonzero(sub)
        leaf = (inner[0] + 1 + xs.min(), inner[1] + 1 + ys.min(), inner[0] + 2 + xs.max(), inner[1] + 2 + ys.max())
        if RP._grow(np.zeros_like(I), leaf, q) != (x0, y0, x1, y1):
            return True
    return False


# ---- directions ----------------------------------------------------------------------------------------------------------
def tall_leaf(H=32767, w=40):
    """A w x H page of 3-row bars every 8 rows from row 0 and a single-row bar at row H - 1: one block H tall whose row bands
    start at index 0 and end at index H - 1."""
    m = np.zeros((H, w), bool)
    m[np.arange(H) % 8 < 3] = True
    m[H - 1] = True
    m[H - 5:H - 1] = False
    return _rgb(m)


def _diag(h, w, phase=0):
    y, x = np.mgrid[0:h, 0:w]
    return (x + y + phase) % 3 == 0


def tie_pages(s=600):
    """(rule, image): pages whose one block ties A = B under each of the four direction rules: a square of one band each way
    (w = h); vertical stripes (one row band, 2 b_c = h); horizontal stripes (one column band, w = 2 b_r); and a 3 x 5 grid of
    patches with 10-pixel gaps (G_y (n_c - 1) = 20 * 4 = G_x (n_r - 1) = 40 * 2).  Patches are diagonal hatching, under half
    ink, so every row and column of a band is non-white."""
    out = [("one band each", _rgb(_diag(s, s)))]
    m = np.zeros((2 * s, 3 * s + 20), bool)
    for k in range(3):
        m[:, k * (s + 10):k * (s + 10) + s] = _diag(2 * s, s)
    out.append(("one row band", _rgb(m)))
    out.append(("one column band", _rgb(np.ascontiguousarray(m.T))))
    p = s // 2
    m = np.zeros((3 * p + 20, 5 * p + 40), bool)
    for r in range(3):
        for c in range(5):
            m[r * (p + 10):r * (p + 10) + p, c * (p + 10):c * (p + 10) + p] = _diag(p, p)
    out.append(("grid", _rgb(m)))
    return out


def test_tie_pages_tie_under_each_rule():
    rules = []
    for name, img in tie_pages():
        got = MP.find_blocks(img)
        assert len(got["blocks"]) == 1, (name, got["blocks"])
        assert got["undecided"] == [0], name
        ink = B.grey(img) <= got["threshold"]
        x0, y0, x1, y1 = got["blocks"][0]
        leaf = got["blocks"][0]
        (nr, _, _), (nc, _, _) = MP.leaf_bands(ink, np.zeros_like(ink), leaf)
        rules.append((nr > 1, nc > 1))
    assert rules == [(False, False), (False, True), (True, False), (True, True)]


def test_tall_leaf_bands_from_0_to_the_last_index():
    img = tall_leaf(4099)
    got = MP.find_blocks(img)
    assert got["blocks"] == [(0, 0, 40, 4099)] and got["directions"] == ["horizontal"]
    ink = B.grey(img) <= got["threshold"]
    rows = ink.sum(axis=1) > 0
    assert rows[0] and rows[-1] and not rows[-2]


# ---- windowed references -------------------------------------------------------------------------------------------------
def corner_content():
    """A 700 x 1200 crop of paper 240 and grey 30: a ruled table, a dark panel with white plus signs, a hatched figure and
    dark plus signs."""
    g = np.full((700, 1200), PAPER, np.int64)
    for y in range(60, 300, 60):
        g[y, 60:660] = 30
    for x in range(60, 661, 150):
        g[60:241, x] = 30
    g[360:520, 60:600] = 30
    for y in range(380, 500, 40):
        for x in range(80, 560, 30):
            _plus(g, x, y, 15, PAPER)
    g[320:550, 700:1140][_diag(230, 440)] = 30
    for y in range(560, 660, 25):
        for x in range(60, 1140, 20):
            _plus(g, x, y, 15, 30)
    return _grey_img(g)


CORNER_OPTS = dict(polarity="dark", rules=True, rule_length=600, figures=True, figure_size=150, block_direction=True,
                   panel_size=60)


def shifted(res, dx, dy):
    def sh(r):
        return (r[0] + dx, r[1] + dy, r[2] + dx, r[3] + dy)
    out = dict(res, blocks=[sh(b) for b in res["blocks"]], rejected=[sh(b) for b in res["rejected"]])
    for key in ("figures", "panels"):
        if key in out:
            out[key] = [sh(b) for b in out[key]]
    return out


def test_corner_crop_of_a_page_is_the_crop_shifted():
    """The twin of a page's crop rectangle is the twin of the crop alone, shifted: the device reads the far corner of a page
    past 2^31 bytes through such a rectangle."""
    c = corner_content()
    page = np.full((900, 1500, 3), PAPER, np.uint8)
    page[200:, 300:] = c
    ref = PP.find_blocks(c, **CORNER_OPTS)
    assert PP.find_blocks(page, rect=(300, 200, 1500, 900), **CORNER_OPTS) == shifted(ref, 300, 200)
    assert ref["rule_pixels"] > 0 and ref["panels"] and ref["figures"] and "light" in ref["polarities"]
    assert len(ref["blocks"]) >= 3


def light_margin(H, W, k, box):
    """The crop (x0, y0, x1, y1) of an H x W page that the windowed reference of ``box`` reads: box with a margin of 2 (k // 2)
    cut to the page.  The closing at a pixel reads the max filter within k // 2, which reads pixels within k // 2 of those."""
    x0, y0, x1, y1 = box
    m = 2 * (k // 2)
    return max(0, x0 - m), max(0, y0 - m), min(W, x1 + m), min(H, y1 + m)


def light_window_reference(crop, crop_rect, k, polarity, box):
    """L.even of the whole page restricted to ``box``, from its crop (light_margin) at crop_rect alone."""
    a, b = crop_rect[:2]
    x0, y0, x1, y1 = box
    return L.even(crop, k, polarity)[y0 - b:y1 - b, x0 - a:x1 - a]


def test_light_window_reference_equals_the_whole_page_twin():
    rng = np.random.default_rng(5)
    page = rng.integers(0, 256, (300, 420, 3), dtype=np.uint8)
    for k in (3, 5, 31):
        for pol in ("dark", "light"):
            whole = L.even(page, k, pol)
            for box in ((0, 0, 40, 30), (380, 270, 420, 300), (100, 100, 160, 140), (0, 250, 420, 300)):
                a, b, c, d = cr = light_margin(300, 420, k, box)
                np.testing.assert_array_equal(light_window_reference(page[b:d, a:c], cr, k, pol, box),
                                              whole[box[1]:box[3], box[0]:box[2]])


def light_edge_sizes(k):
    """The sides n = k // 2, k // 2 + 1, k - 1, k and k + 1 of a window k: the segment and skip branches of the passes."""
    r = k // 2
    return [r, r + 1, k - 1, k, k + 1]


def _closing_brute(page, k):
    r = k // 2
    h, w = page.shape[:2]
    mx = np.empty_like(page)
    for y in range(h):
        for x in range(w):
            mx[y, x] = page[max(0, y - r):y + r + 1, max(0, x - r):x + r + 1].reshape(-1, page.shape[2]).max(axis=0)
    out = np.empty_like(page)
    for y in range(h):
        for x in range(w):
            out[y, x] = mx[max(0, y - r):y + r + 1, max(0, x - r):x + r + 1].reshape(-1, page.shape[2]).min(axis=0)
    return out


@pytest.mark.parametrize("k", [5, 7])
def test_light_edge_sizes_close_as_the_definition(k):
    """At every pair of edge sides the twin's closing is the brute-force min of maxes over the window cut to the page, and a
    window of k + 2 gives another page (the control)."""
    rng = np.random.default_rng(k)
    differ = 0
    for h in light_edge_sizes(k):
        for w in light_edge_sizes(k):
            page = rng.integers(0, 256, (h, w, 3), dtype=np.uint8)
            np.testing.assert_array_equal(L.closing(page, k), _closing_brute(page, k))
            differ += not np.array_equal(L.even(page, k, "dark"), L.even(page, k + 2, "dark"))
    assert differ > 0


def flat_lines(h, w, n=10, seed=4):
    """A line table of n curled lines across [0, w) down an h-row frame."""
    rng = np.random.default_rng(seed)
    rows = []
    for k in range(n):
        y = 20.0 + (h - 40) * k / max(1, n - 1)
        mu = (y, y + rng.uniform(-6, 6), y + rng.uniform(-6, 6), y + rng.uniform(-6, 6))
        rows.append((1.0, float(w - 2), *mu, (((mu[0] + mu[1]) + mu[2]) + mu[3]) / 4, 0.0, float(w)))
    return np.array(sorted(rows, key=lambda r: r[6]), np.float64)


def test_flat_lines_bend_the_field():
    t = flat_lines(32767, 64)
    src = F.field(t, 64, 200)
    assert not np.array_equal(src[:, 10], np.arange(200) + 0.5)
