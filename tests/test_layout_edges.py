"""The text-layout twins at the edges of the kernels' contracts, without a GPU: every input tests/test_gpu_layout_edges.py
builds is made here by a seeded generator, and each test shows that the input reaches its edge in the numpy twin (a table
filled exactly to its limit and one past it, a tie that only the tie rule decides, a level still open at the last level).
The GPU file then compares the kernels with the twins on exactly these inputs."""
import numpy as np
import pytest
from scipy import ndimage

from oracle import blocks as B
from oracle import curled_blocks as C
from oracle import pages as P
from oracle import quad_pages as Q
from oracle import skewed_blocks as SB

INK, PAPER = 10, 240


def _rgb(mask, fg=INK, bg=PAPER):
    """A uint8 [h, w, 3] image: fg where mask, bg elsewhere."""
    return np.where(np.asarray(mask, bool)[..., None], np.uint8(fg), np.uint8(bg)).repeat(3, axis=2)


def _ink(img):
    g = B.grey(img)
    t = B.otsu(g)
    return g <= t


# ---- generators ----------------------------------------------------------------------------------------------------------
def lines_block(n, w=40, t=3, gap=3):
    """n level lines t rows thick, gap rows apart (and from the borders): exactly n kept lines in the twin."""
    m = np.zeros((n * (t + gap) + gap, w), bool)
    for k in range(n):
        m[gap + k * (t + gap):gap + k * (t + gap) + t, 4:w - 4] = True
    return _rgb(m)


def alternating_block(L, w=16):
    """L rows whose profile has the most runs a profile of L bins can hold, (L + 1) // 2, the first and the last row inked: every
    even row for odd L; for even L every even row up to L - 4, then row L - 1."""
    m = np.zeros((L, w), bool)
    m[0:L - 1 if L % 2 == 0 else L:2] = True
    if L % 2 == 0:
        m[L - 2] = False
        m[L - 1] = True
    return _rgb(m)


def lattice_page(ny, nx):
    """Isolated pixels at every even (y, x) of a (2 ny - 1) x (2 nx - 1) page: ny nx nodes in one level of the XY-cut."""
    m = np.zeros((2 * ny - 1, 2 * nx - 1), bool)
    m[::2, ::2] = True
    return _rgb(m)


def staircase_page(n_bars, t=2, gap=3):
    """Nested L-shaped bars: a bar across the top of the remaining region, then one down its left side, and so on.  Each level
    of the XY-cut (gaps 1) peels one bar off, so n_bars > 24 leaves the last region open at level 24.  Less than half of the page
    is ink, so its polarity is dark."""
    side = (n_bars // 2 + 1) * (t + gap) + 8
    m = np.zeros((side, side), bool)
    x0, y0 = 0, 0
    for k in range(n_bars):
        if k % 2 == 0:
            m[y0:y0 + t, x0:] = True
            y0 += t + gap
        else:
            m[y0:, x0:x0 + t] = True
            x0 += t + gap
    return _rgb(m)


def plus_grid(n):
    """n plus signs of 5 x 5 pixels on a full grid (32 x 32 for 1024, 41 x 25 for 1025), 6 columns and 3 rows apart: S = 5, and
    every plus is a block of the twin."""
    per_row = 32 if n == 1024 else 41
    rows = n // per_row
    assert rows * per_row == n
    m = np.zeros((rows * 8 + 3, per_row * 11 + 6), bool)
    for k in range(n):
        y, x = 3 + 8 * (k // per_row), 6 + 11 * (k % per_row)
        m[y + 2, x:x + 5] = True
        m[y:y + 5, x + 2] = True
    return _rgb(m)


def chevron_block(theta=6.0, w=360, n_lines=5, pitch=40):
    """Lines rising at theta degrees towards the middle from both sides, the crop mirror-symmetric about its vertical axis:
    every +-i pair of the angle search ties exactly."""
    h = n_lines * pitch + 80
    m = np.zeros((h, w), bool)
    half = w // 2
    rise = np.floor((half - np.arange(half)) * np.tan(np.radians(theta))).astype(int)
    for k in range(n_lines):
        y = 60 + k * pitch + rise
        for d in range(2):
            ok = (y + d >= 0) & (y + d < h)
            m[(y + d)[ok], np.arange(half)[ok]] = True
    m[:, half:] = m[:, :half][:, ::-1]
    return _rgb(m)


def component_images(rng=None):
    """Paper components (bright, the paper polarity) built to stress the union-find: name -> image."""
    rng = rng or np.random.default_rng(7)
    out = {}
    h, w = 200, 203                                    # a serpentine through every 32 x 32 tile
    m = np.zeros((h, w), bool)
    for k, y in enumerate(range(0, h, 4)):
        m[y, :] = True
        if y + 4 < h:
            m[y:y + 4, w - 1 if k % 2 == 0 else 0] = True
    out["serpentine"] = m
    n = 161                                            # a square spiral
    m = np.zeros((n, n), bool)
    x0, y0, x1, y1 = 0, 0, n - 1, n - 1
    while x0 <= x1 and y0 <= y1:
        m[y0, x0:x1 + 1] = True
        m[y0:y1 + 1, x1] = True
        if y1 - y0 >= 2:
            m[y1, x0 + 2:x1 + 1] = True
        if x1 - x0 >= 4:
            m[y0 + 2:y1 + 1, x0 + 2] = True
        x0, y0, x1, y1 = x0 + 2, y0 + 2, x1 - 2, y1 - 2
        if x1 - x0 < 2:
            break
    out["spiral"] = m
    m = np.zeros((130, 190), bool)                     # a comb whose teeth cross every tile border
    m[0:3, :] = True
    m[:, 1::6] = True
    out["comb"] = m
    m = np.zeros((96, 97), bool)                       # diagonal-only contacts: apart under 4-connectivity
    m[(np.add.outer(np.arange(96), np.arange(97)) % 2) == 0] = True
    m[::5] = False
    out["diagonal"] = m
    m = rng.random((70, 66)) < 0.55                    # components touching all four borders, and random clusters
    m[0, :] = m[-1, :] = m[:, 0] = m[:, -1] = True
    out["borders"] = m
    for wd in (1, 31, 32, 33, 45):                      # image widths of 1, 31, 32, 33 and a non-multiple of 32
        out[f"width{wd}"] = rng.random((77, wd)) < 0.6
    return {k: _rgb(v, fg=PAPER, bg=INK) for k, v in out.items()}


def tie_hull_images():
    """Paper shapes whose hulls have many edges parallel to their diagonals, so that the largest quad ties."""
    yy, xx = np.mgrid[0:160, 0:160] - 80
    shapes = dict(disc=xx ** 2 + yy ** 2 <= 71 ** 2, diamond=np.abs(xx) + np.abs(yy) <= 57,
                  octagon=(np.abs(xx) + np.abs(yy) <= 57) & (np.abs(xx) <= 38) & (np.abs(yy) <= 38),
                  small_disc=xx ** 2 + yy ** 2 <= 23 ** 2)
    yy, xx = np.mgrid[0:520, 0:520] - 260
    shapes["big_disc"] = xx ** 2 + yy ** 2 <= 255 ** 2
    return {k: _rgb(v, fg=PAPER, bg=INK) for k, v in shapes.items()}


def curve_runs_block(n_runs):
    """One strip (strips=1) of n_runs runs: accepted at 256, MN_CURVE_ERR_RUNS at 257."""
    return lines_block(n_runs, w=64)


def curve_lines_block(n_lines):
    """Two strips of 32 pixels: n_lines - 1 lines in strip 0, then one more in strip 1 below them; n_lines kept lines."""
    t, gap = 3, 3
    m = np.zeros((n_lines * (t + gap) + gap, 64), bool)
    for k in range(n_lines):
        y = gap + k * (t + gap)
        if k < n_lines - 1:
            m[y:y + t, 2:30] = True
        else:
            m[y:y + t, 34:62] = True
    return _rgb(m)


def link_bound_block():
    """Five strips of 32 pixels, 4096 rows: strips 0, 1 and 2 each hold 256 runs on rows no other of them inks, so 768 lines are
    open at strip 3; strip 3 holds 256 runs on strip 0's rows, so the link weighs 768 open lines and 256 new runs; strip 4 is
    blank.  Each of strip 0's lines continues in strip 3 and keeps (two runs, need 2): 256 kept lines."""
    m = np.zeros((4096, 160), bool)
    for k in range(256):
        for s in range(4):
            y = 4 * (4 * k + (0 if s == 3 else s))
            m[y:y + 2, 32 * s + 1:32 * s + 31] = True
    return _rgb(m)


def bit31_block(n_lines=6):
    """32 strips of 32 pixels and level lines across them all: each line's sample mask sets bit 31, the int32 sign bit."""
    return lines_block(n_lines, w=1024, t=6, gap=10)


def uneven_strips_block(rng, n_s=5):
    """w = 32 n_s + 31: strips of 38 and 39 pixels, so 32-pixel tiles straddle strip borders; wavy lines of random ink."""
    w, h = 32 * n_s + 31, 220
    m = np.zeros((h, w), bool)
    x = np.arange(w)
    for k in range(6):
        y = (20 + 32 * k + 4 * np.sin(x / 23.0 + k)).astype(int)
        for d in range(4):
            m[y + d, x] = rng.random(w) < 0.8
    return _rgb(m)


# ---- references --------------------------------------------------------------------------------------------------------
def min_index_labels(mask, structure=None):
    """Each pixel's component label as the smallest raster index y w + x of its component (scipy.ndimage.label, 4-connected
    unless ``structure``), -1 off the mask; and the component sizes at those indices (0 elsewhere), flat."""
    lab, n = ndimage.label(mask, structure=structure)
    first = np.full(n + 1, mask.size, np.int64)
    np.minimum.at(first, lab.ravel(), np.arange(mask.size))
    size = np.bincount(lab.ravel(), minlength=n + 1)
    out = np.where(lab > 0, first[lab], -1)
    count = np.zeros(mask.size, np.int64)
    count[first[1:]] = size[1:]
    return out, count


def largest_quad_last(hull):
    """The brute force keeping the last maximal tuple instead of the first (a negative control)."""
    v = np.array(hull, np.int64)
    k, best = len(v), (-1, None)

    def t2(i, m, j):
        return abs(int(Q._cross(v[i], v[m], v[j])))
    for i in range(k - 3):
        for j in range(i + 2, k - 1):
            la = max(range(i + 1, j), key=lambda a: (t2(i, a, j), a))
            lb = max(range(j + 1, k), key=lambda b: (t2(j, b, i), b))
            s = t2(i, la, j) + t2(j, lb, i)
            if s >= best[0]:
                best = (s, (i, la, j, lb))
    return best


def two_pointer_quad(hull):
    """The device's search restated: per first index i, apexes a and c that only move forward as j grows, each stopping at the
    first of two equal apexes; the first (i, j) of the largest area."""
    v = [tuple(p) for p in hull]
    k, best = len(v), (-1, None)

    def t2(i, m, j):
        return abs(Q._cross(v[i], v[m], v[j]))
    for i in range(k - 3):
        a, c = i + 1, i + 3
        for j in range(i + 2, k - 1):
            while a + 1 < j and t2(i, a + 1, j) > t2(i, a, j):
                a += 1
            c = max(c, j + 1)
            while c + 1 < k and t2(j, c + 1, i) > t2(j, c, i):
                c += 1
            s = t2(i, a, j) + t2(j, c, i)
            if s > best[0]:
                best = (s, (i, a, j, c))
    return best


def choose_greater(idx, scores):
    """The skew choice with ties to the greater index (a negative control)."""
    return max(range(len(idx)), key=lambda p: (scores[p], -abs(idx[p]), idx[p]))


def _runs(text):
    d = np.diff(np.concatenate([[0], text.astype(np.int8), [0]]))
    return np.nonzero(d == 1)[0], np.nonzero(d == -1)[0]


# ---- the twins at the edges ----------------------------------------------------------------------------------------------
def test_otsu_hist_is_otsu():
    rng = np.random.default_rng(0)
    for g in (rng.integers(0, 256, (50, 70)), np.full((3, 3), 7), rng.integers(100, 103, (9, 11)), B.grey(lines_block(5))):
        assert B.otsu_hist(np.bincount(g.reshape(-1), minlength=256)) == B.otsu(g)
    big = np.zeros(256, np.int64)                       # a 32767 x 32767 block: about 2^30 pixels in one bin
    big[[INK, PAPER]] = 32767 * 40 * 256, 32767 * 32767 - 32767 * 40 * 256
    assert B.otsu_hist(big) == INK


def big_page_lines(H, W):
    """The ink rows of the large device-built page of the GPU file: lines 40 rows thick, 160 apart, over columns [100, W - 100),
    from row 100 to about 15/16 of the page."""
    return [(y, y + 40) for y in range(100, H - H // 16, 160)]


@pytest.mark.parametrize("direction", ["horizontal", "vertical"])
def test_banded_reference_is_find_lines(direction):
    rng = np.random.default_rng(4)
    imgs = [lines_block(9, w=70), _rgb(rng.random((90, 75)) < 0.2), 255 - lines_block(5, w=41), alternating_block(41),
            _rgb(np.zeros((7, 5), bool)), np.ascontiguousarray(lines_block(6, w=50).transpose(1, 0, 2))]
    for k, img in enumerate(imgs):
        h, w = img.shape[:2]
        for rect in ((0, 0, w, h), (3, 2, w - 1, h - 4)):
            x0, y0, x1, y1 = rect
            crop = img[y0:y1, x0:x1]
            want = B.find_lines(img, rect, direction)
            for rows in (1, 7, 512):
                got = SB.find_lines_banded(lambda a, b: crop[a:b], y1 - y0, x1 - x0, (x0, y0), direction, rows=rows)
                assert got == want, (k, rect, rows)
    H = W = 2000                                       # the large page's layout, scaled down: its lines exactly
    m = np.zeros((H, W), bool)
    for a, b in big_page_lines(H, W):
        m[a:b, 100:W - 100] = True
    img = _rgb(m)
    got = SB.find_lines_banded(lambda a, b: img[a:b], H, W, (0, 0), direction, rows=300)
    assert got == B.find_lines(img, (0, 0, W, H), direction)
    assert len(got["lines"]) == (12 if direction == "horizontal" else 1)


@pytest.mark.parametrize("n", [256, 257])
def test_lines_block_reaches_the_line_limit(n):
    img = lines_block(n)
    rect = (0, 0, img.shape[1], img.shape[0])
    if n == 256:
        assert len(B.find_lines(img, rect)["lines"]) == 256
        with pytest.MonkeyPatch.context() as mp:      # the limit written as >= 256 refuses it
            mp.setattr(B, "MAX_LINES", 255)
            with pytest.raises(ValueError, match="256 lines exceed"):
                B.find_lines(img, rect)
    else:
        with pytest.raises(ValueError, match="257 lines exceed"):
            B.find_lines(img, rect)


@pytest.mark.parametrize("L", [32767, 32766, 9, 10])
def test_alternating_block_fills_the_run_scratch(L):
    ink = _ink(alternating_block(L))
    a, e = _runs(ink.sum(axis=1) >= 1)
    assert len(a) == (L + 1) // 2 and ink[0].any() and ink[-1].any()
    assert len(B.find_lines(alternating_block(L), (0, 0, 16, L))["lines"]) == 1


def test_lattice_pages_reach_the_node_limit():
    ink = _ink(lattice_page(256, 256))
    assert ink.shape == (511, 511)
    assert len(P.xy_cut(ink, False, 1, 1)) == 65536 == min(P.MAX_NODES, 512 * 512 // 4)
    with pytest.raises(ValueError, match="more than 65536 nodes"):
        P.xy_cut(_ink(lattice_page(256, 257)), False, 1, 1)
    with pytest.MonkeyPatch.context() as mp:           # the limit written as >= refuses exactly 65536
        mp.setattr(P, "MAX_NODES", 65535)
        with pytest.raises(ValueError):
            P.xy_cut(ink, False, 1, 1)
    small = _ink(lattice_page(16, 16))                 # the host bound (h + 1) (w + 1) / 4, attained
    assert len(P.xy_cut(small, False, 1, 1)) == 32 * 32 // 4 == 256


def test_staircase_page_is_open_at_level_24():
    img = staircase_page(30)
    ink = _ink(img)
    leaves = P.xy_cut(ink, False, 1, 1)
    res = P.find_blocks(img, None, "horizontal", "auto", 1, 1)
    assert res["ink"] == "dark"
    with pytest.MonkeyPatch.context() as mp:
        for levels in (23, 25):                        # one level more would still cut: level 24 closed open nodes
            mp.setattr(P, "LEVELS", levels)
            assert P.xy_cut(ink, False, 1, 1) != leaves
            other = P.find_blocks(img, None, "horizontal", "auto", 1, 1)
            assert (other["blocks"], other["rejected"]) != (res["blocks"], res["rejected"])


@pytest.mark.parametrize("n", [1024, 1025])
def test_plus_grid_reaches_the_block_limit(n):
    img = plus_grid(n)
    if n == 1024:
        res = P.find_blocks(img)
        assert len(res["blocks"]) == 1024 and res["text_size"] == 5 and not res["rejected"]
    else:
        with pytest.raises(ValueError, match="1025 blocks exceed"):
            P.find_blocks(img)


def test_chevron_ties_every_plus_minus_pair():
    img = chevron_block()
    ink = _ink(img)
    assert np.array_equal(ink, ink[:, ::-1])
    tab = SB.angles("auto", 20.0)
    assert len(tab) == 801
    idx = [i for i, _ in tab]
    c = np.array([np.cos(np.radians(t)) for _, t in tab])
    s = np.array([np.sin(np.radians(t)) for _, t in tab])
    scores = [SB.score(r) for r in SB.profiles(ink, c, s)]
    assert all(scores[400 - d] == scores[400 + d] for d in range(401))
    p = SB.choose(idx, scores)
    assert idx[p] < 0 and scores[p] == max(scores) > scores[400]
    assert idx[choose_greater(idx, scores)] == -idx[p]
    ref = SB.find_lines(img, (0, 0, img.shape[1], img.shape[0]), max_skew=20.0)
    assert ref["detail"]["chosen"] == p


def test_component_labels_and_controls():
    imgs = component_images()
    for name, img in imgs.items():
        mask, _ = Q.paper(img)
        lab, count = min_index_labels(mask)
        label, size, _ = Q.page_component(mask)
        assert label == int(lab.ravel()[np.argmax(np.where(count > 0, count * mask.size - np.arange(mask.size), -1))])
        assert size == count.max()
        if name in ("serpentine", "spiral"):
            assert (lab[mask] == lab[mask][0]).all(), name        # one component through every tile
        if name == "diagonal":
            eight, _ = min_index_labels(mask, np.ones((3, 3), int))
            assert not np.array_equal(lab, eight)
    m, _ = Q.paper(imgs["comb"])
    assert m[:, 1::6].all() and m.shape[0] > 96


def test_tie_hulls_need_the_tie_rule():
    differs = 0
    for name, img in tie_hull_images().items():
        mask, _ = Q.paper(img)
        _, _, members = Q.page_component(mask)
        hull = Q.monotone_chain(Q.row_points(members))
        best = Q.largest_quad(hull)
        assert two_pointer_quad(hull) == best, name
        last = largest_quad_last(hull)
        assert last[0] == best[0]
        differs += last[1] != best[1]
    assert differs == len(tie_hull_images())


@pytest.mark.parametrize("n", [256, 257])
def test_curve_strip_run_limit(n):
    img = curve_runs_block(n)
    ref = C.find_lines(img, (0, 0, 64, img.shape[0]), strips=1)
    if n == 256:
        assert len(ref["detail"]["runs"][0]) == 256 and ref["detail"]["header"][0] == C.OK
    else:
        assert list(ref["detail"]["header"][[0, 3, 4]]) == [C.ERR_RUNS, 0, 257]


@pytest.mark.parametrize("n", [256, 257])
def test_curve_kept_line_limit(n):
    img = curve_lines_block(n)
    ref = C.find_lines(img, (0, 0, 64, img.shape[0]), strips=2)
    assert [len(r) for r in ref["detail"]["runs"]] == [n - 1, 1]
    if n == 256:
        assert ref["detail"]["header"][0] == C.OK and ref["detail"]["header"][1] == 256
    else:
        assert list(ref["detail"]["header"][[0, 4]]) == [C.ERR_LINES, 257]


def test_link_bound_block_fills_the_link():
    img = link_bound_block()
    ref = C.find_lines(img, (0, 0, 160, 4096), strips=5)
    runs = ref["detail"]["runs"]
    assert [len(r) for r in runs] == [256, 256, 256, 256, 0]
    rows = [{a for a, *_ in r} for r in runs[:4]]
    assert not (rows[0] & rows[1]) and not (rows[0] & rows[2]) and not (rows[1] & rows[2]) and rows[3] == rows[0]
    header, table = ref["detail"]["header"], ref["detail"]["table"]
    assert header[0] == C.OK and header[1] == 256 and (table[:, 2] == 2).all() and (table[:, 1] == 3).all()


def test_bit31_block_sets_the_sign_bit():
    img = bit31_block()
    ref = C.find_lines(img, (0, 0, 1024, img.shape[0]), strips=32)
    table = ref["detail"]["table"]
    assert len(table) == 6 and (table[:, 5] == -1).all()


def test_uneven_strips_straddle_tiles():
    img = uneven_strips_block(np.random.default_rng(3))
    xb = C.bounds(img.shape[1], 5)
    assert set(np.diff(xb)) == {38, 39} and any(b % 32 for b in xb[1:-1])
    ref = C.find_lines(img, (0, 0, img.shape[1], img.shape[0]), strips=5)
    assert ref["detail"]["header"][0] == C.OK and ref["detail"]["header"][1] >= 5
