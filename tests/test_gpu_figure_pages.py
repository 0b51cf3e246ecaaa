"""Figures on the device (DESIGN.md section 7b, "Figures"): one find_blocks call of every drawn page, seeded random pages with
photos, charts and text pieces, and pages without figures against the numpy twins bit for bit, with its launch count; no
cross-talk with pages without figures; a figure page beside a skewed page; the 1024-figure limit and a 32767-pixel page; and
restore_regions with a figure page against the same call given the found blocks."""
import numpy as np
import pytest
import torch

from oracle import figure_pages as FP
from oracle import pages as P
from oracle import quad_pages as Q

from test_figure_pages import (_meets, blotch_photo, chart, column_page, framed_photo_page, headline_page, lone_photo,
                               photographed_photo_page, smooth_photo, table_beside_photo, threshold_page, wide_photo_page,
                               wrapped_page)
from test_gpu_pages import _same

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda:0")


def _random_figures(rng):
    """A random page of text pieces with photos (smooth or blotched) and outlined charts: (image, twin keyword arguments)."""
    h, w = int(rng.integers(120, 500)), int(rng.integers(160, 900))
    img = np.full((h, w, 3), 235, np.uint8)
    ink = rng.random((h, w)) < 0.004
    for _ in range(int(rng.integers(4, 40))):            # glyph-sized pieces
        y, x = int(rng.integers(0, h - 12)), int(rng.integers(0, w - 20))
        ink[y:y + int(rng.integers(6, 14)), x:x + int(rng.integers(3, 20)):2] = True
    img[ink] = 20
    for _ in range(int(rng.integers(1, 4))):
        ph, pw = int(rng.integers(10, h // 2)), int(rng.integers(10, w // 2))
        y, x = int(rng.integers(0, h - ph)), int(rng.integers(0, w - pw))
        kind = int(rng.integers(0, 3))
        img[y:y + ph, x:x + pw] = (smooth_photo(rng, ph, pw) if kind == 0 else blotch_photo(rng, ph, pw) if kind == 1
                                   else chart(rng, ph, pw) if ph > 120 and pw > 60 else 20)
    kw = dict(figure_size=int(rng.integers(2, 80))) if rng.random() < 0.4 else {}
    if rng.random() < 0.3:
        kw["rect"] = (int(rng.integers(0, w // 4)), int(rng.integers(0, h // 4)), w - int(rng.integers(0, w // 4)), h)
    if rng.random() < 0.2:
        kw["direction"] = "vertical"
    return img, kw


def _lattice(n):
    """n 2 x 2 squares on a 3-pixel lattice, 32 to a row."""
    rows = -(-n // 32)
    m = np.zeros((3 * rows + 3, 3 * 32 + 3), bool)
    for k in range(n):
        r, c = divmod(k, 32)
        m[2 + 3 * r:4 + 3 * r, 2 + 3 * c:4 + 3 * c] = True
    return np.where(m[..., None], 20, 235).astype(np.uint8).repeat(3, axis=2)


def _wide():
    """A 32767-pixel-wide page: words of three strokes, and a dark figure 300 x 50 ending in the page's last column (its last
    bitmap word); a picture's row must hold 32767 / 128 ink pixels not to be white at the page's first cut."""
    m = np.zeros((60, 32767), bool)
    for x in range(10, 32400, 40):
        m[20:32, x:x + 9:3] = True
    m[5:55, 32767 - 300:] = True
    return np.where(m[..., None], 20, 235).astype(np.uint8).repeat(3, axis=2)


def _pages(rng):
    """[(image, TextPage, the twin's keyword arguments, whether the page has figures)]."""
    from marconet_b200 import pipeline
    TP = pipeline.TextPage
    photo, _ = column_page("photo")
    out = [(photo, {}), (column_page("chart")[0], {}), (column_page("dark")[0], {}), (framed_photo_page()[0], {}),
           (wide_photo_page()[0], {}), (wrapped_page()[0], {}), (headline_page(), {}),
           (np.ascontiguousarray(photo.transpose(1, 0, 2)[:, ::-1]), dict(direction="vertical")), (255 - photo, {}),
           (table_beside_photo()[0], dict(rules=True, rule_length=150)), (_wide(), dict(figure_size=40)),
           (photo, dict(rect=(30, 480, 900, 1150))), (lone_photo(), dict(figure_size=100)),
           (threshold_page(), dict(figure_size=30)), (threshold_page(), dict(figure_size=31)),
           (photographed_photo_page(), dict(quad="auto"))]
    out += [_random_figures(rng) for _ in range(20)]
    pages = [(img, TP(figures="auto", rules="auto" if kw.get("rules") else None, rule_length=kw.get("rule_length"),
                      **{k: v for k, v in kw.items() if k not in ("rules", "rule_length")}), kw, True) for img, kw in out]
    plain = [(photo, {}), (wrapped_page()[0], dict(gap_x=7))] + [out[k] for k in range(16, len(out), 5) if "figure_size" not in out[k][1]]
    pages += [(img, TP(**kw), kw, False) for img, kw in plain]
    return pages


def _twin(img, kw, figures):
    try:
        if "quad" in kw:                                 # a photographed page: its blocks are windows of R
            return FP.find_quad_blocks(img, Q.accepted(Q.find_corners(img), img.shape))
        return FP.find_blocks(img, **kw) if figures else P.find_blocks(img, **kw)
    except ValueError as e:
        return dict(error=str(e))


def _rects(got):
    return dict(got, blocks=[b.window if b.quad is not None else tuple(b.rect) for b in got["blocks"]])


def _call(pipeline, dimgs, pages):
    """pipeline.find_blocks' device path (corner search, rectification and layout) over uploaded images."""
    rects = [(0, 0, im.shape[1], im.shape[0]) if pg.rect is None else pg.rect for im, pg in zip(dimgs, pages)]
    return pipeline._find_pages(dict(enumerate(dimgs)), [(k, pg, r) for k, (pg, r) in enumerate(zip(pages, rects))])[0]


def test_figure_pages_equal_twin(monkeypatch):
    """Every dict, block, rejected leaf and figure of one call equals the twin's (a photographed page's as windows and
    rectangles of R); its layout takes 3 rule launches and 1 figure launch more than a plain one, and its pages without figures
    get the tables of a call without the figure pages."""
    from marconet_b200 import _lib, ops, pipeline
    rng = np.random.default_rng(0)
    items = _pages(rng)
    dimgs = [torch.from_numpy(im).to(DEV) for im, *_ in items]
    layout, find_blocks = [], ops.find_blocks

    def counted(*a, **k):                                # the layout's launches, apart from the corner search and warp
        n0 = ops.LAUNCHES
        res = find_blocks(*a, **k)
        layout.append(ops.LAUNCHES - n0)
        return res
    monkeypatch.setattr(ops, "find_blocks", counted)
    got = _call(pipeline, dimgs, [pg for _, pg, *_ in items])
    assert layout == [5 + 6 * _lib.PAGE_LEVELS + 3 + 1]
    assert [len(g["figures"]) for g in got if isinstance(g, dict) and "quad" in g] == [1]
    n_figures = 0
    for k, ((img, pg, kw, figures), g) in enumerate(zip(items, got)):
        ref = _twin(img, kw, figures)
        if "error" in ref:
            assert isinstance(g, str) and ref["error"].split()[0] == g.split()[0], (k, g, ref)
            continue
        assert not isinstance(g, str), (k, g)
        assert _rects(g) == ref, (k, _rects(g), ref)
        n_figures += len(ref.get("figures", []))
    assert n_figures >= 30
    plain = [k for k, item in enumerate(items) if not item[3]]
    alone = _call(pipeline, [dimgs[k] for k in plain], [items[k][1] for k in plain])
    assert [got[k] for k in plain] == alone


def test_launch_counts():
    """A call with figure pages and no rules or skew takes 5 + 6 * 24 + 1 launches; one without figure pages takes exactly the
    launches it took before, 5 + 6 * 24."""
    from marconet_b200 import _lib, ops, pipeline
    img, _ = column_page("photo")
    d = [torch.from_numpy(img).to(DEV)] * 2
    n0 = ops.LAUNCHES
    with_figures = _call(pipeline, d, [pipeline.TextPage(figures="auto"), pipeline.TextPage()])
    assert ops.LAUNCHES - n0 == 5 + 6 * _lib.PAGE_LEVELS + 1
    n0 = ops.LAUNCHES
    without = _call(pipeline, d, [pipeline.TextPage(), pipeline.TextPage()])
    assert ops.LAUNCHES - n0 == 5 + 6 * _lib.PAGE_LEVELS
    assert with_figures[1] == without[1] == without[0] and len(with_figures[0]["figures"]) == 1


def test_skewed_call_gives_a_figure_page_its_tables():
    from marconet_b200 import _lib, ops, pipeline
    photo, _ = column_page("photo")
    other, _ = wide_photo_page()
    dimgs = [torch.from_numpy(photo).to(DEV), torch.from_numpy(other).to(DEV)]
    alone = _call(pipeline, dimgs[:1], [pipeline.TextPage(figures="auto")])
    n0 = ops.LAUNCHES
    mixed = _call(pipeline, dimgs, [pipeline.TextPage(figures="auto"), pipeline.TextPage(skew="auto")])
    assert ops.LAUNCHES - n0 == 7 + 6 * _lib.PAGE_LEVELS + 1
    assert mixed[0] == alone[0] and len(alone[0]["figures"]) == 1
    assert _rects(alone[0]) == FP.find_blocks(photo)


def test_figure_limit():
    """With figure_size=2 a lattice of exactly 1024 figures is accepted and one of 1025 is refused, as the twin does."""
    from marconet_b200 import pipeline
    ok, over = _lattice(1024), _lattice(1025)
    got = pipeline.find_blocks([ok], [[pipeline.TextPage(figures="auto", figure_size=2)]])[0][0]
    assert len(got["figures"]) == 1024 and _rects(got) == FP.find_blocks(ok, figure_size=2)
    with pytest.raises(ValueError, match="image 0, page 0: 1025 figures exceed the 1024 a text page may hold"):
        pipeline.find_blocks([over], [[pipeline.TextPage(figures="auto", figure_size=2)]])
    with pytest.raises(ValueError, match="1025 figures exceed the 1024"):
        FP.find_blocks(over, figure_size=2)


def test_restore_regions_figure_page_equals_the_found_blocks(gpu_models):
    from marconet_b200 import pipeline
    m = gpu_models["encoder"], gpu_models["tspgan"], gpu_models["sr"]
    img, _ = column_page("photo")
    pg = pipeline.TextPage(figures="auto")
    found = pipeline.find_blocks([img], [[pg]])[0][0]
    assert len(found["blocks"]) == 4 and len(found["figures"]) == 1
    kw = dict(scale=2, feather=3, to_host=True)
    a = pipeline.restore_regions(*m, [img], [[pg]], **kw)[0]
    b = pipeline.restore_regions(*m, [img], [found["blocks"]], **kw)[0]
    np.testing.assert_array_equal(a["image"], b["image"])
    assert {k: v for k, v in a["regions"][0].items() if k != "regions"} == found
    _same(a["regions"][0]["regions"], b["regions"])
    lines = [tuple(r) for blk in a["regions"][0]["regions"] for r in blk["lines"]]
    assert len(lines) == 48 and not any(_meets(r, f) for r in lines for f in found["figures"])
