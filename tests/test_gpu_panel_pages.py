"""Reversed panels on the device (DESIGN.md section 7b, "Reversed panels"): one find_blocks call of every drawn page, seeded
random panel pages and edge pages (a 32767-pixel-wide page whose panel ends in its last bitmap word, lattices of 1024 and 1025
panels) against the numpy twin bit for bit, with its launch count; no cross-talk with pages without panels; a panel page beside
a skewed page; and restore_regions with the banner page against the same call given the found blocks."""
import numpy as np
import pytest
import torch

from oracle import pages as P
from oracle import panel_pages as PP
from oracle import quad_pages as Q
from oracle import ruled_pages as RP

from test_gpu_pages import _same
from test_figure_pages import column_page
from test_panel_pages import (FILL, PAPER, _inside, _put, banner_page, blurred_photo, bold_glyph_page, button_page,
                              gradient_page, photographed_banner, shaded_table, sidebar_page, threshold_pages,
                              vertical_sidebar_page)

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda:0")


def _wide():
    """A 32767-pixel-wide page: words along it and a dark panel with a white word that ends in the page's last column (its last
    bitmap word)."""
    img = np.full((60, 32767, 3), PAPER, np.uint8)
    for x in range(20, 31000, 400):
        _put(img, "words %d" % x, (x, 40), 0.6)
    img[8:52, 32767 - 1500:] = FILL                    # wide enough that its text rows stay ink at the root's width
    _put(img, "LAST PANEL", (32767 - 1400, 40), 0.8, 250, 2)
    return img


def _lattice(n):
    """n dark 6 x 6 squares on a 10-pixel lattice, 32 to a row: with panel_size 2 each is a panel."""
    rows = -(-n // 32)
    img = np.full((10 * rows + 10, 330, 3), PAPER, np.uint8)
    for k in range(n):
        r, c = divmod(k, 32)
        img[10 + 10 * r:16 + 10 * r, 10 + 10 * c:16 + 10 * c] = FILL
    return img


def random_panel_page(rng):
    """A seeded page: dark lines of text, 1 to 3 flat dark panels of random fill holding white lines, sometimes a blurred dark
    photo, a random crop, direction (the transposed page read vertically), polarity (the negative), rules, figures and block
    direction.  (image, the twin's keyword arguments)."""
    h, w = int(rng.integers(300, 700)), int(rng.integers(400, 900))
    img = np.full((h, w, 3), int(rng.integers(225, 250)), np.uint8)
    for k in range(int(rng.integers(3, 10))):
        _put(img, "line %d of text" % k + " word" * int(rng.integers(0, 4)), (int(rng.integers(5, w // 3)), 30 + 30 * k),
              float(rng.uniform(0.5, 0.9)), int(rng.integers(0, 60)))
    for _ in range(int(rng.integers(1, 4))):
        pw, ph = int(rng.integers(60, w // 2)), int(rng.integers(30, h // 3))
        x, y = int(rng.integers(0, w - pw)), int(rng.integers(0, h - ph))
        img[y:y + ph, x:x + pw] = int(rng.integers(5, 90))
        for k in range(max(1, (ph - 10) // 28)):
            _put(img, "PANEL %d" % k, (x + 6, y + 24 + 28 * k), float(rng.uniform(0.5, 0.8)), int(rng.integers(200, 256)),
                  int(rng.integers(1, 3)))
    if rng.random() < 0.4:
        ph, pw = int(rng.integers(40, h // 2)), int(rng.integers(40, w // 2))
        y, x = int(rng.integers(0, h - ph)), int(rng.integers(0, w - pw))
        img[y:y + ph, x:x + pw] = blurred_photo(rng, ph, pw)
    kw = {}
    if rng.random() < 0.3:
        img = np.ascontiguousarray(img.transpose(1, 0, 2)[:, ::-1])
        kw["direction"] = "vertical"
    if rng.random() < 0.3:
        img = 255 - img
    H, W = img.shape[:2]
    if rng.random() < 0.3:
        x0, y0 = int(rng.integers(0, W // 4)), int(rng.integers(0, H // 4))
        kw["rect"] = (x0, y0, int(rng.integers(x0 + W // 2, W + 1)), int(rng.integers(y0 + H // 2, H + 1)))
    for key in ("rules", "figures", "block_direction"):
        if rng.random() < 0.3:
            kw[key] = True
    if rng.random() < 0.3:
        kw["panel_size"] = int(rng.integers(2, 40))
    return img, kw


def _pages(rng):
    """[(image, TextPage, the twin's keyword arguments, whether the page has panels)]."""
    from marconet_b200 import pipeline
    banner, _ = banner_page()
    table = shaded_table()[0]
    side = sidebar_page(photo=True)[0]
    V = dict(direction="vertical")
    plain_side = sidebar_page()[0]
    out = [(banner, {}), (table, dict(rules=True, rule_length=200)), (plain_side, {}), (plain_side, dict(figures=True)),
           (side, dict(figures=True)), (side, {}), (button_page()[0], {}), (bold_glyph_page("I"), {}), (bold_glyph_page("O"), {}),
           (gradient_page(), {}), (vertical_sidebar_page()[0], dict(block_direction=True)),
           (np.ascontiguousarray(banner.transpose(1, 0, 2)[:, ::-1]), V), (255 - banner, {}),
           (banner, dict(rect=(20, 40, 790, 480))), (photographed_banner(), dict(quad="auto")),
           (banner[150:], {}), (banner[150:], dict(rules=True, figures=True, block_direction=True))]
    T = lambda im: np.ascontiguousarray(im.transpose(1, 0, 2)[:, ::-1])   # read vertically: the transposed page
    out += [(T(plain_side), V), (T(table), dict(V, rules=True, rule_length=200)), (column_page("photo")[0], {}),
            (column_page("photo")[0], dict(figures=True))]
    out += [(img, dict(panel_size=p)) for img, p, _ in threshold_pages()]
    out += [random_panel_page(rng) for _ in range(20)]
    out += [(_wide(), dict(panel_size=20)), (_lattice(1024), dict(panel_size=2)), (_lattice(1025), dict(panel_size=2))]
    TP = pipeline.TextPage

    def page(kw, panels=True):
        return TP(rules="auto" if kw.get("rules") else None, rule_length=kw.get("rule_length"),
                  figures="auto" if kw.get("figures") else None,
                  block_direction="auto" if kw.get("block_direction") else None, panels="auto" if panels else None,
                  panel_size=kw.get("panel_size") if panels else None, quad=kw.get("quad"), rect=kw.get("rect"),
                  direction=kw.get("direction", "horizontal"))
    pages = [(img, page(kw), kw, True) for img, kw in out]
    plain = [(banner, {}), (table, dict(rules=True, rule_length=200)), (side, dict(figures=True))]
    pages += [(img, page(kw, False), kw, False) for img, kw in plain]
    return pages


def _twin(img, kw, panels):
    try:
        if "quad" in kw:                                 # a photographed page: its blocks are windows of R
            return PP.find_quad_blocks(img, Q.accepted(Q.find_corners(img), img.shape))
        if panels:
            return PP.find_blocks(img, **kw)
        if kw.get("figures"):
            from oracle import figure_pages as FP
            return FP.find_blocks(img, **{k: v for k, v in kw.items() if k != "figures"})
        if kw.get("rules"):
            return RP.find_blocks(img, **{k: v for k, v in kw.items() if k != "rules"})
        return P.find_blocks(img, **kw)
    except ValueError as e:
        return dict(error=str(e))


def _as_twin(got, panels):
    """A find_blocks dict in the twin's terms: blocks as rectangles (windows of R on a quad page), with panels their
    polarities, and with block_direction their directions."""
    out = dict(got, blocks=[b.window if b.quad is not None else tuple(b.rect) for b in got["blocks"]])
    if panels:
        out["polarities"] = [b.polarity for b in got["blocks"]]
    if "block_direction" in got:
        out["directions"] = [b.direction for b in got["blocks"]]
    return out


def _call(pipeline, dimgs, pages):
    """pipeline.find_blocks' device path (corner search, rectification and layout) over uploaded images."""
    rects = [(0, 0, im.shape[1], im.shape[0]) if pg.rect is None else pg.rect for im, pg in zip(dimgs, pages)]
    return pipeline._find_pages(dict(enumerate(dimgs)), [(k, pg, r) for k, (pg, r) in enumerate(zip(pages, rects))])[0]


def test_panel_pages_equal_twin(monkeypatch):
    """Every dict, block and polarity of one call equals the twin's; its layout takes 3 rule launches, 1 figure launch, 1
    direction launch and 2 panel launches more than a plain one, and its pages without panels get the tables of a call without
    the panel pages."""
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
    assert layout == [5 + 6 * _lib.PAGE_LEVELS + 3 + 1 + 1 + 2]
    n_panels = n_light = 0
    errors = []
    for k, ((img, pg, kw, panels), g) in enumerate(zip(items, got)):
        ref = _twin(img, kw, panels)
        if "error" in ref:
            assert isinstance(g, str) and ref["error"].split()[0] == g.split()[0], (k, g, ref)
            errors.append(g)
            continue
        assert not isinstance(g, str), (k, g)
        assert _as_twin(g, panels) == ref, (k, _as_twin(g, panels), ref)
        if panels:
            n_panels += len(ref["panels"])
            n_light += sum(p != "auto" for p in ref["polarities"])
    assert errors == ["1025 panels exceed the 1024 a text page may hold"]
    assert n_panels >= 1024 + 30 and n_light >= 60, (n_panels, n_light)
    wide = got[[k for k, it in enumerate(items) if it[0].shape[1] == 32767][0]]
    assert wide["panels"][-1][2] == 32767 and any(b.polarity == "light" for b in wide["blocks"])
    plain = [k for k, item in enumerate(items) if not item[3]]
    alone = _call(pipeline, [dimgs[k] for k in plain], [items[k][1] for k in plain])
    assert [got[k] for k in plain] == alone


def test_threshold_pages_give_their_pinned_panels():
    """The exact thresholds of the panel test on the device: a flat count of half is no panel and one pixel more is, a tied mode
    goes to the smaller grey, and a shorter side of p is a panel and p - 1 is not."""
    from marconet_b200 import pipeline
    pages = threshold_pages()
    got = _call(pipeline, [torch.from_numpy(img).to(DEV) for img, _, _ in pages],
                [pipeline.TextPage(panels="auto", panel_size=p) for _, p, _ in pages])
    assert [g["panels"] for g in got] == [panels for _, _, panels in pages]


def test_launch_counts():
    """A call with panel pages takes exactly 2 launches more than the same call without them, and its other pages get their
    tables."""
    from marconet_b200 import _lib, ops, pipeline
    img, _ = banner_page()
    table = shaded_table()[0]
    d = [torch.from_numpy(img).to(DEV), torch.from_numpy(table).to(DEV)]
    for extra, more in (({}, 0), (dict(rules="auto", rule_length=200), 3)):
        n0 = ops.LAUNCHES
        with_panels = _call(pipeline, d, [pipeline.TextPage(panels="auto"), pipeline.TextPage(**extra)])
        assert ops.LAUNCHES - n0 == 5 + 6 * _lib.PAGE_LEVELS + more + 2
        n0 = ops.LAUNCHES
        without = _call(pipeline, d, [pipeline.TextPage(), pipeline.TextPage(**extra)])
        assert ops.LAUNCHES - n0 == 5 + 6 * _lib.PAGE_LEVELS + more
        assert with_panels[1] == without[1]
    assert with_panels[0]["panels"] == [(30, 60, 771, 151)] and without[0]["rejected"] == [(30, 60, 771, 151)]


def test_skewed_call_gives_a_panel_page_its_tables():
    from marconet_b200 import _lib, ops, pipeline
    img = sidebar_page(photo=True)[0]
    dimgs = [torch.from_numpy(img).to(DEV), torch.from_numpy(banner_page()[0]).to(DEV)]
    pg = pipeline.TextPage(panels="auto", figures="auto")
    alone = _call(pipeline, dimgs[:1], [pg])
    n0 = ops.LAUNCHES
    mixed = _call(pipeline, dimgs, [pg, pipeline.TextPage(skew="auto")])
    assert ops.LAUNCHES - n0 == 7 + 6 * _lib.PAGE_LEVELS + 1 + 2
    assert mixed[0] == alone[0]
    assert _as_twin(alone[0], True) == PP.find_blocks(img, figures=True)


def test_restore_regions_banner_page_equals_the_found_blocks(gpu_models, monkeypatch):
    """The banner and the first dark line.  Module graphs are off, so that the call's new line batches leave no recorded
    graphs, and their memory, to the tests after it."""
    from marconet_b200 import ops, pipeline
    monkeypatch.setattr(ops, "MODULE_GRAPHS", False)
    m = gpu_models["encoder"], gpu_models["tspgan"], gpu_models["sr"]
    img, banner = banner_page()
    img = np.ascontiguousarray(img[:232])
    pg = pipeline.TextPage(panels="auto")
    found = pipeline.find_blocks([img], [[pg]])[0][0]
    assert found["panels"] == [banner]
    kw = dict(scale=2, feather=3, to_host=True)
    a = pipeline.restore_regions(*m, [img], [[pg]], **kw)[0]
    b = pipeline.restore_regions(*m, [img], [found["blocks"]], **kw)[0]
    np.testing.assert_array_equal(a["image"], b["image"])
    assert {k: v for k, v in a["regions"][0].items() if k != "regions"} == found
    _same(a["regions"][0]["regions"], b["regions"])
    light = [e for blk, e in zip(found["blocks"], a["regions"][0]["regions"]) if blk.polarity == "light"]
    assert len(light) == 6 and all(len(e["lines"]) == 1 for e in light)
    assert all(_inside(q, banner) for e in light for q in e["lines"])
