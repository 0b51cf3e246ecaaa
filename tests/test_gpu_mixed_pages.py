"""Mixed directions on the device (DESIGN.md section 7b, "Mixed directions"): one find_blocks call of every drawn page, seeded
random mixed pages and edge pages (a 32767-pixel-wide page, leaves of 4096 and 4097 indices, 1024 auto blocks) against the
numpy twins bit for bit, with its launch count; no cross-talk with pages without "auto"; a direction page beside a skewed
page; and restore_regions with a mixed page against the same call given the found blocks."""
import numpy as np
import pytest
import torch

from oracle import mixed_pages as MP
from oracle import pages as P
from oracle import quad_pages as Q
from oracle import ruled_pages as RP

from test_gpu_pages import _same
from test_mixed_pages import (SINGLE, TIES, _t, image, magazine_page, newspaper_page, photographed_newspaper, random_mixed,
                              ruled_table, text)

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda:0")


def _wide():
    """A 32767-pixel-wide page: one line of 1200 glyphs whose last one ends in the page's last column (its last bitmap word)."""
    rng = np.random.default_rng(11)
    m = np.zeros((60, 32767), bool)
    text(m, rng, 32767 - (1200 * 27 - 3), 18, 1, 1200, track=3)
    assert m[:, -1].any()
    return image(m)


def _chunk_edge(n):
    """A line whose leaf spans exactly n columns, a glyph's band running over column 4096 of it (a profile chunk's end)."""
    rng = np.random.default_rng(n)
    m = np.zeros((50, n + 80), bool)
    text(m, rng, 10, 12, 1, 153, track=3, kind="whole")
    m[:, 10 + n:] = False
    return image(m)


def _lattice():
    """1024 outlines of 6 x 12, 12 x 6 and 12 x 12 pixels on a 26-pixel lattice: 1024 blocks, vertical, horizontal and
    undecided in turn."""
    m = np.zeros((32 * 26 + 14, 32 * 26 + 14), bool)
    for k in range(1024):
        r, c = divmod(k, 32)
        x, y = 14 + 26 * c, 14 + 26 * r
        w, h = ((6, 12), (12, 6), (12, 12))[k % 3]
        m[y:y + h, [x, x + w - 1]] = True
        m[[y, y + h - 1], x:x + w] = True
    return image(m)


def _pages(rng):
    """[(image, TextPage, the twin's keyword arguments, whether the page has "auto")]."""
    from marconet_b200 import pipeline
    TP = pipeline.TextPage
    news, _ = newspaper_page()
    mag, _ = magazine_page()
    V = dict(direction="vertical")
    out = [(news, V), (mag, {}), (newspaper_page(photo=True)[0], dict(V, figures=True)), (ruled_table()[0], dict(rules=True)),
           (photographed_newspaper(), dict(V, quad="auto")), (_t(mag), V), (255 - news, V), (news, dict(V, rect=(30, 100, 990, 700))),
           (mag, dict(rect=(20, 20, 760, 470)))]
    out += [(draw(), d) for draw, *_ in SINGLE.values() for d in ({}, V)]
    out += [(make(), d) for make in TIES.values() for d in ({}, V)]
    out += [random_mixed(rng) for _ in range(20)]
    out += [(_wide(), {}), (_chunk_edge(4096), {}), (_chunk_edge(4097), {}), (_t(_chunk_edge(4096)), V),
            (_t(_chunk_edge(4097)), V), (_lattice(), {})]
    pages = []
    for img, kw in out:
        pg = TP(block_direction="auto", rules="auto" if kw.get("rules") else None, figures="auto" if kw.get("figures") else None,
                **{k: v for k, v in kw.items() if k not in ("rules", "figures")})
        pages.append((img, pg, kw, True))
    plain = [(news, V), (mag, {}), (ruled_table()[0], dict(rules=True))]
    pages += [(img, TP(rules="auto" if kw.get("rules") else None, **{k: v for k, v in kw.items() if k != "rules"}), kw, False)
              for img, kw in plain]
    return pages


def _twin(img, kw, auto):
    try:
        if "quad" in kw:                                 # a photographed page: its blocks are windows of R
            return MP.find_quad_blocks(img, Q.accepted(Q.find_corners(img), img.shape), direction=kw["direction"])
        if auto:
            return MP.find_blocks(img, **kw)
        if kw.get("rules"):
            return RP.find_blocks(img, **{k: v for k, v in kw.items() if k != "rules"})
        return P.find_blocks(img, **kw)
    except ValueError as e:
        return dict(error=str(e))


def _as_twin(got, auto):
    """A find_blocks dict in the twin's terms: blocks as rectangles (windows of R on a quad page), and with "auto" their
    directions."""
    out = dict(got, blocks=[b.window if b.quad is not None else tuple(b.rect) for b in got["blocks"]])
    if auto:
        out["directions"] = [b.direction for b in got["blocks"]]
    return out


def _call(pipeline, dimgs, pages):
    """pipeline.find_blocks' device path (corner search, rectification and layout) over uploaded images."""
    rects = [(0, 0, im.shape[1], im.shape[0]) if pg.rect is None else pg.rect for im, pg in zip(dimgs, pages)]
    return pipeline._find_pages(dict(enumerate(dimgs)), [(k, pg, r) for k, (pg, r) in enumerate(zip(pages, rects))])[0]


def test_mixed_pages_equal_twin(monkeypatch):
    """Every dict, block, direction and undecided list of one call equals the twin's; its layout takes 3 rule launches, 1
    figure launch and 1 direction launch more than a plain one, and its pages without "auto" get the tables of a call without
    the auto pages."""
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
    assert layout == [5 + 6 * _lib.PAGE_LEVELS + 3 + 1 + 1]
    seen = {"horizontal": 0, "vertical": 0}
    n_undecided = 0
    for k, ((img, pg, kw, auto), g) in enumerate(zip(items, got)):
        ref = _twin(img, kw, auto)
        if "error" in ref:
            assert isinstance(g, str) and ref["error"].split()[0] == g.split()[0], (k, g, ref)
            continue
        assert not isinstance(g, str), (k, g)
        assert _as_twin(g, auto) == ref, (k, _as_twin(g, auto), ref)
        if auto:
            for d in ref["directions"]:
                seen[d] += 1
            n_undecided += len(ref["undecided"])
    assert min(seen.values()) >= 100 and n_undecided >= 300, (seen, n_undecided)
    lattice = got[[k for k, it in enumerate(items) if it[0].shape == _lattice().shape][0]]
    assert len(lattice["blocks"]) == 1024 and len(lattice["undecided"]) == 341
    plain = [k for k, item in enumerate(items) if not item[3]]
    alone = _call(pipeline, [dimgs[k] for k in plain], [items[k][1] for k in plain])
    assert [got[k] for k in plain] == alone


def test_launch_counts():
    """A call with direction pages and no rules, figures or skew takes 5 + 6 * 24 + 1 launches; one without takes exactly the
    launches it took before, 5 + 6 * 24."""
    from marconet_b200 import _lib, ops, pipeline
    img, _ = magazine_page()
    d = [torch.from_numpy(img).to(DEV)] * 2
    n0 = ops.LAUNCHES
    auto = _call(pipeline, d, [pipeline.TextPage(block_direction="auto"), pipeline.TextPage()])
    assert ops.LAUNCHES - n0 == 5 + 6 * _lib.PAGE_LEVELS + 1
    n0 = ops.LAUNCHES
    without = _call(pipeline, d, [pipeline.TextPage(), pipeline.TextPage()])
    assert ops.LAUNCHES - n0 == 5 + 6 * _lib.PAGE_LEVELS
    assert auto[1] == without[1] == without[0]
    assert [b.direction for b in auto[0]["blocks"]] == ["horizontal", "horizontal", "vertical"]
    assert [b.rect for b in auto[0]["blocks"]] == [b.rect for b in without[0]["blocks"]]


def test_skewed_call_gives_a_direction_page_its_tables():
    from marconet_b200 import _lib, ops, pipeline
    news, _ = newspaper_page()
    mag, _ = magazine_page()
    dimgs = [torch.from_numpy(news).to(DEV), torch.from_numpy(mag).to(DEV)]
    pg = pipeline.TextPage(direction="vertical", block_direction="auto")
    alone = _call(pipeline, dimgs[:1], [pg])
    n0 = ops.LAUNCHES
    mixed = _call(pipeline, dimgs, [pg, pipeline.TextPage(skew="auto")])
    assert ops.LAUNCHES - n0 == 7 + 6 * _lib.PAGE_LEVELS + 1
    assert mixed[0] == alone[0]
    assert _as_twin(alone[0], True) == MP.find_blocks(news, direction="vertical")


def test_restore_regions_mixed_page_equals_the_found_blocks(gpu_models):
    from marconet_b200 import pipeline
    m = gpu_models["encoder"], gpu_models["tspgan"], gpu_models["sr"]
    img, drawn = magazine_page()
    pg = pipeline.TextPage(block_direction="auto")
    found = pipeline.find_blocks([img], [[pg]])[0][0]
    assert [b.direction for b in found["blocks"]] == [d for _, d, _ in drawn] and found["undecided"] == []
    kw = dict(scale=2, feather=3, to_host=True)
    a = pipeline.restore_regions(*m, [img], [[pg]], **kw)[0]
    b = pipeline.restore_regions(*m, [img], [found["blocks"]], **kw)[0]
    np.testing.assert_array_equal(a["image"], b["image"])
    assert {k: v for k, v in a["regions"][0].items() if k != "regions"} == found
    _same(a["regions"][0]["regions"], b["regions"])
    for blk, entry, (_, d, n) in zip(found["blocks"], a["regions"][0]["regions"], drawn):
        assert len(entry["lines"]) == n
        assert all(isinstance(r, pipeline.VerticalRegion) == (d == "vertical") for r in entry["lines"])
