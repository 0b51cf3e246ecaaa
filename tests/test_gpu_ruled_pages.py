"""Ruled pages on the device (DESIGN.md section 7b, "Ruled pages"): one find_blocks call of ruled pages of every kind, random
pages with random rules, 32767-pixel runs and pages without rules against the numpy twins bit for bit, with its launch count;
a call mixing a skewed page and a ruled page; a photographed table under quad="auto"; and restore_regions with a ruled page
against the same call given the found blocks."""
import numpy as np
import pytest
import torch

from oracle import pages as P
from oracle import quad_pages as Q
from oracle import ruled_pages as RP

from test_gpu_pages import _same
from test_ruled_pages import _img, framed_page, newspaper_page, photographed_table, table_beside_column, table_page

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda:0")


def _random_ruled(rng):
    """A random page of specks and rules: horizontal and vertical segments of random lengths around a random rule length l,
    some exactly l and l - 1 long, crossing word boundaries.  (image, l, or None for the default)."""
    h, w = int(rng.integers(20, 300)), int(rng.integers(20, 700))
    l = int(rng.integers(2, 80))
    ink = rng.random((h, w)) < rng.choice([0.005, 0.03, 0.2])
    for _ in range(int(rng.integers(1, 12))):
        n = int(max(1, l + rng.integers(-2, 3) if rng.random() < 0.5 else rng.integers(1, 4 * l)))
        if rng.random() < 0.5:
            y, x = int(rng.integers(0, h)), int(rng.integers(-n // 2, w))
            ink[y:y + int(rng.integers(1, 3)), max(0, x):x + n] = True
        else:
            y, x = int(rng.integers(-n // 2, h)), int(rng.integers(0, w))
            ink[max(0, y):y + n, x:x + int(rng.integers(1, 3))] = True
    return _img(ink), (l if rng.random() < 0.7 else None)


def _long_runs(vertical):
    """A page 32767 pixels along its rows (columns when ``vertical``): a run of 32767, one of 32766 and a dotted row."""
    m = np.zeros((3, 32767), bool)
    m[0] = True
    m[1, 1:] = True
    m[2, ::3] = True
    return _img(m.T if vertical else m)


def _pages(rng):
    """[(image, TextPage, the twin's keyword arguments, whether the page has rules)]."""
    from marconet_b200 import pipeline
    TP = pipeline.TextPage
    table, _ = table_page(4, 3)
    edge = np.zeros((21, 40), bool)
    edge[2:9, 2:38:3] = edge[12:19, 2:38:3] = True
    edge[10, :20] = True
    out = [(table, {}), (framed_page(5)[0], {}), (table_beside_column()[0], {}), (newspaper_page()[0], {}),
           (np.ascontiguousarray(table.transpose(1, 0, 2)[:, ::-1]), dict(direction="vertical")), (255 - table, {}),
           (_img(edge), dict(rule_length=10)), (_img(edge), dict(rect=(0, 0, 39, 21), rule_length=10))]
    out += [(_long_runs(v), dict(polarity="dark", rule_length=n)) for v, n in ((False, 32767), (True, 32767), (False, 32766))]
    for k in range(24):
        img, l = _random_ruled(rng)
        H, W = img.shape[:2]
        rect = None if k % 3 else (int(rng.integers(0, W // 3)), int(rng.integers(0, H // 3)), W - int(rng.integers(0, W // 3)), H)
        out.append((img, dict(rect=rect, direction="vertical" if k % 5 == 4 else "horizontal", rule_length=l)))
    pages = [(img, TP(rules="auto", **kw), kw, True) for img, kw in out]
    plain = [(table, {}), (newspaper_page()[0], dict(gap_x=7))] + [out[k] for k in range(11, len(out), 6)]
    pages += [(img, TP(**{k: v for k, v in kw.items() if k != "rule_length"}), kw, False) for img, kw in plain]
    return pages


def _twin(img, kw, ruled):
    try:
        return RP.find_blocks(img, **kw) if ruled else P.find_blocks(img, **{k: v for k, v in kw.items() if k != "rule_length"})
    except ValueError as e:
        return dict(error=str(e))


def _rects(got):
    return dict(got, blocks=[tuple(b.rect) for b in got["blocks"]])


def _call(pipeline, dimgs, pages):
    rects = [(0, 0, im.shape[1], im.shape[0]) if pg.rect is None else pg.rect for im, pg in zip(dimgs, pages)]
    return pipeline._find_blocks(dict(enumerate(dimgs)), [(k, pg, r) for k, (pg, r) in enumerate(zip(pages, rects))])


def test_ruled_pages_equal_twin():
    """Every dict and block of one call equals the twin's; the call takes 3 launches more than one without rules, and its pages
    without rules get the tables of a call without the ruled pages."""
    from marconet_b200 import _lib, ops, pipeline
    rng = np.random.default_rng(0)
    items = _pages(rng)
    dimgs = [torch.from_numpy(im).to(DEV) for im, *_ in items]
    n0 = ops.LAUNCHES
    got = _call(pipeline, dimgs, [pg for _, pg, *_ in items])
    assert ops.LAUNCHES - n0 == 5 + 6 * _lib.PAGE_LEVELS + 3
    seen = set()
    for k, ((img, pg, kw, ruled), g) in enumerate(zip(items, got)):
        ref = _twin(img, kw, ruled)
        if "error" in ref:
            assert isinstance(g, str) and ref["error"].split()[0] == g.split()[0], (k, g, ref)
            continue
        assert not isinstance(g, str), (k, g)
        assert _rects(g) == ref, (k, _rects(g), ref)
        if ruled:
            plain = _twin(img, kw, False)
            seen.update(["rules"] if ref["rule_pixels"] else [])
            seen.update(["cut"] if "error" not in plain and len(ref["blocks"]) > len(plain["blocks"]) else [])
            seen.update(["run 32767"] if ref["rule_length"] == 32767 and ref["rule_pixels"] == 32767 else [])
    assert {"cut", "rules", "run 32767"} <= seen, seen
    plain = [k for k, item in enumerate(items) if not item[3]]
    alone = _call(pipeline, [dimgs[k] for k in plain], [items[k][1] for k in plain])
    assert [got[k] for k in plain] == alone


def test_skewed_call_gives_a_ruled_page_its_tables():
    """A call with a skewed page runs every page through the skewed entry point: the ruled page's frame bitmap is the level
    one and its tables are those of a call that holds it alone."""
    from marconet_b200 import _lib, ops, pipeline
    table, _ = table_page(4, 3)
    news, _ = newspaper_page()
    dimgs = [torch.from_numpy(table).to(DEV), torch.from_numpy(news).to(DEV)]
    alone = _call(pipeline, dimgs[:1], [pipeline.TextPage(rules="auto")])
    n0 = ops.LAUNCHES
    mixed = _call(pipeline, dimgs, [pipeline.TextPage(rules="auto"), pipeline.TextPage(skew="auto")])
    assert ops.LAUNCHES - n0 == 7 + 6 * _lib.PAGE_LEVELS + 3
    assert mixed[0] == alone[0] and len(alone[0]["blocks"]) == 13
    assert _rects(alone[0]) == RP.find_blocks(table)


def test_photographed_table_under_quad_auto():
    from marconet_b200 import pipeline
    img = photographed_table()
    got = pipeline.find_blocks([img], [[pipeline.TextPage(quad="auto", rules="auto")]])[0][0]
    quad = Q.accepted(Q.find_corners(img), img.shape)
    want = RP.find_quad_blocks(img, quad)
    assert got["quad"] == want["quad"] and got["size"] == want["size"] and len(want["blocks"]) == 13
    assert [b.window for b in got["blocks"]] == want["blocks"]
    assert {k: got[k] for k in want if k != "blocks"} == {k: v for k, v in want.items() if k != "blocks"}


def test_restore_regions_ruled_page_equals_the_found_blocks(gpu_models):
    from marconet_b200 import pipeline
    m = gpu_models["encoder"], gpu_models["tspgan"], gpu_models["sr"]
    img, _ = table_page(4, 3)
    pg = pipeline.TextPage(rules="auto")
    found = pipeline.find_blocks([img], [[pg]])[0][0]
    assert len(found["blocks"]) == 13
    kw = dict(scale=2, feather=3, to_host=True)
    a = pipeline.restore_regions(*m, [img], [[pg]], **kw)[0]
    b = pipeline.restore_regions(*m, [img], [found["blocks"]], **kw)[0]
    np.testing.assert_array_equal(a["image"], b["image"])
    assert {k: v for k, v in a["regions"][0].items() if k != "regions"} == found
    assert len(a["regions"][0]["regions"]) == 13
    _same(a["regions"][0]["regions"], b["regions"])
