"""Page turns on the device (DESIGN.md section 7b, "Page turns"): one find_blocks call of drawn pages at four turns, seeded
random pages and edge pages against the numpy twin's vote statistics bit for bit; the launch counts; ops.warp_perspective of
turned quads against np.rot90; pipeline.find_blocks, restore_regions and flatten_pages on turned pages against the same calls
given the turned quad, the found blocks and the upright page."""
import numpy as np
import pytest
import torch

from oracle import quad_pages as Q
from oracle import turn_pages as T

from test_gpu_pages import _same
from test_mixed_pages import _t, image, random_mixed, text
from test_ruled_pages import _photo
from test_turn_pages import PAGES, turned

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda:0")


def _wide():
    """A 32767-pixel-wide leaf of 3 lines whose longest ends in the page's last column (its last bitmap word)."""
    rng = np.random.default_rng(31)
    m = np.zeros((120, 32767), bool)
    for i, n in enumerate((1213, 1000, 1100)):
        text(m, rng, 32767 - 1213 * 27 + 3, 10 + 34 * i, 1, n, track=3, kind="whole")
    assert m[:, -1].any()
    return image(m)


def _chunk_edge(n):
    """Lines whose leaf spans n columns with bands across index 4096 of it (a chunk's end) on both axes."""
    rng = np.random.default_rng(n)
    m = np.zeros((110, n + 60), bool)
    for i, c in enumerate((153, 150)):
        text(m, rng, 10, 12 + 34 * i, 1, c, track=3, kind="whole")
    m[:, 10 + n:] = False
    return image(m)


def _tall():
    """131 ragged lines in one leaf over 4096 rows tall, a line across its row 4096 (a chunk's end)."""
    rng = np.random.default_rng(32)
    m = np.zeros((4500, 330), bool)
    for i in range(131):
        text(m, rng, 10, 10 + 34 * i, 1, int(rng.integers(3, 12)), kind="whole")
    return image(m)


def _lattice():
    """1024 blocks of two short lines each on a 40-pixel lattice: 1024 voting leaves."""
    m = np.zeros((32 * 40 + 20, 32 * 40 + 20), bool)
    for k in range(1024):
        r, c = divmod(k, 32)
        x, y = 20 + 40 * c, 20 + 40 * r
        m[y:y + 2, x:x + 14] = True
        m[y + 6:y + 8, x:x + 8 + k % 5] = True
    return image(m)


def _items(rng):
    """[(image, TextPage keywords, twin keywords)]: the drawn pages at four turns, 20 seeded random pages with rules, figures,
    panels and block_direction, and the edge pages."""
    out = []
    for make, d in PAGES.values():
        up = make()
        out += [(turned(up, k), dict(direction=d), dict(direction=d)) for k in range(4)]
    for j in range(20):
        img, kw = random_mixed(rng)
        if j % 4 == 1:
            img[10:14, :] = 20                          # a rule across the page
        extra = [dict(rules="auto"), dict(figures="auto"), dict(panels="auto"), dict(block_direction="auto")][j % 4]
        tw = dict(kw, **{k: True for k in extra if k != "block_direction"})
        out.append((img if "rect" in kw else turned(img, j % 4), dict(kw, **extra), tw))     # a crop stays upright
    out += [(_wide(), {}, {}), (_chunk_edge(4096), {}, {}), (_chunk_edge(4097), {}, {}),
            (_t(_chunk_edge(4096)), dict(direction="vertical"), dict(direction="vertical")),
            (_t(_chunk_edge(4097)), dict(direction="vertical"), dict(direction="vertical")), (_tall(), {}, {}),
            (_t(_tall()), dict(direction="vertical"), dict(direction="vertical")), (_lattice(), {}, {})]
    return out


def test_vote_tables_equal_twin():
    """Every kept leaf's (n_bands, E_lo, E_hi) and direction of one ops.find_blocks call equal the twin's."""
    from marconet_b200 import _lib, ops, pipeline
    rng = np.random.default_rng(5)
    items = _items(rng)
    dimgs = [torch.from_numpy(im).to(DEV) for im, _, _ in items]
    pages = []
    for d, (img, kw, _) in zip(dimgs, items):
        rect = kw.get("rect", (0, 0, img.shape[1], img.shape[0]))
        w, h = rect[2] - rect[0], rect[3] - rect[1]
        pages.append(ops.PageItem(d, rect, kw.get("direction") == "vertical", _lib.INK_AUTO,
                                  rule_length=ops.rule_length(w, h) if "rules" in kw else None,
                                  figure_size=0 if "figures" in kw else None, panel_size=0 if "panels" in kw else None,
                                  directions=True, turns=True))
    out, caps = ops.find_blocks(pages)
    host = pipeline._to_host(out).numpy()
    n_votes, tables = 0, ops.page_tables(host, pages, caps)
    for k, ((img, kw, tw), p, (_, r, leaves, _, _, tv)) in enumerate(zip(items, pages, tables)):
        ref = T.votes(img, **tw)
        kept = [(q, e) for q, e in zip(leaves, tv) if not q["st"] & _lib.PAGE_REJECTED]
        got = [(int(e["n_bands"]), int(e["e_lo"]), int(e["e_hi"])) for _, e in kept]
        assert int(r["error"]) == 0 and got == ref["stats"], (k, got[:8], ref["stats"][:8])
        assert ["vertical" if q["st"] & _lib.PAGE_VERTICAL else "horizontal" for q, _ in kept] == ref["directions"], k
        assert pipeline._turn_votes(p.vertical, leaves, tv) == ref["votes"], k
        n_votes += sum(n >= 2 for n, _, _ in got)
    assert sum(1 for q in tables[-1][2] if not q["st"] & _lib.PAGE_REJECTED) == 1024
    assert n_votes >= 1100
    for (img, kw, _), k in zip(items[:16], [0, 1, 2, 3] * 4):
        assert T.votes(img, **kw)["turn"] == 90 * k


def _call(pipeline, dimgs, pages):
    rects = [(0, 0, im.shape[1], im.shape[0]) if pg.rect is None else pg.rect for im, pg in zip(dimgs, pages)]
    return pipeline._find_pages(dict(enumerate(dimgs)), [(k, pg, r) for k, (pg, r) in enumerate(zip(pages, rects))])[0]


def _without(d, *keys):
    return {k: v for k, v in d.items() if k not in keys}


def test_turned_pages_and_launch_counts():
    """Every drawn page at every turn finds it; its dict is that of TextPage(quad=Q_k) plus turn and turn_votes, and its blocks
    are the upright page's; pass 1 adds the direction and turn launches, a turned page one rectify and one layout; a call
    without turn pages is unchanged."""
    from marconet_b200 import _lib, ops, pipeline
    layout = 5 + 6 * _lib.PAGE_LEVELS
    for name, (make, d) in PAGES.items():
        up = make()
        ref = _call(pipeline, [torch.from_numpy(up).to(DEV)], [pipeline.TextPage(direction=d)])[0]
        for k in range(4):
            img = turned(up, k)
            H, W = img.shape[:2]
            di = torch.from_numpy(img).to(DEV)
            n0 = ops.LAUNCHES
            got = _call(pipeline, [di], [pipeline.TextPage(direction=d, turn="auto")])[0]
            assert ops.LAUNCHES - n0 == layout + 2 + (layout + 1 if k else 0), (name, k)
            assert got["turn"] == 90 * k, (name, k, got["turn_votes"])
            q = pipeline.turn_quad((0, 0, W, H), 90 * k)
            given = _call(pipeline, [di], [pipeline.TextPage(direction=d, turn=90 * k)])[0]
            assert _without(got, "turn_votes") == given
            if k:
                quad = _call(pipeline, [di], [pipeline.TextPage(direction=d, quad=q)])[0]
                assert _without(given, "turn") == quad
                assert [b.window for b in got["blocks"]] == [tuple(b.rect) for b in ref["blocks"]]
            else:
                assert _without(got, "turn", "turn_votes") == ref
    img = PAGES["magazine"][0]()
    d = [torch.from_numpy(img).to(DEV)] * 2
    n0 = ops.LAUNCHES
    plain = _call(pipeline, d, [pipeline.TextPage(), pipeline.TextPage()])
    assert ops.LAUNCHES - n0 == layout
    mixed = _call(pipeline, d, [pipeline.TextPage(turn="auto"), pipeline.TextPage()])
    assert mixed[1] == plain[1]


@pytest.mark.parametrize("h, w", [(1, 37), (37, 1), (33, 64), (64, 33), (100, 100)])
def test_warp_perspective_of_turned_quads_is_rot90(h, w):
    from marconet_b200 import pipeline
    rng = np.random.default_rng(h + 7 * w)
    img = rng.integers(0, 256, (h + 9, w + 5, 3), dtype=np.uint8)
    rect = (2, 4, 2 + w, 4 + h)
    d = torch.from_numpy(img).to(DEV)
    keys = [pipeline._quad_key(0, pipeline.turn_quad(rect, t)) for t in pipeline.TURNS]
    rq = pipeline._rectify({0: d}, keys)
    for k, key in enumerate(keys):
        np.testing.assert_array_equal(rq[key].cpu().numpy(), np.rot90(img[4:4 + h, 2:2 + w], -k))


def test_restore_regions_turned_page(gpu_models):
    from marconet_b200 import pipeline
    m = gpu_models["encoder"], gpu_models["tspgan"], gpu_models["sr"]
    up = PAGES["paragraphs"][0]()
    kw = dict(scale=2, feather=3, to_host=True)
    for k in (1, 2):
        img = turned(up, k)
        H, W = img.shape[:2]
        found = pipeline.find_blocks([img], [[pipeline.TextPage(turn="auto")]])[0][0]
        assert found["turn"] == 90 * k
        a = pipeline.restore_regions(*m, [img], [[pipeline.TextPage(turn="auto")]], **kw)[0]
        b = pipeline.restore_regions(*m, [img], [[pipeline.TextPage(quad=pipeline.turn_quad((0, 0, W, H), 90 * k))]], **kw)[0]
        c = pipeline.restore_regions(*m, [img], [found["blocks"]], **kw)[0]
        np.testing.assert_array_equal(a["image"], b["image"])
        np.testing.assert_array_equal(a["image"], c["image"])
        _same(a["regions"][0]["regions"], c["regions"])
        assert _without(a["regions"][0], "regions") == found


def test_flatten_pages_turns_pages_upright():
    from marconet_b200 import pipeline
    FP = pipeline.FlatPage
    for name, (make, d) in PAGES.items():
        up = make()
        for k in range(4):
            img = turned(up, k)
            res = pipeline.flatten_pages([img], [[FP(direction=d, turn="auto"), FP(direction=d, turn=90 * k),
                                                  FP(direction=d, turn="auto", light="even")]], to_host=True)[0]
            np.testing.assert_array_equal(res[0]["image"], up)
            assert res[0]["turn"] == 90 * k and _without(res[0], "turn_votes", "image") == _without(res[1], "image")
            np.testing.assert_array_equal(res[1]["image"], up)
            assert res[2]["turn"] == 90 * k
    page = PAGES["paragraphs"][0]()
    h, w = page.shape[:2]
    photo = _photo(turned(page, 1), [(112, 118), (112 + h - 10, 110), (112 + h, 112 + w), (106, 116 + w - 6)], 5)
    res = pipeline.flatten_pages([photo], [[FP(quad="auto", turn="auto")]], to_host=True)[0][0]
    found = Q.accepted(Q.find_corners(photo), photo.shape)
    assert res["turn"] == 90
    ref = pipeline.flatten_pages([photo], [[FP(quad=pipeline.turn_quad(found, 90))]], to_host=True)[0][0]
    np.testing.assert_array_equal(res["image"], ref["image"])
    assert res["quad"] == ref["quad"]
