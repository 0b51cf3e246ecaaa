"""Text pages split into blocks on the device (DESIGN.md section 7b, "Text pages"): mn_find_blocks_u8's tables bit for bit
against the numpy twin over about 50 pages in one call, its constant launch count, and pipeline.restore_regions with TextPages
against the same call given the found blocks and given the found lines."""
import cv2
import numpy as np
import pytest
import torch

from oracle import pages as P

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda:0")
WORDS = "THE QUICK BROWN FOX JUMPS OVER A LAZY DOG PACK MY BOX WITH FIVE DOZEN JUGS".split()


def _models(gpu_models):
    return gpu_models["encoder"], gpu_models["tspgan"], gpu_models["sr"]


def _columns_page(rng, widths, n_lines, misalign=False, noise=0):
    """A heading over columns of capital-letter lines (DUPLEX, 33 pixels apart, 60-pixel gutters), as in test_pages.py."""
    pitch, gutter = 33, 60
    W = 40 + sum(widths) + gutter * (len(widths) - 1)
    H = 120 + n_lines * pitch + pitch // 2
    page = np.empty((H, W, 3), np.uint8)
    page[:] = rng.integers(200, 250, 3)
    fg = tuple(int(v) for v in rng.integers(0, 60, 3))
    cv2.putText(page, "HEADING OVER ALL COLUMNS"[:max(8, W // 22)], (20, 42), cv2.FONT_HERSHEY_DUPLEX, 1.0, fg, 2, cv2.LINE_8)
    x = 20
    for c, cw in enumerate(widths):
        for k in range(n_lines):
            t = str(rng.choice(WORDS))
            while True:
                longer = t + " " + str(rng.choice(WORDS))
                if cv2.getTextSize(longer, cv2.FONT_HERSHEY_DUPLEX, 1.0, 2)[0][0] > cw:
                    break
                t = longer
            y = 100 + k * pitch + (pitch // 2 if misalign and c % 2 else 0)
            cv2.putText(page, t, (x, y), cv2.FONT_HERSHEY_DUPLEX, 1.0, fg, 2, cv2.LINE_8)
        x += cw + gutter
    if noise:
        page = np.clip(page.astype(np.int32) + rng.integers(-noise, noise + 1, page.shape), 0, 255).astype(np.uint8)
    return page


def _twin(img, rect, vertical, polarity, gaps):
    try:
        return P.find_blocks(img, rect, "vertical" if vertical else "horizontal", polarity, *gaps)
    except ValueError as e:
        return dict(error=str(e))


def _random_pages(rng):
    """About 50 pages: drawn multi-column pages (noisy, light-on-dark, transposed), random ink, crops read through the page's
    pitch, a 1 x 1 page, a uniform page, a page of 32767 rows, one over the block limit and one over the node limit."""
    imgs = [_columns_page(rng, (300, 300), 5), _columns_page(rng, (200, 350, 250), 4, misalign=True, noise=20),
            255 - _columns_page(rng, (260, 300), 3), np.ascontiguousarray(_columns_page(rng, (300, 300), 4).transpose(1, 0, 2)),
            np.where(rng.random((180, 230, 1)) < 0.03, 10, 240).astype(np.uint8).repeat(3, axis=2),
            np.full((40, 50, 3), 131, np.uint8)]
    tall = np.full((32767, 40, 3), 240, np.uint8)
    tall[(np.arange(32767) // 9) % 40 < 3, 5:35:3] = 10
    pairs = np.full((2, 3 * 1100, 3), 240, np.uint8)
    pairs[0, ::3] = pairs[1, 1::3] = 10
    dots = np.full((600, 600, 3), 240, np.uint8)
    dots[::2, ::2] = 10
    imgs += [tall, pairs, dots]
    items = [(6, None, False, "auto", (None, None)), (7, None, False, "auto", (1, 1)), (8, None, False, "auto", (None, None)),
             (5, (3, 4, 4, 5), False, "auto", (None, None))]
    for k in range(46):
        i = k % 5 if k < 10 else int(rng.integers(0, 6))
        H, W = imgs[i].shape[:2]
        if k < 10 or rng.random() < 0.3:
            rect = None
        else:
            x0, y0 = int(rng.integers(0, W - 1)), int(rng.integers(0, H - 1))
            rect = (x0, y0, int(rng.integers(x0 + 1, W + 1)), int(rng.integers(y0 + 1, H + 1)))
        vertical = i == 3 or (k >= 10 and rng.random() < 0.2)
        polarity = ["auto", "auto", "dark", "light"][int(rng.integers(0, 4))] if k >= 10 else "auto"
        gaps = tuple(int(rng.integers(1, 30)) if rng.random() < 0.2 else None for _ in range(2)) if k >= 10 else (None, None)
        items.append((i, rect, vertical, polarity, gaps))
    return imgs, items


def test_page_tables_equal_twin():
    """Every block, rejected leaf, S, gap, threshold and ink equals the twin's, and every error is the twin's, in the same
    launches for one page as for 50."""
    from marconet_b200 import _lib, ops, pipeline
    rng = np.random.default_rng(0)
    imgs, items = _random_pages(rng)
    dimgs = [torch.from_numpy(im).to(DEV) for im in imgs]
    rects = [r if r is not None else (0, 0, imgs[i].shape[1], imgs[i].shape[0]) for i, r, *_ in items]
    pol = dict(auto=_lib.INK_AUTO, dark=_lib.INK_DARK, light=_lib.INK_LIGHT)
    args = [ops.PageItem(dimgs[i], rect, v, pol[p], *g) for (i, _, v, p, g), rect in zip(items, rects)]
    n0 = ops.LAUNCHES
    ops.find_blocks(args[:1])
    one = ops.LAUNCHES - n0
    n0 = ops.LAUNCHES
    ops.find_blocks(args)
    assert ops.LAUNCHES - n0 == one == 5 + 6 * _lib.PAGE_LEVELS
    dev = pipeline._find_blocks(dict(enumerate(dimgs)), [(i, pipeline.TextPage(r, "vertical" if v else "horizontal", p, *g), rect)
                                                         for (i, r, v, p, g), rect in zip(items, rects)])
    seen = set()
    for k, ((i, _, v, p, g), rect, got) in enumerate(zip(items, rects, dev)):
        ref = _twin(imgs[i], rect, v, p, g)
        if "error" in ref:
            assert isinstance(got, str), (k, got)
            assert ("nodes" in got) == ("nodes" in ref["error"]) and ref["error"].split()[0] == got.split()[0], (k, got, ref)
            seen.add("nodes" if "nodes" in got else "blocks")
            continue
        assert not isinstance(got, str), (k, got, ref)
        assert [tuple(b.rect) for b in got["blocks"]] == ref["blocks"], (k, rect)
        assert all(b.direction == ("vertical" if v else "horizontal") and b.polarity == p for b in got["blocks"])
        for key in ("rejected", "threshold", "ink", "text_size", "gap_x", "gap_y"):
            assert got[key] == ref[key], (k, key, got[key], ref[key])
        seen.add("blocks" if len(ref["blocks"]) > 1 else "none" if not ref["blocks"] else "one")
        seen.update(["rejected"] if ref["rejected"] else [])
        if rect[2] - rect[0] == 1 and rect[3] - rect[1] == 1:
            seen.add("1x1")
        if rect[3] - rect[1] == 32767:
            seen.add("tall")
    assert {"nodes", "blocks", "none", "one", "rejected", "1x1", "tall"} <= seen, seen


def test_find_blocks_matches_twin_and_raises_over_a_limit():
    from marconet_b200 import pipeline
    rng = np.random.default_rng(1)
    page = _columns_page(rng, (300, 300), 4)
    out = pipeline.find_blocks([page, torch.from_numpy(page).to(DEV)],
                               [[pipeline.TextPage()], [pipeline.TextPage((5, 5, 500, 200), "vertical", "dark", 7, 9)]])
    ref = P.find_blocks(page)
    assert len(ref["blocks"]) == 3
    assert dict(out[0][0], blocks=[b.rect for b in out[0][0]["blocks"]]) == ref
    refv = P.find_blocks(page, (5, 5, 500, 200), "vertical", "dark", 7, 9)
    assert [b for b in out[1][0]["blocks"]] == [pipeline.TextBlock(r, "vertical", polarity="dark") for r in refv["blocks"]]
    dots = np.full((600, 600, 3), 240, np.uint8)
    dots[::2, ::2] = 10
    with pytest.raises(ValueError, match="image 1, page 0: more than 65536 nodes"):
        pipeline.find_blocks([page, dots], [[], [pipeline.TextPage()]])


def _same(a, b):
    if isinstance(a, dict):
        assert a.keys() == b.keys()
        for k in a:
            _same(a[k], b[k])
    elif isinstance(a, (list, tuple)):
        assert len(a) == len(b)
        for x, y in zip(a, b):
            _same(x, y)
    elif isinstance(a, (np.ndarray, torch.Tensor)):
        x = a.cpu().numpy() if isinstance(a, torch.Tensor) else a
        y = b.cpu().numpy() if isinstance(b, torch.Tensor) else b
        np.testing.assert_array_equal(x, y)
    else:
        assert a == b


@pytest.mark.parametrize("to_host", [False, True])
def test_restore_regions_pages_equal_the_found_blocks(gpu_models, to_host):
    """A call with pages gives the bytes of the call given their blocks and of the call given their lines, beside rectangles,
    oriented, perspective, curved and vertical regions, a text block and a page with zero blocks."""
    from marconet_b200 import pipeline
    m = _models(gpu_models)
    rng = np.random.default_rng(2)
    page = _columns_page(rng, (260, 260), 3)
    img = np.full((page.shape[0] + 130, page.shape[1] + 20, 3), 238, np.uint8)
    img[:page.shape[0], :page.shape[1]] = page
    H, W = page.shape[:2]
    pg = pipeline.TextPage((0, 0, W, H))
    empty = pipeline.TextPage((W, 0, W + 20, 40))
    blk = pipeline.TextBlock((0, H + 5, 300, H + 60))
    cv2.putText(img, "JUGS OF FIVE", (10, H + 40), cv2.FONT_HERSHEY_DUPLEX, 1.0, (20, 20, 20), 2, cv2.LINE_8)
    others = [(20, H + 70, 120, H + 110), pipeline.OrientedRegion.from_rotated(200, H + 90, 120, 30, 8),
              pipeline.QuadRegion((330, H + 70), (450, H + 65), (455, H + 110), (328, H + 112)),
              pipeline.CurvedRegion.from_arc(520, H + 60, 50, 60, 200, 340), pipeline.VerticalRegion((W - 10, H + 5, W + 15, H + 125))]
    found = pipeline.find_blocks([img], [[pg, empty]])[0]
    assert len(found[0]["blocks"]) == 3 and found[1]["blocks"] == []
    regs = [others[0], pg, others[1], blk, others[2], empty, others[3], others[4]]
    with_blocks = [others[0], *found[0]["blocks"], others[1], blk, others[2], others[3], others[4]]
    lines = pipeline.find_lines([img], [found[0]["blocks"] + [blk]])[0]
    with_lines = [others[0], *[q for r in lines[:3] for q in r["lines"]], others[1], *lines[3]["lines"], others[2], others[3],
                  others[4]]
    kw = dict(scale=2, feather=3, skip_invalid=True, to_host=to_host)
    a = pipeline.restore_regions(*m, [img], [regs], **kw)[0]
    b = pipeline.restore_regions(*m, [img], [with_blocks], **kw)[0]
    c = pipeline.restore_regions(*m, [img], [with_lines], **kw)[0]
    _same(a["image"], b["image"])
    _same(a["image"], c["image"])
    e = a["regions"]
    assert len(e) == len(regs)
    assert {k: v for k, v in e[1].items() if k != "regions"} == found[0]
    _same(e[0], b["regions"][0])
    _same(e[1]["regions"], b["regions"][1:4])
    _same(e[2:5], b["regions"][4:7])
    assert e[5] == dict(found[1], regions=[])
    _same(e[6:], b["regions"][7:])


def test_failing_page_under_skip_invalid(gpu_models):
    """A page over the node limit, and a page one of whose blocks has too many lines, raise, or become dict(error=...) under
    skip_invalid, leaving the rest of the call as the call without them."""
    from marconet_b200 import ops, pipeline
    m = _models(gpu_models)
    img = np.full((2400, 700, 3), 240, np.uint8)
    img[:600, :600][::2, ::2] = 10
    img[600:2400, 620:660][np.arange(1800) % 6 < 2] = 10     # 300 stripes that gap_y keeps in one block of 300 lines
    dots = pipeline.TextPage((0, 0, 600, 600))
    striped = pipeline.TextPage((610, 600, 700, 2400), gap_y=1000)
    regs = [dots, (0, 700, 200, 740), striped]
    with pytest.raises(ValueError, match="image 0, region 0 \\(a text page\\): more than 65536 nodes"):
        pipeline.restore_regions(*m, [img], [regs])
    with pytest.raises(ValueError, match="image 0, region 0 \\(a text page\\), block 0: 300 lines exceed"):
        pipeline.restore_regions(*m, [img], [[striped]])
    n0 = ops.LAUNCHES
    a = pipeline.restore_regions(*m, [img], [regs], skip_invalid=True, to_host=True)[0]
    assert "more than 65536 nodes" in a["regions"][0]["error"]
    assert "block 0: 300 lines exceed" in a["regions"][2]["error"]
    b = pipeline.restore_regions(*m, [img], [regs[1:2]], skip_invalid=True, to_host=True)[0]
    _same(a["image"], b["image"])
    _same(a["regions"][1], b["regions"][0])
    assert n0 < ops.LAUNCHES


def test_calls_without_pages_do_not_run_the_layout(gpu_models, monkeypatch):
    """A restore_regions call without pages issues exactly the launches it issued before: the page path is not entered.  Module
    graphs are off, so that every launch is counted in both calls."""
    from marconet_b200 import ops, pipeline
    m = _models(gpu_models)
    monkeypatch.setattr(ops, "MODULE_GRAPHS", False)
    rng = np.random.default_rng(3)
    img = _columns_page(rng, (260, 260), 2)
    regs = [pipeline.TextBlock((0, 0, img.shape[1], img.shape[0])), (10, 10, 100, 40)]
    before = ops.LAUNCHES
    pipeline.restore_regions(*m, [img], [regs], to_host=True)
    first = ops.LAUNCHES - before

    def refuse(*a, **k):
        raise AssertionError("find_blocks ran for a call without pages")
    monkeypatch.setattr(ops, "find_blocks", refuse)
    before = ops.LAUNCHES
    pipeline.restore_regions(*m, [img], [regs], to_host=True)
    assert ops.LAUNCHES - before == first
