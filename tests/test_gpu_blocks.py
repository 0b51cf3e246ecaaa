"""Text blocks split into lines on the device (DESIGN.md section 7b, "Text blocks"): mn_find_lines_u8's line tables bit for bit
against the numpy twin, its constant launch count, and pipeline.restore_regions with TextBlocks against the same call given the
found lines."""
import cv2
import numpy as np
import pytest
import torch

from oracle import blocks as B

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda:0")
TEXTS = ["The quick brown fox", "jumps over 12 lazy dogs", "pack my box: 5 dozen jugs", "Sphinx of black quartz"]


def _models(gpu_models):
    return gpu_models["encoder"], gpu_models["tspgan"], gpu_models["sr"]


def _page(rng, n_lines, w=360, light=False, noise=0):
    h = 30 + 36 * n_lines
    page = np.empty((h, w, 3), np.uint8)
    page[:] = rng.integers(190, 256, 3)
    for k in range(n_lines):
        cv2.putText(page, TEXTS[k % len(TEXTS)], (8 + 5 * k, 36 + 36 * k), cv2.FONT_HERSHEY_SIMPLEX, 0.7,
                    tuple(int(v) for v in rng.integers(0, 70, 3)), 2, cv2.LINE_AA)
    if noise:
        page = np.clip(page.astype(np.int32) + rng.integers(-noise, noise + 1, page.shape), 0, 255).astype(np.uint8)
    return 255 - page if light else page


def _twin(img, rect, vertical, polarity, knobs):
    try:
        r = B.find_lines(img, rect, "vertical" if vertical else "horizontal", *knobs, polarity=polarity)
    except ValueError as e:
        return dict(error=str(e))
    return r


def _random_blocks(rng):
    """About 50 blocks: crops of drawn pages read through the page's pitch, noisy and light-on-dark pages, vertical blocks,
    random pixels, 1 x 1 and uniform blocks, a block of 32767 rows and one of 300 lines."""
    pages = [_page(rng, 5), _page(rng, 3, light=True), _page(rng, 4, noise=30), rng.integers(0, 256, (90, 70, 3), dtype=np.uint8),
             np.full((40, 50, 3), 131, np.uint8)]
    pages.append(np.ascontiguousarray(_page(rng, 4).transpose(1, 0, 2)))
    tall = np.full((32767, 9, 3), 240, np.uint8)
    tall[(np.arange(32767) // 7) % 40 == 0, 2:7] = 10
    pages.append(tall)
    stripes = np.full((1800, 20, 3), 255, np.uint8)
    stripes[np.arange(1800) % 6 < 3] = 0
    pages.append(stripes)
    items = []
    for k in range(52):
        i = int(rng.integers(0, 6)) if k >= 8 else k
        H, W = pages[i].shape[:2]
        if k < 8 or rng.random() < 0.3:
            rect = (0, 0, W, H)
        elif k in (8, 9) or rng.random() < 0.1:
            x, y = int(rng.integers(0, W)), int(rng.integers(0, H))
            rect = (x, y, x + 1, y + 1)
        else:
            x0, y0 = int(rng.integers(0, W - 1)), int(rng.integers(0, H - 1))
            rect = (x0, y0, int(rng.integers(x0 + 1, W + 1)), int(rng.integers(y0 + 1, H + 1)))
        vertical = i == 5 or (k >= 8 and rng.random() < 0.2)
        polarity = ["auto", "auto", "dark", "light"][int(rng.integers(0, 4))] if k >= 8 else "auto"
        knobs = [int(rng.integers(1, 6)) if rng.random() < 0.2 else None for _ in range(3)] if k >= 8 else [None] * 3
        items.append((i, rect, vertical, polarity, knobs))
    return pages, items


def test_line_tables_equal_twin():
    """Every threshold, polarity, line count and rectangle equals the twin's, in four launches for 52 blocks as for one."""
    from marconet_b200 import _lib, ops
    rng = np.random.default_rng(0)
    pages, items = _random_blocks(rng)
    dpages = [torch.from_numpy(p).to(DEV) for p in pages]
    pol = dict(auto=_lib.INK_AUTO, dark=_lib.INK_DARK, light=_lib.INK_LIGHT)
    args = [(dpages[i], rect, v, pol[p], *knobs) for i, rect, v, p, knobs in items]
    n0 = ops.LAUNCHES
    one = ops.find_lines(args[:1])
    assert ops.LAUNCHES - n0 == 4
    n0 = ops.LAUNCHES
    table = ops.find_lines(args)
    assert ops.LAUNCHES - n0 == 4
    rec = table.cpu().numpy().view(ops.block_lines_dtype())
    assert bytes(one.cpu().numpy()[:16]) == bytes(table.cpu().numpy()[:16])
    seen = set()
    for k, ((i, rect, v, p, knobs), r) in enumerate(zip(items, rec)):
        ref = _twin(pages[i], rect, v, p, knobs)
        n = int(r["n_lines"])
        if "error" in ref:
            assert n < 0 and f"{-n} lines exceed" in ref["error"], (k, n, ref)
            seen.add("over")
            continue
        assert int(r["threshold"]) == ref["threshold"], (k, rect)
        assert ("dark" if r["ink"] == _lib.INK_DARK else "light") == ref["ink"], (k, rect)
        assert n == len(ref["lines"]), (k, rect, n, ref)
        assert [tuple(int(x) for x in q) for q in r["rect"][:n]] == ref["lines"], (k, rect)
        seen.add("lines" if n > 1 else "none" if n == 0 else "one")
        if rect[2] - rect[0] == 1 and rect[3] - rect[1] == 1:
            seen.add("1x1")
        if rect[3] - rect[1] == 32767:
            seen.add("tall")
    assert {"over", "lines", "none", "one", "tall"} <= seen, seen


def test_find_lines_matches_twin_and_raises_over_the_limit():
    from marconet_b200 import pipeline
    rng = np.random.default_rng(1)
    page = _page(rng, 4)
    col = np.ascontiguousarray(_page(rng, 3).transpose(1, 0, 2))
    out = pipeline.find_lines([page, torch.from_numpy(col).to(DEV)],
                              [[pipeline.TextBlock((0, 0, page.shape[1], page.shape[0]))],
                               [pipeline.TextBlock((0, 0, col.shape[1], col.shape[0]), "vertical")]])
    ref = B.find_lines(page, (0, 0, page.shape[1], page.shape[0]))
    assert out[0] == [ref] and len(ref["lines"]) == 4
    refv = B.find_lines(col, (0, 0, col.shape[1], col.shape[0]), "vertical")
    assert out[1] == [dict(refv, lines=[pipeline.VerticalRegion(q) for q in refv["lines"]])] and len(refv["lines"]) == 3
    stripes = np.full((1800, 20, 3), 255, np.uint8)
    stripes[np.arange(1800) % 6 < 3] = 0
    with pytest.raises(ValueError, match="image 0, block 0: 300 lines exceed the 256"):
        pipeline.find_lines([stripes], [[pipeline.TextBlock((0, 0, 20, 1800))]])


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
def test_restore_regions_blocks_equal_the_found_lines(gpu_models, to_host):
    """A call with blocks gives the bytes of the call given their lines: pages and every line's entry, horizontal and vertical,
    beside rectangles, oriented, perspective, curved and vertical regions, and a zero-line block."""
    from marconet_b200 import pipeline
    m = _models(gpu_models)
    rng = np.random.default_rng(2)
    img = np.full((340, 420, 3), 235, np.uint8)
    img[10:112, 10:370] = _page(rng, 2, w=360)
    col = np.ascontiguousarray(_page(rng, 2, w=200).transpose(1, 0, 2))
    img[120:320, 300:402] = col
    hb = pipeline.TextBlock((10, 10, 370, 112))
    vb = pipeline.TextBlock((300, 120, 402, 320), "vertical")
    empty = pipeline.TextBlock((0, 320, 60, 340))
    others = [(20, 200, 120, 240), pipeline.OrientedRegion.from_rotated(150, 220, 120, 30, 8),
              pipeline.QuadRegion((130, 250), (250, 245), (255, 290), (128, 292)),
              pipeline.CurvedRegion.from_arc(150, 230, 80, 105, 220, 320), pipeline.VerticalRegion((260, 130, 290, 250))]
    found = pipeline.find_lines([img], [[hb, vb, empty]])[0]
    assert len(found[0]["lines"]) == 2 and len(found[1]["lines"]) == 2 and found[2]["lines"] == []
    regs = [others[0], hb, others[1], vb, others[2], empty, others[3], others[4]]
    flat = [others[0], *found[0]["lines"], others[1], *found[1]["lines"], others[2], others[3], others[4]]
    kw = dict(scale=2, feather=3, skip_invalid=True, to_host=to_host)
    a = pipeline.restore_regions(*m, [img], [regs], **kw)[0]
    b = pipeline.restore_regions(*m, [img], [flat], **kw)[0]
    _same(a["image"], b["image"])
    e = a["regions"]
    assert len(e) == len(regs)
    for k, blk in ((1, 0), (3, 1), (5, 2)):
        assert {x: e[k][x] for x in ("lines", "threshold", "ink")} == found[blk]
    _same(e[0], b["regions"][0])
    _same(e[1]["regions"], b["regions"][1:3])
    _same(e[2], b["regions"][3])
    _same(e[3]["regions"], b["regions"][4:6])
    _same(e[4], b["regions"][6])
    assert e[5]["regions"] == []
    _same(e[6:], b["regions"][7:])


def test_block_over_the_limit_under_skip_invalid(gpu_models):
    from marconet_b200 import ops, pipeline
    m = _models(gpu_models)
    img = np.full((1800, 40, 3), 255, np.uint8)
    img[np.arange(1800) % 6 < 3, :20] = 0
    regs = [pipeline.TextBlock((0, 0, 20, 1800)), (20, 0, 40, 40)]
    with pytest.raises(ValueError, match="image 0, region 0 \\(a text block\\): 300 lines exceed"):
        pipeline.restore_regions(*m, [img], [regs])
    n0 = ops.LAUNCHES
    a = pipeline.restore_regions(*m, [img], [regs], skip_invalid=True, to_host=True)[0]
    assert "300 lines exceed" in a["regions"][0]["error"]
    b = pipeline.restore_regions(*m, [img], [regs[1:]], skip_invalid=True, to_host=True)[0]
    _same(a["image"], b["image"])
    _same(a["regions"][1], b["regions"][0])
    assert n0 < ops.LAUNCHES
