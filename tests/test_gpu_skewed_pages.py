"""Skewed text pages and windowed blocks on the device (DESIGN.md section 7b, "Skewed pages"): mn_find_blocks_skewed_u8's
tables and mn_find_lines_window_u8's line tables bit for bit against the numpy twin, their constant launch counts, and
pipeline.restore_regions with tilted TextPages against the same call given the found blocks and given the found lines."""
import numpy as np
import pytest
import torch

from oracle import skewed_pages as SP

from test_skewed_pages import drawn_page

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda:0")


def _models(gpu_models):
    return gpu_models["encoder"], gpu_models["tspgan"], gpu_models["sr"]


def _pages(rng):
    """About 40 pages: tilted drawn pages in both directions, noisy, light on dark, crops read through the page's pitch, pages
    with None, a given angle and "auto", a 1 x 1 page and a uniform page."""
    imgs = []
    for k, angle in enumerate((-6.0, 2.5, 9.0, -1.5, 4.0, 0.0)):
        img, _ = drawn_page((220, 240) if k % 2 else (260,), 5, angle, seed=k, vertical=k in (1, 4), misalign=k == 2)
        if k == 2:
            img = np.clip(img.astype(np.int32) + rng.integers(-20, 21, img.shape), 0, 255).astype(np.uint8)
        if k == 3:
            img = 255 - img
        imgs.append(img)
    imgs.append(np.full((40, 50, 3), 131, np.uint8))
    items = [(6, None, False, "auto", "auto"), (6, (3, 4, 4, 5), False, "auto", "auto"), (6, (3, 4, 4, 5), True, "auto", 7.0)]
    for k in range(38):
        i = k % 6
        H, W = imgs[i].shape[:2]
        vertical = i in (1, 4)
        if k < 12 or rng.random() < 0.4:
            rect = None
        else:
            x0, y0 = int(rng.integers(0, W // 3)), int(rng.integers(0, H // 3))
            rect = (x0, y0, int(rng.integers(2 * W // 3, W + 1)), int(rng.integers(2 * H // 3, H + 1)))
        polarity = "light" if i == 3 and k % 3 == 0 else "auto"
        skew = [None, "auto", "auto", float(rng.uniform(-9, 9)), 0.0][k % 5] if k >= 6 else "auto"
        items.append((i, rect, vertical, polarity, skew))
    return imgs, items


def _twin(img, rect, vertical, polarity, skew):
    d = "vertical" if vertical else "horizontal"
    if skew is None:
        from oracle import pages as P
        return dict(P.find_blocks(img, rect, d, polarity), skew=None, detail=None)
    return SP.find_blocks(img, rect, d, polarity, skew=skew)


def test_skewed_page_tables_equal_twin():
    """The chosen index, scores, frame, leaves and blocks equal the twin's, in the same launches for one page as for 40."""
    from marconet_b200 import _lib, ops, pipeline
    rng = np.random.default_rng(0)
    imgs, items = _pages(rng)
    dimgs = [torch.from_numpy(im).to(DEV) for im in imgs]
    rects = [r if r is not None else (0, 0, imgs[i].shape[1], imgs[i].shape[0]) for i, r, *_ in items]
    pol = dict(auto=_lib.INK_AUTO, dark=_lib.INK_DARK, light=_lib.INK_LIGHT)
    args = [ops.PageItem(dimgs[i], rect, v, pol[p], skew=sk) for (i, _, v, p, sk), rect in zip(items, rects)]
    n0 = ops.LAUNCHES
    ops.find_blocks(args[:1])
    one = ops.LAUNCHES - n0
    n0 = ops.LAUNCHES
    out, caps, scores = ops.find_blocks(args, scores=True)
    assert ops.LAUNCHES - n0 == one == 7 + 6 * _lib.PAGE_LEVELS
    host = out.cpu().numpy()
    sdt = ops.skew_block_dtype()
    sk = host[:len(args) * sdt.itemsize].view(sdt)
    dev = pipeline._find_blocks(dict(enumerate(dimgs)), [(i, pipeline.TextPage(r, "vertical" if v else "horizontal", p, skew=s), rect)
                                                         for (i, r, v, p, s), rect in zip(items, rects)])
    seen = set()
    for k, ((i, _, v, p, s), rect, got) in enumerate(zip(items, rects, dev)):
        ref = _twin(imgs[i], rect, v, p, s)
        assert not isinstance(got, str), (k, got)
        det = ref.pop("detail")
        if det is not None:
            assert int(sk[k]["chosen"]) == det["chosen"], (k, int(sk[k]["chosen"]), det["chosen"])
            if det["scores"] is not None:
                assert scores[k].cpu().tolist() == det["scores"], k
            else:
                assert scores[k] is None
            if det["frame"] is not None:
                seen.add("tilted-vertical" if v else "tilted")
                u_min, v_min, L, M = det["frame"]
                # the device's search frame; a vertical page's bitmap is that frame with its axes swapped
                assert (int(sk[k]["M"]), int(sk[k]["L"])) == ((L, M) if v else (M, L)), k
        want_blocks = ref["blocks"]
        if det is not None and det["frame"] is not None:
            assert [b.window for b in got["blocks"]] == want_blocks, (k, rect)
            assert all(b.rect == rect and b.skew == ref["skew"] for b in got["blocks"])
        else:
            assert [tuple(b.rect) for b in got["blocks"]] == want_blocks, (k, rect)
            assert all(b.window is None and b.skew is None for b in got["blocks"])
        for key in ("rejected", "threshold", "ink", "text_size", "gap_x", "gap_y"):
            assert got[key] == ref[key], (k, key, got[key], ref[key])
        if s is None:
            assert "skew" not in got
        else:
            assert got["skew"] == ref["skew"], (k, got["skew"], ref["skew"])
        seen.add(str(s if not isinstance(s, float) or s == 0 else "given"))
        if rect[2] - rect[0] == 1:
            seen.add("1x1")
    assert {"tilted", "tilted-vertical", "None", "auto", "given", "0.0", "1x1"} <= seen, seen


def test_windowed_find_lines_equals_twin():
    """Windowed blocks beside plain and skewed blocks in one call: every window's lines, threshold and ink are the twin's, and
    the windowed part takes four launches whatever its number of blocks."""
    from marconet_b200 import ops, pipeline
    imgs, blocks, refs = [], [], []
    for k, (angle, vertical) in enumerate(((-6.0, False), (3.5, True), (8.0, False), (0.0, False))):
        img, _ = drawn_page((240, 220), 5, angle, seed=20 + k, vertical=vertical)
        d = "vertical" if vertical else "horizontal"
        H, W = img.shape[:2]
        r = SP.find_blocks(img, direction=d, skew=angle if angle else "auto")
        wins = r["blocks"] if r["detail"]["frame"] is not None else [(b[1], b[0], b[3], b[2]) if vertical else b
                                                                      for b in r["blocks"]]
        imgs.append(img)
        for win in wins + [(0, 0, 1, 1)]:
            blocks.append((k, pipeline.TextBlock((0, 0, W, H), d, skew=r["skew"], window=win)))
            refs.append(SP.find_lines(img, (0, 0, W, H), win, r["skew"], d))
        blocks.append((k, pipeline.TextBlock((0, 0, W // 2, H // 2), d)))
        refs.append(None)
        blocks.append((k, pipeline.TextBlock((0, 0, W, H), d, skew="auto")))
        refs.append(None)
    per = [[b for i, b in blocks if i == k] for k in range(len(imgs))]
    got = [r for g in pipeline.find_lines(imgs, per) for r in g]
    for (k, blk), ref, g in zip(blocks, refs, got):
        if ref is None:
            continue
        lines = [q.shape if isinstance(q, pipeline.VerticalRegion) else q for q in g["lines"]]
        want = ref["lines"]
        if blk.skew != 0:
            assert [(tuple(q.tl), tuple(q.tr), tuple(q.bl)) for q in lines] == [tuple(map(tuple, q)) for q in want], blk
        else:
            assert [tuple(q) for q in lines] == [tuple(q) for q in want], blk
        assert (g["threshold"], g["ink"], g["skew"]) == (ref["threshold"], ref["ink"], ref["skew"]), blk
    dimg = torch.from_numpy(imgs[0]).to(DEV)
    wins = [b for i, b in blocks if i == 0 and b.window is not None]
    args = [(dimg, b.rect, False, 0, None, None, None, b.skew, b.window) for b in wins]
    n0 = ops.LAUNCHES
    ops.find_lines_window(args[:1])
    assert ops.LAUNCHES - n0 == 4
    n0 = ops.LAUNCHES
    ops.find_lines_window(args)
    assert ops.LAUNCHES - n0 == 4


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
def test_restore_regions_tilted_page_equals_the_found_blocks(gpu_models, to_host):
    """A tilted page under "auto" gives the bytes of the call given its blocks and of the call given their lines; a level page
    under "auto" gives the bytes of skew=None."""
    from marconet_b200 import pipeline
    m = _models(gpu_models)
    img, _ = drawn_page((220, 220), 3, -4.0, seed=5)
    pg = pipeline.TextPage(skew="auto")
    found = pipeline.find_blocks([img], [[pg]])[0][0]
    assert len(found["blocks"]) == 3 and all(b.window is not None for b in found["blocks"])
    lines = pipeline.find_lines([img], [found["blocks"]])[0]
    kw = dict(scale=2, feather=3, to_host=to_host)
    a = pipeline.restore_regions(*m, [img], [[pg]], **kw)[0]
    b = pipeline.restore_regions(*m, [img], [found["blocks"]], **kw)[0]
    c = pipeline.restore_regions(*m, [img], [[q for r in lines for q in r["lines"]]], **kw)[0]
    _same(a["image"], b["image"])
    _same(a["image"], c["image"])
    assert {k: v for k, v in a["regions"][0].items() if k != "regions"} == found
    _same(a["regions"][0]["regions"], b["regions"])
    level, _ = drawn_page((220, 220), 3, 0.0, seed=6)
    d = pipeline.restore_regions(*m, [level], [[pipeline.TextPage(skew="auto")]], **kw)[0]
    e = pipeline.restore_regions(*m, [level], [[pipeline.TextPage()]], **kw)[0]
    _same(d["image"], e["image"])
    assert d["regions"][0].pop("skew") == 0.0
    _same(d["regions"], e["regions"])


def test_failing_tilted_page_under_skip_invalid(gpu_models):
    """A tilted page one of whose blocks has too many lines raises, or is one dict(error=...) under skip_invalid that restores
    none of its blocks."""
    from marconet_b200 import pipeline
    m = _models(gpu_models)
    img = np.full((2000, 400, 3), 240, np.uint8)
    img[100:1900, 100:300][np.arange(1800) % 6 < 2] = 10          # 300 stripes that gap_y keeps in one block
    R = __import__("cv2").getRotationMatrix2D((200, 1000), 3.0, 1.0)
    img = __import__("cv2").warpAffine(img, R, (400, 2000), flags=0, borderValue=(240, 240, 240))
    regs = [pipeline.TextPage(gap_y=1000, skew=3.0), (0, 0, 200, 40)]
    with pytest.raises(ValueError, match="image 0, region 0 \\(a text page\\), block 0: .* lines exceed"):
        pipeline.restore_regions(*m, [img], [regs])
    a = pipeline.restore_regions(*m, [img], [regs], skip_invalid=True, to_host=True)[0]
    assert set(a["regions"][0]) == {"error"} and "lines exceed" in a["regions"][0]["error"]
    b = pipeline.restore_regions(*m, [img], [regs[1:]], skip_invalid=True, to_host=True)[0]
    _same(a["image"], b["image"])
    _same(a["regions"][1], b["regions"][0])
