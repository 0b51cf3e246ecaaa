"""Skewed text blocks on the device (DESIGN.md section 7b, "Skewed blocks"): mn_find_lines_skewed_u8's scores, chosen angles
and line tables bit for bit against the numpy twin, skew=None blocks bit for bit against mn_find_lines_u8, its constant launch
count, and pipeline.restore_regions with skewed blocks against the same call given the found lines."""
import cv2
import numpy as np
import pytest
import torch

from oracle import skewed_blocks as S

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda:0")
TEXTS = ["The quick brown fox jumps over dogs", "Sphinx of black quartz, judge my vow", "Pack my box with five dozen jugs",
         "How vexingly quick daft zebras jump"]


def _models(gpu_models):
    return gpu_models["encoder"], gpu_models["tspgan"], gpu_models["sr"]


def _page(rng, n_lines, angle, light=False, noise=0, margin=100, w=560):
    """n_lines putText lines 36 pixels apart rotated by ``angle`` degrees counter-clockwise on a plain background."""
    h, W = 30 + 36 * n_lines + 2 * margin, w + 2 * margin
    bg = rng.integers(195, 256, 3)
    page = np.empty((h, W, 3), np.uint8)
    page[:] = bg
    for k in range(n_lines):
        cv2.putText(page, TEXTS[k % len(TEXTS)], (margin + 8, margin + 36 + 36 * k), cv2.FONT_HERSHEY_SIMPLEX, 0.7,
                    tuple(int(v) for v in rng.integers(0, 60, 3)), 2, cv2.LINE_AA)
    rot = cv2.getRotationMatrix2D((W / 2, h / 2), angle, 1.0)
    page = cv2.warpAffine(page, rot, (W, h), flags=cv2.INTER_LINEAR, borderValue=tuple(int(v) for v in bg))
    if noise:
        page = np.clip(page.astype(np.int32) + rng.integers(-noise, noise + 1, page.shape), 0, 255).astype(np.uint8)
    return 255 - page if light else page


def _random_blocks(rng):
    """About 50 blocks: whole rotated pages and crops through their pitch at random angles, given and searched skew, both
    polarities, vertical blocks on transposed pages, 1 x 1, uniform and random blocks, a tall and a wide thin block, and blocks
    with skew None among them."""
    pages = [_page(rng, 5, 3.3), _page(rng, 3, -7.1, light=True), _page(rng, 8, 1.2, noise=25), _page(rng, 2, 12.6),
             rng.integers(0, 256, (90, 70, 3), dtype=np.uint8), np.full((40, 50, 3), 131, np.uint8)]
    pages.append(np.ascontiguousarray(_page(rng, 4, -4.4).transpose(1, 0, 2)))
    tall = np.full((32767, 9, 3), 240, np.uint8)
    tall[(np.arange(32767) // 7) % 40 == 0, 2:7] = 10
    pages.append(tall)
    wide = np.full((12, 8000, 3), 250, np.uint8)
    wide[3:8, (np.arange(8000) // 5) % 3 == 0] = 5
    pages.append(wide)
    fixed = [(0, "auto", 10.0), (1, "auto", 15.0), (2, "auto", 10.0), (3, "auto", 20.0), (6, "auto", 10.0), (7, "auto", 10.0),
             (8, "auto", 3.0), (5, "auto", 10.0), (0, None, 10.0), (6, None, 10.0), (2, 1.2, 10.0), (4, "auto", 10.0)]
    items = []
    for k in range(52):
        if k < len(fixed):
            i, skew, ms = fixed[k]
        else:
            i = int(rng.integers(0, 7))
            u = rng.random()
            skew, ms = ("auto", float(rng.choice([2.5, 10.0, 14.0, 20.0]))) if u < 0.5 else \
                (None, 10.0) if u < 0.65 else (float(rng.uniform(-44, 44)) if u < 0.75 else float(rng.uniform(-15, 15)), 10.0)
        H, W = pages[i].shape[:2]
        if k < len(fixed) or rng.random() < 0.3:
            rect = (0, 0, W, H)
        elif rng.random() < 0.1:
            x, y = int(rng.integers(0, W)), int(rng.integers(0, H))
            rect = (x, y, x + 1, y + 1)
        else:
            x0, y0 = int(rng.integers(0, W - 1)), int(rng.integers(0, H - 1))
            rect = (x0, y0, int(rng.integers(x0 + 1, W + 1)), int(rng.integers(y0 + 1, H + 1)))
        vertical = i == 6 or (k >= len(fixed) and rng.random() < 0.2)
        polarity = ["auto", "auto", "dark", "light"][int(rng.integers(0, 4))] if k >= len(fixed) else "auto"
        knobs = [int(rng.integers(1, 6)) if rng.random() < 0.15 else None for _ in range(3)] if k >= len(fixed) else [None] * 3
        items.append((i, rect, vertical, polarity, knobs, skew, ms))
    items.append((0, (10, 10, 11, 11), False, "auto", [None] * 3, "auto", 10.0))
    return pages, items


def _args(dpages, items):
    from marconet_b200 import _lib
    pol = dict(auto=_lib.INK_AUTO, dark=_lib.INK_DARK, light=_lib.INK_LIGHT)
    return [(dpages[i], rect, v, pol[p], *knobs, skew, ms) for i, rect, v, p, knobs, skew, ms in items]


def test_skewed_tables_equal_twin():
    """Every score, chosen index, chosen frame and line table equals the twin's; skew=None blocks keep mn_find_lines_u8's
    records byte for byte; six launches for 52 blocks as for one."""
    from marconet_b200 import _lib, ops
    rng = np.random.default_rng(0)
    pages, items = _random_blocks(rng)
    dpages = [torch.from_numpy(p).to(DEV) for p in pages]
    args = _args(dpages, items)
    n = len(args)
    n0 = ops.LAUNCHES
    ops.find_lines(args[:1])
    assert ops.LAUNCHES - n0 == 6
    n0 = ops.LAUNCHES
    buf, scores = ops.find_lines(args, scores=True)
    assert ops.LAUNCHES - n0 == 6
    host = buf.cpu().numpy()
    osz = ops.block_lines_dtype().itemsize
    rec, sk = host[:n * osz].view(ops.block_lines_dtype()), host[n * osz:].view(ops.skew_block_dtype())
    plain = [k for k, it in enumerate(items) if it[5] is None]
    n0 = ops.LAUNCHES
    ref_plain = ops.find_lines([a[:7] for k, a in enumerate(args) if k in plain]).cpu().numpy().view(ops.block_lines_dtype())
    assert ops.LAUNCHES - n0 == 4
    for j, k in enumerate(plain):                       # every written word; rows past n_lines and the pad are never written
        a, b = rec[k], ref_plain[j]
        nl = int(a["n_lines"])
        assert (nl, int(a["threshold"]), int(a["ink"])) == (int(b["n_lines"]), int(b["threshold"]), int(b["ink"])), k
        assert bytes(a["rect"][:max(nl, 0)]) == bytes(b["rect"][:max(nl, 0)]), k
    seen = set()
    for k, ((i, rect, v, p, knobs, skew, ms), r, s) in enumerate(zip(items, rec, sk)):
        if skew is None:
            continue
        try:
            ref = S.find_lines(pages[i], rect, "vertical" if v else "horizontal", *knobs, polarity=p, skew=skew, max_skew=ms)
        except ValueError as e:
            assert int(r["n_lines"]) < 0 and f"{-int(r['n_lines'])} lines exceed" in str(e), k
            seen.add("over")
            continue
        d = ref["detail"]
        assert int(r["threshold"]) == ref["threshold"], k
        assert ("dark" if r["ink"] == _lib.INK_DARK else "light") == ref["ink"], k
        assert int(s["n_ang"]) == len(d["i"]) and int(s["chosen"]) == d["chosen"], (k, int(s["chosen"]), d["chosen"])
        assert (float(s["u_min"]), float(s["v_min"]), int(s["L"]), int(s["M"])) == d["frame"], k
        assert (float(s["c"]), float(s["s"])) == (float(d["c"][d["chosen"]]), float(d["s"][d["chosen"]])), k
        if d["scores"] is None:
            assert scores[k] is None
        else:
            assert scores[k].cpu().tolist() == d["scores"], k
            seen.add("search")
        nl = int(r["n_lines"])
        got = [tuple(int(x) for x in q) for q in r["rect"][:nl]]
        if s["s"] == 0:
            assert got == ref["lines"], k
            seen.add("level")
        else:
            assert got == d["frame_lines"], k
            seen.add("vertical" if v else "skewed")
        seen.add("lines" if nl > 1 else "none" if nl == 0 else "one")
        if rect[2] - rect[0] == 1 and rect[3] - rect[1] == 1:
            seen.add("1x1")
        if max(rect[2] - rect[0], rect[3] - rect[1]) >= 8000:
            seen.add("thin")
    assert {"search", "level", "vertical", "skewed", "lines", "none", "one", "1x1", "thin"} <= seen, seen


def test_find_lines_skewed_matches_twin():
    """pipeline.find_lines: OrientedRegions, VerticalRegions of OrientedRegions and the skew key equal the twin's; skew=None
    blocks of the same call return exactly what a call without skewed blocks returns."""
    from marconet_b200 import pipeline
    rng = np.random.default_rng(1)
    page = _page(rng, 6, -3.85)
    col = np.ascontiguousarray(_page(rng, 3, 5.2).transpose(1, 0, 2))
    H, W = page.shape[:2]
    blocks = [[pipeline.TextBlock((0, 0, W, H), skew="auto"), pipeline.TextBlock((0, 0, W, H)),
               pipeline.TextBlock((5, 5, W - 5, H - 5), skew=-3.85)],
              [pipeline.TextBlock((0, 0, col.shape[1], col.shape[0]), "vertical", skew="auto", max_skew=12)]]
    out = pipeline.find_lines([page, torch.from_numpy(col).to(DEV)], blocks)
    ref = S.find_lines(page, (0, 0, W, H), skew="auto")
    assert out[0][0]["skew"] == ref["skew"] and abs(ref["skew"] + 3.85) <= 0.2 and len(out[0][0]["lines"]) == 6
    assert [tuple(q) for q in out[0][0]["lines"]] == [tuple(q) for q in ref["lines"]]
    assert all(isinstance(q, pipeline.OrientedRegion) for q in out[0][0]["lines"])
    assert out[0][1] == pipeline.find_lines([page], [[blocks[0][1]]])[0][0] and "skew" not in out[0][1]
    ref2 = S.find_lines(page, (5, 5, W - 5, H - 5), skew=-3.85)
    assert out[0][2]["skew"] == -3.85 and [tuple(q) for q in out[0][2]["lines"]] == [tuple(q) for q in ref2["lines"]]
    refv = S.find_lines(col, (0, 0, col.shape[1], col.shape[0]), "vertical", skew="auto", max_skew=12)
    assert out[1][0]["skew"] == refv["skew"] and abs(refv["skew"] + 5.2) <= 0.2 and len(refv["lines"]) == 3
    assert [tuple(q.shape) for q in out[1][0]["lines"]] == [tuple(q) for q in refv["lines"]]
    assert all(isinstance(q, pipeline.VerticalRegion) and isinstance(q.shape, pipeline.OrientedRegion) for q in out[1][0]["lines"])
    for key in ("threshold", "ink"):
        assert out[0][0][key] == ref[key] and out[1][0][key] == refv[key]


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
def test_restore_regions_skewed_blocks_equal_the_found_lines(gpu_models, to_host):
    """A call with "auto" blocks gives the bytes of the call given their lines, beside rectangles, oriented, perspective, curved
    and vertical regions and a level block."""
    from marconet_b200 import pipeline
    m = _models(gpu_models)
    rng = np.random.default_rng(2)
    img = np.full((420, 520, 3), 236, np.uint8)
    img[0:162, 0:330] = _page(rng, 2, 4.5, margin=30, w=270)
    img[180:400, 330:482] = np.ascontiguousarray(_page(rng, 2, -3.0, margin=25, w=170).transpose(1, 0, 2))
    img[300:406, 0:250] = _page(rng, 1, 0.0, margin=20, w=210)
    hb = pipeline.TextBlock((0, 0, 330, 162), skew="auto")
    vb = pipeline.TextBlock((330, 180, 482, 400), "vertical", skew="auto")
    lb = pipeline.TextBlock((0, 300, 250, 406), skew="auto")
    others = [(200, 200, 300, 240), pipeline.OrientedRegion.from_rotated(150, 250, 120, 30, 8),
              pipeline.QuadRegion((40, 180), (160, 176), (164, 220), (38, 222)),
              pipeline.CurvedRegion.from_arc(150, 260, 60, 85, 220, 320), pipeline.VerticalRegion((300, 200, 325, 290))]
    found = pipeline.find_lines([img], [[hb, vb, lb]])[0]
    assert len(found[0]["lines"]) == 2 and len(found[1]["lines"]) == 2 and len(found[2]["lines"]) == 1, found
    assert found[0]["skew"] != 0 and found[1]["skew"] != 0
    regs = [others[0], hb, others[1], vb, others[2], lb, others[3], others[4]]
    flat = [others[0], *found[0]["lines"], others[1], *found[1]["lines"], others[2], *found[2]["lines"], others[3], others[4]]
    kw = dict(scale=2, feather=3, skip_invalid=True, to_host=to_host)
    a = pipeline.restore_regions(*m, [img], [regs], **kw)[0]
    b = pipeline.restore_regions(*m, [img], [flat], **kw)[0]
    _same(a["image"], b["image"])
    e = a["regions"]
    assert len(e) == len(regs)
    for k, blk in ((1, 0), (3, 1), (5, 2)):
        assert {x: e[k][x] for x in ("lines", "threshold", "ink", "skew")} == found[blk]
    _same(e[0], b["regions"][0])
    _same(e[1]["regions"], b["regions"][1:3])
    _same(e[2], b["regions"][3])
    _same(e[3]["regions"], b["regions"][4:6])
    _same(e[4], b["regions"][6])
    n3 = len(found[2]["lines"])
    _same(e[5]["regions"], b["regions"][7:7 + n3])
    _same(e[6:], b["regions"][7 + n3:])


def test_level_page_under_auto_gives_the_bytes_of_skew_none(gpu_models):
    from marconet_b200 import pipeline
    m = _models(gpu_models)
    rng = np.random.default_rng(3)
    page = _page(rng, 3, 0.0, margin=10, w=300)
    H, W = page.shape[:2]
    auto = pipeline.restore_regions(*m, [page], [[pipeline.TextBlock((0, 0, W, H), skew="auto")]], scale=2, to_host=True)[0]
    none = pipeline.restore_regions(*m, [page], [[pipeline.TextBlock((0, 0, W, H))]], scale=2, to_host=True)[0]
    _same(auto["image"], none["image"])
    assert auto["regions"][0]["skew"] == 0.0 and auto["regions"][0]["lines"] == none["regions"][0]["lines"]
    assert len(none["regions"][0]["lines"]) == 3
    _same(auto["regions"][0]["regions"], none["regions"][0]["regions"])
