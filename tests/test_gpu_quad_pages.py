"""Perspective pages and blocks on the device (DESIGN.md section 7b, "Perspective pages"): mn_find_page_quads_u8's threshold,
component, hull and quad bit for bit against the numpy twin, the rectified crops and the block and line tables of quad pages and
blocks against the twin in calls mixed with level and skewed items, the launch counts, and pipeline.restore_regions with quad
pages and blocks against the same call given the found blocks and given the found lines."""
import numpy as np
import pytest
import torch

from oracle import blocks as B
from oracle import pages as P
from oracle import quad_pages as Q
from oracle.quad_regions import rectify

from test_gpu_skewed_pages import _models, _same
from test_quad_pages import corners_of, photo
from test_skewed_pages import drawn_page

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda:0")


def _photo(k, pull, widths=(180, 200), n_lines=4, vertical=False, light=False):
    flat, _ = drawn_page(widths, n_lines, 0.0, k, vertical=vertical)
    h, w = flat.shape[:2]
    corners = corners_of(w, h, 60 + 7 * k, 50 + 3 * k, pull)
    return photo(widths, n_lines, corners, seed=k, vertical=vertical, light=light)[0]


def _images(rng):
    """33 images: photographed pages (both directions, noisy, light on dark), a page filling the frame, two paper regions of
    equal size, images without a page, random masks, a 1 x 1 image and uniform images; and each one's polarity."""
    out = []
    pulls = [(0, 0, 0, 0), (40, 0, 0, 0), (0, 50, 0, 0), (0, 0, 30, 0), (0, 0, 0, 45), (25, 0, 20, 0), (0, 35, 0, 25),
             (60, 0, 0, 0)]
    for k, pull in enumerate(pulls):
        out.append((_photo(k, pull, vertical=k in (2, 5)), "auto"))
    noisy = _photo(8, (30, 0, 0, 10)).astype(np.int32)
    out.append((np.clip(noisy + rng.integers(-15, 16, noisy.shape[:2] + (1,)), 0, 255).astype(np.uint8), "auto"))
    out.append((_photo(9, (20, 0, 0, 30), light=True), "light"))
    full, _ = drawn_page((200,), 4, 0.0, 10)
    out.append((full, "auto"))                          # fills the frame
    two = np.full((120, 200, 3), 60, np.uint8)
    two[10:110, 10:90] = 220
    two[10:110, 110:190] = 220                          # equal sizes: the first in raster order wins
    out.append((two, "auto"))
    out.append((np.zeros((50, 70, 3), np.uint8), "auto"))                  # no paper
    small = np.full((100, 120, 3), 40, np.uint8)
    small[10:30, 10:40] = 230                                               # a page under a quarter of the image
    out.append((small, "auto"))
    out.append((np.full((1, 1, 3), 200, np.uint8), "auto"))
    out.append((np.full((37, 45, 3), 128, np.uint8), "auto"))
    out.append((np.full((37, 45, 3), 128, np.uint8), "light"))
    for k in range(16):
        h, w = (int(v) for v in rng.integers(1, 90, 2))
        m = rng.random((h, w)) < rng.uniform(0.2, 0.9)
        img = np.where(m[..., None], 200, 30).astype(np.uint8) + rng.integers(0, 20, (h, w, 3)).astype(np.uint8)
        out.append((img, ("auto", "dark", "light")[k % 3]))
    return out


def _device_quads(images):
    from marconet_b200 import ops, pipeline
    dimg = [torch.from_numpy(img).to(DEV) for img, _ in images]
    n0 = ops.LAUNCHES
    res, hulls = ops.find_page_quads([(d, pipeline._INK[p]) for d, (_, p) in zip(dimg, images)], hulls=True)
    assert ops.LAUNCHES - n0 == 8
    return res.cpu().numpy().view(ops.page_quad_dtype()), [h.cpu().numpy() for h in hulls]


def test_corner_search_equals_twin():
    images = _images(np.random.default_rng(0))
    assert len(images) >= 30
    res, hulls = _device_quads(images)
    for k, ((img, pol), r, hull) in enumerate(zip(images, res, hulls)):
        want = Q.find_corners(img, pol)
        assert int(r["threshold"]) == want["threshold"], k
        assert (int(r["label"]), int(r["size"])) == (want["label"], want["size"]), k
        assert int(r["n_hull"]) == len(want["hull"]), k
        assert [tuple(p) for p in hull[:len(want["hull"])].tolist()] == [tuple(p) for p in want["hull"]], k
        if want["quad"] is None:
            continue
        assert int(r["area2"]) == want["area2"], k
        assert tuple(r["idx"].tolist()) == want["idx"], k
        assert [tuple(r["quad"][2 * m:2 * m + 2].tolist()) for m in range(4)] == [tuple(p) for p in want["quad"]], k


def test_quad_page_and_block_tables_equal_twin():
    from marconet_b200 import ops, pipeline
    imgs = [_photo(k, pull, vertical=k == 1) for k, pull in enumerate([(30, 0, 0, 0), (0, 0, 0, 40), (0, 45, 20, 0)])]
    level, _ = drawn_page((200, 180), 4, 0.0, 4)
    tilted, _ = drawn_page((200, 180), 4, 3.0, 5)
    imgs += [level, tilted]
    H, W = imgs[2].shape[:2]
    given = pipeline.QuadRegion((40.5, 30.0), (W - 35.0, 52.0), (W - 60.0, H - 41.5), (55.0, H - 30.0))
    pages = [[pipeline.TextPage(quad="auto")], [pipeline.TextPage(direction="vertical", quad="auto")],
             [pipeline.TextPage(quad="auto"), pipeline.TextPage(quad=given)], [pipeline.TextPage()],
             [pipeline.TextPage(skew="auto")]]
    n0 = ops.LAUNCHES
    got = pipeline.find_blocks(imgs, pages)
    assert ops.LAUNCHES - n0 == 8 + 1 + 7 + 6 * ops._lib.PAGE_LEVELS          # search, one warp, the skewed call
    for i in range(3):
        for pg, r in zip(pages[i], got[i]):
            quad = pg.quad if pg.quad != "auto" else Q.accepted(Q.find_corners(imgs[i], pg.polarity), imgs[i].shape)
            want = Q.find_blocks(imgs[i], quad, pg.direction, pg.polarity)
            assert r["quad"] == tuple((float(x), float(y)) for x, y in quad)
            assert r["size"] == want["size"]
            assert [b.window for b in r["blocks"]] == [tuple(b) for b in want["blocks"]]
            assert r["rejected"] == [tuple(b) for b in want["rejected"]]
            assert all(b.quad == r["quad"] and b.direction == pg.direction for b in r["blocks"])
            assert {k: r[k] for k in ("threshold", "ink", "text_size", "gap_x", "gap_y")} == \
                {k: want[k] for k in ("threshold", "ink", "text_size", "gap_x", "gap_y")}
    assert got[3][0]["blocks"] == [pipeline.TextBlock(b) for b in P.find_blocks(level)["blocks"]]
    # the rectified crops: one launch over the distinct quads, the bytes of ops.warp_perspective and of the twin
    dimg = {i: torch.from_numpy(im).to(DEV) for i, im in enumerate(imgs)}
    keys = [pipeline._quad_key(2, given), pipeline._quad_key(2, given), pipeline._quad_key(0, got[0][0]["quad"])]
    n0 = ops.LAUNCHES
    rq = pipeline._rectify(dimg, keys)
    assert ops.LAUNCHES - n0 == 1 and len(rq) == 2
    np.testing.assert_array_equal(rq[keys[0]].cpu().numpy(), rectify(imgs[2], given))
    np.testing.assert_array_equal(rq[keys[2]].cpu().numpy(), rectify(imgs[0], got[0][0]["quad"]))
    # quad blocks' lines, mixed with level and skewed blocks in one call
    blocks = [got[0][0]["blocks"], got[1][0]["blocks"], got[2][1]["blocks"] + [pipeline.TextBlock.from_quad(given, (H, W))],
              [pipeline.TextBlock(b) for b in P.find_blocks(level)["blocks"]], [pipeline.TextBlock((0, 0) + tilted.shape[1::-1],
                                                                                                    skew="auto")]]
    n0 = ops.LAUNCHES
    lines = pipeline.find_lines(imgs, blocks)
    assert ops.LAUNCHES - n0 == 1 + 6
    for i in range(3):
        for blk, r in zip(blocks[i], lines[i]):
            want = Q.find_lines(imgs[i], blk.quad, blk.window, blk.direction, polarity=blk.polarity)
            shapes = [q.shape if isinstance(q, pipeline.VerticalRegion) else q for q in r["lines"]]
            assert all(isinstance(q, pipeline.QuadRegion) for q in shapes)
            assert [tuple(q) for q in shapes] == want["lines"]
            assert all(isinstance(q, pipeline.VerticalRegion) == (blk.direction == "vertical") for q in r["lines"])
            assert (r["threshold"], r["ink"]) == (want["threshold"], want["ink"])
    for blk, r in zip(blocks[3], lines[3]):
        assert r["lines"] == B.find_lines(level, blk.rect)["lines"]


def test_calls_without_quads_keep_their_launches():
    from marconet_b200 import ops, pipeline
    img, _ = drawn_page((200, 180), 4, 0.0, 4)
    n0 = ops.LAUNCHES
    pipeline.find_blocks([img], [[pipeline.TextPage()]])
    assert ops.LAUNCHES - n0 == 5 + 6 * ops._lib.PAGE_LEVELS
    n0 = ops.LAUNCHES
    pipeline.find_lines([img], [[pipeline.TextBlock((0, 0, 100, 100))]])
    assert ops.LAUNCHES - n0 == 4


@pytest.mark.parametrize("to_host", [False, True])
def test_restore_regions_quad_pages_equal_the_found_blocks_and_lines(gpu_models, to_host):
    from marconet_b200 import pipeline
    m = _models(gpu_models)
    img = _photo(3, (25, 0, 0, 20), widths=(160, 170), n_lines=3)
    H, W = img.shape[:2]
    given = pipeline.QuadRegion((45.0, 40.5), (W - 30.0, 35.0), (W - 40.0, H - 30.0), (50.0, H - 45.0))
    kw = dict(scale=2, feather=3, to_host=to_host)
    for pg in (pipeline.TextPage(quad="auto"), pipeline.TextPage(quad=given)):
        found = pipeline.find_blocks([img], [[pg]])[0][0]
        assert found["blocks"] and all(b.quad is not None for b in found["blocks"])
        lines = pipeline.find_lines([img], [found["blocks"]])[0]
        a = pipeline.restore_regions(*m, [img], [[pg]], **kw)[0]
        b = pipeline.restore_regions(*m, [img], [found["blocks"]], **kw)[0]
        c = pipeline.restore_regions(*m, [img], [[q for r in lines for q in r["lines"]]], **kw)[0]
        _same(a["image"], b["image"])
        _same(a["image"], c["image"])
        assert {k: v for k, v in a["regions"][0].items() if k != "regions"} == found
        _same(a["regions"][0]["regions"], b["regions"])


def test_restore_regions_quad_block_equals_its_lines(gpu_models):
    from marconet_b200 import pipeline
    m = _models(gpu_models)
    img = _photo(6, (0, 30, 0, 0), widths=(160, 170), n_lines=3)
    H, W = img.shape[:2]
    quad = Q.accepted(Q.find_corners(img), img.shape)
    regs = [(2, 2, 40, 20), pipeline.TextBlock.from_quad(quad, (H, W))]
    found = pipeline.find_lines([img], [[regs[1]]])[0][0]
    assert found["lines"]
    a = pipeline.restore_regions(*m, [img], [regs], scale=2, to_host=True)[0]
    b = pipeline.restore_regions(*m, [img], [[regs[0]] + found["lines"]], scale=2, to_host=True)[0]
    _same(a["image"], b["image"])
    assert a["regions"][1]["lines"] == found["lines"]


def test_skip_invalid_for_quad_pages(gpu_models):
    """A page with no quad, or one whose block fails, raises, or is one dict(error=...) under skip_invalid that restores none of
    its blocks."""
    from marconet_b200 import pipeline
    m = _models(gpu_models)
    dark = np.full((80, 100, 3), 30, np.uint8)
    dark[30:40, 20:80] = 200                            # paper, but far under a quarter of the image
    regs = [pipeline.TextPage(quad="auto"), (0, 0, 60, 30)]
    with pytest.raises(ValueError, match=r"image 0, region 0 \(a text page\): no page found"):
        pipeline.restore_regions(*m, [dark], [regs])
    with pytest.raises(ValueError, match=r"image 0, page 0: no page found"):
        pipeline.find_blocks([dark], [[regs[0]]])
    a = pipeline.restore_regions(*m, [dark], [regs], skip_invalid=True, to_host=True)[0]
    assert set(a["regions"][0]) == {"error"} and "no page found" in a["regions"][0]["error"]
    b = pipeline.restore_regions(*m, [dark], [regs[1:]], skip_invalid=True, to_host=True)[0]
    _same(a["image"], b["image"])
    _same(a["regions"][1], b["regions"][0])
    # a page whose block has too many lines
    img = np.full((2000, 400, 3), 240, np.uint8)
    img[100:1900, 100:300][np.arange(1800) % 6 < 2] = 10          # 300 stripes that gap_y keeps in one block
    q = pipeline.QuadRegion((0.0, 0.0), (400.0, 0.0), (400.0, 2000.0), (0.0, 2000.0))
    regs = [pipeline.TextPage(gap_y=1000, quad=q), (0, 0, 200, 40)]
    with pytest.raises(ValueError, match=r"image 0, region 0 \(a text page\), block 0: .* lines exceed"):
        pipeline.restore_regions(*m, [img], [regs])
    a = pipeline.restore_regions(*m, [img], [regs], skip_invalid=True, to_host=True)[0]
    assert set(a["regions"][0]) == {"error"} and "lines exceed" in a["regions"][0]["error"]
    b = pipeline.restore_regions(*m, [img], [regs[1:]], skip_invalid=True, to_host=True)[0]
    _same(a["image"], b["image"])
    _same(a["regions"][1], b["regions"][0])
