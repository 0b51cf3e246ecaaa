"""Flat pages (DESIGN.md section 7b, "Flat pages") on the GPU: pipeline.flatten_pages bit for bit against the numpy twin in one
call mixing every frame, curl, polarity and edge size; the column table and the remap at the column cap; the launch counts;
and restore_regions on a flattened open book."""
import numpy as np
import pytest
import torch

from oracle import flat_pages as F
from oracle.remap import remap_cubic_u8

from test_curled_blocks import PITCH, curled_page
from test_flat_pages import level_after, mid_spread, open_book

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda:0")


def _same_result(got, want):
    np.testing.assert_array_equal(got["image"], want["image"])
    assert got["kind"] == want["kind"] and tuple(got["size"]) == tuple(want["size"])
    for key in ("skew", "quad", "lines"):
        assert (key in got) == (key in want), key
        if key in got:
            assert got[key] == want[key], key


def test_flatten_pages_equals_the_twin_in_one_mixed_call():
    from marconet_b200 import ops
    from marconet_b200.pipeline import FlatPage, QuadRegion, flatten_pages
    curled, _, _ = curled_page(8, "cylinder", 2 * PITCH, 11)
    light, _, _ = curled_page(6, "cylinder", -PITCH, 12, light=True)
    tilted, _, _ = curled_page(5, "flat", 0, 13)
    book = open_book("cylinder", PITCH, 14, 1.8)
    spread = np.hstack([curled_page(6, "cylinder", PITCH, 15)[0], curled_page(6, "cylinder", -PITCH, 16)[0]])
    blank = np.full((90, 120, 3), 200, np.uint8)
    wide = np.random.default_rng(0).integers(0, 256, (6, 32767, 3), dtype=np.uint8)
    H, W = curled.shape[:2]
    q = QuadRegion((30.0, 20.0), (W - 40.0, 35.0), (W - 30.0, H - 20.0), (20.0, H - 45.0))
    images = [curled, light, tilted, book, blank, wide, spread]
    pages = [[FlatPage(curve="auto"), FlatPage((3, 4, 4, 5)), FlatPage(quad=q), FlatPage(quad=q, curve="auto", strips=6),
              FlatPage((40, 30, W - 20, H - 10), curve="auto")],
             [FlatPage(curve="auto", polarity="light"), FlatPage((10, 10, 300, 200), skew=-4.5)],
             [FlatPage(skew="auto"), FlatPage((20, 15, 500, 180), skew=3.0), FlatPage(direction="vertical", skew=7.0)],
             [FlatPage(quad="auto", curve="auto"), FlatPage(quad="auto")],
             [FlatPage(curve="auto"), FlatPage(quad=QuadRegion((5.0, 5.0), (100.0, 8.0), (110.0, 80.0), (2.0, 85.0)), curve="auto")],
             [FlatPage(), FlatPage((32766, 0, 32767, 6))],
             [FlatPage(curve="auto")]]
    got = flatten_pages(images, pages, to_host=True)
    dev = flatten_pages([torch.from_numpy(im).to(DEV) for im in images[:2]], pages[:2])
    n_curled, tables = 0, {}
    for i, (im, pl, gl, dl) in enumerate(zip(images, pages, got, dev + [None] * 5)):
        for k, (fp, g) in enumerate(zip(pl, gl)):
            want = F.flatten(im, fp)
            _same_result(g, want)
            n_curled += "table" in want
            if "table" in want:
                tables[(i, k)] = want["table"]
            if dl is not None:
                assert dl[k]["image"].is_cuda
                np.testing.assert_array_equal(dl[k]["image"].cpu().numpy(), want["image"])
    assert n_curled >= 6 and (0, 4) in tables
    assert len({(b0, b1) for b0, b1 in tables[(6, 0)][:, 7:9]}) >= 2       # the spread's two columns leave a gutter
    assert got[5][0]["size"] == (32767, 6) and got[0][1]["size"] == (1, 1)
    assert "lines" in got[4][0] and got[4][0]["lines"] == []
    assert max(mid_spread(q) for q in level_after(got[3][0]["image"])) <= 2.0
    assert ops.LAUNCHES > 0


def test_column_table_and_remap_at_the_column_cap():
    from marconet_b200 import ops
    cap = ops.FLAT_MAX_COLUMN_LINES
    rng = np.random.default_rng(1)
    h, w = 4 * cap + 40, 96
    img = rng.integers(0, 256, (h + 20, w + 30, 3), dtype=np.uint8)
    rows = []
    for k in range(cap):
        y = 20.0 + 4 * k
        mu = (y, y + rng.uniform(-2, 2), y + rng.uniform(-2, 2), y + rng.uniform(-1, 1))
        x0, x1 = (0, 60) if k % 2 == 0 else (10, 90)
        rows.append((float(x0 + 2), float(x1 - 3), *mu, (((mu[0] + mu[1]) + mu[2]) + mu[3]) / 4, float(x0), float(x1)))
    table = np.array(sorted(rows, key=lambda r: r[6]), np.float64)
    assert ops.flat_column_lines(table, w) == cap
    src = torch.from_numpy(img).to(DEV)
    dst = torch.empty(h, w, 3, dtype=torch.uint8, device=DEV)
    n = ops.LAUNCHES
    (cols, fld), = ops.flat_remap([(src, dst, "rect", (7, 5), table)], tables=True)
    assert ops.LAUNCHES == n + 2
    cover, M = F.column_values(table, w)
    cols, fld = cols.cpu().numpy(), fld.cpu().numpy()
    np.testing.assert_array_equal(cols[0], cover.sum(axis=0))
    for x in range(w):
        ks = np.nonzero(cover[:, x])[0]
        np.testing.assert_array_equal(fld[x, :len(ks), 0], table[ks, 6])
        np.testing.assert_array_equal(fld[x, :len(ks), 1], M[ks, x])
    assert cols[1, 95] == 89 and cols[2, 95] == -1
    mx, my = F.maps(table, w, h, "rect", (7, 5))
    np.testing.assert_array_equal(dst.cpu().numpy(), remap_cubic_u8(img, mx, my))
    over = np.concatenate([table, table[:1]])
    with pytest.raises(ValueError, match=f"meets {cap + 1} lines"):
        ops.flat_remap([(src, dst, "rect", (7, 5), over)])
    assert ops.LAUNCHES == n + 2


@pytest.mark.parametrize("kind", ["rect", "quad"])
def test_gutter_and_margins_on_the_device(kind):
    """Two side-by-side blocks of curled lines, (0, 30) and (60, 90) of a 96-column frame: the gutter columns take the two-sided
    lerp of their neighbours 29 and 60, and columns 90 to 95 the one-sided displacement of column 89."""
    from marconet_b200 import ops
    from marconet_b200.pipeline import _quad_homography
    rng = np.random.default_rng(2)
    h, w = 200, 96
    img = rng.integers(0, 256, (h + 40, w + 60, 3), dtype=np.uint8)
    rows = []
    for bx0, bx1, base in ((0, 30, 20.0), (60, 90, 27.0)):
        for k in range(5):
            y = base + 35 * k
            mu = (y, y + rng.uniform(-6, 6), y + rng.uniform(-6, 6), y + rng.uniform(-6, 6))
            rows.append((float(bx0 + 1), float(bx1 - 2), *mu, (((mu[0] + mu[1]) + mu[2]) + mu[3]) / 4, float(bx0), float(bx1)))
    table = np.array(sorted(rows, key=lambda r: r[6]), np.float64)
    if kind == "rect":
        m = (13, 9)
    else:
        (a, b, c), (d, e, f), (g, hh, _) = _quad_homography([(20.0, 10.0), (140.0, 25.0), (130.0, 230.0), (8.0, 215.0)])
        m = (a, b, c, d, e, f, g, hh)
    src = torch.from_numpy(img).to(DEV)
    dst = torch.empty(h, w, 3, dtype=torch.uint8, device=DEV)
    (cols, fld), = ops.flat_remap([(src, dst, kind, m, table)], tables=True)
    cols = cols.cpu().numpy()
    cover, M = F.column_values(table, w)
    np.testing.assert_array_equal(cols[0], cover.sum(axis=0))
    assert (cols[0, 30:60] == 0).all() and (cols[1, 30:60] == 29).all() and (cols[2, 30:60] == 60).all()
    assert (cols[1, 90:] == 89).all() and (cols[2, 90:] == -1).all()
    mx, my = F.maps(table, w, h, kind, m)
    yc = np.arange(h) + 0.5
    src_rows = F.field(table, w, h)
    assert np.abs((src_rows[:, 30:60] - yc[:, None]) - (src_rows[:, 29:30] - yc[:, None])).max() > 0.5   # a real lerp
    np.testing.assert_array_equal(dst.cpu().numpy(), remap_cubic_u8(img, mx, my))


def test_launch_counts():
    from marconet_b200 import _lib, ops, pipeline
    from marconet_b200.pipeline import FlatPage, QuadRegion, TextBlock, TextPage, flatten_pages
    page, _, _ = curled_page(6, "cylinder", PITCH, 21)
    H, W = page.shape[:2]
    q = QuadRegion((10.0, 10.0), (W - 10.0, 12.0), (W - 12.0, H - 10.0), (8.0, H - 12.0))
    n = ops.LAUNCHES
    flatten_pages([page], [[FlatPage()]])
    assert ops.LAUNCHES == n                                     # a crop is a copy
    n = ops.LAUNCHES
    flatten_pages([page], [[FlatPage(skew=2.0), FlatPage((0, 0, 200, 100), skew=-3.0)]])
    assert ops.LAUNCHES == n + 1
    n = ops.LAUNCHES
    flatten_pages([page, page], [[FlatPage(curve="auto"), FlatPage(quad=q, curve="auto"), FlatPage(skew=1.0)], [FlatPage(quad=q)]])
    levels = _lib.PAGE_LEVELS
    assert ops.LAUNCHES == n + 1 + (5 + 6 * levels) + 7 + 1 + 2   # rectify, find_blocks, find_lines_curved, warp, field
    n = ops.LAUNCHES
    pipeline.find_blocks([page], [[TextPage(curve="auto")]])
    assert ops.LAUNCHES == n + 5 + 6 * levels
    n = ops.LAUNCHES
    pipeline.find_lines([page], [[TextBlock((0, 0, W, H), curve="auto")]])
    assert ops.LAUNCHES == n + 7


def test_restore_regions_on_a_flattened_open_book(gpu_models):
    from marconet_b200.pipeline import FlatPage, TextPage, flatten_pages, restore_regions
    m = gpu_models["encoder"], gpu_models["tspgan"], gpu_models["sr"]
    photo = open_book("cylinder", 2 * PITCH, 31, 2.0)
    flat = flatten_pages([photo], [[FlatPage(quad="auto", curve="auto")]])[0][0]
    w_f, h_f = flat["size"]
    out = restore_regions(*m, [flat["image"]], [[TextPage()]], scale=2, to_host=True)[0]
    assert out["image"].shape == (2 * h_f, 2 * w_f, 3)
    page = out["regions"][0]
    assert "error" not in page and page["blocks"]
    assert all("error" not in b and b["lines"] and len(b["regions"]) == len(b["lines"]) for b in page["regions"])
    assert sum(len(b["lines"]) for b in page["regions"]) >= 8
