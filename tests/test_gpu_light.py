"""Even lighting (DESIGN.md section 7b, "Even lighting") on the GPU: flatten_pages(..., FlatPage(light="even")) bit for bit
against the numpy twin in one call mixing every frame, both polarities, given, default and oversized windows and the edge
sizes; light=None pages untouched by the light pages beside them; the launch and synchronisation counts; and a shaded curled
page found, traced and restored after evening."""
import numpy as np
import pytest
import torch

from oracle import light as L

from test_curled_blocks import PITCH, curled_page
from test_flat_pages import open_book
from test_light import shade

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda:0")
KEYS = ("skew", "quad", "lines", "light_window", "ink")


def _same_result(got, want):
    np.testing.assert_array_equal(got["image"], want["image"])
    assert got["kind"] == want["kind"] and tuple(got["size"]) == tuple(want["size"])
    for key in KEYS:
        assert (key in got) == (key in want), key
        if key in got:
            assert got[key] == want[key], key


def _mixed():
    from marconet_b200.pipeline import FlatPage, QuadRegion
    shaded = shade(curled_page(8, "cylinder", PITCH, 11)[0], "gradient")
    lit = shade(curled_page(6, "cylinder", -PITCH, 12, light=True)[0], "vignette")
    tilted = shade(curled_page(5, "flat", 0, 13)[0], "vignette")
    book = shade(open_book("cylinder", PITCH, 11, 1.5), "vignette")
    rng = np.random.default_rng(3)
    tall, wide = rng.integers(0, 256, (32767, 6, 3), dtype=np.uint8), rng.integers(0, 256, (6, 32767, 3), dtype=np.uint8)
    dot = np.full((1, 1, 3), 90, np.uint8)
    H, W = shaded.shape[:2]
    q = QuadRegion((30.0, 20.0), (W - 40.0, 35.0), (W - 30.0, H - 20.0), (20.0, H - 45.0))
    even = dict(light="even")
    images = [shaded, lit, tilted, book, tall, wide, dot]
    pages = [[FlatPage(curve="auto", **even), FlatPage((40, 30, W - 20, H - 10), **even, light_window=9), FlatPage(curve="auto"),
              FlatPage(quad=q, **even), FlatPage(quad=q, curve="auto", **even), FlatPage((3, 4, 23, 19), **even, light_window=101),
              FlatPage((100, 50, 400, 300))],
             [FlatPage(curve="auto", polarity="light", **even), FlatPage((10, 10, 300, 200), skew=-4.5, **even),
              FlatPage(**even, polarity="dark", light_window=15)],
             [FlatPage(skew="auto", **even), FlatPage((20, 15, 500, 180), skew=3.0, **even), FlatPage(skew="auto")],
             [FlatPage(quad="auto", curve="auto", **even), FlatPage(quad="auto", **even, light_window=31)],
             [FlatPage(**even, light_window=3), FlatPage(**even, light_window=32767), FlatPage((0, 100, 6, 30000), **even)],
             [FlatPage(**even, light_window=3), FlatPage(**even, light_window=32767)],
             [FlatPage(**even)]]
    return images, pages


def test_flatten_pages_evens_like_the_twin_in_one_mixed_call():
    from marconet_b200.pipeline import flatten_pages
    images, pages = _mixed()
    got = flatten_pages(images[:3] + [torch.from_numpy(im).to(DEV) for im in images[3:]], pages, to_host=True)
    kinds, inks, oversized = set(), set(), 0
    for im, pl, gl in zip(images, pages, got):
        for fp, g in zip(pl, gl):
            want = L.flatten(im, fp)
            _same_result(g, want)
            if fp.light is not None:
                kinds.add((want["kind"], "table" in want, isinstance(fp.skew, str) or isinstance(fp.quad, str)))
                inks.add(want["ink"])
                oversized += want["light_window"] > max(want["size"])
    assert inks == {"dark", "light"} and oversized >= 2
    assert {("rect", True, False), ("rect", False, False), ("quad", False, False), ("quad", True, True), ("quad", False, True),
            ("skew", False, False), ("skew", False, True)} <= kinds
    assert got[4][0]["size"] == (6, 32767) and got[5][0]["size"] == (32767, 6) and got[6][0]["size"] == (1, 1)
    # a device call gives the same pages as the host call
    dev = flatten_pages([torch.from_numpy(images[1]).to(DEV)], [pages[1]])[0]
    for d, g in zip(dev, got[1]):
        assert d["image"].is_cuda
        np.testing.assert_array_equal(d["image"].cpu().numpy(), g["image"])


def test_light_none_pages_are_untouched_by_light_pages_beside_them():
    from marconet_b200.pipeline import flatten_pages
    images, pages = _mixed()
    keep = [[fp for fp in pl if fp.light is None] for pl in pages]
    mixed = flatten_pages(images, pages, to_host=True)
    plain = flatten_pages(images, keep, to_host=True)
    n = 0
    for pl, ml, gl in zip(pages, mixed, plain):
        ml = [m for fp, m in zip(pl, ml) if fp.light is None]
        assert len(ml) == len(gl)
        for m, g in zip(ml, gl):
            assert m.keys() == g.keys() and "ink" not in g
            np.testing.assert_array_equal(m["image"], g["image"])
            assert all(m[key] == g[key] for key in m if key != "image")
            n += 1
    assert n == 3


def test_launches_and_synchronisations():
    from marconet_b200 import _lib, ops
    from marconet_b200.pipeline import FlatPage, flatten_pages
    page = torch.from_numpy(curled_page(6, "cylinder", PITCH, 21)[0]).to(DEV)
    base = [FlatPage(curve="auto"), FlatPage(skew=1.0)]

    def count(extra, to_host=False, pages=None):
        syncs = []
        real = torch.cuda.Stream.synchronize
        torch.cuda.Stream.synchronize = lambda self: (syncs.append(1), real(self))[1]
        try:
            n = ops.LAUNCHES
            flatten_pages([page], [(base if pages is None else pages) + extra], to_host=to_host)
            return ops.LAUNCHES - n, len(syncs)
        finally:
            torch.cuda.Stream.synchronize = real
    levels = _lib.PAGE_LEVELS
    n0, s0 = count([])
    assert n0 == (5 + 6 * levels) + 7 + 1 + 2                   # find_blocks, find_lines_curved, warp, field: as before
    rect = FlatPage((0, 0, 200, 150), light="even")
    assert count([rect]) == (n0 + 6, s0)
    assert count([rect] * 7) == (n0 + 6, s0)
    redo = [FlatPage(curve="auto", light="even"), FlatPage(skew=2.0, light="even")]
    assert count(redo) == (n0 + 10, s0)
    assert count(redo * 3 + [rect]) == (n0 + 10, s0)
    assert count(redo, to_host=True)[1] == count([], to_host=True)[1]
    # without a search or a copy back, only an "auto" ink is waited for, once
    assert count([rect], pages=[]) == (6, 1)
    assert count([rect._replace(polarity="dark")] * 3, pages=[]) == (6, 0)
    assert count([FlatPage()], pages=[]) == (0, 0)


def test_shaded_curled_page_is_found_traced_and_restored_after_evening(gpu_models):
    from marconet_b200.pipeline import FlatPage, TextPage, find_blocks, find_lines, flatten_pages, restore_regions
    page = shade(curled_page(8, "cylinder", PITCH, 11)[0], "gradient")
    assert find_blocks([page], [[TextPage(curve="auto")]])[0][0]["blocks"] == []     # unevened, the page is lost
    flat = flatten_pages([page], [[FlatPage(light="even")]])[0][0]
    assert flat["image"].is_cuda and flat["light_window"] == 27 and flat["ink"] == "dark"
    blocks = find_blocks([flat["image"]], [[TextPage(curve="auto")]])[0][0]["blocks"]
    assert len(blocks) == 1
    lines = find_lines([flat["image"]], [blocks])[0][0]["lines"]
    assert len(lines) == 8
    m = gpu_models["encoder"], gpu_models["tspgan"], gpu_models["sr"]
    out = restore_regions(*m, [flat["image"]], [[TextPage(curve="auto")]], scale=2, to_host=True)[0]
    res = out["regions"][0]
    assert "error" not in res and len(res["regions"]) == 1
    blk = res["regions"][0]
    assert "error" not in blk and len(blk["lines"]) == len(blk["regions"]) == 8
