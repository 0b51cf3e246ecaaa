"""Book spreads (DESIGN.md section 7b, "Book spreads") on the GPU: the device's spine records bit for bit against the numpy twin
on hand-made masks and generated spreads, beside pages that are not spreads; flatten_pages with spread="auto" against the same
call given the two halves; a 32767-wide spread, spines at the ends of the search range and many spreads in one call; the
launch counts; and restore_regions on the two flat pages."""
import numpy as np
import pytest
import torch

from oracle import flat_pages as F
from oracle import spread_pages as SP

from test_curled_blocks import PITCH, curled_page
from test_flat_pages import open_book
from test_spread_pages import book_spread, mask_image, notched

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda:0")


def _device_spines(images, spreads):
    """(quads, spines) of ops.find_page_quads over ``images`` with the spines of ``spreads``, read back as numpy records."""
    from marconet_b200 import _lib, ops
    dev = [torch.from_numpy(im).to(DEV) for im in images]
    quads, spines = ops.find_page_quads([(d, _lib.INK_AUTO) for d in dev], spreads=spreads)
    torch.cuda.synchronize()
    return (quads.cpu().numpy().view(ops.page_quad_dtype()), spines.cpu().numpy().view(ops.page_spine_dtype()))


def _same_spine(got, want, what):
    assert bool(got["found"]) == want["found"], what
    assert tuple(got["st"]) == want["st"] and tuple(got["sb"]) == want["sb"], what
    for key in ("D", "E"):
        assert int(got[key]) == (np.iinfo(np.int64).min if want[key] is None else want[key]), (what, key)


def _masks():
    w, h = 202, 90
    lo, hi = 51, 151
    return [notched(120, 60, top=[(60, 8, 1)], bottom=[(50, 5, 2)]),
            notched(400, 200, top=[(150, 30, 1)], bottom=[(250, 12, 1)]),
            notched(64, 40, top=[(16, 3, 1)], bottom=[(48, 2, 1)]),
            notched(300, 100),
            notched(w, h, top=[(lo - 1, 40, 0), (lo, 20, 0), (100, 10, 1)], bottom=[(lo - 1, 30, 0), (101, 6, 1)]),
            notched(w, h, top=[(hi + 1, 40, 0), (hi, 20, 0), (100, 10, 1)], bottom=[(hi + 1, 30, 0), (hi, 6, 0)]),
            notched(1000, 60, top=[(500, 10, 1)], bottom=[(503, 9, 1)]),
            notched(1000, 60, top=[(500, 10, 1)], bottom=[(503, 10, 1)]),
            notched(150, 50, top=[(75, 2, 1)], bottom=[(70, 2, 1)]),
            notched(120, 60, top=[(60, 8, 1)], bottom=[(50, 5, 2)], pad=0),     # cols[w - 1] set and b(x) = h
            *[notched(m, h, top=[(c + e, 40, 0), (c, 20, 0)], bottom=[(c + e, 30, 0), (c, 6, 0)])
              for m in (201, 203) for c, e in ((-(-m // 4), -1), (m - -(-m // 4), 1))],    # tr.x - tl.x = 1, 3 mod 4
            np.pad(np.ones((48, 1), bool), 6)]                                   # one column wide: none in range


def test_device_spines_equal_the_twin_beside_other_pages():
    masks = [mask_image(m) for m in _masks()]
    spreads = [book_spread(*a)[0] for a in ((8, 6, 0.10, 1.0, 1.5, 1), (6, 8, 0.12, 2.0, 1.8, 2), (7, 5, 0.08, 3.0, 1.3, 3),
                                            (5, 7, 0.15, 1.5, 2.0, 4))]
    light = book_spread(6, 5, 0.12, 1.0, 1.6, 7, light=True)[0]
    others = [open_book("cylinder", PITCH, 14, 1.8), np.full((40, 50, 3), 200, np.uint8)]
    images = others[:1] + masks + spreads + others[1:]
    idx = list(range(1, 1 + len(masks) + len(spreads)))
    from marconet_b200 import _lib, ops
    quads, spines = _device_spines(images, idx)
    base = ops.find_page_quads([(torch.from_numpy(im).to(DEV), _lib.INK_AUTO) for im in images])
    np.testing.assert_array_equal(quads, base.cpu().numpy().view(ops.page_quad_dtype()))   # the corners do not change
    for k, sp in zip(idx, spines):
        want = SP.find_spine(images[k])
        assert [tuple(p) for p in quads[k]["quad"].reshape(4, 2)] == [tuple(p) for p in want["quad"]]
        _same_spine(sp, want["spine"], k)
    assert sum(bool(s["found"]) for s in spines) >= len(spreads) + 5
    lt = ops.find_page_quads([(torch.from_numpy(light).to(DEV), _lib.INK_LIGHT)], spreads=[0])[1]
    want = SP.find_spine(light, "light")["spine"]
    assert want["found"]
    _same_spine(lt.cpu().numpy().view(ops.page_spine_dtype())[0], want, "light")


def _same_page(got, want):
    """The same flat page apart from ``side``; the twin's own ``table`` (its line table) is not a pipeline key."""
    np.testing.assert_array_equal(got["image"], want["image"])
    assert {k for k in got if k != "side"} == {k for k in want if k not in ("side", "table")}
    for key in got:
        if key not in ("image", "side"):
            assert got[key] == want[key], key


def test_flatten_pages_spreads_equal_the_twin_in_one_mixed_call():
    from marconet_b200.pipeline import FlatPage, flatten_pages
    s1, _ = book_spread(8, 6, 0.10, 1.0, 1.5, 1)
    s2, _ = book_spread(6, 8, 0.12, 2.0, 1.8, 2)
    book = open_book("cylinder", PITCH, 14, 1.8)
    page, _, _ = curled_page(5, "flat", 0, 13)
    images = [s1, book, s2, page]
    pages = [[FlatPage(quad="auto", spread="auto", curve="auto"), FlatPage(quad="auto", spread="auto", direction="vertical")],
             [FlatPage(quad="auto", curve="auto")],
             [FlatPage(quad="auto", spread="auto", light="even"), FlatPage(quad="auto", spread="auto")],
             [FlatPage((10, 10, 300, 200)), FlatPage(light="even")]]
    got = flatten_pages(images, pages, to_host=True)
    _same_page(got[1][0], F.flatten(book, pages[1][0]))
    _same_page(got[3][0], F.flatten(page, pages[3][0]))
    for i, k in ((0, 0), (0, 1), (2, 1)):
        want = SP.flatten(images[i], pages[i][k])
        g = got[i][k]
        assert g["kind"] == "spread" and g["quad"] == want["quad"] and g["spine"] == want["spine"]
        assert g["depth"] == want["depth"]
        assert [p["side"] for p in g["pages"]] == [p["side"] for p in want["pages"]]
        for gp, wp in zip(g["pages"], want["pages"]):
            _same_page(gp, wp)
    assert [p["side"] for p in got[0][1]["pages"]] == ["right", "left"]
    # the light spread: each half as its own light page (its own window), checked against the halves given below
    assert [p["light_window"] for p in got[2][0]["pages"]] and got[2][0]["spine"] == got[2][1]["spine"]


@pytest.mark.parametrize("extra", [dict(), dict(curve="auto"), dict(light="even"), dict(curve="auto", light="even", strips=6)])
def test_spread_gives_the_bytes_of_its_halves_given(extra):
    from marconet_b200.pipeline import FlatPage, QuadRegion, flatten_pages
    photo, _ = book_spread(7, 6, 0.12, 1.5, 1.6, 9)
    got = flatten_pages([photo], [[FlatPage(quad="auto", spread="auto", **extra)]], to_host=True)[0][0]
    halves = [FlatPage(quad=QuadRegion(*p["quad"]), **extra) for p in got["pages"]]
    want = flatten_pages([photo], [halves], to_host=True)[0]
    for g, w, side in zip(got["pages"], want, ("left", "right")):
        assert g["side"] == side
        _same_page(g, w)


def test_limits_wide_range_ends_and_many_spreads():
    w = 32767 - 12
    mask = notched(w, 700, top=[(w // 2, 330, 1)], bottom=[(w // 2 + 7, 331, 1)])
    assert mask.shape[1] == 32767
    ends = _masks()[4:6]
    many = [notched(80 + k, 40 + k % 7, top=[((80 + k) // 2 + k % 5 - 2, 2 + k % 4, 1)], bottom=[((80 + k) // 2, 3, 1)])
            for k in range(64)]
    images = [mask_image(m) for m in [mask] + ends + many]
    quads, spines = _device_spines(images, list(range(len(images))))
    for k, (im, sp) in enumerate(zip(images, spines)):
        _same_spine(sp, SP.find_spine(im)["spine"], k)
    assert spines[0]["found"] and tuple(spines[0]["st"]) == (6 + w // 2, 6 + 330)
    assert tuple(spines[1]["st"]) == (6 + 51, 26) and tuple(spines[2]["st"]) == (6 + 151, 26)
    assert tuple(spines[2]["sb"]) == (6 + 151, 6 + 90 - 6)


def test_launch_counts_and_no_spread_found():
    from marconet_b200 import ops
    from marconet_b200.pipeline import FlatPage, flatten_pages
    photo, _ = book_spread(6, 5, 0.12, 1.0, 1.5, 11)
    book = open_book("cylinder", PITCH, 14, 1.8)
    n = ops.LAUNCHES
    flatten_pages([photo, book], [[FlatPage(quad="auto")], [FlatPage(quad="auto")]])
    assert ops.LAUNCHES == n + 8 + 1                             # corner search, rectify
    n = ops.LAUNCHES
    r = flatten_pages([photo, photo, book], [[FlatPage(quad="auto", spread="auto")], [FlatPage(quad="auto", spread="auto")],
                                             [FlatPage(quad="auto")]])
    assert ops.LAUNCHES == n + 8 + 2 + 1                         # the spines' two, whatever the spreads' number
    assert r[0][0]["kind"] == "spread" and r[2][0]["kind"] == "quad"
    n = ops.LAUNCHES
    with pytest.raises(ValueError, match=r"image 1, page 0: no spread found: the top and bottom notches are .* pixels deep, "
                                         r"where .* are needed"):
        flatten_pages([photo, book], [[FlatPage(quad="auto", spread="auto")], [FlatPage(quad="auto", spread="auto")]])
    assert ops.LAUNCHES == n + 8 + 2


def test_restore_regions_on_both_pages_of_a_spread(gpu_models):
    from marconet_b200.pipeline import FlatPage, TextPage, flatten_pages, restore_regions
    m = gpu_models["encoder"], gpu_models["tspgan"], gpu_models["sr"]
    photo, _ = book_spread(6, 4, 0.12, 1.5, 1.5, 21)
    spread = flatten_pages([photo], [[FlatPage(quad="auto", spread="auto", curve="auto")]])[0][0]
    flats = [p["image"] for p in spread["pages"]]
    out = restore_regions(*m, flats, [[TextPage()], [TextPage()]], scale=2, to_host=True)
    for o, f, k in zip(out, flats, (6, 4)):
        assert o["image"].shape == (2 * f.shape[0], 2 * f.shape[1], 3)
        page = o["regions"][0]
        assert "error" not in page and page["blocks"]
        assert all("error" not in b and b["lines"] and len(b["regions"]) == len(b["lines"]) for b in page["regions"])
        assert sum(len(b["lines"]) for b in page["regions"]) >= k
