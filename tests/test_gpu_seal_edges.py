"""The seal and spine kernels at the edges of their contracts, bit for bit against the numpy twins on the inputs that
test_seal_edges.py builds and proves to reach those edges.  Seal tables come through ops.find_blocks + ops.seal_tables and through
a direct call of mn_find_seals_u8 that also hands back the layout copies, which are compared byte for byte with the twin's
layout_copy; user boxes go through mn_seal_layout_u8 directly and through pipeline.find_lines.  Then the 4096-side candidates,
crops past 2^31 bytes, a row-strided view, 65535 sealed pages in one call, and the spines: masks at the ends of the middle half,
65535 spreads in one call and the depth key near its bound.

Each case is tagged with the features it reaches; the last test asserts that every REQUIRED feature was seen and every negative
control failed.  Large cases free their buffers before the next one and are skipped only when torch.cuda.mem_get_info shows too
little free memory."""
import collections
import ctypes
import gc

import numpy as np
import pytest
import torch

from oracle import seal_pages as S
from oracle import spread_pages as SP

import test_seal_edges as E
from test_seal_pages import PAPER, RED, stamp
from test_spread_pages import mask_image, notched

pytestmark = pytest.mark.gpu

SEEN = collections.Counter()
CONTROLS = {}
REQUIRED = {
    "chroma 63 | 64, every channel order, grey 0 and 255", "cell 1 | 2 pixels", "2-pixel run across a cell border",
    "last cells 1, 2, 3 wide and tall", "w = 0 mod 128", "1 x 1 page beside a large one", "NE diagonal at a cell-tile border",
    "NE diagonal at the last cell column", "NW diagonal", "component across many cell tiles", "components one off cell apart",
    "seal_size 8 at side 8 | 7", "seal_size 4096 at side 4096 | 4095", "side 4096 | 4097", "ratio 3:2 | over, both orientations",
    "64 | 65 candidates in one call", "(y0, x0) tie broken by root", "candidates on all four edges of an offset strided crop",
    "rays 0, 45, 90, 180, 270, square and oval", "centre pixel", "rho = 10/32, 26/32, 33/32 exactly", "ring 53 | 54",
    "4 ink == area at the ring's inner end", "32 ink == area | one less", "band stops at k = 10", "no gap: NO_BAND",
    "720 sec == band_ink | one less", "gap 1, 2 and text 8, 9", "all 72 sectors empty", "gap wraps 71 | 0", "tied gap runs",
    "copy at rho = 33/32 and just inside", "overlapping found boxes", "box across 32-pixel tiles", "found = 0 unpainted",
    "user box partly outside", "user box apart", "64 user boxes", "user boxes of side 4096", "user box flush with the image",
    "15642^2 page", "32767 x 7467 page", "crop source past 2^31 bytes", "copy past 2^31 bytes", "65535 sealed pages",
    "spine: last column and row", "spine: middle half 1, 2, 3 mod 4", "spine: no column in range", "spine: 65535 spreads",
    "spine: D >= 2^30 with a column tie"}
FIELDS = ("x0", "y0", "x1", "y1", "root", "ring", "found", "k_bottom", "k_top", "g0", "n_gap", "why", "band_ink")
GIB = 1 << 30


def _dev():
    return torch.device("cuda:0")


def _need(nbytes):
    """Skips the case unless nbytes (and a GiB of headroom) are free on the device, after handing back torch's cached blocks."""
    gc.collect()
    torch.cuda.empty_cache()
    free = torch.cuda.mem_get_info(_dev())[0]
    if free < nbytes + GIB:
        pytest.skip(f"needs {nbytes + GIB} free bytes of device memory, {free} free")


def _up(img):
    return torch.from_numpy(np.ascontiguousarray(img)).to(_dev())


def _records(recs):
    raw = bytes((type(recs[0]) * len(recs))(*recs))
    return torch.frombuffer(bytearray(raw), dtype=torch.uint8).to(_dev())


def _block(img, rect):
    x0, y0, x1, y1 = rect
    from marconet_b200 import _lib
    return _lib.TextBlock(img.data_ptr(), img.stride(0), x0, y0, x1 - x0, y1 - y0)


def direct_seals(items):
    """mn_find_seals_u8 over items (device image, rect, seal_size) in one call: per item (table, copy) as (numpy record, uint8
    CUDA tensor [h, w, 3])."""
    from marconet_b200 import _lib, ops
    tsz = ctypes.sizeof(_lib.SealTable)
    work = torch.empty(len(items) * tsz, dtype=torch.uint8, device=_dev())
    keep, recs, stiles, ctiles = [], [], 0, 0
    for j, (img, rect, ss) in enumerate(items):
        w, h = rect[2] - rect[0], rect[3] - rect[1]
        copy, label, box, cand = (torch.empty(n, dtype=torch.uint8, device=_dev()) for n in ops._seal_areas(w, h))
        keep.append((copy, label, box, cand))
        recs.append(_lib.SealPage(_block(img, rect), copy.data_ptr(), label.data_ptr(), box.data_ptr(), cand.data_ptr(),
                                  work.data_ptr() + j * tsz, ss))
        stiles = max(stiles, -(-w // 32) * -(-h // 32))
        ctiles = max(ctiles, -(-w // 128) * -(-h // 32))
    rec = _records(recs)
    _lib.check(_lib.load().mn_find_seals_u8(rec.data_ptr(), len(items), stiles, ctiles, work.data_ptr(), work.numel(),
                                            ops._stream()), "mn_find_seals_u8")
    tabs = work.cpu().numpy().view(ops.seal_table_dtype())
    out = [(t, k[0].view(r[3] - r[1], r[2] - r[0], 3)) for t, k, (_, r, _) in zip(tabs, keep, items)]
    del keep
    return out


def direct_layout(items):
    """mn_seal_layout_u8 over items (device image, rect, boxes in image pixels): the copies."""
    from marconet_b200 import _lib, ops
    tabs = _records([_lib.SealTable.from_buffer_copy(ops.seal_table(b, r[0], r[1])) for _, r, b in items])
    tsz = ctypes.sizeof(_lib.SealTable)
    copies, recs, tiles = [], [], 0
    for j, (img, r, _) in enumerate(items):
        w, h = r[2] - r[0], r[3] - r[1]
        copies.append(torch.empty((h, w, 3), dtype=torch.uint8, device=_dev()))
        recs.append(_lib.SealPage(_block(img, r), copies[-1].data_ptr(), 0, 0, 0, tabs.data_ptr() + j * tsz, 0))
        tiles = max(tiles, -(-w // 32) * -(-h // 32))
    rec = _records(recs)
    _lib.check(_lib.load().mn_seal_layout_u8(rec.data_ptr(), len(items), tiles, ops._stream()), "mn_seal_layout_u8")
    torch.cuda.synchronize()
    return copies


def _same_table(tab, want, what):
    assert (int(tab["error"]), int(tab["n_cand"]), int(tab["n_seals"])) == (want["error"], want["n_cand"], want["n_seals"]), what
    for s, r in zip(tab["seal"], want["seals"]):
        assert {f: int(s[f]) for f in FIELDS} == r, what


def _found(t):
    return [(s["x0"], s["y0"], s["x1"], s["y1"]) for s in t["seals"] if s["found"]]


def run_cases(cases):
    """cases: (name, crop, seal_size).  One direct call and one ops.find_blocks call over all of them; every table against the
    twin, every copy against its layout_copy byte for byte.  Returns the twin tables by name."""
    from marconet_b200 import _lib, ops
    dimgs = [_up(img) for _, img, _ in cases]
    items = [(d, (0, 0, d.shape[1], d.shape[0]), ss) for d, (_, _, ss) in zip(dimgs, cases)]
    got = direct_seals(items)
    pitems = [ops.PageItem(d, r, False, _lib.INK_AUTO, seal_size=ss) for d, r, ss in items]
    out, _ = ops.find_blocks(pitems)
    tabs = ops.seal_tables(out.cpu().numpy(), pitems)
    twins = {}
    for (name, img, ss), (tab, copy), tab2 in zip(cases, got, tabs):
        want = S.find_seals(img, ss)
        _same_table(tab, want, name)
        _same_table(tab2, want, name)
        np.testing.assert_array_equal(copy.cpu().numpy(), S.layout_copy(img, _found(want)), err_msg=name)
        twins[name] = (want, copy.cpu().numpy())
    return twins


# ---- colour, cells, components, candidates ---------------------------------------------------------------------------------
def test_colour_cells_components_and_candidates():
    chroma, _ = E.chroma_page()
    cases = [("chroma", chroma, 8), ("cells", E.cells_page(), 8), ("chains", E.chain_page(), 8), ("arcs", E.arcs_page(), 8),
             ("sizes", E.size_page(), 8), ("dot", np.full((1, 1, 3), RED, np.uint8), 8)]
    cases += [(f"last {img.shape[1]} x {img.shape[0]}", img, 8) for img in E.last_cell_pages()]
    twins = run_cases(cases)
    SEEN.update(["chroma 63 | 64, every channel order, grey 0 and 255", "cell 1 | 2 pixels", "2-pixel run across a cell border",
                 "last cells 1, 2, 3 wide and tall", "w = 0 mod 128", "1 x 1 page beside a large one",
                 "NE diagonal at a cell-tile border", "NE diagonal at the last cell column", "NW diagonal",
                 "components one off cell apart", "seal_size 8 at side 8 | 7", "(y0, x0) tie broken by root"])
    with pytest.MonkeyPatch.context() as mp:
        mp.setattr(S, "CHROMA", 63)
        CONTROLS["CHROMA 63"] = not np.array_equal(S.layout_copy(chroma, _found(S.find_seals(chroma, 8))), twins["chroma"][1])
    from scipy import ndimage
    with pytest.MonkeyPatch.context() as mp:
        mp.setattr(S, "ndimage", E._four_connected(ndimage))
        CONTROLS["4-connected cells"] = S.find_seals(E.chain_page(), 8) != twins["chains"][0]
    orig = S.candidates
    with pytest.MonkeyPatch.context() as mp:
        mp.setattr(S, "candidates", lambda crop, ss: (lambda n, c: (n, sorted(c, key=lambda e: (e[1], e[0], -e[4]))))(
            *orig(crop, ss)))
        CONTROLS["rank ties to the larger root"] = S.find_seals(E.arcs_page(), 8) != twins["arcs"][0]


def test_band_arc_ray_and_copy_pages():
    cases = [(name, img, 8) for name, img, _ in E.band_pages()]
    cases += [("empty", E.empty_page(), 8), ("ring 53", E.ring_pages()[0], 8), ("ring 54", E.ring_pages()[1], 8)]
    cases += [(name, img, 8) for name, img, _, _ in E.ray_pages()]
    cases += [(f"exact rho {j}", img, 8) for j, (img, _) in enumerate(E.exact_rho_pages())]
    over = np.full((360, 380, 3), PAPER, np.uint8)          # two rings whose boxes overlap, across 32-pixel tiles
    for (x, y, a), colour in (((20, 20, 200), RED), ((200, 180, 160), (40, 60, 190))):
        over[y:y + a, x:x + a][S.seal_mask(E.ring_crop(a, a))] = colour
    cases.append(("overlap", over, 40))
    twins = run_cases(cases)
    boxes = _found(twins["overlap"][0])
    assert len(boxes) == 2 and boxes[0][2] > boxes[1][0] and boxes[0][0] % 32 and boxes[0][2] - boxes[0][0] > 64
    assert twins["ring 53"][0]["seals"][0]["found"] == 0 and twins["ring 54"][0]["seals"][0]["found"] == 1
    SEEN.update(["rays 0, 45, 90, 180, 270, square and oval", "centre pixel", "rho = 10/32, 26/32, 33/32 exactly", "ring 53 | 54",
                 "4 ink == area at the ring's inner end", "32 ink == area | one less", "band stops at k = 10",
                 "no gap: NO_BAND", "720 sec == band_ink | one less", "gap 1, 2 and text 8, 9", "all 72 sectors empty",
                 "gap wraps 71 | 0", "tied gap runs", "copy at rho = 33/32 and just inside", "overlapping found boxes",
                 "box across 32-pixel tiles", "found = 0 unpainted"])
    pages = {name: img for name, img, _ in cases}
    for name, attr, value in (("ring 53", "RING_SECTORS", 53), ("band 32 ink == area", "band", E._band_gt),
                              ("720 sec == band_ink", "arc_gap", E._arc_gap_le)):
        with pytest.MonkeyPatch.context() as mp:
            mp.setattr(S, attr, value)
            CONTROLS[f"{attr} variant"] = S.find_seals(pages[name], 8) != twins[name][0]
    img = pages["exact rho 1"]
    CONTROLS["copy with rho <= 33/32"] = not np.array_equal(E.layout_copy_le(img, _found(twins["exact rho 1"][0])),
                                                           twins["exact rho 1"][1])


def test_64_and_65_candidates_and_an_offset_strided_crop():
    from marconet_b200 import _lib, ops
    from test_gpu_seal_pages import _rings
    run_cases([("64", _rings(64), 8), ("65", _rings(65), 8)])
    SEEN["64 | 65 candidates in one call"] += 1
    # a ring filling a crop at (36, 20) of a view whose rows are 3 W + 16 bytes apart
    H, W = 300, 400
    buf = torch.full((H, 3 * W + 16), 7, dtype=torch.uint8, device=_dev())
    view = buf[:, :3 * W].view(H, W, 3)
    view.fill_(PAPER)
    crop = E.ring_crop(250, 200)
    crop[95:105, 0:4] = RED
    view[20:220, 36:286] = _up(crop)
    rect = (36, 20, 286, 220)
    (tab, copy), = direct_seals([(view, rect, 8)])
    want = S.find_seals(crop, 8)
    assert _found(want) == [(0, 0, 250, 200)]
    _same_table(tab, want, "strided")
    np.testing.assert_array_equal(copy.cpu().numpy(), S.layout_copy(crop, _found(want)))
    out, _ = ops.find_blocks([ops.PageItem(view, rect, False, _lib.INK_AUTO, seal_size=8)])
    _same_table(ops.seal_tables(out.cpu().numpy(), [ops.PageItem(view, rect, False, 0, seal_size=8)])[0], want, "strided")
    assert bool((buf[:, 3 * W:] == 7).all())
    SEEN["candidates on all four edges of an offset strided crop"] += 1


def test_4096_side_candidates():
    cases = [(f"{A} x {B} at {ss}", E.ring_crop(A, B), ss) for A, B, ss, _ in E.BIG]
    _need(sum(4 * img.nbytes for _, img, _ in cases))
    twins = run_cases(cases)
    assert [bool(twins[name][0]["n_seals"]) for name, _, _ in cases] == [c for *_, c in E.BIG]
    SEEN.update(["seal_size 4096 at side 4096 | 4095", "side 4096 | 4097", "ratio 3:2 | over, both orientations",
                 "component across many cell tiles"])


# ---- user boxes -----------------------------------------------------------------------------------------------------------
def test_user_boxes_through_the_layout_entry_and_find_lines():
    from marconet_b200 import pipeline
    img = np.full((4300, 4200, 3), PAPER, np.uint8)
    from test_seal_pages import paragraph
    paragraph(img, 130, 200, 40)
    stamp(img, 300, 300, 120, 110)
    stamp(img, 1820, 1620, 90, 90, colour=(40, 60, 190))
    rect = (100, 150, 1880, 1680)
    many = tuple((110 + 12 * (j % 16), 160 + 30 * (j // 16), 150 + 12 * (j % 16), 200 + 30 * (j // 16)) for j in range(64))
    sets = {"partly outside": ((180, 190, 420, 410), (1720, 1520, 1920, 1720)), "apart": ((3000, 3000, 3060, 3060),),
            "64 boxes": many, "side 4096": ((0, 100, 4096, 4196), (50, 0, 4146, 4096)),
            "flush": ((104, 204, 4200, 4300), (0, 0, 300, 300))}
    dimg = _up(img)
    copies = direct_layout([(dimg, rect, boxes) for boxes in sets.values()])
    x0, y0, x1, y1 = rect
    for (name, boxes), copy in zip(sets.items(), copies):
        want = S.layout_copy(img[y0:y1, x0:x1], [(a - x0, b - y0, c - x0, d - y0) for a, b, c, d in boxes])
        np.testing.assert_array_equal(copy.cpu().numpy(), want, err_msg=name)
        blk = pipeline.TextBlock(rect, seals=boxes)
        got = pipeline.find_lines([img], [[blk]])[0][0]
        assert got == pipeline.find_lines([S.layout_image(img, rect, boxes)], [[blk._replace(seals=())]])[0][0], name
    SEEN.update(["user box partly outside", "user box apart", "64 user boxes", "user boxes of side 4096",
                 "user box flush with the image"])


# ---- sizes ----------------------------------------------------------------------------------------------------------------
def _corner_window():
    return E.stamp_window()


@pytest.mark.parametrize("W, H", [(15642, 15642), (32767, 7467)])
def test_largest_sealed_pages(W, H):
    from marconet_b200 import _lib, ops
    assert ops.page_bytes(W, H, seals=True) <= ops.PAGE_MAX_WORK < ops.page_bytes(W + (W == H), H + 1, seals=True)
    _need(3 * W * H + ops.PAGE_MAX_WORK)
    buf = torch.full((H, W, 3), PAPER, dtype=torch.uint8, device=_dev())
    win = _corner_window()
    ox, oy = (W - 260) // 4 * 4, (H - 260) // 4 * 4
    buf[oy:oy + 260, ox:ox + 260] = _up(win)
    items = [ops.PageItem(buf, (0, 0, W, H), False, _lib.INK_AUTO, seal_size=100)]
    out, _ = ops.find_blocks(items)
    _same_table(ops.seal_tables(out.cpu().numpy(), items)[0], E.windowed(win, ox, oy, W, 100), "largest")
    SEEN[f"{W}^2 page" if W == H else f"{W} x {H} page"] += 1
    del buf, out
    torch.cuda.empty_cache()


def test_32767_square_crops_past_2_31_bytes():
    """A sealed crop in the far corner of a 32767 x 32767 image through ops.find_blocks; then the whole image through the direct
    entry, with stamps at two opposite corners, its copy past 2^31 bytes."""
    from marconet_b200 import _lib, ops
    n = 32767
    _need(2 * 3 * n * n + 5 * (n // 4 + 1) ** 2 * 4 + GIB)
    buf = torch.full((n, n, 3), PAPER, dtype=torch.uint8, device=_dev())
    win = _corner_window()
    X, Y = n - 300, n - 300
    buf[Y + 20:Y + 280, X + 20:X + 280] = _up(win)
    crop = buf[Y:, X:].cpu().numpy()
    assert Y * buf.stride(0) > 2 ** 31
    items = [ops.PageItem(buf, (X, Y, n, n), False, _lib.INK_AUTO, seal_size=100)]
    out, _ = ops.find_blocks(items)
    want = S.find_seals(crop, 100)
    assert want["n_seals"] == 1
    _same_table(ops.seal_tables(out.cpu().numpy(), items)[0], want, "far corner")
    del out
    SEEN["crop source past 2^31 bytes"] += 1
    buf[:260, :260] = _up(win)
    o2 = (n - 260) // 4 * 4
    buf[Y + 20:Y + 280, X + 20:X + 280] = PAPER
    buf[o2:o2 + 260, o2:o2 + 260] = _up(win)
    (tab, copy), = direct_seals([(buf, (0, 0, n, n), 100)])
    t1, t2 = E.windowed(win, 0, 0, n, 100), E.windowed(win, o2, o2, n, 100)
    want = dict(error=0, n_cand=t1["n_cand"] + t2["n_cand"], n_seals=2, seals=t1["seals"] + t2["seals"])
    _same_table(tab, want, "whole")
    for o, t in ((0, t1), (o2, t2)):
        np.testing.assert_array_equal(copy[o:o + 260, o:o + 260].cpu().numpy(),
                                      S.layout_copy(win, [(a - o, b - o, c - o, d - o) for a, b, c, d in _found(t)]))
        copy[o:o + 260, o:o + 260] = buf[o:o + 260, o:o + 260]
    assert (n - 1) * 3 * n > 2 ** 31 and torch.equal(copy, buf)
    SEEN["copy past 2^31 bytes"] += 1
    del buf, copy
    torch.cuda.empty_cache()


def test_65535_sealed_pages():
    from marconet_b200 import _lib, ops
    dots = _up(np.array([[[PAPER] * 3], [RED]], np.uint8).reshape(2, 1, 1, 3))
    last = E.page(200, 200, E.sel(200, 200, [20], range(10, 40)))
    dl = _up(last)
    items = [ops.PageItem(dots[k % 2], (0, 0, 1, 1), False, _lib.INK_AUTO, seal_size=8) for k in range(65534)]
    items.append(ops.PageItem(dl, (0, 0, 200, 200), False, _lib.INK_AUTO, seal_size=8))
    assert sum(ops.page_bytes(p.rect[2], p.rect[3], seals=True) for p in items) <= ops.PAGE_MAX_WORK
    out, _ = ops.find_blocks(items)
    tabs = ops.seal_tables(out.cpu().numpy(), items)
    assert all((int(t["error"]), int(t["n_cand"])) == (0, 0) for t in tabs[:-1])
    want = S.find_seals(last, 8)
    assert want["n_seals"] == 1
    _same_table(tabs[-1], want, "last")
    SEEN["65535 sealed pages"] += 1


# ---- spines ---------------------------------------------------------------------------------------------------------------
def _spines(images, spreads):
    from marconet_b200 import _lib, ops
    quads, spines = ops.find_page_quads([(_up(im), _lib.INK_AUTO) for im in images], spreads=spreads)
    return quads.cpu().numpy().view(ops.page_quad_dtype()), spines.cpu().numpy().view(ops.page_spine_dtype())


def _same_spine(got, want, what):
    assert bool(got["found"]) == want["found"], what
    assert tuple(got["st"]) == want["st"] and tuple(got["sb"]) == want["sb"], what
    for key in ("D", "E"):
        assert int(got[key]) == (np.iinfo(np.int64).min if want[key] is None else want[key]), (what, key)


def test_spines_at_the_ends_of_their_ranges_and_65535_spreads():
    from test_gpu_spread_pages import _masks
    masks = _masks()
    images = [mask_image(m) for m in masks]
    _, spines = _spines(images, list(range(len(images))))
    for k, (im, sp) in enumerate(zip(images, spines)):
        _same_spine(sp, SP.find_spine(im)["spine"], k)
    assert any(int(s["st"][0]) == -1 and int(s["D"]) == np.iinfo(np.int64).min for s in spines)
    SEEN.update(["spine: last column and row", "spine: middle half 1, 2, 3 mod 4", "spine: no column in range"])
    small = [mask_image(notched(20 + k, 12, top=[(10 + k // 2, 3, 1)], bottom=[(9, 2, 1)])) for k in range(5)]
    spread = mask_image(notched(300, 100, top=[(150, 20, 1)], bottom=[(152, 18, 1)]))
    images = [small[k % 5] for k in range(65534)] + [spread]
    _, spines = _spines(images, list(range(65535)))
    want = [SP.find_spine(im)["spine"] for im in small]
    for k in range(65534):
        _same_spine(spines[k], want[k % 5], k)
    w = SP.find_spine(spread)["spine"]
    assert w["found"]
    _same_spine(spines[-1], w, "last")
    SEEN["spine: 65535 spreads"] += 1


def _key_call(mask, quad):
    """mn_find_page_spines_u8 on a hand-made label plane (the page's pixels labelled 7, the rest -1) with best and the quad set
    by hand: the mn_page_spine record."""
    from marconet_b200 import _lib, ops
    h, w = mask.shape
    label = torch.full((h, w), -1, dtype=torch.int32, device=_dev())
    label[torch.from_numpy(mask).to(_dev())] = 7
    best = torch.tensor([(1 << 32) | (~7 & 0xffffffff)], dtype=torch.int64, device=_dev())
    res = torch.zeros(ctypes.sizeof(_lib.PageQuad), dtype=torch.uint8, device=_dev())
    pq = _lib.PageQuad()
    for j, v in enumerate(np.ravel(quad)):
        pq.quad[j] = int(v)
    res.copy_(torch.frombuffer(bytearray(bytes(pq)), dtype=torch.uint8))
    return _key_launch(label, best, res, h, w)


def _key_launch(label, best, res, h, w):
    from marconet_b200 import _lib, ops
    qp = _records([_lib.QuadPage(_lib.TextBlock(0, 0, 0, 0, w, h), label.data_ptr(), 0, 0, best.data_ptr(), 0, res.data_ptr())])
    cols = torch.zeros(2 * w, dtype=torch.int32, device=_dev())
    out = torch.zeros(ctypes.sizeof(_lib.PageSpine), dtype=torch.uint8, device=_dev())
    sp = _records([_lib.SpinePage(qp.data_ptr(), cols.data_ptr(), out.data_ptr())])
    _lib.check(_lib.load().mn_find_page_spines_u8(sp.data_ptr(), 1, -(-w // 32) * -(-h // 32), ops._stream()),
               "mn_find_page_spines_u8")
    torch.cuda.synchronize()
    return out.cpu().numpy().view(ops.page_spine_dtype())[0]


def test_spine_depth_key_near_its_bound():
    n0 = 4 * 33 + 3
    x1, x2 = n0 // 2 - 3, n0 // 2 + 5
    m, quad = E.key_plane(n0, x1, x2)
    got = _key_call(m, quad)
    _same_spine(got, SP.spine(m, quad), "downsized")

    def larger_x(p, q, pts, sign):                  # SP._deepest with ties to the larger column
        best = (None, (-1, -1))
        span = q[0] - p[0]
        for x, y in pts:
            if 4 * (x - p[0]) >= span and 4 * (q[0] - x) >= span:
                d = sign * SP._cross(p, q, (x, y))
                if best[0] is None or d >= best[0]:
                    best = (d, (x, y))
        return best
    with pytest.MonkeyPatch.context() as mp:
        mp.setattr(SP, "_deepest", larger_x)
        want = SP.spine(m, quad)
    CONTROLS["spine ties to the larger column"] = tuple(got["st"]) != want["st"]
    n = 32767
    _need(4 * n * n + GIB)
    x1, x2 = n // 2 - 3, n // 2 + 5
    label = torch.full((n, n), 7, dtype=torch.int32, device=_dev())
    label[:n - 1, x1] = -1
    label[:n - 1, x2] = -1
    best = torch.tensor([(1 << 32) | (~7 & 0xffffffff)], dtype=torch.int64, device=_dev())
    from marconet_b200 import _lib
    pq = _lib.PageQuad()
    for j, v in enumerate(np.ravel(E.key_plane(1, 0, 0)[1]) * n):      # (0, -n), (n, -n), (n, 2 n), (0, 2 n)
        pq.quad[j] = int(v)
    res = torch.frombuffer(bytearray(bytes(pq)), dtype=torch.uint8).to(_dev())
    got = _key_launch(label, best, res, n, n)
    want = E.key_expected(n, x1, x2)
    _same_spine(got, want, "32767")
    assert int(got["D"]) >= 2 ** 30
    SEEN["spine: D >= 2^30 with a column tie"] += 1
    del label
    torch.cuda.empty_cache()


# ---- coverage -------------------------------------------------------------------------------------------------------------
def test_coverage_and_negative_controls():
    print("\nfeature: cases")
    for f in sorted(REQUIRED | set(SEEN)):
        print(f"  {f}: {SEEN[f]}")
    print("negative controls (failed as they must):", CONTROLS)
    print("peak allocated bytes:", torch.cuda.max_memory_allocated(_dev()))
    assert REQUIRED <= {f for f, n in SEEN.items() if n}, REQUIRED - {f for f, n in SEEN.items() if n}
    assert set(CONTROLS) == {"CHROMA 63", "4-connected cells", "rank ties to the larger root", "RING_SECTORS variant",
                             "band variant", "arc_gap variant", "copy with rho <= 33/32", "spine ties to the larger column"}, \
        CONTROLS
    assert all(CONTROLS.values()), CONTROLS
