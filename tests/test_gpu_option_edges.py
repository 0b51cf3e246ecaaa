"""The page options, lighting and flat-remap kernels at the edges of their contracts, bit for bit against the numpy twins on
the inputs that test_option_edges.py builds and proves to reach those edges: rule runs straddling the 1024-bit iterations of
line_runs along rows and columns, figures and panels sharing bitmap words, the panel test's flat radius, modes and half-ink
thresholds, 32767-pixel leaves and exact direction ties, 32767 x 32767 pages and crops past 2^31 bytes, evening at the segment
sizes, in place and past 2^31 bytes, a remap destination past 2^31 bytes and 65535 pages in one call.

Each case is tagged with the features it reaches; the last test asserts that every REQUIRED feature was seen and every negative
control failed, and prints the kernel x feature table.  Large cases free their buffers before the next one and are skipped only
when torch.cuda.mem_get_info shows too little free memory."""
import collections
import gc

import numpy as np
import pytest
import torch

from oracle import figure_pages as FP
from oracle import flat_pages as F
from oracle import light as L
from oracle import mixed_pages as MP
from oracle import pages as P
from oracle import panel_pages as PP
from oracle import ruled_pages as RP
from oracle.remap import remap_cubic_u8

from test_gpu_panel_pages import _as_twin
from test_option_edges import (ALL_INK_OPTIONS, CORNER_OPTS, PAPER, _mode_to_larger, _opts, _outline_control, all_ink_expected,
                               all_ink_figure_expected, corner_content, figure_columns, figure_columns_expected,
                               figure_word_page, flat_lines, flat_pages, half_ink_pages, light_edge_sizes, light_margin,
                               light_window_reference, line_pages, panel_rule_page, panel_word_page, shifted, straddle_pages,
                               tall_leaf, tie_pages)

pytestmark = pytest.mark.gpu

SEEN = collections.defaultdict(collections.Counter)        # kernel -> feature -> cases
CONTROLS = {}                                               # control -> failed as it must
REQUIRED = {
    "rules": {"l straddling 1024 k, rows", "l - 1 straddling 1024 k, rows", "l straddling 1024 k, columns",
              "l - 1 straddling 1024 k, columns", "whole iteration without a zero", "w, h = 1 mod 32", "w, h = 0 mod 32",
              "1 x N", "N x 1", "rule_length 2", "rule_length 32767", "all ink 32767^2", "page > 2^31 bytes"},
    "figures": {"two in one word", "last word at x = 32767", "one word wide", "figure_size 2", "figure_size 32767",
                "1024 figures, largest frows"},
    "panels": {"two in one word", "2 pixels wide", "2 rows", "rule across under rules", "radius m +- 8", "radius m +- 9",
               "mode 0", "mode 255", "half ink", "half + 1 ink", "32767^2 flat panel", "page > 2^31 bytes"},
    "directions": {"32767-tall leaf", "32767-wide leaf", "band at 0", "band at 32766", "tie, one band each", "tie, one row band",
                   "tie, one column band", "tie, grid", "1 x 1"},
    "light": {"page > 2^31 bytes in place, pitched", "scratch > 2^31 bytes", "n = r, r + 1, k - 1, k, k + 1", "65535 pages"},
    "flat_remap": {"dst > 2^31 bytes", "65535 pages"},
    "page call": {"65535 pages, last with every option", "32767^2 with every option beside a small page"},
}
GIB = 1 << 30


def _dev():
    return torch.device("cuda:0")


def _need(nbytes):
    """Skips the case unless nbytes (and a GiB of headroom) are free on the device.  The blocks that earlier tests of the same
    process left in torch's caching allocator are handed back first: mem_get_info counts them as used."""
    gc.collect()
    torch.cuda.empty_cache()
    free = torch.cuda.mem_get_info(_dev())[0]
    if free < nbytes + GIB:
        pytest.skip(f"needs {nbytes + GIB} free bytes of device memory, {free} free "
                    f"({torch.cuda.memory_allocated(_dev())} allocated by this process)")


def _up(img):
    return torch.from_numpy(np.ascontiguousarray(img)).to(_dev())


def _page(**kw):
    """A TextPage of the twin's keyword arguments (rules, figures and block_direction as booleans)."""
    from marconet_b200.pipeline import TextPage
    kw = dict(kw)
    for key in ("rules", "figures", "block_direction", "panels"):
        kw[key] = "auto" if kw.pop(key, False) else None
    return TextPage(**kw)


def _call(items):
    """pipeline._find_blocks over items (device or host image, twin keyword arguments, panels?) in one call; per item the result
    in the twin's terms (or the error message)."""
    from marconet_b200 import pipeline
    dimgs, args = {}, []
    for img, kw, panels in items:
        if id(img) not in dimgs:
            dimgs[id(img)] = (len(dimgs), img if isinstance(img, torch.Tensor) else _up(img))
        i, d = dimgs[id(img)]
        rect = kw.get("rect") or (0, 0, d.shape[1], d.shape[0])
        args.append((i, _page(**kw, panels=panels), rect))
    got = pipeline._find_blocks({i: d for i, d in dimgs.values()}, args)
    return [g if isinstance(g, str) else _as_twin(g, panels) for g, (_, _, panels) in zip(got, items)]


def _plain(got):
    """A result without the options' keys a plain twin does not give."""
    return {k: v for k, v in got.items() if k not in ("directions",)}


# ---- rules ---------------------------------------------------------------------------------------------------------------
def test_rule_runs_across_iterations_and_line_pages():
    pages = straddle_pages() + line_pages()
    got = _call([(img, dict(polarity="dark", rules=True, rule_length=l), False) for _, img, l in pages])
    for (name, img, l), g in zip(pages, got):
        assert _plain(g) == RP.find_blocks(img, polarity="dark", rule_length=l), name
        SEEN["rules"].update({f"rule_length {l}": 1} if l in (2, 32767) else {})
    for name, _, _ in pages:
        axis = "columns" if name.startswith("columns") else "rows"
        if "x" in name and name[0] in "rc":
            SEEN["rules"].update({f"l straddling 1024 k, {axis}": 1, f"l - 1 straddling 1024 k, {axis}": 1,
                                  "whole iteration without a zero": 1})
            SEEN["rules"]["w, h = 1 mod 32" if "3073" in name else "w, h = 0 mod 32"] += 1
    SEEN["rules"].update({"1 x N": 1, "N x 1": 1})
    name, img, l = pages[2]
    CONTROLS["rule_length l + 1"] = RP.find_blocks(img, polarity="dark", rule_length=l + 1) != _plain(got[2])


# ---- figures -------------------------------------------------------------------------------------------------------------
def test_figures_sharing_words_and_at_the_last_word():
    img, narrow = figure_word_page(), figure_word_page(400)
    cols = figure_columns(32767)
    got = _call([(img, dict(polarity="dark", figures=True, figure_size=20), False),
                 (narrow, dict(polarity="dark", figures=True, figure_size=2), False),
                 (cols, dict(polarity="dark", figures=True, figure_size=2), False)])
    for g, im, f in zip(got[:2], (img, narrow), (20, 2)):
        assert _plain(g) == FP.find_blocks(im, polarity="dark", figure_size=f)
    assert got[0]["figures"][:3] == [(4, 2, 30, 30), (31, 2, 60, 30), (64, 2, 96, 30)]
    assert got[0]["figures"][-1][2] == 32767
    assert _plain(got[2]) == figure_columns_expected(32767)
    SEEN["figures"].update({"two in one word": 1, "last word at x = 32767": 1, "one word wide": 1, "figure_size 2": 2,
                            "1024 figures, largest frows": 1})


# ---- panels --------------------------------------------------------------------------------------------------------------
def test_panels_sharing_words_thin_panels_and_a_rule_across():
    word, rule = panel_word_page(), panel_rule_page()
    got = _call([(word, dict(panel_size=2), True), (rule, dict(rules=True, rule_length=250, panel_size=20), True)])
    assert got[0] == PP.find_blocks(word, panel_size=2)
    assert got[1] == PP.find_blocks(rule, rules=True, rule_length=250, panel_size=20)
    assert got[1]["panels"] == [(200, 20, 400, 80)]
    CONTROLS["panel without its outline"] = _outline_control(word, got[0])
    SEEN["panels"].update({"two in one word": 1, "2 pixels wide": 1, "2 rows": 1, "rule across under rules": 1})


def test_panel_test_thresholds():
    pages = flat_pages() + half_ink_pages()
    got = _call([(img, dict(panel_size=20), True) for _, img, _, _ in pages])
    tags = {"m+8": "radius m +- 8", "m-8": "radius m +- 8", "m+9": "radius m +- 9", "m-9": "radius m +- 9", "mode 0": "mode 0",
            "mode 255": "mode 255", "half + 0": "half ink", "half + 1": "half + 1 ink"}
    for (name, img, leaf, want), g in zip(pages, got):
        assert g == PP.find_blocks(img, panel_size=20), name
        assert (leaf in g["panels"]) == want, name
        SEEN["panels"][tags.get(name.split(",")[0], "tie")] += 1
    nine = [(img, g) for (name, img, _, _), g in zip(pages, got) if name == "m+9"]
    with pytest.MonkeyPatch.context() as mp:
        mp.setattr(PP, "FLAT", 9)
        CONTROLS["flat radius 9"] = all(PP.find_blocks(img, panel_size=20) != g for img, g in nine)
        mp.setattr(PP, "flat", _mode_to_larger)
        tie = [(img, g) for (name, img, _, _), g in zip(pages, got) if name == "tie to the smaller"]
        mp.setattr(PP, "FLAT", 8)
        CONTROLS["mode ties to the larger grey"] = all(PP.find_blocks(img, panel_size=20) != g for img, g in tie)


# ---- directions ----------------------------------------------------------------------------------------------------------
def test_directions_at_full_span_and_ties():
    tall = tall_leaf()
    wide = np.ascontiguousarray(tall.transpose(1, 0, 2))
    ties = tie_pages(2000)
    dot = np.full((1, 1, 3), 10, np.uint8)
    imgs = [tall, wide] + [im for _, im in ties] + [dot]
    got = _call([(im, dict(block_direction=True), False) for im in imgs])
    for im, g in zip(imgs, got):
        assert g == MP.find_blocks(im)
    assert got[0]["blocks"] == [(0, 0, 40, 32767)] and got[1]["blocks"] == [(0, 0, 32767, 40)]
    for (name, _), g in zip(ties, got[2:6]):
        assert g["undecided"] == [0], name
        SEEN["directions"][f"tie, {name}"] += 1
    SEEN["directions"].update({"32767-tall leaf": 1, "32767-wide leaf": 1, "band at 0": 2, "band at 32766": 2, "1 x 1": 1})


# ---- whole pages ---------------------------------------------------------------------------------------------------------
def test_32767_square_pages_and_a_corner_past_2_31_bytes():
    """The all-ink 32767 x 32767 page under each option against the closed form (|U| = 32767^2 with rule length 2; one flat
    panel; one figure of figure size 32767), with every option beside a small page whose tables equal its call alone; then a
    page of paper with corner_content in its far corner, read through a crop rectangle past 2^31 bytes."""
    n = 32767
    _need(3 * n * n + GIB)
    buf = torch.zeros((n, n, 3), dtype=torch.uint8, device=_dev())
    for o in ALL_INK_OPTIONS:
        o = _opts(o, n)
        g, = _call([(buf, dict(polarity="dark", **o), True)])
        assert g == all_ink_expected(n, **o), o
    g, = _call([(buf, dict(polarity="dark", figures=True, figure_size=n), False)])
    assert g == all_ink_figure_expected(n)
    SEEN["rules"].update({"all ink 32767^2": 1, "rule_length 2": 1})
    SEEN["figures"]["figure_size 32767"] += 1
    SEEN["panels"]["32767^2 flat panel"] += 1
    small = panel_word_page()
    every = dict(rules=True, rule_length=250, figures=True, block_direction=True, panel_size=2)
    alone, = _call([(small, every, True)])
    big, beside = _call([(buf, dict(polarity="dark", **_opts(ALL_INK_OPTIONS[1], n)), True), (small, every, True)])
    assert beside == alone == PP.find_blocks(small, **every)
    assert big == all_ink_expected(n, **_opts(ALL_INK_OPTIONS[1], n))
    SEEN["page call"]["32767^2 with every option beside a small page"] += 1

    buf.fill_(PAPER)
    c = corner_content()
    X, Y = n - c.shape[1], n - c.shape[0]
    assert Y * buf.stride(0) > 2 ** 31
    buf[Y:, X:] = _up(c)
    g, = _call([(buf, dict(rect=(X, Y, n, n), **CORNER_OPTS), True)])
    want = shifted(PP.find_blocks(c, **CORNER_OPTS), X, Y)
    assert g == want and want["rule_pixels"] > 0 and want["panels"] and want["figures"]
    SEEN["rules"]["page > 2^31 bytes"] += 1
    SEEN["panels"]["page > 2^31 bytes"] += 1
    del buf
    torch.cuda.empty_cache()


def test_65535_pages_the_last_with_every_option():
    from marconet_b200 import ops
    rng = np.random.default_rng(31)
    imgs = [np.full((7, 9, 3), PAPER, np.uint8)] + [np.where(rng.random((int(h), int(w), 1)) < 0.2, 10, PAPER).astype(np.uint8)
                                                  .repeat(3, axis=2) for h, w in zip(rng.integers(1, 30, 7), rng.integers(1, 30, 7))]
    last = panel_word_page()
    every = dict(rules=True, rule_length=250, figures=True, block_direction=True, panel_size=2)
    items = [(imgs[k % len(imgs)], {}, False) for k in range(65534)] + [(last, every, True)]
    assert sum(ops.page_bytes(im.shape[1], im.shape[0]) for im, _, _ in items) <= ops.PAGE_MAX_WORK
    got = _call(items)
    refs = [P.find_blocks(im) for im in imgs]
    for k, g in enumerate(got[:-1]):
        assert _plain(g) == refs[k % len(imgs)], k
    assert got[-1] == PP.find_blocks(last, **every)
    SEEN["page call"]["65535 pages, last with every option"] += 1


# ---- even lighting -------------------------------------------------------------------------------------------------------
def test_even_light_at_the_segment_sizes():
    from marconet_b200 import _lib, ops
    rng = np.random.default_rng(41)
    cases = []
    for k in (5, 7):
        for h in light_edge_sizes(k):
            for w in light_edge_sizes(k):
                for pol in ("dark", "light"):
                    cases.append((rng.integers(0, 256, (h, w, 3), dtype=np.uint8), k, pol))
    srcs = [_up(p) for p, _, _ in cases]
    dsts = [torch.empty_like(s) for s in srcs]
    ink = {"dark": _lib.INK_DARK, "light": _lib.INK_LIGHT}
    ops.even_light([(s, s, d, k, ink[pol]) for s, d, (_, k, pol) in zip(srcs, dsts, cases)])
    differ = 0
    for d, (p, k, pol) in zip(dsts, cases):
        got = d.cpu().numpy()
        np.testing.assert_array_equal(got, L.even(p, k, pol))
        differ += not np.array_equal(got, L.even(p, k + 2, pol))
    CONTROLS["window k + 2"] = differ > 0
    SEEN["light"]["n = r, r + 1, k - 1, k, k + 1"] += 1


def test_even_light_in_place_past_2_31_bytes():
    """A 32767 x 22000 page (2.16e9 bytes, so both scratch planes pass 2^31 bytes too) evened in place in a pitched view whose
    16 row guard bytes stay unchanged, against the windowed reference at its corners and middle."""
    from marconet_b200 import _lib, ops
    H, W, k = 32767, 22000, 7
    _need(3 * (H * (3 * W + 16)) + GIB)
    gen = torch.Generator(device=_dev()).manual_seed(43)
    buf = torch.randint(0, 256, (H, 3 * W + 16), dtype=torch.uint8, device=_dev(), generator=gen)
    page = buf[:, :3 * W].view(H, W, 3)
    assert 3 * H * W > 2 ** 31 and (H - 1) * buf.stride(0) > 2 ** 31
    guard = buf[:, 3 * W:].clone()
    boxes = [(0, 0, 64, 48), (W - 64, H - 48, W, H), (W // 2, H // 2, W // 2 + 64, H // 2 + 48), (W - 30, 0, W, 40)]
    crops = []
    for box in boxes:
        a, b, c, d = cr = light_margin(H, W, k, box)
        crops.append((cr, page[b:d, a:c].cpu().numpy(), page[min(H - 1, b + 1):min(H, d + 1), a:c].cpu().numpy()))
    ops.even_light([(page, page, page, k, _lib.INK_DARK)])
    shifted_differs = True
    for box, (cr, crop, crop1) in zip(boxes, crops):
        x0, y0, x1, y1 = box
        got = page[y0:y1, x0:x1].cpu().numpy()
        np.testing.assert_array_equal(got, light_window_reference(crop, cr, k, "dark", box))
        if crop1.shape == crop.shape:
            shifted_differs &= not np.array_equal(got, light_window_reference(crop1, cr, k, "dark", box))
    CONTROLS["a page with its rows shifted by one"] = shifted_differs
    assert torch.equal(buf[:, 3 * W:], guard)
    SEEN["light"].update({"page > 2^31 bytes in place, pitched": 1, "scratch > 2^31 bytes": 1})
    del buf, page, guard
    torch.cuda.empty_cache()


def test_even_light_65535_pages():
    from marconet_b200 import _lib, ops
    rng = np.random.default_rng(45)
    src = rng.integers(0, 256, (13, 4, 5, 3), dtype=np.uint8)
    ds = _up(src)
    dst = torch.empty((65535, 4, 5, 3), dtype=torch.uint8, device=_dev())
    ks = (3, 5, 7)
    ops.even_light([(ds[i % 13], ds[i % 13], dst[i], ks[i % 3], _lib.INK_DARK if i % 2 else _lib.INK_LIGHT)
                    for i in range(65535)])
    got = dst.cpu().numpy()
    memo = {}
    for i in range(65535):
        key = (i % 13, i % 3, i % 2)
        if key not in memo:
            memo[key] = L.even(src[i % 13], ks[i % 3], "dark" if i % 2 else "light")
        np.testing.assert_array_equal(got[i], memo[key], err_msg=str(i))
    SEEN["light"]["65535 pages"] += 1


# ---- flat remap ----------------------------------------------------------------------------------------------------------
def test_flat_remap_destination_past_2_31_bytes():
    """A 32767 x 64 flat page written into the far columns of a pitched buffer, its last rows past 2^31 bytes; every byte
    outside it stays unchanged."""
    from marconet_b200 import ops
    H, w, pitch = 32767, 64, 3 * 32768 + 16
    _need(H * pitch + GIB)
    rng = np.random.default_rng(47)
    src = rng.integers(0, 256, (H, 80, 3), dtype=np.uint8)
    buf = torch.full((H, pitch), 77, dtype=torch.uint8, device=_dev())
    x0 = pitch - 16 - 3 * w
    dst = buf[:, x0:x0 + 3 * w].view(H, w, 3)
    assert (H - 1) * pitch + x0 > 2 ** 31
    t = flat_lines(H, w)
    ops.flat_remap([(_up(src), dst, "rect", (5, 0), t)])
    mx, my = F.maps(t, w, H, "rect", (5, 0))
    want = remap_cubic_u8(src, mx, my)
    got = dst.cpu().numpy()
    np.testing.assert_array_equal(got, want)
    CONTROLS["a flat page with its rows shifted by one"] = not np.array_equal(got[1:], want[:-1])
    dst.fill_(77)
    assert bool((buf == 77).all().item())
    SEEN["flat_remap"]["dst > 2^31 bytes"] += 1
    del buf, dst
    torch.cuda.empty_cache()


def test_flat_remap_65535_pages():
    from marconet_b200 import ops
    rng = np.random.default_rng(49)
    src = rng.integers(0, 256, (13, 8, 9, 3), dtype=np.uint8)
    ds = _up(src)
    dst = torch.empty((65535, 6, 7, 3), dtype=torch.uint8, device=_dev())
    none = np.zeros((0, 9), np.float64)
    ops.flat_remap([(ds[i % 13], dst[i], "rect", (i % 3, 1), none) for i in range(65535)])
    got = dst.cpu().numpy()
    memo = {}
    for i in range(65535):
        key = (i % 13, i % 3)
        if key not in memo:
            mx, my = F.maps(none, 7, 6, "rect", (i % 3, 1))
            memo[key] = remap_cubic_u8(src[i % 13], mx, my)
        np.testing.assert_array_equal(got[i], memo[key], err_msg=str(i))
    SEEN["flat_remap"]["65535 pages"] += 1


# ---- coverage ------------------------------------------------------------------------------------------------------------
def test_coverage_and_negative_controls():
    print("\nkernel x feature: cases")
    for k in REQUIRED:
        feats = sorted(REQUIRED[k] | {f for f, n in SEEN[k].items() if n})
        print(f"  {k:11s} " + "  ".join(f"{f}={SEEN[k][f]}" for f in feats))
    print("negative controls (failed as they must):", CONTROLS)
    print("peak allocated bytes:", torch.cuda.max_memory_allocated(_dev()))
    for k, want in REQUIRED.items():
        assert want <= {f for f, n in SEEN[k].items() if n}, (k, want - {f for f, n in SEEN[k].items() if n})
    assert set(CONTROLS) == {"rule_length l + 1", "flat radius 9", "mode ties to the larger grey", "panel without its outline",
                             "window k + 2", "a page with its rows shifted by one", "a flat page with its rows shifted by one"}, \
        CONTROLS
    assert all(CONTROLS.values()), CONTROLS
