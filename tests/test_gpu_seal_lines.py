"""Seal centre lines on the device (DESIGN.md section 7b, "Seal centre lines"): the line tables of one find_blocks call of drawn
and seeded random stamp pages, mixed with seal pages without the option and pages with rules, figures, panels and block
directions, against the numpy twin bit for bit; launch counts; a 4096-pixel seal on a 32767-wide page; 64 seals with lines; the
line limit; and restore_regions against the same call given the found arcs, lines and blocks."""
import cv2
import numpy as np
import pytest
import torch

from oracle import seal_lines as L

from test_gpu_pages import _same
from test_seal_lines import DRAWN, inner_line, seal_page
from test_seal_pages import BLUE, PAPER, RED, paragraph, stamp

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda:0")


def _check_lines(tab, ltab, recs):
    """A page's device line table against the twin's records (None: a zero record)."""
    n = min(int(tab["n_cand"]), 64) if not tab["error"] else 0
    for j in range(64):
        d = ltab["seal"][j]
        r = recs[j] if j < n else None
        if r is None:
            assert not d.tobytes().strip(b"\0"), j
            continue
        assert {f: int(d[f]) for f in L.FIELDS} == {f: r[f] for f in L.FIELDS}, j
        assert [tuple(int(v) for v in b) for b in d["box"][:r["n_lines"]]] == r["boxes"], j
        assert not d["box"][r["n_lines"]:].any() and not d["pad"].any()


def random_line_page(rng):
    """A seeded page with 1 or 2 stamps with 0 to 5 centre lines (random turn, ratio, colour and star).  (image, TextPage)."""
    from marconet_b200 import pipeline
    h, w = int(rng.integers(600, 800)), int(rng.integers(700, 900))
    img = np.full((h, w, 3), int(rng.integers(230, 250)), np.uint8)
    paragraph(img, 20, 40, 3, scale=0.6)
    for k in range(int(rng.integers(1, 3))):
        rx = int(rng.integers(90, 130))
        ry = int(rx * rng.uniform(0.75, 1.0))
        cx, cy = (rx + 10 + k * (w - 2 * rx - 20), int(rng.integers(ry + 150, h - ry - 5)))
        rot = float(rng.uniform(-25, 25))
        colour = RED if rng.integers(2) else BLUE
        n = int(rng.integers(0, 6))
        stamp(img, cx, cy, rx, ry, colour, rot=rot, star=n < 2 and bool(rng.integers(2)))
        r = min(rx, ry)
        for m in range(n):                                      # under the star when there is one, else across the centre
            dy = (0.45 if n == 1 else -0.3 + 0.15 * m) * r
            img[inner_line(h, w, cx, cy, "ABCDEFG"[:int(rng.integers(3, 8))], dy, 0.07 * r, rot)] = colour
    opts = [dict(), dict(rules="auto"), dict(figures="auto"), dict(panels="auto"), dict(block_direction="auto")]
    return img, pipeline.TextPage(seals="auto", seal_lines="auto", **opts[int(rng.integers(len(opts)))])


def _run(pages):
    """One pipeline._find_blocks call over (image, TextPage) pairs, and the raw tables of one ops.find_blocks call."""
    from marconet_b200 import ops, pipeline
    dimgs = [torch.from_numpy(im).to(DEV) for im, _ in pages]
    items = [(i, pg, pipeline._check_page(pg, *im.shape[:2], "page")) for i, (im, pg) in enumerate(pages)]
    n0 = ops.LAUNCHES
    with torch.cuda.device(DEV):
        got = pipeline._find_blocks(dimgs, items)
    launches = ops.LAUNCHES - n0
    pitems = [ops.PageItem(d, r, False, 0, seal_size=None if pg.seals is None else
                           pg.seal_size or pipeline.seal_size(r[2] - r[0], r[3] - r[1]), seal_lines=pg.seal_lines is not None)
              for d, (_, pg, r) in zip(dimgs, items)]
    out, caps = ops.find_blocks(pitems)
    host = out.cpu().numpy()
    return got, launches, items, pitems, host, caps


def test_line_tables_match_the_twin_and_other_pages_are_unchanged():
    from marconet_b200 import ops, pipeline
    rng = np.random.default_rng(11)
    pages = [(seal_page(**kw)[0], pipeline.TextPage(seals="auto", seal_lines="auto")) for kw in DRAWN.values()]
    pages += [random_line_page(rng) for _ in range(24)]
    plain = [(seal_page(**DRAWN["company"])[0], pipeline.TextPage(seals="auto")),
             (seal_page(**DRAWN["oval invoice seal"])[0], pipeline.TextPage(seals="auto", rules="auto")),
             (seal_page(lines=())[0], pipeline.TextPage(panels="auto"))]
    mixed = [p for pair in zip(pages, plain + [None] * len(pages)) for p in pair if p is not None]
    got, launches, items, pitems, host, caps = _run(mixed)
    assert launches == (5 + 6 * 24 + 3 * any(pg.rules for _, pg in mixed) + any(pg.figures for _, pg in mixed)
                        + any(pg.block_direction for _, pg in mixed) + 2 * any(pg.panels for _, pg in mixed) + 6 + 1)
    n_lines = 0
    for (im, pg), (_, _, rect), p, tab, ltab in zip(mixed, items, pitems, ops.seal_tables(host, pitems),
                                                    ops.seal_line_tables(host, pitems)):
        if pg.seal_lines is None:
            assert ltab is None
            continue
        _, recs = L.page_lines(im, rect, p.seal_size)
        _check_lines(tab, ltab, recs)
        n_lines += sum(r["n_lines"] for r in recs if r)
    assert n_lines >= 30
    # the pages without the option give what a call without the line pages gives
    alone = _run(plain)[0]
    assert [g for (_, pg), g in zip(mixed, got) if pg.seal_lines is None] == alone
    # and the line pages' blocks are those of seals="auto"
    for (im, pg), g in zip(mixed, got):
        if pg.seal_lines is not None:
            base = pipeline.find_blocks([im], [[pg._replace(seal_lines=None)]])[0][0]
            assert g["blocks"] == base["blocks"] and [s["box"] for s in g["seals"]] == [s["box"] for s in base["seals"]]


def test_launch_counts():
    from marconet_b200 import ops, pipeline
    img = seal_page()[0]
    for pgs in ([pipeline.TextPage(seals="auto")], [pipeline.TextPage(seals="auto")] * 3):
        n0 = ops.LAUNCHES
        a = pipeline.find_blocks([img], [[p._replace(seal_lines="auto") for p in pgs]])[0]
        n1 = ops.LAUNCHES
        b = pipeline.find_blocks([img], [pgs])[0]
        assert (n1 - n0) - (ops.LAUNCHES - n1) == 1
        assert [x["blocks"] for x in a] == [x["blocks"] for x in b]
    n0 = ops.LAUNCHES
    pipeline.find_blocks([img], [[pipeline.TextPage()]])
    assert ops.LAUNCHES - n0 == 5 + 6 * 24


def test_largest_seal_on_a_wide_page():
    """A 4096-pixel stamp with a centre line at the right end of a 32767-wide page: its line table equals the twin's."""
    from marconet_b200 import ops
    h, w = 4200, 32767
    img = np.full((h, w, 3), PAPER, np.uint8)
    cx, cy, r = w - 2050, 2100, 2046
    box = stamp(img, cx, cy, r, r, RED, glyphs="ABCDEFGH")[0]      # 4095 pixels wide, to w - 2
    img[cy, w - 2] = RED                                           # one more column on the ring: 4096, to w - 1
    img[inner_line(h, w, cx, cy, "ABCDE", 0.45 * r, 0.17 * r)] = RED
    assert box[2] == w - 2 and box[2] - box[0] == 4095
    pitems = [ops.PageItem(torch.from_numpy(img).to(DEV), (0, 0, w, h), False, 0, seal_size=1000, seal_lines=True)]
    out, _ = ops.find_blocks(pitems)
    host = out.cpu().numpy()
    tab, ltab = ops.seal_tables(host, pitems)[0], ops.seal_line_tables(host, pitems)[0]
    t = {"error": int(tab["error"]), "seals": [{f: int(s[f]) for f in ("x0", "y0", "x1", "y1", "found", "k_top")}
                                               for s in tab["seal"][:int(tab["n_cand"])]]}
    assert [(s["x1"] - s["x0"], s["x1"]) for s in t["seals"] if s["found"]] == [(4096, w - 1)]
    recs = [L.line_record(img, s) if s["found"] else None for s in t["seals"]]
    _check_lines(tab, ltab, recs)
    assert sum(r["n_lines"] for r in recs if r) >= 1


def _lattice(n, lines_per_seal=1):
    """n red rings of radius 60 with lines_per_seal centre lines each (4 rows high, 3 rows apart), 16 to a row."""
    rows = -(-n // 16)
    img = np.full((130 * rows + 20, 16 * 130 + 20, 3), PAPER, np.uint8)
    for k in range(n):
        r, c = divmod(k, 16)
        cx, cy = 75 + 130 * c, 75 + 130 * r
        stamp(img, cx, cy, 60, 60, RED, glyphs="", star=False)
        for m in range(lines_per_seal):
            img[cy - 17 + 7 * m:cy - 13 + 7 * m, cx - 15:cx + 15] = RED
    return img


def test_64_seals_with_lines_and_the_line_limit():
    from marconet_b200 import ops
    for img in (_lattice(64), _lattice(2, L.MAX_LINES), _lattice(2, L.MAX_LINES + 1)):
        pitems = [ops.PageItem(torch.from_numpy(img).to(DEV), (0, 0, img.shape[1], img.shape[0]), False, 0, seal_size=80,
                               seal_lines=True)]
        out, _ = ops.find_blocks(pitems)
        host = out.cpu().numpy()
        tab, ltab = ops.seal_tables(host, pitems)[0], ops.seal_line_tables(host, pitems)[0]
        t, recs = L.page_lines(img, None, 80)
        _check_lines(tab, ltab, recs)
        assert t["n_seals"] == int(tab["n_seals"]) and t["n_seals"] in (64, 2)
    assert [r["n_found"] for r in recs if r] == [L.MAX_LINES + 1] * 2 and [r["n_lines"] for r in recs if r] == [L.MAX_LINES] * 2


@pytest.mark.parametrize("kw", [dict(), dict(rot=15.0), DRAWN["oval invoice seal"]])
def test_restore_regions_equals_the_found_arcs_lines_and_blocks(gpu_models, monkeypatch, kw):
    from marconet_b200 import ops, pipeline
    monkeypatch.setattr(ops, "MODULE_GRAPHS", False)
    m = gpu_models["encoder"], gpu_models["tspgan"], gpu_models["sr"]
    img, box, _, masks = seal_page(h=560, w=700, cx=400, cy=380, **kw)
    pg = pipeline.TextPage(seals="auto", seal_lines="auto")
    found = pipeline.find_blocks([img], [[pg]])[0][0]
    arcs = [s["region"] for s in found["seals"] if s["region"] is not None]
    lines = [ln["region"] for s in found["seals"] for ln in s["lines"] if ln["region"] is not None]
    assert len(arcs) == 1 and len(lines) == len(masks)
    kw2 = dict(scale=2, feather=3, to_host=True)
    a = pipeline.restore_regions(*m, [img], [[pg]], **kw2)[0]
    b = pipeline.restore_regions(*m, [img], [arcs + lines + found["blocks"]], **kw2)[0]
    np.testing.assert_array_equal(a["image"], b["image"])
    entry = a["regions"][0]
    assert {k: v for k, v in entry.items() if k not in ("regions", "seal_regions", "seal_line_regions")} == found
    _same(entry["seal_regions"], b["regions"][:len(arcs)])
    _same(entry["seal_line_regions"], b["regions"][len(arcs):len(arcs) + len(lines)])
    _same(entry["regions"], b["regions"][len(arcs) + len(lines):])
