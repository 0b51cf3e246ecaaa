"""Seals on the device (DESIGN.md section 7b, "Seals"): the seal tables of one find_blocks call of seeded random pages, mixed
with pages without seals and with rules, figures, panels and block directions, against the numpy twin bit for bit; their
layouts against the same pages' layout copies; launch counts; a 32767-wide page; the 64-candidate limit; restore_regions
against the same call given the found arcs and blocks; a page without seal colour; and a photographed contract."""
import cv2
import numpy as np
import pytest
import torch

from oracle import seal_pages as S

from test_gpu_pages import _same
from test_seal_pages import BLUE, PAPER, RED, contract_page, paragraph, stamp

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda:0")
FIELDS = ("x0", "y0", "x1", "y1", "root", "ring", "found", "k_bottom", "k_top", "g0", "n_gap", "why", "band_ink")


def random_seal_page(rng):
    """A seeded page of paragraphs with 0 to 2 stamps (red or blue, round or oval, turned by hand, over the text or not) and a
    random crop, seal size and layout options.  (image, TextPage)."""
    from marconet_b200 import pipeline
    h, w = int(rng.integers(500, 800)), int(rng.integers(600, 900))
    img = np.full((h, w, 3), int(rng.integers(230, 250)), np.uint8)
    for k in range(int(rng.integers(2, 5))):
        paragraph(img, int(rng.integers(10, 80)), 40 + 150 * k, int(rng.integers(2, 5)), scale=float(rng.uniform(0.5, 0.8)))
    for _ in range(int(rng.integers(0, 3))):
        rx = int(rng.integers(60, 120))
        ry = int(rx * rng.uniform(0.75, 1.3))
        cx, cy = int(rng.integers(rx + 2, w - rx - 2)), int(rng.integers(ry + 2, h - ry - 2))
        stamp(img, cx, cy, rx, ry, RED if rng.integers(2) else BLUE, rot=float(rng.uniform(-20, 20)))
    x0, y0 = int(rng.integers(0, 30)), int(rng.integers(0, 30))
    opts = [dict(), dict(rules="auto"), dict(figures="auto"), dict(panels="auto"), dict(block_direction="auto")]
    kw = opts[int(rng.integers(len(opts)))]
    seals = dict(seals="auto", seal_size=int(rng.integers(40, 90))) if rng.integers(4) else {}
    return img, pipeline.TextPage((x0, y0, w - int(rng.integers(0, 30)), h - int(rng.integers(0, 30))), **kw, **seals)


def _twin_table(img, pg, rect):
    x0, y0, x1, y1 = rect
    return S.find_seals(img[y0:y1, x0:x1], pg.seal_size or S.default_seal_size(x1 - x0, y1 - y0))


def test_seal_tables_and_layouts_match_the_twin():
    from marconet_b200 import ops, pipeline
    rng = np.random.default_rng(5)
    pages = [random_seal_page(rng) for _ in range(36)]
    pages.append((contract_page()[0], pipeline.TextPage(seals="auto")))
    pages.append((contract_page(rx=130, ry=95, colour=BLUE, rot=15.0)[0], pipeline.TextPage(seals="auto", rules="auto")))
    dimgs = [torch.from_numpy(im).to(DEV) for im, _ in pages]
    items = [(i, pg, pipeline._check_page(pg, *im.shape[:2], "page")) for i, (im, pg) in enumerate(pages)]
    n0 = ops.LAUNCHES
    with torch.cuda.device(DEV):
        got = pipeline._find_blocks(dimgs, items)
    assert ops.LAUNCHES - n0 == (5 + 6 * 24 + 3 * any(pg.rules for _, pg in pages) + any(pg.figures for _, pg in pages)
                                 + any(pg.block_direction for _, pg in pages) + 2 * any(pg.panels for _, pg in pages) + 6)
    # the raw seal tables, bit for bit
    pitems = [ops.PageItem(d, r, False, 0, seal_size=None if pg.seals is None else
                           pg.seal_size or pipeline.seal_size(r[2] - r[0], r[3] - r[1]))
              for d, (_, pg, r) in zip(dimgs, items)]
    out, _ = ops.find_blocks(pitems)
    n_found = 0
    for (im, pg), (_, _, rect), tab in zip(pages, items, ops.seal_tables(out.cpu().numpy(), pitems)):
        if tab is None:
            continue
        t = _twin_table(im, pg, rect)
        assert (int(tab["error"]), int(tab["n_cand"]), int(tab["n_seals"])) == (t["error"], t["n_cand"], t["n_seals"])
        for s, r in zip(tab["seal"], t["seals"]):
            assert {f: int(s[f]) for f in FIELDS} == r
        n_found += t["n_seals"]
    assert n_found >= 20
    # each sealed page's layout is the layout of its twin layout copy, with the seals given to the blocks they meet
    for (im, pg), (_, _, rect), res in zip(pages, items, got):
        if pg.seals is None:
            continue
        boxes = [s["box"] for s in res["seals"]]
        _, twin_boxes = S.page_seals(im, rect, pg.seal_size)
        assert boxes == twin_boxes
        copy = S.layout_image(im, rect, boxes)
        plain = pipeline.find_blocks([copy], [[pg._replace(seals=None, seal_size=None)]])[0][0]
        assert [b._replace(seals=()) for b in res["blocks"]] == plain["blocks"]
        assert all(b.seals == pipeline._meeting(res["seals"], b.rect) for b in res["blocks"])
        assert {k: v for k, v in res.items() if k not in ("blocks", "seals", "seal_size")} == \
            {k: v for k, v in plain.items() if k != "blocks"}


def test_launch_counts_and_pages_without_seals():
    from marconet_b200 import ops, pipeline
    img = contract_page()[0]
    other = contract_page(over=False)[0]
    for extra in ({}, dict(rules="auto")):
        n0 = ops.LAUNCHES
        a = pipeline.find_blocks([img, other], [[pipeline.TextPage(seals="auto")], [pipeline.TextPage(**extra)]])
        n1 = ops.LAUNCHES
        b = pipeline.find_blocks([img, other], [[pipeline.TextPage()], [pipeline.TextPage(**extra)]])
        n2 = ops.LAUNCHES
        assert (n1 - n0) - (n2 - n1) == 6
        assert a[1] == b[1]
    blk = pipeline.TextBlock((30, 270, 700, 450), seals=tuple(s["box"] for s in a[0][0]["seals"]))
    n0 = ops.LAUNCHES
    sealed = pipeline.find_lines([img], [[blk, pipeline.TextBlock((30, 40, 700, 200))]])[0]
    n1 = ops.LAUNCHES
    plain = pipeline.find_lines([img], [[blk._replace(seals=()), pipeline.TextBlock((30, 40, 700, 200))]])[0]
    assert (n1 - n0) - (ops.LAUNCHES - n1) == 1
    assert sealed[1] == plain[1]
    copy = S.layout_image(img, (0, 0, img.shape[1], img.shape[0]), blk.seals)
    assert sealed[0] == pipeline.find_lines([copy], [[blk._replace(seals=())]])[0][0]
    assert len(sealed[0]["lines"]) == 5


def test_wide_page_with_a_seal_at_its_right_end():
    """A 32767-wide page with a stamp at its right end and one near its middle: both are found, and their tables equal the
    twin's; the right one's arc lies past the 2^14 pixels a curved region's remap reaches, so it has no region, and says why."""
    from marconet_b200 import ops, pipeline
    img = np.full((300, 32767, 3), PAPER, np.uint8)
    for x in range(20, 32000, 800):
        cv2.putText(img, "words %d" % x, (x, 40), cv2.FONT_HERSHEY_SIMPLEX, 0.6, (20, 20, 20), 1, cv2.LINE_AA)
    middle = stamp(img, 15000, 150, 120, 120, BLUE)[0]
    box = stamp(img, 32767 - 121, 150, 120, 120, RED)[0]
    assert box[2] >= 32767 - 2
    pg = pipeline.TextPage(seals="auto")
    pitems = [ops.PageItem(torch.from_numpy(img).to(DEV), (0, 0, 32767, 300), False, 0, seal_size=100)]
    out, _ = ops.find_blocks(pitems)
    tab = ops.seal_tables(out.cpu().numpy(), pitems)[0]
    t = S.find_seals(img, 100)
    assert t["n_seals"] == 2
    for s, r in zip(tab["seal"], t["seals"]):
        assert {f: int(s[f]) for f in FIELDS} == r
    res = pipeline.find_blocks([img], [[pg._replace(seal_size=100)]])[0][0]
    assert [s["box"] for s in res["seals"]] == [middle, box]
    assert res["seals"][0]["arc"] is not None and res["seals"][1]["arc"] is None
    assert "int16 remap" in res["seals"][1]["why"] and res["seals"][1]["band"] is not None


def _rings(n):
    """n small red rings on a 32-pixel lattice, 16 to a row: each one a candidate at seal size 8."""
    rows = -(-n // 16)
    img = np.full((32 * rows + 32, 560, 3), PAPER, np.uint8)
    for k in range(n):
        r, c = divmod(k, 16)
        cv2.circle(img, (24 + 32 * c, 24 + 32 * r), 9, RED, 2)
    return img


def test_the_candidate_limit():
    from marconet_b200 import pipeline
    img = _rings(64)
    res = pipeline.find_blocks([img], [[pipeline.TextPage(seals="auto", seal_size=8)]])[0][0]
    t = S.find_seals(img, 8)
    assert t["n_cand"] == 64 and len(res["seals"]) == t["n_seals"]
    assert [s["box"] for s in res["seals"]] == [(s["x0"], s["y0"], s["x1"], s["y1"]) for s in t["seals"] if s["found"]]
    with pytest.raises(ValueError, match="image 0, page 0: 65 seal candidates exceed the 64 a text page may hold"):
        pipeline.find_blocks([_rings(65)], [[pipeline.TextPage(seals="auto", seal_size=8)]])


def test_page_without_seal_colour_is_unchanged():
    from marconet_b200 import pipeline
    img = np.full((500, 700, 3), PAPER, np.uint8)
    paragraph(img, 30, 50, 8)
    a = pipeline.find_blocks([img], [[pipeline.TextPage(seals="auto")]])[0][0]
    b = pipeline.find_blocks([img], [[pipeline.TextPage()]])[0][0]
    assert a.pop("seals") == [] and a.pop("seal_size") == 41
    assert a == b


@pytest.mark.parametrize("rx, ry, rot", [(110, 110, 0.0), (130, 95, 0.0), (95, 125, -15.0)])
def test_restore_regions_equals_the_found_arcs_and_blocks(gpu_models, monkeypatch, rx, ry, rot):
    """A round stamp, and oval ones (the invoice stamp) whose arcs need more segments than a circle's."""
    from marconet_b200 import ops, pipeline
    monkeypatch.setattr(ops, "MODULE_GRAPHS", False)
    m = gpu_models["encoder"], gpu_models["tspgan"], gpu_models["sr"]
    img = contract_page(h=520, w=700, rx=rx, ry=ry, rot=rot)[0]
    pg = pipeline.TextPage(seals="auto")
    found = pipeline.find_blocks([img], [[pg]])[0][0]
    arcs = [s["region"] for s in found["seals"] if s["region"] is not None]
    assert len(arcs) == 1 and any(b.seals for b in found["blocks"])
    kw = dict(scale=2, feather=3, to_host=True)
    a = pipeline.restore_regions(*m, [img], [[pg]], **kw)[0]
    b = pipeline.restore_regions(*m, [img], [arcs + found["blocks"]], **kw)[0]
    np.testing.assert_array_equal(a["image"], b["image"])
    entry = a["regions"][0]
    assert {k: v for k, v in entry.items() if k not in ("regions", "seal_regions")} == found
    _same(entry["seal_regions"], b["regions"][:len(arcs)])
    _same(entry["regions"], b["regions"][len(arcs):])
    plain = np.full_like(img, PAPER)
    paragraph(plain, 40, 60, 5)
    c = pipeline.restore_regions(*m, [plain], [[pipeline.TextPage(seals="auto")]], **kw)[0]
    d = pipeline.restore_regions(*m, [plain], [[pipeline.TextPage()]], **kw)[0]
    np.testing.assert_array_equal(c["image"], d["image"])


def test_sealed_and_skewed_items_share_a_call():
    """A sealed page beside a skewed page in one find_blocks call, and a sealed block beside a skewed block in one find_lines
    call, give what each gives in a call of its own."""
    from marconet_b200 import ops, pipeline
    img = contract_page()[0]
    tilted = np.full((400, 700, 3), PAPER, np.uint8)
    paragraph(tilted, 40, 60, 8)
    tilted = cv2.warpAffine(tilted, cv2.getRotationMatrix2D((350, 200), 4.0, 1.0), (700, 400), borderValue=(PAPER,) * 3)
    sealed_pg, skewed_pg = pipeline.TextPage(seals="auto"), pipeline.TextPage(skew="auto")
    n0 = ops.LAUNCHES
    both = pipeline.find_blocks([img, tilted], [[sealed_pg], [skewed_pg]])
    assert ops.LAUNCHES - n0 == 7 + 6 * 24 + 6
    assert both[0][0] == pipeline.find_blocks([img], [[sealed_pg]])[0][0]
    assert both[1][0] == pipeline.find_blocks([tilted], [[skewed_pg]])[0][0]
    blk = pipeline.TextBlock((30, 270, 700, 450), seals=tuple(s["box"] for s in both[0][0]["seals"]))
    sk = pipeline.TextBlock((20, 30, 680, 330), skew="auto")
    n0 = ops.LAUNCHES
    mixed = pipeline.find_lines([img, tilted], [[blk], [sk]])
    assert ops.LAUNCHES - n0 == 6 + 1
    assert mixed[0][0] == pipeline.find_lines([img], [[blk]])[0][0] and len(mixed[0][0]["lines"]) == 5
    assert mixed[1][0] == pipeline.find_lines([tilted], [[sk]])[0][0]


def test_photographed_contract_through_flatten_pages():
    from marconet_b200 import pipeline
    page, box, _ = contract_page(h=700, w=900, over=False)
    h, w = page.shape[:2]
    H, W = int(h * 1.3), int(w * 1.3)
    dst = np.float32([[W * 0.10, H * 0.12], [W * 0.90, H * 0.09], [W * 0.88, H * 0.90], [W * 0.12, H * 0.88]])
    hom = cv2.getPerspectiveTransform(np.float32([[0, 0], [w, 0], [w, h], [0, h]]), dst)
    photo = cv2.warpPerspective(page, hom, (W, H), dst=np.full((H, W, 3), 40, np.uint8), flags=cv2.INTER_LINEAR,
                                borderMode=cv2.BORDER_TRANSPARENT)
    flat = pipeline.flatten_pages([photo], [[pipeline.FlatPage(quad="auto")]], to_host=True)[0][0]["image"]
    res = pipeline.find_blocks([np.ascontiguousarray(flat)], [[pipeline.TextPage(seals="auto")]])[0][0]
    assert len(res["seals"]) == 1
    t, boxes = S.page_seals(np.ascontiguousarray(flat))
    assert [s["box"] for s in res["seals"]] == boxes
