"""The image kernels at the edges of their contracts, bit for bit against the windowed references (test_image_edges.py pins those
against the whole-page twins and live cv2): destinations and pages past 2^31 bytes, 32767-pixel sources at s = 8, far maps,
perspective block widths, pitched views, chains of 64 regions, 65535 regions in one launch, and the refusals.

Each case is tagged with the features it reaches; the last test asserts that every REQUIRED feature was seen and every negative
control failed, and prints the kernel x feature table.  Large cases free their buffers before the next one and are skipped only
when torch.cuda.mem_get_info shows too little free memory."""
import collections

import numpy as np
import pytest
import torch

from oracle import curved_regions, image_ops, remap, warp_affine, warp_perspective
from test_gpu_curved_regions import _entry, _maps, _mixed_page

pytestmark = pytest.mark.gpu

SEEN = collections.defaultdict(collections.Counter)        # kernel -> feature -> cases
CONTROLS = {}                                               # control -> failed as it must
REQUIRED = {
    "resize": {"dst > 2^31 bytes", "32767 source", "cn=1", "cn=3", "cn=4", "pitched", "1x1", "1xN", "batch"},
    "warp_affine": {"dst > 2^31 bytes", "32767 source", "far map +", "far map -", "off the destination", "batch"},
    "warp_perspective": {"32767 source", "far map +", "far map -", "block widths", "batch"},
    "remap_curved": {"32767 source", "map near +2^14", "map near -2^14", "batch"},
    "composite": {"page > 2^31 bytes", "s = 8 far column", "page view", "page borders", "feather 0", "feather > region",
                  "chain >= 64", "65535 regions", "8 segments"},
    "refusal": {"65536 items", "32768-side warp source", "negative feather", "map the pipeline refuses", "65536 regions"},
}
GIB = 1 << 30


def _dev():
    return torch.device("cuda:0")


def _need(nbytes):
    free = torch.cuda.mem_get_info(_dev())[0]
    if free < nbytes + GIB:
        pytest.skip(f"needs {nbytes + GIB} free bytes of device memory, {free} free")


def _guarded(h, w, cn, guard=16, fill=0xA5):
    """A [h, w, cn] view of a buffer whose rows carry ``guard`` bytes past the pixels, every byte ``fill``."""
    buf = torch.full((h, w * cn + guard), fill, dtype=torch.uint8, device=_dev())
    return buf, buf[:, :w * cn].view(h, w, cn)


def _guards_intact(buf, w, cn, fill=0xA5):
    return bool((buf[:, w * cn:] == fill).all().item())


def _rows(view, rows):
    return view[torch.as_tensor(rows, device=_dev())].cpu().numpy()


# ---- resize --------------------------------------------------------------------------------------------------------------
def test_resize_destination_past_2_31_bytes():
    from marconet_b200 import ops
    H, W, s = 6144, 8192, 4
    _need(s * s * H * W * 3 + H * W * 3 + 64 * s * H)
    rng = np.random.default_rng(1)
    img = rng.integers(0, 256, (H, W, 3), dtype=np.uint8)
    src = torch.from_numpy(img).to(_dev())
    buf, dst = _guarded(s * H, s * W, 3)
    pitch = buf.stride(0)
    assert buf.numel() > 2 ** 31
    ops.resize_cubic([(src, dst)])
    k = 2 ** 31 // pitch
    rows = np.unique(np.concatenate([[0, s * H - 1, k - 1, k, k + 1], rng.choice(s * H, 64, replace=False)]))
    got = _rows(dst, rows)
    assert np.array_equal(got, image_ops.resize_cubic_rows(img, (s * W, s * H), rows))
    assert _guards_intact(buf, s * W, 3)
    SEEN["resize"]["dst > 2^31 bytes"] += 1
    del buf, dst, src
    torch.cuda.empty_cache()


@pytest.mark.parametrize("h, w", [(32767, 40), (40, 32767)])
def test_resize_of_32767_sources_at_s8(h, w):
    from marconet_b200 import ops
    s = 8
    rng = np.random.default_rng(h)
    img = rng.integers(0, 256, (h, w, 3), dtype=np.uint8)
    buf, dst = _guarded(s * h, s * w, 3)
    ops.resize_cubic([(torch.from_numpy(img).to(_dev()), dst)])
    rows = np.unique(np.concatenate([[0, 1, s * h - 2, s * h - 1], rng.choice(s * h, 64, replace=False)]))
    assert np.array_equal(_rows(dst, rows), image_ops.resize_cubic_rows(img, (s * w, s * h), rows))
    assert _guards_intact(buf, s * w, 3)
    if h > w:                            # the last 8 vector elements of every row: the split moved by 8 must fail
        cols = np.arange(s * w - 3, s * w)
        got = dst[:, -3:].cpu().numpy()
        assert np.array_equal(got, image_ops.resize_cubic_rows(img, (s * w, s * h), np.arange(s * h), cols))
        moved = image_ops.resize_cubic_rows(img, (s * w, s * h), np.arange(s * h), cols, split_shift=-8)
        CONTROLS["vector/tail split moved by 8"] = not np.array_equal(got, moved)
    SEEN["resize"]["32767 source"] += 1


def test_resize_batch_of_odd_shapes_and_pitches():
    from marconet_b200 import ops
    rng = np.random.default_rng(2)
    for cn in (1, 3, 4):
        shapes = [(1, 1, 5, 3), (1, 17, 3, 130), (9, 1, 40, 2), (23, 51, 92, 204), (40, 30, 13, 11), (7, 300, 61, 2049)]
        items, keep = [], []
        for h, w, dh, dw in shapes:
            img = rng.integers(0, 256, (h, w, cn), dtype=np.uint8)
            wide = torch.from_numpy(rng.integers(0, 256, (h, w + 5, cn), dtype=np.uint8)).to(_dev())
            wide[:, 2:2 + w] = torch.from_numpy(img).to(_dev())
            src = wide[:, 2:2 + w]                                       # a pitched view into a wider image
            buf, dst = _guarded(dh, dw, cn, guard=13)
            items.append((src, dst))
            keep.append((img, buf, dst, dh, dw))
        ops.resize_cubic(items)
        for img, buf, dst, dh, dw in keep:
            assert np.array_equal(dst.cpu().numpy(), image_ops.resize_cubic_rows(img, (dw, dh), np.arange(dh)))
            assert _guards_intact(buf, dw, cn)
        SEEN["resize"].update({f"cn={cn}": 1, "pitched": 1, "1x1": 1, "1xN": 1, "batch": 1})


# ---- rectify -------------------------------------------------------------------------------------------------------------
def _warp_check(kind, items):
    """items: (src numpy, dst shape (dh, dw), M or curve); one launch, every destination compared in full."""
    from marconet_b200 import ops
    srcs = [torch.from_numpy(s).to(_dev()) for s, _, _ in items]
    outs = [_guarded(dh, dw, s.shape[2], guard=11) for s, (dh, dw), _ in items]
    call = dict(warp_affine=ops.warp_affine, warp_perspective=ops.warp_perspective, remap_curved=ops.remap_curved)[kind]
    call([(sd, dst, m) for sd, (_, dst), (_, _, m) in zip(srcs, outs, items)])
    for (s, (dh, dw), m), (buf, dst) in zip(items, outs):
        if kind == "warp_affine":
            ref = warp_affine.warp_affine_cubic_u8(s, m, (dw, dh))
        elif kind == "warp_perspective":
            ref = warp_perspective.warp_perspective_cubic_u8(s, m, (dw, dh))
        else:
            ref = _remap_ref(s, m, dh, dw)
        assert np.array_equal(dst.cpu().numpy(), ref), (kind, s.shape, (dh, dw))
        assert _guards_intact(buf, dw, s.shape[2])


def _remap_ref(src, curve, dh, dw):
    from marconet_b200 import pipeline
    maps = pipeline.CurvedMaps((dw, dh), curve.c, 1.0, 1.0, 1, curve.top, curve.bottom, (), ())
    mx, my = curved_regions.crop_map(maps)
    return remap.remap_cubic_u8(src, mx, my)


def test_warp_affine_edges():
    rng = np.random.default_rng(3)
    tall = rng.integers(0, 256, (32767, 40, 3), dtype=np.uint8)
    wide = rng.integers(0, 256, (40, 32767, 3), dtype=np.uint8)
    small = rng.integers(0, 256, (61, 47, 4), dtype=np.uint8)[..., :3].copy()
    big = float(2 ** 20 - 1200)
    items = [(wide, (16, 300), [[1.0, 0.0, 32500.3], [0.0, 1.0, 12.7]]),
             (tall, (40, 64), [[0.0, 1.0, 0.4], [-1.0, 0.0, 32760.1]]),
             (small, (17, 1025), [[1.0, 0.0, big], [0.0, 1.0, -big]]),
             (small, (1, 63), [[-1.0, 0.0, -big + 64], [0.0, -1.0, big]]),
             (small, (15, 65), [[0.731, -0.412, 20.3], [0.388, 0.911, -3.7]]),
             (small, (16, 64), [[1.0 / 32, 0.01, 30.0], [-0.02, 1.0 / 32, 30.0]])]
    _warp_check("warp_affine", items)
    SEEN["warp_affine"].update({"32767 source": 1, "far map +": 1, "far map -": 1, "off the destination": 1, "batch": 1})


def test_warp_affine_destination_past_2_31_bytes():
    from marconet_b200 import ops
    dh, dw = 32768, 22000
    _need(dh * (dw * 3 + 16))
    rng = np.random.default_rng(4)
    img = rng.integers(0, 256, (300, 200, 3), dtype=np.uint8)
    m = [[200.0 / dw, 0.013, -2.3], [-0.0011, 300.0 / dh, 1.7]]
    buf, dst = _guarded(dh, dw, 3)
    assert buf.numel() > 2 ** 31
    ops.warp_affine([(torch.from_numpy(img).to(_dev()), dst, m)])
    k = 2 ** 31 // buf.stride(0)
    rows = np.unique(np.concatenate([[0, dh - 1, k - 1, k, k + 1], rng.choice(dh, 32, replace=False)]))
    xq, yq = warp_affine.warp_coords(m, np.arange(dw), rows)
    assert np.array_equal(_rows(dst, rows), warp_affine.warp_sample_u8(img, xq, yq))
    assert _guards_intact(buf, dw, 3)
    SEEN["warp_affine"]["dst > 2^31 bytes"] += 1
    del buf, dst
    torch.cuda.empty_cache()


def test_warp_perspective_edges():
    rng = np.random.default_rng(5)
    wide = rng.integers(0, 256, (40, 32767, 3), dtype=np.uint8)
    small = rng.integers(0, 256, (53, 71, 3), dtype=np.uint8)
    big = float(2 ** 24)
    items = [(wide, (16, 300), [[1.0, 0.0, 32500.3], [0.0, 1.0, 12.7], [1e-6, 2e-6, 1.0]]),
             (small, (16, 64), [[1.0, 0.0, big], [0.0, 1.0, -big], [0.0, 0.0, 1.0]]),
             (small, (17, 65), [[-1.0, 0.0, -big], [0.0, -1.0, big], [1e-9, 0.0, 1.0]])]
    for dh in (1, 15, 16, 17):
        for dw in (63, 64, 65, 1025):
            items.append((small, (dh, dw), [[71.0 / dw, 0.02, 0.3], [-0.01, 53.0 / dh, 0.1], [1e-3 / dw, 2e-3 / dh, 0.9]]))
    _warp_check("warp_perspective", items)
    SEEN["warp_perspective"].update({"32767 source": 1, "far map +": 1, "far map -": 1, "block widths": 1, "batch": 1})


def _line_curve(x0, y0, x1, y1, h, k):
    from marconet_b200.ops import CurveTable
    xs, ys = np.linspace(x0, x1, 3 * k + 1), np.linspace(y0, y1, 3 * k + 1)
    top = tuple((float(x), float(y)) for x, y in zip(xs, ys))
    bottom = tuple((float(x), float(y) + h) for x, y in zip(xs, ys))
    return CurveTable(1.0, tuple(np.linspace(0, 1, k + 1)), top, bottom)


def test_remap_curved_edges():
    rng = np.random.default_rng(6)
    wide = rng.integers(0, 256, (40, 32767, 3), dtype=np.uint8)
    lim = 2.0 ** 14 - 2
    items = [(wide, (30, 300), _line_curve(lim - 300, 3, lim, 9, 20, 3)),
             (wide, (10, 80), _line_curve(-lim, 3, -lim + 80, 3, 8, 1)),
             (wide, (64, 64), _line_curve(100.3, -lim + 5, 180.7, -lim + 9, 30, 8))]
    _warp_check("remap_curved", items)
    SEEN["remap_curved"].update({"32767 source": 1, "map near +2^14": 1, "map near -2^14": 1, "batch": 1})


# ---- composites ----------------------------------------------------------------------------------------------------------
KERNEL = {"rect": "composite_regions", "oriented": "composite_regions_affine", "quad": "composite_regions_quad",
          "curved": "composite_regions_curved"}


def _kind_filter(regs, kind):
    from marconet_b200.pipeline import CurvedRegion, OrientedRegion, QuadRegion
    keep = dict(rect=(), oriented=(OrientedRegion,), quad=(OrientedRegion, QuadRegion),
                curved=(OrientedRegion, QuadRegion, CurvedRegion))[kind]
    return [r for r in regs if isinstance(r, keep) or not isinstance(r, (OrientedRegion, QuadRegion, CurvedRegion))]


def _compose_and_check(kind, page, HW, regs, s, feather, rng, windows_of=None, control=None):
    """One composite launch of ``kind`` over the device page (a view) for regions of a source image of HW, exactly as
    restore_regions calls it; each region's footprint box padded by 2 compared with compose_window over the device's own
    background bytes, everything outside every box byte-equal to the background.  Returns the plan."""
    from marconet_b200 import ops, pipeline
    plan = pipeline.plan_regions([HW], [regs], scale=s, feather=feather)
    ok = list(range(len(plan)))
    maps = [_maps(p, s, None) for p in plan]
    srs = [rng.integers(0, 256, (128, m.t_width, 3) if m is not None else (int(rng.integers(4, 40)), int(rng.integers(4, 90)), 3),
                        dtype=np.uint8) for m in maps]
    ts = [torch.from_numpy(t).to(_dev()) for t in srs]
    chains = pipeline.region_chains(plan, ok)
    ph, pw = page.shape[:2]
    boxes = [(max(0, p.out[0] - 2), max(0, p.out[1] - 2), min(pw, p.out[2] + 2), min(ph, p.out[3] + 2)) for p in plan]
    before = {b: page[b[1]:b[3], b[0]:b[2]].cpu().numpy() for b in set(boxes)}
    saved = page.clone()
    items = [(page, ts[k], plan[k].out, chain) for k, chain in zip(ok, chains)]
    if kind == "rect":
        ops.composite_regions(items, feather)
    else:
        getattr(ops, KERNEL[kind])([it + (_entry(m, s),) for it, m in zip(items, maps)], feather)
    after = {b: page[b[1]:b[3], b[0]:b[2]].cpu().numpy() for b in set(boxes)}
    for k, b in enumerate(boxes):
        near = [j for j, p in enumerate(plan) if max(b[0], p.out[0]) < min(b[2], p.out[2]) and max(b[1], p.out[1]) < min(b[3], p.out[3])]
        ref = curved_regions.compose_window(before[b], b[:2], (ph, pw), [regs[j] for j in near], [srs[j] for j in near], s,
                                            feather)
        assert np.array_equal(after[b], ref), (kind, k, regs[k], b)
        if control is not None and k == control[0]:
            CONTROLS[control[1]] = not np.array_equal(after[b], control[2](before[b], b[:2], (ph, pw), [regs[j] for j in near],
                                                                             [srs[j] for j in near], s, feather))
    for b in boxes:                                  # the boxes put back: every other byte must be the background's
        page[b[1]:b[3], b[0]:b[2]] = saved[b[1]:b[3], b[0]:b[2]]
    assert torch.equal(page, saved)
    del saved
    return plan


def _page_for(img, s, pitch_extra=0):
    """The device background of img at scale s (ops.resize_cubic; test_resize_* check those bytes), as a view into a buffer
    ``pitch_extra`` pixels wider."""
    from marconet_b200 import ops
    H, W = img.shape[:2]
    buf = torch.zeros((s * H, s * W + pitch_extra, 3), dtype=torch.uint8, device=_dev())
    page = buf[:, :s * W]
    ops.resize_cubic([(torch.from_numpy(img).to(_dev()), page)])
    return buf, page


@pytest.mark.parametrize("kind", ["rect", "oriented", "quad", "curved"])
@pytest.mark.parametrize("feather", [0, 5, 400])
def test_composite_mixed_page_as_a_view(kind, feather):
    rng = np.random.default_rng(hash((kind, feather)) % 2 ** 32)
    H, W, s = 40, 70, 4
    img = rng.integers(0, 256, (H, W, 3), dtype=np.uint8)
    _, page = _page_for(img, s, pitch_extra=7)
    regs = _kind_filter(_mixed_page(rng, H, W), kind)
    regs += [(0, 0, 3, 2), (W - 4, H - 3, W, H), (0, H - 5, W, H)]                 # every page border, and all of them
    _compose_and_check(kind, page, (H, W), regs, s, feather, rng)
    SEEN["composite"].update({"page view": 1, "page borders": 1, "feather 0" if feather == 0 else "feather > region"
                              if feather == 400 else "feather 5": 1})


def _far_regs(H, W, rng):
    from marconet_b200.pipeline import CurvedRegion, OrientedRegion, QuadRegion
    x = W - 60.0
    regs = [(W - 50, 2, W, 30), OrientedRegion.from_rotated(x + 20, 30, 70, 16, 8), QuadRegion((x, 36), (W - 2, 34), (W - 3, 52),
                                                                                               (x + 2, 50))]
    xs = np.linspace(16220.0, 16370.0, 25)          # a curved crop map stays below 2^14: as far right as it may go
    top = tuple((float(v), 12.0 + 3 * np.sin(v / 9)) for v in xs)
    regs.append(CurvedRegion(top, tuple((a, b + 14) for a, b in top)))             # 8 segments, past page column 2^17
    regs.append(OrientedRegion.from_rotated(W - 8, H - 6, 14, 10, 135))              # past the far corner, clipped
    return regs


def test_composite_s8_far_column_of_a_32767_wide_image():
    rng = np.random.default_rng(8)
    H, W, s = 64, 32767, 8
    img = rng.integers(0, 256, (H, W, 3), dtype=np.uint8)
    _, page = _page_for(img, s)
    regs = _far_regs(H, W, rng)
    assert len(regs[3].top) == 25
    def no_border_alpha(bg, origin, page_hw, rects, srs, s_, f):
        return curved_regions.compose_window(bg, origin, (10 ** 7, 10 ** 7), rects, srs, s_, f)
    _compose_and_check("curved", page, (H, W), regs, s, 6, rng, control=(0, "alpha ignoring page borders", no_border_alpha))
    SEEN["composite"].update({"s = 8 far column": 1, "8 segments": 1})


def test_composite_on_a_page_past_2_31_bytes():
    H, W, s = 6144, 8192, 4
    _need(s * s * H * W * 3 + H * W * 3)
    rng = np.random.default_rng(9)
    img = rng.integers(0, 256, (H, W, 3), dtype=np.uint8)
    buf, page = _page_for(img, s)
    y = H - 100
    from marconet_b200.pipeline import CurvedRegion, OrientedRegion, QuadRegion
    regs = [(r + 10, y, r + 60, y + 20) for r in range(0, 600, 200)]
    regs += [OrientedRegion.from_rotated(W - 100, y, 120, 20, 11), QuadRegion((W - 300, y - 10), (W - 200, y - 14),
                                                                               (W - 198, y + 12), (W - 301, y + 10)),
             CurvedRegion.from_arc(W - 600, H - 40, 80, 60, 150, 30), (W - 40, H - 20, W, H)]
    assert s * (y - 20) * s * W * 3 > 2 ** 31
    _compose_and_check("curved", page, (H, W), regs, s, 8, rng)
    SEEN["composite"]["page > 2^31 bytes"] += 1
    del buf, page
    torch.cuda.empty_cache()


def test_composite_chain_of_64_mixed_regions():
    from marconet_b200.pipeline import CurvedRegion, OrientedRegion, QuadRegion
    rng = np.random.default_rng(10)
    H, W, s = 60, 90, 2
    img = rng.integers(0, 256, (H, W, 3), dtype=np.uint8)
    _, page = _page_for(img, s)
    regs = []
    for i in range(66):
        cx, cy = 45 + rng.uniform(-6, 6), 30 + rng.uniform(-5, 5)
        k = i % 4
        if k == 0:
            regs.append((int(cx) - 12, int(cy) - 6, int(cx) + 10, int(cy) + 5))
        elif k == 1:
            regs.append(OrientedRegion.from_rotated(cx, cy, rng.uniform(10, 30), rng.uniform(4, 10), rng.uniform(-180, 180)))
        elif k == 2:
            regs.append(QuadRegion((cx - 12, cy - 5), (cx + 12, cy - 7), (cx + 13, cy + 6), (cx - 11, cy + 5)))
        else:
            regs.append(CurvedRegion.from_arc(cx, cy + 20, 26, 18, 120, 60))

    def reversed_chain(bg, origin, page_hw, rects, srs, s_, f):
        return curved_regions.compose_window(bg, origin, page_hw, rects[::-1], srs[::-1], s_, f)
    plan = _compose_and_check("curved", page, (H, W), regs, s, 3, rng, control=(65, "chain order reversed", reversed_chain))
    from marconet_b200 import pipeline
    assert max(len(c) for c in pipeline.region_chains(plan, list(range(len(plan))))) >= 64
    SEEN["composite"]["chain >= 64"] += 1


def test_composite_65535_regions_in_one_launch():
    from marconet_b200 import ops
    rng = np.random.default_rng(11)
    H, W, s = 512, 1024, 1
    img = rng.integers(0, 256, (H, W, 3), dtype=np.uint8)
    _, page = _page_for(img, s)
    rects = [(x, y, x + 2, y + 3) for y in range(0, 512, 4) for x in range(0, 1024, 2)][:65535]     # s = 1: out = rect
    srs = rng.integers(0, 256, (65535, 2, 3, 3), dtype=np.uint8)
    ts = torch.from_numpy(srs).to(_dev())
    before = page.cpu().numpy()
    chains = [[k] for k in range(65535)]
    launches = ops.LAUNCHES
    ops.composite_regions([(page, ts[k], rects[k], chains[k]) for k in range(65535)], 1)
    assert ops.LAUNCHES == launches + 1
    got = page.cpu().numpy()
    for row in (0, 1, 64, 127):                  # whole rows of regions: one window per 4 source rows
        y = 4 * row
        ks = [k for k in range(row * 512, min(65535, row * 512 + 512))]
        ref = curved_regions.compose_window(before[y:y + 4], (0, y), (H, W), [rects[k] for k in ks], [srs[k] for k in ks], s, 1)
        assert np.array_equal(got[y:y + 4], ref), row
    assert np.array_equal(got[508:, 1022:], before[508:, 1022:])    # the 65536th slot holds no region
    SEEN["composite"]["65535 regions"] += 1


def test_perspective_block_width_control():
    """Negative control: the twin with 32-column block origins fails on a destination wider than a block (the block origin
    moves a few fixed-point coordinates by one 1/32 step; the source is large enough that those pixels read real bytes)."""
    from marconet_b200 import ops
    src = np.random.default_rng(5).integers(0, 256, (120, 1200, 3), dtype=np.uint8)
    m = np.array([[0.9, 0.05, 3.3], [-0.04, 1.1, 2.2], [3e-4, -2e-4, 1.0]]) * np.float64(1 / 3)
    dh, dw = 100, 2049
    buf, dst = _guarded(dh, dw, 3)
    ops.warp_perspective([(torch.from_numpy(src).to(_dev()), dst, m)])
    got = dst.cpu().numpy()
    assert np.array_equal(got, warp_perspective.warp_perspective_cubic_u8(src, m, (dw, dh)))
    with pytest.MonkeyPatch.context() as mp:
        mp.setattr(warp_perspective, "block_width", lambda d: 32)
        bad = warp_perspective.warp_perspective_cubic_u8(src, m, (dw, dh))
    CONTROLS["perspective block width 32"] = not np.array_equal(got, bad)


def test_fp64_fx_control():
    """Negative control: past column 2^17 at a non-integer scale, taps from an fp64 fx fail the resize comparison."""
    from marconet_b200 import ops
    from test_image_edges import taps_fp64
    rng = np.random.default_rng(13)
    img = rng.integers(0, 256, (40, 32767, 3), dtype=np.uint8)
    dh, dw = 301, 250001
    buf, dst = _guarded(dh, dw, 3)
    ops.resize_cubic([(torch.from_numpy(img).to(_dev()), dst)])
    rows = np.array([0, 150, 300])
    got = _rows(dst, rows)
    assert np.array_equal(got, image_ops.resize_cubic_rows(img, (dw, dh), rows))
    with pytest.MonkeyPatch.context() as mp:
        mp.setattr(image_ops, "taps_at", taps_fp64)
        CONTROLS["fp32 fx rounding done in fp64"] = not np.array_equal(got, image_ops.resize_cubic_rows(img, (dw, dh), rows))


# ---- refusals ------------------------------------------------------------------------------------------------------------
def test_refusals_before_any_launch(gpu_models, monkeypatch):
    from marconet_b200 import ops, pipeline
    before = ops.LAUNCHES
    t = torch.zeros((4, 4, 3), dtype=torch.uint8, device=_dev())
    with pytest.raises(ValueError, match="at most 65535"):
        ops.resize_cubic([(t, t)] * 65536)
    with pytest.raises(ValueError, match="at most 65535"):
        ops.composite_regions([(t, t, (0, 0, 1, 1), [0])] * 65536, 0)
    SEEN["refusal"]["65536 items"] += 1
    tall = torch.zeros((32768, 1, 3), dtype=torch.uint8, device=_dev())
    with pytest.raises(ValueError, match="32768x1 source exceeds OpenCV's int16 source coordinates"):
        ops.warp_affine([(tall, t, [[1, 0, 0], [0, 1, 0]])])
    with pytest.raises(ValueError, match="32768x1 source exceeds OpenCV's int16 source coordinates"):
        ops.warp_perspective([(tall, t, [[1, 0, 0], [0, 1, 0], [0, 0, 1]])])
    with pytest.raises(ValueError, match="32768x1 source exceeds OpenCV's int16 source coordinates"):
        ops.remap_curved([(tall, t, _line_curve(0, 0, 3, 0, 3, 1))])
    SEEN["refusal"]["32768-side warp source"] += 1
    with pytest.raises(ValueError, match="feather -1 < 0"):
        ops.composite_regions([(t, t, (0, 0, 1, 1), [0])], -1)
    SEEN["refusal"]["negative feather"] += 1
    with pytest.raises(ValueError, match="exceeds OpenCV's 32-bit fixed-point coordinates"):
        pipeline.restore_regions(gpu_models["encoder"], gpu_models["tspgan"], gpu_models["sr"], [np.zeros((64, 32767, 3), np.uint8)],
                                 [[pipeline.OrientedRegion.from_rotated(32700, 60, 40, 1.5, 3)]], scale=8)
    SEEN["refusal"]["map the pipeline refuses"] += 1
    assert ops.LAUNCHES == before

    # a call whose blocks split into more than 65535 lines stops after the layout, before any model runs
    calls = []
    monkeypatch.setattr(pipeline, "_find_lines", lambda dimg, items, rq=None: [
        dict(lines=[(x, y, x + 1, y + 1) for y in range(b[2][1], b[2][1] + 16) for x in range(b[2][0], b[2][0] + 16)],
             threshold=0, ink=0) for b in items])
    monkeypatch.setattr(pipeline, "restore_images", lambda *a, **k: calls.append(1))
    blocks = [pipeline.TextBlock((16 * i, 0, 16 * i + 16, 16)) for i in range(257)]
    with pytest.raises(ValueError, match="65792 regions in one call"):
        pipeline.restore_regions(gpu_models["encoder"], gpu_models["tspgan"], gpu_models["sr"],
                                 [np.zeros((16, 16 * 257, 3), np.uint8)], [blocks], scale=1)
    assert ops.LAUNCHES == before and not calls
    SEEN["refusal"]["65536 regions"] += 1


# ---- coverage ------------------------------------------------------------------------------------------------------------
def test_coverage_and_negative_controls():
    feats = sorted({f for v in SEEN.values() for f in v} | {f for v in REQUIRED.values() for f in v})
    print("\nkernel x feature: cases")
    for k in REQUIRED:
        print(f"  {k:18s} " + "  ".join(f"{f}={SEEN[k][f]}" for f in feats if f in REQUIRED[k] or SEEN[k][f]))
    print("negative controls (failed as they must):", CONTROLS)
    for k, want in REQUIRED.items():
        assert want <= {f for f, n in SEEN[k].items() if n}, (k, want - set(SEEN[k]))
    assert set(CONTROLS) == {"vector/tail split moved by 8", "perspective block width 32", "fp32 fx rounding done in fp64",
                             "alpha ignoring page borders", "chain order reversed"}, CONTROLS
    assert all(CONTROLS.values()), CONTROLS
