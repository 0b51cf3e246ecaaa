"""The image kernels' references at the edges of their contracts, on the CPU.

  - the windowed references (oracle.image_ops.resize_cubic_rows and the compose_window of each region twin) equal the whole-page
    ones on small pages of every region kind, for windows at the corners, on the borders and across footprints;
  - the restatements equal live cv2 (IPP off) at the extremes the kernels accept: 32767-pixel sources resized at s = 8, warps
    whose fixed-point coordinates approach their documented bounds, perspective block widths around 64 and remap maps near
    +-2^14;
  - the maps the planner accepts at its own limits (32767-pixel sides, s = 8, regions at the far corner, the largest angles,
    foreshortening 4, curved maps near 2^14) keep the fixed-point values the kernels form inside those bounds;
  - a restore_regions call of more than 65535 regions is refused before anything runs on the device."""
import math

import numpy as np
import pytest

from oracle import curved_regions, image_ops, oriented_regions, quad_regions, regions, remap, warp_affine, warp_perspective
from test_gpu_curved_regions import _curved, _mixed_page


@pytest.fixture
def cv2_no_ipp():
    import cv2
    was = cv2.ipp.useIPP()
    cv2.ipp.setUseIPP(False)
    yield cv2
    cv2.ipp.setUseIPP(was)


# ---- windowed references ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("cn", [1, 3, 4])
def test_resize_rows_equal_whole_resize(cn):
    rng = np.random.default_rng(cn)
    for h, w, dh, dw in [(1, 1, 1, 1), (1, 1, 7, 5), (1, 13, 8, 104), (9, 1, 36, 3), (23, 51, 92, 204), (17, 29, 40, 33),
                         (40, 30, 13, 11)]:
        img = rng.integers(0, 256, (h, w, cn), dtype=np.uint8)
        whole = image_ops.resize_cubic_u8(img, dw / w, dh / h)
        assert np.array_equal(image_ops.resize_cubic_rows(img, (dw, dh), np.arange(dh)), whole)
        rows, cols = np.sort(rng.choice(dh, min(dh, 5), replace=False)), np.sort(rng.choice(dw, min(dw, 7), replace=False))
        assert np.array_equal(image_ops.resize_cubic_rows(img, (dw, dh), rows, cols), whole[rows][:, cols])


def _windows(page_hw, boxes):
    """Windows (x0, y0, x1, y1) of a page: its four corners, a strip along each border, the whole page and, for each footprint
    box, windows centred on its corners and one inside it."""
    H, W = page_hw
    out = [(0, 0, 9, 7), (W - 9, 0, W, 7), (0, H - 7, 9, H), (W - 9, H - 7, W, H), (0, 0, W, 3), (0, H - 3, W, H),
           (0, 0, 4, H), (W - 4, 0, W, H), (0, 0, W, H)]
    for x0, y0, x1, y1 in boxes:
        for cx, cy in ((x0, y0), (x1, y0), (x0, y1), (x1, y1), ((x0 + x1) // 2, (y0 + y1) // 2)):
            out.append((max(0, cx - 6), max(0, cy - 5), min(W, cx + 7), min(H, cy + 4)))
    return out


@pytest.mark.parametrize("twin, kinds", [(regions, "rect"), (oriented_regions, "oriented"), (quad_regions, "quad"),
                                         (curved_regions, "curved")])
@pytest.mark.parametrize("s, feather", [(1, 0), (2, 3), (3, 200)])
def test_compose_window_equals_compose(twin, kinds, s, feather):
    from marconet_b200 import pipeline
    rng = np.random.default_rng(7 * s + feather)
    H, W = 23, 51
    regs = _mixed_page(rng, H, W)
    keep = dict(rect=(), oriented=(pipeline.OrientedRegion,), quad=(pipeline.OrientedRegion, pipeline.QuadRegion),
                curved=(pipeline.OrientedRegion, pipeline.QuadRegion, pipeline.CurvedRegion))[kinds]
    regs = [r for r in regs if isinstance(r, keep) or not isinstance(r, (pipeline.OrientedRegion, pipeline.QuadRegion,
                                                                         pipeline.CurvedRegion))]
    plan = pipeline.plan_regions([(H, W)], [regs], scale=s, feather=feather)
    srs = [rng.integers(0, 256, (int(rng.integers(8, 40)), int(rng.integers(8, 60)), 3), dtype=np.uint8) for _ in regs]
    srs[int(rng.integers(len(srs)))] = None                 # a failed region keeps the background
    img = rng.integers(0, 256, (H, W, 3), dtype=np.uint8)
    whole = twin.compose(img, regs, srs, s, feather)
    bg = regions.background(img, s)
    page_hw = bg.shape[:2]
    for x0, y0, x1, y1 in _windows(page_hw, [p.out for p in plan]):
        got = twin.compose_window(bg[y0:y1, x0:x1], (x0, y0), page_hw, regs, srs, s, feather)
        assert np.array_equal(got, whole[y0:y1, x0:x1]), (x0, y0, x1, y1)


def test_compose_window_alpha_counts_page_borders():
    """A rectangle on the page's far corner feathers only its inner sides: the window at the corner takes the page's sides from
    page_hw, not from the window.  Negative control: an alpha that ignores the page border fails the comparison."""
    rng = np.random.default_rng(3)
    img = rng.integers(0, 256, (20, 30, 3), dtype=np.uint8)
    t = rng.integers(0, 256, (16, 24, 3), dtype=np.uint8)
    bg = regions.background(img, 2)
    whole = regions.compose(img, [(0, 0, 12, 9)], [t], 2, 6)
    got = regions.compose_window(bg[:6, :6], (0, 0), bg.shape[:2], [(0, 0, 12, 9)], [t], 2, 6)
    assert np.array_equal(got, whole[:6, :6])
    got = regions.compose_window(bg[-6:, -6:], (54, 34), bg.shape[:2], [(18, 12, 30, 20)], [t], 2, 6)
    whole = regions.compose(img, [(18, 12, 30, 20)], [t], 2, 6)
    assert np.array_equal(got, whole[-6:, -6:])
    wrong = regions.compose_window(bg[-6:, -6:], (54, 34), (10 ** 6, 10 ** 6), [(18, 12, 30, 20)], [t], 2, 6)
    assert not np.array_equal(wrong, whole[-6:, -6:])


# ---- the restatements against live cv2 at the extremes ---------------------------------------------------------------
def _sample_rows(rng, n, k=24):
    return np.unique(np.concatenate([[0, 1, n // 2, n - 2, n - 1], rng.choice(n, min(n, k), replace=False)]))


@pytest.mark.parametrize("h, w, dsize", [(32767, 40, (320, 262136)), (40, 32767, (262136, 320)), (40, 32767, (250001, 301)),
                                         (32767, 3, (7, 262133))])
def test_resize_of_32767_sources_equals_cv2(cv2_no_ipp, h, w, dsize):
    rng = np.random.default_rng(h + w)
    img = rng.integers(0, 256, (h, w, 3), dtype=np.uint8)
    ref = cv2_no_ipp.resize(img, dsize, interpolation=cv2_no_ipp.INTER_CUBIC)
    rows = _sample_rows(rng, dsize[1])
    assert np.array_equal(image_ops.resize_cubic_rows(img, dsize, rows), ref[rows])
    if dsize == (320, 262136):           # every row's last 8 vector elements: the split moved by 8 must show (negative control)
        cols = np.arange(317, 320)
        assert np.array_equal(image_ops.resize_cubic_rows(img, dsize, np.arange(dsize[1]), cols), ref[:, cols])
        moved = image_ops.resize_cubic_rows(img, dsize, np.arange(dsize[1]), cols, split_shift=-8)
        assert not np.array_equal(moved, ref[:, cols])
    if dsize == (250001, 301):           # past column 2^17 fx keeps ~7 fraction bits in fp32 (at s = 8 it is exact): fp64 must show
        with pytest.MonkeyPatch.context() as mp:
            mp.setattr(image_ops, "taps_at", taps_fp64)
            assert not np.array_equal(image_ops.resize_cubic_rows(img, dsize, rows), ref[rows])


def taps_fp64(ds, scale):
    """image_ops.taps_at with fx kept in fp64 until the tap quantisation (negative control of the fp32 rounding)."""
    ds = np.asarray(ds, np.int64)
    f = (ds + 0.5) * scale - 0.5
    s = np.floor(f)
    c = image_ops.cubic_coeffs((f - s).astype(np.float32))
    return s.astype(np.int64), np.rint(c * np.float32(image_ops.COEF_SCALE)).astype(np.int64).T.reshape(len(ds), 4)


def _cubic_flags(cv2):
    return cv2.INTER_CUBIC | cv2.WARP_INVERSE_MAP


@pytest.mark.parametrize("dh, dw", [(1, 63), (15, 64), (16, 65), (17, 1025), (16, 64), (40, 300)])
def test_warp_affine_near_the_bounds_equals_cv2(cv2_no_ipp, dh, dw):
    rng = np.random.default_rng(dh * dw)
    src = rng.integers(0, 256, (61, 47, 3), dtype=np.uint8)
    big = float(2 ** 20 - dw - 64)
    for m in ([[1.0, 0.0, big], [0.0, 1.0, -big]],                 # far outside: every pixel replicated from a corner
              [[-1.0, 0.0, -big + 2 * dw], [0.0, -1.0, big]],
              [[0.731, -0.412, 20.3], [0.388, 0.911, -3.7]],
              [[700.25 / dw, 0.0, -3.1], [0.0, 63.0 / dh, 0.43]],   # a zoom that spans the source
              [[1.0 / 32, 0.01, 30.0], [-0.02, 1.0 / 32, 30.0]]):
        ref = cv2_no_ipp.warpAffine(src, np.asarray(m), (dw, dh), flags=_cubic_flags(cv2_no_ipp),
                                    borderMode=cv2_no_ipp.BORDER_REPLICATE)
        assert np.array_equal(warp_affine.warp_affine_cubic_u8(src, m, (dw, dh)), ref.reshape(dh, dw, 3)), m


@pytest.mark.parametrize("dh", [1, 15, 16, 17])
@pytest.mark.parametrize("dw", [63, 64, 65, 1025])
def test_warp_perspective_block_widths_equal_cv2(cv2_no_ipp, dh, dw):
    rng = np.random.default_rng(dh * 1000 + dw)
    src = rng.integers(0, 256, (53, 71, 3), dtype=np.uint8)
    big = float(2 ** 24)
    for m in ([[0.9, 0.05, 3.3], [-0.04, 1.1, 2.2], [3e-4, -2e-4, 1.0]],
              [[71.0 / dw, 0.0, 0.0], [0.0, 53.0 / dh, 0.0], [1e-3 / dw, 2e-3 / dh, 0.9]],
              [[1.0, 0.0, big], [0.0, 1.0, -big], [0.0, 0.0, 1.0]],            # far outside, 32 X / W near 2^29
              [[-1.0, 0.0, -big], [0.0, -1.0, big], [1e-9, 0.0, 1.0]]):
        ref = cv2_no_ipp.warpPerspective(src, np.asarray(m), (dw, dh), flags=_cubic_flags(cv2_no_ipp),
                                         borderMode=cv2_no_ipp.BORDER_REPLICATE)
        got = warp_perspective.warp_perspective_cubic_u8(src, m, (dw, dh))
        assert np.array_equal(got, ref.reshape(dh, dw, 3)), m


def test_perspective_block_width_matters(cv2_no_ipp):
    """Negative control: block origins 32 columns apart instead of 64 give other bytes."""
    src = np.random.default_rng(5).integers(0, 256, (53, 71, 3), dtype=np.uint8)
    m = np.array([[0.9, 0.05, 3.3], [-0.04, 1.1, 2.2], [3e-4, -2e-4, 1.0]]) * np.float64(1 / 3)
    dsize = (1025, 17)
    ref = cv2_no_ipp.warpPerspective(src, m, dsize, flags=_cubic_flags(cv2_no_ipp), borderMode=cv2_no_ipp.BORDER_REPLICATE)
    xq, yq = warp_perspective.warp_coords(m, np.arange(1025), np.arange(17), dsize)
    assert np.array_equal(warp_affine.warp_sample_u8(src, xq, yq), ref)
    with pytest.MonkeyPatch.context() as mp:
        mp.setattr(warp_perspective, "block_width", lambda d: 32)
        xq2, yq2 = warp_perspective.warp_coords(m, np.arange(1025), np.arange(17), dsize)
    assert not (np.array_equal(xq2, xq) and np.array_equal(yq2, yq))


@pytest.mark.parametrize("w", [64, 32766])
def test_remap_near_2_14_equals_cv2(cv2_no_ipp, w):
    rng = np.random.default_rng(w)
    src = rng.integers(0, 256, (37, w, 3), dtype=np.uint8)
    lim = 2.0 ** 14 - 1
    mx = np.concatenate([rng.uniform(lim - 40, lim, (9, 30)), rng.uniform(-lim, -lim + 40, (9, 30)),
                         np.round(rng.uniform(lim - 40, lim, (9, 30)) * 64) / 64]).astype(np.float32)
    my = np.concatenate([rng.uniform(-3, 40, (18, 30)), rng.uniform(-lim, lim, (9, 30))]).astype(np.float32)
    ref = cv2_no_ipp.remap(src, mx, my, cv2_no_ipp.INTER_CUBIC, borderMode=cv2_no_ipp.BORDER_REPLICATE)
    assert np.array_equal(remap.remap_cubic_u8(src, mx, my), ref)


def test_32767_sources_are_cv2_shifted_by_one_pixel(cv2_no_ipp):
    """cv2's warps and remap assert every source side below SHRT_MAX = 32767, yet the kernels and the planner take 32767 (the
    int16 coordinates cannot saturate there either).  What they compute there is OpenCV's arithmetic: on a 32767-wide source
    the restatements equal cv2 on the 32766-wide crop without column 0 under the map moved one pixel left, for maps that read the
    far columns (every fixed-point step is exact, so the shift moves Xq by exactly 32)."""
    from marconet_b200 import pipeline
    rng = np.random.default_rng(32767)
    src = rng.integers(0, 256, (9, 32767, 3), dtype=np.uint8)
    crop = np.ascontiguousarray(src[:, 1:])
    with pytest.raises(cv2_no_ipp.error, match="SHRT_MAX"):
        cv2_no_ipp.warpAffine(src, np.eye(2, 3), (8, 4), flags=_cubic_flags(cv2_no_ipp), borderMode=cv2_no_ipp.BORDER_REPLICATE)
    dw, dh = 300, 7
    for tx in (32480.40625, 32600.0, 32766.96875):          # up to and past the far border (replicated)
        m = np.array([[1.0, 0.0, tx], [0.0, 1.0, 0.25]])
        ref = cv2_no_ipp.warpAffine(crop, m - [[0, 0, 1], [0, 0, 0]], (dw, dh), flags=_cubic_flags(cv2_no_ipp),
                                    borderMode=cv2_no_ipp.BORDER_REPLICATE)
        assert np.array_equal(warp_affine.warp_affine_cubic_u8(src, m, (dw, dh)), ref), tx
        m3 = np.vstack([m, [0.0, 0.0, 1.0]])
        ref = cv2_no_ipp.warpPerspective(crop, m3 - [[0, 0, 1], [0, 0, 0], [0, 0, 0]], (dw, dh),
                                         flags=_cubic_flags(cv2_no_ipp), borderMode=cv2_no_ipp.BORDER_REPLICATE)
        assert np.array_equal(warp_perspective.warp_perspective_cubic_u8(src, m3, (dw, dh)), ref), tx
    mx = (np.round(rng.uniform(32400, 32800, (7, 40)) * 64) / 64).astype(np.float32)
    my = (np.round(rng.uniform(-2, 10, (7, 40)) * 64) / 64).astype(np.float32)
    ref = cv2_no_ipp.remap(crop, mx - np.float32(1), my, cv2_no_ipp.INTER_CUBIC, borderMode=cv2_no_ipp.BORDER_REPLICATE)
    assert np.array_equal(remap.remap_cubic_u8(src, mx, my), ref)
    regs = [pipeline.OrientedRegion.from_rotated(32000, 20, 40, 30, 10),
            pipeline.QuadRegion(*[(32000 + x, y) for x, y in ((0, 5), (40, 5), (40, 35), (0, 35))]),
            pipeline.CurvedRegion(tuple((16000.0 + 10 * k, 5.0) for k in range(4)), tuple((16000.0 + 10 * k, 35.0) for k in range(4)))]
    pipeline.plan_regions([(40, 32767)], [regs], scale=1)
    for r in regs:
        with pytest.raises(ValueError, match="image 32768x40 exceeds 32767"):
            pipeline.plan_regions([(40, 32768)], [[r]], scale=1)


# ---- the planner's maps at its limits --------------------------------------------------------------------------------
def _affine_extremes(m, box):
    """max |X0|, max |adelta| and max |X0 + adelta| over the box, in 1/1024 pixel, from the kernels' formula in fp64."""
    x0, y0, x1, y1 = box
    xs, ys = np.arange(x0, x1, dtype=np.float64), np.arange(y0, y1, dtype=np.float64)
    worst = [0, 0, 0]
    for r in np.asarray(m, np.float64):
        row = np.rint((r[1] * ys + r[2]) * 1024) + 16
        delta = np.rint(r[0] * xs * 1024)
        s = max(abs(row.max() + delta.max()), abs(row.min() + delta.min()), abs(row.max() + delta.min()),
                abs(row.min() + delta.max()))
        worst = [max(worst[0], np.abs(row).max()), max(worst[1], np.abs(delta).max()), max(worst[2], s)]
    return worst


def _perspective_extremes(n, box, page_hw):
    """max |fX|, |fY| (before the clamp) over the box's border pixels, block origins counted from the page's column 0."""
    x0, y0, x1, y1 = box
    H, W = page_hw
    bw = warp_perspective.block_width((W, H))
    n = np.asarray(n, np.float64)
    pts = [(x, y) for x in range(x0, x1) for y in (y0, y1 - 1)] + [(x, y) for x in (x0, x1 - 1) for y in range(y0, y1)]
    xs, ys = np.array([p[0] for p in pts]), np.array([p[1] for p in pts], np.float64)
    xb, x1_ = (xs - xs % bw).astype(np.float64), (xs % bw).astype(np.float64)
    row = [n[r, 0] * xb + n[r, 1] * ys + n[r, 2] for r in range(3)]
    w = row[2] + n[2, 0] * x1_
    assert (w > 0).all()
    w = 32.0 / w
    return max(np.abs((row[r] + n[r, 0] * x1_) * w).max() for r in range(2))


def _accepted(H, W, s, reg):
    from marconet_b200 import pipeline
    try:
        return pipeline.plan_regions([(H, W)], [[reg]], scale=s)[0]
    except ValueError:
        return None


def _far_oriented(H, W):
    from marconet_b200.pipeline import OrientedRegion
    regs = []
    for angle in (0, 29.9, 45, 89.99, 135, 179.9, -90, -150):
        for w, h in ((60, 4.5), (60, 8), (300, 2), (30, 30), (2000, 16), (24, 1.2)):
            for cx, cy in ((W - 1, H - 1), (W - 1, 1), (1, H - 1), (W / 2, H / 2)):
                regs.append(OrientedRegion.from_rotated(cx, cy, w, h, angle))
    return regs


@pytest.mark.parametrize("H, W", [(64, 32767), (32767, 64)])
def test_oriented_maps_at_the_limits_stay_in_fixed_point(H, W):
    from marconet_b200 import pipeline
    s, seen, refused, near = 8, 0, 0, 0
    for reg in _far_oriented(H, W):
        p = _accepted(H, W, s, reg)
        if p is None:
            refused += 1
            continue
        seen += 1
        m = pipeline.oriented_maps(reg, s)
        x0, y0, adelta = _affine_extremes(m.page_map, p.out)
        assert max(x0, adelta, y0) < 2 ** 30 + 64, (reg, x0, adelta, y0)     # each int, and their int32 sum
        near += y0 > 2 ** 28
        w_r, h_r = m.size
        assert max(_affine_extremes(m.matrix, (0, 0, w_r, h_r))) < 2 ** 30
    assert seen > 50 and (H > W or refused + near > 0), (seen, refused, near)     # the column step grows along x


def _far_quads(H, W, rng):
    from marconet_b200.pipeline import QuadRegion
    out = []
    for _ in range(400):
        cx, cy = (W - 1, H - 1) if rng.random() < 0.5 else (rng.uniform(0, W), rng.uniform(0, H))
        w, h = rng.uniform(3, 300), rng.uniform(1.2, 40)
        a = math.radians(rng.uniform(-180, 180))
        g = rng.uniform(1, 4)                    # the far side's length over the near side's: foreshortening up to 4
        pts = [(-w / 2, -h / 2), (w / 2, -h / 2 * g), (w / 2, h / 2 * g), (-w / 2, h / 2)]
        if rng.random() < 0.5:
            pts = [(-x, y) for x, y in pts][::-1]
            pts = [pts[1], pts[0], pts[3], pts[2]]
        c, s_ = math.cos(a), math.sin(a)
        out.append(QuadRegion(*((cx + c * x - s_ * y, cy + s_ * x + c * y) for x, y in pts)))
    return out


@pytest.mark.parametrize("H, W", [(64, 32767), (32767, 64)])
def test_quad_maps_at_the_limits_stay_in_fixed_point(H, W):
    from marconet_b200 import pipeline
    rng = np.random.default_rng(H)
    s, seen, worst = 8, 0, 0.0
    for reg in _far_quads(H, W, rng):
        p = _accepted(H, W, s, reg)
        if p is None:
            continue
        seen += 1
        m = pipeline.quad_maps(reg, s)
        x0, y0, x1, y1 = p.out
        if (x1 - x0) * (y1 - y0) > 4e6:
            continue
        worst = max(worst, _perspective_extremes(m.page_map, p.out, (s * H, s * W)))
        assert worst < 2 ** 30
    assert seen > 40, seen


@pytest.mark.parametrize("H, W", [(64, 32767), (32767, 64)])
def test_curved_maps_at_the_limits_stay_in_remap_range(H, W):
    from marconet_b200 import pipeline
    rng = np.random.default_rng(W)
    seen, refused, reach = 0, 0, 0.0
    regs = [_curved(rng, H, W) for _ in range(30)]
    big = max(H, W)
    for x in (16300.0, 16383.0, 16390.0, big - 200.0):     # straight lines that end near and past 2^14 along the long side
        k = 4
        xs = np.linspace(x - 180, x, 3 * k + 1)
        if H > W:
            regs.append(pipeline.CurvedRegion(tuple((20.0, v) for v in xs), tuple((10.0, v) for v in xs)))
        else:
            regs.append(pipeline.CurvedRegion(tuple((v, 10.0) for v in xs), tuple((v, 20.0) for v in xs)))
    for reg in regs:
        p = _accepted(H, W, 8, reg)
        if p is None:
            refused += 1
            continue
        seen += 1
        mx, my = curved_regions.crop_map(pipeline.curved_maps(p.curved, 1))
        r = max(np.abs(mx).max(), np.abs(my).max())
        assert r < 2 ** 14, (reg, r)
        reach = max(reach, r)
    assert seen >= 30 and refused >= 1 and reach > 16000, (seen, refused, reach)


# ---- the 65535-region limit of restore_regions -------------------------------------------------------------------------
def test_plan_regions_refuses_more_than_65535_regions():
    from marconet_b200 import pipeline
    shapes = [(64, 256)] * 257
    regs = [[(x, y, x + 1, y + 1) for y in range(0, 64, 4) for x in range(0, 256, 16)] for _ in shapes]     # 256 per image
    assert sum(map(len, regs)) == 65792
    with pytest.raises(ValueError, match="65792 regions in one call.*at most 65535"):
        pipeline.plan_regions(shapes, regs, scale=1)
    regs = regs[:-1]
    regs[-1] = regs[-1][:-1]
    assert sum(map(len, regs)) == 65535
    assert len(pipeline.plan_regions(shapes[:-1], regs, scale=1)) == 65535


def test_restore_regions_refuses_before_any_launch(monkeypatch):
    from marconet_b200 import ops, pipeline
    calls = []
    monkeypatch.setattr(pipeline, "restore_images", lambda *a, **k: calls.append(1))
    monkeypatch.setattr(pipeline, "_device_images", lambda *a, **k: calls.append(2))
    imgs = [np.zeros((64, 256, 3), np.uint8)] * 257
    regs = [[(x, y, x + 1, y + 1) for y in range(0, 64, 4) for x in range(0, 256, 16)] for _ in imgs]
    before = ops.LAUNCHES
    with pytest.raises(ValueError, match="65792 regions in one call"):
        pipeline.restore_regions(None, None, None, imgs, regs, scale=1)
    assert ops.LAUNCHES == before and not calls
