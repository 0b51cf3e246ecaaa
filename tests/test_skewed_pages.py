"""Skewed text pages and windowed blocks (DESIGN.md section 7b, "Skewed pages") on the host: the twin on tilted `putText` pages
of a heading over columns, level pages, the axis swap of the frame, windowed blocks, every validation error of find_blocks,
find_lines and restore_regions (raised before anything reaches a device), and the build of the new kernels."""
import math
import os
import re
import subprocess

import cv2
import numpy as np
import pytest

from marconet_b200 import ops, pipeline
from oracle import blocks as B
from oracle import pages as P
from oracle import skewed_blocks as SB
from oracle import skewed_pages as SP

from test_pages import _columns_page

WORDS = "THE BROWN FOX LEAPS OVER A LAZY DOG PACK MY BOX WITH FIVE DOZEN MUGS".split()   # no descending capitals


def drawn_page(widths, n_lines, angle, seed, misalign=False, vertical=False):
    """A heading over columns (DUPLEX capitals, 33-pixel pitch, 60-pixel gutters) turned by ``angle`` degrees about the page
    centre with cv2.warpAffine (nearest neighbour), and the turned ink masks of the heading and of each column's lines.
    ``vertical`` transposes the drawn page first: a title column right of columns of vertical lines."""
    rng = np.random.default_rng(seed)
    pitch, gutter, margin = 33, 60, 80
    W = 2 * margin + sum(widths) + gutter * (len(widths) - 1)
    H = 2 * margin + 70 + n_lines * pitch
    heading = np.zeros((H, W), np.uint8)
    cv2.putText(heading, "HEADING OVER ALL COLUMNS"[:max(8, (W - 2 * margin) // 22)], (margin, margin + 24),
                cv2.FONT_HERSHEY_DUPLEX, 1.0, 255, 2, cv2.LINE_8)
    masks, x = [heading], margin
    for c, cw in enumerate(widths):
        lines = []
        for k in range(n_lines):
            m = np.zeros((H, W), np.uint8)
            t = str(rng.choice(WORDS))
            while True:
                longer = t + " " + str(rng.choice(WORDS))
                if cv2.getTextSize(longer, cv2.FONT_HERSHEY_DUPLEX, 1.0, 2)[0][0] > cw:
                    break
                t = longer
            y = margin + 90 + k * pitch + (pitch // 2 if misalign and c % 2 else 0)
            cv2.putText(m, t, (x, y), cv2.FONT_HERSHEY_DUPLEX, 1.0, 255, 2, cv2.LINE_8)
            lines.append(m)
        masks.append(lines)
        x += cw + gutter
    if vertical:
        masks = [masks[0].T[:, ::-1].copy()] + [[m.T[:, ::-1].copy() for m in col] for col in masks[1:]]
        H, W = W, H
    R = cv2.getRotationMatrix2D((W / 2, H / 2), angle, 1.0)
    turn = lambda m: cv2.warpAffine(m, R, (W, H), flags=cv2.INTER_NEAREST) > 0
    masks = [turn(masks[0])] + [[turn(m) for m in col] for col in masks[1:]]
    ink = masks[0] | np.any([m for col in masks[1:] for m in col], axis=0)
    return np.where(ink[..., None], 20, 235).astype(np.uint8).repeat(3, axis=2), masks


def _line_mask(q, shape, grow):
    """Pixels whose centre lies inside line q (an integer rectangle, or a corner triple tl, tr, bl) grown by ``grow``."""
    ys, xs = np.mgrid[0:shape[0], 0:shape[1]] + 0.5
    if isinstance(q[0], (int, np.integer)):
        x0, y0, x1, y1 = q
        return (xs >= x0 - grow) & (xs <= x1 + grow) & (ys >= y0 - grow) & (ys <= y1 + grow)
    (ax, ay), (bx, by), (cx, cy) = q
    ex, ey, fx, fy = bx - ax, by - ay, cx - ax, cy - ay
    le, lf = math.hypot(ex, ey), math.hypot(fx, fy)
    a = ((xs - ax) * ex + (ys - ay) * ey) / le
    b = ((xs - ax) * fx + (ys - ay) * fy) / lf
    return (a >= -grow) & (a <= le + grow) & (b >= -grow) & (b <= lf + grow)


def _check_page(img, masks, angle, vertical):
    direction = "vertical" if vertical else "horizontal"
    H, W = img.shape[:2]
    r = SP.find_blocks(img, direction=direction, skew="auto", max_skew=15.0 if abs(angle) > 10 else 10.0)
    assert abs(r["skew"] - angle) <= 0.2, (r["skew"], angle)
    assert len(r["blocks"]) == len(masks), r["blocks"]
    groups = [[masks[0]]] + masks[1:]
    # each block holds exactly one drawn group, in reading order: the heading (the title column right of a vertical page) first,
    # then the columns left to right (the transposed columns top to bottom)
    order = list(range(1, len(masks)))
    tilted = r["detail"]["frame"] is not None
    for blk, g in zip(r["blocks"], [0] + order):
        if tilted:
            got = SP.find_lines(img, (0, 0, W, H), blk, r["skew"], direction)
            member = SP.members(H, W, vertical, r["skew"], blk)
        else:
            got = B.find_lines(img, blk, direction)
            member = np.zeros((H, W), bool)
            member[blk[1]:blk[3], blk[0]:blk[2]] = True
        for other, grp in enumerate(groups):
            inside = [bool((m & member).any()) for m in grp]
            assert all(inside) if other == g else not any(inside), (blk, g, other)
        lines = got["lines"]
        if vertical and not tilted:
            lines = [q.shape if hasattr(q, "shape") else q for q in lines]
        assert len(lines) == len(groups[g]), (g, len(lines), len(groups[g]))
        regions = [_line_mask(q, (H, W), 0.5) for q in lines]
        for k, m in enumerate(groups[g]):
            assert not (m & ~regions[k]).any(), (g, k)
            for k2, reg in enumerate(regions):
                if k2 != k:
                    assert not (m & _line_mask(lines[k2], (H, W), -0.5)).any(), (g, k, k2)
    return r


ANGLES = [0.5, -0.5, 1.0, -2.0, 3.0, -4.5, 7.5, -10.0, 14.0, -14.0]


@pytest.mark.parametrize("angle", ANGLES)
@pytest.mark.parametrize("widths,misalign", [((300, 300), False), ((260, 320, 240), True)])
def test_drawn_tilted_pages(angle, widths, misalign):
    img, masks = drawn_page(widths, 8, angle, seed=int(10 * abs(angle)) + len(widths), misalign=misalign)
    _check_page(img, masks, angle, vertical=False)


@pytest.mark.parametrize("angle", [0.5, -2.0, 5.0, -14.0])
def test_drawn_tilted_vertical_pages(angle):
    img, masks = drawn_page((300, 300), 8, angle, seed=7, vertical=True)
    _check_page(img, masks, angle, vertical=True)


def test_the_three_degree_two_column_page():
    """A heading over two 12-line columns, turned by 3 degrees: one block per column, each of its drawn lines."""
    img, masks = drawn_page((300, 300), 12, 3.0, seed=0)
    r = _check_page(img, masks, 3.0, vertical=False)
    assert len(r["blocks"]) == 3


@pytest.mark.parametrize("direction", ["horizontal", "vertical"])
def test_level_pages_give_the_dict_of_skew_none(direction):
    img, _ = _columns_page(np.random.default_rng(3), (300, 300), 12)
    if direction == "vertical":
        img = np.ascontiguousarray(img.transpose(1, 0, 2))
    want = P.find_blocks(img, direction=direction)
    for skew in ("auto", 0, 0.0):
        got = SP.find_blocks(img, direction=direction, skew=skew)
        assert got.pop("detail")["frame"] is None
        assert got == dict(want, skew=0.0)


def test_axis_swap_of_the_frame():
    """u(X, Y, c, -s) = v_t and v(X, Y, c, -s) = u_t with every operation rounded, so the untransposed frame at the negated angle
    is the transposed frame with its axes swapped, and its bitmap the transpose."""
    rng = np.random.default_rng(0)
    for _ in range(200):
        h, w = (int(v) for v in rng.integers(1, 300, 2))
        th = float(rng.uniform(-20, 20))
        c, s = math.cos(math.radians(th)), math.sin(math.radians(th))
        ys, xs = np.mgrid[0:h, 0:w].astype(np.float64)
        u, v = SB._uv(ys, xs, h, w, c, -s)
        ut, vt = SB._uv(xs, ys, w, h, c, s)
        assert np.array_equal(u, vt) and np.array_equal(v, ut)
        f, ft = SB.frame(h, w, np.array([c]), np.array([-s])), SB.frame(w, h, np.array([c]), np.array([s]))
        assert (f[0], f[1], f[2], f[3]) == (ft[1], ft[0], ft[3], ft[2])
        ink = rng.random((h, w)) < 0.05
        assert np.array_equal(SP.frame_bitmap(ink, c, -s), SP.frame_bitmap(ink.T, c, s).T)


@pytest.mark.parametrize("direction", ["horizontal", "vertical"])
def test_windows_at_zero_are_sub_rectangles(direction):
    img, _ = _columns_page(np.random.default_rng(5), (300, 300), 12)
    H, W = img.shape[:2]
    vertical = direction == "vertical"
    for x0, y0, x1, y1 in P.find_blocks(img, direction=direction)["blocks"] + [(0, 0, W, H), (5, 7, 9, 8)]:
        win = (y0, x0, y1, x1) if vertical else (x0, y0, x1, y1)
        got = SP.find_lines(img, (0, 0, W, H), win, 0.0, direction)
        want = B.find_lines(img, (x0, y0, x1, y1), direction)
        assert (got["lines"], got["threshold"], got["ink"]) == (want["lines"], want["threshold"], want["ink"])


def test_windows_are_disjoint_and_hold_their_profile():
    img, _ = drawn_page((300, 300), 8, -6.0, seed=4)
    H, W = img.shape[:2]
    r = SP.find_blocks(img, skew="auto")
    sets = [SP.members(H, W, False, r["skew"], b) for b in r["blocks"]]
    assert not (np.sum(sets, axis=0) > 1).any()
    for b, m in zip(r["blocks"], sets):
        got = SP.find_lines(img, (0, 0, W, H), b, r["skew"])
        assert not (got["detail"]["ink"] & ~m).any()
        px0, py0, px1, py1 = SP.footprint(H, W, False, r["skew"], b)
        assert np.array_equal(ops.window_footprint(W, H, False, *SP.block_frame(H, W, False, r["skew"])[:4], b),
                              (px0, py0, px1, py1))
        ys, xs = np.nonzero(m)
        assert xs.min() >= px0 and xs.max() < px1 and ys.min() >= py0 and ys.max() < py1


def test_empty_window_has_no_lines():
    img, _ = drawn_page((300,), 4, 8.0, seed=1)
    H, W = img.shape[:2]
    _, _, _, _, L, M = SP.block_frame(H, W, False, 8.0)
    r = SP.find_lines(img, (0, 0, W, H), (0, 0, 1, 1), 8.0)      # a corner cell of the frame holds no pixel centre
    assert r["lines"] == [] and not SP.members(H, W, False, 8.0, (0, 0, 1, 1)).any()


def _img(h=120, w=160):
    return np.full((h, w, 3), 235, np.uint8)


@pytest.mark.parametrize("kw,msg", [
    (dict(skew="level"), "skew must be"), (dict(skew=45.0), "skew must be"), (dict(skew=float("nan")), "skew must be"),
    (dict(skew="auto", max_skew=25), "max_skew"), (dict(skew=3.0, max_skew=5.0), "max_skew is given")])
def test_find_blocks_rejects_bad_skew_before_any_launch(kw, msg):
    with pytest.raises(ValueError, match=rf"image 0, page 0: .*{msg}"):
        pipeline.find_blocks([_img()], [[pipeline.TextPage(**kw)]])


@pytest.mark.parametrize("kw,msg", [
    (dict(window=(0, 0, 10, 10)), "not a given angle"), (dict(skew="auto", window=(0, 0, 10, 10)), "not a given angle"),
    (dict(skew=3.0, window=(0, 0, 10)), "four integers"), (dict(skew=3.0, window=(0, 0, 10.0, 10)), "four integers"),
    (dict(skew=3.0, window=(5, 0, 5, 10)), "empty or outside"), (dict(skew=3.0, window=(0, 0, 10, 10 ** 6)), "empty or outside"),
    (dict(skew=3.0, window=(-1, 0, 10, 10)), "empty or outside")])
def test_windows_are_checked_before_any_launch(kw, msg):
    blk = pipeline.TextBlock((0, 0, 160, 120), **kw)
    with pytest.raises(ValueError, match=rf"image 0, block 0: .*{msg}"):
        pipeline.find_lines([_img()], [[blk]])
    with pytest.raises(ValueError, match=rf"image 0, region 0 \(a text block\): .*{msg}"):
        pipeline.restore_regions(None, None, None, [_img()], [[blk]])


def test_window_bound_is_the_frame_at_that_angle():
    _, _, L, M = ops.skew_frames(160, 120, False, ops.skew_cos_sin([10.0]))
    blk = pipeline.TextBlock((0, 0, 160, 120), skew=10.0, window=(0, 0, int(M[0]), int(L[0])))
    assert pipeline._check_block(blk, 120, 160, "b") == (0, 0, 160, 120)
    with pytest.raises(ValueError, match="outside"):
        pipeline._check_block(blk._replace(window=(0, 0, int(M[0]) + 1, int(L[0]))), 120, 160, "b")


def test_page_limits_are_checked_before_any_launch(monkeypatch):
    # a frame side over 32767: a 32767 x 6000 page turned by 10 degrees
    with pytest.raises(ValueError, match="image 0, page 0: a side of the page's rotated frame"):
        pipeline._check_page(pipeline.TextPage((0, 0, 32767, 6000), skew=10.0), 6000, 32767, "image 0, page 0")
    with pytest.raises(ValueError, match="profile values"):
        pipeline._check_page(pipeline.TextPage((0, 0, 30000, 30000), skew="auto", max_skew=20), 30000, 30000, "p")
    level = ops.skew_page_bytes(1000, 800, False, ops.skew_cos_sin([0.0]))
    searched = ops.skew_page_bytes(1000, 800, False, ops.skew_cos_sin(ops.skew_table("auto", 10.0, False)))
    assert searched > level + 401 * 4 * 800                 # the profiles and scores of the search count
    monkeypatch.setattr(ops, "PAGE_MAX_WORK", level)
    pipeline._check_page(pipeline.TextPage((0, 0, 1000, 800), skew=0.0), 800, 1000, "p")
    with pytest.raises(ValueError, match="bytes of work memory"):
        pipeline._check_page(pipeline.TextPage((0, 0, 1000, 800), skew="auto"), 800, 1000, "p")
    with pytest.raises(ValueError, match="text pages need more"):
        pipeline._check_page_work([(0, pipeline.TextPage(skew=1.0), (0, 0, 400, 400))] * 4)


def test_new_kernels_build_without_spills(tmp_path):
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    if not os.path.exists(nvcc):
        pytest.skip("nvcc not found")
    src = os.path.join(os.path.dirname(ops.__file__), "csrc", "block_ops.cu")
    r = subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-Xcompiler", "-fPIC",
                        "-DMN_BUILD", "-Xptxas", "-v", "-c", src, "-o", str(tmp_path / "b.o")], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    for kernel in ("page_frame_bits_kernel", "window_hist_kernel", "window_profile_kernel"):
        props = re.search(rf"Function properties for \S*{kernel}\S*\n(.*)\n", r.stderr)
        assert props, kernel
        assert "0 bytes spill stores, 0 bytes spill loads" in props.group(1), props.group(1)
