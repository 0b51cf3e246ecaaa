"""Text regions in whole pages end to end (host uint8 in, host uint8 out, every copy inside the timed region):
pipeline.restore_regions against the host path a user writes without it -- restore_images(to_host=True) on the regions cut out of
the pages, then cv2's cubic resize of every page and of every restored region (IPP off) and the numpy feather blend
(oracle/regions.py).

    MN_MODULE_GRAPHS=0 python tools/bench_regions.py [--pages 8] [--lines 12] [--passes 3] [--scale 4] [--max-angle 0]
                                                     [--perspective 0] [--curved]

The pages are seeded: tools/bench_images.make_image_set lines (the reference test set's sizes and lines 2 to 4 times wider than the
LQ canvas) pasted one under another onto a noise background, each line a region with its character boxes.  The arms alternate pass
by pass; both must give the same bytes.  The two new kernels (mn_resize_cubic_u8_batched, mn_composite_regions_u8) are timed with
CUDA events around their launches inside the restore_regions passes.  MN_MODULE_GRAPHS defaults to 0 here: recorded module graphs
of 16-character crop batches outgrow an 80 GB card (DESIGN.md section 7b).  Prints one JSON line per arm and one for the kernels,
with the card's name and power limit read in the same run.  Not part of the product path.

With --max-angle DEG > 0 every line is pasted turned by a seeded angle in [-DEG, DEG] and given as a pipeline.OrientedRegion
(DESIGN.md section 7b, "Oriented text regions").  The host arm then rectifies each line with cv2.warpAffine, runs
restore_images(to_host=True) on the crops, resizes the pages with cv2, warps each restored line back with cv2.warpAffine and
blends it over its footprint with the numpy feather (oracle/oriented_regions.py); the timed kernels are mn_warp_affine_u8_batched,
mn_resize_cubic_u8_batched and mn_composite_regions_affine_u8.

With --perspective K > 1 every line is pasted seen in perspective: its far (right) end shrunk by a seeded foreshortening ratio in
[1, K] and given as a pipeline.QuadRegion (DESIGN.md section 7b, "Perspective text regions").  The host arm then rectifies each
line with cv2.warpPerspective, runs restore_images(to_host=True) on the crops, resizes the pages with cv2, warps each restored line
back with cv2.warpPerspective and blends it over its footprint with the numpy feather (oracle/quad_regions.py); the timed kernels
are mn_warp_perspective_u8_batched, mn_resize_cubic_u8_batched and mn_composite_regions_quad_u8.

With --vertical every line becomes a column of upright characters: its first --cells character cells (each cut at its box and
resized, nearest pixel, to a square of the line's height) stacked down the page, the columns side by side, each given as a
pipeline.VerticalRegion of its rectangle with boxes in the column's frame (DESIGN.md section 7b, "Vertical text columns").  The
host arm then lays every column out as a line with numpy (oracle/vertical_regions.py), runs restore_images(to_host=True) on the
lines, puts each restored line back into a column with numpy, resizes the pages and each column with cv2 and blends with the
numpy feather; the timed kernels are mn_vertical_layout_u8_batched, mn_vertical_unlayout_u8_batched, mn_resize_cubic_u8_batched
and mn_composite_regions_u8.

With --curved every line is pasted on a curve, alternately a seal-like arc of 40 to 120 degrees (pipeline.CurvedRegion.from_arc)
and a two-segment S-curve, and given as a pipeline.CurvedRegion (DESIGN.md section 7b, "Curved text regions").  The lines are the
reference test set's sizes up to 49 rows, so that the host arm's numpy inversion stays within minutes.  The host arm then
rectifies each line with cv2.remap through the numpy twin's crop maps (oracle/curved_regions.py), runs
restore_images(to_host=True) on the crops, resizes the pages with cv2, inverts every pixel of each footprint box with the twin,
remaps each restored line back with cv2.remap and blends it with the numpy feather; the timed kernels are
mn_remap_curved_u8_batched, mn_resize_cubic_u8_batched and mn_composite_regions_curved_u8.

--profile adds one restore_regions pass under torch.profiler (after the timed passes, in the same run) and prints the device time
of every kernel of that pass by name.
"""
import argparse
import json
import os
import sys
import time

os.environ.setdefault("MN_MODULE_GRAPHS", "0")

import numpy as np  # noqa: E402
import torch  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))


def make_pages(n_pages, n_lines, seed=0):
    """n_pages noise pages, each holding n_lines make_image_set lines one under another (8-pixel gaps, left margin 8 + 4k):
    (pages, regions, labels, boxes), boxes in page coordinates."""
    from bench_images import make_image_set
    images, labels, boxes = make_image_set(n_pages * n_lines, seed)
    rng = np.random.default_rng(seed + 1)
    pages, rects, labs, bxs = [], [], [], []
    for p in range(n_pages):
        idx = range(p * n_lines, (p + 1) * n_lines)
        W = max(images[i].shape[1] + 8 + 4 * (k % 8) for k, i in enumerate(idx)) + 8
        H = sum(images[i].shape[0] + 8 for i in idx) + 8
        page = rng.integers(0, 256, (H, W, 3), dtype=np.uint8)
        rr, ll, bb, y = [], [], [], 8
        for k, i in enumerate(idx):
            h, w = images[i].shape[:2]
            x = 8 + 4 * (k % 8)
            page[y:y + h, x:x + w] = images[i]
            rr.append((x, y, x + w, y + h))
            ll.append(labels[i])
            bb.append([[b[0] + x, b[1] + y, b[2] + x, b[3] + y] for b in boxes[i]])
            y += h + 8
        pages.append(page)
        rects.append(rr)
        labs.append(ll)
        bxs.append(bb)
    return pages, rects, labs, bxs


def make_rotated_pages(n_pages, n_lines, max_angle, seed=0):
    """make_pages' lines, each turned by a seeded angle in [-max_angle, max_angle] and pasted (nearest pixel) one under another
    by their bounding boxes onto a noise page: (pages, regions, labels, boxes), regions OrientedRegions and boxes in each line's
    own frame."""
    import cv2
    from bench_images import make_image_set
    from marconet_b200.pipeline import OrientedRegion, oriented_maps
    images, labels, boxes = make_image_set(n_pages * n_lines, seed)
    rng = np.random.default_rng(seed + 1)
    pages, regs, labs, bxs = [], [], [], []
    for p in range(n_pages):
        idx = range(p * n_lines, (p + 1) * n_lines)
        angles = rng.uniform(-max_angle, max_angle, n_lines)
        ext = []
        for i, a in zip(idx, angles):
            h, w = images[i].shape[:2]
            c, sn = abs(np.cos(np.radians(a))), abs(np.sin(np.radians(a)))
            ext.append((w * c + h * sn, w * sn + h * c))
        W = int(max(e[0] for e in ext)) + 24
        H = int(sum(e[1] + 8 for e in ext)) + 16
        page = rng.integers(0, 256, (H, W, 3), dtype=np.uint8)
        rr, y = [], 8.0
        for i, a, (bw, bh) in zip(idx, angles, ext):
            h, w = images[i].shape[:2]
            reg = OrientedRegion.from_rotated(8 + bw / 2, y + bh / 2, w, h, a)
            m = oriented_maps(reg, 1)
            assert m.size == (w, h)
            warped = cv2.warpAffine(images[i], m.matrix, (W, H), flags=cv2.INTER_NEAREST)
            inside = cv2.warpAffine(np.ones((h, w), np.uint8), m.matrix, (W, H), flags=cv2.INTER_NEAREST).astype(bool)
            page[inside] = warped[inside]
            rr.append(reg)
            y += bh + 8
        pages.append(page)
        regs.append(rr)
        labs.append([labels[i] for i in idx])
        bxs.append([boxes[i] for i in idx])
    return pages, regs, labs, bxs


def make_perspective_pages(n_pages, n_lines, max_ratio, seed=0):
    """make_pages' lines, each seen in perspective -- its right side shrunk about its middle by a seeded ratio in [1, max_ratio] --
    and pasted (nearest pixel, resized to its rectified crop's size) one under another onto a noise page: (pages, regions,
    labels, boxes), regions QuadRegions and boxes in each line's rectified frame."""
    import cv2
    from bench_images import make_image_set
    from marconet_b200.pipeline import QuadRegion, quad_maps
    images, labels, boxes = make_image_set(n_pages * n_lines, seed)
    rng = np.random.default_rng(seed + 1)
    pages, regs, labs, bxs = [], [], [], []
    for p in range(n_pages):
        idx = range(p * n_lines, (p + 1) * n_lines)
        ratios = rng.uniform(1, max_ratio, n_lines)
        W = max(images[i].shape[1] for i in idx) + 24
        H = sum(images[i].shape[0] + 8 for i in idx) + 8
        page = rng.integers(0, 256, (H, W, 3), dtype=np.uint8)
        rr, bb, y = [], [], 8
        for i, k in zip(idx, ratios):
            h, w = images[i].shape[:2]
            d = (h - h / k) / 2
            reg = QuadRegion((8, y), (8 + w, y + d), (8 + w, y + h - d), (8, y + h))
            qm = quad_maps(reg, 1)
            (w_r, h_r), m = qm.size, qm.matrix
            line = cv2.resize(images[i], qm.size, interpolation=cv2.INTER_NEAREST)
            warped = cv2.warpPerspective(line, m, (W, H), flags=cv2.INTER_NEAREST)
            inside = cv2.warpPerspective(np.ones((h_r, w_r), np.uint8), m, (W, H), flags=cv2.INTER_NEAREST).astype(bool)
            page[inside] = warped[inside]
            fx, fy = w_r / w, h_r / h
            bb.append([[min(b[0] * fx, w_r), b[1] * fy, min(b[2] * fx, w_r), b[3] * fy] for b in boxes[i]])
            rr.append(reg)
            y += h + 8
        pages.append(page)
        regs.append(rr)
        labs.append([labels[i] for i in idx])
        bxs.append(bb)
    return pages, regs, labs, bxs


def make_curved_pages(n_pages, n_lines, seed=0):
    """Lines of the reference test set's sizes up to 49 rows, each bent into an arc (even lines: 40 to 120 degrees, read left to
    right over its top) or a two-segment S-curve (odd lines) and pasted (nearest pixel, each crop pixel to its rounded crop-map
    position) one under another onto a noise page: (pages, regions, labels, boxes), regions CurvedRegions and boxes in each line's
    rectified frame."""
    from bench_images import TESTSET_SIZES
    from marconet_b200.pipeline import CurvedRegion, curved_maps
    from oracle import curved_regions as R
    rng = np.random.default_rng(seed + 1)
    sizes = [hw for hw in TESTSET_SIZES if hw[0] <= 49]
    pages, regs, labs, bxs = [], [], [], []
    for p in range(n_pages):
        lines, W, H = [], 0, 8.0
        for j in range(n_lines):
            h, w = sizes[(p * n_lines + j) % len(sizes)]
            if j % 2 == 0:
                phi = np.radians(rng.uniform(40, 120))
                r = w / phi
                half = np.degrees(phi) / 2
                ro = r + h / 2
                bw, bh = 2 * ro * np.sin(phi / 2), ro - (r - h / 2) * np.cos(phi / 2)
                reg = CurvedRegion.from_arc(8 + bw / 2, H + ro, ro, r - h / 2, 90 + half, 90 - half)
            else:
                amp = rng.uniform(0.02, 0.06) * w
                xs = np.linspace(0, w, 7)
                ys = H + amp + amp * np.array([0, -1, 1, 0, -1, 1, 0])
                bw, bh = w, h + 2 * amp
                reg = CurvedRegion(tuple((8 + x, y) for x, y in zip(xs, ys)), tuple((8 + x, y + h) for x, y in zip(xs, ys)))
            lines.append((reg, h, w))
            W, H = max(W, int(bw) + 24), H + bh + 8
        H = int(H) + 8
        page = rng.integers(0, 256, (H, W, 3), dtype=np.uint8)
        rr, ll, bb = [], [], []
        for reg, h, w in lines:
            m = curved_maps(reg, 1)
            (w_r, h_r) = m.size
            pitch = 28 * h_r / 32
            k = max(1, int(w_r // pitch))
            line = rng.integers(0, 256, (h_r, w_r, 3), dtype=np.uint8)
            mx, my = R.crop_map(m)
            xi, yi = np.rint(mx).astype(np.int64), np.rint(my).astype(np.int64)
            inside = (xi >= 0) & (xi < W) & (yi >= 0) & (yi < H)
            page[yi[inside], xi[inside]] = line[inside]
            rr.append(reg)
            bb.append([[int(j * pitch + 0.15 * pitch), 0, int(j * pitch + 0.85 * pitch), h_r] for j in range(k)])
            ll.append(rng.integers(0, 6735, k).tolist())
        pages.append(page)
        regs.append(rr)
        labs.append(ll)
        bxs.append(bb)
    return pages, regs, labs, bxs


def make_vertical_pages(n_pages, n_cols, max_cells, seed=0):
    """make_image_set lines turned into columns: each line's first max_cells characters, cut at their boxes and resized (nearest
    pixel) to h x h squares, stacked one under another and the columns pasted side by side (8-pixel gaps) onto a noise page:
    (pages, regions, labels, boxes), regions VerticalRegions of rectangles and boxes in each column's frame."""
    import cv2
    from bench_images import make_image_set
    from marconet_b200.pipeline import VerticalRegion
    images, labels, boxes = make_image_set(n_pages * n_cols, seed)
    rng = np.random.default_rng(seed + 1)
    pages, regs, labs, bxs = [], [], [], []
    for p in range(n_pages):
        idx = range(p * n_cols, (p + 1) * n_cols)
        cols, ll, bb = [], [], []
        for i in idx:
            h = images[i].shape[0]
            chars = boxes[i][:max_cells]
            cols.append(np.concatenate([cv2.resize(images[i][:, b[0]:b[2]], (h, h), interpolation=cv2.INTER_NEAREST)
                                        for b in chars], 0))
            ll.append(labels[i][:len(chars)])
            bb.append([[1, k * h + 1, h - 1, (k + 1) * h - 1] for k in range(len(chars))])
        W = sum(c.shape[1] + 8 for c in cols) + 8
        H = max(c.shape[0] for c in cols) + 16
        page = rng.integers(0, 256, (H, W, 3), dtype=np.uint8)
        rr, x = [], 8
        for c in cols:
            page[8:8 + c.shape[0], x:x + c.shape[1]] = c
            rr.append(VerticalRegion((x, 8, x + c.shape[1], 8 + c.shape[0])))
            x += c.shape[1] + 8
        pages.append(page)
        regs.append(rr)
        labs.append(ll)
        bxs.append(bb)
    return pages, regs, labs, bxs


def host_path_vertical(m, pages, regs, labels, boxes, s, feather, max_lines):
    """numpy layout of every column, restore_images on the lines, numpy inverse layout, cv2 background and cv2 resize of each
    restored column onto its rectangle, the numpy blend."""
    import cv2
    from marconet_b200 import pipeline
    from oracle import regions
    from oracle import vertical_regions as V
    lines, labs, lbx, cells = [], [], [], []
    for pg, rr, ll, bb in zip(pages, regs, labels, boxes):
        for reg, lab, bx in zip(rr, ll, bb):
            x0, y0, x1, y1 = reg.shape
            c = V.cells(y1 - y0, x1 - x0, boxes=bx)
            lines.append(V.layout(pg[y0:y1, x0:x1], c))
            labs.append(lab)
            lbx.append(V.line_boxes(c, x1 - x0, bx))
            cells.append(c)
    res = pipeline.restore_images(*m, lines, labs, lbx, max_lines=max_lines, to_host=True)
    out, k = [], 0
    for pg, rr in zip(pages, regs):
        o = cv2.resize(pg, (0, 0), fx=s, fy=s, interpolation=cv2.INTER_CUBIC)
        for reg in rr:
            x0, y0, x1, y1 = reg.shape
            tc = V.unlayout(res[k]["sr_u8"], cells[k], x1 - x0)
            r = (s * x0, s * y0, s * x1, s * y1)
            p = cv2.resize(np.ascontiguousarray(tc[..., ::-1]), (r[2] - r[0], r[3] - r[1]), interpolation=cv2.INTER_CUBIC)
            o[r[1]:r[3], r[0]:r[2]] = regions.blend(o[r[1]:r[3], r[0]:r[2]], p, regions.alpha(r, o.shape[:2], feather))
            k += 1
        out.append(o)
    return out


def host_path_curved(m, pages, regs, labels, boxes, s, feather, max_lines):
    """cv2.remap rectify through the twin's crop maps, restore_images on the crops, cv2 background, the twin's inversion of every
    pixel of each footprint box, cv2.remap of each restored line back at those T coordinates and the numpy blend."""
    import cv2
    from marconet_b200 import pipeline
    from oracle import curved_regions as R
    crops, labs, bxs = [], [], []
    for pg, rr, ll, bb in zip(pages, regs, labels, boxes):
        for reg, lab, bx in zip(rr, ll, bb):
            mx, my = R.crop_map(pipeline.curved_maps(reg, 1))
            crops.append(cv2.remap(pg, mx.astype(np.float32), my.astype(np.float32), cv2.INTER_CUBIC,
                                   borderMode=cv2.BORDER_REPLICATE))
            labs.append(lab)
            bxs.append(bx)
    res = pipeline.restore_images(*m, crops, labs, bxs, max_lines=max_lines, to_host=True)
    out, k = [], 0
    for pg, rr in zip(pages, regs):
        o = cv2.resize(pg, (0, 0), fx=s, fy=s, interpolation=cv2.INTER_CUBIC)
        for reg in rr:
            t = res[k]["sr_u8"]
            th, tw = t.shape[:2]
            n = pipeline.curved_maps(reg, s, tw)
            x0, y0, x1, y1 = pipeline.curved_footprint_box(reg, s, o.shape[:2])
            qx, qy = np.meshgrid((np.arange(x0, x1) + 0.5) / s, (np.arange(y0, y1) + 0.5) / s)
            ok, mm, tt, bb = R.invert(n, qx, qy)
            u, v = R.t_maps(n, mm, tt, bb, (th, tw))
            u, v = np.where(ok, u, 0).reshape(qx.shape).astype(np.float32), np.where(ok, v, 0).reshape(qx.shape).astype(np.float32)
            xq, yq = np.rint(u * np.float32(32)).astype(np.int64), np.rint(v * np.float32(32)).astype(np.int64)
            mask = ok.reshape(qx.shape) & (xq >= -16) & (xq < 32 * tw - 16) & (yq >= -16) & (yq < 32 * th - 16)
            a = R.feather_alpha(xq, yq, (th, tw), n.kx, n.ky, feather)
            p = cv2.remap(np.ascontiguousarray(t[..., ::-1]), u, v, cv2.INTER_CUBIC, borderMode=cv2.BORDER_REPLICATE)
            sl = o[y0:y1, x0:x1]
            sl[mask] = R.blend(sl, p, a)[mask]
            k += 1
        out.append(o)
    return out


def host_path_perspective(m, pages, regs, labels, boxes, s, feather, max_lines):
    """cv2 rectify, restore_images on the crops, cv2 background and cv2 warp of each restored line back (onto the rows and
    columns up to its footprint's far corner: at least 64 columns and 16 rows, so that cv2's 64-column blocks start where the
    whole page's do), the numpy blend."""
    import cv2
    from marconet_b200 import pipeline
    from oracle import quad_regions as regions
    flags = cv2.INTER_CUBIC | cv2.WARP_INVERSE_MAP
    crops, labs, bxs = [], [], []
    for pg, rr, ll, bb in zip(pages, regs, labels, boxes):
        for reg, lab, bx in zip(rr, ll, bb):
            mp = pipeline.quad_maps(reg, 1)
            crops.append(cv2.warpPerspective(pg, mp.matrix, mp.size, flags=flags, borderMode=cv2.BORDER_REPLICATE))
            labs.append(lab)
            bxs.append(bx)
    res = pipeline.restore_images(*m, crops, labs, bxs, max_lines=max_lines, to_host=True)
    out, k = [], 0
    for pg, rr in zip(pages, regs):
        o = cv2.resize(pg, (0, 0), fx=s, fy=s, interpolation=cv2.INTER_CUBIC)
        for reg in rr:
            t = res[k]["sr_u8"]
            (x0, y0, x1, y1), _, _, mask, a = regions.quad_footprint(t.shape, reg, s, o.shape[:2], feather)
            n = pipeline.quad_maps(reg, s, t.shape[1]).page_map
            dw, dh = max(x1, 64), max(y1, 16)
            p = cv2.warpPerspective(np.ascontiguousarray(t[..., ::-1]), n, (dw, dh), flags=flags, borderMode=cv2.BORDER_REPLICATE)
            sl = o[y0:y1, x0:x1]
            sl[mask] = regions.blend(sl, p[y0:y1, x0:x1], a)[mask]
            k += 1
        out.append(o)
    return out


def host_path_oriented(m, pages, regs, labels, boxes, s, feather, max_lines):
    """cv2 rectify, restore_images on the crops, cv2 background and cv2 warp of each restored line back (onto the rows and
    columns up to its footprint's far corner, so that its fixed-point coordinates are the whole page's), the numpy blend."""
    import cv2
    from marconet_b200 import pipeline
    from oracle import oriented_regions as regions
    flags = cv2.INTER_CUBIC | cv2.WARP_INVERSE_MAP
    crops, labs, bxs = [], [], []
    for pg, rr, ll, bb in zip(pages, regs, labels, boxes):
        for reg, lab, bx in zip(rr, ll, bb):
            mp = pipeline.oriented_maps(reg, 1)
            crops.append(cv2.warpAffine(pg, mp.matrix, mp.size, flags=flags, borderMode=cv2.BORDER_REPLICATE))
            labs.append(lab)
            bxs.append(bx)
    res = pipeline.restore_images(*m, crops, labs, bxs, max_lines=max_lines, to_host=True)
    out, k = [], 0
    for pg, rr in zip(pages, regs):
        o = cv2.resize(pg, (0, 0), fx=s, fy=s, interpolation=cv2.INTER_CUBIC)
        for reg in rr:
            t = res[k]["sr_u8"]
            (x0, y0, x1, y1), _, _, mask, a = regions.oriented_footprint(t.shape, reg, s, o.shape[:2], feather)
            n = pipeline.oriented_maps(reg, s, t.shape[1]).page_map
            p = cv2.warpAffine(np.ascontiguousarray(t[..., ::-1]), n, (x1, y1), flags=flags, borderMode=cv2.BORDER_REPLICATE)
            sl = o[y0:y1, x0:x1]
            sl[mask] = regions.blend(sl, p[y0:y1, x0:x1], a)[mask]
            k += 1
        out.append(o)
    return out


def host_path(m, pages, rects, labels, boxes, s, feather, max_lines):
    """restore_images on the cut-out regions, then cv2 resizes and the numpy blend on the host."""
    import cv2
    from marconet_b200 import pipeline
    from oracle import regions
    crops, labs, rel = [], [], []
    for pg, rr, ll, bb in zip(pages, rects, labels, boxes):
        for (x0, y0, x1, y1), lab, bx in zip(rr, ll, bb):
            crops.append(pg[y0:y1, x0:x1])
            labs.append(lab)
            rel.append([[b[0] - x0, b[1] - y0, b[2] - x0, b[3] - y0] for b in bx])
    res = pipeline.restore_images(*m, crops, labs, rel, max_lines=max_lines, to_host=True)
    out, k = [], 0
    for pg, rr in zip(pages, rects):
        o = cv2.resize(pg, (0, 0), fx=s, fy=s, interpolation=cv2.INTER_CUBIC)
        for x0, y0, x1, y1 in rr:
            r = (s * x0, s * y0, s * x1, s * y1)
            p = cv2.resize(np.ascontiguousarray(res[k]["sr_u8"][..., ::-1]), (r[2] - r[0], r[3] - r[1]), interpolation=cv2.INTER_CUBIC)
            o[r[1]:r[3], r[0]:r[2]] = regions.blend(o[r[1]:r[3], r[0]:r[2]], p, regions.alpha(r, o.shape[:2], feather))
            k += 1
        out.append(o)
    return out


def _card():
    import subprocess
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True,
                       text=True)
    name, _, power = q.stdout.strip().partition(", ")
    return {"gpu": name or torch.cuda.get_device_name(0), "power_limit": power or None}


def main():
    import cv2
    ap = argparse.ArgumentParser()
    ap.add_argument("--pages", type=int, default=8)
    ap.add_argument("--lines", type=int, default=12)
    ap.add_argument("--passes", type=int, default=3)
    ap.add_argument("--scale", type=int, default=4)
    ap.add_argument("--max-lines", type=int, default=8)
    ap.add_argument("--max-angle", type=float, default=0.0, help="turn every line by up to this many degrees (oriented regions)")
    ap.add_argument("--perspective", type=float, default=0.0,
                    help="shrink every line's far end by a foreshortening ratio up to this (> 1; perspective regions)")
    ap.add_argument("--vertical", action="store_true", help="vertical text columns (--lines columns per page)")
    ap.add_argument("--cells", type=int, default=16, help="characters per column with --vertical")
    ap.add_argument("--curved", action="store_true", help="arcs and S-curves (curved regions)")
    ap.add_argument("--profile", action="store_true", help="one more restore_regions pass under torch.profiler")
    args = ap.parse_args()
    if args.vertical and (args.max_angle > 0 or args.perspective):
        sys.exit("--vertical does not combine with --max-angle or --perspective")
    if args.perspective and (args.max_angle > 0 or not 1 < args.perspective <= 4):
        sys.exit("--perspective takes a ratio in (1, 4] and does not combine with --max-angle")
    if args.curved and (args.vertical or args.max_angle > 0 or args.perspective):
        sys.exit("--curved does not combine with --vertical, --max-angle or --perspective")
    if not torch.cuda.is_available():
        sys.exit("bench_regions.py needs a CUDA device")
    cv2.ipp.setUseIPP(False)
    from marconet_b200 import _lib, pipeline
    from marconet_b200.models import networks
    from marconet_b200.testing import synth
    dev = torch.device("cuda:0")
    sds = synth.make_checkpoints(0)
    m = []
    for key, cls in (("encoder", networks.TextContextEncoderV2), ("tspgan", networks.TSPGAN), ("sr", networks.TSPSRNet)):
        net = cls()
        net.load_state_dict(sds[key], strict=True)
        m.append(net.eval().to(dev))
    oriented, perspective = args.max_angle > 0, args.perspective > 1
    if args.vertical:
        pages, rects, labels, boxes = make_vertical_pages(args.pages, args.lines, args.cells)
    elif args.curved:
        pages, rects, labels, boxes = make_curved_pages(args.pages, args.lines)
    elif perspective:
        pages, rects, labels, boxes = make_perspective_pages(args.pages, args.lines, args.perspective)
    elif oriented:
        pages, rects, labels, boxes = make_rotated_pages(args.pages, args.lines, args.max_angle)
    else:
        pages, rects, labels, boxes = make_pages(args.pages, args.lines)
    s, feather = args.scale, 2 * args.scale

    lib = _lib.load()
    if args.vertical:
        events = {"mn_vertical_layout_u8_batched": [], "mn_vertical_unlayout_u8_batched": [], "mn_resize_cubic_u8_batched": [],
                  "mn_composite_regions_u8": []}
    elif args.curved:
        events = {"mn_remap_curved_u8_batched": [], "mn_resize_cubic_u8_batched": [], "mn_composite_regions_curved_u8": []}
    elif perspective:
        events = {"mn_warp_perspective_u8_batched": [], "mn_resize_cubic_u8_batched": [], "mn_composite_regions_quad_u8": []}
    elif oriented:
        events = {"mn_warp_affine_u8_batched": [], "mn_resize_cubic_u8_batched": [], "mn_composite_regions_affine_u8": []}
    else:
        events = {"mn_resize_cubic_u8_batched": [], "mn_composite_regions_u8": []}
    timing = [False]
    for name in events:
        fn = getattr(lib, name)

        def timed(*a, _fn=fn, _name=name):
            if not timing[0]:
                return _fn(*a)
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            rc = _fn(*a)
            e1.record()
            events[_name].append((e0, e1))
            return rc
        setattr(lib, name, timed)

    def api():
        out = pipeline.restore_regions(*m, pages, rects, labels, boxes, scale=s, feather=feather, max_lines=args.max_lines,
                                       to_host=True)
        return [o["image"] for o in out]

    def host():
        path = host_path_vertical if args.vertical else host_path_curved if args.curved else \
            host_path_perspective if perspective else \
            host_path_oriented if oriented else host_path
        return path(m, pages, rects, labels, boxes, s, feather, args.max_lines)

    arms = {"restore_regions": api, "host_path": host}
    outs = {name: fn() for name, fn in arms.items()}                 # warm-up pass of each arm
    same = all(np.array_equal(a, b) for a, b in zip(outs["restore_regions"], outs["host_path"]))
    diff = max(int(np.abs(a.astype(np.int16) - b.astype(np.int16)).max()) for a, b in zip(outs["restore_regions"], outs["host_path"]))
    times = {name: [] for name in arms}
    for _ in range(args.passes):
        for name, fn in arms.items():
            timing[0] = name == "restore_regions"
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            fn()
            torch.cuda.synchronize()
            times[name].append(time.perf_counter() - t0)
            timing[0] = False
    torch.cuda.synchronize()
    card = _card()
    out_px = sum(s * s * p.shape[0] * p.shape[1] for p in pages)
    common = dict(pages=args.pages, lines_per_page=args.lines, scale=s, feather=feather, max_lines=args.max_lines,
                  max_angle=args.max_angle, **({"perspective": args.perspective} if perspective else {}),
                  **({"vertical": True, "cells_per_column": args.cells} if args.vertical else {}),
                  **({"curved": True} if args.curved else {}),
                  page_sizes=[list(p.shape[:2]) for p in pages], output_megapixels=round(out_px / 1e6, 2),
                  module_graphs=os.environ.get("MN_MODULE_GRAPHS"), same_bytes=same, max_abs_diff=diff, **card)
    for name, ts in times.items():
        print(json.dumps(dict(metric="regions_e2e", arm=name, pass_s=[round(t, 4) for t in ts],
                              pages_per_s=round(args.pages / min(ts), 3), **common)), flush=True)
    kern = {name: [e0.elapsed_time(e1) for e0, e1 in ev] for name, ev in events.items()}
    print(json.dumps(dict(metric="regions_kernels", **{f"{k}_ms": [round(v, 4) for v in vs] for k, vs in kern.items()},
                          background_gbytes_per_s=round(3 * out_px / (min(kern["mn_resize_cubic_u8_batched"]) * 1e-3) / 1e9, 1),
                          **common)), flush=True)
    if args.profile:
        from torch.profiler import ProfilerActivity, profile
        with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
            api()
            torch.cuda.synchronize()
        dev_ms = {}
        for ev in prof.events():
            if ev.device_type == torch.autograd.DeviceType.CUDA:
                dev_ms.setdefault(ev.name, []).append(ev.device_time_total / 1e3)
        total = sum(sum(v) for v in dev_ms.values())
        top = sorted(dev_ms.items(), key=lambda kv: -sum(kv[1]))
        print(json.dumps(dict(metric="regions_profile", device_ms_total=round(total, 3),
                              kernels={k: dict(calls=len(v), ms=round(sum(v), 4)) for k, v in top
                                       if "vertical" in k or "curved" in k or "composite" in k or "resize_cubic" in k or k in dict(top[:8])},
                              **common)), flush=True)
    if not same:
        sys.exit("the arms' bytes differ")


if __name__ == "__main__":
    main()
