"""CPU restatement of OpenCV's 8-bit perspective warp (TEST INFRASTRUCTURE ONLY): cv2.warpPerspective(src, M, dsize,
flags=INTER_CUBIC | WARP_INVERSE_MAP, borderMode=BORDER_REPLICATE) on uint8 HWC images, OpenCV's OWN code path
(modules/imgproc/src/imgwarp.cpp: WarpPerspectiveInvoker's fixed-point coordinates, formed block by block, then remap's cubic
sampler exactly as the affine warp uses it), the arithmetic mn_warp_perspective_u8_batched and mn_composite_regions_quad_u8
compute (DESIGN.md section 7b, "Perspective text regions").  The sampler and its 2-D table are oracle.warp_affine's.

PINNED: bit-exact against cv2 4.13.0 with ``cv2.ipp.setUseIPP(False)`` (tests/test_quad_regions.py).
"""
import numpy as np

from .warp_affine import INTER_TAB, warp_sample_u8

INT_MIN, INT_MAX = -2.0 ** 31, 2.0 ** 31 - 1


def block_width(dsize):
    """The width of WarpPerspectiveInvoker's column blocks for a destination of dsize = (width, height): BLOCK_SZ = 32,
    bh0 = min(16, height), bw0 = min(1024 / bh0, width) (64 columns once the destination has 16 rows and 64 columns)."""
    dw, dh = dsize
    return min(32 * 32 // min(32 // 2, dh), dw)


def warp_coords(M, xs, ys, dsize):
    """cv2.warpPerspective's fixed-point source coordinates (WARP_INVERSE_MAP) of destination columns xs and rows ys of a
    destination of dsize = (width, height): int64 (Xq, Yq) [len(ys), len(xs)] in 1/32 source pixel.  OpenCV walks the destination
    in column blocks of bw = block_width(dsize) and forms, at each block's first column xb, X0 = fl(fl(fl(M00 xb) + fl(M01 y)) +
    M02), Y0 and W0 likewise; then per column x = xb + x1: W = fl(W0 + fl(M20 x1)), W = W ? fl(32 / W) : 0,
    fX = clamp(fl(fl(X0 + fl(M00 x1)) W), INT_MIN, INT_MAX), Xq = cvRound(fX) (fp64, round half to even, no contraction).  The
    block origin changes the rounding, so it is part of the result: a destination wider than a block pins it against cv2.  The
    source pixel is Xq >> 5 and the fraction Xq & 31; cv2's int16 storage of Xq >> 5 changes no value with replicated borders
    and source sides <= 32767."""
    M = np.asarray(M, np.float64).reshape(3, 3)
    bw = block_width(dsize)
    xs = np.asarray(xs, np.int64)
    xb, x1 = (xs - xs % bw).astype(np.float64)[None, :], (xs % bw).astype(np.float64)[None, :]
    ys = np.asarray(ys, np.float64)[:, None]
    row = [M[r, 0] * xb + M[r, 1] * ys + M[r, 2] for r in range(3)]
    w = row[2] + M[2, 0] * x1
    nz = w != 0
    w = np.where(nz, np.float64(INTER_TAB) / np.where(nz, w, 1.0), 0.0)
    q = []
    for r in range(2):
        f = np.clip((row[r] + M[r, 0] * x1) * w, INT_MIN, INT_MAX)
        q.append(np.rint(f).astype(np.int64))
    return q[0], q[1]


def warp_perspective_cubic_u8(src, M, dsize):
    """cv2.warpPerspective(src, M, dsize, flags=INTER_CUBIC | WARP_INVERSE_MAP, borderMode=BORDER_REPLICATE) for uint8 HWC
    images, OpenCV's own code path (IPP off): M (3 x 3) maps destination pixel indices to source pixel indices (homogeneous);
    dsize = (width, height)."""
    dw, dh = dsize
    xq, yq = warp_coords(M, np.arange(dw), np.arange(dh), dsize)
    return warp_sample_u8(np.asarray(src), xq, yq)
