"""CPU restatement of OpenCV's 8-bit affine warp (TEST INFRASTRUCTURE ONLY): cv2.warpAffine(src, M, dsize,
flags=INTER_CUBIC | WARP_INVERSE_MAP, borderMode=BORDER_REPLICATE) on uint8 HWC images, OpenCV's OWN code path
(modules/imgproc/src/imgwarp.cpp: WarpAffineInvoker's fixed-point coordinates, initInterTab2D's 2-D cubic table and
remapBicubic with FixedPtCast<int, uchar, 15>), the arithmetic mn_warp_affine_u8_batched and mn_composite_regions_affine_u8
compute (DESIGN.md section 7b, "Oriented text regions").  The 1-D weights are oracle.image_ops.cubic_coeffs (interpolateCubic,
A = -0.75, fp32).

PINNED: bit-exact against cv2 4.13.0 with ``cv2.ipp.setUseIPP(False)`` (tests/test_oriented_regions.py).
"""
import functools

import numpy as np

from .image_ops import cubic_coeffs

INTER_BITS = 5                   # warpAffine / remap: 1/32-pixel source coordinates
INTER_TAB = 1 << INTER_BITS
AB_BITS = 10                     # warpAffine's fixed-point step: coordinates in 1/1024 pixel before the >> (AB_BITS - INTER_BITS)
AB_SCALE = 1 << AB_BITS
REMAP_COEF_SCALE = 1 << 15       # INTER_REMAP_COEF_SCALE: the 2-D cubic taps in 1/32768


@functools.lru_cache(maxsize=None)
def warp_taps():
    """int64 [32, 32, 4, 4]: remap's 2-D INTER_CUBIC table (imgwarp.cpp initInterTab2D, fixed point), indexed by the y fraction,
    the x fraction, the tap row and the tap column: rint(fl(vy * vx) * 32768), saturated to int16, of the fp32 interpolateCubic weights at i/32, and
    where the 16 taps do not sum to 32768 the difference is taken off the smallest (sum too large) or added to the largest (too
    small) of the four taps at rows and columns 2 and 3, the first one found in row-major order.  OpenCV starts that search at
    ksize/2 = 2 for every kernel size, so for the 4 x 4 cubic kernel it is the lower-right 2 x 2 of the central 4 taps, not the
    central 2 x 2; taking rows and columns 1 and 2 instead differs from cv2 on 1/32-zoom warps."""
    t1 = np.stack([cubic_coeffs(np.float32(i) * np.float32(1.0 / INTER_TAB)) for i in range(INTER_TAB)])
    tab = np.zeros((INTER_TAB, INTER_TAB, 4, 4), np.int64)
    for i in range(INTER_TAB):
        for j in range(INTER_TAB):
            it = np.rint(np.multiply(t1[i][:, None], t1[j][None, :], dtype=np.float32) * np.float32(REMAP_COEF_SCALE))
            it = np.clip(it, -32768, 32767).astype(np.int64)                # saturate_cast<short>: 32768 at (0, 0) -> 32767
            diff = int(it.sum()) - REMAP_COEF_SCALE
            if diff:
                mk = Mk = (2, 2)
                for k in ((2, 2), (2, 3), (3, 2), (3, 3)):
                    if it[k] < it[mk]:
                        mk = k
                    elif it[k] > it[Mk]:
                        Mk = k
                it[Mk if diff < 0 else mk] -= diff
            tab[i, j] = it
    return tab


def warp_coords(M, xs, ys):
    """cv2.warpAffine's fixed-point source coordinates (imgwarp.cpp WarpAffineInvoker, WARP_INVERSE_MAP) of destination columns
    xs and rows ys: int64 (Xq, Yq) [len(ys), len(xs)] in 1/32 source pixel, X0 = cvRound((M01*y + M02)*1024) + 16 plus
    adelta[x] = cvRound(M00*x*1024), then >> 5 (fp64, round half to even, no contraction).  The source pixel is Xq >> 5 and the
    fraction Xq & 31.  cv2 then stores Xq >> 5 as int16; with replicated borders and source sides <= 32767 that saturation never
    changes a value, so it is not restated here."""
    M = np.asarray(M, np.float64)
    xs = np.asarray(xs, np.float64)
    ys = np.asarray(ys, np.float64)
    q = []
    for r in range(2):
        delta = np.rint(M[r, 0] * xs * AB_SCALE).astype(np.int64)
        row = np.rint((M[r, 1] * ys + M[r, 2]) * AB_SCALE).astype(np.int64) + AB_SCALE // INTER_TAB // 2
        q.append((row[:, None] + delta[None, :]) >> (AB_BITS - INTER_BITS))
    return q[0], q[1]


def warp_sample_u8(src, xq, yq):
    """remapBicubic<FixedPtCast<int, uchar, 15>> with BORDER_REPLICATE at fixed-point coordinates (xq, yq) (warp_coords): the
    16 taps around (xq >> 5, yq >> 5) with replicated borders, weighted by warp_taps()[yq & 31, xq & 31], (sum + 2^14) >> 15
    saturated.  src uint8 [h, w, cn] -> uint8 [*xq.shape, cn]."""
    h, w, cn = src.shape
    tab = warp_taps()
    ix, iy = xq >> INTER_BITS, yq >> INTER_BITS
    wt = tab[yq & (INTER_TAB - 1), xq & (INTER_TAB - 1)]                 # [..., 4, 4]
    s = src.astype(np.int64)
    acc = np.zeros(xq.shape + (cn,), np.int64)
    for r in range(4):
        yy = np.clip(iy + r - 1, 0, h - 1)
        for c in range(4):
            acc += s[yy, np.clip(ix + c - 1, 0, w - 1)] * wt[..., r, c][..., None]
    return np.clip((acc + (1 << 14)) >> 15, 0, 255).astype(np.uint8)


def warp_affine_cubic_u8(src, M, dsize):
    """cv2.warpAffine(src, M, dsize, flags=INTER_CUBIC | WARP_INVERSE_MAP, borderMode=BORDER_REPLICATE) for uint8 HWC images,
    OpenCV's own code path (IPP off): M (2 x 3) maps destination pixel indices to source pixel indices; dsize = (width, height)."""
    dw, dh = dsize
    xq, yq = warp_coords(M, np.arange(dw), np.arange(dh))
    return warp_sample_u8(np.asarray(src), xq, yq)
