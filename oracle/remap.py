"""CPU restatement of OpenCV's 8-bit remap with float maps (TEST INFRASTRUCTURE ONLY): cv2.remap(src, mapx, mapy,
INTER_CUBIC, borderMode=BORDER_REPLICATE) with fp32 maps on uint8 HWC images, OpenCV's OWN code path (IPP off).  remap first
turns the float maps into fixed-point coordinates in 1/32 pixel, Xq = cvRound(fl32(mapx) * 32) (round half to even; the
product is exact), and then samples exactly as warpAffine does: oracle.warp_affine.warp_sample_u8 at (Xq, Yq).  This is the
arithmetic mn_remap_curved_u8_batched computes (DESIGN.md section 7b, "Curved text regions").

PINNED: bit-exact against cv2 4.13.0 with ``cv2.ipp.setUseIPP(False)`` (tests/test_curved_regions.py), maps at exact multiples
of 1/64 included.
"""
import numpy as np

from .warp_affine import warp_sample_u8


def remap_coords(mapx, mapy):
    """int64 (Xq, Yq): the fixed-point coordinates rint(fl32(map) * 32) of remap's float maps."""
    f32 = np.float32
    xq = np.rint(np.multiply(np.asarray(mapx, f32), f32(32), dtype=f32)).astype(np.int64)
    yq = np.rint(np.multiply(np.asarray(mapy, f32), f32(32), dtype=f32)).astype(np.int64)
    return xq, yq


def remap_cubic_u8(src, mapx, mapy):
    """cv2.remap(src, mapx, mapy, INTER_CUBIC, borderMode=BORDER_REPLICATE) for a uint8 [h, w, cn] image and float maps of the
    destination's shape (fp64 maps are rounded to fp32 first, as the caller would store them)."""
    xq, yq = remap_coords(mapx, mapy)
    return warp_sample_u8(np.asarray(src), xq, yq)
