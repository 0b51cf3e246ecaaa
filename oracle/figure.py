"""CPU restatement of the four-panel figure the reference's test_sr.py writes per image (TEST INFRASTRUCTURE ONLY;
pipeline.restore_image(figure=True) / restore_images(figure=True), DESIGN.md section 7b).

Reference call sites (paths relative to the reference repo):
  test_sr.py:98       ShowLQ = cv2.resize(img, (0,0), fx=128/h, fy=128/h, INTER_CUBIC)       (panel 1, oracle/image_ops.py)
  test_sr.py:214-230  ShowLocs: the box markers drawn on a copy of ShowLQ                       (panel 2, marker_intervals)
  test_sr.py:198-201  ShowSR                                                                    (panel 3, the call's sr_u8)
  test_sr.py:206-211  prior = cv2.resize(hstack(prior*0.5+0.5), (S, 128)) * 255                (panel 4, resize_linear_f32)
  test_sr.py:231      cv2.imwrite(np.vstack((ShowLQ[:,:,::-1], ShowLocs[:,:,::-1], ShowSR, prior)))

Third-party arithmetic restated: OpenCV's own float32 INTER_LINEAR resize (imgproc/src/resize.cpp: fx = (float)((dx+0.5)*scale_x
- 0.5), sx = cvFloor(fx), fx -= sx, clamped to (0, 0) left of the image and to (sw-1, 0) right of it, then
S[sx]*(1-fx) + S[sx+1]*fx as fp32 multiply, multiply, add; the vertical pass is the identity at 128 -> 128 rows) and
cv2.imwrite's float -> uint8 conversion (cvRound: round half to even, saturated).  Pinned against cv2 4.13 (IPP off) in
tests/test_figure.py.
"""
import numpy as np

from .image_ops import resize_cubic_u8

PANEL = 128
PAD_X, PAD_Y = 2, 1             # test_sr.py:215,219: pad, padr


def show_width(h, w):
    """S: the width of ShowLQ, cv2's dsize for fx = 128/h (round half to even)."""
    return int(np.rint(w * (PANEL / h)))


def canvas_width(h, w):
    """Wc: 512 for a line that fits the LQ canvas, else 4*ceil(lq_w/4) (pipeline.whole_line_width)."""
    lq_w = int(np.rint(w * (32 / h)))
    return 512 if lq_w <= 512 else 4 * (-(-lq_w // 4))


def locs_f32(boxes, h, lq_width):
    """test_sr.py:118-134: boxes -> fp32 (centre, half-width) / lq_width, Python-float arithmetic stored as fp32."""
    out = np.zeros(2 * len(boxes), np.float32)
    for i, box in enumerate(boxes):
        x1, _, x2, _ = [float(v) for v in box]
        out[2 * i] = ((x1 + x2) / 2.0 * 32.0 / h) / lq_width
        out[2 * i + 1] = ((x2 - x1) / 2.0 * 32.0 / h) / lq_width
    return out


def marker_intervals(locs, S, M):
    """The columns test_sr.py:218-230 paints on a width-S row with img_max_width = M: (top, bottom) lists of [start, stop)
    column ranges, top = rows 0-63 (x = centre - width, pad 2), bottom = rows 64-127 (y = centre + width, pad 1).  Python slice
    rules: clipped to [0, S], a negative stop counts from the end, empty ranges dropped."""
    top, bot = [], []
    for c in range(len(locs) // 2):
        center, width = int(float(locs[2 * c]) * M), int(float(locs[2 * c + 1]) * M)
        x, y = center - width, center + width
        for out, a, b in ((top, max(0, x - PAD_X), min(x + PAD_X, M)), (bot, max(0, y - PAD_Y), min(y + PAD_Y, M))):
            start, stop, _ = slice(a, b).indices(S)
            if stop > start:
                out.append((start, stop))
    return top, bot


def show_locs(show_lq, top, bot):
    """ShowLocs (image channel order): ShowLQ with (255, 0, 0) at the top markers and (0, 0, 255) at the bottom markers."""
    out = show_lq.copy()
    for a, b in top:
        out[:64, a:b] = (255, 0, 0)
    for a, b in bot:
        out[64:, a:b] = (0, 0, 255)
    return out


def resize_linear_f32(src, dw):
    """cv2.resize(src, (dw, src.shape[0]), interpolation=INTER_LINEAR) for a float32 [H, sw, C] array (OpenCV's own path)."""
    h, sw, cn = src.shape
    if dw == sw:
        return src.copy()
    scale = 1.0 / (dw / sw)
    fx = ((np.arange(dw) + 0.5) * scale - 0.5).astype(np.float32)
    sx = np.floor(fx).astype(np.int64)
    fx = (fx - sx.astype(np.float32)).astype(np.float32)
    lo = sx < 0
    fx[lo], sx[lo] = 0, 0
    hi = sx >= sw - 1
    fx[hi], sx[hi] = 0, sw - 1
    s1 = np.minimum(sx + 1, sw - 1)
    a0 = (np.float32(1) - fx)[None, :, None]
    return src[:, sx] * a0 + src[:, s1] * fx[None, :, None]        # fp32 multiply, multiply, add (no FMA)


def prior_panel(priors, S):
    """Panel 4 at width S: priors fp32 [n, 3, 128, 128] (the generator's images, in [-1, 1]) -> uint8 [128, S, 3], channels
    NOT flipped (test_sr.py:206-211,231)."""
    p = priors.astype(np.float32) * np.float32(0.5) + np.float32(0.5)
    strip = np.ascontiguousarray(np.concatenate(list(p.transpose(0, 2, 3, 1)), axis=1))
    x = resize_linear_f32(strip, S) * np.float32(255)
    return np.clip(np.rint(x), 0, 255).astype(np.uint8)


def figure_bytes(img, boxes, priors, sr_u8):
    """The figure of one image: uint8 [512, W, 3], W = sr_u8's width -- ShowLQ, ShowLocs (both channel-flipped), sr_u8 and the
    prior panel, each computed at width S and cropped to W (DESIGN.md section 7b)."""
    h, w = img.shape[:2]
    S, wc = show_width(h, w), canvas_width(h, w)
    W = sr_u8.shape[1]
    lq = resize_cubic_u8(img, PANEL / h, PANEL / h)
    assert lq.shape[:2] == (PANEL, S) and W <= S, (lq.shape, S, W)
    top, bot = marker_intervals(locs_f32(boxes, h, wc), S, 4 * wc)
    locs = show_locs(lq, top, bot)
    return np.concatenate([lq[:, :W, ::-1], locs[:, :W, ::-1], sr_u8, prior_panel(priors, S)[:, :W]], axis=0)
