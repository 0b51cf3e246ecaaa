"""CPU restatement of the host pre/post-processing around the MARCONet nets (TEST INFRASTRUCTURE ONLY).

Reference call sites (paths relative to the reference repo):
  test_sr.py:98-111   LQ = cv2.resize(img, (0,0), fx=32/h, fy=32/h, INTER_CUBIC); zero-pad to 32x512;
                      ToTensor; Normalize((.5,.5,.5),(.5,.5,.5))
  test_sr.py:198-201  sr*0.5+0.5 -> HWC -> channel flip -> np.clip(.,0,1)*255 ; cv2.imwrite (:231) rounds to uint8

Third-party arithmetic outside the reference project: OpenCV ``cv2.resize(..., INTER_CUBIC)`` on 8-bit images
(requirements.txt: ``opencv-python``, no version pin; 4.13.0 is installed in this image).  This file restates OpenCV's OWN
implementation (modules/imgproc/src/resize.cpp: interpolateCubic with A = -0.75, 11-bit fixed-point tap tables, integer
horizontal pass, vertical pass = the baseline-SSE vector body ``VResizeCubicVec_32s8u`` in fp32 (separate multiply and add,
taps accumulated from row 3 to row 0, round-half-even) for the first floor(W*cn/8)*8 elements of a row and the fixed-point
scalar tail ``(sum + 2^21) >> 22`` for the rest).

PINNED: bit-exact against cv2 4.13.0 with ``cv2.ipp.setUseIPP(False)`` on ~2M random output pixels (tests/test_oracle_image.py,
tests/golden/resize_cubic.npz).  With Intel IPP enabled (the pip wheel's default on x86) cv2 dispatches this call to IPP's
closed-source cubic kernel, whose results differ from OpenCV's own by +-1 LSB on ~5 % of the pixels (and depend on the CPU);
that variant cannot be restated and is NOT what this file (or the CUDA kernel) reproduces.
"""
import numpy as np

COEF_BITS = 11
COEF_SCALE = 1 << COEF_BITS      # INTER_RESIZE_COEF_SCALE
SIMD_LANES = 8                   # v_int16 lanes of the baseline (SSE) build: the vector body handles multiples of 8 elements


def cubic_coeffs(x):
    """interpolateCubic (imgproc/src/resize.cpp), fp32, same operation order."""
    x = np.float32(x)
    a = np.float32(-0.75)
    one = np.float32(1)
    c0 = ((a * (x + one) - np.float32(5) * a) * (x + one) + np.float32(8) * a) * (x + one) - np.float32(4) * a
    c1 = ((a + np.float32(2)) * x - (a + np.float32(3))) * x * x + one
    c2 = ((a + np.float32(2)) * (one - x) - (a + np.float32(3))) * (one - x) * (one - x) + one
    c3 = one - c0 - c1 - c2
    return np.array([c0, c1, c2, c3], dtype=np.float32)


def taps_at(ds, scale):
    """tap_tables for the destination indices ds only: (ofs, taps) int64 [n], [n, 4]."""
    ds = np.asarray(ds, np.int64)
    f = ((ds + 0.5) * scale - 0.5).astype(np.float32)       # double arithmetic, then (float)
    s = np.floor(f)                                         # cvFloor
    f = np.subtract(f, s, dtype=np.float32)
    taps = np.rint(cubic_coeffs(f) * np.float32(COEF_SCALE)).astype(np.int64).T   # saturate_cast<short> = cvRound
    return s.astype(np.int64), taps.reshape(len(ds), 4)


def tap_tables(dst, scale):
    """Per destination index: first source index - 1 ... and the four 11-bit fixed-point taps (xofs/ialpha, yofs/ibeta)."""
    return taps_at(np.arange(dst), scale)


def dsize_for(h, w, fx, fy):
    """cv::resize with dsize = (0,0): saturate_cast<int>(size * scale) = round half to even."""
    return int(np.rint(h * fy)), int(np.rint(w * fx))


def resize_cubic_u8(img, fx, fy):
    """cv2.resize(img, (0, 0), fx=fx, fy=fy, interpolation=cv2.INTER_CUBIC) for uint8 HWC images (OpenCV's own code path)."""
    h, w, cn = img.shape
    dh, dw = dsize_for(h, w, fx, fy)
    if dh <= 0 or dw <= 0:
        raise ValueError("resize: empty destination (cv2 asserts !dsize.empty())")
    xo, xa = tap_tables(dw, 1.0 / fx)
    yo, ya = tap_tables(dh, 1.0 / fy)
    src = img.astype(np.int64)
    hbuf = np.zeros((h, dw, cn), np.int64)                  # HResizeCubic: int32 rows, replicate border
    for j in range(4):
        hbuf += src[:, np.clip(xo + j - 1, 0, w - 1), :] * xa[:, j][None, :, None]
    rows = [hbuf[np.clip(yo + j - 1, 0, h - 1)] for j in range(4)]
    beta = [ya[:, j][:, None, None] for j in range(4)]
    fixed = (rows[0] * beta[0] + rows[1] * beta[1] + rows[2] * beta[2] + rows[3] * beta[3] + (1 << (2 * COEF_BITS - 1))) >> (2 * COEF_BITS)
    fixed = np.clip(fixed, 0, 255).astype(np.uint8)
    scale = np.float32(1.0) / np.float32(COEF_SCALE * COEF_SCALE)
    bf = [(ya[:, j].astype(np.float32) * scale)[:, None, None] for j in range(4)]
    rf = [r.astype(np.float32) for r in rows]
    acc = rf[3] * bf[3]
    for k in (2, 1, 0):
        acc = rf[k] * bf[k] + acc                           # fp32 multiply, fp32 add (no FMA in the baseline build)
    vec = np.clip(np.rint(acc), 0, 255).astype(np.uint8)    # v_round + saturating pack
    out = fixed.reshape(dh, dw * cn).copy()
    nvec = (dw * cn // SIMD_LANES) * SIMD_LANES
    out[:, :nvec] = vec.reshape(dh, dw * cn)[:, :nvec]
    return out.reshape(dh, dw, cn)


def resize_cubic_rows(img, dsize, rows, cols=None, split_shift=0):
    """Destination rows ``rows`` (and columns ``cols``, default all) of cv2.resize(img, dsize, interpolation=INTER_CUBIC) for a
    uint8 HWC image, dsize = (dw, dh), computed without the rest of the destination: the dsize form's scales 1/((double)dw/w)
    and 1/((double)dh/h), and the vector body / fixed-point tail split decided by the element's index in the full destination
    row (the first floor(dw*cn/8)*8 elements are the vector body).  ``split_shift`` moves that split (negative controls only).
    Returns uint8 [len(rows), len(cols), cn]."""
    h, w, cn = img.shape
    dw, dh = dsize
    rows = np.asarray(rows, np.int64)
    cols = np.arange(dw) if cols is None else np.asarray(cols, np.int64)
    xo, xa = taps_at(cols, 1.0 / (dw / w))
    yo, ya = taps_at(rows, 1.0 / (dh / h))
    xi = [np.clip(xo + j - 1, 0, w - 1) for j in range(4)]
    nvec = (dw * cn // SIMD_LANES) * SIMD_LANES + split_shift
    vec_el = (cols[:, None] * cn + np.arange(cn)[None, :]) < nvec          # [len(cols), cn]
    scale = np.float32(1.0) / np.float32(COEF_SCALE * COEF_SCALE)
    out = np.empty((len(rows), len(cols), cn), np.uint8)
    step = max(1, (1 << 22) // (4 * max(len(cols), w) * cn))               # rows per chunk: bounded int64 buffers
    for r0 in range(0, len(rows), step):
        sl = slice(r0, r0 + step)
        yy = np.clip(yo[sl, None] + np.arange(4)[None, :] - 1, 0, h - 1)   # [n, 4] source rows
        src = img[yy.reshape(-1)].astype(np.int64)                          # [n*4, w, cn]
        hb = sum(src[:, xi[j], :] * xa[:, j][None, :, None] for j in range(4)).reshape(len(yy), 4, len(cols), cn)
        beta = ya[sl]
        fixed = sum(hb[:, j] * beta[:, j, None, None] for j in range(4))
        fixed = np.clip((fixed + (1 << (2 * COEF_BITS - 1))) >> (2 * COEF_BITS), 0, 255)
        bf = (beta.astype(np.float32) * scale)[:, :, None, None]
        rf = hb.astype(np.float32)
        acc = rf[:, 3] * bf[:, 3]
        for k in (2, 1, 0):
            acc = rf[:, k] * bf[:, k] + acc                                 # fp32 multiply, fp32 add (no FMA)
        vec = np.clip(np.rint(acc), 0, 255)
        out[sl] = np.where(vec_el[None], vec, fixed).astype(np.uint8)
    return out


def preprocess_lq(img, out_h=32, out_w=512):
    """test_sr.py:98-111: uint8 HWC image -> (LQ fp32 [1, 3, out_h, out_w] in [-1, 1], resized width)."""
    h = img.shape[0]
    lq = resize_cubic_u8(img, out_h / h, out_h / h)
    if lq.shape[1] > out_w:
        raise ValueError(f"LQ width {lq.shape[1]} exceeds {out_w} (test_sr.py:109 skips such images)")
    canvas = np.zeros((out_h, out_w, img.shape[2]), np.uint8)
    canvas[:, :lq.shape[1]] = lq
    t = canvas.transpose(2, 0, 1).astype(np.float32) / np.float32(255)       # ToTensor
    t = (t - np.float32(0.5)) / np.float32(0.5)                              # Normalize
    return t[None], lq.shape[1]


def postprocess_sr(sr):
    """test_sr.py:198-201,231: fp32 [B,3,H,W] in [-1,1] -> uint8 [B,H,W,3] with the channel flip; the bytes cv2.imwrite stores."""
    x = sr.astype(np.float32) * np.float32(0.5) + np.float32(0.5)
    x = np.transpose(x, (0, 2, 3, 1))[..., ::-1]
    x = np.clip(x, 0, 1) * np.float32(255.0)
    return np.clip(np.rint(x), 0, 255).astype(np.uint8)
