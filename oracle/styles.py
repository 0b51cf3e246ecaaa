"""numpy twin of pipeline.interpolate_styles (DESIGN.md section 7b, "Font-style interpolation"): the style lerp of test_w.py:107
with its rounding spelled out (mn_style_lerp), the 8-bit strip test_w.py:109-114 writes for one style (mn_prior_tiles_u8), and
the assembly of a content line wider than the canvas from its detection windows.
TEST INFRASTRUCTURE ONLY."""
import numpy as np


def scale_pair(s):
    """(s32, t32) = (float32(s), float32(1 - s)), 1 - s computed in double (Python floats) as the script's ``1 - scale``."""
    s = float(s)
    return np.float32(s), np.float32(1.0 - s)


def lerp(w1, w2, s):
    """fl(fl(w1 * s32) + fl(w2 * t32)) in fp32, each operation rounded on its own: torch's ``w1 * s + w2 * (1 - s)`` on fp32
    tensors and Python-float s (test_w.py:107)."""
    s32, t32 = scale_pair(s)
    a = np.multiply(np.asarray(w1, np.float32), s32, dtype=np.float32)
    b = np.multiply(np.asarray(w2, np.float32), t32, dtype=np.float32)
    return np.add(a, b, dtype=np.float32)


def strip(priors):
    """Generator images fp32 [n, 3, 128, 128] in [-1, 1] -> the uint8 [128, 128 n, 3] strip cv2.imwrite stores for
    hstack(prior*0.5 + 0.5) * 255.0 (test_w.py:109-114): cvRound with saturation, channels not flipped."""
    p = np.asarray(priors, np.float32)
    v = np.add(np.multiply(p, np.float32(0.5), dtype=np.float32), np.float32(0.5), dtype=np.float32)
    q = np.rint(np.multiply(v, np.float32(255.0), dtype=np.float32))
    return np.clip(q, 0, 255).astype(np.uint8).transpose(2, 0, 3, 1).reshape(p.shape[2], -1, 3)


def merge_with_windows(h, w, rows):
    """oracle.predict.merge that also returns, per merged character, (window, index among the window's kept characters)."""
    pairs = []
    for k, (labs, x1s, x2s) in enumerate(rows):
        for j, (lab, x1, x2) in enumerate(zip(labs, x1s, x2s)):
            lo = min(max(min(x1, x2), 0.0), float(w))
            hi = min(max(max(x1, x2), 0.0), float(w))
            pairs.append((int(lab), (lo + hi) / 2.0, (k, j)))
    order = sorted(range(len(pairs)), key=lambda i: (pairs[i][1], i))
    return [pairs[i][0] for i in order], [pairs[i][2] for i in order]


def assemble(window_priors, owners):
    """Strip of a wide content line at one style: window_priors[k] = the generator images of window k's kept characters
    (fp32 [n_k, 3, 128, 128]), owners = merge_with_windows' (window, index) per merged character."""
    return strip(np.stack([window_priors[k][j] for k, j in owners]))
