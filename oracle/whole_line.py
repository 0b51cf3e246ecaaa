"""CPU restatement of restoring a text line wider than the 32x512 LQ canvas with its SR decoder run ONCE on the whole line
(TEST INFRASTRUCTURE ONLY; pipeline.restore_images(whole_lines=True), DESIGN.md section 7b): the decoder's LQ of the whole image
and the columns of its output that form the line.  The resize arithmetic is oracle/image_ops.py's."""
import numpy as np

from .image_ops import preprocess_lq


def whole_line_width(h, w, out_h=32):
    """(lq_w, Wc) of a line decoded in one piece: lq_w = cv2's dsize width for fx = fy = out_h/h, and the decoder canvas
    Wc = 4*ceil(lq_w/4) -- the reference's stride-2 convs and x2 up-samples need W % 4 == 0 (its torch.cat fails otherwise)."""
    lq_w = int(np.rint(w * (out_h / h)))
    return lq_w, 4 * (-(-lq_w // 4))


def preprocess_lq_whole_line(img, out_h=32):
    """The decoder's LQ of a line wider than the canvas: the cubic resize of the WHOLE image to height out_h, zero-filled to
    Wc columns.  Returns (lq fp32 [1, 3, out_h, Wc], lq_w, Wc)."""
    lq_w, wc = whole_line_width(img.shape[0], img.shape[1], out_h)
    lq, got = preprocess_lq(img, out_h, wc)
    assert got == lq_w
    return lq, lq_w, wc


def whole_line_bytes(h, w, wc, sr_u8):
    """Output columns of a line decoded in one piece: [0, min(rint(w*128/h), 4*Wc)) of its SR bytes [128, 4*Wc, 3]."""
    return sr_u8[:, :min(int(np.rint(w * (128 / h))), 4 * wc)].copy()
