"""CPU restatement of restoring a text line crop by crop (TEST INFRASTRUCTURE ONLY): what a user who cuts a line wider than the
32x512 LQ canvas by hand does around test_sr.py, which skips such lines (:107-110) -- run the script's data flow on each crop
and paste each crop's SR columns back into one image.  The per-crop arithmetic is oracle/image_ops.py's."""
import numpy as np

from .image_ops import preprocess_lq


def preprocess_lq_crop(img, a, b, out_h=32, out_w=512):
    """What a user who crops a long line by hand feeds test_sr.py: columns [a, b) of the image as an image of its own."""
    return preprocess_lq(np.ascontiguousarray(img[:, a:b]), out_h, out_w)


def stitch_sr(h, w, cuts, crops, sr_u8):
    """Write-back of a line restored crop by crop: sr_u8[k] is crop k's SR bytes [128, 2048, 3] (postprocess_sr of its line) and
    [cuts[k], cuts[k+1]) / crops[k] its core and crop in source columns.  Output column x of the h x w line sits at source column
    x*h/128 (ShowLQ's scale, test_sr.py:99), so core k fills output columns [r(cuts[k]), r(cuts[k+1])) with r(x) = rint(x*128/h),
    read from its SR bytes shifted left by r(crops[k][0]).  One crop: ShowSR = sr[:, :ShowLQ.shape[1]] (test_sr.py:201), which
    numpy clamps to the SR width."""
    r = lambda x: int(np.rint(x * (128 / h)))          # noqa: E731  (round half to even, like cv::resize's dsize)
    if len(crops) == 1:
        return sr_u8[0][:, :r(w)].copy()
    out = np.zeros((sr_u8[0].shape[0], r(w), sr_u8[0].shape[2]), np.uint8)
    for k, (a, _) in enumerate(crops):
        o0, o1 = r(cuts[k]), r(cuts[k + 1])
        out[:, o0:o1] = sr_u8[k][:, o0 - r(a):o1 - r(a)]
    return out
