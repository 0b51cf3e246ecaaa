"""Self-contained line-restoration flow on top of the three modules (SURVEY.md section 8f rows n3 / n4).

The reference's ``test_sr.py`` takes character labels and boxes from a third-party YOLO + OCR front-end; the original
single-model flow uses the encoder's own predictions instead: CTC-style de-duplicated argmax labels (test_w.py:34-40) and
boxes converted from the encoder's (left, right) pairs to (centre, half-width) exactly as the training model does
(Train/tspgan/models/tspgan_model.py:331-337).  restore_lines decodes labels on the host, bit-exactly like the reference;
predict_characters decodes them, and the boxes, on the device (mn_decode_predictions) for images of any width.  Everything
numeric runs through the module API (and therefore through the CUDA kernels).
"""
import itertools
import math
import numbers
import threading
from typing import NamedTuple

import torch

ALPHABET_SIZE = 6735          # classes [0, 6735) are characters, 6735 is the CTC blank (utils/alphabets.py, test_w.py:38)


def decode_labels(logits_row, n_alphabet=ALPHABET_SIZE):
    """argmax over classes, drop repeats and blanks (reference test_w.py:34-40).  ``logits_row``: [T, 6736]."""
    idx = torch.max(logits_row.detach(), 1)[1].cpu()
    out = []
    for i in range(idx.shape[0]):
        if not (i > 0 and idx[i - 1] == idx[i]) and idx[i] < n_alphabet:
            out.append(int(idx[i]))
    return out


def lr_to_center_halfwidth(locs_lr):
    """(left, right) pairs -> (centre, half-width) pairs, fp32, as Train/tspgan/models/tspgan_model.py:331-337."""
    out = locs_lr.clone()
    out[:, 0::2] = (locs_lr[:, 1::2] + locs_lr[:, 0::2]) / 2.0
    out[:, 1::2] = (locs_lr[:, 1::2] - locs_lr[:, 0::2]) / 2.0
    return out


def load_checkpoint(model, path_or_dict, prefer_ema=True, strict=True):
    """Load a reference-format checkpoint into one of the three modules.

    Accepts the released files' layout ``{'params': sd}`` (test_sr.py:43-51), BasicSR training checkpoints that also carry
    ``'params_ema'`` (Train/options/train.yml:69 uses it for the generator), a bare state_dict, and DDP ``module.`` prefixes."""
    ck = torch.load(path_or_dict, map_location="cpu") if isinstance(path_or_dict, (str, bytes)) or hasattr(path_or_dict, "read") else path_or_dict
    if isinstance(ck, dict) and ("params" in ck or "params_ema" in ck):
        key = "params_ema" if (prefer_ema and "params_ema" in ck) else ("params" if "params" in ck else "params_ema")
        ck = ck[key]
    sd = {(k[7:] if k.startswith("module.") else k): v for k, v in ck.items()}
    return model.load_state_dict(sd, strict=strict)


@torch.no_grad()
def restore_lines(encoder, tspgan, sr, lq, labels=None, locs=None, max_chars=16, check_range=True):
    """LQ lines [B,3,32,512] -> dict(sr, prior, labels, locs, w, logits).

    labels: optional list (per line) of int64 [n_b, 1] tensors; default = the encoder's decoded labels (at most ``max_chars``).
    locs:   optional [B, 2*n] (centre, half-width) in units of the line width; default = converted encoder boxes.
    check_range: synchronise at the end and look at the fp16-range flags (ops.poll_range); when a tensor-core conv overflowed the
    fp16 hi/lo split its layer is re-routed to the bf16 split and the step is re-run until no run re-routes a layer (``_rerun``)
    -- the caller never sees the overflowed result."""
    def step():
        return _step(encoder, tspgan, sr, lq, labels, locs, max_chars=max_chars)
    return _rerun(step, lq.device) if check_range else step()


def _step(encoder, tspgan, sr, lq, labels, locs, max_chars=16, owner=None, lq_sr=None, widths=None):
    """One pass of the three modules over a batch -> restore_lines' dict.  The encoder reads ``lq`` (32x512 crops), TSPSRNet
    reads ``lq_sr`` (default: lq, one decoder line per crop) with ``widths``.  labels: one int64 [n_b, 1] tensor per decoder line
    (None: the encoder's decoded labels, at most ``max_chars``); locs None: the encoder's boxes.  One TSPGAN call generates every
    character; character j takes the style w[owner[j]] (default: the crop of its own line)."""
    logits, locs_lr, w = encoder(lq)
    if labels is None:
        labels = [torch.tensor(decode_labels(logits[b])[:max_chars], dtype=torch.long).reshape(-1, 1) for b in range(lq.shape[0])]
    if locs is None:
        locs = lr_to_center_halfwidth(locs_lr)
    counts = [int(l.shape[0]) for l in labels]
    dev = lq.device
    if sum(counts) > 0:
        if owner is None:
            owner = [b for b, c in enumerate(counts) for _ in range(c)]
        # through pinned memory, which the caching host allocator keeps until the copy has read it: a non_blocking copy straight
        # from this temporary gave styles that differed from run to run once the modules replay CUDA graphs
        styles = w.index_select(0, torch.tensor(owner, dtype=torch.long).pin_memory().to(dev, non_blocking=True))
        img, f64, f32_ = tspgan(styles=styles, labels=torch.cat([l for l in labels if l.shape[0] > 0]), noise=None)
        priors, p64, p32 = list(img.split(counts)), list(f64.split(counts)), list(f32_.split(counts))
    else:
        priors = [torch.zeros(0, 3, 128, 128, device=dev) for _ in counts]
        p64 = [torch.zeros(0, 256, 64, 64, device=dev) for _ in counts]
        p32 = [torch.zeros(0, 512, 32, 32, device=dev) for _ in counts]
    out = sr(lq if lq_sr is None else lq_sr, p64, p32, locs, widths=widths)
    return dict(sr=out, prior=priors, labels=labels, locs=locs, w=w, logits=logits)


def _rerun(step, device):
    """``step()``, then a synchronisation and a look at the fp16-range flags (ops.poll_range): a tensor-core conv that overflowed
    the fp16 hi/lo split has been re-routed to the bf16 split, and the step runs again.  One overflow can hide the next: its NaN
    becomes 0 after a ReLU, so a layer further on overflows only once the earlier one is re-routed (the encoder on a line
    x1000 takes five runs).  So the step re-runs for as long as a run re-routes a layer -- each layer at most once, hence a bounded loop -- and
    stops when a run raises no flag or flags only layers already on the bf16 split (their input itself held Inf / NaN).
    A re-route made inside the step counts too: every module forward polls the flags at its start without synchronising, so a
    later module of the same step (or a later chunk of a sweep) can already re-route a layer that overflowed earlier in it."""
    from . import ops
    while True:
        before = len(ops.RANGE_EVENTS)
        out = step()
        torch.cuda.synchronize(device)
        ops.poll_range(device)
        if not any(what == "rerouted to bf16x3" for _, what in ops.RANGE_EVENTS[before:]):
            return out


def boxes_to_locs(boxes, h, lq_width=512):
    """test_sr.py:118-134: detector boxes [x1, y1, x2, y2] in the ORIGINAL image -> locs [1, 2n] (centre, half-width) in units of
    the LQ canvas width.  Python-float arithmetic exactly as the script, stored as fp32."""
    locs = torch.zeros(1, len(boxes) * 2, dtype=torch.float32)
    for i, box in enumerate(boxes):
        x1, _, x2, _ = [float(v) for v in box]
        center, width = (x1 + x2) / 2.0, (x2 - x1) / 2.0
        locs[0, 2 * i] = (center * 32.0 / h) / lq_width
        locs[0, 2 * i + 1] = (width * 32.0 / h) / lq_width
    return locs


def figure_markers(locs, S, M):
    """The box markers of test_sr.py's ShowLocs panel (:214-230) on a width-S row, with img_max_width = M (2048 in the script):
    locs = one line's fp32 (centre, half-width) pairs.  Returns (top, bottom): the [start, stop) column ranges painted in rows
    0-63 (x = centre - width, pad 2) and rows 64-127 (y = centre + width, pad 1), by the script's own Python slice rules --
    clipped to [0, S], a negative stop counting from the end; empty ranges are dropped."""
    top, bot = [], []
    for c in range(len(locs) // 2):
        center, width = int(float(locs[2 * c]) * M), int(float(locs[2 * c + 1]) * M)
        x, y = center - width, center + width
        for out, a, b in ((top, max(0, x - 2), min(x + 2, M)), (bot, max(0, y - 1), min(y + 1, M))):
            start, stop, _ = slice(a, b).indices(S)
            if stop > start:
                out.append((start, stop))
    return top, bot


def _figure_markers_for(h, w, boxes):
    """figure_markers of an h x w image: locs = boxes_to_locs(boxes, h, Wc), M = 4*Wc, S = ShowLQ's width (DESIGN.md 7b)."""
    from .ops import round_half_even
    wc = whole_line_width(h, w)[1]
    return figure_markers(boxes_to_locs(boxes, h, wc)[0].tolist(), round_half_even(w * (128 / h)), 4 * wc)


def _to_host(flat):
    """One pinned device->host copy of ``flat``; returns the pinned tensor once the copy has finished."""
    pinned = torch.empty(flat.numel(), dtype=torch.uint8, pin_memory=True)
    pinned.copy_(flat, non_blocking=True)
    torch.cuda.current_stream(flat.device).synchronize()
    return pinned


@torch.no_grad()
def restore_image(encoder, tspgan, sr, img_u8, labels=None, boxes=None, figure=False):
    """One text-line image end to end on the device (the body of test_sr.py's loop, :98-201, with the labels / boxes the
    detector and OCR produced): uint8 [h, w, 3] image (host numpy / tensor or CUDA tensor) -> dict(sr_u8 [128, W, 3] uint8 bytes
    as cv2.imwrite would store them, cropped to the line's width; sr fp32; lq; lq_width).
    Pre- and post-processing run as CUDA kernels (mn_preprocess_lq_u8 / mn_postprocess_sr_u8).
    ``figure=True`` adds ``figure``: the uint8 [512, W, 3] image test_sr.py writes (:206-231; ShowLQ, ShowLocs, ShowSR, prior;
    DESIGN.md section 7b), composed on the device (mn_figure_u8); ``sr_u8`` is then its view ``figure[256:384]``.
    ``boxes=None``: the encoder predicts them (predict_characters), and the labels too when ``labels`` is None (given labels are
    paired in order with the predicted boxes); the result then gains ``labels`` and ``boxes``.  Only for a line that fits the
    canvas: restore_images predicts on lines of any width."""
    img = torch.as_tensor(img_u8)
    h = img.shape[0]
    predicted = None
    if boxes is None:
        img = _as_image(img, 0)
        lq_w = whole_line_width(h, img.shape[1])[0]
        if lq_w > 512:
            raise ValueError(f"LQ width {lq_w} exceeds 512: restore_image predicts characters only on a line that fits the "
                             f"canvas; restore_images(..., labels=None, boxes=None) reads lines of any width")
        labels, boxes = predicted = _use_prediction(0, labels, _predict(encoder, [img], 1, 64)[0])
    elif labels is None:
        raise ValueError("boxes without labels (predicted labels pair only with predicted boxes)")
    res = _restore_one(encoder, tspgan, sr, img, labels, boxes, figure)
    if predicted is not None:
        res["labels"], res["boxes"] = predicted
    return res


def _restore_one(encoder, tspgan, sr, img, labels, boxes, figure):
    """restore_image with labels and boxes."""
    from . import ops
    dev = next(encoder.parameters()).device
    h = img.shape[0]
    img = img.to(dev, non_blocking=True).contiguous()
    lq, lq_w = ops.preprocess_lq(img)
    locs_host = boxes_to_locs(boxes, h, lq.shape[-1])
    locs = locs_host.to(dev)
    _, _, w = encoder(lq)
    lab = torch.as_tensor(labels, dtype=torch.long).reshape(-1, 1)
    if lab.shape[0] == 0:
        raise ValueError("no character labels (test_sr.py:160-162 skips such images)")
    img_prior, f64, f32_ = tspgan(styles=w[:1].repeat(lab.shape[0], 1), labels=lab, noise=None)
    out = sr(lq, [f64], [f32_], locs)
    show_w = ops.round_half_even(img.shape[1] * (128 / h))    # ShowLQ = cv2.resize(img, fx=128/h, ...) (test_sr.py:98)
    if not figure:
        sr_u8 = ops.postprocess_sr(out)[0, :, :show_w]        # ShowSR = sr[:, :ShowLQ.shape[1]] (test_sr.py:201)
        return dict(sr_u8=sr_u8, sr=out, lq=lq, lq_width=lq_w, prior=img_prior, locs=locs)
    fig = torch.empty((512, min(show_w, out.shape[-1]), 3), dtype=torch.uint8, device=dev)
    ops.postprocess_sr_pieces(out, [(0, 0, fig[256:384])])
    top, bot = figure_markers(locs_host[0].tolist(), show_w, 4 * lq.shape[-1])
    ops.figure_panels([(img, fig, top, bot, list(img_prior))])
    return dict(sr_u8=fig[256:384], figure=fig, sr=out, lq=lq, lq_width=lq_w, prior=img_prior, locs=locs)


# ---------------------------------------------------------------------------------------------------------------------
# Lines of any width, many images per call.  test_sr.py restores one image per call and skips lines wider than the 32x512 LQ
# canvas (:107-110, "crop it into shorter segments").  Here every image is cut between characters into crops that fit the canvas,
# every crop of every image becomes one line of a batch, and each crop's core columns are written back into its image.  Each crop
# is exactly what the script computes on a hand-made crop (the resize sees the crop alone; its characters, boxes shifted).
# ---------------------------------------------------------------------------------------------------------------------
class Segment(NamedTuple):
    """One crop of a text-line image, in integer source columns: ``core`` [c_k, c_k+1) is the part of the line it restores,
    ``crop`` [a_k, b_k) what it reads (the core plus context on both sides), ``chars`` [i0, i1) the characters it owns and
    ``boxes`` their detector boxes shifted by -a_k."""
    core: tuple
    crop: tuple
    chars: tuple
    boxes: list


def plan_segments(h, w, boxes, canvas=512, context=16, labels=None, name="image"):
    """Cut an h x w text-line image with detector boxes [x1, y1, x2, y2] (source pixels, reading order) into Segments whose
    crops fit the 32 x ``canvas`` LQ canvas.

    An image that fits (round_half_even(w*32/h) <= canvas) is one segment: crop = core = the whole image.  Otherwise cuts
    0 = c_0 < ... < c_S = w never fall strictly inside a character span [floor(x1), ceil(x2)) (overlapping spans stay together);
    a crop is its core plus m = ceil(context*h/32) columns of context per side, clipped to the image, with (b-a)*32/h <= canvas-0.5.
    Greedy: each segment takes as many characters as fit and cuts in the middle of the gap that follows them; where the middle
    does not fit, or would leave the next character unable to fit its own segment, the cut moves to the nearest gap column that
    does.  A gap wider than the canvas yields segments without characters.  Characters belong to the segment whose core holds
    their span (zero-width boxes: their centre).
    Raises ValueError naming ``name`` and the character: a label count that differs from the box count, a box outside the image,
    box centres that decrease, a character (or run of overlapping characters) wider than the canvas with its context."""
    import math
    from .ops import round_half_even
    h, w, n = int(h), int(w), len(boxes)
    if h < 1 or w < 1:
        raise ValueError(f"{name}: empty image ({h}x{w})")
    if labels is not None and len(labels) != n:
        raise ValueError(f"{name}: {len(labels)} labels for {n} boxes")
    spans, centres = [], []
    for i, box in enumerate(boxes):
        x1, _, x2, _ = [float(v) for v in box]
        if not 0 <= x1 <= x2 <= w:
            raise ValueError(f"{name}, character {i}: box {[float(v) for v in box]} is outside the image (columns [0, {w}])")
        c = (x1 + x2) / 2.0
        if centres and c < centres[-1]:
            raise ValueError(f"{name}, character {i}: box centre {c} lies left of character {i - 1}'s ({centres[-1]}); "
                             f"boxes must be in reading order")
        spans.append((math.floor(x1), math.ceil(x2)))
        centres.append(c)
    if round_half_even(w * (32 / h)) <= canvas:
        return [Segment((0, w), (0, w), (0, n), [list(b) for b in boxes])]
    m = -(-context * h // 32)
    maxw = (2 * canvas - 1) * h // 64                    # widest crop: cols * 32 / h <= canvas - 0.5
    if maxw <= 2 * m:
        raise ValueError(f"{name}: {context} pixels of context leave no room in a {canvas}-pixel canvas")

    def crop_cols(lo, hi):                               # width of the crop around core [lo, hi)
        return min(w, hi + m) - max(0, lo - m)

    clusters = []                                        # [start, end, first char, last char] of runs of overlapping spans
    for i in sorted(range(n), key=lambda i: spans[i]):
        s, e = spans[i]
        if e <= s:
            continue
        if clusters and s < clusters[-1][1]:
            cl = clusters[-1]
            cl[1], cl[2], cl[3] = max(cl[1], e), min(cl[2], i), max(cl[3], i)
        else:
            clusters.append([s, e, i, i])
    for s, e, i0, i1 in clusters:
        if crop_cols(s, e) > maxw:
            who = f"character {i0}" if i0 == i1 else f"characters {i0} to {i1} (overlapping boxes)"
            raise ValueError(f"{name}, {who}: columns [{s}, {e}) with {m} columns of context per side are wider than the "
                             f"{canvas}-pixel LQ canvas at height {h}; a single character cannot be split")
    # gaps between clusters: closed ranges of columns where a cut may fall, and the cluster that follows each
    gaps = []
    lo = 0
    for s, e, _, _ in clusters:
        gaps.append((lo, s, e))
        lo = e
    gaps.append((lo, w, None))
    cuts = [0]
    while cuts[-1] < w:
        c = cuts[-1]
        a = max(0, c - m)
        if w - a <= maxw:
            cuts.append(w)
            break
        cmax = a + maxw - m                              # furthest cut whose crop fits
        L, R, nxt_end = [g for g in gaps if g[0] <= cmax and g[1] > c][-1]
        need = L
        if nxt_end is not None:                          # the segment that starts at the cut must reach the next cluster's end
            need = max(L, min(w, nxt_end + m) - maxw + m)
        cuts.append(min(max((L + R) // 2, need, L, c + 1), R, cmax))
    import bisect
    owner = [min(len(cuts) - 2, bisect.bisect_right(cuts, ctr) - 1) for ctr in centres]
    segs = []
    for k in range(len(cuts) - 1):
        i0 = bisect.bisect_left(owner, k)
        i1 = bisect.bisect_right(owner, k)
        a, b = max(0, cuts[k] - m), min(w, cuts[k + 1] + m)
        segs.append(Segment((cuts[k], cuts[k + 1]), (a, b), (i0, i1), [[bx[0] - a, bx[1], bx[2] - a, bx[3]] for bx in boxes[i0:i1]]))
    return segs


def stitch_pieces(h, w, segments, sr_width=2048):
    """Where each segment's SR columns land: (output width, [(segment index, out_x0, src_x0, width)]).  Output column x of an
    h x w image lies at source column x*h/128 (ShowLQ's scale, test_sr.py:99): segment k fills [r(c_k), r(c_k+1)) from its own SR
    output shifted left by r(a_k), r(x) = round_half_even(x*128/h).  A single-segment image is restore_image's
    ``sr[:, :round_half_even(w*128/h)]``, clamped to the SR width as that slice is."""
    from .ops import round_half_even

    def r(x):
        return round_half_even(x * (128 / h))
    if len(segments) == 1:
        width = min(r(w), sr_width)
        return width, [(0, 0, 0, width)]
    out = []
    for k, s in enumerate(segments):
        o0, o1 = r(s.core[0]), r(s.core[1])
        if o1 > o0:
            out.append((k, o0, o0 - r(s.crop[0]), o1 - o0))
    return r(w), out


_TLS = threading.local()


def _staging(nbytes, device):
    """Per-thread, per-device pinned host buffer for the host->device copy of a batch's images, reused once its last copy (the
    event, recorded after it) has finished."""
    stages = _TLS.__dict__.setdefault("stages", {})
    st = stages.get(device.index)
    if st is None or st[0].numel() < nbytes:
        st = (torch.empty(max(nbytes, 1 << 20), dtype=torch.uint8, pin_memory=True), torch.cuda.Event())
        stages[device.index] = st
    else:
        st[1].synchronize()
    return st


def _as_image(img, i):
    if not isinstance(img, torch.Tensor):
        import numpy as np
        img = torch.from_numpy(np.ascontiguousarray(img))
    if img.dtype != torch.uint8 or img.dim() != 3 or img.shape[2] != 3 or img.shape[0] < 1 or img.shape[1] < 1:
        raise ValueError(f"image {i}: expected a uint8 [h, w, 3] image, got {img.dtype} {tuple(img.shape)}")
    return img


def _device_images(ids, imgs, dev):
    """The batch's images on the device: CUDA images as they are (dense pixels), host images through ONE pinned host->device
    copy.  Returns {image index: uint8 CUDA view}."""
    dimg, host = {}, []
    for i in ids:
        t = imgs[i]
        if not t.is_cuda:
            host.append(i)
            continue
        t = t.to(dev)
        if t.stride(2) != 1 or t.stride(1) != 3:
            t = t.contiguous()
        dimg[i] = t
    if host:
        nbytes = sum(imgs[i].numel() for i in host)
        stage, ev = _staging(nbytes, dev)
        o = 0
        for i in host:
            stage[o:o + imgs[i].numel()].view(imgs[i].shape).copy_(imgs[i])
            o += imgs[i].numel()
        dbuf = stage[:nbytes].to(dev, non_blocking=True)
        ev.record()
        o = 0
        for i in host:
            dimg[i] = dbuf[o:o + imgs[i].numel()].view(imgs[i].shape)
            o += imgs[i].numel()
    return dimg


def whole_line_width(h, w, canvas=512):
    """(lq_w, Wc): the LQ width of an h x w image (cv2's dsize for fx = fy = 32/h) and the width of its decoder line.  A line that
    fits the canvas keeps the 512 canvas; a wider one decodes in one piece at Wc = 4*ceil(lq_w/4) (the reference's stride-2 convs
    and x2 up-samples need W % 4 == 0)."""
    from .ops import round_half_even
    lq_w = round_half_even(w * (32 / h))
    return lq_w, (canvas if lq_w <= canvas else 4 * (-(-lq_w // 4)))


def pack_by_columns(widths, max_lines, canvas=512):
    """Decoder batches of lines with their own widths: lines sorted by width, a batch of k lines only while
    k * (its widest line) <= max_lines * canvas (peak activation memory stays that of max_lines canvas-wide lines); a line wider
    than that forms a batch of its own.  Returns lists of indices into ``widths``."""
    order = sorted(range(len(widths)), key=lambda j: widths[j])
    batches, cur = [], []
    for j in order:
        if cur and (len(cur) + 1) * widths[j] > max_lines * canvas:
            batches.append(cur)
            cur = []
        cur.append(j)
    if cur:
        batches.append(cur)
    return batches


class LineBatch(NamedTuple):
    """One batch of restore_images, planned on the host (plan_batches).  Images are indices into the call's lists."""
    crops: list         # encoder rows: (image, a, b), source columns resized onto the 32x512 canvas
    lines: list         # decoder lines: (image, x0, x1), source columns
    widths: list        # each decoder line's LQ width: Wc for a whole line wider than the canvas, else 512
    counts: list        # characters per decoder line
    labels: list        # the batch's labels, line by line, each line's in label order
    owner: list         # the encoder row (index into crops) whose style each character takes: the crop that owns it
    locs: torch.Tensor  # fp32 [lines, 2*max(1, max(counts))]: boxes_to_locs of each line's boxes at its width, zero-padded
    pieces: list        # stitch: (line, src_x0, image, out_x0, width)
    done: list          # images whose last line is in this batch: their figures are composed after it
    reuse: bool         # every decoder line is its own encoder crop at 512: the decoder reads the encoder's LQ


def plan_batches(shapes, labels, boxes, plans, max_lines, whole_lines=False):
    """restore_images' batches, on the host.  shapes / labels / boxes / plans: per image, its (h, w), label list, detector boxes
    and plan_segments' Segments; an image whose plan is None is left out.  A decoder line is one crop at 512 or, with
    ``whole_lines``, a whole image wider than the canvas at Wc (whole_line_width).  Lines keep image and segment order;
    pack_by_columns forms the batches (with every width 512: consecutive chunks of max_lines lines).
    Returns ({image: output width}, [LineBatch])."""
    from .ops import round_half_even
    out_w, lines = {}, []       # (image, x0, x1, width, segment indices, boxes, [(src_x0, out_x0, width)])
    for i, segs in enumerate(plans):
        if segs is None:
            continue
        h, w = shapes[i]
        wc = whole_line_width(h, w)[1] if whole_lines else 512
        if wc > 512:
            out_w[i] = min(round_half_even(w * (128 / h)), 4 * wc)
            lines.append((i, 0, w, wc, range(len(segs)), boxes[i], [(0, 0, out_w[i])]))
            continue
        out_w[i], pieces = stitch_pieces(h, w, segs)
        for k, s in enumerate(segs):
            lines.append((i, *s.crop, 512, [k], s.boxes, [(src, x0, wd) for kk, x0, src, wd in pieces if kk == k]))
    groups = pack_by_columns([line[3] for line in lines], max_lines)
    last = {lines[j][0]: g for g, idx in enumerate(groups) for j in idx}
    batches = []
    for g, idx in enumerate(groups):
        crops, dec, widths, counts, labs, owner, pieces = [], [], [], [], [], [], []
        for b, j in enumerate(idx):
            i, x0, x1, wd, ks, _, pcs = lines[j]
            n0 = len(labs)
            for k in ks:
                s = plans[i][k]
                owner += [len(crops)] * (s.chars[1] - s.chars[0])
                labs += labels[i][s.chars[0]:s.chars[1]]
                crops.append((i, *s.crop))
            dec.append((i, x0, x1))
            widths.append(wd)
            counts.append(len(labs) - n0)
            pieces += [(b, src, i, o0, pw) for src, o0, pw in pcs]
        locs = torch.zeros(len(idx), 2 * max(1, max(counts)), dtype=torch.float32)
        for b, j in enumerate(idx):
            if counts[b]:
                locs[b, :2 * counts[b]] = boxes_to_locs(lines[j][5], shapes[lines[j][0]][0], widths[b])[0]
        done = [i for i in dict.fromkeys(i for i, _, _ in dec) if last[i] == g]
        batches.append(LineBatch(crops, dec, widths, counts, labs, owner, locs, pieces, done,
                                 crops == dec and max(widths) == 512))
    return out_w, batches


# ---------------------------------------------------------------------------------------------------------------------
# Predicted characters (DESIGN.md section 7b).  Without a detector, the encoder's own CTC labels and (left, right) boxes stand in
# for test_sr.py's YOLO + OCR front-end: the line is read through detection windows that fit the canvas, each window's characters
# are decoded on the device (mn_decode_predictions), and a character belongs to the window whose core holds its box centre.
# ---------------------------------------------------------------------------------------------------------------------
class Window(NamedTuple):
    """One detection window of a text-line image: ``crop`` [a, b) the source columns the encoder reads (resized onto the 32x512
    canvas as test_sr.py resizes a hand-cut crop), ``core`` [lo, hi) the source columns whose predicted characters it owns."""
    crop: tuple
    core: tuple


def plan_windows(h, w, canvas=512, overlap=64):
    """Where the encoder looks on an h x w image.  A line that fits (round_half_even(w*32/h) <= canvas) is one window (0, w) whose
    core is the whole real line.  A wider one: windows of W* = (2*canvas-1)*h // 64 source columns (the widest crop that fits the
    canvas, as in plan_segments) at stride s = W* - v, v = ceil(overlap*h/32) (``overlap`` LQ pixels), K = 1 + ceil((w-W*)/s)
    windows, the last one [w - W*, w).  The core boundary between windows k and k+1 is floor((a_k+1 + b_k)/2); the first core
    starts at -inf and the last ends at +inf, so the cores partition the real line."""
    from .ops import round_half_even
    h, w = int(h), int(w)
    if h < 1 or w < 1:
        raise ValueError(f"empty image ({h}x{w})")
    if not 0 <= overlap <= 256:
        raise ValueError(f"overlap must lie in [0, 256] LQ pixels, got {overlap}")
    inf = float("inf")
    if round_half_even(w * (32 / h)) <= canvas:
        return [Window((0, w), (-inf, inf))]
    wmax = (2 * canvas - 1) * h // 64
    s = wmax - (-(-int(overlap) * h // 32))
    k = 1 + -(-(w - wmax) // s)
    crops = [(j * s, j * s + wmax) for j in range(k - 1)] + [(w - wmax, w)]
    cuts = [-inf] + [(crops[j + 1][0] + crops[j][1]) // 2 for j in range(k - 1)] + [inf]
    return [Window(crops[j], (cuts[j], cuts[j + 1])) for j in range(k)]


def merge_predictions(h, w, windows, rows):
    """One image's characters from its windows' decoded rows: rows[k] = (labels, x1s, x2s), the characters window k kept in
    decode order with their boxes in source columns.  Concatenated in window order, each box clamped to the image
    ([clamp(min(x1, x2), 0, w), 0, clamp(max(x1, x2), 0, w), h]), then stable-sorted by box centre (pairs stay together).
    Returns (labels, boxes)."""
    merged = _merge_windows(h, w, windows, rows)
    return [m[0] for m in merged], [m[1] for m in merged]


def _merge_windows(h, w, windows, rows):
    """merge_predictions' characters as (label, box, index of the window that kept it), in merged order."""
    pairs = []
    for k, ((labs, x1s, x2s), _) in enumerate(zip(rows, windows)):
        for lab, x1, x2 in zip(labs, x1s, x2s):
            lo, hi = min(max(min(x1, x2), 0.0), float(w)), min(max(max(x1, x2), 0.0), float(w))
            pairs.append((int(lab), [lo, 0, hi, h], k))
    pairs.sort(key=lambda p: (p[1][0] + p[1][2]) / 2.0)
    return pairs


def _predict(encoder, imgs, max_lines, overlap):
    """predict_characters on validated uint8 [h, w, 3] tensors."""
    from . import ops
    dev = next(encoder.parameters()).device
    plans = [plan_windows(im.shape[0], im.shape[1], overlap=overlap) for im in imgs]
    rows = [(i, k) for i, p in enumerate(plans) for k in range(len(p))]
    if not rows:
        return []
    with torch.cuda.device(dev):
        table, out = ops.prediction_table([(plans[i][k].crop[0], 16.0 * imgs[i].shape[0], *plans[i][k].core) for i, k in rows], dev)
        dimg = _device_images(range(len(imgs)), imgs, dev)
        for r0 in range(0, len(rows), max_lines):
            batch = rows[r0:r0 + max_lines]
            lq, _ = ops.preprocess_lq_crops([(dimg[i], *plans[i][k].crop) for i, k in batch])
            logits, locs_lr, _ = encoder(lq)
            ops.decode_predictions(logits, locs_lr, table, r0)
        rec = _to_host(out).numpy().view(ops.pred_dtype())
    res, r = [], 0
    for i, p in enumerate(plans):
        dec = []
        for k in range(len(p)):
            n = int(rec[r]["n_kept"])
            dec.append((rec[r]["label"][:n].tolist(), rec[r]["x1"][:n].tolist(), rec[r]["x2"][:n].tolist()))
            r += 1
        labels, boxes = merge_predictions(imgs[i].shape[0], imgs[i].shape[1], p, dec)
        res.append(dict(labels=labels, boxes=boxes, windows=p))
    return res


@torch.no_grad()
def predict_characters(encoder, images, max_lines=8, overlap=64):
    """The characters TextContextEncoderV2 predicts on text-line images of any width, in place of a detector + OCR front-end
    (the reference's single-model flow, SURVEY.md section 8f row n3; DESIGN.md section 7b, "Predicted characters").

    images: uint8 [h, w, 3] numpy arrays or CPU / CUDA tensors.  Each image is read through plan_windows' detection windows, each
    window resized onto the 32x512 canvas exactly as preprocess_lq_crops resizes a crop.  Per batch of at most ``max_lines``
    windows (image, then window order): one crop launch, the encoder, one mn_decode_predictions launch (argmax, CTC collapse,
    first 16 characters, boxes in source columns, core test) into one device table for the call; then one pinned device->host
    copy and one synchronisation.  Host images go to the device once, in one pinned copy.
    Returns one dict per image: labels (ints), boxes ([x1, 0, x2, h] floats, clamped to the image, sorted by centre; what
    restore_images takes) and windows (the plan)."""
    if max_lines < 1:
        raise ValueError("max_lines must be >= 1")
    return _predict(encoder, [_as_image(im, i) for i, im in enumerate(images)], max_lines, overlap)


def _use_prediction(i, lab, pred):
    """The labels and boxes image i restores with, given its prediction: the predicted ones, or the given labels paired in
    order with the predicted boxes (the reference README's manual-label mode)."""
    if lab is None:
        if not pred["labels"]:
            raise ValueError(f"image {i}: the encoder predicted no character")
        return list(pred["labels"]), pred["boxes"]
    lab = [int(v) for v in torch.as_tensor(lab, dtype=torch.long).reshape(-1).tolist()]
    if len(lab) != len(pred["labels"]):
        raise ValueError(f"image {i}: {len(lab)} labels given, the encoder predicted {len(pred['labels'])} characters")
    return lab, pred["boxes"]


@torch.no_grad()
def restore_images(encoder, tspgan, sr, images, labels=None, boxes=None, max_lines=8, context=16, skip_invalid=False,
                   to_host=False, whole_lines=False, figure=False, overlap=64):
    """Text-line images of any sizes end to end, batched: the flow of restore_image for every image, each cut into crops that
    fit the 32x512 LQ canvas (plan_segments) and every crop of every image run as one line of a batch of at most ``max_lines``.

    images: uint8 [h_i, w_i, 3] numpy arrays or CPU / CUDA tensors; labels / boxes: one list per image, as restore_image takes.
    Every image is planned and validated before any launch (a label outside the generator's classes raises IndexError, as the
    module would); with ``skip_invalid`` a bad image's entry becomes dict(error=...) and the others still run.  Per batch: one
    host->device copy of the batch's host images through pinned memory, one crop kernel (mn_preprocess_lq_u8_batched), the
    encoder, one TSPGAN call for all characters (each crop's characters take that crop's style w, as on a hand-made crop),
    TSPSRNet, a synchronisation and ops.poll_range (the batch re-runs while a run re-routes a layer for fp16 range, see
    ``_rerun``), then one stitch kernel (mn_postprocess_sr_u8_pieces) into the images' outputs.
    Returns one dict per image: sr_u8 (uint8 [128, W_i, 3], W_i = round_half_even(w_i*128/h_i), on the device, or numpy through
    one pinned device->host copy with ``to_host``) and segments (the plan).  A single-segment image gives restore_image's bytes.

    ``whole_lines=True`` decodes every line wider than the canvas (lq_w = round_half_even(w*32/h) > 512) in ONE piece, so that no
    column sees a crop edge: its decoder LQ is the cubic resize of the whole image to height 32, zero-filled to
    Wc = 4*ceil(lq_w/4) columns, its locs are boxes_to_locs(boxes, h, Wc), and its output is columns
    [0, min(round_half_even(w*128/h), 4*Wc)) of TSPSRNet(lq, [p64], [p32], locs) -- the reference module run on the whole line.
    The encoder, whose patch and positional embeddings are sized for the 32x512 canvas, still runs on the plan's crops, and each
    character's prior takes the style w of the crop that owns it.  Lines that fit the canvas are computed as without the flag.
    Decoder lines of different widths share a batch (TSPSRNet's ``widths``); a batch holds k lines only while
    k * (its widest Wc) <= max_lines * 512.  Per batch: one host->device copy, one crop kernel for the encoder crops, one for
    the decoder lines when the batch holds a line wider than the canvas, the encoder, one TSPGAN call, one ragged TSPSRNet call,
    the fp16-range re-run, one stitch kernel.  Both modes run the batches of plan_batches through the same loop.

    ``figure=True`` (either mode) adds ``figure`` to every result: the uint8 [512, W_i, 3] image test_sr.py writes (:206-231;
    DESIGN.md section 7b) -- ShowLQ and ShowLocs (markers at locs = boxes_to_locs(boxes, h, Wc), img_max_width = 4*Wc), the
    image's sr_u8, and the priors this call generated (each character's in the style of the crop that owns it), all cropped to
    sr_u8's width.  ``sr_u8`` becomes the view ``figure[256:384]``, its bytes unchanged.  The batch that holds an image's last
    crop composes its figure: one more launch (mn_figure_u8) per batch, and the prior images are kept until then.  With
    ``to_host`` the figures come back through the same single pinned copy.  Error entries have no figure.

    Without a detector: ``labels`` / ``boxes`` may be None, or lists with None entries.  An image whose boxes are None is first
    read by the encoder (predict_characters, with ``max_lines`` and ``overlap``): labels None takes the predicted labels and
    boxes; given labels are paired in order with the predicted boxes (their counts must match).  Labels None with given boxes
    is a ValueError.  The call then is restore_images(images, labels, boxes) with the predicted values, every option applying on
    top, and those results gain ``labels`` and ``boxes`` (what the restoration used).  No character predicted, a count mismatch
    or a predicted box plan_segments rejects are ValueErrors naming the image (error entries with ``skip_invalid``).  Images
    with both labels and boxes given do not enter the prediction stage."""
    from . import ops
    n = len(images)
    labels = [None] * n if labels is None else labels
    boxes = [None] * n if boxes is None else boxes
    if not (len(labels) == len(boxes) == n):
        raise ValueError(f"{n} images, {len(labels)} label lists, {len(boxes)} box lists")
    if max_lines < 1:
        raise ValueError("max_lines must be >= 1")
    dev = next(encoder.parameters()).device
    n_cls = tspgan.TextGenerator.input_text.TextEmbeddings.shape[0]
    results, imgs, labs, plans = [None] * n, [None] * n, [None] * n, [None] * n
    boxes, predicted, ask = list(boxes), {}, {}
    for i in range(n):                                   # the prediction stage: images without boxes
        try:
            if boxes[i] is None:
                ask[i] = _as_image(images[i], i)
            elif labels[i] is None:
                raise ValueError(f"image {i}: boxes without labels (predicted labels pair only with predicted boxes)")
        except ValueError as e:
            if not skip_invalid:
                raise
            results[i] = dict(error=f"{type(e).__name__}: {e}")
    for i, pred in zip(ask, _predict(encoder, list(ask.values()), max_lines, overlap) if ask else []):
        try:
            predicted[i] = _use_prediction(i, labels[i], pred)
            boxes[i] = predicted[i][1]
        except ValueError as e:
            if not skip_invalid:
                raise
            results[i] = dict(error=f"{type(e).__name__}: {e}")
    for i in range(n):
        if results[i] is not None:
            continue
        try:
            img = _as_image(images[i], i)
            lab = predicted[i][0] if i in predicted else \
                [int(v) for v in torch.as_tensor(labels[i], dtype=torch.long).reshape(-1).tolist()]
            if not lab:
                raise ValueError(f"image {i}: no character labels (test_sr.py:168-170 skips such images)")
            segs = plan_segments(img.shape[0], img.shape[1], boxes[i], labels=lab, context=context, name=f"image {i}")
            bad = [j for j, v in enumerate(lab) if not 0 <= v < n_cls]
            if bad:
                raise IndexError(f"image {i}, character {bad[0]}: label {lab[bad[0]]} outside [0, {n_cls}) "
                                 f"(reference: empty embedding slice, networks.py:211)")
        except (ValueError, IndexError) as e:
            if not skip_invalid:
                raise
            results[i] = dict(error=f"{type(e).__name__}: {e}")
            continue
        imgs[i], labs[i], plans[i] = img, lab, segs
    if all(p is None for p in plans):
        return results
    out_w, batches = plan_batches([None if im is None else im.shape[:2] for im in imgs], labs, boxes, plans, max_lines,
                                  whole_lines)
    rows = 512 if figure else 128
    with torch.cuda.device(dev):
        offs, total = {}, 0
        for i, wd in out_w.items():
            offs[i] = total
            total += rows * wd * 3
        flat = torch.empty(total, dtype=torch.uint8, device=dev)
        figs = {i: flat[o:o + rows * out_w[i] * 3].view(rows, out_w[i], 3) for i, o in offs.items()}
        outs = {i: f[256:384] for i, f in figs.items()} if figure else figs
        priors = {i: [] for i in out_w}
        for bt in batches:
            dimg = _device_images(dict.fromkeys(i for i, _, _ in bt.lines), imgs, dev)
            lq, _ = ops.preprocess_lq_crops([(dimg[i], a, b) for i, a, b in bt.crops])
            lq_sr = lq if bt.reuse else ops.preprocess_lq_crops([(dimg[i], a, b) for i, a, b in bt.lines], out_w=max(bt.widths))[0]
            lab = list(torch.tensor(bt.labels, dtype=torch.long).reshape(-1, 1).split(bt.counts))
            res = _rerun(lambda: _step(encoder, tspgan, sr, lq, lab, bt.locs, owner=bt.owner, lq_sr=lq_sr, widths=bt.widths), dev)
            if bt.pieces:
                ops.postprocess_sr_pieces(res["sr"], [(b, src, outs[i][:, x0:x0 + wd]) for b, src, i, x0, wd in bt.pieces])
            if figure:
                for (i, _, _), p in zip(bt.lines, res["prior"]):      # lines in label order: the priors in label order
                    priors[i] += list(p)
                if bt.done:
                    ops.figure_panels([(dimg[i], figs[i]) + _figure_markers_for(*imgs[i].shape[:2], boxes[i]) + (priors.pop(i),)
                                       for i in bt.done])
        if to_host:
            pinned = _to_host(flat)
            figs = {i: pinned[o:o + rows * out_w[i] * 3].view(rows, out_w[i], 3).numpy() for i, o in offs.items()}
            outs = {i: f[256:384] for i, f in figs.items()} if figure else figs
    for i in out_w:
        results[i] = dict(sr_u8=outs[i], segments=plans[i])
        if figure:
            results[i]["figure"] = figs[i]
        if i in predicted:
            results[i]["labels"], results[i]["boxes"] = predicted[i]
    return results


# ---------------------------------------------------------------------------------------------------------------------
# Font-style interpolation (DESIGN.md section 7b, "Font-style interpolation"): test_w.py's mode, batched.  The script encodes two
# images, decodes image 1's characters, and generates them in the style w1*s + w2*(1-s) for 11 scales, one generator call per
# scale.  Here every (pair, scale, character) style row of a call is built by one mn_style_lerp launch, the generator runs over
# chunks of those rows and mn_prior_tiles_u8 writes each image into its strip as the 8-bit PNG bytes the script stores.
# ---------------------------------------------------------------------------------------------------------------------
class SweepRow(NamedTuple):
    """One generator image of interpolate_styles: character ``char`` of pair ``pair``'s strip ``scale``, in the style
    w[w1]*s + w[w2]*(1-s) (rows of the call's encoder style table)."""
    pair: int
    scale: int
    char: int
    w1: int
    w2: int
    label: int


def plan_sweep(chars, donors, n_scales, max_chars):
    """interpolate_styles' generator rows, on the host.  chars[p]: pair p's characters in strip order as (style row, label), or
    None for a pair left out; donors[p]: its donor's style row.  Returns (rows in (pair, scale, character) order, chunks [r0, r1)
    of at most ``max_chars`` consecutive rows: one generator call each)."""
    rows = [SweepRow(p, k, c, w1, donors[p], lab) for p, cs in enumerate(chars) if cs
            for k in range(n_scales) for c, (w1, lab) in enumerate(cs)]
    return rows, [(r0, min(r0 + max_chars, len(rows))) for r0 in range(0, len(rows), max_chars)]


def _pair_image(img, p, which):
    try:
        return _as_image(img, p)
    except (ValueError, TypeError) as e:
        raise ValueError(f"pair {p}: the {which} is not a uint8 [h, w, 3] image ({e})") from None


@torch.no_grad()
def interpolate_styles(encoder, tspgan, pairs, scales=tuple(i / 10 for i in range(11)), max_lines=8, max_chars=128, overlap=64,
                       to_host=False, skip_invalid=False):
    """test_w.py's font-style interpolation (:95-114) for many (content, donor) pairs of text-line images, on the device.

    pairs: (content, donor) uint8 [h, w, 3] images (numpy arrays or CPU / CUDA tensors, as restore_images takes them; the arrays
    test_w.py holds after cv2.cvtColor).  scales: non-empty sequence of finite numbers; the style at scale s is w1*s + w2*(1-s)
    (test_w.py:107), w1 the content's and w2 the donor's, so s = 1 is the content's own style.
    Returns one dict per pair: strips (uint8 [len(scales), 128, 128 n, 3]: strip k holds the n characters' generator images at
    scales[k], the bytes cv2.imwrite stores for w_{s:.2f}.png; on the device, or numpy through ONE pinned copy with ``to_host``),
    labels (the n characters, in strip order) and windows (the content's plan_windows plan).

    A content line that fits the canvas (round_half_even(w*32/h) <= 512) gives test_w.py's bytes: its characters are all of
    clear_labels(logits[0]) (up to 64), its style the encoder w of the whole image.  A wider one is read through plan_windows(h, w,
    overlap): its characters are predict_characters' labels in the same order, each in the style of the detection window that
    kept it.  Donors must fit the canvas.  A donor wider than the canvas, a content line without a decoded character or a
    malformed image make the pair invalid: ValueError naming the pair, or dict(error=...) with ``skip_invalid``.

    Read stage: one pinned host->device copy of the host images; per batch of at most ``max_lines`` encoder rows (fitting
    content, then wide-content windows, then donors): one crop launch, the encoder, one mn_decode_labels launch for the fitting
    content rows and one mn_decode_predictions launch for the windows; one pinned device->host copy and one synchronisation.
    Sweep stage: one pinned copy of the style rows, labels and tile table; one mn_style_lerp launch; per chunk of at most
    ``max_chars`` rows the generator (run eagerly: no module graph is recorded, since the chunk shapes vary from call to call) and
    one mn_prior_tiles_u8 launch; one synchronisation, and a re-run when the fp16-range guard re-routed a layer (ops.poll_range)."""
    import ctypes
    import math
    import numpy as np
    from . import _lib, ops
    if max_lines < 1:
        raise ValueError("max_lines must be >= 1")
    if max_chars < 1:
        raise ValueError("max_chars must be >= 1")
    if not 0 <= overlap <= 256:
        raise ValueError(f"overlap must lie in [0, 256] LQ pixels, got {overlap}")
    scales = list(scales)
    if not scales or any(isinstance(v, bool) or not isinstance(v, (int, float)) or not math.isfinite(v) for v in scales):
        raise ValueError(f"scales must be a non-empty sequence of finite numbers, got {scales}")
    scales = [float(v) for v in scales]
    dev = next(encoder.parameters()).device
    n = len(pairs)
    results, imgs, plans = [None] * n, [], {}

    def failed(p, e):
        if not skip_invalid:
            raise e
        results[p] = dict(error=f"{type(e).__name__}: {e}")

    for p, pair in enumerate(pairs):
        try:
            if not isinstance(pair, (tuple, list)) or len(pair) != 2:
                raise ValueError(f"pair {p}: expected a (content, donor) pair of images")
            content, donor = _pair_image(pair[0], p, "content"), _pair_image(pair[1], p, "donor")
            lq_w = whole_line_width(*donor.shape[:2])[0]
            if lq_w > 512:
                raise ValueError(f"pair {p}: the donor's LQ width {lq_w} exceeds the 512-pixel canvas (a line wider than the canvas "
                                 f"has no single style w; test_w.py:88 exits on it)")
        except ValueError as e:
            failed(p, e)
            continue
        plans[p] = (plan_windows(*content.shape[:2], overlap=overlap), len(imgs), len(imgs) + 1)
        imgs += [content, donor]
    # encoder rows (image, a, b, pair, window), kind by kind: fitting content, wide-content windows, donors
    fit = [(ci, 0, imgs[ci].shape[1], p, 0) for p, (win, ci, _) in plans.items() if len(win) == 1]
    wide = [(ci, *wn.crop, p, k) for p, (win, ci, _) in plans.items() if len(win) > 1 for k, wn in enumerate(win)]
    donors = [(di, 0, imgs[di].shape[1], p, -1) for p, (_, _, di) in plans.items()]
    rows = fit + wide + donors
    if not rows:
        return results
    isz_p, isz_l = ctypes.sizeof(_lib.CharPred), ctypes.sizeof(_lib.LabelRow)
    with torch.cuda.device(dev):
        rec = torch.empty(len(wide) * isz_p + len(fit) * isz_l, dtype=torch.uint8, device=dev)
        ptable = ops.prediction_table([(a, 16.0 * imgs[i].shape[0], *plans[p][0][k].core) for i, a, _, p, k in wide], dev,
                                      out=rec)[0] if wide else None
        labs_d = rec[len(wide) * isz_p:]
        wtab = torch.empty((len(rows), 512), dtype=torch.float32, device=dev)
        dimg = _device_images(range(len(imgs)), imgs, dev)
        nf, nw = len(fit), len(fit) + len(wide)
        for r0 in range(0, len(rows), max_lines):
            r1 = min(r0 + max_lines, len(rows))
            lq, _ = ops.preprocess_lq_crops([(dimg[i], a, b) for i, a, b, _, _ in rows[r0:r1]])
            logits, locs_lr, w = encoder(lq)
            wtab[r0:r1].copy_(w)
            if r0 < nf:
                ops.decode_labels(logits[:min(r1, nf) - r0], labs_d, r0)
            if max(r0, nf) < min(r1, nw):
                a0, a1 = max(r0, nf) - r0, min(r1, nw) - r0
                ops.decode_predictions(logits[a0:a1], locs_lr[a0:a1], ptable, r0 + a0 - nf)
        host = _to_host(rec).numpy()
    pred = host[:len(wide) * isz_p].view(ops.pred_dtype())
    labs = host[len(wide) * isz_p:].view(ops.label_dtype())
    chars, donor_row = [None] * n, [None] * n
    for r, (_, _, _, p, _) in enumerate(donors):
        donor_row[p] = nw + r
    for r, (_, _, _, p, _) in enumerate(fit):
        chars[p] = [(r, int(v)) for v in labs[r]["label"][:int(labs[r]["n"])]]
    first = {}
    for r, (ci, _, _, p, k) in enumerate(wide):
        first.setdefault(p, nf + r)
    for p, r0 in first.items():
        win, ci, _ = plans[p]
        dec = []
        for k in range(len(win)):
            m = int(pred[r0 - nf + k]["n_kept"])
            rr = pred[r0 - nf + k]
            dec.append((rr["label"][:m].tolist(), rr["x1"][:m].tolist(), rr["x2"][:m].tolist()))
        chars[p] = [(r0 + k, lab) for lab, _, k in _merge_windows(*imgs[ci].shape[:2], win, dec)]
    for p in plans:
        if not chars[p]:
            chars[p] = None
            failed(p, ValueError(f"pair {p}: no character decoded from the content"))
    srows, chunks = plan_sweep(chars, donor_row, len(scales), max_chars)
    if not srows:
        return results
    with torch.cuda.device(dev):
        offs, total = {}, 0
        for p, cs in enumerate(chars):
            if cs:
                offs[p] = total
                total += len(scales) * 128 * 128 * len(cs) * 3
        flat = torch.empty(total, dtype=torch.uint8, device=dev)

        def strips_of(buf):
            return {p: buf[o:o + len(scales) * 128 * 128 * len(chars[p]) * 3].view(len(scales), 128, 128 * len(chars[p]), 3)
                    for p, o in offs.items()}
        strips = strips_of(flat)
        tiles = ops.prior_tile_rows([(strips[r.pair][r.scale], r.char) for r in srows])
        lerp = ops.lerp_rows([(r.w1, r.w2, scales[r.scale]) for r in srows], len(rows))
        host_tab = tiles + lerp + np.asarray([r.label for r in srows], np.int64).tobytes()
        pinned = torch.empty(len(host_tab), dtype=torch.uint8, pin_memory=True)
        pinned.numpy()[:] = np.frombuffer(host_tab, np.uint8)
        tab = pinned.to(dev, non_blocking=True)
        lerp_d = tab[len(tiles):len(tiles) + len(lerp)]
        lab_d = tab[len(tiles) + len(lerp):].view(torch.int64)
        flag = torch.zeros(1, dtype=torch.int32, device=dev)

        def sweep():
            styles = ops.style_lerp(wtab, lerp_d, len(srows))
            with ops.deferred_checks(flag):          # device-side label check; also keeps the generator off its module graphs
                for r0, r1 in chunks:
                    img, _, _ = tspgan(styles=styles[r0:r1], labels=lab_d[r0:r1].view(-1, 1), noise=None)
                    ops.prior_tiles(img, tab, r0)
        _rerun(sweep, dev)
        ops.raise_deferred(int(flag.item()))
        if to_host:
            strips = {p: s.numpy() for p, s in strips_of(_to_host(flat)).items()}
    for p in offs:
        results[p] = dict(strips=strips[p], labels=[lab for _, lab in chars[p]], windows=plans[p][0])
    return results


# ---------------------------------------------------------------------------------------------------------------------
# Text regions in whole images (DESIGN.md section 7b, "Text regions in whole images").  A photo, scan or screenshot with a few
# rectangles of small text: the page is upscaled by s with OpenCV's cubic resize, each rectangle is restored as a text-line image
# of its own (restore_images on a view of the uploaded page), its 128-row result is resized onto the rectangle's s-times output
# and blended in with a linear ramp of F output pixels along every side that is not on the page border.
# ---------------------------------------------------------------------------------------------------------------------
class RegionPlan(NamedTuple):
    """One region of restore_regions, planned on the host: region ``region`` of image ``image``, ``rect`` (x0, y0, x1, y1) in
    source pixels, ``out`` the same rectangle in output pixels, ``overlaps`` the indices (into the plan) of the earlier regions
    of the same image whose rectangles meet this one, and the labels and boxes restore_images gets for the crop (boxes shifted
    by (-x0, -y0); None: predicted).  An oriented region (DESIGN.md 7b, "Oriented text regions") also has ``oriented`` (the
    OrientedRegion), ``matrix`` (M, its rectified crop's map) and ``size`` ((w_r, h_r), the crop's size); its ``rect`` is the
    bounding box of its corners in source pixels clipped to the image, ``out`` the bounding box of its footprint in output pixels,
    ``overlaps`` compares the ``out`` boxes, and its boxes are in the crop's frame, unshifted.  A perspective region (DESIGN.md
    7b, "Perspective text regions") has ``quad`` (the QuadRegion) instead of ``oriented``, and ``matrix`` is its 3 x 3 M.  A
    vertical column (DESIGN.md 7b, "Vertical text columns") is planned as its shape, with ``out`` sized for its restored column,
    and has ``vertical`` (its VerticalPlan); its ``boxes`` are the given boxes moved onto the line L.  A curved region (DESIGN.md
    7b, "Curved text regions") has ``curved`` (the CurvedRegion, its points as float pairs) and ``size``, no ``matrix``; its
    ``rect`` is the bounding box of its control points clipped to the image and ``out`` curved_footprint_box's."""
    image: int
    region: int
    rect: tuple
    out: tuple
    overlaps: list
    labels: list
    boxes: list
    oriented: tuple = None
    matrix: object = None
    size: tuple = None
    quad: tuple = None
    vertical: tuple = None
    curved: tuple = None


class OrientedRegion(NamedTuple):
    """A text line as a parallelogram (DESIGN.md 7b, "Oriented text regions"): its top-left, top-right and bottom-left corners as
    it is read, (x, y) points in continuous image coordinates (pixel (i, j) covers [j, j+1) x [i, i+1)).  e = tr - tl runs along
    the line and f = bl - tl down it.  The rectangle (x0, y0, x1, y1) is OrientedRegion((x0, y0), (x1, y0), (x0, y1))."""
    tl: tuple
    tr: tuple
    bl: tuple

    @classmethod
    def from_rotated(cls, cx, cy, w, h, angle):
        """The w x h line centred at (cx, cy), turned ``angle`` degrees counter-clockwise as seen on screen (y points down):
        e = w (cos a, -sin a), f = h (sin a, cos a), tl = c - e/2 - f/2."""
        a = math.radians(angle)
        ex, ey, fx, fy = w * math.cos(a), -w * math.sin(a), h * math.sin(a), h * math.cos(a)
        tlx, tly = cx - ex / 2 - fx / 2, cy - ey / 2 - fy / 2
        return cls((tlx, tly), (tlx + ex, tly + ey), (tlx + fx, tly + fy))


class OrientedMaps(NamedTuple):
    """oriented_maps' result: ``matrix`` M (fp64 [2, 3]: rectified crop pixel indices -> image pixel indices), ``size``
    (w_r, h_r), ``page_map`` N (fp64 [2, 3]: output page pixel indices -> pixel indices of the restored line T), ``kx`` and
    ``ky`` (the feather slopes, fp32 values) and ``t_width`` (W_T)."""
    matrix: object
    size: tuple
    page_map: object
    kx: float
    ky: float
    t_width: int


def oriented_maps(region, scale, t_width=None, t_height=128):
    """The fp64 maps of an OrientedRegion (DESIGN.md 7b, "Oriented text regions"), computed here once for the kernels and the
    numpy twin alike.  w_r = round_half_even(|e|), h_r = round_half_even(|f|);
      M = [[ex/w_r, fx/h_r, tlx + 0.5 ex/w_r + 0.5 fx/h_r - 0.5], [ey/w_r, fy/h_r, tly + 0.5 ey/w_r + 0.5 fy/h_r - 0.5]];
    N takes output pixel (X, Y) at scale s to T's pixel indices (a W_T - 0.5, H_T b - 0.5), where ((X + 0.5)/s, (Y + 0.5)/s) - tl
    = a e + b f; kx = fl32(s |e x f| / (|f| W_T)), ky = fl32(s |e x f| / (H_T |e|)).  W_T (``t_width``) defaults to
    round_half_even(w_r 128 / h_r), the width restore_images gives a line that fits its canvas; pass T's own width otherwise.
    H_T (``t_height``) is 128, restore_images' height, except for a vertical column's restored T_col (DESIGN.md 7b, "Vertical
    text columns").  For integer axis-aligned corners M = [[1, 0, x0], [0, 1, y0]] exactly."""
    import numpy as np
    from .ops import round_half_even
    (tlx, tly), (trx, try_), (blx, bly) = ((float(p[0]), float(p[1])) for p in region)
    ex, ey, fx, fy = trx - tlx, try_ - tly, blx - tlx, bly - tly
    le, lf = math.hypot(ex, ey), math.hypot(fx, fy)
    w_r, h_r = round_half_even(le), round_half_even(lf)
    a, b, c, d = ex / w_r, fx / h_r, ey / w_r, fy / h_r
    m = np.array([[a, b, tlx + 0.5 * a + 0.5 * b - 0.5], [c, d, tly + 0.5 * c + 0.5 * d - 0.5]], np.float64)
    wt = round_half_even(w_r * (128 / h_r)) if t_width is None else int(t_width)
    s, cross, h, ht = scale, ex * fy - ey * fx, 0.5 / scale, t_height
    n = np.array([[wt * fy / (s * cross), -wt * fx / (s * cross), wt * (fy * (h - tlx) - fx * (h - tly)) / cross - 0.5],
                  [-ht * ey / (s * cross), ht * ex / (s * cross), ht * (ex * (h - tly) - ey * (h - tlx)) / cross - 0.5]],
                 np.float64)
    kx = float(np.float32(s * abs(cross) / (lf * wt)))
    ky = float(np.float32(s * abs(cross) / (le * ht)))
    return OrientedMaps(m, (w_r, h_r), n, kx, ky, wt)


def footprint_box(region, maps, scale, page_hw, t_height=128):
    """(X0, Y0, X1, Y1): output pixels that hold every pixel of the region's footprint, on a page of page_hw = (H, W) output
    pixels.  The parallelogram is widened by one T pixel on every side (far more than the 1/32-pixel rounding of the fixed-point
    coordinates) and each pixel whose centre it may cover is taken.  t_height: T's height, as oriented_maps took it."""
    (tlx, tly), (trx, try_), (blx, bly) = ((float(p[0]), float(p[1])) for p in region)
    ex, ey, fx, fy = trx - tlx, try_ - tly, blx - tlx, bly - tly
    da, db = 1 / maps.t_width, 1 / t_height
    xs = [tlx + a * ex + b * fx for a in (-da, 1 + da) for b in (-db, 1 + db)]
    ys = [tly + a * ey + b * fy for a in (-da, 1 + da) for b in (-db, 1 + db)]
    s, (ph, pw) = scale, page_hw
    return (max(0, math.floor(s * min(xs) - 0.5)), max(0, math.floor(s * min(ys) - 0.5)),
            min(pw, math.ceil(s * max(xs) - 0.5) + 1), min(ph, math.ceil(s * max(ys) - 0.5) + 1))


def _fixed_point_fits(m, box):
    """cv2.warpAffine's int32 fixed-point coordinates (1/1024 pixel) of every destination pixel of box = (x0, y0, x1, y1) under
    m stay below 2^30: both the row start (m1 y + m2) * 1024 and the column step m0 x * 1024."""
    x0, y0, x1, y1 = box
    return all(abs(r[0]) * x1 + max(abs(r[1] * y0 + r[2]), abs(r[1] * y1 + r[2])) < 2.0 ** 20 for r in m)


def _plan_oriented(reg, H, W, scale, name, column=None):
    """Validates an OrientedRegion of an H x W image: (maps, rect, out).  column: None, or for the shape of a VerticalRegion a
    function of the crop's (w_r, h_r) that returns the column's restored size (W_c, H_c), which then sizes N and ``out``."""
    try:
        pts = [(float(p[0]), float(p[1])) for p in reg]
        if len(pts) != 3 or any(len(p) != 2 for p in reg):
            raise ValueError
    except (TypeError, ValueError):
        raise ValueError(f"{name}: expected three (x, y) corners, got {reg!r}") from None
    if not all(math.isfinite(v) for p in pts for v in p):
        raise ValueError(f"{name}: corners {pts} are not finite")
    (tlx, tly), (trx, try_), (blx, bly) = pts
    ex, ey, fx, fy = trx - tlx, try_ - tly, blx - tlx, bly - tly
    le, lf, cross = math.hypot(ex, ey), math.hypot(fx, fy), ex * fy - ey * fx
    if le < 1 or lf < 1:
        raise ValueError(f"{name}: sides |e| = {le:.4g} and |f| = {lf:.4g} must both be at least 1 pixel")
    if cross <= 0:
        raise ValueError(f"{name}: the region is mirrored (e x f = {cross:.4g} <= 0; give tl, tr, bl as the line is read)")
    if cross < 0.5 * le * lf:
        raise ValueError(f"{name}: the region is sheared past |e x f| >= |e| |f| / 2")
    cx, cy = tlx + ex / 2 + fx / 2, tly + ey / 2 + fy / 2
    if not (0 <= cx < W and 0 <= cy < H):
        raise ValueError(f"{name}: the centre ({cx:.6g}, {cy:.6g}) is outside the {W}x{H} image")
    maps = oriented_maps(pts, scale)
    (w_r, h_r), wt = maps.size, maps.t_width
    if max(w_r, h_r, wt, H, W) > 32767:
        raise ValueError(f"{name}: crop {w_r}x{h_r}, restored width {wt} or image {W}x{H} exceeds 32767 pixels "
                         f"(OpenCV's warp holds source coordinates as int16)")
    ht = 128
    if column is not None:
        wt, ht = column(w_r, h_r)
        maps = oriented_maps(pts, scale, wt, ht)
    out = footprint_box(pts, maps, scale, (scale * H, scale * W), ht)
    if not _fixed_point_fits(maps.page_map, out):
        raise ValueError(f"{name}: the map onto its {out} output box exceeds OpenCV's 32-bit fixed-point coordinates")
    xs, ys = (tlx, trx, blx, trx + fx), (tly, try_, bly, try_ + fy)
    rect = (max(0, math.floor(min(xs))), max(0, math.floor(min(ys))), min(W, math.ceil(max(xs))), min(H, math.ceil(max(ys))))
    return maps, rect, out


class QuadRegion(NamedTuple):
    """A text line seen in perspective (DESIGN.md 7b, "Perspective text regions"): its top-left, top-right, bottom-right and
    bottom-left corners as it is read, (x, y) points in continuous image coordinates (pixel (i, j) covers [j, j+1) x [i, i+1)).
    The rectangle (x0, y0, x1, y1) is QuadRegion((x0, y0), (x1, y0), (x1, y1), (x0, y1))."""
    tl: tuple
    tr: tuple
    br: tuple
    bl: tuple


class QuadMaps(NamedTuple):
    """quad_maps' result: ``matrix`` M (fp64 [3, 3]: rectified crop pixel indices -> image pixel indices, homogeneous), ``size``
    (w_r, h_r), ``page_map`` N (fp64 [3, 3]: output page pixel indices -> pixel indices of the restored line T), ``kx`` and ``ky``
    (the feather slopes, fp32 values), ``t_width`` (W_T) and ``homography`` H (the unit square -> the quad, rows of floats)."""
    matrix: object
    size: tuple
    page_map: object
    kx: float
    ky: float
    t_width: int
    homography: tuple


def _quad_homography(pts):
    """Heckbert's closed-form H taking the unit square's (0, 0), (1, 0), (1, 1), (0, 1) to p0..p3, as rows (a, b, c), (d, e, f),
    (g, h, 1)."""
    (x0, y0), (x1, y1), (x2, y2), (x3, y3) = pts
    sx, sy = x0 - x1 + x2 - x3, y0 - y1 + y2 - y3
    dx1, dx2, dy1, dy2 = x1 - x2, x3 - x2, y1 - y2, y3 - y2
    den = dx1 * dy2 - dx2 * dy1
    g = (sx * dy2 - sy * dx2) / den
    h = (dx1 * sy - dy1 * sx) / den
    return (x1 - x0 + g * x1, x3 - x0 + h * x3, x0), (y1 - y0 + g * y1, y3 - y0 + h * y3, y0), (g, h, 1.0)


def quad_maps(region, scale, t_width=None, t_height=128):
    """The fp64 maps of a QuadRegion (DESIGN.md 7b, "Perspective text regions"), computed here once in plain Python floats with a
    fixed operation order for the kernels and the numpy twin alike.  w_r = round_half_even(max(|tr - tl|, |br - bl|)),
    h_r = round_half_even(max(|bl - tl|, |br - tr|)); with H = [[a, b, c], [d, e, f], [g, h, 1]] the unit square -> quad
    homography, M's rows are [(a - 0.5 g)/w_r, (b - 0.5 h)/h_r, c - 0.5 + 0.5 (a - 0.5 g)/w_r + 0.5 (b - 0.5 h)/h_r], the same with
    d, e, f, and [g/w_r, h/h_r, 1 + 0.5 g/w_r + 0.5 h/h_r].  N = A_T adj(H) A_page, A_page = [[1/s, 0, 0.5/s], [0, 1/s, 0.5/s],
    [0, 0, 1]], A_T = [[W_T, 0, -0.5], [0, H_T, -0.5], [0, 0, 1]], all nine entries divided by its third row's value at the
    footprint's centre (the page pixel of H(0.5, 0.5)).  kx = fl32(s A / (L_f W_T)), ky = fl32(s A / (L_e H_T)): A the shoelace
    area, L_e the mean of the top and bottom side lengths, L_f of the left and right ones.  W_T (``t_width``) defaults to
    round_half_even(w_r 128 / h_r); pass T's own width otherwise.  H_T (``t_height``) is 128 except for a vertical column's T_col.  For integer axis-aligned corners M = [[1, 0, x0], [0, 1, y0],
    [0, 0, 1]] exactly, and at h = 32, s = 4, N = [[1, 0, -4 x0], [0, 1, -4 y0], [0, 0, 1]]."""
    import numpy as np
    from .ops import round_half_even
    pts = [(float(p[0]), float(p[1])) for p in region]
    (x0, y0), (x1, y1), (x2, y2), (x3, y3) = pts
    top, bottom = math.hypot(x1 - x0, y1 - y0), math.hypot(x2 - x3, y2 - y3)
    left, right = math.hypot(x3 - x0, y3 - y0), math.hypot(x2 - x1, y2 - y1)
    w_r, h_r = round_half_even(max(top, bottom)), round_half_even(max(left, right))
    hom = _quad_homography(pts)
    (a, b, c), (d, e, f), (g, h, _) = hom
    ra, rb, rd, re, rg, rh = (a - 0.5 * g) / w_r, (b - 0.5 * h) / h_r, (d - 0.5 * g) / w_r, (e - 0.5 * h) / h_r, g / w_r, h / h_r
    m = np.array([[ra, rb, c - 0.5 + 0.5 * ra + 0.5 * rb], [rd, re, f - 0.5 + 0.5 * rd + 0.5 * re],
                  [rg, rh, 1.0 + 0.5 * rg + 0.5 * rh]], np.float64)
    wt = round_half_even(w_r * (128 / h_r)) if t_width is None else int(t_width)
    s = scale
    adj = ((e - f * h, c * h - b, b * f - c * e), (f * g - d, a - c * g, c * d - a * f), (d * h - e * g, b * g - a * h, a * e - b * d))
    hs = 0.5 / s
    k = [(r[0] / s, r[1] / s, r[0] * hs + r[1] * hs + r[2]) for r in adj]
    n = [[wt * k[0][j] - 0.5 * k[2][j] for j in range(3)], [t_height * k[1][j] - 0.5 * k[2][j] for j in range(3)], list(k[2])]
    cw = 0.5 * g + 0.5 * h + 1.0
    xc, yc = s * ((0.5 * a + 0.5 * b + c) / cw) - 0.5, s * ((0.5 * d + 0.5 * e + f) / cw) - 0.5
    den = n[2][0] * xc + n[2][1] * yc + n[2][2]
    n = np.array([[v / den for v in row] for row in n], np.float64)
    area = 0.5 * abs((x0 * y1 - x1 * y0) + (x1 * y2 - x2 * y1) + (x2 * y3 - x3 * y2) + (x3 * y0 - x0 * y3))
    l_e, l_f = 0.5 * (top + bottom), 0.5 * (left + right)
    kx = float(np.float32(s * area / (l_f * wt)))
    ky = float(np.float32(s * area / (l_e * t_height)))
    return QuadMaps(m, (w_r, h_r), n, kx, ky, wt, hom)


def quad_footprint_box(maps, scale, page_hw, t_height=128):
    """(X0, Y0, X1, Y1): output pixels that hold every pixel of a quad's footprint, on a page of page_hw = (H, W) output pixels:
    the images under H of the corners of [-1/W_T, 1 + 1/W_T] x [-1/H_T, 1 + 1/H_T] (the quad widened by one T pixel on every
    side; H_T = t_height, as quad_maps took it), each pixel whose centre their hull may cover.  None when H's denominator is not
    positive at one of those corners."""
    (a, b, c), (d, e, f), (g, h, _) = maps.homography
    da, db = 1 / maps.t_width, 1 / t_height
    xs, ys = [], []
    for u in (-da, 1 + da):
        for v in (-db, 1 + db):
            w = g * u + h * v + 1.0
            if not w > 0:
                return None
            xs.append((a * u + b * v + c) / w)
            ys.append((d * u + e * v + f) / w)
    s, (ph, pw) = scale, page_hw
    return (max(0, math.floor(s * min(xs) - 0.5)), max(0, math.floor(s * min(ys) - 0.5)),
            min(pw, math.ceil(s * max(xs) - 0.5) + 1), min(ph, math.ceil(s * max(ys) - 0.5) + 1))


def _plan_quad(reg, H, W, scale, name, column=None):
    """Validates a QuadRegion of an H x W image: (maps, rect, out); column as _plan_oriented takes it."""
    try:
        pts = [(float(p[0]), float(p[1])) for p in reg]
        if len(pts) != 4 or any(len(p) != 2 for p in reg):
            raise ValueError
    except (TypeError, ValueError):
        raise ValueError(f"{name}: expected four (x, y) corners, got {reg!r}") from None
    if not all(math.isfinite(v) for p in pts for v in p):
        raise ValueError(f"{name}: corners {pts} are not finite")
    sides = [math.hypot(pts[(k + 1) % 4][0] - pts[k][0], pts[(k + 1) % 4][1] - pts[k][1]) for k in range(4)]
    if min(sides) < 1:
        raise ValueError(f"{name}: sides {[round(v, 4) for v in sides]} must all be at least 1 pixel")
    for k, corner in enumerate(("tl", "tr", "br", "bl")):
        (px, py), (nx, ny), (qx, qy) = pts[k], pts[(k + 1) % 4], pts[k - 1]
        turn = (nx - px) * (qy - py) - (ny - py) * (qx - px)
        if turn <= 0:
            raise ValueError(f"{name}: the quad is not strictly convex in reading order (turn {turn:.4g} <= 0 at {corner}; "
                             f"give tl, tr, br, bl as the line is read)")
        if turn < 0.5 * sides[k] * sides[k - 1]:
            raise ValueError(f"{name}: the interior angle at {corner} is outside [30, 150] degrees")
    cx, cy = sum(p[0] for p in pts) / 4, sum(p[1] for p in pts) / 4
    if not (0 <= cx < W and 0 <= cy < H):
        raise ValueError(f"{name}: the centre ({cx:.6g}, {cy:.6g}) is outside the {W}x{H} image")
    g, h, _ = _quad_homography(pts)[2]
    ws = (1.0, 1.0 + g, 1.0 + h, 1.0 + g + h)
    if not min(ws) > 0 or max(ws) > 4 * min(ws):
        raise ValueError(f"{name}: the foreshortening {max(ws) / min(ws) if min(ws) > 0 else math.inf:.4g} exceeds 4")
    maps = quad_maps(pts, scale)
    (w_r, h_r), wt = maps.size, maps.t_width
    if max(w_r, h_r, wt, H, W) > 32767:
        raise ValueError(f"{name}: crop {w_r}x{h_r}, restored width {wt} or image {W}x{H} exceeds 32767 pixels "
                         f"(OpenCV's warp holds source coordinates as int16)")
    ht = 128
    if column is not None:
        wt, ht = column(w_r, h_r)
        maps = quad_maps(pts, scale, wt, ht)
    out = quad_footprint_box(maps, scale, (scale * H, scale * W), ht)
    n = maps.page_map
    corners = [] if out is None else [(x, y) for x in (out[0], out[2] - 1) for y in (out[1], out[3] - 1)]
    dens = [n[2][0] * x + n[2][1] * y + n[2][2] for x, y in corners]
    if out is None or not min(dens) > 0:
        raise ValueError(f"{name}: the page map's denominator is not positive over the footprint box {out}")
    reach = max(abs(n[r][0] * x + n[r][1] * y + n[r][2]) for r in range(2) for x, y in corners)
    if 32 * reach / min(dens) >= 2.0 ** 30:
        raise ValueError(f"{name}: the map onto its {out} output box exceeds OpenCV's 32-bit fixed-point coordinates")
    xs, ys = [p[0] for p in pts], [p[1] for p in pts]
    rect = (max(0, math.floor(min(xs))), max(0, math.floor(min(ys))), min(W, math.ceil(max(xs))), min(H, math.ceil(max(ys))))
    return maps, rect, out


class CurvedRegion(NamedTuple):
    """A text line on a curve (DESIGN.md 7b, "Curved text regions"): ``top`` and ``bottom`` are chains of k cubic Beziers
    (1 <= k <= 8), 3k+1 (x, y) points each in continuous image coordinates (pixel (i, j) covers [j, j+1) x [i, i+1)); segment m of
    a curve is its points 3m .. 3m+3.  Both run in reading order, ``top`` along the characters' heads.  The line is rectified
    into a straight crop whose column a runs along the mid curve by arc length between segments and uniformly in t within one
    (ABCNet's BezierAlign), and whose row b runs from top to bottom along the straight ruling between T(t) and B(t)."""
    top: tuple
    bottom: tuple

    @classmethod
    def from_arc(cls, cx, cy, r_top, r_bottom, start, end):
        """Text on a circle centred at (cx, cy): the top edge at radius r_top, the bottom edge at r_bottom, read from angle
        ``start`` to ``end`` (degrees, counter-clockwise on screen: a point is (cx + r cos a, cy - r sin a)), 0 < |end - start| <
        360.  The top of a seal read left to right is start 150, end 30, r_top > r_bottom.  The arc is split into
        k = ceil(|end - start| / 90) equal segments whose handles lie along the tangents at r (4/3) tan(phi/4), phi the segment's
        signed span."""
        span = float(end) - float(start)
        if not 0 < abs(span) < 360:
            raise ValueError(f"from_arc: the span end - start = {span:g} degrees must satisfy 0 < |span| < 360")
        k = math.ceil(abs(span) / 90)
        h = 4 / 3 * math.tan(math.radians(span / k) / 4)

        def curve(r):
            pts = []
            for m in range(k):
                a0, a1 = math.radians(start + span * m / k), math.radians(start + span * (m + 1) / k)
                p0 = (cx + r * math.cos(a0), cy - r * math.sin(a0))
                p3 = (cx + r * math.cos(a1), cy - r * math.sin(a1))
                if m == 0:
                    pts.append(p0)
                pts += [(p0[0] - h * r * math.sin(a0), p0[1] - h * r * math.cos(a0)),       # p0 + h dP/da(a0)
                        (p3[0] + h * r * math.sin(a1), p3[1] + h * r * math.cos(a1)), p3]    # p3 - h dP/da(a1)
            return tuple(pts)
        return cls(curve(float(r_top)), curve(float(r_bottom)))


class CurvedMaps(NamedTuple):
    """curved_maps' result: ``size`` (w_r, h_r), ``c`` the column fractions [c_0 = 0, ..., c_k = 1], ``kx`` and ``ky`` (the
    feather slopes, fp32 values), ``t_width`` (W_T), ``top`` and ``bottom`` (the curves' points as float pairs), ``lengths``
    (the mid curve's sampled length L_m per segment) and ``rulings`` (every sampled ruling length |B(t_i) - T(t_i)|, segment by
    segment)."""
    size: tuple
    c: tuple
    kx: float
    ky: float
    t_width: int
    top: tuple
    bottom: tuple
    lengths: tuple
    rulings: tuple

    def curve(self, scale):
        """The kernels' curve table (ops.CurveTable) at page scale ``scale``."""
        from .ops import CurveTable
        return CurveTable(float(scale), self.c, self.top, self.bottom)


def bezier_point(p, t):
    """De Casteljau's point of the cubic Bezier p (4 (x, y) points) at t: s = 1 - t and three levels of lerps
    fl(fl(s A) + fl(t B)) per coordinate, in plain Python floats (every operation rounded on its own)."""
    s = 1.0 - t
    out = []
    for k in (0, 1):
        a0, a1, a2 = s * p[0][k] + t * p[1][k], s * p[1][k] + t * p[2][k], s * p[2][k] + t * p[3][k]
        b0, b1 = s * a0 + t * a1, s * a1 + t * a2
        out.append(s * b0 + t * b1)
    return out[0], out[1]


def _curve_points(region):
    """(top, bottom, k): the region's points as float pairs.  Raises TypeError / ValueError for anything else."""
    top, bottom = ([(float(p[0]), float(p[1])) for p in c] for c in region)
    if any(len(p) != 2 for c in region for p in c):
        raise ValueError
    return tuple(top), tuple(bottom), (len(top) - 1) // 3


def _curve_samples(top, bottom, k):
    """Per segment, the 33 samples t_i = i/32 of (T, B): the mid curve's lengths L_m (sqrt of fl(fl(dx dx) + fl(dy dy)) between
    consecutive Mid = fl(0.5 fl(T + B)), summed in order) and every ruling length, in order."""
    lengths, rulings = [], []
    for m in range(k):
        tp, bp = top[3 * m:3 * m + 4], bottom[3 * m:3 * m + 4]
        L, prev = 0.0, None
        for i in range(33):
            (tx, ty), (bx, by) = bezier_point(tp, i / 32), bezier_point(bp, i / 32)
            rx, ry = bx - tx, by - ty
            rulings.append(math.sqrt(rx * rx + ry * ry))
            mid = (0.5 * (tx + bx), 0.5 * (ty + by))
            if prev is not None:
                dx, dy = mid[0] - prev[0], mid[1] - prev[1]
                L += math.sqrt(dx * dx + dy * dy)
            prev = mid
        lengths.append(L)
    return lengths, rulings


def curved_maps(region, scale, t_width=None, t_height=128):
    """The maps of a CurvedRegion (DESIGN.md 7b, "Curved text regions"), computed here once in plain Python floats with a fixed
    operation order for the kernels and the numpy twin alike.  Per segment m, 33 samples at t_i = i/32 give the mid curve's
    length L_m (_curve_samples) and the ruling lengths; L = L_0 + ... + L_{k-1} in order, c_m = (L_0 + ... + L_{m-1}) / L
    (c_0 = 0, c_k = 1), w_r = round_half_even(L), h_r = round_half_even(the longest sampled ruling), W_T (``t_width``) defaults to
    round_half_even(w_r 128 / h_r); kx = fl32(s L / W_T), ky = fl32(s h / H_T), h the mean sampled ruling length (summed in
    order) and H_T = ``t_height``."""
    import numpy as np
    from .ops import round_half_even
    top, bottom, k = _curve_points(region)
    lengths, rulings = _curve_samples(top, bottom, k)
    L = 0.0
    c = [0.0]
    for v in lengths:
        L += v
    acc = 0.0
    for m in range(1, k):
        acc += lengths[m - 1]
        c.append(acc / L)
    c.append(1.0)
    w_r, h_r = round_half_even(L), round_half_even(max(rulings))
    wt = round_half_even(w_r * (128 / h_r)) if t_width is None else int(t_width)
    hsum = 0.0
    for v in rulings:
        hsum += v
    kx = float(np.float32(scale * L / wt))
    ky = float(np.float32(scale * (hsum / len(rulings)) / t_height))
    return CurvedMaps((w_r, h_r), tuple(c), kx, ky, wt, top, bottom, tuple(lengths), tuple(rulings))


def curved_footprint_box(region, scale, page_hw):
    """(X0, Y0, X1, Y1): the output pixels that hold every pixel of a curved region's footprint on a page of page_hw = (H, W)
    output pixels: the bounding box of all its control points (which holds both curves and every ruling between them) at scale s,
    widened by one pixel and clipped to the page."""
    top, bottom, _ = _curve_points(region)
    xs, ys = [p[0] for p in top + bottom], [p[1] for p in top + bottom]
    s, (ph, pw) = scale, page_hw
    return (max(0, math.floor(s * min(xs)) - 1), max(0, math.floor(s * min(ys)) - 1),
            min(pw, math.ceil(s * max(xs)) + 1), min(ph, math.ceil(s * max(ys)) + 1))


def _bezier_rows(maps, b):
    """numpy fp64 [2, w_r]: the crop map (x, y) of row b (a float) at every column, as mn_remap_curved_u8_batched computes it."""
    import numpy as np
    w_r, k = maps.size[0], len(maps.c) - 1
    a = (np.arange(w_r, dtype=np.float64) + 0.5) / w_r
    c = np.asarray(maps.c, np.float64)
    m = np.searchsorted(c[1:k], a, side="right")
    t = (a - c[m]) / (c[m + 1] - c[m])
    s = 1.0 - t
    out = []
    for k_ in (0, 1):
        pts = []
        for curve in (maps.top, maps.bottom):
            p = np.asarray(curve, np.float64)[:, k_]
            v = [p[3 * m + j] for j in range(4)]
            a0, a1, a2 = s * v[0] + t * v[1], s * v[1] + t * v[2], s * v[2] + t * v[3]
            b0, b1 = s * a0 + t * a1, s * a1 + t * a2
            pts.append(s * b0 + t * b1)
        out.append((1.0 - b) * pts[0] + b * pts[1] - 0.5)
    return np.stack(out)


def _plan_curved(reg, H, W, scale, name):
    """Validates a CurvedRegion of an H x W image: (maps, rect, out)."""
    try:
        top, bottom, k = _curve_points(reg)
        if len(reg) != 2:
            raise ValueError
    except (TypeError, ValueError):
        raise ValueError(f"{name}: expected two curves of (x, y) points, got {reg!r}") from None
    if not all(math.isfinite(v) for p in top + bottom for v in p):
        raise ValueError(f"{name}: the control points are not all finite")
    if len(top) != len(bottom) or len(top) % 3 != 1 or not 1 <= k <= 8:
        raise ValueError(f"{name}: the curves have {len(top)} and {len(bottom)} points; both need 3k+1 points, 1 <= k <= 8")
    import numpy as np
    from .ops import round_half_even
    lengths, rulings = _curve_samples(top, bottom, k)
    h_r = round_half_even(max(rulings))
    if h_r < 1 or round_half_even(sum(lengths)) < 1:
        raise ValueError(f"{name}: the band is {max(rulings):.4g} pixels high and {sum(lengths):.4g} long (at least 1 each)")
    for m, v in enumerate(lengths):
        if v < h_r / 8:
            raise ValueError(f"{name}: segment {m}'s mid curve is {v:.4g} pixels long, below h_r / 8 = {h_r / 8:g}")
    for m in range(k):
        tp, bp = top[3 * m:3 * m + 4], bottom[3 * m:3 * m + 4]
        turn, lo, hi, prev = 0.0, 0.0, 0.0, None
        for i in range(33):
            t = i / 32
            (tx, ty), (bx, by) = bezier_point(tp, t), bezier_point(bp, t)
            dt = [3 * ((1 - t) ** 2 * (p[1][j] - p[0][j]) + 2 * (1 - t) * t * (p[2][j] - p[1][j]) + t * t * (p[3][j] - p[2][j]))
                  for p in (tp, bp) for j in (0, 1)]
            rx, ry = bx - tx, by - ty
            for b in (0.0, 0.25, 0.5, 0.75, 1.0):
                jac = ((1 - b) * dt[0] + b * dt[2]) * ry - ((1 - b) * dt[1] + b * dt[3]) * rx
                if not jac > 0:
                    raise ValueError(f"{name}: the band folds or runs against its reading order (Jacobian {jac:.4g} <= 0 at "
                                     f"segment {m}, t = {t:g}, b = {b:g}; give top and bottom as the line is read)")
            if prev is not None:
                turn += math.atan2(prev[0] * ry - prev[1] * rx, prev[0] * rx + prev[1] * ry)
                lo, hi = min(lo, turn), max(hi, turn)
            prev = (rx, ry)
        if hi - lo > math.pi / 2:
            raise ValueError(f"{name}: the ruling B - T turns by {math.degrees(hi - lo):.4g} degrees within segment {m} "
                             f"(at most 90)")
    if max(rulings) > 4 * min(rulings):
        raise ValueError(f"{name}: the longest ruling {max(rulings):.4g} is more than 4 times the shortest {min(rulings):.4g}")
    maps = curved_maps((top, bottom), scale)
    c = maps.c
    m = max(j for j in range(k) if c[j] <= 0.5)
    t = (0.5 - c[m]) / (c[m + 1] - c[m])
    (tx, ty), (bx, by) = bezier_point(top[3 * m:3 * m + 4], t), bezier_point(bottom[3 * m:3 * m + 4], t)
    cx, cy = 0.5 * tx + 0.5 * bx, 0.5 * ty + 0.5 * by
    if not (0 <= cx < W and 0 <= cy < H):
        raise ValueError(f"{name}: the mid point ({cx:.6g}, {cy:.6g}) is outside the {W}x{H} image")
    (w_r, h_r), wt = maps.size, maps.t_width
    if max(w_r, h_r, wt, H, W) > 32767:
        raise ValueError(f"{name}: crop {w_r}x{h_r}, restored width {wt} or image {W}x{H} exceeds 32767 pixels "
                         f"(OpenCV's remap holds source coordinates as int16)")
    reach = max(np.abs(_bezier_rows(maps, b)).max() for b in (0.5 / h_r, (h_r - 0.5) / h_r))
    if not reach < 2.0 ** 14:
        raise ValueError(f"{name}: the crop map reaches {reach:.6g} pixels, beyond OpenCV's int16 remap coordinates (2^14)")
    out = curved_footprint_box((top, bottom), scale, (scale * H, scale * W))
    xs, ys = [p[0] for p in top + bottom], [p[1] for p in top + bottom]
    rect = (max(0, math.floor(min(xs))), max(0, math.floor(min(ys))), min(W, math.ceil(max(xs))), min(H, math.ceil(max(ys))))
    return maps, rect, out


class VerticalRegion(NamedTuple):
    """A column of upright characters read top to bottom (DESIGN.md 7b, "Vertical text columns").  ``shape`` is its footprint: an
    integer rectangle (x0, y0, x1, y1), an OrientedRegion or a QuadRegion, with tl -> tr across the column and tl -> bl down it.
    Its crop C (img[y0:y1, x0:x1], or the shape's rectified crop) is cut into character cells laid side by side as a horizontal
    line, which is restored and put back into a column.  ``cells``: the number of equal cells when no boxes are given (default:
    round_half_even(h_r / w_r), glyphs being about square)."""
    shape: object
    cells: object = None


class VerticalPlan(NamedTuple):
    """vertical_plan's result for a column crop C of ``size`` (w_r, h_r): ``cells`` the boundaries [c_0 = 0, ..., c_n = h_r],
    ``heights`` t_k = c_{k+1} - c_k, ``line_height`` H_L = max t_k, ``pads`` p_k = (H_L - t_k) // 2, ``t_size`` (W_c, H_c) =
    (R(w_r), R(h_r)), the restored column's size, and ``boxes`` the given boxes moved onto the line L [H_L, n w_r] (None when
    they are predicted)."""
    cells: list
    size: tuple
    heights: list
    line_height: int
    pads: list
    t_size: tuple
    boxes: list


def vertical_r(y, line_height):
    """R(y) = round_half_even(y (128 / H_L)): where row or column y of the line L lands in its restored line T (stitch_pieces'
    r(x), so that R(n w_r) is T's width)."""
    from .ops import round_half_even
    return round_half_even(y * (128 / line_height))


def vertical_plan(w_r, h_r, cells=None, boxes=None, name="column"):
    """The cell plan of a w_r x h_r column crop (DESIGN.md 7b, "Vertical text columns"), in integers and fp64.  With boxes
    [x1, y1, x2, y2] (C's frame, reading order), c_k = floor((y2_{k-1} + y1_k) / 2) for k = 1 .. n-1; else c_k = (k h_r) // n with
    n = ``cells`` or clamp(round_half_even(h_r / w_r), 1, h_r).  Raises ValueError, naming ``name``: cells not an integer in
    [1, h_r] or given with boxes, a box outside C, box centres that go up, boundaries not strictly increasing inside (0, h_r)
    (these name the character), a
    line n w_r or a restored size W_c, H_c or W_T = R(n w_r) over 32767 pixels."""
    from .ops import round_half_even
    if cells is not None and boxes is not None:
        raise ValueError(f"{name}: cells and boxes are both given (boxes fix the cells)")
    if boxes is not None:
        bx = []
        for k, b in enumerate(boxes):
            b = [float(v) for v in b]
            if len(b) != 4 or not (0 <= b[0] <= b[2] <= w_r and 0 <= b[1] <= b[3] <= h_r):
                raise ValueError(f"{name}, character {k}: box {b} is outside the column crop [0, {w_r}] x [0, {h_r}]")
            bx.append(b)
        c = [0]
        for k in range(1, len(bx)):
            y, y0 = (bx[k][1] + bx[k][3]) / 2, (bx[k - 1][1] + bx[k - 1][3]) / 2
            if y < y0:
                raise ValueError(f"{name}, character {k}: the box's centre {y:g} lies above the previous character's {y0:g} "
                                 f"(boxes are listed in reading order, down the column)")
            c.append(math.floor((bx[k - 1][3] + bx[k][1]) / 2))
            if not c[-2] < c[-1] < h_r:
                raise ValueError(f"{name}, character {k}: the cell boundary {c[-1]} between it and the previous character is "
                                 f"not strictly inside ({c[-2]}, {h_r})")
        c.append(h_r)
    else:
        if cells is None:
            n = min(max(round_half_even(h_r / w_r), 1), h_r)
        elif isinstance(cells, bool) or not isinstance(cells, int) or not 1 <= cells <= h_r:
            raise ValueError(f"{name}: cells must be an integer in [1, {h_r}] (the crop's rows), got {cells!r}")
        else:
            n = cells
        c = [(k * h_r) // n for k in range(n + 1)]
    n = len(c) - 1
    t = [c[k + 1] - c[k] for k in range(n)]
    hl = max(t)
    p = [(hl - v) // 2 for v in t]
    wc, hc, wt = vertical_r(w_r, hl), vertical_r(h_r, hl), vertical_r(n * w_r, hl)
    if max(n * w_r, wc, hc, wt) > 32767:
        raise ValueError(f"{name}: line width {n * w_r}, restored column {wc}x{hc} or restored line width {wt} exceeds 32767 pixels")
    lb = None if boxes is None else [[k * w_r + b[0], p[k] + b[1] - c[k], k * w_r + b[2], p[k] + b[3] - c[k]]
                                     for k, b in enumerate(bx)]
    return VerticalPlan(c, (w_r, h_r), t, hl, p, (wc, hc), lb)


def layout_cells(vp):
    """ops.vertical_layout's table: (c_k, p_k, t_k) per cell."""
    return [(vp.cells[k], vp.pads[k], vp.heights[k]) for k in range(len(vp.heights))]


def unlayout_cells(vp, t_width):
    """ops.vertical_unlayout's table for a restored line T of width W_T = t_width: (R(c_k), R(p_k), R(p_k + t_k), R(k w_r),
    min(R((k+1) w_r), W_T)) per cell."""
    hl, w = vp.line_height, vp.size[0]
    return [(vertical_r(vp.cells[k], hl), vertical_r(vp.pads[k], hl), vertical_r(vp.pads[k] + vp.heights[k], hl),
             vertical_r(k * w, hl), min(vertical_r((k + 1) * w, hl), t_width)) for k in range(len(vp.heights))]


def column_boxes(vp, boxes):
    """Boxes predicted on the line L -> the column crop C's frame, each through the cell that holds its centre: x - k w_r clipped
    to [0, w_r], y - p_k + c_k clipped to [c_k, c_{k+1}]."""
    w, n, out = vp.size[0], len(vp.heights), []
    for b in boxes:
        k = min(max(math.floor((b[0] + b[2]) / 2 / w), 0), n - 1)
        lo, hi, dy = vp.cells[k], vp.cells[k + 1], vp.cells[k] - vp.pads[k]
        out.append([min(max(b[0] - k * w, 0), w), min(max(b[1] + dy, lo), hi), min(max(b[2] - k * w, 0), w),
                    min(max(b[3] + dy, lo), hi)])
    return out


def _per_image(v, n, what):
    v = [None] * n if v is None else list(v)
    if len(v) != n:
        raise ValueError(f"{what}: {len(v)} entries for {n}")
    return v


class TextBlock(NamedTuple):
    """A block of text lines inside an image (DESIGN.md 7b, "Text blocks").  ``rect``: an integer rectangle (x0, y0, x1, y1)
    around the lines.  ``direction``: "horizontal" (lines read top to bottom) or "vertical" (columns read right to left).
    ``min_ink``, ``gap``, ``min_height``: positive integers in place of the segmentation's defaults.  ``polarity``: "auto" (the
    minority side of the Otsu threshold is ink), "dark" or "light".  find_lines splits it into lines; restore_regions restores
    each line in its place.  ``skew`` (DESIGN.md 7b, "Skewed blocks"): None (level lines), a given angle in degrees with
    |skew| < 45, counter-clockwise on screen as OrientedRegion.from_rotated's, or "auto": the angle is searched on the device
    within +-``max_skew`` degrees (in (0, 20], only with "auto") and the lines are OrientedRegions of that angle."""
    rect: object
    direction: str = "horizontal"
    min_ink: object = None
    gap: object = None
    min_height: object = None
    polarity: str = "auto"
    skew: object = None
    max_skew: float = 10.0


_INK = {"auto": 0, "dark": 1, "light": 2}


def _check_block(blk, H, W, name):
    """The rectangle (x0, y0, x1, y1) of the TextBlock ``blk`` of an H x W image, validated.  Raises ValueError naming ``name``."""
    try:
        if isinstance(blk.rect, (OrientedRegion, QuadRegion, CurvedRegion, VerticalRegion)):
            raise ValueError
        x0, y0, x1, y1 = (int(v) for v in blk.rect)
        if (x0, y0, x1, y1) != tuple(blk.rect):
            raise ValueError
    except (TypeError, ValueError):
        raise ValueError(f"{name}: a text block is an integer rectangle (x0, y0, x1, y1), got {blk.rect!r} (oriented, "
                         f"perspective and curved blocks are not supported)") from None
    if not (0 <= x0 < x1 <= W and 0 <= y0 < y1 <= H):
        raise ValueError(f"{name}: rectangle {(x0, y0, x1, y1)} is empty or outside the {W}x{H} image")
    if max(x1 - x0, y1 - y0) > 32767:
        raise ValueError(f"{name}: a side of rectangle {(x0, y0, x1, y1)} exceeds 32767 pixels")
    if blk.direction not in ("horizontal", "vertical"):
        raise ValueError(f"{name}: direction must be 'horizontal' or 'vertical', got {blk.direction!r}")
    if blk.polarity not in _INK:
        raise ValueError(f"{name}: polarity must be 'auto', 'dark' or 'light', got {blk.polarity!r}")
    for what in ("min_ink", "gap", "min_height"):
        v = getattr(blk, what)
        if v is not None and (isinstance(v, bool) or not isinstance(v, int) or not 1 <= v < 2 ** 31):
            raise ValueError(f"{name}: {what} must be a positive integer, got {v!r}")
    sk, ms = blk.skew, blk.max_skew
    auto = isinstance(sk, str) and sk == "auto"
    if not (sk is None or auto or (isinstance(sk, numbers.Real) and not isinstance(sk, bool) and math.isfinite(sk)
                                   and abs(sk) < 45)):
        raise ValueError(f"{name}: skew must be None, 'auto' or a finite angle in degrees with |skew| < 45, got {sk!r}")
    if isinstance(ms, bool) or not isinstance(ms, numbers.Real) or not 0 < ms <= 20:
        raise ValueError(f"{name}: max_skew must be a number of degrees in (0, 20], got {ms!r}")
    if ms != 10.0 and not auto:
        raise ValueError(f"{name}: max_skew is given, but skew is {sk!r}, not 'auto'")
    if sk is not None:
        from . import ops
        vertical = blk.direction == "vertical"
        table = ops.skew_table(sk, ms, vertical)
        stride = ops.skew_stride(x1 - x0, y1 - y0, vertical, ops.skew_cos_sin(table))
        if len(table) > 1 and len(table) * stride > ops.SKEW_MAX_PROFILE:
            raise ValueError(f"{name}: the angle search needs {len(table)} angles x {stride} bins, over the "
                             f"{ops.SKEW_MAX_PROFILE} profile values a block may use (narrow max_skew or split the block)")
    return x0, y0, x1, y1


def _find_lines(dimg, items):
    """ops.find_lines over items (image index, TextBlock, rect) of the uploaded images ``dimg``, its table back through one pinned
    copy and one synchronisation.  Returns per item dict(lines, threshold, ink), or the error message of a block with too many
    lines."""
    from . import ops
    recs = ops.find_lines([(dimg[i], rect, blk.direction == "vertical", _INK[blk.polarity], blk.min_ink, blk.gap, blk.min_height,
                            blk.skew, blk.max_skew) for i, blk, rect in items])
    host = _to_host(recs).numpy()
    n_osz = len(items) * ops.block_lines_dtype().itemsize
    table = host[:n_osz].view(ops.block_lines_dtype())
    skew = host[n_osz:].view(ops.skew_block_dtype()) if len(host) > n_osz else [None] * len(items)
    out = []
    for (i, blk, rect), t, sk in zip(items, table, skew):
        n = int(t["n_lines"])
        if n < 0:
            out.append(f"{-n} lines exceed the {ops._lib.BLOCK_MAX_LINES} a text block may hold")
            continue
        lines = [tuple(int(v) for v in q) for q in t["rect"][:n]]
        vertical = blk.direction == "vertical"
        if blk.skew is not None and sk["s"] != 0:
            lines = skew_lines(rect, vertical, float(sk["c"]), float(sk["s"]), float(sk["u_min"]), float(sk["v_min"]), lines)
        elif vertical:
            lines = [VerticalRegion(q) for q in lines]
        res = dict(lines=lines, threshold=int(t["threshold"]), ink="dark" if t["ink"] == ops._lib.INK_DARK else "light")
        if blk.skew is not None:
            table_angles = ops.skew_table(blk.skew, blk.max_skew, vertical)
            angle = table_angles[int(sk["chosen"])]
            res["skew"] = float(blk.skew) if not isinstance(blk.skew, str) else 0.0 - angle if vertical else angle
        out.append(res)
    return out


def skew_lines(rect, vertical, c, s, u_min, v_min, frame_lines):
    """The lines of a skewed block (DESIGN.md 7b, "Skewed blocks") from its frame lines (c0, l0, c1, l1): edges a = u_min - 0.5
    + c and b = v_min - 0.5 + l along e = (c, -s) and f = (s, c) from the crop's centre O, each corner O + a e + b f in fp64.
    OrientedRegions top to bottom, or for a vertical block (whose frame is the transposed crop) VerticalRegions of
    OrientedRegions, tl -> tr across the column, right to left."""
    x0, y0, x1, y1 = rect
    ox, oy = (y0 + (y1 - y0) / 2, x0 + (x1 - x0) / 2) if vertical else (x0 + (x1 - x0) / 2, y0 + (y1 - y0) / 2)
    ex, ey, fx, fy = c, -s, s, c
    out = []
    for c0, l0, c1, l1 in frame_lines:
        a0, a1 = u_min - 0.5 + c0, u_min - 0.5 + c1
        b0, b1 = v_min - 0.5 + l0, v_min - 0.5 + l1
        tl = (ox + a0 * ex + b0 * fx, oy + a0 * ey + b0 * fy)
        tr = (ox + a1 * ex + b0 * fx, oy + a1 * ey + b0 * fy)
        bl = (ox + a0 * ex + b1 * fx, oy + a0 * ey + b1 * fy)
        out.append(VerticalRegion(OrientedRegion(tl[::-1], bl[::-1], tr[::-1])) if vertical else OrientedRegion(tl, tr, bl))
    return out[::-1] if vertical else out


@torch.no_grad()
def find_lines(images, blocks):
    """The lines of text blocks (DESIGN.md 7b, "Text blocks"): Otsu's threshold of each block's grey crop, the ink's row profile
    (column profile for a vertical block) and its runs, merged across small gaps, short ones dropped, padded.

    images: uint8 [H, W, 3] numpy arrays or CPU / CUDA tensors, in any channel order; blocks: per image, a list of TextBlocks.
    Every block of the call goes through the same four launches (ops.find_lines), and its line table comes back in one pinned
    copy and one synchronisation; host images go to the device in one pinned copy.
    Returns per image a list with one dict per block: lines, integer rectangles (x0, y0, x1, y1) in image pixels top to bottom
    (VerticalRegions of such rectangles, right to left, for a vertical block), each one a region restore_regions takes;
    threshold, Otsu's t; ink, "dark" or "light".  Raises ValueError naming the image and the block, before any launch, for a
    block restore_regions would reject, and after the segmentation for a block of more than 256 lines.
    A block with ``skew`` (DESIGN.md 7b, "Skewed blocks") has its angle searched (or given) on the device and is split in the
    rotated frame; a call that holds one runs every block through ops.find_lines' six launches.  Its dict gains ``skew``, the
    angle used in degrees, and its lines are OrientedRegions (VerticalRegions of OrientedRegions for a vertical block), or the
    rectangles of skew=None when the angle is exactly 0."""
    imgs = [_as_image(im, i) for i, im in enumerate(images)]
    blocks = _per_image(blocks, len(imgs), "blocks (one list per image)")
    items, names = [], []
    for i, im in enumerate(imgs):
        for r, blk in enumerate(blocks[i] or []):
            names.append(f"image {i}, block {r}")
            if not isinstance(blk, TextBlock):
                raise ValueError(f"{names[-1]}: expected a TextBlock, got {blk!r}")
            items.append((i, blk, _check_block(blk, im.shape[0], im.shape[1], names[-1])))
    out = [[] for _ in imgs]
    if not items:
        return out
    dev = next((im.device for im in imgs if im.is_cuda), torch.device("cuda", torch.cuda.current_device()))
    with torch.cuda.device(dev):
        res = _find_lines(_device_images(sorted({i for i, _, _ in items}), imgs, dev), items)
    for (i, _, _), name, r in zip(items, names, res):
        if isinstance(r, str):
            raise ValueError(f"{name}: {r}")
        out[i].append(r)
    return out


def _plan_blocks(shapes, regions, labels, boxes):
    """restore_regions' text blocks, validated before any launch: [(image, region index, TextBlock, rect)], and the region lists
    with each block in place of its rectangle (plan_regions validates the other regions on them)."""
    n = len(shapes)
    regions, labels, boxes = (_per_image(v, n, f"{what} (one list per image)") for v, what in
                              ((regions, "regions"), (labels, "labels"), (boxes, "boxes")))
    blocks, stand_in = [], []
    for i, (H, W) in enumerate(shapes):
        rects = list(regions[i] or [])
        labs = _per_image(labels[i], len(rects), f"image {i}: labels (one entry per region)")
        bxs = _per_image(boxes[i], len(rects), f"image {i}: boxes (one entry per region)")
        for r, reg in enumerate(rects):
            if isinstance(reg, TextBlock):
                name = f"image {i}, region {r} (a text block)"
                if labs[r] is not None or bxs[r] is not None:
                    raise ValueError(f"{name}: labels or boxes are given, but its lines are only found on the device (call "
                                     f"find_lines and give the lines with their labels)")
                rects[r] = _check_block(reg, H, W, name)
                blocks.append((i, r, reg, rects[r]))
        stand_in.append(rects)
    return blocks, stand_in


def _expand_blocks(regions, labels, boxes, blocks, found, skip_invalid, shapes=None, scale=4, feather=None):
    """The region, label and box lists with each text block replaced in place by its lines, and per image the layout of its given
    regions: None for a region, the block's find_lines result (or dict(error=...) under ``skip_invalid``) for a block.  A block
    with too many lines, a vertical line that vertical_plan rejects, or an oriented line of a skewed block that plan_regions
    rejects (on the image of ``shapes`` at ``scale`` and ``feather``) raises ValueError without ``skip_invalid``."""
    found = {(i, r): res for (i, r, _, _), res in zip(blocks, found)}
    n = len(regions)
    labels, boxes = _per_image(labels, n, "labels"), _per_image(boxes, n, "boxes")
    out_r, out_l, out_b, layout = [], [], [], []
    for i in range(n):
        rects = list(regions[i] or [])
        labs, bxs = _per_image(labels[i], len(rects), "labels"), _per_image(boxes[i], len(rects), "boxes")
        rs, ls, bs, lay = [], [], [], []
        for r, reg in enumerate(rects):
            res = found.get((i, r))
            if res is None:
                rs.append(reg), ls.append(labs[r]), bs.append(bxs[r]), lay.append(None)
                continue
            name = f"image {i}, region {r} (a text block)"
            err = f"{name}: {res}" if isinstance(res, str) else None
            try:
                for k, q in enumerate(res["lines"] if err is None else []):
                    if isinstance(q, OrientedRegion) or isinstance(q, VerticalRegion) and isinstance(q.shape, OrientedRegion):
                        try:
                            plan_regions([shapes[i]], [[q]], None, None, scale, feather)
                        except ValueError as e:
                            raise ValueError(f"{name}, line {k}: {str(e).split(': ', 1)[-1]}") from None
                    elif isinstance(q, VerticalRegion):
                        vertical_plan(q.shape[2] - q.shape[0], q.shape[3] - q.shape[1], name=f"{name}, line {k}")
            except ValueError as e:
                err = str(e)
            if err is not None:
                if not skip_invalid:
                    raise ValueError(err)
                lay.append(dict(error=err))
                continue
            rs += res["lines"]
            ls += [None] * len(res["lines"])
            bs += [None] * len(res["lines"])
            lay.append(res)
        out_r.append(rs)
        out_l.append(None if labels[i] is None else ls)
        out_b.append(None if boxes[i] is None else bs)
        layout.append(lay)
    return out_r, out_l, out_b, layout


def _regroup_blocks(out, layout):
    """restore_regions' result with each block's line entries gathered into the block's own entry, in place."""
    for img, lay in zip(out, layout):
        flat, o, img["regions"] = img["regions"], 0, []
        for res in lay:
            if res is None:
                img["regions"].append(flat[o])
                o += 1
            elif "error" in res:
                img["regions"].append(res)
            else:
                img["regions"].append(dict(res, regions=flat[o:o + len(res["lines"])]))
                o += len(res["lines"])


def plan_regions(shapes, regions, labels=None, boxes=None, scale=4, feather=None):
    """restore_regions' host plan, validated before any launch.  shapes: (H, W) per image; regions: per image, a list of integer
    half-open rectangles (x0, y0, x1, y1) and OrientedRegions; labels / boxes: None, or per image None or a list with one entry
    per region (None: predicted, else the region's labels / its detector boxes [x1, y1, x2, y2], in IMAGE coordinates for a
    rectangle and in the rectified crop's frame for an oriented region).  Returns the RegionPlans of every region, image by
    image in region order.
    Raises ValueError: scale not an integer in [1, 8], feather < 0, and, naming the image and the region, a rectangle that is
    empty or leaves the image, an oriented region with corners that are not finite, a side shorter than 1 pixel, mirrored or
    sheared past |e x f| < |e| |f| / 2, its centre outside the image, a crop, restored width or image side over 32767 pixels or
    a page map beyond OpenCV's fixed-point range, a label / box count mismatch, boxes without labels, a box outside the region's
    columns ([x0, x1] for a rectangle, [0, w_r] for an oriented region).  QuadRegions are validated likewise (DESIGN.md 7b,
    "Perspective text regions"): corners not finite, a side shorter than 1 pixel, not strictly convex in reading order, an
    interior angle outside [30, 150] degrees, foreshortening beyond 4, the centre outside the image, a side over 32767 pixels,
    a page map whose denominator is not positive over the footprint box or whose fixed-point coordinates leave +-2^30.
    A VerticalRegion (DESIGN.md 7b, "Vertical text columns") is validated as its shape, its labels and boxes in its crop C's frame,
    and further rejected for a shape that is itself a VerticalRegion or a CurvedRegion and for vertical_plan's errors.
    A CurvedRegion (DESIGN.md 7b, "Curved text regions") is rejected for points that are not finite, curves without 3k+1 points,
    with different k or k outside [1, 8], a band under one pixel, a segment whose mid curve is shorter than h_r / 8, a Jacobian of
    P(t, b) = (1 - b) T + b B that is not positive on the 33 x 5 grid of a segment (folds, mirrored or reversed reading order), a
    ruling B - T that turns by more than 90 degrees within a segment, a longest ruling over 4 times the shortest, the mid point
    at a = 0.5 outside the image, a side over 32767 pixels and a crop map beyond +-2^14; its labels and boxes are in its crop's
    frame."""
    if isinstance(scale, bool) or not isinstance(scale, int) or not 1 <= scale <= 8:
        raise ValueError(f"scale must be an integer in [1, 8], got {scale!r}")
    if feather is not None and (isinstance(feather, bool) or not isinstance(feather, int) or feather < 0):
        raise ValueError(f"feather must be an integer >= 0 output pixels, got {feather!r}")
    n = len(shapes)
    regions, labels, boxes = (_per_image(v, n, f"{what} (one list per image)") for v, what in
                              ((regions, "regions"), (labels, "labels"), (boxes, "boxes")))
    plan = []
    for i, (H, W) in enumerate(shapes):
        rects = list(regions[i] or [])
        labs = _per_image(labels[i], len(rects), f"image {i}: labels (one entry per region)")
        bxs = _per_image(boxes[i], len(rects), f"image {i}: boxes (one entry per region)")
        first = len(plan)
        s = scale
        for r, rect in enumerate(rects):
            name = f"image {i}, region {r}"
            maps, column, vplan = None, None, []
            lab, bx = labs[r], bxs[r]
            if isinstance(rect, VerticalRegion):
                vreg, rect = rect, rect.shape
                if isinstance(rect, VerticalRegion):
                    raise ValueError(f"{name}: the shape of a VerticalRegion is itself a VerticalRegion")
                if isinstance(rect, CurvedRegion):
                    raise ValueError(f"{name}: the shape of a VerticalRegion is a CurvedRegion (curved columns are not supported)")
                if lab is not None:
                    lab = [int(v) for v in torch.as_tensor(lab, dtype=torch.long).reshape(-1).tolist()]
                if bx is not None and lab is None:
                    raise ValueError(f"{name}: boxes without labels (predicted labels pair only with predicted boxes)")
                if bx is not None and len(lab) != len(bx):
                    raise ValueError(f"{name}: {len(lab)} labels for {len(bx)} boxes")

                def column(w_r, h_r, _v=vreg, _bx=bx, _name=name, _out=vplan):
                    _out.append(vertical_plan(w_r, h_r, _v.cells, _bx, _name))
                    return _out[0].t_size
            if isinstance(rect, OrientedRegion):
                maps, (x0, y0, x1, y1), out = _plan_oriented(rect, H, W, s, name, column)
                cols = (0, maps.size[0])
            elif isinstance(rect, QuadRegion):
                maps, (x0, y0, x1, y1), out = _plan_quad(rect, H, W, s, name, column)
                cols = (0, maps.size[0])
            elif isinstance(rect, CurvedRegion):
                maps, (x0, y0, x1, y1), out = _plan_curved(rect, H, W, s, name)
                cols = (0, maps.size[0])
            else:
                try:
                    x0, y0, x1, y1 = (int(v) for v in rect)
                    if (x0, y0, x1, y1) != tuple(rect):
                        raise ValueError
                except (TypeError, ValueError):
                    raise ValueError(f"{name}: expected an integer rectangle (x0, y0, x1, y1) or an OrientedRegion, "
                                     f"got {rect!r}") from None
                if not (0 <= x0 < x1 <= W and 0 <= y0 < y1 <= H):
                    raise ValueError(f"{name}: rectangle {(x0, y0, x1, y1)} is empty or outside the {W}x{H} image")
                out, cols = (s * x0, s * y0, s * x1, s * y1), (x0, x1)
                if column is not None:
                    column(x1 - x0, y1 - y0)
            if column is not None:
                bx = vplan[0].boxes
            elif lab is not None:
                lab = [int(v) for v in torch.as_tensor(lab, dtype=torch.long).reshape(-1).tolist()]
            if bx is not None and column is None:
                if lab is None:
                    raise ValueError(f"{name}: boxes without labels (predicted labels pair only with predicted boxes)")
                if len(lab) != len(bx):
                    raise ValueError(f"{name}: {len(lab)} labels for {len(bx)} boxes")
                for k, b in enumerate(bx):
                    b = [float(v) for v in b]
                    if len(b) != 4 or not cols[0] <= b[0] <= b[2] <= cols[1]:
                        raise ValueError(f"{name}, character {k}: box {b} is outside the region's columns [{cols[0]}, {cols[1]}]")
                dx, dy = (0, 0) if maps else (x0, y0)
                bx = [[float(b[0]) - dx, float(b[1]) - dy, float(b[2]) - dx, float(b[3]) - dy] for b in bx]
            overlaps = [first + j for j, q in enumerate(plan[first:]) if max(out[0], q.out[0]) < min(out[2], q.out[2])
                        and max(out[1], q.out[1]) < min(out[3], q.out[3])]
            corners = tuple((float(p[0]), float(p[1])) for p in rect) if maps and not isinstance(rect, CurvedRegion) else ()
            if isinstance(rect, CurvedRegion):
                plan.append(RegionPlan(i, r, (x0, y0, x1, y1), out, overlaps, lab, bx, size=maps.size,
                                       curved=CurvedRegion(maps.top, maps.bottom)))
                continue
            if isinstance(rect, QuadRegion):
                extra = (None, maps.matrix, maps.size, QuadRegion(*corners))
            else:
                extra = (OrientedRegion(*corners), maps.matrix, maps.size) if maps else ()
            plan.append(RegionPlan(i, r, (x0, y0, x1, y1), out, overlaps, lab, bx, *extra, vertical=vplan[0] if vplan else None))
    return plan


def region_chains(plan, ok):
    """The chains mn_composite_regions_u8 reads: for each region k of ``ok`` (increasing indices into the plan: the regions that
    are composed), the positions in ``ok`` of every region of ok whose rectangle meets k's, k included, in order."""
    later = {k: [] for k in range(len(plan))}
    for k, p in enumerate(plan):
        for j in p.overlaps:
            later[j].append(k)
    index = {k: j for j, k in enumerate(ok)}
    return [[index[j] for j in plan[k].overlaps + [k] + later[k] if j in index] for k in ok]


def _flat_views(shapes, dev):
    """uint8 [h, w, 3] views, one per (h, w) of ``shapes``, packed in one device buffer."""
    n = [3 * h * w for h, w in shapes]
    buf = torch.empty(sum(n), dtype=torch.uint8, device=dev)
    return [buf[o - k:o].view(h, w, 3) for k, o, (h, w) in zip(n, itertools.accumulate(n), shapes)]


def _to_host_all(tensors):
    """Device tensors -> numpy arrays of the same shapes, through ONE pinned buffer and one synchronisation."""
    total = sum(t.numel() for t in tensors)
    pinned = torch.empty(max(total, 1), dtype=torch.uint8, pin_memory=True)
    out, o = [], 0
    for t in tensors:
        v = pinned[o:o + t.numel()].view(t.shape)
        v.copy_(t, non_blocking=True)
        out.append(v)
        o += t.numel()
    if tensors:
        torch.cuda.current_stream(tensors[0].device).synchronize()
    return [v.numpy() for v in out]


@torch.no_grad()
def restore_regions(encoder, tspgan, sr, images, regions, labels=None, boxes=None, scale=4, feather=None, max_lines=8, context=16,
                    overlap=64, whole_lines=False, skip_invalid=False, to_host=False):
    """Restore rectangles of small text inside whole images and compose them into the images upscaled ``scale`` times
    (DESIGN.md section 7b, "Text regions in whole images").

    images: uint8 [H, W, 3] numpy arrays or CPU / CUDA tensors, in any channel order; regions: per image, a list of integer
    rectangles (x0, y0, x1, y1), 0 <= x0 < x1 <= W, 0 <= y0 < y1 <= H, and OrientedRegions, in the order they compose; labels /
    boxes: as plan_regions takes them (boxes in image coordinates; None entries are predicted, exactly as restore_images
    predicts).
    scale s: an integer in [1, 8]; feather F >= 0 output pixels (default 2 s).
    The result of an image is out = B = cv2.resize(img, (0, 0), fx=s, fy=s, INTER_CUBIC) (OpenCV's own path), then for each region
    that did not fail, in order, over its rectangle R = [s x0, s x1) x [s y0, s y1):
      P = cv2.resize(T[..., ::-1], (s (x1 - x0), s (y1 - y0)), INTER_CUBIC), T = restore_images' sr_u8 of img[y0:y1, x0:x1];
      out = sat_u8(rint(fl(fl(a P) + fl(fl(1 - a) out)))), a = min(1, fl((float)d + 0.5) / F), d the distance to the nearest
      side of R that is not on the image border (a = 1 when F = 0 or no side counts).
    One call: the host images go to the device in one pinned copy; restore_images runs on views of the uploaded images (every
    region of every image shares its batches; max_lines, context, overlap, whole_lines and skip_invalid are passed on); one
    launch computes every background (mn_resize_cubic_u8_batched) and one composes every region (mn_composite_regions_u8).
    Returns one dict per image: image (uint8 [s H, s W, 3]) and regions, one entry per region: dict(sr_u8, segments, labels,
    boxes) -- boxes in image coordinates, predicted ones shifted back -- or, with ``skip_invalid``, dict(error=...) for a region
    restore_images rejected, whose rectangle keeps the background.  Results stay on the device, or come back as numpy arrays
    through one pinned buffer and one synchronisation with ``to_host``.  plan_regions' errors are raised whatever skip_invalid.
    An OrientedRegion (DESIGN.md 7b, "Oriented text regions") is restored from its rectified crop
    C = cv2.warpAffine(img, M, (w_r, h_r), INTER_CUBIC | WARP_INVERSE_MAP, BORDER_REPLICATE) (oriented_maps; every crop of the
    call in one mn_warp_affine_u8_batched launch), its labels and boxes given and returned in C's frame, and its entry gains
    ``matrix`` (M) and ``size`` ((w_r, h_r)).  Its T is warped back by N onto its footprint with a feather on all four sides, and
    a call that holds one composes every region with mn_composite_regions_affine_u8 instead of mn_composite_regions_u8.
    A QuadRegion (DESIGN.md 7b, "Perspective text regions") is handled alike through quad_maps: C = cv2.warpPerspective(img, M,
    (w_r, h_r), INTER_CUBIC | WARP_INVERSE_MAP, BORDER_REPLICATE) (every quad of the call in one mn_warp_perspective_u8_batched
    launch), T warped back by the 3 x 3 N, and a call that holds one composes every region with mn_composite_regions_quad_u8.
    A VerticalRegion (DESIGN.md 7b, "Vertical text columns") takes its shape's crop C (rectified in its kind's launch), lays its
    cells side by side as the line L (vertical_plan; every column of the call in one mn_vertical_layout_u8_batched launch before
    restore_images), restores L to T and puts T back into the column T_col [H_c, W_c] (one mn_vertical_unlayout_u8_batched launch
    after it), which is composed as its shape composes T.  Its labels and boxes are given and returned in C's frame; its entry's
    sr_u8 is T_col, and it gains line_u8 (T) and cells ([c_0, ..., c_n]).
    A CurvedRegion (DESIGN.md 7b, "Curved text regions") is restored from its rectified crop C = cv2.remap(img, fl32(mapx),
    fl32(mapy), INTER_CUBIC, BORDER_REPLICATE) with curved_maps' crop map (every curved crop of the call in one
    mn_remap_curved_u8_batched launch), its labels and boxes given and returned in C's frame, and its entry gains ``size``
    ((w_r, h_r)).  Each page pixel of its footprint is inverted onto T by bisection along the curves, feathered on all four
    sides, and a call that holds one composes every region with mn_composite_regions_curved_u8.
    A TextBlock (DESIGN.md 7b, "Text blocks") is split into lines on the uploaded images first (find_lines: every block of the
    call in the same four launches, one pinned copy of the line table and one synchronisation), and its lines, rectangles or
    VerticalRegions, take its place in the region list; the call then goes on as if they had been given.  No labels or boxes
    may be given for a block.  Its entry is dict(lines, threshold, ink, regions), regions one entry per line as above; a block
    of more than 256 lines, or with a vertical line vertical_plan rejects, raises, or is dict(error=...) with ``skip_invalid``.
    A skewed block (DESIGN.md 7b, "Skewed blocks") takes the place of its OrientedRegion lines alike, and its entry gains
    ``skew``; a line plan_regions rejects makes the block's error."""
    from . import ops
    imgs = [_as_image(im, i) for i, im in enumerate(images)]
    shapes = [im.shape[:2] for im in imgs]
    blocks, stand_in = _plan_blocks(shapes, regions, labels, boxes)
    plan = plan_regions(shapes, stand_in if blocks else regions, labels, boxes, scale, feather)
    feather = 2 * scale if feather is None else feather
    if not imgs:
        return []
    dev = next(encoder.parameters()).device
    with torch.cuda.device(dev):
        dimg = _device_images(range(len(imgs)), imgs, dev)
        if blocks:                                       # every block's lines take its place in the region list
            found = _find_lines(dimg, [(i, blk, rect) for i, _, blk, rect in blocks])
            regions, labels, boxes, layout = _expand_blocks(regions, labels, boxes, blocks, found, skip_invalid, shapes, scale,
                                                            feather)
            plan = plan_regions(shapes, regions, labels, boxes, scale, feather)
        crops = [dimg[p.image][p.rect[1]:p.rect[3], p.rect[0]:p.rect[2]] for p in plan]
        oriented = [k for k, p in enumerate(plan) if p.oriented is not None]
        quads = [k for k, p in enumerate(plan) if p.quad is not None]
        curved = [k for k, p in enumerate(plan) if p.curved is not None]
        if oriented or quads or curved:                  # every region of a kind rectified in one launch
            n_crop = [3 * plan[k].size[0] * plan[k].size[1] for k in oriented + quads + curved]
            cbuf = torch.empty(sum(n_crop), dtype=torch.uint8, device=dev)
            o = 0
            for k, nb in zip(oriented + quads + curved, n_crop):
                crops[k] = cbuf[o:o + nb].view(plan[k].size[1], plan[k].size[0], 3)
                o += nb
            if oriented:
                ops.warp_affine([(dimg[plan[k].image], crops[k], plan[k].matrix) for k in oriented])
            if quads:
                ops.warp_perspective([(dimg[plan[k].image], crops[k], plan[k].matrix) for k in quads])
            if curved:
                ops.remap_curved([(dimg[plan[k].image], crops[k], curved_maps(plan[k].curved, scale).curve(scale))
                                  for k in curved])
        verts = [k for k, p in enumerate(plan) if p.vertical is not None]
        if verts:                                        # every column laid out as a line in one launch
            lines = _flat_views([(plan[k].vertical.line_height, len(plan[k].vertical.heights) * plan[k].vertical.size[0])
                                 for k in verts], dev)
            ops.vertical_layout([(crops[k], line, layout_cells(plan[k].vertical)) for k, line in zip(verts, lines)])
            for k, line in zip(verts, lines):
                crops[k] = line
        res = restore_images(encoder, tspgan, sr, crops, [p.labels for p in plan], [p.boxes for p in plan], max_lines=max_lines,
                             context=context, skip_invalid=skip_invalid, whole_lines=whole_lines, overlap=overlap) if plan else []
        ts = {k: r["sr_u8"] for k, r in enumerate(res) if "error" not in r}
        vok = [k for k in verts if k in ts]
        if vok:                                          # every restored line put back into its column in one launch
            cols = _flat_views([plan[k].vertical.t_size[::-1] for k in vok], dev)
            ops.vertical_unlayout([(ts[k], col, unlayout_cells(plan[k].vertical, ts[k].shape[1])) for k, col in zip(vok, cols)])
            ts.update(zip(vok, cols))
        sizes = [scale * scale * im.shape[0] * im.shape[1] * 3 for im in imgs]
        flat = torch.empty(sum(sizes), dtype=torch.uint8, device=dev)
        offs = [sum(sizes[:i]) for i in range(len(imgs))]
        pages = [flat[o:o + n].view(scale * im.shape[0], scale * im.shape[1], 3) for o, n, im in zip(offs, sizes, imgs)]
        ops.resize_cubic([(dimg[i], pages[i]) for i in range(len(imgs))])
        ok = [k for k, r in enumerate(res) if "error" not in r]
        if ok:                                           # a column composes its T_col where any other region composes its T
            items = [(pages[plan[k].image], ts[k], plan[k].out, chain) for k, chain in zip(ok, region_chains(plan, ok))]
            if curved:
                maps = [curved_maps(plan[k].curved, scale, *ts[k].shape[1::-1]) if plan[k].curved is not None else
                        quad_maps(plan[k].quad, scale, *ts[k].shape[1::-1]) if plan[k].quad is not None else
                        oriented_maps(plan[k].oriented, scale, *ts[k].shape[1::-1]) if plan[k].oriented is not None else None
                        for k in ok]
                ops.composite_regions_curved([it + (m and ((m.curve(scale) if isinstance(m, CurvedMaps) else m.page_map),
                                                           m.kx, m.ky),) for it, m in zip(items, maps)], feather)
            elif quads:
                maps = [quad_maps(plan[k].quad, scale, *ts[k].shape[1::-1]) if plan[k].quad is not None else
                        oriented_maps(plan[k].oriented, scale, *ts[k].shape[1::-1]) if plan[k].oriented is not None else None
                        for k in ok]
                ops.composite_regions_quad([it + (m and (m.page_map, m.kx, m.ky),) for it, m in zip(items, maps)], feather)
            elif oriented:
                maps = [None if plan[k].oriented is None else oriented_maps(plan[k].oriented, scale, *ts[k].shape[1::-1])
                        for k in ok]
                ops.composite_regions_affine([it + (m and (m.page_map, m.kx, m.ky),) for it, m in zip(items, maps)], feather)
            else:
                ops.composite_regions(items, feather)
        srs, lines = ts, {k: res[k]["sr_u8"] for k in vok}
        if to_host:
            host = _to_host_all([flat] + list(srs.values()) + list(lines.values()))
            pages = [host[0][o:o + n].reshape(pg.shape) for o, n, pg in zip(offs, sizes, pages)]
            srs = dict(zip(srs, host[1:1 + len(srs)]))
            lines = dict(zip(lines, host[1 + len(srs):]))
    out = [dict(image=pages[i], regions=[]) for i in range(len(imgs))]
    for k, p in enumerate(plan):
        r = res[k]
        if "error" in r:
            entry = dict(error=r["error"])
        elif "boxes" in r and p.vertical is not None:
            entry = dict(sr_u8=srs[k], segments=r["segments"], labels=r["labels"], boxes=column_boxes(p.vertical, r["boxes"]))
        elif "boxes" in r:
            x0, y0 = (0, 0) if p.oriented or p.quad or p.curved else p.rect[:2]
            entry = dict(sr_u8=srs[k], segments=r["segments"], labels=r["labels"],
                         boxes=[[b[0] + x0, b[1] + y0, b[2] + x0, b[3] + y0] for b in r["boxes"]])
        else:
            entry = dict(sr_u8=srs[k], segments=r["segments"], labels=p.labels, boxes=boxes[p.image][p.region])
        if p.vertical is not None and "error" not in r:
            entry.update(line_u8=lines[k], cells=list(p.vertical.cells))
        if (p.oriented or p.quad) and "error" not in r:
            entry.update(matrix=p.matrix.copy(), size=p.size)
        if p.curved and "error" not in r:
            entry.update(size=p.size)
        out[p.image]["regions"].append(entry)
    if blocks:
        _regroup_blocks(out, layout)
    return out


# ---------------------------------------------------------------------------------------------------------------------
# Per-layer precision plan (SURVEY.md section 8f row n4): fp16x3 / bf16x3 / fp32 and a power-of-two input scale per conv layer,
# chosen on calibration inputs against the exact fp32 kernels.  Needed the day real checkpoints replace the synthetic ones: the
# default fp16 hi/lo split (conv_tc2.cu) has fp32-grade mantissa but fp16's exponent range.
# ---------------------------------------------------------------------------------------------------------------------
def conv_layers(*modules):
    """Every ops.ConvWeight of the (already used, hence packed) modules, in pack order."""
    from . import ops
    out, seen = [], set()

    def walk(o):
        if isinstance(o, ops.ConvWeight):
            if id(o) not in seen:
                seen.add(id(o)); out.append(o)
        elif isinstance(o, dict):
            for v in o.values():
                walk(v)
        elif isinstance(o, (list, tuple)):
            for v in o:
                walk(v)

    for m in modules:
        for sub in m.modules():
            walk(getattr(sub, "_packed", None))
    return out


@torch.no_grad()
def tune_precision(encoder, tspgan, sr, lq, labels=None, locs=None, target_absmax=1024.0, fp32_fallback=1e-3, compare=True):
    """Calibrate the per-layer precision plan on (lq, labels, locs) -- representative LR lines -- and install it (ops.PLAN).

    pass 1 (range-safe bf16 split everywhere): max |input| of every tensor-core conv -> x_scale = 2^k with
            |x| * x_scale ~ ``target_absmax`` (64x headroom below 65504, inputs down to 2^-24 * target keep full hi/lo precision);
    pass 2 (``compare``): every such layer also runs through the exact fp32 kernel and through both split formats; the format with
            the smaller relative max-abs error wins, and a layer whose best error still exceeds ``fp32_fallback`` (relative to its
            output's max) runs on the fp32 CUDA-core kernel;
    pass 3: the plan is verified -- one more step, no range flag may rise.
    Returns a list of dict(name, absmax, x_scale, precision, err_f16x3, err_bf16x3), one per tensor-core conv layer."""
    import math
    from . import ops
    dev = lq.device
    with torch.cuda.device(dev):
        old_default = ops.default_precision()
        restore_lines(encoder, tspgan, sr, lq, labels, locs, check_range=False)     # packs the weights
        layers = conv_layers(encoder, tspgan, sr)
        for cw in layers:
            cw.set_plan(x_scale=1.0)
            cw.precision = None
            ops.PLAN[cw.name] = (None, 1.0)
        ops.PLAN_VERSION += 1
        try:
            ops.set_default_precision(ops.PREC_BF16X3_TC)
            with ops.calibration(dev) as cal:
                restore_lines(encoder, tspgan, sr, lq, labels, locs, check_range=False)
            res = cal.results()
        finally:
            ops.set_default_precision(old_default)
        ops.poll_range(dev, reroute=False)
        for cw, r in res.items():
            a = r["absmax"]
            k = 0 if not (a > 0 and math.isfinite(a)) else max(-24, min(24, round(math.log2(target_absmax / a))))
            cw.set_plan(x_scale=2.0 ** k)
        errs = {}
        if compare:
            with ops.calibration(dev, compare=True) as cal:
                restore_lines(encoder, tspgan, sr, lq, labels, locs, check_range=False)
            errs = cal.results()
            ops.poll_range(dev, reroute=False)
        report = []
        for cw, r in res.items():
            e = errs.get(cw, {})
            e16, ebf = e.get("err_f16x3", float("nan")), e.get("err_bf16x3", float("nan"))
            prec = ops.PREC_F16X3_TC
            if compare and cw in errs:
                prec = ops.PREC_F16X3_TC if (e16 <= ebf or not math.isfinite(ebf)) and math.isfinite(e16) else ops.PREC_BF16X3_TC
                if not (min(e16, ebf) <= fp32_fallback):
                    prec = ops.PREC_FP32_SIMT
            cw.set_plan(precision=prec)
            report.append(dict(name=cw.name, absmax=r["absmax"], x_scale=cw.x_scale, precision=prec, err_f16x3=e16, err_bf16x3=ebf))
        restore_lines(encoder, tspgan, sr, lq, labels, locs, check_range=False)
        torch.cuda.synchronize(dev)
        ops.check_range(dev)
    return report


def save_precision_plan(path):
    """ops.PLAN -> JSON {layer name: [precision or null, x_scale]}."""
    import json
    from . import ops
    with open(path, "w") as f:
        json.dump({k: [v[0], v[1]] for k, v in ops.PLAN.items()}, f, indent=1, sort_keys=True)


def load_precision_plan(path_or_dict, *modules):
    """Install a saved plan; already-packed layers of ``modules`` are updated in place, later packs pick it up by name."""
    import json
    from . import ops
    plan = json.load(open(path_or_dict)) if isinstance(path_or_dict, str) else path_or_dict
    for k, (prec, xs) in plan.items():
        ops.PLAN[k] = (None if prec is None else int(prec), float(xs))
    for cw in conv_layers(*modules):
        if cw.name in ops.PLAN:
            cw.precision, cw.x_scale = ops.PLAN[cw.name]
    ops.PLAN_VERSION += 1
    return plan
