"""Self-contained line-restoration flow on top of the three modules (SURVEY.md section 8f rows n3 / n4).

The reference's ``test_sr.py`` takes character labels and boxes from a third-party YOLO + OCR front-end; the original
single-model flow uses the encoder's own predictions instead: CTC-style de-duplicated argmax labels (test_w.py:34-40) and
boxes converted from the encoder's (left, right) pairs to (centre, half-width) exactly as the training model does
(Train/tspgan/models/tspgan_model.py:331-337).  Integer outputs (labels) are computed on the host, bit-exactly like the
reference; everything numeric runs through the module API (and therefore through the CUDA kernels).
"""
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
    fp16 hi/lo split its layer is re-routed to the bf16 split and the step is re-run (at most 3 times) -- the caller never sees
    the Inf/NaN result."""
    if check_range:
        from . import ops
        for attempt in range(4):
            out = restore_lines(encoder, tspgan, sr, lq, labels, locs, max_chars, check_range=False)
            torch.cuda.synchronize(lq.device)
            if not ops.poll_range(lq.device) or attempt == 3:
                return out
    logits, locs_lr, w = encoder(lq)
    if labels is None:
        labels = []
        for b in range(lq.shape[0]):
            lab = decode_labels(logits[b])[:max_chars]
            labels.append(torch.tensor(lab, dtype=torch.long).reshape(-1, 1))
    if locs is None:
        locs = lr_to_center_halfwidth(locs_lr)
    counts = [int(l.shape[0]) for l in labels]
    total = sum(counts)
    p64, p32, priors = [], [], []
    if total > 0:
        styles = torch.cat([w[b:b + 1].expand(counts[b], -1) for b in range(lq.shape[0]) if counts[b] > 0], dim=0)
        lab_all = torch.cat([l for l in labels if l.shape[0] > 0], dim=0)
        img, f64, f32_ = tspgan(styles=styles, labels=lab_all, noise=None)       # one generator call for every character
        o = 0
        for n in counts:
            p64.append(f64[o:o + n]); p32.append(f32_[o:o + n]); priors.append(img[o:o + n]); o += n
    else:
        dev = lq.device
        for _ in counts:
            p64.append(torch.zeros(0, 256, 64, 64, device=dev)); p32.append(torch.zeros(0, 512, 32, 32, device=dev))
            priors.append(torch.zeros(0, 3, 128, 128, device=dev))
    out = sr(lq, p64, p32, locs)
    return dict(sr=out, prior=priors, labels=labels, locs=locs, w=w, logits=logits)


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
def restore_image(encoder, tspgan, sr, img_u8, labels, boxes, figure=False):
    """One text-line image end to end on the device (the body of test_sr.py's loop, :98-201, with the labels / boxes the
    detector and OCR produced): uint8 [h, w, 3] image (host numpy / tensor or CUDA tensor) -> dict(sr_u8 [128, W, 3] uint8 bytes
    as cv2.imwrite would store them, cropped to the line's width; sr fp32; lq; lq_width).
    Pre- and post-processing run as CUDA kernels (mn_preprocess_lq_u8 / mn_postprocess_sr_u8).
    ``figure=True`` adds ``figure``: the uint8 [512, W, 3] image test_sr.py writes (:206-231; ShowLQ, ShowLocs, ShowSR, prior;
    DESIGN.md section 7b), composed on the device (mn_figure_u8); ``sr_u8`` is then its view ``figure[256:384]``."""
    from . import ops
    dev = next(encoder.parameters()).device
    img = torch.as_tensor(img_u8)
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


@torch.no_grad()
def restore_images(encoder, tspgan, sr, images, labels, boxes, max_lines=8, context=16, skip_invalid=False, to_host=False,
                   whole_lines=False, figure=False):
    """Text-line images of any sizes end to end, batched: the flow of restore_image for every image, each cut into crops that
    fit the 32x512 LQ canvas (plan_segments) and every crop of every image run as one line of a batch of at most ``max_lines``.

    images: uint8 [h_i, w_i, 3] numpy arrays or CPU / CUDA tensors; labels / boxes: one list per image, as restore_image takes.
    Every image is planned and validated before any launch (a label outside the generator's classes raises IndexError, as the
    module would); with ``skip_invalid`` a bad image's entry becomes dict(error=...) and the others still run.  Per batch: one
    host->device copy of the batch's host images through pinned memory, one crop kernel (mn_preprocess_lq_u8_batched), the
    encoder, one TSPGAN call for all characters (each crop's characters take that crop's style w, as on a hand-made crop),
    TSPSRNet, a synchronisation and ops.poll_range (the batch re-runs, at most 3 times, when a layer was re-routed for fp16
    range), then one stitch kernel (mn_postprocess_sr_u8_pieces) into the images' outputs.
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
    the decoder lines, the encoder, one TSPGAN call, one ragged TSPSRNet call, the fp16-range re-run, one stitch kernel.

    ``figure=True`` (either mode) adds ``figure`` to every result: the uint8 [512, W_i, 3] image test_sr.py writes (:206-231;
    DESIGN.md section 7b) -- ShowLQ and ShowLocs (markers at locs = boxes_to_locs(boxes, h, Wc), img_max_width = 4*Wc), the
    image's sr_u8, and the priors this call generated (each character's in the style of the crop that owns it), all cropped to
    sr_u8's width.  ``sr_u8`` becomes the view ``figure[256:384]``, its bytes unchanged.  The batch that holds an image's last
    crop composes its figure: one more launch (mn_figure_u8) per batch, and the prior images are kept until then.  With
    ``to_host`` the figures come back through the same single pinned copy.  Error entries have no figure."""
    from . import ops
    n = len(images)
    if not (len(labels) == len(boxes) == n):
        raise ValueError(f"{n} images, {len(labels)} label lists, {len(boxes)} box lists")
    if max_lines < 1:
        raise ValueError("max_lines must be >= 1")
    dev = next(encoder.parameters()).device
    n_cls = tspgan.TextGenerator.input_text.TextEmbeddings.shape[0]
    results, imgs, labs, plans = [None] * n, [None] * n, [None] * n, [None] * n
    for i in range(n):
        try:
            img = _as_image(images[i], i)
            lab = [int(v) for v in torch.as_tensor(labels[i], dtype=torch.long).reshape(-1).tolist()]
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
    valid = [i for i in range(n) if plans[i] is not None]
    if not valid:
        return results
    if whole_lines:
        return _restore_whole_lines(encoder, tspgan, sr, imgs, labs, boxes, plans, valid, results, max_lines, to_host, dev, figure)
    rows = 512 if figure else 128
    with torch.cuda.device(dev):
        layout, total = {}, 0
        for i in valid:
            width, pieces = stitch_pieces(imgs[i].shape[0], imgs[i].shape[1], plans[i])
            layout[i] = (total, width, pieces)
            total += rows * width * 3
        flat = torch.empty(total, dtype=torch.uint8, device=dev)
        figs = {i: flat[o:o + rows * wd * 3].view(rows, wd, 3) for i, (o, wd, _) in layout.items()}
        outs = {i: f[256:384] for i, f in figs.items()} if figure else figs
        lines = [(i, k) for i in valid for k in range(len(plans[i]))]
        last_batch = {i: b0 for b0 in range(0, len(lines), max_lines) for i, _ in lines[b0:b0 + max_lines]}
        priors = {i: [] for i in valid}
        for b0 in range(0, len(lines), max_lines):
            batch = lines[b0:b0 + max_lines]
            dimg = _device_images(dict.fromkeys(i for i, _ in batch), imgs, dev)
            segs = [plans[i][k] for i, k in batch]
            lq, _ = ops.preprocess_lq_crops([(dimg[i], s.crop[0], s.crop[1]) for (i, _), s in zip(batch, segs)])
            counts = [s.chars[1] - s.chars[0] for s in segs]
            lab_all = torch.tensor([v for (i, _), s in zip(batch, segs) for v in labs[i][s.chars[0]:s.chars[1]]],
                                   dtype=torch.long).reshape(-1, 1)
            locs = torch.zeros(len(batch), 2 * max(1, max(counts)), dtype=torch.float32)
            for b, ((i, _), s) in enumerate(zip(batch, segs)):
                if counts[b]:
                    locs[b, :2 * counts[b]] = boxes_to_locs(s.boxes, imgs[i].shape[0], lq.shape[-1])[0]
            for attempt in range(4):
                _, _, w = encoder(lq)
                p64, p32, img_p = [], [], None
                if lab_all.shape[0] > 0:
                    styles = torch.cat([w[b:b + 1].expand(c, -1) for b, c in enumerate(counts) if c > 0], dim=0)
                    img_p, f64, f32_ = tspgan(styles=styles, labels=lab_all, noise=None)
                    o = 0
                    for c in counts:
                        p64.append(f64[o:o + c]); p32.append(f32_[o:o + c]); o += c
                else:
                    p64 = [torch.zeros(0, 256, 64, 64, device=dev) for _ in counts]
                    p32 = [torch.zeros(0, 512, 32, 32, device=dev) for _ in counts]
                out = sr(lq, p64, p32, locs)
                torch.cuda.synchronize(dev)
                if not ops.poll_range(dev) or attempt == 3:
                    break
            pieces = []
            for b, (i, k) in enumerate(batch):
                for kk, x0, src, wd in layout[i][2]:
                    if kk == k:
                        pieces.append((b, src, outs[i][:, x0:x0 + wd]))
            if pieces:
                ops.postprocess_sr_pieces(out, pieces)
            if figure:
                o = 0
                for (i, _), c in zip(batch, counts):            # crops in label order: the characters' priors in label order
                    priors[i] += list(img_p[o:o + c]) if c else []
                    o += c
                done = [i for i in dict.fromkeys(i for i, _ in batch) if last_batch[i] == b0]
                if done:
                    ops.figure_panels([(dimg[i], figs[i]) + _figure_markers_for(*imgs[i].shape[:2], boxes[i]) + (priors.pop(i),)
                                       for i in done])
        if to_host:
            pinned = _to_host(flat)
            figs = {i: pinned[o:o + rows * wd * 3].view(rows, wd, 3).numpy() for i, (o, wd, _) in layout.items()}
            outs = {i: f[256:384] for i, f in figs.items()} if figure else figs
    for i in valid:
        results[i] = dict(sr_u8=outs[i], segments=plans[i])
        if figure:
            results[i]["figure"] = figs[i]
    return results


def _restore_whole_lines(encoder, tspgan, sr, imgs, labs, boxes, plans, valid, results, max_lines, to_host, dev, figure):
    """restore_images(whole_lines=True) after validation: one decoder line per image (see restore_images)."""
    from . import ops
    rows = 512 if figure else 128
    with torch.cuda.device(dev):
        geo = {i: whole_line_width(imgs[i].shape[0], imgs[i].shape[1]) for i in valid}
        layout, total = {}, 0
        for i in valid:
            h, w = imgs[i].shape[:2]
            wc = geo[i][1]
            width = min(ops.round_half_even(w * (128 / h)), 4 * wc)
            layout[i] = (total, width)
            total += rows * width * 3
        flat = torch.empty(total, dtype=torch.uint8, device=dev)
        figs = {i: flat[o:o + rows * wd * 3].view(rows, wd, 3) for i, (o, wd) in layout.items()}
        outs = {i: f[256:384] for i, f in figs.items()} if figure else figs
        for bidx in pack_by_columns([geo[i][1] for i in valid], max_lines):
            batch = [valid[j] for j in bidx]
            dimg = _device_images(batch, imgs, dev)
            crops = [(i, s) for i in batch for s in plans[i]]              # encoder crops, 512 canvas
            lq_enc, _ = ops.preprocess_lq_crops([(dimg[i], s.crop[0], s.crop[1]) for i, s in crops])
            widths = [geo[i][1] for i in batch]
            canvas = max(widths)
            if canvas == 512:                 # only lines that fit: each is its single crop, exactly as without whole_lines
                lq = lq_enc
            else:
                lq, _ = ops.preprocess_lq_crops([(dimg[i], 0, imgs[i].shape[1]) for i in batch], out_w=canvas)
            counts = [len(labs[i]) for i in batch]
            owner = []                                                   # encoder crop (row of lq_enc) of every character
            c0 = 0
            for i in batch:
                for s in plans[i]:
                    owner += [c0] * (s.chars[1] - s.chars[0])
                    c0 += 1
            owner_t = torch.tensor(owner, dtype=torch.long).to(dev, non_blocking=True)
            lab_all = torch.tensor([v for i in batch for v in labs[i]], dtype=torch.long).reshape(-1, 1)
            locs = torch.zeros(len(batch), 2 * max(counts), dtype=torch.float32)
            for b, i in enumerate(batch):
                locs[b, :2 * counts[b]] = boxes_to_locs(boxes[i], imgs[i].shape[0], widths[b])[0]
            for attempt in range(4):
                _, _, w = encoder(lq_enc)
                img_p, f64, f32_ = tspgan(styles=w.index_select(0, owner_t), labels=lab_all, noise=None)
                p64, p32, o = [], [], 0
                for c in counts:
                    p64.append(f64[o:o + c]); p32.append(f32_[o:o + c]); o += c
                out = sr(lq, p64, p32, locs, widths=widths)
                torch.cuda.synchronize(dev)
                if not ops.poll_range(dev) or attempt == 3:
                    break
            ops.postprocess_sr_pieces(out, [(b, 0, outs[i]) for b, i in enumerate(batch)])
            if figure:                                          # every image of the batch is complete
                offs = [0]
                for c in counts:
                    offs.append(offs[-1] + c)
                ops.figure_panels([(dimg[i], figs[i]) + _figure_markers_for(*imgs[i].shape[:2], boxes[i]) +
                                   (list(img_p[offs[b]:offs[b + 1]]),) for b, i in enumerate(batch)])
        if to_host:
            pinned = _to_host(flat)
            figs = {i: pinned[o:o + rows * wd * 3].view(rows, wd, 3).numpy() for i, (o, wd) in layout.items()}
            outs = {i: f[256:384] for i, f in figs.items()} if figure else figs
    for i in valid:
        results[i] = dict(sr_u8=outs[i], segments=plans[i])
        if figure:
            results[i]["figure"] = figs[i]
    return results


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
