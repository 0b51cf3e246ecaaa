"""Torch-tensor wrappers over the C ABI (include/marconet_b200.h).

PyTorch is plumbing here: it owns device memory and the current CUDA stream; every
computation below is a kernel from libmarconet_b200.so.  Activations are NHWC fp32 views
``[N, H, W, C]`` with ``stride(-1) == 1`` whose pixel stride (``cs``) may exceed C (channel
slices of a concatenation buffer).
"""
import ctypes
import functools
import math
from typing import NamedTuple

import torch

from . import _lib
from ._lib import (ACT_GELU, ACT_LRELU02, ACT_NONE, ACT_RELU, ACT_RSQRT_EPS, ACT_SIGMOID, ACT_TANH,  # noqa: F401
                   PREC_BF16X3_TC, PREC_F16X1_TC, PREC_F16X3_TC, PREC_FP32_SIMT, ConvParams, Window)

import os as _os
import threading as _threading

_WS = {}
_WS_BYTES = 96 << 20
# per-thread launch context (graph.py captures per thread; two host threads must never see each other's scratch or error flag)
_TLS = _threading.local()
# 0 fp32 CUDA-core, 1 fp16x3 wgmma (default: parity-grade tensor-core path), 2 bf16x3 wgmma, 3 fp16x1 wgmma (not parity grade)
_DEFAULT_PRECISION = int(_os.environ.get("MN_PRECISION", PREC_F16X3_TC))
LAUNCHES = 0   # number of C-ABI kernel-launching calls issued (bench.py reports it)


def set_default_precision(p):
    global _DEFAULT_PRECISION
    _DEFAULT_PRECISION = int(p)


def graph_key():
    """Everything process-global that a captured CUDA graph of this library bakes in."""
    return (_DEFAULT_PRECISION, PLAN_VERSION, MAX_CTAS)


def graphs_allowed():
    """Module-level graph replay is off inside another capture, inside ops.deferred_checks (GraphedLines owns the step then) and
    while a calibration records per-layer statistics."""
    return (MODULE_GRAPHS and getattr(_TLS, "deferred_flag", None) is None and getattr(_TLS, "calib", None) is None
            and not torch.cuda.is_current_stream_capturing())


MODULE_GRAPHS = _os.environ.get("MN_MODULE_GRAPHS", "1") != "0"


def set_max_ctas(n):
    """Cap the persistent conv kernels at n CTAs (0 = all SMs); returns the previous cap."""
    global MAX_CTAS
    MAX_CTAS = int(n)
    return _lib.load().mn_set_max_ctas(int(n))


def default_precision():
    return _DEFAULT_PRECISION


def _stream():
    """The current stream of the CURRENT device.  Every wrapper checks (``_require_cuda``) that its tensors live on the current
    device, and the module forwards switch to their input's device (``torch.cuda.device(x.device)``), so a model on cuda:1 driven
    from a process whose current device is cuda:0 launches on cuda:1's stream, never on cuda:0's with cuda:1 pointers."""
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def on_device(t):
    """Context manager: make ``t``'s device current (stream, SM count, dynamic-smem attributes all follow the current device)."""
    return torch.cuda.device(t.device)


def _ptr(t):
    return None if t is None else ctypes.c_void_p(t.data_ptr())


def _require_cuda(t, name):
    if not isinstance(t, torch.Tensor) or not t.is_cuda:
        raise RuntimeError(f"marconet_b200: {name} must be a CUDA tensor (there is no CPU path)")
    if t.dtype != torch.float32:
        raise RuntimeError(f"marconet_b200: {name} must be float32, got {t.dtype}")
    if t.device.index != torch.cuda.current_device():
        raise RuntimeError(f"marconet_b200: {name} lives on {t.device} but the current CUDA device is cuda:{torch.cuda.current_device()}; "
                           f"call through the module API (it switches devices) or wrap the call in torch.cuda.device(...)")


def nhwc_info(t, name="tensor"):
    """(N, H, W, C, cs) of an NHWC view; verifies the stride pattern."""
    _require_cuda(t, name)
    if t.dim() != 4:
        raise RuntimeError(f"{name}: expected 4-D NHWC view, got {tuple(t.shape)}")
    n, h, w, c = t.shape
    sn, sh, sw, sc = t.stride()
    cs = sw if w > 1 else (sh if h > 1 else (sn if n > 1 else c))
    ok = (sc == 1 or c == 1) and (w == 1 or sw == cs) and (h == 1 or sh == w * cs) and (n == 1 or sn == h * w * cs)
    if not ok:
        raise RuntimeError(f"{name}: not a dense NHWC view (shape {tuple(t.shape)}, strides {t.stride()})")
    return n, h, w, c, cs


def workspace(device):
    """Split-K scratch of the conv kernels: one per device (single stream, like the reference scripts) unless a caller that runs
    convolutions on a second stream installs its own with ``use_workspace`` (per host thread)."""
    ov = getattr(_TLS, "ws_override", None)
    if ov is not None:
        return ov
    key = device.index if device.index is not None else torch.cuda.current_device()
    ws = _WS.get(key)
    if ws is None:
        ws = torch.empty(_WS_BYTES // 4, dtype=torch.float32, device=device)
        _WS[key] = ws
    return ws


class use_workspace:
    """Context manager: convolutions launched inside use ``ws`` (fp32 CUDA tensor) as their split-K scratch, so that they can run
    on another stream concurrently with convolutions that use the per-device scratch."""

    def __init__(self, ws):
        self.ws, self.prev = ws, None

    def __enter__(self):
        self.prev = getattr(_TLS, "ws_override", None)
        _TLS.ws_override = self.ws
        return self.ws

    def __exit__(self, *exc):
        _TLS.ws_override = self.prev
        return False


PLAN = {}     # layer name -> (precision or None, x_scale): the per-layer precision plan of this process (pipeline.tune_precision)
PLAN_VERSION = 0   # bumped whenever a layer's plan changes: captured CUDA graphs bake the plan in and key on it
MAX_CTAS = 0       # mirror of mn_set_max_ctas (grid sizes are baked into captured graphs)


class ConvWeight:
    """A conv/linear weight in kernel layout: fp32 K-major [KH*KW*Cin, Cout] plus (lazily) the hi/lo 16-bit
    planes [taps][Cout][Cin] the tensor-core path consumes (mn_conv_pack_weights_tc).

    Per-layer precision plan (SURVEY 8f n4; set by pipeline.tune_precision or by the range guard):
      ``precision``  None = the process default, else one of PREC_* for this layer;
      ``x_scale``    power of two applied to the layer's INPUT inside the kernel before the fp16 hi/lo split and undone
                     exactly in the epilogue, so that |x * x_scale| stays inside fp16's range (mn_conv_params.x_scale)."""

    __slots__ = ("w", "taps", "cin", "cout", "_tc", "name", "precision", "x_scale", "tag", "__weakref__")
    _next_tag = 1
    _by_tag = {}
    _slots = {}        # tag -> range-flag slot of the live layers that have launched on the tensor cores

    def __init__(self, w, taps, name=None):
        import weakref
        self.w = w
        self.taps = taps
        self.cin = w.shape[0] // taps
        self.cout = w.shape[1]
        self._tc = {}
        self.tag = ConvWeight._next_tag
        ConvWeight._next_tag += 1
        self.name = name or f"conv#{self.tag}[{taps}x{self.cin}->{self.cout}]"
        self.precision, self.x_scale = PLAN.get(self.name, (None, 1.0))      # plans survive re-packing (keyed by layer name)
        ConvWeight._by_tag[self.tag] = weakref.ref(self, functools.partial(ConvWeight._release, self.tag))

    @classmethod
    def _release(cls, tag, _ref=None):
        """The layer with this tag died: forget it and give its range-flag slot back."""
        cls._by_tag.pop(tag, None)
        slot = cls._slots.pop(tag, None)
        if slot is not None:
            _RANGE_POOL.give(slot)

    def range_slot(self):
        """This layer's own element of the range-flag arrays: taken at its first tensor-core launch, released when it dies."""
        slot = ConvWeight._slots.get(self.tag)
        if slot is None:
            slot = ConvWeight._slots[self.tag] = _RANGE_POOL.take()
        return slot

    def set_plan(self, precision=None, x_scale=None):
        """Set this layer's precision / input scale and remember it under the layer's name (ops.PLAN)."""
        if precision is not None:
            self.precision = int(precision)
        if x_scale is not None:
            self.x_scale = float(x_scale)
        PLAN[self.name] = (self.precision, self.x_scale)
        global PLAN_VERSION
        PLAN_VERSION += 1

    @classmethod
    def from_tag(cls, tag):
        r = cls._by_tag.get(int(tag))
        return None if r is None else r()

    @property
    def shape(self):
        return self.w.shape

    def tc_capable(self):
        return self.cin % 64 == 0 and self.cout % 64 == 0

    def tc(self, precision):
        key = PREC_BF16X3_TC if precision == PREC_BF16X3_TC else PREC_F16X3_TC
        got = self._tc.get(key)
        if got is None:
            n = self.taps * self.cin * self.cout
            hi = torch.empty(n, dtype=torch.int16, device=self.w.device)
            lo = torch.empty(n, dtype=torch.int16, device=self.w.device)
            sc = torch.empty(2, dtype=torch.float32, device=self.w.device)
            with torch.cuda.device(self.w.device):
                _lib.check(_lib.load().mn_conv_pack_weights_tc(_ptr(self.w), self.taps, self.cin, self.cout, key, _ptr(hi), _ptr(lo),
                                                               _ptr(sc), _stream()), "mn_conv_pack_weights_tc")
            got = (hi, lo, sc)
            self._tc[key] = got
        return got


# ---- fp16-range guard (ADVICE r1 / VERDICT r1 2.iii) ------------------------------------------------------------------
# The default tensor-core precision splits fp32 operands into fp16 hi/lo pairs: an activation with |x * x_scale| >= 65504 would
# become Inf.  Every tensor-core conv is launched with a pointer to its layer's own element of a per-device flag array in PINNED
# HOST memory; the operand-split stage stores the layer's tag into it when |x * x_scale| reaches 65504 (or Inf; NaN is not seen).
# The host reads the flags without any CUDA call: at the start of every module forward (``poll_range``: the offending layer is
# re-routed to the bf16 split, which has fp32's exponent range, and a warning names it) and in ``check_range`` (raises
# FloatingPointError; GraphedLines.check and pipeline.restore_lines call it after their synchronisation, the latter re-runs the
# step with the new plan).  The flag is the guarantee, not the overflowed call's own output: its dot products hold Inf/NaN, but a
# ReLU epilogue (fmaxf) turns NaN and -Inf into 0, so that output may be finite and plausible.
_RANGE_FLAGS = {}
_RANGE_SLOTS = 2048
RANGE_EVENTS = []        # (layer name, action) log of re-routes, newest last


class _SlotPool:
    """Indices [0, size) handed out one per live layer; released ones are reused first."""

    def __init__(self, size):
        self.size, self.next, self.free = size, 0, []

    def take(self):
        if not self.free and self.next == self.size:
            import gc
            gc.collect()                # dead layers still held by reference cycles give their slots back
        if self.free:
            return self.free.pop()
        if self.next == self.size:
            raise RuntimeError(f"marconet_b200: more than {self.size} live tensor-core conv layers; the fp16-range guard has one "
                               f"flag slot per layer (ops._RANGE_SLOTS)")
        self.next += 1
        return self.next - 1

    def give(self, slot):
        self.free.append(slot)


_RANGE_POOL = _SlotPool(_RANGE_SLOTS)


def range_flags(device):
    """Per-device int32[_RANGE_SLOTS] in pinned host memory; element ``cw.range_slot()`` belongs to layer ``cw`` while it lives."""
    key = device.index if device.index is not None else torch.cuda.current_device()
    f = _RANGE_FLAGS.get(key)
    if f is None:
        f = torch.zeros(_RANGE_SLOTS, dtype=torch.int32).pin_memory()
        _RANGE_FLAGS[key] = f
    return f


def poll_range(device, reroute=True):
    """Non-synchronising look at the device's range flags.  Returns the offending ConvWeights (empty list: none) and clears the
    flags; with ``reroute`` every such layer is switched to the bf16 hi/lo split for all later calls."""
    f = _RANGE_FLAGS.get(device.index if device.index is not None else torch.cuda.current_device())
    if f is None:
        return []
    arr = f.numpy()
    if not arr.any():
        return []
    tags = [int(t) for t in arr[arr != 0]]
    arr[:] = 0
    hits = []
    import warnings
    for tag in tags:
        cw = ConvWeight.from_tag(tag)
        if cw is None:
            continue
        hits.append(cw)
        if not reroute:
            continue
        if cw.precision == PREC_BF16X3_TC:      # already on the wide-range split: the input itself held Inf / NaN
            RANGE_EVENTS.append((cw.name, "non-finite input"))
            warnings.warn(f"marconet_b200: non-finite values reached conv layer {cw.name}")
        else:
            cw.set_plan(precision=PREC_BF16X3_TC)
            RANGE_EVENTS.append((cw.name, "rerouted to bf16x3"))
            warnings.warn(f"marconet_b200: |activation * {cw.x_scale:g}| >= 65504 at conv layer {cw.name}: the fp16 hi/lo split "
                          f"overflowed (that call's output is wrong: Inf/NaN, or 0 after a ReLU); the layer now uses the bf16 split (MN_PREC_BF16X3_TC). "
                          f"Run pipeline.tune_precision() for a calibrated per-layer plan.")
    return hits


def check_range(device):
    """Raise FloatingPointError when a tensor-core conv saw an operand outside its representable range since the last
    poll.  The caller must have synchronised with the work it asks about."""
    hits = poll_range(device)
    if hits:
        names = ", ".join(cw.name for cw in hits[:6]) + (" ..." if len(hits) > 6 else "")
        raise FloatingPointError(f"marconet_b200: fp16 operand range exceeded (or non-finite input) at conv layer(s) {names}; they "
                                 f"have been re-routed to the bf16 split -- re-run the step")


class calibration:
    """Context manager: every tensor-core conv launched inside records max |x * x_scale| of its input (mn_conv_params.x_absmax)
    and, with ``compare=True``, its relative max-abs error against the exact fp32 kernel for both split formats.
    ``results()`` (synchronises) -> {ConvWeight: dict(absmax=..., err_f16x3=..., err_bf16x3=..., out_absmax=...)}."""

    SLOTS = 4096

    def __init__(self, device, compare=False):
        self.device, self.compare = torch.device(device), compare
        self.buf = torch.zeros(self.SLOTS, dtype=torch.float32, device=self.device)
        self.slots, self.errs, self.prev = {}, {}, None

    def __enter__(self):
        self.prev = getattr(_TLS, "calib", None)
        _TLS.calib = self
        return self

    def __exit__(self, *exc):
        _TLS.calib = self.prev
        return False

    def slot(self, cw):
        i = self.slots.get(cw)
        if i is None:
            i = len(self.slots)
            if i >= self.SLOTS:
                raise RuntimeError("calibration: too many layers")
            self.slots[cw] = i
        return self.buf[i:i + 1]

    def results(self):
        torch.cuda.synchronize(self.device)
        host = self.buf.cpu()
        out = {}
        for cw, i in self.slots.items():
            rec = dict(absmax=float(host[i]) / cw.x_scale)
            for k, v in self.errs.get(cw, {}).items():
                rec[k] = max(float(t) for t in v)
            out[cw] = rec
        return out


TC_FALLBACKS = {}      # shape key -> (layer name, GFLOP, reason): convs that a tensor-core default ran on the fp32 CUDA-core kernel


def _note_fallback(cw, key, flop, reason):
    """A tensor-core precision was the default but this conv runs on the exact fp32 kernel (unsupported geometry: Cin/Cout not
    multiples of 64, stride != 1, tiny launch ...).  Logged ONCE per shape so that a checkpoint with different channel counts does
    not quietly run 6x slower (VERDICT r1); ``ops.TC_FALLBACKS`` keeps the list, bench.py reports it."""
    if key in TC_FALLBACKS:
        return
    name = cw.name if cw is not None else "unnamed"
    TC_FALLBACKS[key] = (name, flop / 1e9, reason)
    import logging
    logging.getLogger("marconet_b200").info("conv %s %s runs on the fp32 CUDA-core kernel: %s", name, key, reason)


TC_MIN_FLOP = 3.0e7    # tiny launches are latency-bound either way and stay on the exact fp32 path


def conv2d(x, w, kh, kw, stride=(1, 1), pad=(0, 0), bias=None, out_scale=None, residual=None,
           res_broadcast=False, act=ACT_NONE, gain=1.0, out=None, out2=None, y2_scale=None,
           valid_w=None, precision=None, want_y=True, split_k=0, gn=None, gn_fuse=True, out2_ptrs=None, gn_stats=False, plan=None):
    """mn_conv2d_nhwc.  ``w`` is the packed [KH*KW*Cin, Cout] matrix.  Returns y (or (y, y2)).
    ``plan``: a dict that receives what was launched (mn_conv2d_plan): ``kernel`` ("small" / "simt" / "tc1" / "tc2"), ``precision``,
    ``nt``, ``TN``, ``TH``, ``TW``, ``splits`` (split-K), ``gn_fused``, ``gn_stats_out`` (statistics from the epilogue), ``x_scale`` and,
    for the tensor-core kernels (0 otherwise), ``cs`` (cluster size), ``m_tiles``, ``work_items``, ``hstages`` / ``bstages`` (ring
    depths) and ``ctas`` (the grid under the current ``set_max_ctas`` cap).
    ``gn=(mean_rstd, gamma, beta)``: the conv input is swish(GroupNorm(x)); fused into the halo-tiled tensor-core kernel's operand-split
    stage when ``gn_fuse`` is true and the plan honours it (that kernel, one sample per pixel tile), otherwise applied by
    mn_groupnorm_apply first; ``gn_fuse=False`` forces the two passes.
    (Default on since the fused instantiation runs four lanes per halo row with the GroupNorm constants in registers: all eight
    normalise passes gone, 1.3 % per line on the same box; its first form -- one lane per row, per-row
    global loads of mean / rstd -- measured 8.7 vs 7.1 ms.)
    ``gn_stats=True``: also return the GroupNorm statistics (mean / rstd [N, Cout/32, 2]) of the OUTPUT, for the GroupNorm that
    follows this conv (networks.py:508-512): accumulated by the tensor-core kernel's epilogue (mn_conv_params.gn_stats_out, no read
    pass over y) when the plan honours it, by mn_groupnorm_stats otherwise.  Returns (y, mean_rstd).
    The library decides what runs (mn_conv2d_plan: asked once, and again only after a fall-back to fp32); this wrapper only picks the precision requested -- explicit, then
    the layer's plan, then the process default -- and keeps a default tensor-core request away from tiny launches (TC_MIN_FLOP) and
    from raw weights, which have no tensor-core planes."""
    global LAUNCHES
    lib = _lib.load()
    n, h, wd, cin, x_cs = nhwc_info(x, "x")
    cw = w if isinstance(w, ConvWeight) else None
    if cw is not None:
        w = cw.w
    cout = w.shape[1]
    if w.shape[0] != kh * kw * cin:
        raise RuntimeError(f"conv2d: packed weight has {w.shape[0]} rows, expected {kh * kw * cin}")
    oh = (h + 2 * pad[0] - kh) // stride[0] + 1
    ow = (wd + 2 * pad[1] - kw) // stride[1] + 1
    p = ConvParams()
    p.x = x.data_ptr(); p.N = n; p.H = h; p.W = wd; p.Cin = cin; p.x_cs = x_cs
    p.w = w.data_ptr(); p.KH = kh; p.KW = kw; p.stride_h, p.stride_w = stride; p.pad_h, p.pad_w = pad; p.Cout = cout
    y = None
    if want_y:
        y = out if out is not None else torch.empty((n, oh, ow, cout), dtype=torch.float32, device=x.device)
        yn, yh, yw, yc, y_cs = nhwc_info(y, "out")
        if (yn, yh, yw, yc) != (n, oh, ow, cout):
            raise RuntimeError(f"conv2d: out has shape {tuple(y.shape)}, expected {(n, oh, ow, cout)}")
        p.y = y.data_ptr(); p.y_cs = y_cs
    y2 = None
    if out2_ptrs is not None:
        # second output scattered through per-sample base pointers (int64 device tensor [N], possibly PEER-GPU addresses):
        # mn_conv_params.y2_ptrs; dense [OH, OW, Cout] blocks.  Nothing local is allocated for it.
        if out2 is not None or out2_ptrs.dtype != torch.int64 or not out2_ptrs.is_cuda or out2_ptrs.numel() != n or not out2_ptrs.is_contiguous():
            raise RuntimeError("conv2d: out2_ptrs must be a contiguous int64 CUDA tensor with one pointer per sample (and out2 unset)")
        p.y2 = out2_ptrs.data_ptr(); p.y2_cs = cout; p.y2_ptrs = out2_ptrs.data_ptr()
        if y2_scale is not None:
            p.y2_scale = y2_scale.data_ptr(); p.y2_scale_stride = y2_scale.stride(0)
    if out2 is not None:
        y2 = out2 if isinstance(out2, torch.Tensor) else torch.empty((n, oh, ow, cout), dtype=torch.float32, device=x.device)
        _, _, _, _, y2_cs = nhwc_info(y2, "out2")
        p.y2 = y2.data_ptr(); p.y2_cs = y2_cs
        if y2_scale is not None:
            p.y2_scale = y2_scale.data_ptr(); p.y2_scale_stride = y2_scale.stride(0)
    if bias is not None:
        p.bias = bias.data_ptr()
    if out_scale is not None:
        p.out_scale = out_scale.data_ptr(); p.out_scale_stride = out_scale.stride(0)
    if residual is not None:
        rinfo = nhwc_info(residual, "residual")
        p.residual = residual.data_ptr(); p.res_cs = rinfo[4]; p.res_broadcast_n = 1 if res_broadcast else 0
    p.act = act; p.act_gain = gain
    if valid_w is not None:
        p.valid_w = valid_w.data_ptr()
    ws = workspace(x.device)
    p.workspace = ws.data_ptr(); p.workspace_bytes = ws.numel() * 4
    p.split_k = split_k
    prec = precision if precision is not None else (cw.precision if (cw is not None and cw.precision is not None) else _DEFAULT_PRECISION)
    # the optional requests of the halo-tiled tensor-core kernel: the plan says which of them it honours
    if gn is not None and gn_fuse:
        p.gn_mean_rstd = gn[0].data_ptr(); p.gn_gamma = gn[1].data_ptr(); p.gn_beta = gn[2].data_ptr(); p.gn_swish = 1
    if gn_stats and y is not None and out2_ptrs is None:
        p.gn_stats_out = 1          # the plan reads the pointer as NULL / non-NULL only: the buffer follows once the plan accepts
    p.precision = prec
    cp = _lib.ConvPlan()
    if prec != PREC_FP32_SIMT:
        flop = 2.0 * n * oh * ow * cout * kh * kw * cin
        if cw is None:
            why = "a raw weight has no tensor-core planes (pass a ConvWeight)"
        elif precision is None and flop < TC_MIN_FLOP:
            why = f"below TC_MIN_FLOP ({flop / 1e6:.1f} MFLOP)"
        else:
            why = lib.mn_last_error().decode(errors="replace") if lib.mn_conv2d_plan(ctypes.byref(p), ctypes.byref(cp)) else None
        if why is not None:
            if precision is not None:
                raise RuntimeError("conv2d: tensor-core precision requested explicitly but this layer/shape is not supported: " + why)
            _note_fallback(cw, (n, h, wd, cin, cout, kh, kw, stride), flop, why)
            prec = p.precision = PREC_FP32_SIMT
    if prec == PREC_FP32_SIMT:
        _lib.check(lib.mn_conv2d_plan(ctypes.byref(p), ctypes.byref(cp)), "mn_conv2d_plan")
    else:
        hi, lo, sc = cw.tc(prec)
        p.w_tc_hi = hi.data_ptr(); p.w_tc_lo = lo.data_ptr(); p.w_tc_scale = sc.data_ptr()
        p.x_scale = cw.x_scale
        p.range_flag = range_flags(x.device).data_ptr() + 4 * cw.range_slot(); p.range_tag = cw.tag
        calib = getattr(_TLS, "calib", None)
        if calib is not None:
            p.x_absmax = calib.slot(cw).data_ptr()
    stats_ws = None
    if cp.gn_stats_out:
        stats_ws = torch.zeros((n * (cout // 32) * 2,), dtype=torch.float64, device=x.device)
    p.gn_stats_out = _ptr(stats_ws)
    if not cp.gn_fused:
        p.gn_mean_rstd = p.gn_gamma = p.gn_beta = None; p.gn_swish = 0
        if gn is not None:          # normalise into a temporary first
            xg = groupnorm_apply(x, gn[0], gn[1], gn[2], valid_w=valid_w)
            p.x = xg.data_ptr(); p.x_cs = xg.shape[3]
    _lib.check(lib.mn_conv2d_nhwc(ctypes.byref(p), _stream()), "mn_conv2d_nhwc")
    LAUNCHES += 1
    if plan is not None:
        plan.update(kernel=_lib.CONV_KERNELS[cp.kernel], precision=cp.precision, nt=cp.nt, TN=cp.TN, TH=cp.TH, TW=cp.TW, splits=cp.splits,
                    gn_fused=bool(cp.gn_fused), gn_stats_out=bool(cp.gn_stats_out), x_scale=p.x_scale if p.x_scale > 0 else 1.0,
                    cs=cp.cs, m_tiles=cp.m_tiles, work_items=cp.work_items, hstages=cp.hstages, bstages=cp.bstages, ctas=cp.ctas)
    calib = getattr(_TLS, "calib", None)
    if calib is not None and calib.compare and cw is not None and prec != PREC_FP32_SIMT and precision is None:
        # tuning tool only (pipeline.tune_precision): the same layer through the exact fp32 kernel and both split formats
        _TLS.calib = None
        try:
            opts = dict(stride=stride, pad=pad, bias=bias, out_scale=out_scale, residual=residual, res_broadcast=res_broadcast, act=act,
                        gain=gain, valid_w=valid_w, split_k=split_k, gn=gn)
            ref = conv2d(x, cw, kh, kw, precision=PREC_FP32_SIMT, **opts)
            scale = ref.abs().max().clamp_min(1e-30)
            rec = calib.errs.setdefault(cw, {})
            rec.setdefault("out_absmax", []).append(scale)
            for name, cand in (("err_f16x3", PREC_F16X3_TC), ("err_bf16x3", PREC_BF16X3_TC)):
                got = conv2d(x, cw, kh, kw, precision=cand, **opts)
                rec.setdefault(name, []).append(torch.nan_to_num((got - ref).abs().max() / scale, nan=float("inf")))
        finally:
            _TLS.calib = calib
    if gn_stats:
        if stats_ws is not None:
            mr = torch.empty((n, cout // 32, 2), dtype=torch.float32, device=x.device)
            _lib.check(lib.mn_groupnorm_finalize(_ptr(stats_ws), n, oh, ow, cout, 32, 1e-6, _ptr(valid_w), _ptr(mr), _stream()), "mn_groupnorm_finalize")
            LAUNCHES += 2
        else:
            mr = groupnorm_stats(y, valid_w=valid_w)
        return y, mr
    if y2 is not None:
        return (y, y2) if want_y else y2
    return y


def linear(x2d, w, bias=None, act=ACT_NONE, gain=1.0, residual=None, out=None, precision=None):
    """nn.Linear as a 1x1 conv on [M,1,1,K]; ``w`` packed [K, Cout]; x2d: [M, K] contiguous."""
    global LAUNCHES
    m, k = x2d.shape
    wt = w.w if isinstance(w, ConvWeight) else w
    nout = wt.shape[1]
    if m <= 64 and k % 32 == 0 and nout % 16 == 0 and precision is None and x2d.is_contiguous() and \
            (residual is None or residual.is_contiguous()):
        y = out if out is not None else torch.empty((m, nout), dtype=torch.float32, device=x2d.device)
        _lib.check(_lib.load().mn_linear_small_m(_ptr(x2d), _ptr(wt), _ptr(bias), _ptr(residual), _ptr(y), m, k, nout, act, gain,
                                                 _stream()), "mn_linear_small_m")
        LAUNCHES += 1
        return y
    res = None if residual is None else residual.reshape(m, 1, 1, -1)
    o = None if out is None else out.reshape(m, 1, 1, -1)
    y = conv2d(x2d.reshape(m, 1, 1, k), w, 1, 1, bias=bias, act=act, gain=gain, residual=res, out=o, precision=precision)
    return y.reshape(m, -1)


def patch_embed(feat, w, bias, pe):
    """TextViT patch embedding on the NHWC feature map in place (textvit_arch.py:33-36,68-69):
    feat [B, 8, 8*T, C] -> tokens [B*T, D] = Linear(rearrange(feat, 'b (p1) (t p2) c -> b t (p1 p2 c)')) + pe[T, D].
    ``w`` is the packed [8*8*C, D] weight (K order p1, p2, c)."""
    global LAUNCHES
    b, fh, fw, c, cs = nhwc_info(feat, "feat")
    if fh != 8 or fw % 8 != 0 or cs != c:
        raise RuntimeError("patch_embed: expects a dense [B, 8, 8*T, C] feature map")
    t = fw // 8
    k, d = w.shape
    if k != 64 * c or t > 64 or tuple(pe.shape) != (t, d):
        raise RuntimeError("patch_embed: weight / positional embedding do not match the feature map")
    y = torch.empty((b * t, d), dtype=torch.float32, device=feat.device)
    ws = workspace(feat.device)         # outer K slices (deep K, few column tiles): partial tiles + a deterministic reduce kernel
    _lib.check(_lib.load().mn_linear_small_m_ws(_ptr(feat), 8 * c, 8 * fw * c, 8 * c, fw * c, _ptr(w), _ptr(bias), _ptr(pe), 0, _ptr(y),
                                                b, t, k, d, ACT_NONE, 1.0, _ptr(ws), ws.numel() * 4, _stream()), "mn_linear_small_m_ws")
    LAUNCHES += 2
    return y


def pixelnorm(x):
    global LAUNCHES
    _require_cuda(x, "x")
    y = torch.empty_like(x)
    _lib.check(_lib.load().mn_pixelnorm(_ptr(x), _ptr(y), x.shape[0], x.shape[1], _stream()), "mn_pixelnorm")
    LAUNCHES += 1
    return y


# ---- deferred error checks (CUDA-graph capture / pipelined callers, SURVEY 8f n1) -----------------------------------
# The module API raises on a bad label or an empty character window BEFORE launching, which costs a device->host round
# trip per call.  Inside ``deferred_checks(flag)`` the same conditions are evaluated by device kernels that OR a bit into
# ``flag`` (int32[1] on the device: bit 0 = label out of range, bit 1 = empty window); the caller reads it with the results.
ERR_LABEL, ERR_WINDOW = 1, 2


class deferred_checks:
    def __init__(self, flag):
        if flag is not None and (flag.dtype != torch.int32 or not flag.is_cuda or flag.numel() != 1):
            raise RuntimeError("deferred_checks: flag must be an int32[1] CUDA tensor")
        self.flag, self.prev = flag, None

    def __enter__(self):
        self.prev = getattr(_TLS, "deferred_flag", None)
        _TLS.deferred_flag = self.flag
        return self.flag

    def __exit__(self, *exc):
        _TLS.deferred_flag = self.prev
        return False


def deferred_flag():
    return getattr(_TLS, "deferred_flag", None)


def raise_deferred(flag_value):
    """Turn a flag value read back from the device into the exception the eager path raises."""
    if flag_value & ERR_LABEL:
        raise IndexError("character label out of range (reference: empty embedding slice, networks.py:211)")
    if flag_value & ERR_WINDOW:
        raise RuntimeError("empty character window (the reference fails on the empty slice at networks.py:443)")


def check_labels(labels_dev, classes, flag):
    """labels_dev: int64 [n] on the device -> clamped copy; raises bit 0 of ``flag`` on the device when out of range."""
    global LAUNCHES
    n = labels_dev.numel()
    out = torch.empty_like(labels_dev)
    _lib.check(_lib.load().mn_check_labels(_ptr(labels_dev), _ptr(out), n, classes, _ptr(flag), _stream()), "mn_check_labels")
    LAUNCHES += 1
    return out


def char_windows(locs_dev, line_first_dev, counts, width, half, flag):
    """Device restatement of models.networks.char_windows: returns (win int32[Nc,4], valid int32[Nc], owner int32[B,W])."""
    global LAUNCHES
    _require_cuda(locs_dev, "locs")
    if locs_dev.dtype != torch.float32 or locs_dev.dim() != 2 or locs_dev.stride(1) != 1:
        raise RuntimeError("char_windows: locs must be fp32 [B, 2n] with unit inner stride")
    b, nc = len(counts), sum(counts)
    if locs_dev.shape[0] < b or (counts and locs_dev.shape[1] < 2 * max(counts)):
        raise RuntimeError("char_windows: locs has fewer entries than characters")
    dev = locs_dev.device
    win = torch.empty((nc, 4), dtype=torch.int32, device=dev)
    valid = torch.empty((nc,), dtype=torch.int32, device=dev)
    owner = torch.empty((b, width), dtype=torch.int32, device=dev)
    _lib.check(_lib.load().mn_char_windows(_ptr(locs_dev), locs_dev.stride(0), _ptr(line_first_dev), b, max(counts), width, half,
                                           _ptr(win), _ptr(valid), _ptr(owner), _ptr(flag), _stream()), "mn_char_windows")
    LAUNCHES += 1
    return win, valid, owner


def char_windows_ragged(locs_dev, line_first_dev, line_w_dev, counts, width, half, flag):
    """mn_char_windows for lines of their own widths: line b's centres and clipping use ``line_w_dev[b]`` (device int32 [B], each
    <= ``width``, the width of the owner map); owner is -1 from column line_w[b] on.  Returns (win, valid, owner) as char_windows."""
    global LAUNCHES
    _require_cuda(locs_dev, "locs")
    if locs_dev.dtype != torch.float32 or locs_dev.dim() != 2 or locs_dev.stride(1) != 1:
        raise RuntimeError("char_windows_ragged: locs must be fp32 [B, 2n] with unit inner stride")
    b, nc = len(counts), sum(counts)
    if locs_dev.shape[0] < b or (counts and locs_dev.shape[1] < 2 * max(counts)):
        raise RuntimeError("char_windows_ragged: locs has fewer entries than characters")
    if line_w_dev.dtype != torch.int32 or not line_w_dev.is_cuda or line_w_dev.numel() != b or not line_w_dev.is_contiguous():
        raise RuntimeError("char_windows_ragged: line_w must be a contiguous int32 CUDA tensor with one width per line")
    dev = locs_dev.device
    win = torch.empty((nc, 4), dtype=torch.int32, device=dev)
    valid = torch.empty((nc,), dtype=torch.int32, device=dev)
    owner = torch.empty((b, width), dtype=torch.int32, device=dev)
    _lib.check(_lib.load().mn_char_windows_ragged(_ptr(locs_dev), locs_dev.stride(0), _ptr(line_first_dev), _ptr(line_w_dev), b, max(counts),
                                                  width, half, _ptr(win), _ptr(valid), _ptr(owner), _ptr(flag), _stream()),
               "mn_char_windows_ragged")
    LAUNCHES += 1
    return win, valid, owner


def select_text(emb, labels_dev, s, n, l):
    """emb: [classes, C]; labels_dev: int64 [n*l] on device; s: [n, C] view (row stride s.stride(0)) or None."""
    global LAUNCHES
    c = emb.shape[1]
    out = torch.empty((n, 4, 4 * l, c), dtype=torch.float32, device=emb.device)
    _lib.check(_lib.load().mn_select_text(_ptr(emb), _ptr(labels_dev), _ptr(s), 0 if s is None else s.stride(0),
                                          _ptr(out), n, l, c, _stream()), "mn_select_text")
    LAUNCHES += 1
    return out


def demod(s, wsq):
    """s: [N, Cin] view; wsq: [Cin, Cout] -> [N, Cout]."""
    global LAUNCHES
    n, cin = s.shape
    cout = wsq.shape[1]
    out = torch.empty((n, cout), dtype=torch.float32, device=s.device)
    _lib.check(_lib.load().mn_demod(_ptr(s), s.stride(0), _ptr(wsq), _ptr(out), n, cin, cout, _stream()), "mn_demod")
    LAUNCHES += 1
    return out


def make_demod_table(entries, device):
    """entries: [(wsq tensor [cin,cout], s_off, out_off)] -> (device byte tensor holding mn_demod_desc[], n, max_cout, total_out)."""
    import numpy as np
    arr = (_lib.DemodDesc * len(entries))()
    mx = 0
    for i, (wsq, s_off, out_off) in enumerate(entries):
        arr[i].wsq = wsq.data_ptr(); arr[i].s_off = s_off; arr[i].cin = wsq.shape[0]; arr[i].cout = wsq.shape[1]; arr[i].out_off = out_off
        mx = max(mx, wsq.shape[1])
    raw = torch.from_numpy(np.frombuffer(bytes(arr), dtype=np.uint8).copy()).to(device)
    return raw, len(entries), mx


def demod_batched(s_all, table, out_total):
    """One launch for every styled conv's demodulation vector; returns [N, out_total]."""
    global LAUNCHES
    raw, n_layers, mx = table
    n = s_all.shape[0]
    out = torch.empty((n, out_total), dtype=torch.float32, device=s_all.device)
    _lib.check(_lib.load().mn_demod_batched(_ptr(s_all), s_all.stride(0), _ptr(raw), n_layers, mx, _ptr(out), out_total, n, _stream()),
               "mn_demod_batched")
    LAUNCHES += 1
    return out


def resample_modulate(x, s=None, up=False, out=None):
    global LAUNCHES
    n, h, w, c, x_cs = nhwc_info(x, "x")
    oh, ow = (2 * h, 2 * w) if up else (h, w)
    y = out if out is not None else torch.empty((n, oh, ow, c), dtype=torch.float32, device=x.device)
    _, _, _, _, y_cs = nhwc_info(y, "out")
    _lib.check(_lib.load().mn_resample_modulate(_ptr(x), x_cs, _ptr(y), y_cs, _ptr(s), 0 if s is None else s.stride(0),
                                                n, h, w, c, 1 if up else 0, _stream()), "mn_resample_modulate")
    LAUNCHES += 1
    return y


def resample_up2_ragged(x, valid_w, s=None, out=None):
    """Bilinear x2 of a ragged batch (mn_resample_modulate_ragged): sample n is the first ``valid_w[n]`` columns of x (device int32
    [N]); the output is zero from column 2*valid_w[n] on.  ``s``: optional per-sample channel scale [N, C] view."""
    global LAUNCHES
    n, h, w, c, x_cs = nhwc_info(x, "x")
    if valid_w.dtype != torch.int32 or not valid_w.is_cuda or valid_w.numel() != n or not valid_w.is_contiguous():
        raise RuntimeError("resample_up2_ragged: valid_w must be a contiguous int32 CUDA tensor with one width per sample")
    y = out if out is not None else torch.empty((n, 2 * h, 2 * w, c), dtype=torch.float32, device=x.device)
    yn, yh, yw, yc, y_cs = nhwc_info(y, "out")
    if (yn, yh, yw, yc) != (n, 2 * h, 2 * w, c):
        raise RuntimeError(f"resample_up2_ragged: out has shape {tuple(y.shape)}, expected {(n, 2 * h, 2 * w, c)}")
    _lib.check(_lib.load().mn_resample_modulate_ragged(_ptr(x), x_cs, _ptr(y), y_cs, _ptr(s), 0 if s is None else s.stride(0), _ptr(valid_w),
                                                       n, h, w, c, _stream()), "mn_resample_modulate_ragged")
    LAUNCHES += 1
    return y


def torgb(x, s, w, bias, skip=None):
    global LAUNCHES
    n, h, wd, c, x_cs = nhwc_info(x, "x")
    out = torch.empty((n, h, wd, 3), dtype=torch.float32, device=x.device)
    _lib.check(_lib.load().mn_torgb(_ptr(x), x_cs, _ptr(s), s.stride(0), _ptr(w), _ptr(bias), _ptr(skip), _ptr(out),
                                    n, h, wd, c, _stream()), "mn_torgb")
    LAUNCHES += 1
    return out


def groupnorm_swish(x, gamma, beta, cpg=32, eps=1e-6, swish=True, valid_w=None, out=None):
    global LAUNCHES
    n, h, w, c, x_cs = nhwc_info(x, "x")
    y = out if out is not None else torch.empty((n, h, w, c), dtype=torch.float32, device=x.device)
    _, _, _, _, y_cs = nhwc_info(y, "out")
    stats = torch.empty((n * (c // cpg) * 3,), dtype=torch.float64, device=x.device)
    _lib.check(_lib.load().mn_groupnorm_swish(_ptr(x), x_cs, _ptr(y), y_cs, _ptr(gamma), _ptr(beta), n, h, w, c, cpg,
                                              eps, 1 if swish else 0, _ptr(valid_w), _ptr(stats), _stream()),
               "mn_groupnorm_swish")
    LAUNCHES += 3
    return y


def groupnorm_stats(x, cpg=32, eps=1e-6, valid_w=None):
    """Per (sample, group) mean / rstd [N, C/cpg, 2] of an NHWC view (mn_groupnorm_stats)."""
    global LAUNCHES
    n, h, w, c, x_cs = nhwc_info(x, "x")
    g = c // cpg
    ws = torch.empty((n * g * 2,), dtype=torch.float64, device=x.device)
    mr = torch.empty((n, g, 2), dtype=torch.float32, device=x.device)
    _lib.check(_lib.load().mn_groupnorm_stats(_ptr(x), x_cs, n, h, w, c, cpg, eps, _ptr(valid_w), _ptr(ws), _ptr(mr), _stream()),
               "mn_groupnorm_stats")
    LAUNCHES += 3
    return mr


def groupnorm_apply(x, mr, gamma, beta, cpg=32, swish=True, valid_w=None, out=None):
    global LAUNCHES
    n, h, w, c, x_cs = nhwc_info(x, "x")
    y = out if out is not None else torch.empty((n, h, w, c), dtype=torch.float32, device=x.device)
    _, _, _, _, y_cs = nhwc_info(y, "out")
    _lib.check(_lib.load().mn_groupnorm_apply(_ptr(x), x_cs, _ptr(y), y_cs, _ptr(gamma), _ptr(beta), _ptr(mr), n, h, w, c, cpg,
                                              1 if swish else 0, _ptr(valid_w), _stream()), "mn_groupnorm_apply")
    LAUNCHES += 1
    return y


def adain_concat(prior, feat, win_dev, nc, wp):
    global LAUNCHES
    pn, h, pw, c, p_cs = nhwc_info(prior, "prior")
    b, fh, w, fc, f_cs = nhwc_info(feat, "feat")
    if pn != nc or pw != wp or fh != h or fc != c:
        raise RuntimeError("adain_concat: shape mismatch")
    out = torch.empty((nc, h, wp, 2 * c), dtype=torch.float32, device=feat.device)
    stats = torch.empty((nc * c * 6,), dtype=torch.float64, device=feat.device)
    _lib.check(_lib.load().mn_adain_concat(_ptr(prior), p_cs, _ptr(feat), f_cs, _ptr(win_dev), _ptr(out), nc, h, wp, w, c,
                                           _ptr(stats), _stream()), "mn_adain_concat")
    LAUNCHES += 3
    return out


def window_scatter(feat, scale, shift, owner_dev, win_dev, wp, out=None):
    global LAUNCHES
    b, h, w, c, f_cs = nhwc_info(feat, "feat")
    y = out if out is not None else torch.empty((b, h, w, c), dtype=torch.float32, device=feat.device)
    _, _, _, _, y_cs = nhwc_info(y, "out")
    _lib.check(_lib.load().mn_window_scatter(_ptr(feat), f_cs, _ptr(scale), _ptr(shift), _ptr(owner_dev), _ptr(win_dev),
                                             _ptr(y), y_cs, b, h, w, wp, c, _stream()), "mn_window_scatter")
    LAUNCHES += 1
    return y


def swish(x):
    """x * sigmoid(x) on a CUDA tensor of any shape (reference networks.py:492-493)."""
    global LAUNCHES
    _require_cuda(x, "x")
    x = x.contiguous()
    y = torch.empty_like(x)
    _lib.check(_lib.load().mn_swish(_ptr(x), _ptr(y), x.numel(), _stream()), "mn_swish")
    LAUNCHES += 1
    return y


def calc_mean_std_4d(feat, eps=1e-5):
    """reference networks.py:518-525 on an NCHW CUDA tensor -> (mean [B,C,1,1], std [B,C,1,1]) (unbiased variance + eps)."""
    global LAUNCHES
    _require_cuda(feat, "feat")
    if feat.dim() != 4:
        raise AssertionError("The input feature should be 4D tensor.")
    b, c, h, w = feat.shape
    x = feat.contiguous()
    mean = torch.empty((b, c, 1, 1), dtype=torch.float32, device=feat.device)
    std = torch.empty((b, c, 1, 1), dtype=torch.float32, device=feat.device)
    _lib.check(_lib.load().mn_row_mean_std(_ptr(x), _ptr(mean), _ptr(std), b * c, h * w, eps, _stream()), "mn_row_mean_std")
    LAUNCHES += 1
    return mean, std


def adaptive_instance_normalization(prior_feat, lq_feat):
    """reference networks.py:528-533 on NCHW CUDA tensors with equal [B, C]."""
    global LAUNCHES
    lm, ls = calc_mean_std_4d(lq_feat)
    pm, ps = calc_mean_std_4d(prior_feat)
    if lm.shape != pm.shape:
        raise RuntimeError("adaptive_instance_normalization: prior and lq features disagree on [B, C]")
    b, c, h, w = prior_feat.shape
    x = prior_feat.contiguous()
    out = torch.empty_like(x)
    _lib.check(_lib.load().mn_adain_rows(_ptr(x), _ptr(pm), _ptr(ps), _ptr(lm), _ptr(ls), _ptr(out), b * c, h * w, _stream()), "mn_adain_rows")
    LAUNCHES += 1
    return out


def layernorm(x2d, gamma, beta, eps=1e-5):
    global LAUNCHES
    _require_cuda(x2d, "x")
    rows, dim = x2d.shape
    y = torch.empty_like(x2d)
    _lib.check(_lib.load().mn_layernorm(_ptr(x2d), _ptr(y), _ptr(gamma), _ptr(beta), rows, dim, eps, _stream()), "mn_layernorm")
    LAUNCHES += 1
    return y


def token_mix(x, gamma, beta, w, bias, eps=1e-5):
    """x: [B,T,D] contiguous -> [B,To,D]."""
    global LAUNCHES
    b, t, d = x.shape
    to = w.shape[0]
    out = torch.empty((b, to, d), dtype=torch.float32, device=x.device)
    _lib.check(_lib.load().mn_token_mix(_ptr(x), _ptr(gamma), _ptr(beta), _ptr(w), _ptr(bias), _ptr(out), b, t, to, d, eps,
                                        _stream()), "mn_token_mix")
    LAUNCHES += 1
    return out


def attention(qkv, heads=8, dh=64):
    """qkv: [B,S,3*heads*dh] contiguous -> [B,S,heads*dh]."""
    global LAUNCHES
    b, s, _ = qkv.shape
    out = torch.empty((b, s, heads * dh), dtype=torch.float32, device=qkv.device)
    _lib.check(_lib.load().mn_attention(_ptr(qkv), _ptr(out), b, s, heads, dh, dh ** -0.5, _stream()), "mn_attention")
    LAUNCHES += 1
    return out


def nchw_to_nhwc(x, out=None):
    global LAUNCHES
    _require_cuda(x, "x")
    n, c, h, w = x.shape
    x = x.contiguous()
    y = out if out is not None else torch.empty((n, h, w, c), dtype=torch.float32, device=x.device)
    _, _, _, _, y_cs = nhwc_info(y, "out")
    _lib.check(_lib.load().mn_nchw_to_nhwc(_ptr(x), _ptr(y), n, c, h, w, y_cs, _stream()), "mn_nchw_to_nhwc")
    LAUNCHES += 1
    return y


def nhwc_to_nchw(x):
    global LAUNCHES
    n, h, w, c, x_cs = nhwc_info(x, "x")
    y = torch.empty((n, c, h, w), dtype=torch.float32, device=x.device)
    _lib.check(_lib.load().mn_nhwc_to_nchw(_ptr(x), x_cs, _ptr(y), n, c, h, w, _stream()), "mn_nhwc_to_nchw")
    LAUNCHES += 1
    return y


def as_nhwc(x_nchw):
    """NCHW-shaped tensor -> NHWC view, zero-copy when the input is channels_last."""
    n, c, h, w = x_nchw.shape
    v = x_nchw.permute(0, 2, 3, 1)
    if v.is_contiguous():
        return v
    return nchw_to_nhwc(x_nchw)


def as_nchw_view(x_nhwc):
    """NHWC tensor -> NCHW-shaped view (channels_last strides); what the modules return."""
    return x_nhwc.permute(0, 3, 1, 2)


# ---- script pre/post-processing on the device (SURVEY 8f n2) ---------------------------------------------------------
def round_half_even(v):
    """cv::saturate_cast<int>(double) = cvRound: round half to even (how cv::resize derives dsize from fx, fy)."""
    return int(round(v))          # Python's round() is round-half-even on floats


def preprocess_lq(img_u8, out_h=32, out_w=512, return_resized=False):
    """test_sr.py:98-111 on the device.  img_u8: uint8 [h, w, 3] CUDA tensor (the BGR image the script reads) ->
    (lq fp32 [1, 3, out_h, out_w], resized width).  Bit-identical to OpenCV's own INTER_CUBIC + ToTensor + Normalize."""
    global LAUNCHES
    if not isinstance(img_u8, torch.Tensor) or not img_u8.is_cuda:
        raise RuntimeError("marconet_b200: img must be a CUDA tensor (there is no CPU path)")
    if img_u8.dtype != torch.uint8 or img_u8.dim() != 3 or not img_u8.is_contiguous():
        raise RuntimeError("preprocess_lq: expects a contiguous uint8 [h, w, c] image")
    h, w, cn = img_u8.shape
    fx = fy = out_h / h                                   # Python float division, like the script's fx=32/h
    dh, dw = round_half_even(h * fy), round_half_even(w * fx)
    if dw > out_w:
        raise ValueError(f"LQ width {dw} exceeds {out_w}: crop the line into shorter segments (test_sr.py:107-109)")
    lq = torch.empty((1, cn, out_h, out_w), dtype=torch.float32, device=img_u8.device)
    small = torch.empty((dh, dw, cn), dtype=torch.uint8, device=img_u8.device) if return_resized else None
    _lib.check(_lib.load().mn_preprocess_lq_u8(_ptr(img_u8), h, w, cn, fx, fy, dh, dw, _ptr(lq), _ptr(small), out_h, out_w, _stream()),
               "mn_preprocess_lq_u8")
    LAUNCHES += 1
    return (lq, dw, small) if return_resized else (lq, dw)


def postprocess_sr(sr):
    """test_sr.py:198-201 (+ cv2.imwrite's rounding): fp32 [B, C, H, W] (any strides) -> uint8 [B, H, W, C], channels flipped."""
    global LAUNCHES
    _require_cuda(sr, "sr")
    if sr.dtype != torch.float32 or sr.dim() != 4:
        raise RuntimeError("postprocess_sr: expects an fp32 [B, C, H, W] tensor")
    b, c, h, w = sr.shape
    out = torch.empty((b, h, w, c), dtype=torch.uint8, device=sr.device)
    sn, sc, sh, sw = sr.stride()
    _lib.check(_lib.load().mn_postprocess_sr_u8(_ptr(sr), sn, sc, sh, sw, _ptr(out), b, c, h, w, _stream()), "mn_postprocess_sr_u8")
    LAUNCHES += 1
    return out


class _Pack:
    """The one uint8 device buffer of a batched call, which the kernels read their records and tables from.  ``area`` places
    its areas in order, each at the next multiple of its alignment; ``alloc`` allocates it, its length a multiple of the
    largest alignment (as a C struct's), and returns its address, to which the records' pointers add the areas' offsets;
    ``upload`` copies the host bytes of the areas that have them in one host-to-device copy."""

    def __init__(self):
        self.end, self.align = 0, 1

    def area(self, nbytes, align=1):
        """The offset of ``nbytes`` new bytes at the next multiple of ``align``."""
        o = -(-self.end // align) * align
        self.end, self.align = o + nbytes, max(self.align, align)
        return o

    def alloc(self, device):
        self.buf = torch.empty(-(-self.end // self.align) * self.align, dtype=torch.uint8, device=device)
        return self.buf.data_ptr()

    def upload(self, *areas):
        """Copies (offset, bytes) areas, in increasing order, as the one range from the first area to the end of the last, with
        zeros between them.  Returns the buffer."""
        lo = areas[0][0]
        host = bytearray(areas[-1][0] + len(areas[-1][1]) - lo)
        for o, b in areas:
            host[o - lo:o - lo + len(b)] = b
        self.buf[lo:lo + len(host)].copy_(torch.frombuffer(host, dtype=torch.uint8))
        return self.buf

    @classmethod
    def of(cls, ctype, recs, device):
        """The buffer of one table of C records (which point outside it), allocated and uploaded."""
        pack = cls()
        pack.area(len(recs) * ctypes.sizeof(ctype))
        pack.alloc(device)
        return pack.upload((0, bytes((ctype * len(recs))(*recs))))


def _check_items(items, what, noun, field=0):
    """The device of a batched call's items, that of field ``field`` of the first one, after checking their number (one launch
    holds 1 to 65535)."""
    if not items:
        raise ValueError(f"{what}: no {noun}s")
    if len(items) > 65535:
        raise ValueError(f"{what}: at most 65535 {noun}s per launch")
    return items[0][field].device


def _check_channels(items, what):
    """The channel count cn of a batched image call, that of its first source (3 unless that is a 3-D tensor), 1 to 4."""
    src = items[0][0]
    cn = src.shape[2] if isinstance(src, torch.Tensor) and src.dim() == 3 else 3
    if not 1 <= cn <= 4:
        raise RuntimeError(f"{what}: {cn} channels (1 to 4)")
    return cn


def preprocess_lq_crops(crops, out_h=32, out_w=512):
    """test_sr.py:98-111 for many crops in one launch (mn_preprocess_lq_u8_batched).  crops: list of (img, x0, x1), img a uint8
    [h, w, cn] CUDA tensor with dense pixels (stride(1) == cn, stride(2) == 1, any row stride) read in place, [x0, x1) the crop's
    source columns.  Each crop is resized as an image of its own (its border is replicated): crop i of the result is
    bit-identical to ``preprocess_lq(img[:, x0:x1].contiguous())``.  Returns (lq fp32 [n, cn, out_h, out_w], resized widths)."""
    global LAUNCHES
    if not crops:
        raise ValueError("preprocess_lq_crops: no crops")
    cn = None
    recs, widths = [], []
    for i, (img, x0, x1) in enumerate(crops):
        if not isinstance(img, torch.Tensor) or not img.is_cuda:
            raise RuntimeError("marconet_b200: img must be a CUDA tensor (there is no CPU path)")
        if img.device.index != torch.cuda.current_device():
            raise RuntimeError(f"preprocess_lq_crops: crop {i} lives on {img.device}, the current device is cuda:{torch.cuda.current_device()}")
        if img.dtype != torch.uint8 or img.dim() != 3 or img.stride(2) != 1 or img.stride(1) != img.shape[2] or img.stride(0) < img.shape[1] * img.shape[2]:
            raise RuntimeError(f"preprocess_lq_crops: crop {i}: expects a uint8 [h, w, c] image with dense pixels")
        h, w, c = img.shape
        if cn is None:
            cn = c
        if c != cn or not 1 <= c <= 4:
            raise RuntimeError(f"preprocess_lq_crops: crop {i} has {c} channels, expected {cn} (1 to 4)")
        x0, x1 = int(x0), int(x1)
        if not 0 <= x0 < x1 <= w:
            raise ValueError(f"preprocess_lq_crops: crop {i}: columns [{x0}, {x1}) are not a non-empty range of the {w}-wide image")
        fx = fy = out_h / h
        dh, dw = round_half_even(h * fy), round_half_even((x1 - x0) * fx)
        if dw > out_w or dh > out_h or dw < 1 or dh < 1:
            raise ValueError(f"crop {i}: LQ size {dh}x{dw} does not fit the {out_h}x{out_w} canvas: crop the line into shorter segments "
                             f"(test_sr.py:107-109)")
        recs.append(_lib.LqCrop(img.data_ptr() + x0 * cn, img.stride(0), h, x1 - x0, cn, fx, fy, dh, dw))
        widths.append(dw)
    dev = crops[0][0].device
    table = _Pack.of(_lib.LqCrop, recs, dev)
    lq = torch.empty((len(recs), cn, out_h, out_w), dtype=torch.float32, device=dev)
    _lib.check(_lib.load().mn_preprocess_lq_u8_batched(_ptr(table), len(recs), cn, _ptr(lq), out_h, out_w, _stream()),
               "mn_preprocess_lq_u8_batched")
    LAUNCHES += 1
    return lq, widths


def postprocess_sr_pieces(sr, pieces):
    """test_sr.py:198-201 for column ranges of several SR lines into several images, one launch (mn_postprocess_sr_u8_pieces).
    sr: fp32 [B, C, H, W] (any strides: the channels_last view TSPSRNet returns is read in place).  pieces: list of
    (line, src_x0, dst), dst a uint8 CUDA view [H, width, C] with dense pixels (typically ``out[:, x0:x0 + width]`` of an image):
    dst receives columns [src_x0, src_x0 + width) of line ``line`` as ``postprocess_sr`` bytes."""
    global LAUNCHES
    _require_cuda(sr, "sr")
    if sr.dim() != 4:
        raise RuntimeError("postprocess_sr_pieces: expects an fp32 [B, C, H, W] tensor")
    if not pieces:
        raise ValueError("postprocess_sr_pieces: no pieces")
    b, c, h, w = sr.shape
    recs, mx = [], 0
    for i, (line, x0, dst) in enumerate(pieces):
        line, x0 = int(line), int(x0)
        if not isinstance(dst, torch.Tensor) or dst.device != sr.device or dst.dtype != torch.uint8 or dst.dim() != 3:
            raise RuntimeError(f"postprocess_sr_pieces: piece {i}: dst must be a uint8 [H, width, C] tensor on {sr.device}")
        if dst.shape[0] != h or dst.shape[2] != c or dst.stride(2) != 1 or dst.stride(1) != c or dst.shape[1] < 1:
            raise RuntimeError(f"postprocess_sr_pieces: piece {i}: dst {tuple(dst.shape)} (strides {dst.stride()}) is not a dense "
                               f"[{h}, width, {c}] view")
        width = dst.shape[1]
        if not (0 <= line < b and 0 <= x0 and x0 + width <= w):
            raise ValueError(f"postprocess_sr_pieces: piece {i}: line {line}, columns [{x0}, {x0 + width}) outside the [{b}, {w}] SR output")
        recs.append(_lib.SrPiece(line, x0, width, dst.data_ptr(), dst.stride(0)))
        mx = max(mx, width)
    table = _Pack.of(_lib.SrPiece, recs, sr.device)
    sn, sc, sh, sw = sr.stride()
    _lib.check(_lib.load().mn_postprocess_sr_u8_pieces(_ptr(sr), sn, sc, sh, sw, c, h, w, _ptr(table), len(recs), mx, _stream()),
               "mn_postprocess_sr_u8_pieces")
    LAUNCHES += 1


def figure_panels(items):
    """Panels 1, 2 and 4 of test_sr.py's figure (:206-231) for many images in one launch (mn_figure_u8; DESIGN.md section 7b).
    items: list of (img, fig, top, bottom, priors):
      img     uint8 [h, w, 3] CUDA tensor with dense pixels (any row stride), read in place;
      fig     uint8 [512, W, 3] CUDA view with dense pixels, W <= S = round_half_even(w*128/h); rows 0-255 and 384-511 are
              written, rows 256-383 (the SR panel) are not;
      top, bottom  the ShowLocs marker column ranges [start, stop) of rows 0-63 and 64-127 (pipeline.figure_markers);
      priors  non-empty list of fp32 [3, 128, 128] CUDA views (any strides), the characters' generator images in label order."""
    import numpy as np
    global LAUNCHES
    dev = _check_items(items, "figure_panels", "image", 1)
    psz = ctypes.sizeof(_lib.FigurePrior)
    pack = _Pack()
    pack.area(len(items) * ctypes.sizeof(_lib.FigureImage))
    p_off = pack.area(sum(len(it[4]) for it in items) * psz)
    m_off = pack.area(8 * max(1, sum(len(it[2]) + len(it[3]) for it in items)))
    base = pack.alloc(dev)
    recs, prs, marks, mx = [], [], [], 0
    for i, (img, fig, top, bot, priors) in enumerate(items):
        _dense_u8(img, dev, 3, f"figure_panels: image {i}: img")
        _dense_u8(fig, dev, 3, f"figure_panels: image {i}: fig")
        h, w = img.shape[:2]
        S = round_half_even(w * (128 / h))
        W = fig.shape[1]
        if fig.shape[0] != 512 or not 1 <= W <= S or round_half_even(h * (128 / h)) != 128:
            raise ValueError(f"figure_panels: image {i}: figure {tuple(fig.shape)} is not [512, W, 3] with 1 <= W <= S = {S}")
        if not priors:
            raise ValueError(f"figure_panels: image {i}: no prior images")
        for a, b in list(top) + list(bot):
            if not 0 <= int(a) < int(b) <= S:
                raise ValueError(f"figure_panels: image {i}: marker columns [{a}, {b}) are not a non-empty range of [0, {S}]")
        recs.append(_lib.FigureImage(img.data_ptr(), img.stride(0), fig.data_ptr(), fig.stride(0), base + m_off + 8 * len(marks),
                                     base + p_off + psz * len(prs), h, w, S, W, len(top), len(bot), len(priors)))
        marks += [(int(a), int(b)) for a, b in list(top) + list(bot)]
        for k, p in enumerate(priors):
            if not isinstance(p, torch.Tensor) or p.device != dev or p.dtype != torch.float32 or tuple(p.shape) != (3, 128, 128):
                raise RuntimeError(f"figure_panels: image {i}, character {k}: prior must be an fp32 [3, 128, 128] tensor on {dev}")
            prs.append(_lib.FigurePrior(p.data_ptr(), *p.stride()))
        mx = max(mx, W)
    buf = pack.upload((0, bytes((_lib.FigureImage * len(recs))(*recs))), (p_off, bytes((_lib.FigurePrior * len(prs))(*prs))),
                      (m_off, np.asarray(marks or [(0, 0)], dtype=np.int32).tobytes()))
    _lib.check(_lib.load().mn_figure_u8(_ptr(buf), len(recs), mx, _stream()), "mn_figure_u8")
    LAUNCHES += 1


# ---- characters predicted by the encoder on detection windows (DESIGN.md 7b, "Predicted characters") -----------------
PRED_SLOTS = _lib.PRED_SLOTS


def pred_dtype():
    """numpy view of an mn_char_pred record (the output of mn_decode_predictions)."""
    import numpy as np
    return np.dtype([("x1", "<f8", PRED_SLOTS), ("x2", "<f8", PRED_SLOTS), ("label", "<i4", PRED_SLOTS), ("n_kept", "<i4"),
                     ("n_decoded", "<i4")])


def prediction_table(windows, device, out=None):
    """windows: one (a, scale, lo, hi) per encoder row -- the window's first source column, source columns per unit of canvas
    width (16*h), its core [lo, hi) -> (rows, out): the device table of mn_pred_row records and the device buffer of
    mn_char_pred records they point to (row r writes record r; read it back as ``pred_dtype()``).  ``out``: a uint8 CUDA buffer
    (8-byte aligned) to hold the records instead of a new one."""
    if not windows:
        raise ValueError("prediction_table: no rows")
    isz = ctypes.sizeof(_lib.CharPred)
    if out is None:
        out = torch.empty(len(windows) * isz, dtype=torch.uint8, device=device)
    elif out.dtype != torch.uint8 or out.device != torch.device(device) or out.numel() < len(windows) * isz or out.data_ptr() % 8:
        raise ValueError(f"prediction_table: out must be an 8-byte aligned uint8 buffer of >= {len(windows) * isz} bytes on {device}")
    recs = [_lib.PredRow(float(a), float(s), float(lo), float(hi), out.data_ptr() + r * isz) for r, (a, s, lo, hi) in enumerate(windows)]
    return _Pack.of(_lib.PredRow, recs, device), out


def decode_predictions(logits, locs_lr, rows, first=0, n_alphabet=6735):
    """mn_decode_predictions, one launch: encoder row b of logits (fp32 [B, T, 6736], T <= 64) and locs_lr (fp32 [B, 32], the
    (left, right) pairs) -> argmax, CTC collapse, the first 16 characters' boxes in source columns and the core test, into the
    record that entry first + b of ``rows`` (prediction_table) points to.  Both tensors are read in place."""
    global LAUNCHES
    _require_cuda(logits, "logits")
    _require_cuda(locs_lr, "locs_lr")
    if logits.dtype != torch.float32 or logits.dim() != 3 or logits.stride(2) != 1 or logits.stride(1) != logits.shape[2]:
        raise RuntimeError("decode_predictions: logits must be fp32 [B, T, C] with dense rows")
    b, t, c = logits.shape
    if locs_lr.dtype != torch.float32 or locs_lr.dim() != 2 or locs_lr.shape[0] != b or locs_lr.shape[1] < 2 * PRED_SLOTS \
            or locs_lr.stride(1) != 1:
        raise RuntimeError(f"decode_predictions: locs_lr must be fp32 [{b}, >= {2 * PRED_SLOTS}] with dense rows")
    if not isinstance(rows, torch.Tensor) or rows.device != logits.device or rows.dtype != torch.uint8 \
            or not 0 <= first or (first + b) * ctypes.sizeof(_lib.PredRow) > rows.numel():
        raise ValueError(f"decode_predictions: rows [{first}, {first + b}) are not in the table")
    _lib.check(_lib.load().mn_decode_predictions(_ptr(logits), logits.stride(0), t, c, _ptr(locs_lr), locs_lr.stride(0),
                                                 rows.data_ptr() + first * ctypes.sizeof(_lib.PredRow), b, n_alphabet, _stream()),
               "mn_decode_predictions")
    LAUNCHES += 1


# ---- font-style interpolation (test_w.py:95-114; DESIGN.md 7b, "Font-style interpolation") ------------------------------
LABEL_SLOTS = _lib.LABEL_SLOTS


def label_dtype():
    """numpy view of an mn_label_row record (the output of mn_decode_labels)."""
    import numpy as np
    return np.dtype([("n", "<i4"), ("label", "<i4", LABEL_SLOTS)])


def decode_labels(logits, out, first=0, n_alphabet=6735):
    """mn_decode_labels, one launch: every character of encoder row b of logits (fp32 [B, T, 6736], T <= 64, read in place) --
    the argmax and CTC collapse of decode_predictions over all T timesteps (test_w.py:34-40) -- into record first + b of ``out``
    (a uint8 CUDA buffer of mn_label_row records; read it back as ``label_dtype()``)."""
    global LAUNCHES
    _require_cuda(logits, "logits")
    if logits.dim() != 3 or logits.stride(2) != 1 or logits.stride(1) != logits.shape[2]:
        raise RuntimeError("decode_labels: logits must be fp32 [B, T, C] with dense rows")
    b, t, c = logits.shape
    isz = ctypes.sizeof(_lib.LabelRow)
    if not isinstance(out, torch.Tensor) or out.device != logits.device or out.dtype != torch.uint8 or out.data_ptr() % 4 \
            or not 0 <= first or (first + b) * isz > out.numel():
        raise ValueError(f"decode_labels: records [{first}, {first + b}) are not in the output buffer")
    _lib.check(_lib.load().mn_decode_labels(_ptr(logits), logits.stride(0), t, c, out.data_ptr() + first * isz, b, n_alphabet,
                                            _stream()), "mn_decode_labels")
    LAUNCHES += 1


def lerp_rows(rows, n_w):
    """rows: (w1, w2, scale) per style row, w1 / w2 row indices of a style table with n_w rows and scale a finite Python number ->
    bytes of mn_lerp_row records with s = float32(scale), t = float32(1 - scale) (1 - scale computed in double, as test_w.py's
    ``1 - scale``)."""
    import math
    recs = []
    for r, (w1, w2, scale) in enumerate(rows):
        w1, w2, scale = int(w1), int(w2), float(scale)
        if not (0 <= w1 < n_w and 0 <= w2 < n_w) or not math.isfinite(scale):
            raise ValueError(f"lerp_rows: row {r}: styles ({w1}, {w2}) of {n_w}, scale {scale}")
        recs.append(_lib.LerpRow(w1, w2, scale, 1.0 - scale))
    return bytes((_lib.LerpRow * len(recs))(*recs))


def style_lerp(w, rows, n_rows):
    """mn_style_lerp, one launch: w fp32 [n_w, dim] (unit inner stride), rows a uint8 CUDA tensor holding n_rows mn_lerp_row
    records (lerp_rows) -> fp32 [n_rows, dim], row r = w[w1]*s + w[w2]*t with every operation rounded on its own."""
    global LAUNCHES
    _require_cuda(w, "w")
    if w.dim() != 2 or w.stride(1) != 1:
        raise RuntimeError("style_lerp: w must be fp32 [n, dim] with unit inner stride")
    if not isinstance(rows, torch.Tensor) or rows.device != w.device or rows.dtype != torch.uint8 or rows.data_ptr() % 4 \
            or n_rows < 1 or n_rows * ctypes.sizeof(_lib.LerpRow) > rows.numel():
        raise ValueError(f"style_lerp: the table does not hold {n_rows} rows")
    out = torch.empty((n_rows, w.shape[1]), dtype=torch.float32, device=w.device)
    _lib.check(_lib.load().mn_style_lerp(_ptr(w), w.stride(0), _ptr(rows), n_rows, w.shape[1], _ptr(out), out.stride(0), _stream()),
               "mn_style_lerp")
    LAUNCHES += 1
    return out


def prior_tile_rows(tiles):
    """tiles: (strip, c) per generator image, strip a contiguous uint8 CUDA [128, 128 n, 3] view (one style's strip) and c < n
    the character's column -> bytes of mn_prior_tile records pointing at strip[:, 128 c:128 c + 128]."""
    recs = []
    for r, (strip, c) in enumerate(tiles):
        c = int(c)
        if not isinstance(strip, torch.Tensor) or not strip.is_cuda or strip.dtype != torch.uint8 or strip.dim() != 3 \
                or strip.shape[0] != 128 or strip.shape[2] != 3 or strip.shape[1] % 128 or not strip.is_contiguous():
            raise RuntimeError(f"prior_tile_rows: row {r}: the strip must be a contiguous uint8 [128, 128 n, 3] CUDA tensor")
        if not 0 <= c < strip.shape[1] // 128:
            raise ValueError(f"prior_tile_rows: row {r}: character {c} outside the {strip.shape[1] // 128}-character strip")
        recs.append(_lib.PriorTile(strip.data_ptr() + 384 * c, strip.stride(0)))
    return bytes((_lib.PriorTile * len(recs))(*recs))


def prior_tiles(priors, tiles, first=0):
    """mn_prior_tiles_u8, one launch: generator image n of priors (fp32 [N, 3, 128, 128], any strides: the channels_last
    output is read in place) -> 8-bit tile at record first + n of ``tiles`` (a uint8 CUDA tensor of prior_tile_rows records),
    the bytes cv2.imwrite stores for prior*0.5 + 0.5 times 255 (test_w.py:109-114)."""
    global LAUNCHES
    _require_cuda(priors, "priors")
    if priors.dim() != 4 or tuple(priors.shape[1:]) != (3, 128, 128):
        raise RuntimeError("prior_tiles: priors must be fp32 [N, 3, 128, 128]")
    n = priors.shape[0]
    isz = ctypes.sizeof(_lib.PriorTile)
    if not isinstance(tiles, torch.Tensor) or tiles.device != priors.device or tiles.dtype != torch.uint8 or tiles.data_ptr() % 8 \
            or not 0 <= first or (first + n) * isz > tiles.numel() or not 1 <= n <= 65535:
        raise ValueError(f"prior_tiles: records [{first}, {first + n}) are not in the table (at most 65535 per launch)")
    _lib.check(_lib.load().mn_prior_tiles_u8(_ptr(priors), *priors.stride(), tiles.data_ptr() + first * isz, n, _stream()),
               "mn_prior_tiles_u8")
    LAUNCHES += 1


# ---- text regions in whole images (DESIGN.md 7b, "Text regions in whole images") -----------------------------------------
def _dense_u8(t, dev, cn, what):
    """Checks a uint8 [h, w, cn] CUDA view with dense pixels (any row stride) on ``dev``."""
    if not isinstance(t, torch.Tensor) or t.device != dev or t.dtype != torch.uint8 or t.dim() != 3 or t.shape[2] != cn \
            or t.shape[0] < 1 or t.shape[1] < 1 or t.stride(2) != 1 or t.stride(1) != cn or t.stride(0) < cn * t.shape[1]:
        raise RuntimeError(f"{what} must be a non-empty uint8 [h, w, {cn}] tensor with dense pixels on {dev}")


def resize_cubic(items):
    """cv2.resize(src, (dw, dh), interpolation=INTER_CUBIC) -- OpenCV's own 8-bit path, as preprocess_lq -- for many images in one
    launch (mn_resize_cubic_u8_batched).  items: list of (src, dst), uint8 [h, w, cn] and [dh, dw, cn] CUDA views with dense
    pixels (any row stride; dst may exceed 2^31 bytes).  The scales are the dsize form's 1/((double)dw/w) and 1/((double)dh/h);
    for dw = s*w, dh = s*h they equal 1/s, so dst is also cv2.resize(src, (0, 0), fx=s, fy=s, interpolation=INTER_CUBIC)."""
    global LAUNCHES
    dev = _check_items(items, "resize_cubic", "image")
    cn = _check_channels(items, "resize_cubic")
    recs, mx = [], 0
    for i, (src, dst) in enumerate(items):
        _dense_u8(src, dev, cn, f"resize_cubic: image {i}: src")
        _dense_u8(dst, dev, cn, f"resize_cubic: image {i}: dst")
        (h, w), (dh, dw) = src.shape[:2], dst.shape[:2]
        recs.append(_lib.ResizeImage(src.data_ptr(), src.stride(0), h, w, dst.data_ptr(), dst.stride(0), dh, dw,
                                     1.0 / (dw / w), 1.0 / (dh / h)))
        mx = max(mx, dh * dw)
    table = _Pack.of(_lib.ResizeImage, recs, dev)
    _lib.check(_lib.load().mn_resize_cubic_u8_batched(_ptr(table), len(recs), cn, mx, _stream()), "mn_resize_cubic_u8_batched")
    LAUNCHES += 1


def _region_records(regions, feather, what, record, tables=None):
    """Validated mn_region records of composite_regions' (page, sr, rect, chain, ...) tuples, the largest rectangle's pixel
    count, the call's allocated buffer, the (offset, bytes) of the chains in it and the offset of its ``tables`` bytes of curve
    tables (None without them).  The buffer holds the ``record``-type table, the chains, then the 8-byte aligned tables."""
    import numpy as np
    dev = _check_items(regions, what, "region")
    if feather < 0:
        raise ValueError(f"{what}: feather {feather} < 0")
    pack = _Pack()
    pack.area(len(regions) * ctypes.sizeof(record))
    c_off = pack.area(4 * max(1, sum(len(r[3]) for r in regions)))
    t_off = None if tables is None else pack.area(tables, 8)
    c_base = pack.alloc(dev) + c_off
    recs, chains, mx = [], [], 0
    for i, (page, sr, rect, chain) in enumerate(r[:4] for r in regions):
        _dense_u8(page, dev, 3, f"{what}: region {i}: page")
        _dense_u8(sr, dev, 3, f"{what}: region {i}: sr")
        x0, y0, x1, y1 = (int(v) for v in rect)
        ph, pw = page.shape[:2]
        if not (0 <= x0 < x1 <= pw and 0 <= y0 < y1 <= ph):
            raise ValueError(f"{what}: region {i}: rectangle {(x0, y0, x1, y1)} is not a non-empty part of the {ph}x{pw} page")
        chain = [int(j) for j in chain]
        if i not in chain or any(b <= a for a, b in zip(chain, chain[1:])) or not 0 <= chain[0] or chain[-1] >= len(regions) \
                or any(regions[j][0].data_ptr() != page.data_ptr() for j in chain):
            raise ValueError(f"{what}: region {i}: chain {chain} is not an increasing list of regions of its page "
                             f"that holds the region itself")
        recs.append(_lib.Region(page.data_ptr(), page.stride(0), sr.data_ptr(), sr.stride(0), c_base + 4 * len(chains), ph, pw,
                                sr.shape[0], sr.shape[1], x0, y0, x1, y1, feather, len(chain)))
        chains += chain
        mx = max(mx, (x1 - x0) * (y1 - y0))
    return recs, mx, pack, (c_off, np.asarray(chains or [0], dtype=np.int32).tobytes()), t_off


def composite_regions(regions, feather):
    """Restored regions composed over their pages in one launch (mn_composite_regions_u8; DESIGN.md 7b).  regions: list of
    (page, sr, rect, chain):
      page   uint8 [H, W, 3] CUDA view with dense pixels holding the background (written in place);
      sr     uint8 [h, w, 3] CUDA view with dense pixels: the region's restored bytes in cv2.imwrite order, read in place;
      rect   (x0, y0, x1, y1), the region's rectangle in page pixels, non-empty and inside the page;
      chain  indices into ``regions`` of every region of the same page whose rectangle meets this one, itself included, increasing.
    ``feather`` >= 0: the ramp width F in page pixels.  Inside its rectangle each region's cubic resize P of sr (channels flipped
    back) is blended over the page with weight a = min(1, fl((float)d + 0.5)/F), d the distance to the nearest side not on the
    page border; regions later in the list compose over earlier ones, and each pixel is written once."""
    global LAUNCHES
    recs, mx, pack, chains, _ = _region_records(regions, int(feather), "composite_regions", _lib.Region)
    buf = pack.upload((0, bytes((_lib.Region * len(recs))(*recs))), chains)
    _lib.check(_lib.load().mn_composite_regions_u8(_ptr(buf), len(recs), mx, _stream()), "mn_composite_regions_u8")
    LAUNCHES += 1


def warp_affine(items):
    """cv2.warpAffine(src, M, (dw, dh), flags=INTER_CUBIC | WARP_INVERSE_MAP, borderMode=BORDER_REPLICATE) -- OpenCV's own 8-bit
    path (IPP off) -- for many images in one launch (mn_warp_affine_u8_batched; DESIGN.md 7b, "Oriented text regions").  items:
    list of (src, dst, M): uint8 [h, w, cn] and [dh, dw, cn] CUDA views with dense pixels (any row stride), h, w <= 32767, and M
    a 2 x 3 map from dst pixel indices to src pixel indices whose fixed-point coordinates over dst stay below 2^30 / 1024 pixels
    in magnitude (pipeline.oriented_maps keeps them so)."""
    _warp(items, "warp_affine", 2, _lib.WarpImage, "mn_warp_affine_u8_batched")


def warp_perspective(items):
    """cv2.warpPerspective(src, M, (dw, dh), flags=INTER_CUBIC | WARP_INVERSE_MAP, borderMode=BORDER_REPLICATE) -- OpenCV's own
    8-bit path (IPP off) -- for many images in one launch (mn_warp_perspective_u8_batched; DESIGN.md 7b, "Perspective text
    regions").  items: list of (src, dst, M) as warp_affine takes them, M a 3 x 3 homogeneous map from dst pixel indices to src
    pixel indices whose denominator is positive over dst and whose fixed-point coordinates stay below 2^30 / 32 pixels in
    magnitude (pipeline.quad_maps keeps them so)."""
    _warp(items, "warp_perspective", 3, _lib.WarpPerspectiveImage, "mn_warp_perspective_u8_batched")


def _warp(items, what, rows, record, symbol):
    """One launch of ``symbol`` over warp_affine's / warp_perspective's items, M ``rows`` x 3."""
    global LAUNCHES
    dev = _check_items(items, what, "image")
    cn = _check_channels(items, what)
    recs, mx = [], 0
    for i, (src, dst, m) in enumerate(items):
        _dense_u8(src, dev, cn, f"{what}: image {i}: src")
        _dense_u8(dst, dev, cn, f"{what}: image {i}: dst")
        (h, w), (dh, dw) = src.shape[:2], dst.shape[:2]
        if max(h, w) > 32767:
            raise ValueError(f"{what}: image {i}: a {h}x{w} source exceeds OpenCV's int16 source coordinates")
        m = [float(v) for row in m for v in row]
        if len(m) != 3 * rows:
            raise ValueError(f"{what}: image {i}: M must be {rows} x 3")
        recs.append(record(src.data_ptr(), src.stride(0), h, w, dst.data_ptr(), dst.stride(0), dh, dw, (ctypes.c_double * (3 * rows))(*m)))
        mx = max(mx, dh * dw)
    table = _Pack.of(record, recs, dev)
    _lib.check(getattr(_lib.load(), symbol)(_ptr(table), len(recs), cn, mx, _stream()), symbol)
    LAUNCHES += 1


def composite_regions_affine(regions, feather):
    """composite_regions for pages that hold oriented regions (mn_composite_regions_affine_u8; DESIGN.md 7b, "Oriented text
    regions"), one launch.  regions: list of (page, sr, rect, chain, maps) as composite_regions takes them, maps None for a
    rectangle (composed exactly as composite_regions composes it) or (N, kx, ky) for an oriented region: N (2 x 3, fp64) maps page
    pixels to sr's pixel indices, kx, ky its fp32 feather slopes, and rect is the bounding box of its footprint in page pixels
    (pipeline.oriented_maps).  A page pixel belongs to an oriented region where its fixed-point sr coordinates fall in
    [-1/2, w - 1/2) x [-1/2, h - 1/2)."""
    global LAUNCHES
    recs, mx, pack, chains, _ = _region_records(regions, int(feather), "composite_regions_affine", _lib.RegionAffine)
    out = []
    for i, (r, rec) in enumerate(zip(regions, recs)):
        maps = r[4]
        if maps is None:
            out.append(_lib.RegionAffine(rec, _lib.REGION_RECT, 0.0, 0.0, 0, (ctypes.c_double * 6)()))
            continue
        n, kx, ky = maps
        n = [float(v) for row in n for v in row]
        if len(n) != 6 or not (kx > 0 and ky > 0):
            raise ValueError(f"composite_regions_affine: region {i}: expected (N 2 x 3, kx > 0, ky > 0)")
        out.append(_lib.RegionAffine(rec, _lib.REGION_AFFINE, kx, ky, 0, (ctypes.c_double * 6)(*n)))
    buf = pack.upload((0, bytes((_lib.RegionAffine * len(out))(*out))), chains)
    _lib.check(_lib.load().mn_composite_regions_affine_u8(_ptr(buf), len(out), mx, _stream()), "mn_composite_regions_affine_u8")
    LAUNCHES += 1


def composite_regions_quad(regions, feather):
    """composite_regions_affine for pages that also hold perspective regions (mn_composite_regions_quad_u8; DESIGN.md 7b,
    "Perspective text regions"), one launch.  regions: list of (page, sr, rect, chain, maps) as composite_regions_affine takes
    them; maps may also be (N, kx, ky) with N 3 x 3 (fp64): a perspective region whose page map is homogeneous, with a positive
    denominator over rect, the bounding box of its footprint in page pixels (pipeline.quad_maps).  The footprint test is the
    affine one on its fixed-point sr coordinates."""
    global LAUNCHES
    recs, mx, pack, chains, _ = _region_records(regions, int(feather), "composite_regions_quad", _lib.RegionQuad)
    out = []
    for i, (r, rec) in enumerate(zip(regions, recs)):
        maps = r[4]
        if maps is None:
            out.append(_lib.RegionQuad(rec, _lib.REGION_RECT, 0.0, 0.0, 0, (ctypes.c_double * 9)()))
            continue
        n, kx, ky = maps
        n = [float(v) for row in n for v in row]
        if len(n) not in (6, 9) or not (kx > 0 and ky > 0):
            raise ValueError(f"composite_regions_quad: region {i}: expected (N 2 x 3 or 3 x 3, kx > 0, ky > 0)")
        kind = _lib.REGION_AFFINE if len(n) == 6 else _lib.REGION_PERSPECTIVE
        out.append(_lib.RegionQuad(rec, kind, kx, ky, 0, (ctypes.c_double * 9)(*n)))
    buf = pack.upload((0, bytes((_lib.RegionQuad * len(out))(*out))), chains)
    _lib.check(_lib.load().mn_composite_regions_quad_u8(_ptr(buf), len(out), mx, _stream()), "mn_composite_regions_quad_u8")
    LAUNCHES += 1


class CurveTable(NamedTuple):
    """A curved region's curve table (DESIGN.md 7b, "Curved text regions"; layout in include/marconet_b200.h): ``scale`` s (the
    page's; unused when rectifying), the column fractions ``c`` [c_0 = 0, ..., c_k = 1] and the ``top`` and ``bottom`` curves,
    3k+1 (x, y) points each (segment m: points 3m .. 3m+3)."""
    scale: float
    c: tuple
    top: tuple
    bottom: tuple

    def values(self, what):
        """The fp64 table: s, c_0 .. c_k, the top points, the bottom points (x, y interleaved).  Raises ValueError naming ``what``."""
        import numpy as np
        k = len(self.c) - 1
        top = np.asarray(self.top, np.float64).reshape(-1)
        bottom = np.asarray(self.bottom, np.float64).reshape(-1)
        if not 1 <= k <= 8 or top.size != 6 * k + 2 or bottom.size != 6 * k + 2 or float(self.c[0]) != 0.0 \
                or float(self.c[-1]) != 1.0:
            raise ValueError(f"{what}: expected 1 <= k <= 8 segments, c_0 = 0, c_k = 1 and 3k+1 (x, y) points per curve")
        return np.concatenate([[float(self.scale)], np.asarray(self.c, np.float64), top, bottom]), k


def remap_curved(items):
    """Curved text regions rectified, every crop in one launch (mn_remap_curved_u8_batched; DESIGN.md 7b, "Curved text regions"):
    cv2.remap(src, mapx, mapy, INTER_CUBIC, borderMode=BORDER_REPLICATE) with the fp32 crop maps of each region's curves, OpenCV's
    own 8-bit path (IPP off).  items: list of (src, dst, curve): uint8 [h, w, cn] and [h_r, w_r, cn] CUDA views with dense pixels
    (any row stride), h, w <= 32767, and curve a CurveTable whose crop map stays below 2^14 pixels in magnitude
    (pipeline.plan_regions keeps it so).  The curve tables go up with the records in one copy."""
    global LAUNCHES
    dev = _check_items(items, "remap_curved", "image")
    cn = _check_channels(items, "remap_curved")
    tables = []
    for i, (src, dst, curve) in enumerate(items):
        _dense_u8(src, dev, cn, f"remap_curved: image {i}: src")
        _dense_u8(dst, dev, cn, f"remap_curved: image {i}: dst")
        if max(src.shape[:2]) > 32767:
            raise ValueError(f"remap_curved: image {i}: a {src.shape[0]}x{src.shape[1]} source exceeds OpenCV's int16 source "
                             f"coordinates")
        tables.append(curve.values(f"remap_curved: image {i}"))
    pack = _Pack()
    pack.area(len(items) * ctypes.sizeof(_lib.RemapCurvedImage))
    t_off = pack.area(8 * sum(t.size for t, _ in tables))
    base, o, recs, mx = pack.alloc(dev) + t_off, 0, [], 0
    for (src, dst, _), (t, k) in zip(items, tables):
        (h, w), (dh, dw) = src.shape[:2], dst.shape[:2]
        recs.append(_lib.RemapCurvedImage(src.data_ptr(), src.stride(0), h, w, dst.data_ptr(), dst.stride(0), dh, dw, base + 8 * o,
                                          k, 0))
        o += t.size
        mx = max(mx, dh * dw)
    buf = pack.upload((0, bytes((_lib.RemapCurvedImage * len(recs))(*recs))), (t_off, b"".join(t.tobytes() for t, _ in tables)))
    _lib.check(_lib.load().mn_remap_curved_u8_batched(_ptr(buf), len(recs), cn, mx, _stream()), "mn_remap_curved_u8_batched")
    LAUNCHES += 1


FLAT_MAX_COLUMN_LINES = _lib.FLAT_MAX_COLUMN_LINES


def flat_column_lines(lines, width):
    """The most lines of an fp64 line table (pipeline.flat_line_table) that one of ``width`` frame columns meets."""
    import numpy as np
    if len(lines) == 0:
        return 0
    d = np.zeros(width + 1, np.int64)
    np.add.at(d, np.asarray(lines[:, 7], np.int64), 1)
    np.add.at(d, np.asarray(lines[:, 8], np.int64), -1)
    return int(np.cumsum(d).max())


def flat_remap(items, tables=False):
    """Curled pages flattened through their dewarp field, every page in two launches (mn_flat_columns_batched, then
    mn_flat_remap_u8_batched; DESIGN.md 7b, "Flat pages").  items: list of (src, dst, kind, m, lines): src the uint8 [h, w, cn]
    photo and dst the [dh, dw, cn] flat page, CUDA views with dense pixels (any row stride), h, w <= 32767; kind "rect" (m = (x0,
    y0)) or "quad" (m = the unit-square homography's a .. h); lines the page's fp64 [n, 9] line table (pipeline.flat_line_table)
    with block ranges inside [0, dw].  The records and line tables go up in one copy.  ``tables`` (tests): also return per page
    the int32 CUDA view [3, dw] of its column counts and neighbours, and the fp64 view [dw, stride, 2] of its (Y, M) pairs.
    Raises ValueError naming the page, before any launch, for a column met by more than FLAT_MAX_COLUMN_LINES lines."""
    import numpy as np
    global LAUNCHES
    dev = _check_items(items, "flat_remap", "page")
    cn = _check_channels(items, "flat_remap")
    tabs, strides = [], []
    for i, (src, dst, kind, m, lines) in enumerate(items):
        what = f"flat_remap: page {i}"
        _dense_u8(src, dev, cn, f"{what}: src")
        _dense_u8(dst, dev, cn, f"{what}: dst")
        if max(src.shape[:2]) > 32767:
            raise ValueError(f"{what}: a {src.shape[0]}x{src.shape[1]} source exceeds OpenCV's int16 source coordinates")
        if kind not in ("rect", "quad") or len(m) != (2 if kind == "rect" else 8):
            raise ValueError(f"{what}: expected kind 'rect' with (x0, y0) or 'quad' with H's eight values")
        t = np.ascontiguousarray(lines, np.float64).reshape(-1, _lib.FLAT_LINE_DOUBLES)
        dw = dst.shape[1]
        if len(t) and not (np.all(t[:, 7] >= 0) and np.all(t[:, 7] < t[:, 8]) and np.all(t[:, 8] <= dw)
                           and np.all(t[:, 7] == np.floor(t[:, 7])) and np.all(t[:, 8] == np.floor(t[:, 8]))):
            raise ValueError(f"{what}: a line's block range is not an integer range inside the {dw} columns")
        stride = flat_column_lines(t, dw)
        if stride > FLAT_MAX_COLUMN_LINES:
            raise ValueError(f"{what}: a column meets {stride} lines, over the {FLAT_MAX_COLUMN_LINES} a column may hold")
        tabs.append(t)
        strides.append(max(1, stride))
    pack = _Pack()                  # the records, then every line table, then each page's column table and (Y, M) pairs
    pack.area(len(items) * ctypes.sizeof(_lib.FlatPage))
    los = [pack.area(8 * t.size, 8) for t in tabs]
    offs = [(lo, pack.area(12 * d.shape[1], 8), pack.area(16 * d.shape[1] * stride, 8))
            for (_, d, *_), lo, stride in zip(items, los, strides)]
    base, recs, mx, mw = pack.alloc(dev), [], 0, 0
    for (src, dst, kind, m, _), t, stride, (lo, co, fo) in zip(items, tabs, strides, offs):
        (h, w), (dh, dw) = src.shape[:2], dst.shape[:2]
        recs.append(_lib.FlatPage(src.data_ptr(), src.stride(0), h, w, dst.data_ptr(), dst.stride(0), dh, dw, base + lo, base + co,
                                  base + fo, len(t), stride, _lib.FLAT_RECT if kind == "rect" else _lib.FLAT_QUAD, 0,
                                  (ctypes.c_double * 8)(*[float(v) for v in m])))
        mx, mw = max(mx, dh * dw), max(mw, dw)
    buf = pack.upload((0, bytes((_lib.FlatPage * len(recs))(*recs))), (los[0], b"".join(t.tobytes() for t in tabs)))
    lib = _lib.load()
    _lib.check(lib.mn_flat_columns_batched(base, len(recs), mw, _stream()), "mn_flat_columns_batched")
    _lib.check(lib.mn_flat_remap_u8_batched(base, len(recs), cn, mx, _stream()), "mn_flat_remap_u8_batched")
    LAUNCHES += 2
    if not tables:
        return None
    return [(buf[co:co + 12 * d.shape[1]].view(torch.int32).view(3, d.shape[1]),
             buf[fo:fo + 16 * d.shape[1] * s].view(torch.float64).view(d.shape[1], s, 2))
            for (_, d, *_), s, (_, co, fo) in zip(items, strides, offs)]


LIGHT_MAX_WINDOW = 32767


def light_window(w, h):
    """The default evening window of a w x h frame (DESIGN.md 7b, "Even lighting"): max(3, 2 floor(min(w, h) / 40) + 1), a
    heuristic that holds a line of ordinary text."""
    return max(3, 2 * (min(w, h) // 40) + 1)


def even_light(items, inks=None):
    """Pages evened by their paper, every page in six launches (mn_even_light_u8; DESIGN.md 7b, "Even lighting"): E = rint(255 F
    / B) per channel, B the grey closing of F with a k x k window cut to the page, complemented on read and write for light ink.
    items: list of (frame, src, dst, k, polarity): src and dst uint8 [h, w, 3] CUDA views with dense pixels (any row stride) of
    the same size, sides <= 32767 (dst may be src: evened in place); k an odd int in [3, 32767]; frame the [h_f, w_f, 3] view
    whose histogram and Otsu threshold choose the ink under polarity _lib.INK_AUTO (else the polarity given).
    ``inks``: None, or per item the int32 CUDA view of 4 values an earlier call returned: its ink is used as it is on the device,
    frame and polarity are ignored and the call takes four launches.  Returns the int32 CUDA tensor [n, 4] of every page's
    (0, threshold, ink, 0), whose rows an evening of the same pages may take as ``inks``; None when ``inks`` is given."""
    global LAUNCHES
    dev = _check_items(items, "even_light", "page", 1)
    if inks is not None and len(inks) != len(items):
        raise ValueError("even_light: one ink per page")
    n = len(items)
    tiles, lines = 1, 1
    for i, (frame, src, dst, k, polarity) in enumerate(items):
        what = f"even_light: page {i}"
        _dense_u8(src, dev, 3, f"{what}: src")
        _dense_u8(dst, dev, 3, f"{what}: dst")
        h, w = src.shape[:2]
        if tuple(dst.shape) != tuple(src.shape) or max(h, w) > 32767:
            raise ValueError(f"{what}: src {tuple(src.shape)} and dst {tuple(dst.shape)} differ or have a side over 32767")
        if isinstance(k, bool) or not isinstance(k, int) or not 3 <= k <= LIGHT_MAX_WINDOW or k % 2 == 0:
            raise ValueError(f"{what}: the window must be an odd int in [3, {LIGHT_MAX_WINDOW}], got {k!r}")
        if inks is None:
            _dense_u8(frame, dev, 3, f"{what}: frame")
            if max(frame.shape[:2]) > 32767 or polarity not in (_lib.INK_AUTO, _lib.INK_DARK, _lib.INK_LIGHT):
                raise ValueError(f"{what}: a frame side over 32767 or a bad polarity {polarity!r}")
            tiles = max(tiles, -(-frame.shape[0] // 32) * -(-frame.shape[1] // 32))
        elif not (isinstance(inks[i], torch.Tensor) and inks[i].device == dev and inks[i].dtype == torch.int32
                  and inks[i].numel() == 4 and inks[i].is_contiguous()):
            raise ValueError(f"{what}: an ink must be an int32 CUDA view of 4 values on {dev}")
        lines = max(lines, h * -(-w // k), w * -(-h // k))
    pack = _Pack()                  # the crop records, the page records, the threshold work, then each page's two planes
    pack.area(n * ctypes.sizeof(_lib.TextBlock))
    o_rec = pack.area(n * ctypes.sizeof(_lib.LightPage))
    o_work = pack.area(1024 * n if inks is None else 0, 8)
    planes = [[pack.area(3 * src.shape[0] * src.shape[1], 8) for _ in range(2)] for _, src, *_ in items]
    base = pack.alloc(dev)
    if inks is None:                # apart from the work, so that the scratch planes are freed with the call
        table = torch.zeros(n, 4, dtype=torch.int32, device=dev)
        inks, threshold = table.unbind(0), 1
    else:
        threshold = 0
    blocks, recs = [], []
    for i, ((frame, src, dst, k, polarity), pl) in enumerate(zip(items, planes)):
        if threshold:
            fh, fw = frame.shape[:2]
            tb = _lib.TextBlock(frame.data_ptr(), frame.stride(0), 0, 0, fw, fh, 0, polarity, 0, 0, 0, 0, base + o_work + 1024 * i,
                                0, 0, inks[i].data_ptr())
        else:
            tb = _lib.TextBlock(0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, inks[i].data_ptr())
        blocks.append(tb)
        recs.append(_lib.LightPage(tb, src.data_ptr(), src.stride(0), dst.data_ptr(), dst.stride(0), src.shape[0], src.shape[1], k, 0,
                                   base + pl[0], base + pl[1]))
    pack.upload((0, bytes((_lib.TextBlock * n)(*blocks))), (o_rec, bytes((_lib.LightPage * n)(*recs))))
    if threshold:
        _lib.check(_lib.load().mn_even_light_u8(base, base + o_rec, n, 1, tiles, lines, base + o_work, 1024 * n, _stream()),
                   "mn_even_light_u8")
        LAUNCHES += 6
        return table
    _lib.check(_lib.load().mn_even_light_u8(0, base + o_rec, n, 0, 0, lines, 0, 0, _stream()), "mn_even_light_u8")
    LAUNCHES += 4
    return None


def even_light_bytes(w, h, frame=None):
    """Device bytes of evening a w x h page beyond the page itself: its two scratch planes and, when ``frame`` (w_f, h_f) is
    given, the evened frame the page's searches read."""
    n = 2 * (-(-3 * w * h // 8) * 8) + 1024 + 16
    if frame is not None:
        n += 3 * frame[0] * frame[1]
    return n


def composite_regions_curved(regions, feather):
    """composite_regions_quad for pages that also hold curved regions (mn_composite_regions_curved_u8; DESIGN.md 7b, "Curved text
    regions"), one launch.  regions: list of (page, sr, rect, chain, maps) as composite_regions_quad takes them; maps may also be
    (curve, kx, ky) with curve a CurveTable whose scale is the page's: a curved region, rect the bounding box of its control points
    in page pixels widened by one pixel (pipeline.curved_footprint_box).  Rectangles, oriented and perspective regions are
    composed exactly as composite_regions_quad composes them.  The records, chains and curve tables go up in one copy."""
    import numpy as np
    global LAUNCHES
    tables = {}
    for i, r in enumerate(regions):
        if r[4] is not None and isinstance(r[4][0], CurveTable):
            t, k = r[4][0].values(f"composite_regions_curved: region {i}")
            if not t[0] >= 1:
                raise ValueError(f"composite_regions_curved: region {i}: scale {t[0]} < 1")
            tables[i] = (t, k)
    recs, mx, pack, chains, t_off = _region_records(regions, int(feather), "composite_regions_curved", _lib.RegionCurved,
                                                    tables=8 * sum(t.size for t, _ in tables.values()))
    out, o = [], 0
    for i, (r, rec) in enumerate(zip(regions, recs)):
        maps = r[4]
        if maps is None:
            out.append(_lib.RegionCurved(_lib.RegionQuad(rec, _lib.REGION_RECT, 0.0, 0.0, 0, (ctypes.c_double * 9)()), None, 0, 0))
            continue
        n, kx, ky = maps
        if not (kx > 0 and ky > 0):
            raise ValueError(f"composite_regions_curved: region {i}: feather slopes kx = {kx}, ky = {ky} must be > 0")
        if i in tables:
            t, k = tables[i]
            out.append(_lib.RegionCurved(_lib.RegionQuad(rec, _lib.REGION_CURVED, kx, ky, 0, (ctypes.c_double * 9)()),
                                         pack.buf.data_ptr() + t_off + 8 * o, k, 0))
            o += t.size
            continue
        n = [float(v) for row in n for v in row]
        if len(n) not in (6, 9):
            raise ValueError(f"composite_regions_curved: region {i}: expected (N 2 x 3 or 3 x 3, kx, ky) or (CurveTable, kx, ky)")
        kind = _lib.REGION_AFFINE if len(n) == 6 else _lib.REGION_PERSPECTIVE
        out.append(_lib.RegionCurved(_lib.RegionQuad(rec, kind, kx, ky, 0, (ctypes.c_double * 9)(*n)), None, 0, 0))
    buf = pack.upload((0, bytes((_lib.RegionCurved * len(out))(*out))), chains,
                      (t_off, b"".join(tables[i][0].tobytes() for i in sorted(tables))))
    _lib.check(_lib.load().mn_composite_regions_curved_u8(_ptr(buf), len(out), mx, _stream()), "mn_composite_regions_curved_u8")
    LAUNCHES += 1


def _vertical_gather(items, what, width, symbol):
    """One launch of ``symbol`` over vertical_layout's / vertical_unlayout's items, ``width`` int32 values per cell."""
    import numpy as np
    global LAUNCHES
    dev = _check_items(items, what, "column")
    tables = []
    for i, (src, dst, cells) in enumerate(items):
        _dense_u8(src, dev, 3, f"{what}: column {i}: src")
        _dense_u8(dst, dev, 3, f"{what}: column {i}: dst")
        t = np.asarray(cells, dtype=np.int64).reshape(-1, width)
        (sh, sw), (dh, dw) = src.shape[:2], dst.shape[:2]
        if width == 3:                                   # (c_k, p_k, t_k): rows [c_k, c_k + t_k) of C, columns [0, w)
            ok = len(t) >= 1 and dw % len(t) == 0 and dw // len(t) <= sw and (t[:, 2] >= 1).all() and (t[:, 0] >= 0).all() \
                and (t[:, 0] + t[:, 2] <= sh).all()
        else:                                            # rows [min(R(p), R(p+t) - 1), R(p+t)), columns [min(lo, hi - 1), hi)
            ok = len(t) >= 1 and t[0, 0] == 0 and (np.diff(t[:, 0]) >= 0).all() and (t[:, 2] <= sh).all() \
                and (np.minimum(t[:, 1], t[:, 2] - 1) >= 0).all() and (t[:, 4] <= sw).all() \
                and (np.minimum(t[:, 3], t[:, 4] - 1) >= 0).all()
        if not ok or t.max() >= 2 ** 31:
            raise ValueError(f"{what}: column {i}: its cell table reads outside the {sh}x{sw} source")
        tables.append(t.astype(np.int32))
    pack = _Pack()
    pack.area(len(items) * ctypes.sizeof(_lib.VerticalColumn))
    t_off = pack.area(4 * sum(t.size for t in tables))
    base, o, recs, mx = pack.alloc(dev) + t_off, 0, [], 0
    for (src, dst, _), t in zip(items, tables):
        dh, dw = dst.shape[:2]
        recs.append(_lib.VerticalColumn(src.data_ptr(), src.stride(0), dst.data_ptr(), dst.stride(0), base + 4 * o, dh, dw, len(t),
                                        dw // len(t) if width == 3 else 0))
        o += t.size
        mx = max(mx, dh * dw)
    buf = pack.upload((0, bytes((_lib.VerticalColumn * len(recs))(*recs))), (t_off, b"".join(t.tobytes() for t in tables)))
    _lib.check(getattr(_lib.load(), symbol)(_ptr(buf), len(recs), mx, _stream()), symbol)
    LAUNCHES += 1


def vertical_layout(items):
    """Vertical text columns laid out as horizontal lines, every column in one launch (mn_vertical_layout_u8_batched; DESIGN.md
    7b, "Vertical text columns").  items: list of (C, L, cells): uint8 [h_r, w_r, 3] and [H_L, n w_r, 3] CUDA views with dense
    pixels (any row stride; C may be read in place through a page's pitch), cells the n (c_k, p_k, t_k) of
    pipeline.vertical_plan: L[i, k w_r + j] = C[c_k + clamp(i - p_k, 0, t_k - 1), j]."""
    _vertical_gather(items, "vertical_layout", 3, "mn_vertical_layout_u8_batched")


def block_lines_dtype():
    """numpy view of an mn_block_lines record (the output of mn_find_lines_u8)."""
    import numpy as np
    return np.dtype([("n_lines", "<i4"), ("threshold", "<i4"), ("ink", "<i4"), ("pad", "<i4"),
                     ("rect", "<i4", (_lib.BLOCK_MAX_LINES, 4))])


SKEW_MAX_PROFILE = 1 << 24     # int32 values of one skewed block's angle profiles (64 MB)


def skew_table(skew, max_skew, vertical):
    """The frame angles of a skewed block's search (DESIGN.md 7b, "Skewed blocks"), in degrees: i / 20 for |i| <= round(20
    max_skew) with skew "auto", else the given angle, negated for a vertical block (whose frame is the transposed crop)."""
    if isinstance(skew, str):
        n = round(20 * max_skew)
        return [i / 20 for i in range(-n, n + 1)]
    return [-float(skew) if vertical else float(skew)]


def skew_cos_sin(angles):
    """fp64 (c, s) of frame angles in degrees, computed on the host: the device has no trigonometry."""
    return [(math.cos(math.radians(t)), math.sin(math.radians(t))) for t in angles]


def skew_stride(w, h, vertical, cs):
    """The largest number of bins L of a w x h crop's frames over the (c, s) of ``cs``, as the device computes it."""
    import numpy as np
    wt, ht = (h, w) if vertical else (w, h)
    c, s = (np.array([p[k] for p in cs], np.float64) for k in (0, 1))
    xs, ys = (0.5 - wt / 2, wt - 0.5 - wt / 2), (0.5 - ht / 2, ht - 0.5 - ht / 2)
    v = np.stack([x * s + y * c for x in xs for y in ys])
    return int((np.floor(v.max(axis=0) - v.min(axis=0)) + 1).max())


def skew_frames(w, h, vertical, cs):
    """(u_min, v_min, L, M) of a w x h crop's frames (transposed for a vertical crop) at each (c, s) of ``cs``, as the device's
    frame_of computes them: fp64 arrays, every operation rounded on its own."""
    import numpy as np
    wt, ht = (h, w) if vertical else (w, h)
    c, s = (np.array([p[k] for p in cs], np.float64) for k in (0, 1))
    xs, ys = (0.5 - wt / 2, wt - 0.5 - wt / 2), (0.5 - ht / 2, ht - 0.5 - ht / 2)
    u = np.stack([x * c - y * s for x in xs for y in ys])
    v = np.stack([x * s + y * c for x in xs for y in ys])
    return (u.min(axis=0), v.min(axis=0), (np.floor(v.max(axis=0) - v.min(axis=0)) + 1).astype(np.int64),
            (np.floor(u.max(axis=0) - u.min(axis=0)) + 1).astype(np.int64))


def skew_block_dtype():
    """numpy view of an mn_skew_block record after mn_find_lines_skewed_u8: the chosen index and frame."""
    import numpy as np
    return np.dtype([("b", np.uint8, ctypes.sizeof(_lib.TextBlock)), ("table", "<u8"), ("scores", "<u8"), ("profiles", "<u8"),
                     ("n_ang", "<i4"), ("stride", "<i4"), ("chosen", "<i4"), ("L", "<i4"), ("M", "<i4"), ("pad", "<i4"),
                     ("u_min", "<f8"), ("v_min", "<f8"), ("c", "<f8"), ("s", "<f8")])


def _check_crop(item, dev, what, knob_names):
    """(x0, y0, w, h) of a layout item (img, rect, vertical, polarity, *knobs), validated as find_lines and find_blocks describe
    it.  Raises naming ``what``."""
    img, rect, _, polarity, *knobs = item
    _dense_u8(img, dev, 3, f"{what}: img")
    x0, y0, x1, y1 = (int(v) for v in rect)
    if not (0 <= x0 < x1 <= img.shape[1] and 0 <= y0 < y1 <= img.shape[0]) or max(x1 - x0, y1 - y0) > 32767:
        raise ValueError(f"{what}: rectangle {(x0, y0, x1, y1)} is empty, outside the "
                         f"{img.shape[1]}x{img.shape[0]} image or has a side over 32767")
    if polarity not in (_lib.INK_AUTO, _lib.INK_DARK, _lib.INK_LIGHT) or any(v is not None and not 1 <= v < 2 ** 31 for v in knobs):
        raise ValueError(f"{what}: bad polarity {polarity!r} or {knob_names} {knobs!r}")
    return x0, y0, x1 - x0, y1 - y0


def _check_skew(skew, max_skew, vertical, what):
    """The (c, s) table of skew / max_skew (find_lines' rules), or ValueError naming ``what``."""
    if skew is None:
        return [(1.0, 0.0)]
    if not (skew == "auto" if isinstance(skew, str) else math.isfinite(skew) and abs(skew) < 45):
        raise ValueError(f"{what}: bad skew {skew!r}")
    if not (isinstance(skew, str) or max_skew == 10.0) or not 0 < max_skew <= 20:
        raise ValueError(f"{what}: max_skew {max_skew!r} is outside (0, 20] or given without 'auto'")
    return skew_cos_sin(skew_table(skew, max_skew, vertical))


def _angle_tables(tables):
    """The fp64 (c, s) bytes of the distinct tables among ``tables``, and the offset of each one in (c, s) entries."""
    import numpy as np
    keys, offs, n = {}, [], 0
    for cs in tables:
        key = tuple(cs)
        if key not in keys:
            keys[key], n = n, n + len(cs)
        offs.append(keys[key])
    return np.array([v for key in keys for p in key for v in p], np.float64).tobytes(), offs


def _skew_block(tb, table, scores, profiles, n_ang, stride):
    """The mn_skew_block record of the crop ``tb`` over the n_ang (c, s) at ``table``; only a search (n_ang > 1) has per-angle
    scores and profiles."""
    return _lib.SkewBlock(tb, table, scores if n_ang > 1 else 0, profiles if n_ang > 1 else 0, n_ang, stride)


def find_lines(blocks, scores=False):
    """Text blocks split into lines, every block in four launches whatever their number (mn_find_lines_u8; DESIGN.md 7b, "Text
    blocks").  blocks: list of (img, rect, vertical, polarity, min_ink, gap, min_height[, skew, max_skew]): img a uint8 [H, W, 3]
    CUDA view with dense pixels (any row stride) read in place, rect (x0, y0, x1, y1) a non-empty crop inside it with sides
    <= 32767, vertical a bool, polarity _lib.INK_AUTO / INK_DARK / INK_LIGHT, and min_ink, gap, min_height positive integers or
    None for the default.  Returns the uint8 CUDA tensor of the blocks' mn_block_lines records, in order (read it back as
    ``block_lines_dtype()``).
    skew (DESIGN.md 7b, "Skewed blocks"): None, "auto" (search +-max_skew degrees) or a given angle in degrees, |skew| < 45.  A
    call with any skewed block goes through mn_find_lines_skewed_u8's six launches instead, every block of it, whatever their
    number; blocks with skew None search the one-entry table (1, 0), which keeps their mn_block_lines records exactly.  The
    tensor then holds the n mn_block_lines records followed by the n mn_skew_block records (``skew_block_dtype()``: the chosen
    index and frame).  ``scores`` (tests): also return, per block, the int64 CUDA view of its per-angle scores (None unless it
    searched).
    seals (DESIGN.md 7b, "Seals"; index 9, blocks with skew None only): None or a list of at most PAGE_MAX_SEALS seal boxes
    (x0, y0, x1, y1) in image pixels.  Such a block is split on its layout copy, the crop with every seal-coloured pixel inside
    a box's inscribed ellipse (rho < 33 / 32) set to paper, made by one more launch (mn_seal_layout_u8) for all sealed blocks
    of the call; a call with skewed blocks reads the copies through its skew records alike.  The copies (seal_block_bytes)
    may use PAGE_MAX_WORK bytes per call."""
    global LAUNCHES
    dev = _check_items(blocks, "find_lines", "block")
    skewed = any(len(b) > 7 and b[7] is not None for b in blocks)
    n = len(blocks)
    osz, rsz = ctypes.sizeof(_lib.BlockLines), ctypes.sizeof(_lib.TextBlock)
    ssz = ctypes.sizeof(_lib.SkewBlock) if skewed else 0
    dims, tables, copies = [], [], 0
    for i, blk in enumerate(blocks):
        what = f"find_lines: block {i}"
        x0, y0, bw, bh = _check_crop(blk[:7], dev, what, "min_ink / gap / min_height")
        vertical, skew, max_skew = blk[2], blk[7] if len(blk) > 7 else None, blk[8] if len(blk) > 8 else 10.0
        cs = _check_skew(skew, max_skew, vertical, what)
        if len(blk) > 9 and blk[9]:
            if skew is not None or len(blk[9]) > _lib.PAGE_MAX_SEALS:
                raise ValueError(f"{what}: a sealed block is level (skew None) and has at most {_lib.PAGE_MAX_SEALS} seals")
            copies += seal_block_bytes(bw, bh)
            if copies > PAGE_MAX_WORK:
                raise ValueError(f"{what}: the sealed blocks up to this one need {copies} bytes of layout copies, over the "
                                 f"{PAGE_MAX_WORK} a call may use")
        stride = (bw if vertical else bh) if skew is None else skew_stride(bw, bh, vertical, cs)
        if len(cs) > 1 and len(cs) * stride > SKEW_MAX_PROFILE:
            raise ValueError(f"{what}: {len(cs)} angles x {stride} bins exceed the {SKEW_MAX_PROFILE} profile values a skewed "
                             f"block may use")
        tables.append(cs)
        dims.append((x0, y0, bw, bh, len(cs), stride))
    tab, t_offs = _angle_tables(tables) if skewed else (b"", [0] * n)
    sealed = [i for i, blk in enumerate(blocks) if len(blk) > 9 and blk[9]]
    m, tsz, spsz = len(sealed), ctypes.sizeof(_lib.SealTable), ctypes.sizeof(_lib.SealPage)
    pack = _Pack()                  # results, skew records, crop records, tables; scores, work (zeroed); scratch; seal records,
    pack.area(n * osz)              # tables and layout copies
    sk, seg, t_off = pack.area(n * ssz), pack.area(n * rsz), pack.area(len(tab))
    score = [pack.area(8 * n_ang if n_ang > 1 else 0) for *_, n_ang, _ in dims]
    work = [(pack.area(4 * 256), pack.area(4 * 3 * L), pack.area(4 * n_ang * L if n_ang > 1 else 0)) for *_, n_ang, L in dims]
    w_end = pack.end
    scratch = [pack.area(4 * (2 * L + 4)) for *_, L in dims]
    sp, st = (pack.area(m * spsz, 16), pack.area(m * tsz, 16)) if sealed else (0, 0)
    copies = {i: pack.area(3 * dims[i][2] * dims[i][3], 16) for i in sealed}
    base = pack.alloc(dev)
    recs, srecs, views, tiles, seal_recs, seal_tabs = [], [], [], 0, [], []
    for i, (blk, (x0, y0, bw, bh, n_ang, stride), sc, (hist, prof, ext), scr, t) in \
            enumerate(zip(blocks, dims, score, work, scratch, t_offs)):
        img, _, vertical, polarity, min_ink, gap, min_height = blk[:7]
        src, pitch = img.data_ptr(), img.stride(0)
        if i in copies:             # the block reads its layout copy through its own crop offsets
            crop = _lib.TextBlock(src, pitch, x0, y0, bw, bh)
            src, pitch = (base + copies[i] - y0 * 3 * bw - 3 * x0) % (1 << 64), 3 * bw
            seal_recs.append(_lib.SealPage(crop, base + copies[i], 0, 0, 0, base + st + len(seal_tabs) * tsz))
            seal_tabs.append(seal_table(blk[9], x0, y0))
        tb = _lib.TextBlock(src, pitch, x0, y0, bw, bh, int(bool(vertical)), polarity, min_ink or 0, gap or 0,
                            min_height or 0, 0, base + hist, base + prof, base + scr, base + i * osz)
        recs.append(tb)
        if skewed:
            srecs.append(_skew_block(tb, base + t_off + 16 * t, base + sc, base + ext, n_ang, stride))
        views.append(pack.buf[sc:sc + 8 * n_ang].view(torch.int64) if n_ang > 1 else None)
        tiles = max(tiles, -(-bw // 32) * -(-bh // 32))
    pack.upload((sk, bytes((_lib.SkewBlock * len(srecs))(*srecs))), (seg, bytes((_lib.TextBlock * n)(*recs))), (t_off, tab),
                *(((sp, bytes((_lib.SealPage * m)(*seal_recs))), (st, b"".join(seal_tabs))) if sealed else ()))
    if sealed:
        _lib.check(_lib.load().mn_seal_layout_u8(base + sp, m, max(-(-dims[i][2] // 32) * -(-dims[i][3] // 32) for i in sealed),
                                                 _stream()), "mn_seal_layout_u8")
        LAUNCHES += 1
    if skewed:
        _lib.check(_lib.load().mn_find_lines_skewed_u8(base + seg, base + sk, n, tiles, base + score[0], w_end - score[0],
                                                       _stream()), "mn_find_lines_skewed_u8")
        LAUNCHES += 6
    else:
        _lib.check(_lib.load().mn_find_lines_u8(base + seg, n, tiles, base + score[0], w_end - score[0], _stream()),
                   "mn_find_lines_u8")
        LAUNCHES += 4
    res = pack.buf[:n * (osz + ssz)]
    return (res, views) if scores else res


def seal_table(boxes, x0=0, y0=0):
    """The bytes of the mn_seal_table of given seal ``boxes`` (x0, y0, x1, y1) of a crop at (x0, y0): each box in crop pixels,
    a found seal, in the order given."""
    t = _lib.SealTable(0, len(boxes), len(boxes))
    for j, (a, b, c, d) in enumerate(boxes):
        t.seal[j] = _lib.Seal(a - x0, b - y0, c - x0, d - y0, -1, 0, 1, -1, -1, -1, -1, 0, 0)
    return bytes(t)


def seal_block_bytes(w, h):
    """Device bytes a sealed w x h block adds to find_lines (DESIGN.md 7b, "Seals"): its layout copy (3 w h), record and seal
    table, with 16 bytes for each area's alignment.  A call's sealed blocks may use PAGE_MAX_WORK bytes in all."""
    return 3 * w * h + ctypes.sizeof(_lib.SealPage) + ctypes.sizeof(_lib.SealTable) + 3 * 16


def _seal_areas(w, h):
    """Byte sizes of one seal page's areas after the results in find_blocks: its layout copy, cell labels, cell boxes and
    candidate list."""
    cells = -(-w // 4) * -(-h // 4)
    return [3 * w * h, 4 * cells, 16 * cells, 32 * _lib.PAGE_MAX_SEALS]


def seal_bytes(w, h):
    """Device bytes a w x h page adds to find_blocks when its seals are found (DESIGN.md 7b, "Seals"): its record, seal table,
    candidate list, cell labels and boxes (one int32 and four per 4 x 4 cell) and its layout copy (3 w h), with 16 bytes for
    each area's alignment."""
    return ctypes.sizeof(_lib.SealPage) + ctypes.sizeof(_lib.SealTable) + sum(_seal_areas(w, h)) + 6 * 16


def window_footprint(w, h, vertical, c, s, u_min, v_min, window):
    """(px0, py0, px1, py1): the crop pixels that hold a window's pixel set, the fp64 bounding box of the window's corner pixel
    centres (X = u c + v s, Y = v c - u s), padded by one pixel and clipped.  The padding covers the rounding of the frame."""
    wt, ht = (h, w) if vertical else (w, h)
    c0, l0, c1, l1 = window
    xs, ys = [], []
    for u in (u_min + c0, u_min + c1):
        for v in (v_min + l0, v_min + l1):
            xs.append(u * c + v * s + wt / 2 - 0.5)
            ys.append(v * c - u * s + ht / 2 - 0.5)
    fx0, fx1 = max(0, math.floor(min(xs)) - 1), min(wt, math.floor(max(xs)) + 2)
    fy0, fy1 = max(0, math.floor(min(ys)) - 1), min(ht, math.floor(max(ys)) + 2)
    return (fy0, fx0, fy1, fx1) if vertical else (fx0, fy0, fx1, fy1)


def find_lines_window(blocks):
    """Windowed text blocks split into lines, every block in four launches whatever their number (mn_find_lines_window_u8;
    DESIGN.md 7b, "Skewed pages").  blocks: list of (img, rect, vertical, polarity, min_ink, gap, min_height, skew, window): as
    find_lines', skew a given finite angle and window (c0, l0, c1, l1) a non-empty integer rectangle inside the crop's frame at
    that angle (the transposed crop at the negated angle for a vertical block).  Returns the uint8 CUDA tensor of the blocks'
    mn_block_lines records, in order, whose rectangles are (c0', l0', c1', l1') in cells of the window."""
    global LAUNCHES
    dev = _check_items(blocks, "find_lines_window", "block")
    n = len(blocks)
    osz, rsz, wsz = ctypes.sizeof(_lib.BlockLines), ctypes.sizeof(_lib.TextBlock), ctypes.sizeof(_lib.WindowBlock)
    dims = []
    for i, blk in enumerate(blocks):
        what = f"find_lines: block {i}"
        img, rect, vertical, polarity, min_ink, gap, min_height, skew, window = blk
        x0, y0, bw, bh = _check_crop(blk[:7], dev, what, "min_ink / gap / min_height")
        if isinstance(skew, str) or skew is None or not math.isfinite(skew) or abs(skew) >= 45:
            raise ValueError(f"{what}: a window needs a given finite angle, got skew {skew!r}")
        (c, s), = _check_skew(skew, 10.0, vertical, what)
        u_min, v_min, L, M = (float(a[0]) for a in skew_frames(bw, bh, vertical, [(c, s)]))
        c0, l0, c1, l1 = (int(v) for v in window)
        if not (0 <= c0 < c1 <= M and 0 <= l0 < l1 <= L):
            raise ValueError(f"{what}: window {(c0, l0, c1, l1)} is empty or outside the {int(M)}x{int(L)} frame")
        fp = window_footprint(bw, bh, vertical, c, s, u_min, v_min, (c0, l0, c1, l1))
        dims.append((x0, y0, bw, bh, c, s, (c0, l0, c1, l1), fp))
    pack = _Pack()                  # results, line records, window records; work (zeroed); scratch
    pack.area(n * osz)
    seg, wrec = pack.area(n * rsz), pack.area(n * wsz)
    work = [(pack.area(4 * 256), pack.area(4 * 3 * (d[6][3] - d[6][1]))) for d in dims]
    w_end = pack.end
    scratch = [pack.area(4 * (2 * (d[6][3] - d[6][1]) + 4)) for d in dims]
    base = pack.alloc(dev)
    recs, wrecs, tiles = [], [], 0
    for i, (blk, (x0, y0, bw, bh, c, s, (c0, l0, c1, l1), (px0, py0, px1, py1)), (hist, prof), scr) in \
            enumerate(zip(blocks, dims, work, scratch)):
        img, _, vertical, polarity, min_ink, gap, min_height = blk[:7]
        knobs = (polarity, min_ink or 0, gap or 0, min_height or 0, 0, base + hist, base + prof, base + scr, base + i * osz)
        recs.append(_lib.TextBlock(img.data_ptr(), img.stride(0), 0, 0, c1 - c0, l1 - l0, 0, *knobs))
        crop = _lib.TextBlock(img.data_ptr(), img.stride(0), x0, y0, bw, bh, int(bool(vertical)), *knobs)
        wrecs.append(_lib.WindowBlock(crop, c, s, c0, l0, c1, l1, px0, py0, px1 - px0, py1 - py0))
        tiles = max(tiles, 1, -(-(px1 - px0) // 32) * -(-(py1 - py0) // 32))
    buf = pack.upload((seg, bytes((_lib.TextBlock * n)(*recs))), (wrec, bytes((_lib.WindowBlock * n)(*wrecs))))
    _lib.check(_lib.load().mn_find_lines_window_u8(base + seg, base + wrec, n, tiles, base + work[0][0], w_end - work[0][0],
                                                   _stream()), "mn_find_lines_window_u8")
    LAUNCHES += 4
    return buf[:n * osz]


CURVE_MAX_STRIPS = _lib.CURVE_MAX_STRIPS
CURVE_MIN_STRIP = 32           # pixels of a strip when there are several: a 32-pixel tile then spans at most two strips
CURVE_MAX_WORK = 1 << 30       # bytes of device memory the curled blocks of one find_lines call may use


def curve_strips(w, strips=None):
    """n_s of a curled block w pixels wide (DESIGN.md 7b, "Curled blocks"): ``strips``, or clamp(w // 48, 1, 32):
    strips 48 to 95 pixels wide, in which a line that climbs one pixel in five still rises less than the gap between lines."""
    return int(strips) if strips is not None else min(CURVE_MAX_STRIPS, max(1, w // 48))


def _curve_areas(h, n_s):
    """Byte sizes of one curled block's int32 areas: its work (histogram, profile, strip profiles, run counts), which the call
    zeroes, and its scratch (segmentation scratch of the block and of its strips, run table, link state)."""
    cap = _lib.CURVE_RUN_CAP
    return [4 * 256, 4 * 3 * h, 4 * 3 * n_s * h, 4 * n_s], [4 * (2 * h + 4), 4 * n_s * (2 * h + 4), 4 * 4 * cap * n_s, 4 * 7 * cap * n_s]


def curve_block_bytes(w, h, strips=None):
    """Device bytes of one curled block of w x h pixels in a find_lines_curved call: its records, work and scratch."""
    work, scratch = _curve_areas(h, curve_strips(w, strips))
    return sum(work + scratch) + sum(ctypes.sizeof(t) for t in (_lib.BlockLines, _lib.CurveLines, _lib.TextBlock, _lib.CurveBlock))


def curve_lines_dtype():
    """numpy view of an mn_curve_lines record (the link table of mn_find_lines_curved_u8)."""
    import numpy as np
    return np.dtype([("header", "<i4", (8,)), ("lines", "<i4", (_lib.BLOCK_MAX_LINES, _lib.CURVE_LINE_INTS))])


def find_lines_curved(blocks, tables=False):
    """Curled text blocks traced line by line across column strips, every block in seven launches whatever the number of blocks
    and strips (mn_find_lines_curved_u8; DESIGN.md 7b, "Curled blocks").  blocks: list of (img, rect, polarity, min_ink, gap,
    min_height, strips): as find_lines' horizontal blocks, strips a positive integer or None for the default (curve_strips), at
    most CURVE_MAX_STRIPS and each strip at least CURVE_MIN_STRIP pixels wide when there are several.  Returns the uint8 CUDA
    tensor of the n mn_block_lines records (the lines of curve=None) followed by the n mn_curve_lines records
    (``curve_lines_dtype()``).  ``tables`` (tests): also return per block dict(profiles, nruns, runs), int32 CUDA views of its strip
    profiles [n_s, 3, h], run counts [n_s] and run table [n_s, CURVE_RUN_CAP, 4].  Raises ValueError naming the block, before
    any launch, for a call whose blocks need more than CURVE_MAX_WORK bytes."""
    global LAUNCHES
    dev = _check_items(blocks, "find_lines_curved", "block")
    n = len(blocks)
    osz, csz = ctypes.sizeof(_lib.BlockLines), ctypes.sizeof(_lib.CurveLines)
    rsz, bsz = ctypes.sizeof(_lib.TextBlock), ctypes.sizeof(_lib.CurveBlock)
    dims, total = [], 0
    for i, blk in enumerate(blocks):
        what = f"find_lines_curved: block {i}"
        x0, y0, bw, bh = _check_crop((blk[0], blk[1], False, *blk[2:6]), dev, what, "min_ink / gap / min_height")
        strips = blk[6]
        n_s = curve_strips(bw, strips)
        if not 1 <= n_s <= CURVE_MAX_STRIPS or (n_s > 1 and bw // n_s < CURVE_MIN_STRIP):
            raise ValueError(f"{what}: {n_s} strips of a {bw}-pixel block: at most {CURVE_MAX_STRIPS}, each at least "
                             f"{CURVE_MIN_STRIP} pixels wide")
        total += curve_block_bytes(bw, bh, strips)
        if total > CURVE_MAX_WORK:
            raise ValueError(f"{what}: the blocks up to this one need {total} bytes, over the {CURVE_MAX_WORK} a call may use")
        dims.append((x0, y0, bw, bh, n_s))
    pack = _Pack()                  # results, link tables, line records, curve records; work (zeroed); scratch
    pack.area(n * osz)
    pack.area(n * csz)
    seg, crec = pack.area(n * rsz), pack.area(n * bsz)
    areas = [_curve_areas(d[3], d[4]) for d in dims]
    work = [[pack.area(a) for a in w] for w, _ in areas]
    w_end = pack.end
    scratch = [[pack.area(a) for a in s] for _, s in areas]
    base = pack.alloc(dev)
    recs, crecs, views, tiles = [], [], [], 0
    cap = _lib.CURVE_RUN_CAP
    for i, (blk, (x0, y0, bw, bh, n_s), (hist, prof, sprof, nruns), (scr, sscr, runs, link)) in \
            enumerate(zip(blocks, dims, work, scratch)):
        img, _, polarity, min_ink, gap, min_height, _ = blk
        tb = _lib.TextBlock(img.data_ptr(), img.stride(0), x0, y0, bw, bh, 0, polarity, min_ink or 0, gap or 0, min_height or 0,
                            0, base + hist, base + prof, base + scr, base + i * osz)
        recs.append(tb)
        crecs.append(_lib.CurveBlock(tb, base + sprof, base + nruns, base + runs, base + sscr, base + link,
                                     base + n * osz + i * csz, n_s))
        if tables:
            views.append(dict(profiles=pack.buf[sprof:sprof + 12 * n_s * bh].view(torch.int32).view(n_s, 3, bh),
                              nruns=pack.buf[nruns:nruns + 4 * n_s].view(torch.int32),
                              runs=pack.buf[runs:runs + 16 * cap * n_s].view(torch.int32).view(n_s, cap, 4)))
        tiles = max(tiles, -(-bw // 32) * -(-bh // 32))
    pack.upload((seg, bytes((_lib.TextBlock * n)(*recs))), (crec, bytes((_lib.CurveBlock * n)(*crecs))))
    _lib.check(_lib.load().mn_find_lines_curved_u8(base + seg, base + crec, n, tiles, max(d[4] for d in dims), base + work[0][0],
                                                   w_end - work[0][0], _stream()), "mn_find_lines_curved_u8")
    LAUNCHES += 7
    res = pack.buf[:n * (osz + csz)]
    return (res, views) if tables else res


PAGE_MAX_WORK = 1 << 30        # bytes of device memory one find_blocks call may use


class PageItem(NamedTuple):
    """One page of a find_blocks call (its docstring gives the fields' meaning)."""
    img: object
    rect: object
    vertical: bool
    polarity: int
    gap_x: object = None
    gap_y: object = None
    skew: object = None
    max_skew: float = 10.0
    rule_length: object = None
    figure_size: object = None
    directions: bool = False
    panel_size: object = None
    seal_size: object = None
    seal_lines: bool = False
    turns: bool = False


def page_cap(w, h):
    """Nodes one level of a w x h page may hold: disjoint rectangles with ink, pairwise apart by a white pixel, so at most
    (h + 1) (w + 1) / 4, and at most the node limit."""
    return min(_lib.PAGE_MAX_NODES, (h + 1) * (w + 1) // 4)


def rule_length(w, h):
    """The default rule length of a w x h page frame (DESIGN.md 7b, "Ruled pages"): max(32, min(w, h) // 16).  A heuristic: a
    glyph stroke at least this long counts as a rule."""
    return max(32, min(w, h) // 16)


def skew_page_frame(w, h, vertical, cs):
    """(L, M, stride) of a w x h page's frame bitmaps over the (c, s) of ``cs``: the most rows and columns a bitmap may have (the
    search frame's axes swapped for a vertical page) and the most bins of its search frames.  The one-entry table (1, 0) gives
    the crop's own (h, w) and its bins."""
    if cs == [(1.0, 0.0)]:
        return h, w, w if vertical else h
    _, _, L, M = skew_frames(w, h, vertical, cs)
    return (int(M.max()), int(L.max()), int(L.max())) if vertical else (int(L.max()), int(M.max()), int(L.max()))


def _page_areas(L, M, cap, n_ang, stride, rules, figures, panels):
    """Byte sizes of one page's work areas in find_blocks, in their order: the per-angle scores of a search (n_ang > 1), the
    histogram, the threshold record, the ink bitmap (L rows of ceil(M / 32) words), two level lists and three per-node counts
    of cap nodes, the angle profiles of a search, a ruled page's U plane (as the ink bitmap) and the transposed bitmap's
    scratch (M rows of ceil(L / 32) words), a figure page's F plane, and a panel page's U plane when it has no rules (the
    panels' outlines join the rules' plane when it has)."""
    plane, search = 4 * L * -(-M // 32), n_ang > 1
    return [8 * n_ang if search else 0, 4 * 256, ctypes.sizeof(_lib.BlockLines), plane, 2 * 12 * cap, 3 * 4 * cap,
            4 * n_ang * stride if search else 0, plane + 4 * M * -(-L // 32) if rules else 0, plane if figures else 0,
            plane if panels and not rules else 0]


def page_bytes(w, h, vertical=False, cs=None, rules=False, figures=False, panels=False, seals=False, seal_lines=False,
               turns=False):
    """Device bytes of one w x h page in find_blocks, with or without ``rules``, ``figures`` and ``panels``: its records,
    result and leaf table, a figure page's table of PAGE_MAX_FIGURES and a panel page's table of PAGE_MAX_PANELS page nodes,
    its work areas and 64 bytes for the call's 16-byte alignments.  ``cs``: None in a call without skewed pages, else the
    (c, s) table the page searches ([(1.0, 0.0)] for a page with skew None), which adds the search record, the table and 16
    bytes for its alignment; the page's bitmaps are then those of its largest frame.  ``seals``: with seal_bytes, and
    ``seal_lines`` with seal_line_bytes.  ``turns``: with its vote table of one mn_page_turn per leaf and 16 bytes for its
    alignment."""
    n_ang = len(cs) if cs else 1
    L, M, stride = skew_page_frame(w, h, vertical, cs or [(1.0, 0.0)])
    cap = page_cap(M, L)
    tables = 12 * (cap + (_lib.PAGE_MAX_FIGURES if figures else 0) + (_lib.PAGE_MAX_PANELS if panels else 0))
    search = ctypes.sizeof(_lib.SkewBlock) + 16 * n_ang + 16 if cs else 0
    return (ctypes.sizeof(_lib.PageResult) + ctypes.sizeof(_lib.TextBlock) + ctypes.sizeof(_lib.TextPage) + tables + search
            + sum(_page_areas(L, M, cap, n_ang, stride, rules, figures, panels)) + 64 + (seal_bytes(w, h) if seals else 0)
            + (seal_line_bytes() if seal_lines else 0) + (ctypes.sizeof(_lib.PageTurn) * cap + 16 if turns else 0))


def seal_line_bytes():
    """Device bytes a page with seal_lines adds to find_blocks (DESIGN.md 7b, "Seal centre lines"): its record and line table,
    with 16 bytes for each area's alignment.  The rows of the line search live in shared memory."""
    return ctypes.sizeof(_lib.CentrePage) + ctypes.sizeof(_lib.SealLineTable) + 2 * 16


def rule_page_bytes(w, h):
    """Device bytes a w x h page adds to find_blocks when it has rules (page_bytes): its U plane and the transposed bitmap's
    scratch."""
    return page_bytes(w, h, rules=True) - page_bytes(w, h)


def figure_page_bytes(w, h):
    """Device bytes a w x h page adds to find_blocks when it has figures (page_bytes): its F plane and figure table."""
    return page_bytes(w, h, figures=True) - page_bytes(w, h)


def panel_page_bytes(w, h, ruled):
    """Device bytes a w x h page adds to find_blocks when it has panels (page_bytes): its panel table, and the plane of U
    that takes the panels' outlines unless the page is ``ruled`` and has one."""
    return page_bytes(w, h, rules=ruled, panels=True) - page_bytes(w, h, rules=ruled)


def skew_page_bytes(w, h, vertical, cs):
    """Device bytes of one w x h page searched over ``cs`` in a find_blocks call with skewed pages (page_bytes)."""
    return page_bytes(w, h, vertical, cs)


def _check_page_options(page, what):
    """Refuses, naming ``what``, a PageItem's rule_length, figure_size or panel_size that is not None or an integer in
    [2, 32767] (figure_size and panel_size may be 0, their default) and its directions that is not None, False or True, or
    any of them set on a page with skew.  They are checked in their field order."""
    for knob, zero in (("rule_length", False), ("figure_size", True), ("directions", None), ("panel_size", True)):
        v = getattr(page, knob)
        if zero is None:                                # directions: a bool
            bad, want = (v is not None and not isinstance(v, bool)) or (v and page.skew is not None), "None, False or True"
        else:
            bad = v is not None and (isinstance(v, bool) or not isinstance(v, int) or not (zero and v == 0 or 2 <= v <= 32767)
                                     or page.skew is not None)
            want = f"{'0 or ' if zero else ''}an integer in [2, 32767]"
        if bad:
            raise ValueError(f"{what}: {knob} {v!r} is not {want} on a page with skew None")
    v = page.seal_size
    if v is not None and (isinstance(v, bool) or not isinstance(v, int) or not 8 <= v <= 4096 or page.skew is not None):
        raise ValueError(f"{what}: seal_size {v!r} is not an integer in [8, 4096] on a page with skew None")
    v = page.seal_lines
    if not isinstance(v, bool) or (v and page.seal_size is None):
        raise ValueError(f"{what}: seal_lines {v!r} is not False, or True on a page with a seal_size")
    v = page.turns
    if not isinstance(v, bool) or (v and (page.skew is not None or page.seal_size is not None or not page.directions)):
        raise ValueError(f"{what}: turns {v!r} is not False, or True on a page with directions, skew None and no seal_size")


def find_blocks(pages, scores=False):
    """Text pages split into blocks by a recursive XY-cut (mn_find_blocks_u8; DESIGN.md 7b, "Text pages"), every page of the call
    in 5 + 6 * 24 launches whatever the number of pages and nodes.  pages: list of PageItem records, or of tuples of their
    leading fields in order.  img: a uint8 [H, W, 3] CUDA view with dense pixels (any row stride) read in place.  rect:
    (x0, y0, x1, y1), a non-empty crop inside it with sides <= 32767.  vertical: a bool.  polarity: _lib.INK_AUTO / INK_DARK /
    INK_LIGHT.  gap_x, gap_y: positive integers, or None for the default.  Returns (out, caps): out the uint8 CUDA tensor of the pages' mn_page_result records followed by each
    page's leaf table of caps[i] mn_page_node entries; page_tables reads its host copy back.
    skew, max_skew (DESIGN.md 7b, "Skewed pages"): as find_lines'.  A call with any skewed page goes through
    mn_find_blocks_skewed_u8's 7 + 6 * 24 launches instead, every page of it; pages with skew None search the one-entry table
    (1, 0) and keep their tables exactly.  out then starts with the n mn_skew_block records (the chosen index and frame) and
    the leaves are in frame cells.  ``scores`` (tests): also return, per page, the int64 CUDA view of its per-angle scores
    (None unless it searched).
    rule_length (DESIGN.md 7b, "Ruled pages"): None, or an integer in [2, 32767] on a page with skew None, whose ink pixels in
    a maximal row or column run of at least that many pixels are its rules U.  A call with such a page issues 3 more launches
    whatever the number of pages; its records gain rule_pixels (|U|).
    figure_size (DESIGN.md 7b, "Figures"): None, or on a page with skew None 0 (the figure size 3 S) or an integer f in
    [2, 32767]: its pass-1 leaves whose shorter side is at least f are its figures, taken out of its ink before pass 2.  A call
    with such a page issues 1 more launch whatever the number of pages; its records gain figure_size and n_figures, and out
    ends with each such page's table of _lib.PAGE_MAX_FIGURES mn_page_node figures, in the order of the pages.
    directions (DESIGN.md 7b, "Mixed directions"): False (or None), or True on a page with skew None: each of its kept leaves
    has its own direction tested, _lib.PAGE_VERTICAL set in its st when it is vertical and _lib.PAGE_UNDECIDED when the test is
    undecided (it then takes the page's direction).  A call with such a page issues 1 more launch whatever the number of
    pages and needs no more memory.
    panel_size (DESIGN.md 7b, "Reversed panels"): None, or on a page with skew None 0 (the panel size S) or an integer p in
    [2, 32767]: its pass-1 leaves of shorter side at least p that are over half ink and flat-filled are its panels, whose
    insides are cut as ink of the other polarity inside a rule outline (with rule_length, after the rules U have left the
    ink: a fill with runs of at least rule_length is no panel).  A call with such a page issues 2 more launches whatever the
    number of pages; its records gain panel_size and n_panels, and out ends, after the figure tables, with each such page's
    table of _lib.PAGE_MAX_PANELS mn_page_node panels, in the order of the pages.
    seal_size (DESIGN.md 7b, "Seals"): None, or on a page with skew None an integer in [8, 4096]: the page's seals are found
    (mn_find_seals_u8's 6 launches for all such pages of the call, before the layout) and its layout runs on its layout copy,
    the crop with the seals' own ink set to paper.  out then starts with each such page's mn_seal_table, in the order of the
    pages (seal_tables reads them back).
    seal_lines (DESIGN.md 7b, "Seal centre lines"): False, or True on a page with a seal_size: each found seal's turn, arc band
    and centre lines are found (mn_find_seal_lines_u8's 1 launch for all such pages of the call, after mn_find_seals_u8).  out
    then has, after the seal tables, each such page's mn_seal_line_table, in the order of the pages (seal_line_tables reads
    them back).
    turns (DESIGN.md 7b, "Page turns"): False, or True on a page with directions (skew None, no seal_size): each kept leaf's
    bands along its direction give its vote entry (n_bands, e_lo, e_hi) in the page's table of caps[i] _lib.PageTurn records
    (1 more launch for all such pages of the call, after the direction launch).  The table lies in out at the first 16-byte
    boundary after the page's leaf table (page_tables reads it back).
    A page without one of these options gets the tables of a call without it."""
    global LAUNCHES
    dev = _check_items(pages, "find_blocks", "page")
    pages = [PageItem(*p) for p in pages]
    skewed = any(p.skew is not None for p in pages)
    n = len(pages)
    rsz, bsz, psz = (ctypes.sizeof(t) for t in (_lib.PageResult, _lib.TextBlock, _lib.TextPage))
    ssz = ctypes.sizeof(_lib.SkewBlock) if skewed else 0
    dims, tables, areas, need = [], [], [], 0
    for i, p in enumerate(pages):
        what = f"find_blocks: page {i}"
        x0, y0, bw, bh = _check_crop(p[:6], dev, what, "gap_x / gap_y")
        cs = _check_skew(p.skew, p.max_skew, p.vertical, what)
        _check_page_options(p, what)
        opts = (p.rule_length is not None, p.figure_size is not None, p.panel_size is not None)   # rules, figures, panels
        L, M, stride = skew_page_frame(bw, bh, p.vertical, cs)
        need += page_bytes(bw, bh, p.vertical, cs if skewed else None, *opts, seals=p.seal_size is not None,
                           seal_lines=p.seal_lines, turns=p.turns)
        if max(L, M) > 32767:
            raise ValueError(f"{what}: a frame side of {max(L, M)} exceeds 32767")
        if len(cs) > 1 and len(cs) * stride > SKEW_MAX_PROFILE:
            raise ValueError(f"{what}: {len(cs)} angles x {stride} bins exceed the {SKEW_MAX_PROFILE} profile values a skewed "
                             f"page may use")
        cap = page_cap(M, L)
        tables.append(cs)
        dims.append((x0, y0, bw, bh, cap, M, len(cs), stride, opts))
        areas.append(_page_areas(L, M, cap, len(cs), stride, *opts))
    if need > PAGE_MAX_WORK:
        raise ValueError(f"find_blocks: the pages need more than the {PAGE_MAX_WORK} bytes of work memory a call may use")
    tab, t_offs = _angle_tables(tables) if skewed else (b"", [0] * n)
    sealed = [i for i, p in enumerate(pages) if p.seal_size is not None]
    m, spsz, tsz = len(sealed), ctypes.sizeof(_lib.SealPage), ctypes.sizeof(_lib.SealTable)
    lined = [i for i in sealed if pages[i].seal_lines]
    ml, cpsz, lsz = len(lined), ctypes.sizeof(_lib.CentrePage), ctypes.sizeof(_lib.SealLineTable)
    pack = _Pack()                  # records, tables, the seal and line tables and the skew records, which come back with the
    pack.area(n * bsz)              # results in one copy; then the results, leaves, figure and panel tables and each page's
    pg, t_off = pack.area(n * psz), pack.area(len(tab))     # work, which the call zeroes; then the seal pages' cells and copies
    if sealed:
        sp = pack.area(m * spsz, 16)
        cp = pack.area(ml * cpsz, 16)
        pack.area(m * tsz, 16)
        pack.area(ml * lsz, 16)
    pack.area(n * ssz)
    out0 = pack.area(n * rsz, 16)
    sk0 = out0 - n * ssz            # the skew records end where the results begin, the line tables where they begin and the
    lt0 = sk0 - ml * lsz            # seal tables where those begin
    st0 = lt0 - m * tsz
    leaves = []
    for d, p in zip(dims, pages):                   # a turn page's vote table follows its leaves at the next 16-byte boundary
        leaves.append(pack.area(12 * d[4]))
        if p.turns:
            pack.area(ctypes.sizeof(_lib.PageTurn) * d[4], 16)
    figs = [pack.area(12 * _lib.PAGE_MAX_FIGURES) if d[8][1] else None for d in dims]
    pans = [pack.area(12 * _lib.PAGE_MAX_PANELS) if d[8][2] else None for d in dims]
    out1 = pack.end
    work = [[pack.area(a[0], 16)] + [pack.area(s) for s in a[1:]] for a in areas]
    w_end = pack.end
    scells = {i: [pack.area(a, 16) for a in _seal_areas(dims[i][2], dims[i][3])] for i in sealed}
    base = pack.alloc(dev)
    blocks, srecs, recs, views, tiles, seal_recs, centre_recs, stiles, ctiles = [], [], [], [], 0, [], [], 0, 0
    for i, (p, (x0, y0, bw, bh, cap, M, n_ang, stride, (rules, figures, panels)), wk, lv, f, pn, t) in \
            enumerate(zip(pages, dims, work, leaves, figs, pans, t_offs)):
        sc, hist, lines, bits, lists, counts, prof, rbits, fbits, pbits = (base + o for o in wk)
        src, pitch = p.img.data_ptr(), p.img.stride(0)
        if i in scells:             # the page's layout reads its copy through its own crop offsets
            copy, label, box, cand = (base + o for o in scells[i])
            seal_recs.append(_lib.SealPage(_lib.TextBlock(src, pitch, x0, y0, bw, bh), copy, label, box, cand,
                                           base + st0 + len(seal_recs) * tsz, p.seal_size))
            if p.seal_lines:
                centre_recs.append(_lib.CentrePage(seal_recs[-1].b, seal_recs[-1].out, base + lt0 + len(centre_recs) * lsz))
            src, pitch = (copy - y0 * 3 * bw - 3 * x0) % (1 << 64), 3 * bw
            stiles = max(stiles, -(-bw // 32) * -(-bh // 32))
            ctiles = max(ctiles, -(-bw // (4 * 32)) * -(-bh // (4 * 8)))
        tb = _lib.TextBlock(src, pitch, x0, y0, bw, bh, int(bool(p.vertical)), p.polarity, 0, 0, 0, 0, hist, 0, 0, lines)
        blocks.append(tb)
        if skewed:
            srecs.append(_skew_block(tb, base + t_off + 16 * t, sc, prof, n_ang, stride))
        recs.append(_lib.TextPage(tb, bits, (ctypes.c_void_p * 2)(lists, lists + 12 * cap), base + lv, counts, counts + 4 * cap,
                                  counts + 8 * cap, base + out0 + i * rsz, -(-M // 32), cap, p.gap_x or 0, p.gap_y or 0,
                                  rbits=rbits if rules else pbits if panels else None, rule_length=p.rule_length or 0,
                                  fbits=fbits if figures else None, figs=base + f if figures else None,
                                  figure_size=p.figure_size or 0,
                                  dirs=int(bool(p.directions)) | (_lib.PAGE_DIRS_TURN if p.turns else 0),
                                  pans=base + pn if panels else None, panel_size=p.panel_size or 0))
        views.append(pack.buf[wk[0]:wk[0] + 8 * n_ang].view(torch.int64) if n_ang > 1 else None)
        tiles = max(tiles, -(-bw // 32) * -(-bh // 32))
    buf = pack.upload((0, bytes((_lib.TextBlock * n)(*blocks))), (pg, bytes((_lib.TextPage * n)(*recs))), (t_off, tab),
                      *(((sp, bytes((_lib.SealPage * m)(*seal_recs))),) if sealed else ()),
                      *(((cp, bytes((_lib.CentrePage * ml)(*centre_recs))),) if lined else ()),
                      (sk0, bytes((_lib.SkewBlock * len(srecs))(*srecs))))
    if sealed:
        _lib.check(_lib.load().mn_find_seals_u8(base + sp, m, stiles, ctiles, base + st0, m * tsz, _stream()), "mn_find_seals_u8")
        LAUNCHES += 6
    if lined:
        _lib.check(_lib.load().mn_find_seal_lines_u8(base + cp, ml, _stream()), "mn_find_seal_lines_u8")
        LAUNCHES += 1
    ruled, figured, directed, paneled = (any(p.rule_length is not None for p in pages), any(f is not None for f in figs),
                                         any(p.directions for p in pages), any(pn is not None for pn in pans))
    turned = any(p.turns for p in pages)
    flags = ((_lib.PAGE_RULES if ruled else 0) | (_lib.PAGE_FIGURES if figured else 0) | (_lib.PAGE_DIRECTIONS if directed else 0)
             | (_lib.PAGE_PANELS if paneled else 0) | (_lib.PAGE_TURNS if turned else 0))
    entry, head = ("mn_find_blocks_skewed_u8", (base, base + sk0)) if skewed else ("mn_find_blocks_u8", (base,))
    w_bytes = (w_end if sealed else len(buf)) - out0
    _lib.check(getattr(_lib.load(), entry)(*head, base + pg, n, tiles, flags, base + out0, w_bytes, _stream()), entry)
    LAUNCHES += (7 if skewed else 5) + 6 * _lib.PAGE_LEVELS + 3 * ruled + figured + directed + 2 * paneled + turned
    res = buf[st0:out1], [d[4] for d in dims]
    return res + (views,) if scores else res


def page_tables(host, pages, caps):
    """Per page of a find_blocks call, numpy views of its tables in ``host``, the uint8 host copy of the call's out:
    (skew, res, leaves, figures, panels, turns).  skew is its mn_skew_block record (None in a call without skewed pages), res
    its mn_page_result record, and leaves, figures and panels its mn_page_node entries, as many as res counts; figures is None
    unless the page has a figure_size, panels None unless it has a panel_size.  turns is a turn page's mn_page_turn entries
    (page_turn_dtype()), one per leaf, else None."""
    sdt, rdt, ndt, tdt = skew_block_dtype(), page_result_dtype(), page_node_dtype(), page_turn_dtype()
    n = len(pages)
    host = host[ctypes.sizeof(_lib.SealTable) * sum(p.seal_size is not None for p in pages)
                + ctypes.sizeof(_lib.SealLineTable) * sum(p.seal_lines for p in pages):]
    o = n * sdt.itemsize if any(p.skew is not None for p in pages) else 0
    skews = host[:o].view(sdt) if o else [None] * n
    res = host[o:o + n * rdt.itemsize].view(rdt)
    host = host[o:]                                     # from the results on, 16-byte aligned as in the device buffer
    pos, tables = n * rdt.itemsize, []                  # every leaf table (and vote table), then the figure and panel tables
    for p, cap in zip(pages, caps):
        lv, pos, tv = pos, pos + 12 * cap, None
        if p.turns:
            t0 = -(-pos // 16) * 16
            tv, pos = host[t0:t0 + tdt.itemsize * cap].view(tdt), t0 + tdt.itemsize * cap
        tables.append((host[lv:lv + 12 * cap].view(ndt), tv))
    nodes = host[pos:].view(ndt)
    f = 0
    t = _lib.PAGE_MAX_FIGURES * sum(p.figure_size is not None for p in pages)
    out = []
    for p, sk, r, (lv, tv) in zip(pages, skews, res, tables):
        figs = pans = None
        if p.figure_size is not None:
            figs, f = nodes[f:f + _lib.PAGE_MAX_FIGURES][:int(r["n_figures"])], f + _lib.PAGE_MAX_FIGURES
        if p.panel_size is not None:
            pans, t = nodes[t:t + _lib.PAGE_MAX_PANELS][:int(r["n_panels"])], t + _lib.PAGE_MAX_PANELS
        out.append((sk, r, lv[:int(r["n_leaves"])], figs, pans, None if tv is None else tv[:int(r["n_leaves"])]))
    return out


def page_turn_dtype():
    """numpy view of an mn_page_turn record."""
    import numpy as np
    return np.dtype([("n_bands", "<i4"), ("pad", "<i4"), ("e_lo", "<i8"), ("e_hi", "<i8")])


def seal_tables(host, pages):
    """Per page of a find_blocks call, the numpy view of its mn_seal_table in ``host`` (seal_table_dtype()), or None for a page
    without seal_size."""
    tdt = seal_table_dtype()
    tabs = iter(host[:tdt.itemsize * sum(p.seal_size is not None for p in pages)].view(tdt))
    return [None if p.seal_size is None else next(tabs) for p in pages]


def seal_line_tables(host, pages):
    """Per page of a find_blocks call, the numpy view of its mn_seal_line_table in ``host`` (seal_line_table_dtype()), or None
    for a page without seal_lines."""
    ldt, o = seal_line_table_dtype(), ctypes.sizeof(_lib.SealTable) * sum(p.seal_size is not None for p in pages)
    tabs = iter(host[o:o + ldt.itemsize * sum(p.seal_lines for p in pages)].view(ldt))
    return [next(tabs) if p.seal_lines else None for p in pages]


def seal_line_table_dtype():
    """numpy view of an mn_seal_line_table record."""
    import numpy as np
    rec = np.dtype([(f, "<i4") for f, _ in _lib.SealLines._fields_[:-2]] + [("pad", "<i4", (2,)),
                                                                            ("box", "<i4", (_lib.SEAL_MAX_LINES, 4))])
    return np.dtype([("seal", rec, (_lib.PAGE_MAX_SEALS,))])


def seal_table_dtype():
    """numpy view of an mn_seal_table record."""
    import numpy as np
    seal = np.dtype([(f, "<i4") for f, _ in _lib.Seal._fields_[:-1]] + [("pad", "<i4", (3,))])
    return np.dtype([("error", "<i4"), ("n_cand", "<i4"), ("n_seals", "<i4"), ("pad", "<i4"),
                     ("seal", seal, (_lib.PAGE_MAX_SEALS,))])


def page_result_dtype():
    """numpy view of an mn_page_result record."""
    import numpy as np
    return np.dtype([(f, "<i4") for f, _ in _lib.PageResult._fields_])


def page_node_dtype():
    """numpy view of an mn_page_node record (x0, y0, x1, y1 in the page's crop, st)."""
    import numpy as np
    return np.dtype([("x0", "<i2"), ("y0", "<i2"), ("x1", "<i2"), ("y1", "<i2"), ("st", "<i4")])


def _quad_areas(w, h):
    """Byte sizes of one w x h image's areas in find_page_quads: histogram, threshold record, page key, row extents (2 h),
    labels and counts (h w each) and the hull stack (4 h + 8 points), each rounded to 16 bytes."""
    sizes = (4 * 256, ctypes.sizeof(_lib.BlockLines), 8, 8 * h, 4 * h * w, 4 * h * w, 8 * (4 * h + 8))
    return [-(-s // 16) * 16 for s in sizes]


def quad_page_bytes(w, h):
    """Device bytes of one w x h image in find_page_quads: its records, its result and its areas."""
    return (ctypes.sizeof(_lib.TextBlock) + ctypes.sizeof(_lib.QuadPage) + ctypes.sizeof(_lib.PageQuad) + 32
            + sum(_quad_areas(w, h)))


def spine_page_bytes(w):
    """Device bytes of one w pixels wide spread in find_page_quads beyond its image's (DESIGN.md 7b, "Book spreads"): its record,
    its result and its column extents (2 w int32)."""
    return ctypes.sizeof(_lib.SpinePage) + ctypes.sizeof(_lib.PageSpine) + 32 + -(-8 * w // 16) * 16


def find_page_quads(pages, hulls=False, labels=False, spreads=()):
    """Page corners (mn_find_page_quads_u8; DESIGN.md 7b, "Perspective pages"), every image of the call in 8 launches whatever
    their number.  pages: list of (img, polarity): img a uint8 [H, W, 3] CUDA view with dense pixels (any row stride), H, W <=
    32767, read in place whole; polarity _lib.INK_AUTO / INK_DARK / INK_LIGHT (paper is grey <= t for INK_LIGHT, else grey > t).
    Returns the uint8 CUDA tensor of the pages' mn_page_quad records, in order (read it back as ``page_quad_dtype()``).
    ``spreads`` (DESIGN.md 7b, "Book spreads"): the indices of the pages whose spine is searched too, on their component and
    corners, by mn_find_page_spines_u8's 2 more launches whatever their number; the call then returns (quads, spines), spines
    the uint8 CUDA tensor of their mn_page_spine records in the order given (``page_spine_dtype()``), in a table of its own
    after the quads'.  Without spreads the call is exactly the one before: no spine memory and no more launches.
    ``hulls`` (tests): also return, per page, the int32 [4 H + 8, 2] CUDA view of its hull stack, whose first n_hull rows are
    the hull.  ``labels`` (tests): also return, per page, the int32 CUDA views of its compressed labels [H, W] (each paper pixel's
    component root, the smallest raster index y W + x of the component; -1 elsewhere) and pixel counts [H W] (a component's
    size at its root, 0 elsewhere)."""
    global LAUNCHES
    dev = _check_items(pages, "find_page_quads", "page")
    n = len(pages)
    spreads = [int(k) for k in spreads]
    if any(not 0 <= k < n for k in spreads) or len(set(spreads)) != len(spreads):
        raise ValueError(f"find_page_quads: spreads must be distinct page indices in [0, {n}), got {spreads!r}")
    m = len(spreads)
    bsz, psz, rsz = (ctypes.sizeof(t) for t in (_lib.TextBlock, _lib.QuadPage, _lib.PageQuad))
    ssz, spsz = ctypes.sizeof(_lib.SpinePage), ctypes.sizeof(_lib.PageSpine)
    for i, (img, polarity) in enumerate(pages):
        _check_crop((img, (0, 0, img.shape[1], img.shape[0]), False, polarity), dev, f"find_page_quads: page {i}", "")
    if (sum(quad_page_bytes(img.shape[1], img.shape[0]) for img, _ in pages)
            + sum(spine_page_bytes(pages[k][0].shape[1]) for k in spreads) > PAGE_MAX_WORK):
        raise ValueError(f"find_page_quads: the pages need more than the {PAGE_MAX_WORK} bytes of work memory a call may use")
    pack = _Pack()                  # records; then the results and the work, which the call zeroes
    pack.area(n * bsz)
    qp, sp = pack.area(n * psz), pack.area(m * ssz)
    out0, sres = pack.area(n * rsz, 16), pack.area(m * spsz)
    work = [[pack.area(s, 16) for s in _quad_areas(img.shape[1], img.shape[0])] for img, _ in pages]
    cols = [pack.area(8 * pages[k][0].shape[1], 16) for k in spreads]
    base = pack.alloc(dev)
    blocks, recs, views, lviews, tiles = [], [], [], [], 0
    for i, ((img, polarity), (hist, lines, best, ext, label, count, hull)) in enumerate(zip(pages, work)):
        h_, w_ = img.shape[:2]
        tb = _lib.TextBlock(img.data_ptr(), img.stride(0), 0, 0, w_, h_, 0, polarity, 0, 0, 0, 0, base + hist, 0, 0, base + lines)
        blocks.append(tb)
        recs.append(_lib.QuadPage(tb, base + label, base + count, base + ext, base + best, base + hull, base + out0 + i * rsz))
        views.append(pack.buf[hull:hull + 8 * (4 * h_ + 8)].view(torch.int32).view(-1, 2))
        lviews.append((pack.buf[label:label + 4 * h_ * w_].view(torch.int32).view(h_, w_),
                       pack.buf[count:count + 4 * h_ * w_].view(torch.int32)))
        tiles = max(tiles, -(-w_ // 32) * -(-h_ // 32))
    spines = [_lib.SpinePage(base + qp + k * psz, base + c, base + sres + j * spsz) for j, (k, c) in enumerate(zip(spreads, cols))]
    buf = pack.upload((0, bytes((_lib.TextBlock * n)(*blocks))), (qp, bytes((_lib.QuadPage * n)(*recs))),
                      (sp, bytes((_lib.SpinePage * m)(*spines))))
    _lib.check(_lib.load().mn_find_page_quads_u8(base, base + qp, n, tiles, base + out0, len(buf) - out0, _stream()),
               "mn_find_page_quads_u8")
    LAUNCHES += 8
    res = buf[out0:out0 + n * rsz]
    if spreads:
        stiles = max(-(-pages[k][0].shape[1] // 32) * -(-pages[k][0].shape[0] // 32) for k in spreads)
        _lib.check(_lib.load().mn_find_page_spines_u8(base + sp, m, stiles, _stream()), "mn_find_page_spines_u8")
        LAUNCHES += 2
        res = (res, buf[sres:sres + m * spsz])
    else:
        res = (res,)
    out = res + ((views,) if hulls else ()) + ((lviews,) if labels else ())
    return out if len(out) > 1 else res[0]


def page_quad_dtype():
    """numpy view of an mn_page_quad record."""
    import numpy as np
    return np.dtype([("threshold", "<i4"), ("label", "<i4"), ("size", "<i4"), ("n_hull", "<i4"), ("area2", "<i8"),
                     ("idx", "<i4", (4,)), ("quad", "<i4", (8,))])


def page_spine_dtype():
    """numpy view of an mn_page_spine record."""
    import numpy as np
    return np.dtype([("found", "<i4"), ("st", "<i4", (2,)), ("sb", "<i4", (2,)), ("pad", "<i4"), ("D", "<i8"), ("E", "<i8")])


def vertical_unlayout(items):
    """Restored lines put back into columns, every column in one launch (mn_vertical_unlayout_u8_batched; DESIGN.md 7b,
    "Vertical text columns").  items: list of (T, T_col, cells): uint8 [128, W_T, 3] and [H_c, W_c, 3] CUDA views with dense
    pixels (T read in place through its pitch), cells the n (R(c_k), R(p_k), R(p_k + t_k), R(k w_r), min(R((k+1) w_r), W_T)) of
    pipeline.unlayout_cells.  Row i of T_col belongs to the last cell k with R(c_k) <= i and reads T at row
    clamp(R(p_k) + i - R(c_k), R(p_k), R(p_k + t_k) - 1), column clamp(R(k w_r) + j, R(k w_r), min(R((k+1) w_r), W_T) - 1)."""
    _vertical_gather(items, "vertical_unlayout", 5, "mn_vertical_unlayout_u8_batched")
