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


def _table(ctype, records, device):
    """Host-built array of C records -> device byte tensor (the kernels read their descriptors from device memory)."""
    import numpy as np
    arr = (ctype * len(records))(*records)
    return torch.from_numpy(np.frombuffer(bytes(arr), dtype=np.uint8).copy()).to(device)


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
    table = _table(_lib.LqCrop, recs, dev)
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
    table = _table(_lib.SrPiece, recs, sr.device)
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
    if not items:
        raise ValueError("figure_panels: no images")
    if len(items) > 65535:
        raise ValueError("figure_panels: at most 65535 images per launch")
    dev = items[0][1].device
    n_prior = sum(len(it[4]) for it in items)
    n_marks = sum(len(it[2]) + len(it[3]) for it in items)
    isz, psz = ctypes.sizeof(_lib.FigureImage), ctypes.sizeof(_lib.FigurePrior)
    buf = torch.empty(len(items) * isz + n_prior * psz + 8 * max(1, n_marks), dtype=torch.uint8, device=dev)
    base = buf.data_ptr()
    p_off, m_off = len(items) * isz, len(items) * isz + n_prior * psz
    recs, prs, marks, mx = [], [], [], 0
    for i, (img, fig, top, bot, priors) in enumerate(items):
        for name, t in (("img", img), ("fig", fig)):
            if not isinstance(t, torch.Tensor) or t.device != dev or t.dtype != torch.uint8 or t.dim() != 3 or t.shape[2] != 3 \
                    or t.stride(2) != 1 or t.stride(1) != 3 or t.stride(0) < 3 * t.shape[1]:
                raise RuntimeError(f"figure_panels: image {i}: {name} must be a uint8 [., ., 3] tensor with dense pixels on {dev}")
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
    host = bytes((_lib.FigureImage * len(recs))(*recs)) + bytes((_lib.FigurePrior * len(prs))(*prs)) + \
        np.asarray(marks or [(0, 0)], dtype=np.int32).tobytes()
    buf.copy_(torch.frombuffer(bytearray(host), dtype=torch.uint8))
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
    return _table(_lib.PredRow, recs, device), out


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
    if not items:
        raise ValueError("resize_cubic: no images")
    if len(items) > 65535:
        raise ValueError("resize_cubic: at most 65535 images per launch")
    dev = items[0][0].device
    cn = items[0][0].shape[2] if isinstance(items[0][0], torch.Tensor) and items[0][0].dim() == 3 else 3
    if not 1 <= cn <= 4:
        raise RuntimeError(f"resize_cubic: {cn} channels (1 to 4)")
    recs, mx = [], 0
    for i, (src, dst) in enumerate(items):
        _dense_u8(src, dev, cn, f"resize_cubic: image {i}: src")
        _dense_u8(dst, dev, cn, f"resize_cubic: image {i}: dst")
        (h, w), (dh, dw) = src.shape[:2], dst.shape[:2]
        recs.append(_lib.ResizeImage(src.data_ptr(), src.stride(0), h, w, dst.data_ptr(), dst.stride(0), dh, dw,
                                     1.0 / (dw / w), 1.0 / (dh / h)))
        mx = max(mx, dh * dw)
    table = _table(_lib.ResizeImage, recs, dev)
    _lib.check(_lib.load().mn_resize_cubic_u8_batched(_ptr(table), len(recs), cn, mx, _stream()), "mn_resize_cubic_u8_batched")
    LAUNCHES += 1


def _region_records(regions, feather, what, record, extra=0):
    """Validated mn_region records of composite_regions' (page, sr, rect, chain, ...) tuples, their chains, the largest rectangle's
    pixel count and a device buffer for the ``record``-type table followed by the chains (and ``extra`` bytes after them)."""
    if not regions:
        raise ValueError(f"{what}: no regions")
    if len(regions) > 65535:
        raise ValueError(f"{what}: at most 65535 regions per launch")
    if feather < 0:
        raise ValueError(f"{what}: feather {feather} < 0")
    dev = regions[0][0].device
    n_chain = sum(len(r[3]) for r in regions)
    isz = ctypes.sizeof(record)
    buf = torch.empty(len(regions) * isz + 4 * max(1, n_chain) + extra, dtype=torch.uint8, device=dev)
    c_base = buf.data_ptr() + len(regions) * isz
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
    return recs, chains, mx, buf


def _upload_records(buf, recs, chains):
    import numpy as np
    host = bytes((type(recs[0]) * len(recs))(*recs)) + np.asarray(chains or [0], dtype=np.int32).tobytes()
    buf.copy_(torch.frombuffer(bytearray(host), dtype=torch.uint8))


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
    recs, chains, mx, buf = _region_records(regions, int(feather), "composite_regions", _lib.Region)
    _upload_records(buf, recs, chains)
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
    if not items:
        raise ValueError(f"{what}: no images")
    if len(items) > 65535:
        raise ValueError(f"{what}: at most 65535 images per launch")
    dev = items[0][0].device
    cn = items[0][0].shape[2] if isinstance(items[0][0], torch.Tensor) and items[0][0].dim() == 3 else 3
    if not 1 <= cn <= 4:
        raise RuntimeError(f"{what}: {cn} channels (1 to 4)")
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
    table = _table(record, recs, dev)
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
    recs, chains, mx, buf = _region_records(regions, int(feather), "composite_regions_affine", _lib.RegionAffine)
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
    _upload_records(buf, out, chains)
    _lib.check(_lib.load().mn_composite_regions_affine_u8(_ptr(buf), len(out), mx, _stream()), "mn_composite_regions_affine_u8")
    LAUNCHES += 1


def composite_regions_quad(regions, feather):
    """composite_regions_affine for pages that also hold perspective regions (mn_composite_regions_quad_u8; DESIGN.md 7b,
    "Perspective text regions"), one launch.  regions: list of (page, sr, rect, chain, maps) as composite_regions_affine takes
    them; maps may also be (N, kx, ky) with N 3 x 3 (fp64): a perspective region whose page map is homogeneous, with a positive
    denominator over rect, the bounding box of its footprint in page pixels (pipeline.quad_maps).  The footprint test is the
    affine one on its fixed-point sr coordinates."""
    global LAUNCHES
    recs, chains, mx, buf = _region_records(regions, int(feather), "composite_regions_quad", _lib.RegionQuad)
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
    _upload_records(buf, out, chains)
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


def _align8(n):
    return (n + 7) & ~7


def remap_curved(items):
    """Curved text regions rectified, every crop in one launch (mn_remap_curved_u8_batched; DESIGN.md 7b, "Curved text regions"):
    cv2.remap(src, mapx, mapy, INTER_CUBIC, borderMode=BORDER_REPLICATE) with the fp32 crop maps of each region's curves, OpenCV's
    own 8-bit path (IPP off).  items: list of (src, dst, curve): uint8 [h, w, cn] and [h_r, w_r, cn] CUDA views with dense pixels
    (any row stride), h, w <= 32767, and curve a CurveTable whose crop map stays below 2^14 pixels in magnitude
    (pipeline.plan_regions keeps it so).  The curve tables go up with the records in one copy."""
    import numpy as np
    global LAUNCHES
    if not items:
        raise ValueError("remap_curved: no images")
    if len(items) > 65535:
        raise ValueError("remap_curved: at most 65535 images per launch")
    dev = items[0][0].device
    cn = items[0][0].shape[2] if isinstance(items[0][0], torch.Tensor) and items[0][0].dim() == 3 else 3
    if not 1 <= cn <= 4:
        raise RuntimeError(f"remap_curved: {cn} channels (1 to 4)")
    tables = []
    for i, (src, dst, curve) in enumerate(items):
        _dense_u8(src, dev, cn, f"remap_curved: image {i}: src")
        _dense_u8(dst, dev, cn, f"remap_curved: image {i}: dst")
        if max(src.shape[:2]) > 32767:
            raise ValueError(f"remap_curved: image {i}: a {src.shape[0]}x{src.shape[1]} source exceeds OpenCV's int16 source "
                             f"coordinates")
        tables.append(curve.values(f"remap_curved: image {i}"))
    isz = ctypes.sizeof(_lib.RemapCurvedImage)
    n_tab = sum(t.size for t, _ in tables)
    buf = torch.empty(len(items) * isz + 8 * n_tab, dtype=torch.uint8, device=dev)
    base, o, recs, mx = buf.data_ptr() + len(items) * isz, 0, [], 0
    for (src, dst, _), (t, k) in zip(items, tables):
        (h, w), (dh, dw) = src.shape[:2], dst.shape[:2]
        recs.append(_lib.RemapCurvedImage(src.data_ptr(), src.stride(0), h, w, dst.data_ptr(), dst.stride(0), dh, dw, base + 8 * o,
                                          k, 0))
        o += t.size
        mx = max(mx, dh * dw)
    host = bytes((_lib.RemapCurvedImage * len(recs))(*recs)) + np.concatenate([t for t, _ in tables]).tobytes()
    buf.copy_(torch.frombuffer(bytearray(host), dtype=torch.uint8))
    _lib.check(_lib.load().mn_remap_curved_u8_batched(_ptr(buf), len(recs), cn, mx, _stream()), "mn_remap_curved_u8_batched")
    LAUNCHES += 1


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
    n_tab = sum(t.size for t, _ in tables.values())
    recs, chains, mx, buf = _region_records(regions, int(feather), "composite_regions_curved", _lib.RegionCurved,
                                            extra=8 + 8 * n_tab)
    isz = ctypes.sizeof(_lib.RegionCurved)
    head = len(regions) * isz + 4 * max(1, len(chains))
    t_off = _align8(buf.data_ptr() + head) - buf.data_ptr()
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
                                         buf.data_ptr() + t_off + 8 * o, k, 0))
            o += t.size
            continue
        n = [float(v) for row in n for v in row]
        if len(n) not in (6, 9):
            raise ValueError(f"composite_regions_curved: region {i}: expected (N 2 x 3 or 3 x 3, kx, ky) or (CurveTable, kx, ky)")
        kind = _lib.REGION_AFFINE if len(n) == 6 else _lib.REGION_PERSPECTIVE
        out.append(_lib.RegionCurved(_lib.RegionQuad(rec, kind, kx, ky, 0, (ctypes.c_double * 9)(*n)), None, 0, 0))
    host = bytes((_lib.RegionCurved * len(out))(*out)) + np.asarray(chains or [0], dtype=np.int32).tobytes()
    host += bytes(t_off - head)
    if tables:
        host += np.concatenate([tables[i][0] for i in sorted(tables)]).tobytes()
    buf[:len(host)].copy_(torch.frombuffer(bytearray(host), dtype=torch.uint8))
    _lib.check(_lib.load().mn_composite_regions_curved_u8(_ptr(buf), len(out), mx, _stream()), "mn_composite_regions_curved_u8")
    LAUNCHES += 1


def _vertical_gather(items, what, width, symbol):
    """One launch of ``symbol`` over vertical_layout's / vertical_unlayout's items, ``width`` int32 values per cell."""
    import numpy as np
    global LAUNCHES
    if not items:
        raise ValueError(f"{what}: no columns")
    if len(items) > 65535:
        raise ValueError(f"{what}: at most 65535 columns per launch")
    dev = items[0][0].device
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
    isz = ctypes.sizeof(_lib.VerticalColumn)
    n_int = sum(t.size for t in tables)
    buf = torch.empty(len(items) * isz + 4 * n_int, dtype=torch.uint8, device=dev)
    base, o, recs, mx = buf.data_ptr() + len(items) * isz, 0, [], 0
    for (src, dst, _), t in zip(items, tables):
        dh, dw = dst.shape[:2]
        recs.append(_lib.VerticalColumn(src.data_ptr(), src.stride(0), dst.data_ptr(), dst.stride(0), base + 4 * o, dh, dw, len(t),
                                        dw // len(t) if width == 3 else 0))
        o += t.size
        mx = max(mx, dh * dw)
    host = bytes((_lib.VerticalColumn * len(recs))(*recs)) + b"".join(t.tobytes() for t in tables)
    buf.copy_(torch.frombuffer(bytearray(host), dtype=torch.uint8))
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


def skew_block_dtype():
    """numpy view of an mn_skew_block record after mn_find_lines_skewed_u8: the chosen index and frame."""
    import numpy as np
    return np.dtype([("b", np.uint8, ctypes.sizeof(_lib.TextBlock)), ("table", "<u8"), ("scores", "<u8"), ("profiles", "<u8"),
                     ("n_ang", "<i4"), ("stride", "<i4"), ("chosen", "<i4"), ("L", "<i4"), ("M", "<i4"), ("pad", "<i4"),
                     ("u_min", "<f8"), ("v_min", "<f8"), ("c", "<f8"), ("s", "<f8")])


def find_lines(blocks, scores=False):
    """Text blocks split into lines, every block in four launches whatever their number (mn_find_lines_u8; DESIGN.md 7b, "Text
    blocks").  blocks: list of (img, rect, vertical, polarity, min_ink, gap, min_height[, skew, max_skew]): img a uint8 [H, W, 3]
    CUDA view with dense pixels (any row stride) read in place, rect (x0, y0, x1, y1) a non-empty crop inside it with sides
    <= 32767, vertical a bool, polarity _lib.INK_AUTO / INK_DARK / INK_LIGHT, and min_ink, gap, min_height positive integers or
    None for the default.  Returns the uint8 CUDA tensor of the blocks' mn_block_lines records, in order (read it back as
    ``block_lines_dtype()``).
    skew (DESIGN.md 7b, "Skewed blocks"): None, "auto" (search +-max_skew degrees) or a given angle in degrees, |skew| < 45.  A
    call with any skewed block goes through mn_find_lines_skewed_u8's six launches instead, every block of it, whatever their
    number; blocks with skew None keep their mn_block_lines records exactly.  The tensor then holds the n mn_block_lines records
    followed by the n mn_skew_block records (``skew_block_dtype()``: the chosen index and frame).  ``scores`` (tests): also
    return, per block, the int64 CUDA view of its per-angle scores (None unless it searched)."""
    import numpy as np
    global LAUNCHES
    if not blocks:
        raise ValueError("find_lines: no blocks")
    if len(blocks) > 65535:
        raise ValueError("find_lines: at most 65535 blocks per launch")
    if any(len(b) > 7 and b[7] is not None for b in blocks):
        return _find_lines_skewed(blocks, scores)
    blocks = [b[:7] for b in blocks]
    dev = blocks[0][0].device
    osz, rsz = ctypes.sizeof(_lib.BlockLines), ctypes.sizeof(_lib.TextBlock)
    dims = []
    for i, (img, rect, vertical, polarity, *knobs) in enumerate(blocks):
        _dense_u8(img, dev, 3, f"find_lines: block {i}: img")
        x0, y0, x1, y1 = (int(v) for v in rect)
        if not (0 <= x0 < x1 <= img.shape[1] and 0 <= y0 < y1 <= img.shape[0]) or max(x1 - x0, y1 - y0) > 32767:
            raise ValueError(f"find_lines: block {i}: rectangle {(x0, y0, x1, y1)} is empty, outside the "
                             f"{img.shape[1]}x{img.shape[0]} image or has a side over 32767")
        if polarity not in (_lib.INK_AUTO, _lib.INK_DARK, _lib.INK_LIGHT) or \
                any(v is not None and not 1 <= v < 2 ** 31 for v in knobs):
            raise ValueError(f"find_lines: block {i}: bad polarity {polarity!r} or min_ink / gap / min_height {knobs!r}")
        dims.append((x0, y0, x1 - x0, y1 - y0, y1 - y0 if not vertical else x1 - x0))
    n_work = sum(256 + 3 * d[4] for d in dims)
    n_scratch = sum(2 * d[4] + 4 for d in dims)
    head = len(blocks) * (osz + rsz)
    buf = torch.empty(head + 4 * (n_work + n_scratch), dtype=torch.uint8, device=dev)
    out, work = buf.data_ptr(), buf.data_ptr() + head
    scratch, w, s, recs, tiles = work + 4 * n_work, 0, 0, [], 0
    for i, ((img, _, vertical, polarity, min_ink, gap, min_height), (x0, y0, bw, bh, L)) in enumerate(zip(blocks, dims)):
        recs.append(_lib.TextBlock(img.data_ptr(), img.stride(0), x0, y0, bw, bh, int(bool(vertical)), polarity, min_ink or 0,
                                   gap or 0, min_height or 0, 0, work + 4 * w, work + 4 * (w + 256), scratch + 4 * s, out + i * osz))
        w += 256 + 3 * L
        s += 2 * L + 4
        tiles = max(tiles, -(-bw // 32) * -(-bh // 32))
    rec = buf[len(blocks) * osz:head]
    rec.copy_(torch.from_numpy(np.frombuffer(bytes((_lib.TextBlock * len(recs))(*recs)), dtype=np.uint8).copy()))
    _lib.check(_lib.load().mn_find_lines_u8(_ptr(rec), len(recs), tiles, work, 4 * n_work, _stream()), "mn_find_lines_u8")
    LAUNCHES += 4
    out = buf[:len(blocks) * osz]
    return (out, [None] * len(blocks)) if scores else out


def _find_lines_skewed(blocks, want_scores):
    """find_lines for a call that holds a skewed block: mn_find_lines_skewed_u8 over every block.  A block without skew searches
    the one-entry table (1, 0), which leaves its crop record and so its mn_block_lines record as mn_find_lines_u8 writes it."""
    import numpy as np
    global LAUNCHES
    dev = blocks[0][0].device
    n = len(blocks)
    osz, ssz, rsz = ctypes.sizeof(_lib.BlockLines), ctypes.sizeof(_lib.SkewBlock), ctypes.sizeof(_lib.TextBlock)
    dims, tables, keys = [], [], {}
    for i, blk in enumerate(blocks):
        img, rect, vertical, polarity, *knobs = blk[:7]
        skew, max_skew = blk[7] if len(blk) > 7 else None, blk[8] if len(blk) > 8 else 10.0
        _dense_u8(img, dev, 3, f"find_lines: block {i}: img")
        x0, y0, x1, y1 = (int(v) for v in rect)
        if not (0 <= x0 < x1 <= img.shape[1] and 0 <= y0 < y1 <= img.shape[0]) or max(x1 - x0, y1 - y0) > 32767:
            raise ValueError(f"find_lines: block {i}: rectangle {(x0, y0, x1, y1)} is empty, outside the "
                             f"{img.shape[1]}x{img.shape[0]} image or has a side over 32767")
        if polarity not in (_lib.INK_AUTO, _lib.INK_DARK, _lib.INK_LIGHT) or \
                any(v is not None and not 1 <= v < 2 ** 31 for v in knobs):
            raise ValueError(f"find_lines: block {i}: bad polarity {polarity!r} or min_ink / gap / min_height {knobs!r}")
        if skew is None:
            cs = [(1.0, 0.0)]
        elif skew == "auto" if isinstance(skew, str) else math.isfinite(skew) and abs(skew) < 45:
            if not (isinstance(skew, str) or max_skew == 10.0) or not 0 < max_skew <= 20:
                raise ValueError(f"find_lines: block {i}: max_skew {max_skew!r} is outside (0, 20] or given without 'auto'")
            cs = skew_cos_sin(skew_table(skew, max_skew, vertical))
        else:
            raise ValueError(f"find_lines: block {i}: bad skew {skew!r}")
        stride = skew_stride(x1 - x0, y1 - y0, vertical, cs)
        if len(cs) > 1 and len(cs) * stride > SKEW_MAX_PROFILE:
            raise ValueError(f"find_lines: block {i}: {len(cs)} angles x {stride} bins exceed the {SKEW_MAX_PROFILE} profile "
                             f"values a skewed block may use")
        key = tuple(cs)
        if key not in keys:
            keys[key] = sum(len(t) for t in tables)
            tables.append(cs)
        dims.append((x0, y0, x1 - x0, y1 - y0, len(cs), stride, keys[key]))
    n_tab = sum(len(t) for t in tables)
    n_scores = sum(d[4] for d in dims if d[4] > 1)
    n_work = sum(256 + 3 * d[5] + (d[4] * d[5] if d[4] > 1 else 0) for d in dims)
    n_scratch = sum(2 * d[5] + 4 for d in dims)
    head = n * (osz + ssz + rsz) + 16 * n_tab
    buf = torch.empty(head + 8 * n_scores + 4 * (n_work + n_scratch), dtype=torch.uint8, device=dev)
    out, sk, seg = buf.data_ptr(), buf.data_ptr() + n * osz, buf.data_ptr() + n * (osz + ssz)
    tab, work = seg + n * rsz, buf.data_ptr() + head
    w32, scratch = work + 8 * n_scores, work + 8 * n_scores + 4 * n_work
    recs, srecs, views, w, s, o, tiles = [], [], [], 0, 0, 0, 0
    for i, (blk, (x0, y0, bw, bh, n_ang, stride, t)) in enumerate(zip(blocks, dims)):
        img, _, vertical, polarity, min_ink, gap, min_height = blk[:7]
        prof = w32 + 4 * (w + 256)
        tb = _lib.TextBlock(img.data_ptr(), img.stride(0), x0, y0, bw, bh, int(bool(vertical)), polarity, min_ink or 0, gap or 0,
                            min_height or 0, 0, w32 + 4 * w, prof, scratch + 4 * s, out + i * osz)
        recs.append(tb)
        srecs.append(_lib.SkewBlock(tb, tab + 16 * t, work + 8 * o if n_ang > 1 else 0, prof + 4 * 3 * stride if n_ang > 1 else 0,
                                    n_ang, stride, 0, 0, 0, 0, 0.0, 0.0, 0.0, 0.0))
        views.append(buf[head + 8 * o:head + 8 * (o + n_ang)].view(torch.int64) if n_ang > 1 else None)
        o += n_ang if n_ang > 1 else 0
        w += 256 + 3 * stride + (n_ang * stride if n_ang > 1 else 0)
        s += 2 * stride + 4
        tiles = max(tiles, -(-bw // 32) * -(-bh // 32))
    host = bytes((_lib.SkewBlock * n)(*srecs)) + bytes((_lib.TextBlock * n)(*recs)) + \
        np.array([v for t in tables for p in t for v in p], np.float64).tobytes()
    buf[n * osz:head].copy_(torch.from_numpy(np.frombuffer(host, dtype=np.uint8).copy()))
    _lib.check(_lib.load().mn_find_lines_skewed_u8(ctypes.c_void_p(seg), ctypes.c_void_p(sk), n, tiles, work,
                                                   8 * n_scores + 4 * n_work, _stream()), "mn_find_lines_skewed_u8")
    LAUNCHES += 6
    res = buf[:n * (osz + ssz)]
    return (res, views) if want_scores else res


def vertical_unlayout(items):
    """Restored lines put back into columns, every column in one launch (mn_vertical_unlayout_u8_batched; DESIGN.md 7b,
    "Vertical text columns").  items: list of (T, T_col, cells): uint8 [128, W_T, 3] and [H_c, W_c, 3] CUDA views with dense
    pixels (T read in place through its pitch), cells the n (R(c_k), R(p_k), R(p_k + t_k), R(k w_r), min(R((k+1) w_r), W_T)) of
    pipeline.unlayout_cells.  Row i of T_col belongs to the last cell k with R(c_k) <= i and reads T at row
    clamp(R(p_k) + i - R(c_k), R(p_k), R(p_k + t_k) - 1), column clamp(R(k w_r) + j, R(k w_r), min(R((k+1) w_r), W_T) - 1)."""
    _vertical_gather(items, "vertical_unlayout", 5, "mn_vertical_unlayout_u8_batched")
