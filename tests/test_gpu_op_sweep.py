"""Every call of the non-convolution kernels in real forwards of the three modules, checked against the fp64 references of
oracle/op_ref.py, plus the shapes and edges the modules never produce.

A fixture wraps the ops below in ``ops`` (the modules and ``ops.conv2d`` look them up at call time); the forwards run eagerly (no
module graphs).  For each call the wrapper synchronises, copies what the op reads, runs the real op and checks:
  - values against fp64 (op_ref.ratio: |got - ref| <= tol * (bound + |ref|) element by element), or bit for bit for the ops that are
    exact by construction (select_text, window_scatter, check_labels, the window integers, the layout conversion);
  - exact zeros beyond valid widths and window widths (their bound is 0);
  - unchanged bytes outside an ``out=`` channel slice (the SR trunk writes into slices of its concatenation buffers);
  - for resample_modulate, which kernel ran (the alignment rule of mn_resample_modulate, restated in ``_resample_kernel``);
  - for demod_batched, the descriptor table decoded against the module's layers, then every layer's slice.
Negative controls run on the first suitable calls of each op: a reference with the per-sample or per-window rows shifted by one, a
window moved one column, or the skip or scale dropped must fail the same comparison.  The last test runs any workload this session
skipped and TSPGAN / TSPSRNet inside ops.deferred_checks (device labels and windows), asserts that every op and variant was seen and
that every control failed, and prints the op x variant table (calls / worst error-to-tolerance ratio).

The offset-data tests check GroupNorm and AdaIN statistics of data whose mean is k times its std (k up to 3000) with TOL_STATS, the
threshold of the convolution epilogue's statistics."""
import collections

import numpy as np
import pytest
import torch

from marconet_b200.testing.workloads import WORKLOADS, priors, sr_ragged_inputs, tspgan
from oracle import op_ref as R
from oracle.conv_ref import groupnorm_stats64
from test_gpu_conv_sweep import _snapshot, _untouched_outside

pytestmark = pytest.mark.gpu

# |got - ref| <= TOL[op] * (bound + |ref|) (op_ref.py): 4x the worst |got - ref| / (bound + |ref|) of the first H100 run with these
# bounds (NVIDIA H100 80GB HBM3, 700 W): groupnorm_apply 9.3e-8, groupnorm_swish 1.1e-7, adain_concat 2.0e-7, resample_modulate
# 1.3e-7, resample_up2_ragged 1.2e-7, torgb 6.8e-8, demod_batched 2.8e-7, pixelnorm 2.1e-7, layernorm 1.0e-7, token_mix 1.2e-7,
# attention 1.3e-7.  The table of the run is profiles/r12_op_sweep.txt.
TOL = dict(groupnorm_apply=3.8e-7, groupnorm_swish=4.5e-7, adain_concat=8.2e-7, resample_modulate=5.2e-7, resample_up2_ragged=4.7e-7,
           torgb=2.8e-7, demod_batched=1.2e-6, pixelnorm=8.5e-7, layernorm=4.1e-7, token_mix=5.0e-7, attention=5.4e-7)
TOL_STATS = 4e-7           # GroupNorm / AdaIN statistics: the epilogue statistics' threshold of test_gpu_conv_sweep.py

RECORDS = []                                 # dict(op, feats, ratio)
CONTROLS = collections.defaultdict(list)     # op -> [(control, failed as it must)]
WORST = collections.defaultdict(float)       # op -> worst |got - ref| / (bound + |ref|) (for setting TOL)
DONE = set()
KERNELS = collections.Counter()             # resample_modulate: kernel -> calls
WRAPPED = ["groupnorm_stats", "groupnorm_apply", "groupnorm_swish", "adain_concat", "window_scatter", "resample_modulate",
           "resample_up2_ragged", "torgb", "demod_batched", "pixelnorm", "layernorm", "token_mix", "attention", "select_text",
           "check_labels", "char_windows", "char_windows_ragged", "nchw_to_nhwc"]
# the variants each op must have run with by the end of the file ("module": from a module forward)
REQUIRED = {
    "groupnorm_stats": {"C=32", "C=64", "C=256", "C=512", "C=1024", "HW<32", "x_cs>C", "valid_w=1", "module"},
    "groupnorm_apply": {"C=32", "C=64", "C=256", "C=512", "C=1024", "HW<32", "x_cs>C", "valid_w=1", "swish", "no_swish", "out_slice"},
    "groupnorm_swish": {"C=32", "C=64", "C=256", "C=512", "C=1024", "HW<32", "x_cs>C", "valid_w=1", "out_slice"},
    "adain_concat": {"clipped_left", "clipped_right", "overlap3", "x_cs>C", "module"},
    "window_scatter": {"overlap3", "empty_line", "out_cs>C", "module"},
    "resample_modulate": {"up2_kernel", "generic_kernel", "copy", "H=1", "W=1", "W=3", "W=5", "x_cs>C", "y_cs>C", "module"},
    "resample_up2_ragged": {"vw=1", "vw=4k+1", "vw=full", "module"},
    "torgb": {"C=128", "C=256", "C=384", "C=512", "skip", "no_skip", "module"},
    "demod_batched": {"cout%64", "cin%4", "module"},
    "pixelnorm": {"rows%4", "dim%32", "module"},
    "layernorm": {"rows%4", "dim%32", "module"},
    "token_mix": {"To=1", "To=3", "To=5", "D%128", "module"},
    "attention": {"S=1", "S=7", "S=8", "S=9", "S=33", "S=63", "module"},
    "select_text": {"module"},
    "check_labels": {"module"},
    "char_windows": {"module"},
    "char_windows_ragged": {"module"},
    "nchw_to_nhwc": {"module"},
}


def _dev():
    return torch.device("cuda:0")


def _cs(t):
    """Channel stride (pixel pitch) of an NHWC view."""
    return t.stride(2)


def _resample_kernel(s, up):
    """Which kernel mn_resample_modulate runs: the bilinear x2 specialisation needs the style slice (if any) 16-byte aligned with a
    row stride that is a multiple of 4 floats; otherwise the generic kernel (which also does the plain copy, up=False)."""
    if not up:
        return "copy"
    if s is None or (s.stride(0) % 4 == 0 and s.data_ptr() % 16 == 0):
        return "up2_kernel"
    return "generic_kernel"


def _overlap3(wins):
    """Some column is covered by three windows of one line."""
    cover = collections.Counter()
    for line, x1, x2, _ in wins:
        for x in range(x1, x2):
            cover[(line, x)] += 1
    return bool(cover) and max(cover.values()) >= 3


class Checker:
    def __init__(self, ops):
        self.ops, self.enabled, self.in_module = ops, True, False
        self.orig = {name: getattr(ops, name) for name in WRAPPED}
        self.wsq = {}              # data_ptr -> wsq tensor of a demodulation table
        self.tables = {}           # data_ptr of a module's table -> its packed "styled" entries
        self.kernels = []          # the kernel of every resample_modulate call of this test

    def wrap(self, name):
        def call(*args, **kw):
            if not self.enabled:
                return self.orig[name](*args, **kw)
            torch.cuda.synchronize()
            return getattr(self, "_" + name)(*args, **kw)
        return call

    # ---- bookkeeping ----------------------------------------------------------------------------------------------------
    def _record(self, op, feats, r, tol=None, where=""):
        if self.in_module:
            feats = set(feats) | {"module"}
        if tol is not None:
            WORST[op] = max(WORST[op], r * tol)
        RECORDS.append(dict(op=op, feats=set(feats), ratio=r))
        assert r <= 1.0, f"{op} {where}: error / tolerance {r:.3g}"

    def _controls(self, op, cands):
        """cands: [(name, fails)] where fails() says whether the wrong reference fails the comparison (None: not applicable here)."""
        done = {c for c, _ in CONTROLS[op]}
        for name, fails in cands:
            if name in done:
                continue
            f = fails()
            if f is not None:
                CONTROLS[op].append((name, bool(f)))

    # ---- GroupNorm --------------------------------------------------------------------------------------------------------
    def _gn_feats(self, x, vw_host, out=None):
        n, h, w, c = x.shape
        f = {f"C={c}"}
        if h * w < 32:
            f.add("HW<32")
        if _cs(x) > c:
            f.add("x_cs>C")
        if vw_host is not None:
            f.add("valid_w")
            if 1 in vw_host:
                f.add("valid_w=1")
        if out is not None and _cs(out) > c:
            f.add("out_slice")
        return f

    def _groupnorm_stats(self, x, cpg=32, eps=1e-6, valid_w=None):
        vw = None if valid_w is None else valid_w.cpu().tolist()
        x0 = x.clone()
        mr = self.orig["groupnorm_stats"](x, cpg=cpg, eps=eps, valid_w=valid_w)
        torch.cuda.synchronize()
        ref = groupnorm_stats64(x0, valid_w=vw, eps=eps)
        e = R.stats_err(mr, ref)
        self._record("groupnorm_stats", self._gn_feats(x, vw), e / TOL_STATS, TOL_STATS, str(tuple(x.shape)))
        n = x.shape[0]
        self._controls("groupnorm_stats", [("shift", lambda: None if n < 2 or torch.equal(ref, ref.roll(1, 0)) else
                                            R.stats_err(mr, ref.roll(-1, 0)) > TOL_STATS)])
        return mr

    def _check_gn_out(self, op, x0, y, ref, bound, vw, snap, feats, ctrl):
        tol = TOL[op]
        r = R.ratio(y, ref, bound, tol)
        assert _untouched_outside(snap), f"{op} {tuple(y.shape)}: bytes outside the output slice changed"
        self._record(op, feats, r, tol, str(tuple(y.shape)))
        self._controls(op, [("shift", lambda: None if ctrl is None else R.ratio(y, ctrl[0], ctrl[1], tol) > 1.0)])

    def _groupnorm_apply(self, x, mr, gamma, beta, cpg=32, swish=True, valid_w=None, out=None):
        vw = None if valid_w is None else valid_w.cpu().tolist()
        x0, mr0 = x.clone(), mr.clone()
        snap = _snapshot(out)
        y = self.orig["groupnorm_apply"](x, mr, gamma, beta, cpg=cpg, swish=swish, valid_w=valid_w, out=out)
        torch.cuda.synchronize()
        ref, bound = R.groupnorm_apply_ref(x0, mr0, gamma, beta, swish, vw)
        ctrl = None
        if x.shape[0] > 1:
            ctrl = R.groupnorm_apply_ref(x0, mr0.roll(-1, 0), gamma, beta, swish, vw)
        feats = self._gn_feats(x, vw, out) | {"swish" if swish else "no_swish"}
        self._check_gn_out("groupnorm_apply", x0, y, ref, bound, vw, snap, feats, ctrl)
        return y

    def _groupnorm_swish(self, x, gamma, beta, cpg=32, eps=1e-6, swish=True, valid_w=None, out=None):
        vw = None if valid_w is None else valid_w.cpu().tolist()
        x0 = x.clone()
        snap = _snapshot(out)
        y = self.orig["groupnorm_swish"](x, gamma, beta, cpg=cpg, eps=eps, swish=swish, valid_w=valid_w, out=out)
        torch.cuda.synchronize()
        mr = groupnorm_stats64(x0, valid_w=vw, eps=eps)
        ref, bound = R.groupnorm_apply_ref(x0, mr, gamma, beta, swish, vw, own_stats=True)
        ctrl = None if x.shape[0] < 2 else R.groupnorm_apply_ref(x0, mr.roll(-1, 0), gamma, beta, swish, vw, own_stats=True)
        feats = self._gn_feats(x, vw, out) | {"swish" if swish else "no_swish"}
        self._check_gn_out("groupnorm_swish", x0, y, ref, bound, vw, snap, feats, ctrl)
        return y

    # ---- AdaIN + concat / window write-back ---------------------------------------------------------------------------
    def _adain_concat(self, prior, feat, win_dev, nc, wp):
        p0, f0 = prior.clone(), feat.clone()
        wins = [tuple(r) for r in win_dev.cpu().tolist()]
        out = self.orig["adain_concat"](prior, feat, win_dev, nc, wp)
        torch.cuda.synchronize()
        c = prior.shape[3]
        ref, bound, floor = R.adain_concat_ref(p0, f0, wins, wp)
        tol = TOL["adain_concat"]
        r = R.ratio(out[..., :c], ref[..., :c], bound[..., :c], tol, floor[..., :c])
        where = f"{tuple(prior.shape)} {nc} windows"
        assert torch.equal(out[..., c:].double(), ref[..., c:]), f"adain_concat {where}: the feature half is not the window bit for bit"
        feats = set()
        for line, x1, x2, y1 in wins:
            if x2 - x1 < wp:
                feats.add("clipped_left" if x1 == 0 else "clipped_right")
        if _overlap3(wins):
            feats.add("overlap3")
        if _cs(prior) > c or _cs(feat) > c:
            feats.add("x_cs>C")
        self._record("adain_concat", feats, r, tol, where)

        def bad(**kw):
            b, bb, fl = R.adain_concat_ref(p0, f0, wins, wp, **kw)
            if torch.equal(b, ref):
                return None
            return R.ratio(out[..., :c], b[..., :c], bb[..., :c], tol, fl[..., :c]) > 1.0 or not torch.equal(out[..., c:].double(), b[..., c:])
        self._controls("adain_concat", [("shift", lambda: None if nc < 2 else bad(shift=1)), ("move", lambda: bad(move=1))])
        return out

    @staticmethod
    def _scatter_expect(f0, sc, sh, owner, wins, move=0):
        """fp32 f + (f * scale + shift) at every owned column (torch on the CPU: each product and sum rounded on its own)."""
        b, h, w, c = f0.shape
        own = owner.long()
        idx = own.clamp_min(0)
        x1 = torch.tensor([wn[1] for wn in wins] or [0], dtype=torch.long)
        xx = (torch.arange(w)[None, :] - x1[idx] - move).clamp(0, sc.shape[2] - 1)
        s = sc[idx, :, xx].permute(0, 2, 1, 3)          # [B, W, H, C] -> [B, H, W, C]
        t = sh[idx, :, xx].permute(0, 2, 1, 3)
        val = f0 + (f0 * s + t)
        return torch.where((own >= 0)[:, None, :, None], val, f0)

    def _window_scatter(self, feat, scale, shift, owner_dev, win_dev, wp, out=None):
        f0, sc, sh = feat.cpu(), scale.cpu(), shift.cpu()
        owner, wins = owner_dev.cpu(), [tuple(r) for r in win_dev.cpu().tolist()]
        snap = _snapshot(out)
        y = self.orig["window_scatter"](feat, scale, shift, owner_dev, win_dev, wp, out=out)
        torch.cuda.synchronize()
        want = self._scatter_expect(f0, sc, sh, owner, wins)
        where = f"{tuple(feat.shape)} {len(wins)} windows"
        assert torch.equal(y.cpu(), want), f"window_scatter {where}: not f + (f * scale + shift) bit for bit"
        assert _untouched_outside(snap), f"window_scatter {where}: bytes outside the output slice changed"
        feats = set()
        if _overlap3(wins):
            feats.add("overlap3")
        if bool((owner < 0).all(1).any()):
            feats.add("empty_line")
        if out is not None and _cs(out) > feat.shape[3]:
            feats.add("out_cs>C")
        self._record("window_scatter", feats, 0.0, None, where)

        def moved():
            bad = self._scatter_expect(f0, sc, sh, owner, wins, move=1)
            return None if torch.equal(bad, want) else not torch.equal(y.cpu(), bad)
        self._controls("window_scatter", [("move", moved)])
        return y

    # ---- bilinear x2 ------------------------------------------------------------------------------------------------------
    def _resample_modulate(self, x, s=None, up=False, out=None):
        x0, s0 = x.clone(), None if s is None else s.clone()
        kern = _resample_kernel(s, up)
        snap = _snapshot(out)
        y = self.orig["resample_modulate"](x, s, up=up, out=out)
        torch.cuda.synchronize()
        self.kernels.append(kern)
        KERNELS[kern] += 1
        ref, bound = R.resample_ref(x0, s0, up)
        tol = TOL["resample_modulate"]
        r = R.ratio(y, ref, bound, tol)
        n, h, w, c = x.shape
        where = f"{kern} {tuple(x.shape)}"
        assert _untouched_outside(snap), f"resample_modulate {where}: bytes outside the output slice changed"
        feats = {kern, "s" if s is not None else "no_s", f"H={h}" if h == 1 else "H>1"}
        if w in (1, 3, 5):
            feats.add(f"W={w}")
        if _cs(x) > c:
            feats.add("x_cs>C")
        if out is not None and _cs(out) > c:
            feats.add("y_cs>C")
        self._record("resample_modulate", feats, r, tol, where)
        cands = []
        if s is not None:
            cands.append(("drop_scale", lambda: R.ratio(y, *R.resample_ref(x0, None, up), tol) > 1.0))
            cands.append(("shift", lambda: None if n < 2 else R.ratio(y, *R.resample_ref(x0, s0, up, shift=1), tol) > 1.0))
        self._controls("resample_modulate", cands)
        return y

    def _resample_up2_ragged(self, x, valid_w, s=None, out=None):
        vw = valid_w.cpu().tolist()
        x0, s0 = x.clone(), None if s is None else s.clone()
        snap = _snapshot(out)
        y = self.orig["resample_up2_ragged"](x, valid_w, s=s, out=out)
        torch.cuda.synchronize()
        ref, bound = R.resample_ref(x0, s0, True, valid_w=vw)
        tol = TOL["resample_up2_ragged"]
        r = R.ratio(y, ref, bound, tol)
        w = x.shape[2]
        assert _untouched_outside(snap), f"resample_up2_ragged {tuple(x.shape)}: bytes outside the output slice changed"
        feats = {"s" if s is not None else "no_s"}
        for v in vw:
            feats.add("vw=full" if v == w else ("vw=1" if v == 1 else ("vw=4k+1" if v % 4 == 1 else "vw<W")))
        self._record("resample_up2_ragged", feats, r, tol, f"{tuple(x.shape)} valid_w {vw}")
        shifted = vw[1:] + vw[:1]
        self._controls("resample_up2_ragged", [("shift", lambda: None if shifted == vw else
                                                R.ratio(y, *R.resample_ref(x0, s0, True, valid_w=shifted), tol) > 1.0)])
        return y

    # ---- ToRGB / demodulation ---------------------------------------------------------------------------------------------
    def _torgb(self, x, s, w, bias, skip=None):
        x0, s0, sk0 = x.clone(), s.clone(), None if skip is None else skip.clone()
        y = self.orig["torgb"](x, s, w, bias, skip)
        torch.cuda.synchronize()
        ref, bound = R.torgb_ref(x0, s0, w, bias, sk0)
        tol = TOL["torgb"]
        r = R.ratio(y, ref, bound, tol)
        n, c = x.shape[0], x.shape[3]
        self._record("torgb", {f"C={c}", "skip" if skip is not None else "no_skip"}, r, tol, f"{tuple(x.shape)}")
        self._controls("torgb", [
            ("drop_skip", lambda: None if skip is None else R.ratio(y, *R.torgb_ref(x0, s0, w, bias, sk0, drop_skip=True), tol) > 1.0),
            ("shift", lambda: None if n < 2 else R.ratio(y, *R.torgb_ref(x0, s0, w, bias, sk0, shift=1), tol) > 1.0)])
        return y

    def _demod_batched(self, s_all, table, out_total):
        raw, n_layers, mx = table
        descs = (self.ops._lib.DemodDesc * n_layers).from_buffer_copy(raw.cpu().numpy().tobytes())
        s0 = s_all.clone()
        y = self.orig["demod_batched"](s_all, table, out_total)
        torch.cuda.synchronize()
        styled = self.tables.get(raw.data_ptr())
        if styled is not None:              # a module's table: one descriptor per styled convolution, in order
            assert n_layers == len(styled), (n_layers, len(styled))
            for d, e in zip(descs, styled):
                assert (d.wsq, d.s_off, d.cin, d.cout, d.out_off) == (e["wsq"].data_ptr(), e["off"][0], e["wsq"].shape[0], e["cout"],
                                                                      e["demod_off"]), "demodulation descriptor disagrees with its layer"
        assert mx == max(d.cout for d in descs)
        tol = TOL["demod_batched"]
        worst, feats, bad = 0.0, set(), []
        for d in descs:
            wsq = self.wsq[d.wsq]
            got = y[:, d.out_off:d.out_off + d.cout]
            ref, bound = R.demod_ref(s0, wsq, d.s_off)
            worst = max(worst, R.ratio(got, ref, bound, tol))
            if s0.shape[0] > 1:
                bad.append(R.ratio(got, *R.demod_ref(s0, wsq, d.s_off, shift=1), tol) > 1.0)
            if d.cout % 64:
                feats.add("cout%64")
            if d.cin % 4:
                feats.add("cin%4")
        self._record("demod_batched", feats, worst, tol, f"{n_layers} layers, N = {s_all.shape[0]}")
        self._controls("demod_batched", [("shift", lambda: all(bad) if bad else None)])
        return y

    # ---- row ops ----------------------------------------------------------------------------------------------------------
    def _rows(self, op, y, ref, bound, feats, ctrl):
        tol = TOL[op]
        r = R.ratio(y, ref, bound, tol)
        self._record(op, feats, r, tol, str(tuple(y.shape)))
        self._controls(op, [(name, (lambda c=c: None if c is None else R.ratio(y, c[0], c[1], tol) > 1.0)) for name, c in ctrl])

    @staticmethod
    def _row_feats(rows, dim):
        return {"rows%4" if rows % 4 else "rows=4k", "dim%32" if dim % 32 else "dim=32k"}

    def _pixelnorm(self, x):
        x0 = x.clone()
        y = self.orig["pixelnorm"](x)
        torch.cuda.synchronize()
        ref, bound = R.pixelnorm_ref(x0)
        ctrl = None if x.shape[0] < 2 else R.pixelnorm_ref(x0.roll(-1, 0))
        self._rows("pixelnorm", y, ref, bound, self._row_feats(*x.shape), [("shift", ctrl)])
        return y

    def _layernorm(self, x2d, gamma, beta, eps=1e-5):
        x0 = x2d.clone()
        y = self.orig["layernorm"](x2d, gamma, beta, eps)
        torch.cuda.synchronize()
        ref, bound = R.layernorm_ref(x0, gamma, beta, eps)
        ctrl = None if x0.shape[0] < 2 else R.layernorm_ref(x0.roll(-1, 0), gamma, beta, eps)
        self._rows("layernorm", y, ref, bound, self._row_feats(*x0.shape), [("shift", ctrl)])
        return y

    def _token_mix(self, x, gamma, beta, w, bias, eps=1e-5):
        x0 = x.clone()
        y = self.orig["token_mix"](x, gamma, beta, w, bias, eps)
        torch.cuda.synchronize()
        ref, bound = R.token_mix_ref(x0, gamma, beta, w, bias, eps)
        b, t, d = x.shape
        to = w.shape[0]
        feats = {f"To={to}", "D%128" if d % 128 else "D=128k"}
        ctrl = [("shift", None if b < 2 else R.token_mix_ref(x0.roll(-1, 0), gamma, beta, w, bias, eps)),
                ("drop_bias", R.token_mix_ref(x0, gamma, beta, w, torch.zeros_like(bias), eps))]
        self._rows("token_mix", y, ref, bound, feats, ctrl)
        return y

    def _attention(self, qkv, heads=8, dh=64):
        q0 = qkv.clone()
        y = self.orig["attention"](qkv, heads, dh)
        torch.cuda.synchronize()
        ref, bound = R.attention_ref(q0, heads, dh)
        ctrl = None if qkv.shape[0] < 2 else R.attention_ref(q0, heads, dh, shift=1)
        self._rows("attention", y, ref, bound, {f"S={qkv.shape[1]}"}, [("shift", ctrl)])
        return y

    # ---- exact ops --------------------------------------------------------------------------------------------------------
    def _exact(self, op, got, want, where, shifted=None):
        assert torch.equal(got, want), f"{op} {where}: differs from the exact result"
        self._record(op, set(), 0.0, None, where)
        if shifted is None and want.shape[0] > 1:
            shifted = want.roll(1, 0)
        self._controls(op, [("shift", lambda: None if shifted is None or torch.equal(shifted, want) else not torch.equal(got, shifted))])

    def _select_text(self, emb, labels_dev, s, n, l):
        lab = labels_dev.cpu()
        s0 = None if s is None else s.cpu()
        y = self.orig["select_text"](emb, labels_dev, s, n, l)
        torch.cuda.synchronize()
        c = emb.shape[1]

        def expect(lab_):
            e = emb.cpu()[lab_].view(n, l, 1, c).expand(n, l, 4, c).reshape(n, 1, 4 * l, c).expand(n, 4, 4 * l, c)
            return e if s0 is None else e * s0[:, None, None, :c]
        self._exact("select_text", y.cpu(), expect(lab), f"[{n}, {l}]", shifted=expect(lab.roll(1)))
        return y

    def _check_labels(self, labels_dev, classes, flag):
        lab = labels_dev.cpu()
        y = self.orig["check_labels"](labels_dev, classes, flag)
        torch.cuda.synchronize()
        self._exact("check_labels", y.cpu(), lab.clamp(0, classes - 1), f"{lab.numel()} labels")
        return y

    def _windows(self, op, res, locs, counts, width, half, line_w=None):
        from marconet_b200.models import networks
        wins, valid, owner = networks._char_windows_np(locs.cpu().numpy(), counts, width, half, line_w)
        got = [t.cpu().numpy() for t in res]
        where = f"{len(counts)} lines, {sum(counts)} characters"
        assert np.array_equal(got[0], wins) and np.array_equal(got[1], valid) and np.array_equal(got[2], owner), \
            f"{op} {where}: window integers differ from networks._char_windows_np"
        self._record(op, set(), 0.0, None, where)
        moved = wins.copy()
        moved[:, 1:3] += 1
        self._controls(op, [("move", lambda: None if not len(wins) else not np.array_equal(got[0], moved))])

    def _char_windows(self, locs_dev, line_first_dev, counts, width, half, flag):
        res = self.orig["char_windows"](locs_dev, line_first_dev, counts, width, half, flag)
        torch.cuda.synchronize()
        self._windows("char_windows", res, locs_dev, counts, width, half)
        return res

    def _char_windows_ragged(self, locs_dev, line_first_dev, line_w_dev, counts, width, half, flag):
        res = self.orig["char_windows_ragged"](locs_dev, line_first_dev, line_w_dev, counts, width, half, flag)
        torch.cuda.synchronize()
        self._windows("char_windows_ragged", res, locs_dev, counts, width, half, line_w_dev.cpu().tolist())
        return res

    def _nchw_to_nhwc(self, x, out=None):
        x0 = x.clone()
        snap = _snapshot(out)
        y = self.orig["nchw_to_nhwc"](x, out=out)
        torch.cuda.synchronize()
        assert _untouched_outside(snap), "nchw_to_nhwc: bytes outside the output slice changed"
        self._exact("nchw_to_nhwc", y, x0.permute(0, 2, 3, 1), str(tuple(x.shape)))
        return y


@pytest.fixture
def sweep(monkeypatch, gpu_models):
    from marconet_b200 import ops
    chk = Checker(ops)
    monkeypatch.setattr(ops, "MODULE_GRAPHS", False)
    for name in WRAPPED:
        monkeypatch.setattr(ops, name, chk.wrap(name))
    pk = gpu_models["tspgan"].TextGenerator._get_packed(_dev())
    chk.tables[pk["demod_table"][0].data_ptr()] = pk["styled"]
    for e in pk["styled"]:
        chk.wsq[e["wsq"].data_ptr()] = e["wsq"]
    yield chk


def _run(sweep, fn):
    sweep.in_module = True
    try:
        with torch.no_grad():
            fn()
    finally:
        sweep.in_module = False


@pytest.mark.parametrize("name", list(WORKLOADS))
def test_forward_calls_match_fp64(sweep, gpu_models, name):
    _run(sweep, lambda: WORKLOADS[name](gpu_models))
    DONE.add(name)


def _deferred(gm, which):
    """TSPGAN with its labels on the device (check_labels) / TSPSRNet with its boxes on the device (char_windows,
    char_windows_ragged), inside ops.deferred_checks: the error flag must stay 0."""
    from marconet_b200 import ops
    flag = torch.zeros(1, dtype=torch.int32, device=_dev())
    with ops.deferred_checks(flag):
        if which == "tspgan":
            tspgan(gm, 3, 2, labels_on_device=True)
        elif which == "sr_ragged":
            widths, counts = (512, 700, 1264), (12, 20, 44)
            lq, locs = sr_ragged_inputs(widths, counts)
            p64, p32 = priors(counts, 9)
            gm["sr"](lq.to(_dev()), p64, p32, locs.to(_dev()), widths=list(widths))
        else:
            lq, locs = sr_ragged_inputs((512,), (10,))
            p64, p32 = priors((10,), 9)
            gm["sr"](lq.to(_dev()), p64, p32, locs.to(_dev()))
    torch.cuda.synchronize()
    assert int(flag.item()) == 0


@pytest.mark.parametrize("which", ["tspgan", "sr", "sr_ragged"])
def test_deferred_checks_on_the_device(sweep, gpu_models, which):
    _run(sweep, lambda: _deferred(gpu_models, which))
    DONE.add("deferred_" + which)


# ---- direct cases the modules never produce ---------------------------------------------------------------------------
def _t(*shape, seed, scale=1.0, shift=0.0):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(*shape, generator=g) * scale + shift).to(_dev())


def _slice(n, h, w, c, seed, extra=32, scale=1.0, shift=0.0):
    """An NHWC view of C channels starting at channel ``extra`` of a wider buffer (pixel pitch C + 2 * extra)."""
    return _t(n, h, w, c + 2 * extra, seed=seed, scale=scale, shift=shift)[..., extra:extra + c]


@pytest.mark.parametrize("s", [1, 7, 8, 9, 33, 63])
def test_attention_partial_query_chunks(sweep, s):
    """Query chunks of 8 rows: S = 1 / 7 / 9 / 33 / 63 leave a partial last chunk; 33 <= S < 64 a partial second softmax pass."""
    from marconet_b200 import ops
    ops.attention(_t(2, s, 3 * 8 * 64, seed=s), 8, 64)
    assert RECORDS[-1]["op"] == "attention"


@pytest.mark.parametrize("to", [1, 3, 5])
def test_token_mix_output_counts(sweep, to):
    """Output tokens in fours plus a remainder; D = 200 leaves a partial block of 128 features."""
    from marconet_b200 import ops
    b, t, d = 2, 16, 200
    ops.token_mix(_t(b, t, d, seed=to), _t(t, seed=1, scale=0.3, shift=1.0), _t(t, seed=2, scale=0.2), _t(to, t, seed=3, scale=0.25),
                  _t(to, seed=4))


@pytest.mark.parametrize("rows,dim", [(7, 100), (5, 512), (8, 33)])
def test_row_norms_odd_shapes(sweep, rows, dim):
    from marconet_b200 import ops
    ops.layernorm(_t(rows, dim, seed=rows, shift=0.5), _t(dim, seed=5, scale=0.3, shift=1.0), _t(dim, seed=6, scale=0.2))
    ops.pixelnorm(_t(rows, dim, seed=rows + 1))


@pytest.mark.parametrize("skip", [False, True])
@pytest.mark.parametrize("c", [128, 256, 384, 512])
def test_torgb_widths(sweep, c, skip):
    """Every instantiation (4 / 8 / 12 / 16 channels per lane), with and without the bilinear skip; C = 384 is none of the module's."""
    from marconet_b200 import ops
    n, h = 2, 8
    ops.torgb(_slice(n, h, h, c, seed=c), _t(n, c + 4, seed=c + 1)[:, 4:], _t(3, c, seed=c + 2, scale=0.05), _t(3, seed=c + 3),
              _t(n, h // 2, h // 2, 3, seed=c + 4) if skip else None)


@pytest.mark.parametrize("aligned", [True, False])
@pytest.mark.parametrize("h,w", [(1, 1), (1, 3), (1, 5), (3, 5), (4, 9)])
def test_bilinear_x2_both_kernels(sweep, h, w, aligned):
    """An aligned style slice takes the bilinear x2 specialisation, an unaligned one the generic kernel; channel slices on both
    sides (x_cs > C, y_cs > C)."""
    from marconet_b200 import ops
    n, c = 2, 16
    sbuf = _t(n, c + 8, seed=11)
    s = sbuf[:, 4:4 + c] if aligned else sbuf[:, 1:1 + c]
    out = torch.full((n, 2 * h, 2 * w, c + 8), 7.0, device=_dev())[..., 4:4 + c]
    ops.resample_modulate(_slice(n, h, w, c, seed=10 + w), s, up=True, out=out)
    assert sweep.kernels[-1] == ("up2_kernel" if aligned else "generic_kernel")
    ops.resample_modulate(_slice(n, h, w, c, seed=20 + w), s, up=False)


def test_ragged_bilinear_widths(sweep):
    """Widths of 1, of 4k + 1 and of the whole canvas in one batch, with and without a style scale."""
    from marconet_b200 import ops
    n, h, w, c = 4, 3, 12, 8
    vw = torch.tensor([1, 5, w, 9], dtype=torch.int32, device=_dev())
    x = _slice(n, h, w, c, seed=30, extra=4)
    ops.resample_up2_ragged(x, vw)
    out = torch.full((n, 2 * h, 2 * w, c + 8), 7.0, device=_dev())[..., 4:4 + c]
    ops.resample_up2_ragged(x, vw, s=_t(n, c, seed=31), out=out)


def test_demod_batched_odd_layer_shapes(sweep):
    """Layers whose cout is not a multiple of the 64-column tile and whose cin is not a multiple of the 4 k-slices."""
    from marconet_b200 import ops
    n = 3
    w1, w2 = _t(10, 70, seed=40).abs(), _t(7, 130, seed=41).abs()
    for wsq in (w1, w2):
        sweep.wsq[wsq.data_ptr()] = wsq
    table = ops.make_demod_table([(w1, 3, 0), (w2, 20, 70)], _dev())
    ops.demod_batched(_t(n, 40, seed=42), table, 200)


@pytest.mark.parametrize("c", [32, 64, 256, 512, 1024])
def test_groupnorm_widths_and_ragged_samples(sweep, c):
    """Statistics, apply (with and without swish) and the fused pass at every group count the kernels support: H * W < 32, a channel
    slice of a wider buffer on both sides, valid widths including 1."""
    from marconet_b200 import ops
    n, h, w = 3, 2, 5
    x = _slice(n, h, w, c, seed=c, scale=1.5, shift=0.3)
    vw = torch.tensor([w, 1, 3], dtype=torch.int32, device=_dev())
    gamma, beta = _t(c, seed=c + 1, scale=0.3, shift=1.0), _t(c, seed=c + 2, scale=0.2)
    mr = ops.groupnorm_stats(x, valid_w=vw)
    for swish in (True, False):
        out = torch.full((n, h, w, c + 64), 7.0, device=_dev())[..., 32:32 + c]
        ops.groupnorm_apply(x, mr, gamma, beta, swish=swish, valid_w=vw, out=out)
    out = torch.full((n, h, w, c + 64), 7.0, device=_dev())[..., 32:32 + c]
    ops.groupnorm_swish(x, gamma, beta, valid_w=vw, out=out)
    ops.groupnorm_stats(_slice(2, 16, 24, c, seed=c + 3))            # H * W >= 32, several blocks per sample


def _line_case():
    """Three lines 40 columns wide, windows of half 8: line 0 has a window clipped at the left edge, a chain of three overlapping
    windows and one clipped at the right edge; line 1 has no characters; line 2 one window in the middle."""
    w, half = 40, 8
    counts = [5, 0, 1]
    locs = torch.zeros(3, 10)
    locs[0, 0:10:2] = torch.tensor([2, 15, 20, 25, 36]) / w
    locs[2, 0] = 20.0 / w
    return locs, counts, w, half


def test_windows_at_line_edges_and_overlap_chains(sweep):
    from marconet_b200 import ops
    locs, counts, w, half = _line_case()
    b, h, c, wp = len(counts), 4, 64, 2 * half
    flag = torch.zeros(1, dtype=torch.int32, device=_dev())
    first = torch.tensor([0, 5, 5, 6], dtype=torch.int32, device=_dev())
    win, valid, owner = ops.char_windows(locs.to(_dev()), first, counts, w, half, flag)
    win2, _, owner2 = ops.char_windows_ragged(locs.to(_dev()), first, torch.tensor([w, 24, 32], dtype=torch.int32, device=_dev()),
                                              counts, w, half, flag)
    assert int(flag.item()) == 0
    nc = sum(counts)
    feat = _slice(b, h, w, c, seed=50)
    fin = ops.adain_concat(_slice(nc, h, wp, c, seed=51, extra=16), feat, win, nc, wp)
    scale, shift = _t(nc, h, wp, c, seed=52, scale=0.3), _t(nc, h, wp, c, seed=53, scale=0.3)
    out = torch.full((b, h, w, c + 64), 7.0, device=_dev())[..., 32:32 + c]
    ops.window_scatter(feat, scale, shift, owner, win, wp, out=out)
    ops.window_scatter(feat, scale, shift, owner2, win2, wp)
    assert fin.shape == (nc, h, wp, 2 * c)


# ---- statistics of offset data ----------------------------------------------------------------------------------------
OFFSET_ERRS = {}


@pytest.mark.parametrize("k", [1, 30, 300, 3000])
def test_groupnorm_statistics_of_offset_data(sweep, k):
    """mean = k * std, valid widths and a channel slice: the statistics pass, and the statistics the fused pass applied (recovered
    from its un-affine output), against fp64 with TOL_STATS.  Plain fp32 sums of x and x * x lost the variance to cancellation
    (4.9e-4 at k = 300, 3.8e-2 at k = 3000; profiles/r12_offset_stats.txt); each thread now sums about a pivot."""
    from marconet_b200 import ops
    sweep.enabled = False
    n, h, w, c = 2, 32, 32, 256
    x = _slice(n, h, w, c, seed=60 + k, shift=float(k))
    vw = torch.tensor([w, 29], dtype=torch.int32, device=_dev())
    ref = groupnorm_stats64(x, valid_w=[w, 29])
    e_stats = R.stats_err(ops.groupnorm_stats(x, valid_w=vw), ref)
    y = ops.groupnorm_swish(x, torch.ones(c, device=_dev()), torch.zeros(c, device=_dev()), swish=False, valid_w=vw)
    e_fused = R.stats_err(R.affine_stats(x, y, valid_w=[w, 29]), ref)
    OFFSET_ERRS[("groupnorm", k)] = (e_stats, e_fused)
    print(f"\nGroupNorm mean/std = {k}: statistics pass {e_stats:.3e}, fused pass {e_fused:.3e} (|d mean| * rstd, |d rstd| / rstd)")
    assert e_stats <= TOL_STATS and e_fused <= TOL_STATS


@pytest.mark.parametrize("which", ["prior", "feat"])
@pytest.mark.parametrize("k", [1, 30, 300, 3000])
def test_adain_statistics_of_offset_data(sweep, k, which):
    """AdaIN + concat with the prior crops or the feature windows at mean = k * std, against fp64 with TOL_STATS: the statistics'
    error shows in the normalised half (the fp32 rounding of the prior mean is allowed exactly, as a floor)."""
    from marconet_b200 import ops
    sweep.enabled = False
    nc, h, wp, c, w = 4, 32, 32, 64, 128
    prior = _t(nc, h, wp, c, seed=70 + k, shift=float(k) if which == "prior" else 0.0)
    feat = _t(1, h, w, c, seed=71 + k, scale=0.5, shift=0.5 * k if which == "feat" else 0.0)
    wins = [(0, 32 * i, 32 * i + 32, 0) for i in range(nc)]
    out = ops.adain_concat(prior, feat, torch.tensor(wins, dtype=torch.int32, device=_dev()), nc, wp)
    ref, bound, floor = R.adain_concat_ref(prior, feat, wins, wp)
    r = R.ratio(out[..., :c], ref[..., :c], bound[..., :c], 1.0, floor[..., :c])
    OFFSET_ERRS[("adain_" + which, k)] = r
    print(f"\nAdaIN {which} mean/std = {k}: worst (|d| - floor) / (bound + |ref|) = {r:.3e}")
    assert r <= TOL_STATS


def test_coverage_and_negative_controls(sweep, gpu_models):
    """Runs any workload this session skipped, then: every op and variant was seen, every negative control failed."""
    for name, fn in WORKLOADS.items():
        if name not in DONE:
            _run(sweep, lambda: fn(gpu_models))
            DONE.add(name)
    for which in ("tspgan", "sr", "sr_ragged"):
        if "deferred_" + which not in DONE:
            _run(sweep, lambda: _deferred(gpu_models, which))
    table = collections.defaultdict(lambda: [0, 0.0])
    for r in RECORDS:
        for f in ["*"] + sorted(r["feats"]):
            cell = table[(r["op"], f)]
            cell[0] += 1
            cell[1] = max(cell[1], r["ratio"])
    print("\nop x variant: calls / worst error-to-tolerance ratio")
    for op in WRAPPED:
        cells = [f"{f}={table[(op, f)][0]}/{table[(op, f)][1]:.3f}" for f in ["*"] + sorted({f for r in RECORDS if r["op"] == op
                                                                                               for f in r["feats"]})]
        print(f"  {op:20s} " + "  ".join(cells))
    print("worst |got - ref| / (bound + |ref|) per op:", {k: f"{v:.3e}" for k, v in sorted(WORST.items())})
    print("resample_modulate kernels:", dict(KERNELS))
    print("negative controls (failed as they must):", {op: c for op, c in sorted(CONTROLS.items())})
    if OFFSET_ERRS:
        print("offset-data statistics errors:", {f"{a} k={k}": v for (a, k), v in sorted(OFFSET_ERRS.items())})
    for op, want in REQUIRED.items():
        seen = {f for r in RECORDS if r["op"] == op for f in r["feats"]}
        assert want <= seen, f"{op}: never ran with {sorted(want - seen)}"
    for op in WRAPPED:
        assert CONTROLS[op], f"{op}: no call suited a negative control"
        assert all(failed for _, failed in CONTROLS[op]), f"{op}: a negative control passed the comparison: {CONTROLS[op]}"
