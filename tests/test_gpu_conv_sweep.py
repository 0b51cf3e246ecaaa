"""Every convolution / linear call of real forwards of the three modules, checked against the fp64 reference of oracle/conv_ref.py,
one kernel branch at a time.

A fixture wraps ``ops.conv2d``, ``ops.linear`` and ``ops.patch_embed``; the forwards run eagerly (no module graphs).  For each call
the wrapper synchronises, gathers the sampled input patches and everything else the epilogue reads, runs the real op with ``plan=``
(which kernel, tile and split-K actually ran) and checks against fp64:
  - the sampled outputs y, y2 and the per-sample ``y2_ptrs`` destinations, element by element (conv_ref.ratio);
  - columns beyond valid_w are exactly zero over the whole tensor;
  - bytes of the destination buffers outside the output channel slice are unchanged;
  - ``gn_stats`` statistics against fp64 GroupNorm statistics of the stored y, and the ``gn`` constants the call received against
    fp64 statistics of its input.
Negative controls run on the first suitable call of each branch: a reference with the per-sample rows shifted by one sample, or with
the bias or residual dropped, must fail the same comparison.  The last test asserts that every branch and epilogue feature was seen
and prints the coverage table (branch x feature: calls and worst error / tolerance)."""
import collections
import math
import random

import pytest
import torch

from marconet_b200.testing.workloads import SUBSET, WORKLOADS
from oracle import conv_ref as R

pytestmark = pytest.mark.gpu

# |y - ref| <= TOL[precision] * (gain * L_act * (|out_scale| * A + |bias| + |residual|) + |ref|)  (conv_ref.py), per precision that
# ran: 4x the worst error / bound of the first H100 run (profiles/r10_conv_sweep.txt): fp32 5.9e-7, f16x3 4.1e-6, bf16x3 8.7e-6.
# No call runs f16x1 (not parity grade); its entry is a guess.
TOL = {0: 2.4e-6, 1: 1.7e-5, 2: 3.5e-5, 3: 1e-2}
TOL_LINEAR = 1.2e-6        # mn_linear_small_m / patch_embed (fp32 CUDA-core dot products): 4x the worst 2.9e-7
TOL_STATS = 4e-7           # GroupNorm statistics (|d mean| * rstd, |d rstd| / rstd): 4x the worst 9.3e-8 (mean/std = 3000)

RECORDS = []               # one dict per checked call
CONTROLS = collections.defaultdict(list)     # branch -> [(control, failed as it must)]
WORST_ERR = collections.defaultdict(float)   # precision -> worst |y - ref| / bound (for setting TOL)
WORST_STATS = [0.0]         # worst GroupNorm statistics error (for setting TOL_STATS)
DONE = set()               # workloads already run in this session


def _dev():
    return torch.device("cuda:0")


def branch_of(plan):
    k = plan["kernel"]
    if k == "simt":
        return "simt+splitK" if plan["splits"] > 1 else "simt"
    if k == "tc2":
        return f"tc2/nt{plan['nt']}" + ("/TN>1" if plan["TN"] > 1 else "") + ("+splitK" if plan["splits"] > 1 else "")
    return k


def _snapshot(t):
    """(storage view, copy) of the whole allocation under ``t``: compared after the call outside t's own elements."""
    if t is None:
        return None
    full = torch.empty(0, dtype=t.dtype, device=t.device).set_(t.untyped_storage(), 0, (t.untyped_storage().nbytes() // t.element_size(),))
    if full.numel() == t.numel():
        return None
    return t, full, full.clone()


def _untouched_outside(snap):
    if snap is None:
        return True
    t, full, before = snap
    before.as_strided(t.shape, t.stride(), t.storage_offset()).copy_(t)
    return torch.equal(before.view(torch.int32), full.view(torch.int32))


GUARD = 12345.0


def _copy(t):
    return None if t is None else t.clone()


class Checker:
    def __init__(self, ops):
        self.ops, self.enabled, self.tap_buffers = ops, True, {}
        self.guards = []           # guard bands around y2_ptrs destinations: must keep GUARD in every element
        self.orig = dict(conv2d=ops.conv2d, linear=ops.linear, patch_embed=ops.patch_embed)

    # ---- ops.conv2d ---------------------------------------------------------------------------------------------------
    def conv2d(self, x, w, kh, kw, stride=(1, 1), pad=(0, 0), **opts):
        if not self.enabled or opts.get("plan") is not None:
            return self.orig["conv2d"](x, w, kh, kw, stride=stride, pad=pad, **opts)
        torch.cuda.synchronize()
        ops = self.ops
        n, h, wd, cin = x.shape
        w2d = w.w if isinstance(w, ops.ConvWeight) else w
        cout = w2d.shape[1]
        oh, ow = (h + 2 * pad[0] - kh) // stride[0] + 1, (wd + 2 * pad[1] - kw) // stride[1] + 1
        vw = opts.get("valid_w")
        vw_host = None if vw is None else vw.cpu().tolist()
        # copies of what the call reads (its output may overwrite its input or residual); the pixels to check follow the plan
        x0, res0 = x.clone(), _copy(opts.get("residual"))
        os0, y2s0, b0 = _copy(opts.get("out_scale")), _copy(opts.get("y2_scale")), _copy(opts.get("bias"))
        gn = opts.get("gn")
        gn0 = None if gn is None else tuple(t.clone() for t in gn)
        gn_in = None if gn is None else (gn0[0].double(), R.groupnorm_stats64(x0, valid_w=vw_host))
        snaps = [_snapshot(opts.get("out")), _snapshot(opts["out2"] if isinstance(opts.get("out2"), torch.Tensor) else None)]
        plan = {}
        res = self.orig["conv2d"](x, w, kh, kw, stride=stride, pad=pad, plan=plan, **opts)
        torch.cuda.synchronize()
        tiled = plan["kernel"] in ("tc1", "tc2")
        pix = R.sample_pixels(n, oh, ow, th=plan["TH"] if tiled else None, tw=plan["TW"] if tiled else None,
                              tn=plan["TN"] if tiled else None, m_tile=128, valid_w=vw_host, count=200, seed=len(RECORDS))
        d = R.gather(x0, kh, kw, stride, pad, pix, gn=gn0, valid_w=vw if gn is not None else None, residual=res0,
                     res_broadcast=opts.get("res_broadcast", False), out_scale=os0, y2_scale=y2s0, bias=b0)
        if vw is not None:
            d["valid_w"] = vw.long()
        want_y = opts.get("want_y", True)
        y = y2 = mr = None
        if opts.get("gn_stats"):
            y, mr = res
        elif opts.get("out2") is not None:
            y, y2 = res if want_y else (None, res)
        else:
            y = res
        act, gain = opts.get("act", 0), opts.get("gain", 1.0)
        ref = R.conv_ref(d, w2d, act=act, gain=gain)
        tol = TOL[plan["precision"]]
        worst, errs = 0.0, []
        if y is not None:
            errs.append(("y", R.gather_out(y, pix), ref["y"], ref["bound"]))
        if opts.get("out2_ptrs") is not None:
            bufs = [self.tap_buffers[int(p)] for p in opts["out2_ptrs"].cpu().tolist()]
            y2 = torch.stack([b.view(oh, ow, cout) for b in bufs])
        if y2 is not None:
            errs.append(("y2", R.gather_out(y2, pix), ref.get("y2", ref["y"]), ref.get("bound2", ref["bound"])))
        for name, got, want, bound in errs:
            r = R.ratio(got, want, bound, tol)
            WORST_ERR[plan["precision"]] = max(WORST_ERR[plan["precision"]], r * tol)
            worst = max(worst, r)
        br = branch_of(plan)
        where = f"{br} {tuple(x.shape)}->{cout} k{kh} s{stride}"
        assert worst <= 1.0, f"{where}: error / tolerance {worst:.3g}"
        if vw is not None:
            for t in (y, y2):
                for i, v in enumerate(vw_host if t is not None else ()):
                    assert (t[i, :, v:] == 0).all(), f"{where}: sample {i} has nonzero columns beyond valid_w = {v}"
        assert all(_untouched_outside(s) for s in snaps), f"{where}: bytes outside the output slice changed"
        assert all(bool((g == GUARD).all()) for g in self.guards), f"{where}: a store landed outside its y2_ptrs destination"
        stats_err = None
        if mr is not None:
            stats_err = _stats_err(mr, R.groupnorm_stats64(y, valid_w=vw_host))
            WORST_STATS[0] = max(WORST_STATS[0], stats_err)
            assert stats_err <= TOL_STATS, f"{where}: GroupNorm statistics of the output off by {stats_err:.3g}"
        if gn_in is not None:
            e = _stats_err(*gn_in)
            WORST_STATS[0] = max(WORST_STATS[0], e)
            stats_err = max(stats_err or 0.0, e)
            assert e <= TOL_STATS, f"{where}: the GroupNorm constants it received are off by {e:.3g}"
        self._controls(br, d, w2d, act, gain, tol, errs, n, opts)
        feats = _features(opts, plan, y)
        RECORDS.append(dict(branch=br, feats=feats, ratio=worst, precision=plan["precision"], stats_err=stats_err, plan=plan))
        return res

    def _controls(self, br, d, w2d, act, gain, tol, errs, n, kw):
        done = {c for c, _ in CONTROLS[br]}
        todo = []
        if n > 1 and any(kw.get(k) is not None for k in ("out_scale", "y2_scale", "valid_w")) and "shift" not in done:
            todo.append(("shift", dict(shift=1)))
        for k in ("bias", "residual"):
            if kw.get(k) is not None and f"drop_{k}" not in done:
                todo.append((f"drop_{k}", dict(drop=(k,))))
        for name, opt in todo:
            bad = R.conv_ref(d, w2d, act=act, gain=gain, **opt)
            pick = lambda key: bad.get(key, bad["y"])        # noqa: E731  (y2 without y2_scale is y)
            if all(torch.equal(pick(key), want) for key, _, want, _ in errs):
                continue                 # identical rows (one-sample data, full-width windows): nothing to see on this call
            CONTROLS[br].append((name, any(R.ratio(got, pick(key), bound, tol) > 1.0 for key, got, _, bound in errs)))

    # ---- ops.linear / ops.patch_embed ------------------------------------------------------------------------------------
    def linear(self, x2d, w, bias=None, act=0, gain=1.0, residual=None, out=None, precision=None):
        if not self.enabled:
            return self.orig["linear"](x2d, w, bias, act, gain, residual, out, precision)
        torch.cuda.synchronize()
        wt = w.w if isinstance(w, self.ops.ConvWeight) else w
        ref, bound = R.linear_ref(x2d, wt, bias, act, gain, None if residual is None else residual.clone())
        y = self.orig["linear"](x2d, w, bias, act, gain, residual, out, precision)
        torch.cuda.synchronize()
        r = R.ratio(y, ref, bound, TOL_LINEAR)
        assert r <= 1.0, f"linear {tuple(x2d.shape)} x {tuple(wt.shape)}: error / tolerance {r:.3g}"
        RECORDS.append(dict(branch="linear", feats={"act:" + R.ACT_NAMES[act]}, ratio=r, precision=0, stats_err=None))
        return y

    def patch_embed(self, feat, w, bias, pe):
        if not self.enabled:
            return self.orig["patch_embed"](feat, w, bias, pe)
        torch.cuda.synchronize()
        ref, bound = R.patch_embed_ref(feat, w, bias, pe)
        y = self.orig["patch_embed"](feat, w, bias, pe)
        torch.cuda.synchronize()
        r = R.ratio(y, ref, bound, TOL_LINEAR)
        assert r <= 1.0, f"patch_embed {tuple(feat.shape)}: error / tolerance {r:.3g}"
        RECORDS.append(dict(branch="patch_embed", feats=set(), ratio=r, precision=0, stats_err=None))
        return y


def _stats_err(got, ref):
    """max of |d mean| * rstd and |d rstd| / rstd.  The mean is returned in fp32: its own rounding (up to 2^-24 |mean|, which is
    1.8e-4 std at mean/std = 3000) is not counted."""
    got = got.double().to(ref.device)
    em = (((got[..., 0] - ref[..., 0]).abs() - 2.0 ** -24 * ref[..., 0].abs()).clamp_min(0) * ref[..., 1]).max().item()
    er = ((got[..., 1] - ref[..., 1]).abs() / ref[..., 1]).max().item()
    return max(em, er)


def _features(kw, plan, y):
    f = set()
    for k in ("out_scale", "bias", "residual", "valid_w"):
        if kw.get(k) is not None:
            f.add(k)
    if kw.get("res_broadcast"):
        f.add("res_broadcast")
    act = kw.get("act", 0)
    if act != 0:
        f.add("act:" + R.ACT_NAMES[act])
        if act in (R.ACT_TANH, R.ACT_GELU, R.ACT_SIGMOID):
            f.add("runtime_act")
    if kw.get("out2") is not None or kw.get("out2_ptrs") is not None:
        f.add("y2")
    if kw.get("y2_scale") is not None:
        f.add("y2_scale")
    if kw.get("out2_ptrs") is not None:
        f.add("y2_ptrs")
    if y is None:
        f.add("want_y=False")
    if kw.get("gn") is not None:
        f.add("gn_fused" if plan["gn_fused"] else "gn_two_pass")
    if kw.get("gn_stats"):
        f.add("gn_stats_out" if plan["gn_stats_out"] else "gn_stats_pass")
    if plan["x_scale"] != 1.0:
        f.add("x_scale")
    return f


@pytest.fixture
def sweep(monkeypatch):
    from marconet_b200 import ops
    chk = Checker(ops)
    monkeypatch.setattr(ops, "MODULE_GRAPHS", False)
    monkeypatch.setattr(ops, "conv2d", chk.conv2d)
    monkeypatch.setattr(ops, "linear", chk.linear)
    monkeypatch.setattr(ops, "patch_embed", chk.patch_embed)
    old_prec, old_plan = ops.default_precision(), dict(ops.PLAN)
    yield chk
    ops.set_default_precision(old_prec)
    ops.PLAN.clear()
    ops.PLAN.update(old_plan)
    ops.PLAN_VERSION += 1


# ---- workloads (marconet_b200/testing/workloads.py; SUBSET runs the precision variants) -----------------------------------


@pytest.mark.parametrize("name", list(WORKLOADS))
def test_forward_calls_match_fp64(sweep, gpu_models, name):
    with torch.no_grad():
        WORKLOADS[name](gpu_models)
    DONE.add(name)


def _tc_layers(gm, sweep):
    from marconet_b200 import pipeline
    sweep.enabled = False                       # make sure every layer is packed (conv_layers lists packed weights)
    with torch.no_grad():
        for name in SUBSET:
            WORKLOADS[name](gm)
    sweep.enabled = True
    return [cw for cw in pipeline.conv_layers(gm["encoder"], gm["tspgan"], gm["sr"]) if cw.tc_capable()]


@pytest.mark.parametrize("variant", ["bf16x3", "fp32_simt", "x_scale"])
def test_precision_variants(sweep, gpu_models, variant):
    from marconet_b200 import ops
    layers = _tc_layers(gpu_models, sweep)
    saved = [(cw, cw.precision, cw.x_scale) for cw in layers]
    try:
        if variant == "bf16x3":
            for cw in layers:
                cw.set_plan(precision=ops.PREC_BF16X3_TC)
        elif variant == "fp32_simt":
            ops.set_default_precision(ops.PREC_FP32_SIMT)
        else:
            # random powers of two in 2^-6 .. 2^6, capped so that |x * x_scale| stays well inside fp16's range
            sweep.enabled = False
            with ops.calibration(_dev()) as cal, torch.no_grad():
                for name in SUBSET:
                    WORKLOADS[name](gpu_models)
            amax = {cw: r["absmax"] for cw, r in cal.results().items()}
            sweep.enabled = True
            rng = random.Random(5)
            for cw in layers:
                k = rng.randint(-6, 6)
                if cw in amax and amax[cw] > 0:
                    k = min(k, math.floor(math.log2(8192.0 / amax[cw])))
                cw.set_plan(x_scale=2.0 ** k)
        with torch.no_grad():
            for name in SUBSET:
                WORKLOADS[name](gpu_models)
        torch.cuda.synchronize()
        assert ops.poll_range(_dev(), reroute=False) == []
    finally:
        for cw, p, s in saved:
            cw.precision, cw.x_scale = p, s


def test_tap_pointers_equal_the_dense_taps(sweep, gpu_models):
    """TSPGAN with its two feature taps also stored through per-character pointers into separate local buffers (shuffled order):
    every buffer must hold exactly the tap the same call stored densely."""
    n = 6
    order = [3, 0, 5, 1, 4, 2]
    bufs = {64: [torch.full((64 * 64 * 256,), float("nan"), device=_dev()) for _ in range(n)],
            32: [torch.full((32 * 32 * 512,), float("nan"), device=_dev()) for _ in range(n)]}
    ptrs = {}
    for wdt, lst in bufs.items():
        for b in lst:
            sweep.tap_buffers[b.data_ptr()] = b
        ptrs[wdt] = torch.tensor([lst[order[i]].data_ptr() for i in range(n)], dtype=torch.int64, device=_dev())
    g = torch.Generator().manual_seed(8)
    styles = torch.randn(n, 512, generator=g).to(_dev())
    labels = torch.randint(0, 6735, (n, 1), generator=g)
    with torch.no_grad():
        _, f64, f32_ = gpu_models["tspgan"](styles=styles, labels=labels, noise=None, _tap_ptrs=ptrs)
    torch.cuda.synchronize()
    for wdt, dense in ((64, f64), (32, f32_)):
        nhwc = dense.permute(0, 2, 3, 1)
        for i in range(n):
            assert torch.equal(bufs[wdt][order[i]].view(wdt, wdt, -1), nhwc[i]), (wdt, i)
    assert any("y2_ptrs" in r["feats"] for r in RECORDS)


# ---- direct cases the modules never produce ---------------------------------------------------------------------------
def _cw(cout, cin, k, seed, name):
    from marconet_b200 import ops
    g = torch.Generator().manual_seed(seed)
    w4 = torch.randn(cout, cin, k, k, generator=g) / math.sqrt(cin * k * k)
    cw = ops.ConvWeight(w4.permute(2, 3, 1, 0).reshape(k * k * cin, cout).contiguous().to(_dev()), k * k, name=name)
    ops.PLAN.pop(name, None)
    return cw


def _t(*shape, seed, scale=1.0, shift=0.0):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(*shape, generator=g) * scale + shift).to(_dev())


@pytest.mark.parametrize("h,w", [(16, 8), (32, 4), (8, 8), (16, 16)])
def test_groupnorm_input_and_statistics_on_maps_of_several_samples_per_tile(sweep, h, w):
    """16x8 / 32x4 maps hold 128 pixels but their tiles hold two samples: the fused GroupNorm input and the epilogue statistics need
    one sample per tile, so both take the two-pass forms; 16x16 keeps the fused ones.  (Before ops.conv2d asked the plan, the
    16x8 / 32x4 calls raised RuntimeError.)"""
    from marconet_b200 import ops
    n, cin, cout = 3, 64, 64
    x = _t(n, h, w, cin, seed=1, scale=2.0, shift=0.3)
    vw = torch.tensor([w, max(1, w // 2), w - 1], dtype=torch.int32, device=_dev())
    mr = ops.groupnorm_stats(x, valid_w=vw)
    ops.conv2d(x, _cw(cout, cin, 3, 2, f"sweep.gn_{h}x{w}"), 3, 3, pad=(1, 1), bias=_t(cout, seed=3), valid_w=vw,
               gn=(mr, _t(cin, seed=4, scale=0.3, shift=1.0), _t(cin, seed=5, scale=0.2)), gn_stats=True, precision=ops.PREC_F16X3_TC)
    rec = RECORDS[-1]
    assert rec["branch"].startswith("tc2")
    fused = rec["plan"]["TN"] == 1
    assert fused == (h * w > 128), rec
    assert ("gn_fused" in rec["feats"]) == fused and ("gn_stats_out" in rec["feats"]) == fused, rec


@pytest.mark.parametrize("feature", ["plain", "gn_stats_valid_w", "y2_ptrs"])
@pytest.mark.parametrize("h,w", [(4, 16), (2, 32), (1, 64)])
def test_single_sample_tiles_of_64_pixels(sweep, h, w, feature):
    """4x16, 2x32 and 1x64 maps: a 3x3 halo of two samples would exceed the halo buffer, so the plan keeps one sample per tile and
    the tile holds 64 pixels (TH * TW = 64) of its 128 MMA rows.  The rows past the tile must not be stored: not into the next
    sample, not past the end of y (a guard sample after the output), not past a y2_ptrs destination (guard bands), and not into
    the epilogue statistics."""
    from marconet_b200 import ops
    n, cin, cout = 3, 64, 64
    x = _t(n, h, w, cin, seed=40, scale=1.5, shift=0.2)
    cw = _cw(cout, cin, 3, 41, f"sweep.tile64_{h}x{w}")
    out = torch.full((n + 1, h, w, cout), GUARD, device=_dev())[:n]          # the guard sample after y must stay untouched
    kw = dict(pad=(1, 1), bias=_t(cout, seed=42), out_scale=_t(n, cout, seed=43, scale=0.3, shift=1.0), act=ops.ACT_LRELU02,
              gain=2 ** 0.5, out=out, precision=ops.PREC_F16X3_TC)
    if feature == "gn_stats_valid_w":
        vw = torch.tensor([w, w // 2 + 1, 3], dtype=torch.int32, device=_dev())
        mr = ops.groupnorm_stats(x, valid_w=vw)
        kw.update(valid_w=vw, gn=(mr, _t(cin, seed=44, scale=0.3, shift=1.0), _t(cin, seed=45, scale=0.2)), gn_stats=True)
    elif feature == "y2_ptrs":
        blk, guard = h * w * cout, 4096
        big = torch.full((n * (blk + guard) + guard,), GUARD, device=_dev())
        dst = [big[guard + i * (blk + guard):guard + i * (blk + guard) + blk] for i in range(n)]
        sweep.guards[:] = [big[:guard]] + [big[guard + i * (blk + guard) + blk:guard + (i + 1) * (blk + guard)] for i in range(n)]
        for b in dst:
            sweep.tap_buffers[b.data_ptr()] = b
        kw.update(out2_ptrs=torch.tensor([b.data_ptr() for b in dst], dtype=torch.int64, device=_dev()),
                  y2_scale=_t(n, cout, seed=46))
    try:
        ops.conv2d(x, cw, 3, 3, **kw)          # the wrapper checks the guard sample after y and the guard bands
    finally:
        sweep.guards[:] = []
    torch.cuda.synchronize()
    rec = RECORDS[-1]
    assert (rec["plan"]["kernel"], rec["plan"]["TN"], rec["plan"]["TH"] * rec["plan"]["TW"]) == ("tc2", 1, 64), rec
    if feature == "gn_stats_valid_w":
        assert {"gn_fused", "gn_stats_out", "valid_w"} <= rec["feats"], rec
    if feature == "y2_ptrs":
        assert "y2_ptrs" in rec["feats"], rec


@pytest.mark.parametrize("act", ["tanh", "gelu", "sigmoid"])
@pytest.mark.parametrize("shape,branch", [((4, 32, 32, 64, 128), "tc2/nt64"), ((16, 64, 64, 64, 128), "tc2/nt128"),
                                          ((5, 4, 4, 64, 64), "tc2/nt64/TN>1")], ids=["tc2_nt64", "tc2_nt128", "tc2_TN4"])
def test_tc2_runtime_activation_and_broadcast_residual(sweep, act, shape, branch):
    """tanh / GELU / sigmoid (the epilogue's run-time activation) with a residual broadcast over the batch, on the dense one-sample
    tile path at both tile widths and on the per-row path of a multi-sample tile."""
    from marconet_b200 import ops
    n, h, w, cin, cout = shape
    a = {"tanh": ops.ACT_TANH, "gelu": ops.ACT_GELU, "sigmoid": ops.ACT_SIGMOID}[act]
    ops.conv2d(_t(n, h, w, cin, seed=10), _cw(cout, cin, 3, 11, f"sweep.act_{act}_{n}"), 3, 3, pad=(1, 1), bias=_t(cout, seed=12),
               out_scale=_t(n, cout, seed=13, scale=0.3, shift=1.0), residual=_t(1, h, w, cout, seed=14), res_broadcast=True, act=a,
               gain=1.5, precision=ops.PREC_F16X3_TC)
    rec = RECORDS[-1]
    assert rec["branch"] == branch and {"runtime_act", "res_broadcast"} <= rec["feats"], rec


@pytest.mark.parametrize("h,w", [(6, 128), (12, 256)])
def test_per_tap_tiling_with_the_full_epilogue(sweep, h, w):
    """The per-tap tiling (maps the halo tiling cannot cover) with demodulation, residual, y2 and ragged windows."""
    from marconet_b200 import ops
    n, cin, cout = 3, 64, 128
    buf = torch.zeros(n, h, w, cout + 64, device=_dev())
    vw = torch.tensor([w, w // 2 + 3, 17], dtype=torch.int32, device=_dev())
    ops.conv2d(_t(n, h, w, cin, seed=20), _cw(cout, cin, 3, 21, f"sweep.tc1_{h}"), 3, 3, pad=(1, 1), bias=_t(cout, seed=22),
               out_scale=_t(n, 2 * cout, seed=23, scale=0.3, shift=1.0)[:, cout:], residual=_t(n, h, w, cout, seed=24),
               act=ops.ACT_LRELU02, gain=2 ** 0.5, out=buf[..., 32:32 + cout], out2=True, y2_scale=_t(n, cout, seed=25), valid_w=vw,
               precision=ops.PREC_F16X3_TC)
    assert RECORDS[-1]["branch"] == "tc1", RECORDS[-1]


@pytest.mark.parametrize("ratio", [1, 30, 300, 3000])
def test_epilogue_groupnorm_statistics_of_offset_data(sweep, ratio):
    """Epilogue GroupNorm statistics on outputs whose mean is ``ratio`` times their std, against fp64.  Plain fp32 sums of y and y*y
    lost the variance to cancellation here (1.2e-3 relative error at 300); the epilogue now sums about a pivot (conv_tc2.cu GnAcc)."""
    from marconet_b200 import ops
    n, h, w, cin, cout = 2, 32, 32, 128, 128
    bias = torch.full((cout,), float(ratio), device=_dev())
    y, mr = ops.conv2d(_t(n, h, w, cin, seed=30), _cw(cout, cin, 3, 31, "sweep.stats"), 3, 3, pad=(1, 1), bias=bias, gn_stats=True,
                       precision=ops.PREC_F16X3_TC)
    rec = RECORDS[-1]
    print(f"\nmean/std ~ {ratio}: GroupNorm statistics error {rec['stats_err']:.3e} (|d mean| * rstd, |d rstd| / rstd)")
    assert "gn_stats_out" in rec["feats"]


def test_coverage_and_negative_controls(sweep, gpu_models):
    """Runs any workload this session skipped, then: every branch and feature was seen, every negative control failed."""
    for name, fn in WORKLOADS.items():
        if name not in DONE:
            with torch.no_grad():
                fn(gpu_models)
            DONE.add(name)
    table = collections.defaultdict(lambda: [0, 0.0])
    feats_all = sorted({f for r in RECORDS for f in r["feats"]})
    for r in RECORDS:
        for f in ["*"] + sorted(r["feats"]):
            cell = table[(r["branch"], f)]
            cell[0] += 1
            cell[1] = max(cell[1], r["ratio"])
    branches = sorted({r["branch"] for r in RECORDS})
    cols = ["*"] + feats_all
    print("\nbranch x feature: calls / worst error-to-tolerance ratio")
    print(f"{'branch':24s}" + "".join(f"{c[:14]:>16s}" for c in cols))
    for b in branches:
        print(f"{b:24s}" + "".join(f"{table[(b, c)][0]:>7d}/{table[(b, c)][1]:<8.3f}" if (b, c) in table else f"{'':>16s}" for c in cols))
    print("worst |y - ref| / bound per precision:", {k: f"{v:.3e}" for k, v in sorted(WORST_ERR.items())})
    print(f"worst GroupNorm statistics error: {WORST_STATS[0]:.3e}")
    print("negative controls (failed as they must):", {b: c for b, c in sorted(CONTROLS.items())})
    seen = {r["branch"] for r in RECORDS}
    kinds = {"small": "small", "simt": "simt", "simt+splitK": "simt+splitK", "tc1": "tc1",
             "tc2 nt64": "tc2/nt64", "tc2 nt128": "tc2/nt128", "tc2 TN>1": "/TN>1", "tc2 split-K": "tc2/nt"}
    for label, key in kinds.items():
        if label == "tc2 split-K":
            ok = any(b.startswith("tc2") and b.endswith("+splitK") for b in seen)
        elif key.startswith("/"):
            ok = any(key in b for b in seen)
        elif label.startswith("tc2"):
            ok = any(b.startswith(key) for b in seen)
        else:
            ok = key in seen
        assert ok, f"no call ran the {label} branch: {sorted(seen)}"
    fs = {f for r in RECORDS for f in r["feats"]}
    for f in ("gn_fused", "gn_stats_out", "y2_ptrs", "want_y=False", "runtime_act", "x_scale"):
        assert f in fs, f"no call exercised {f}"
    for b in seen - {"linear", "patch_embed"}:
        assert CONTROLS[b], f"branch {b}: no call suited a negative control"
        assert all(failed for _, failed in CONTROLS[b]), f"branch {b}: a negative control passed the comparison: {CONTROLS[b]}"
