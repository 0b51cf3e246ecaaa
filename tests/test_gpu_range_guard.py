"""The fp16 hi/lo split's range management (DESIGN.md §4b) across the tensor-core plan space and through recorded forwards.

The default convolution precision keeps fp32's mantissa but only fp16's exponent range.  What keeps it safe on other checkpoints
is checked here against exact or fp64 references, at the geometries of the plan-space test (test_gpu_conv_plan_space.GEOMS):
  1. the calibration maxima (mn_conv_params.x_absmax, read by pipeline.tune_precision) equal max |x| bit for bit at f16x3 and
     bf16x3, input scales 1, 2^-3 and 2^5, CTA caps 1 and 7, with 1e30 in the channels beside the slice; with the fused GroupNorm
     input they match the fp64 max |swish(GroupNorm(x))| over each sample's valid window;
  2. the range flag at its boundary: 65504 raises (f16x3, f16x1) and its fp32 predecessor does not; with x_scale 2^-1 the boundary
     moves to 131008; bf16x3 raises on Inf only (not 3e38, not NaN); one planted element at the first and the last element and in
     the last k-slice of split-K; Inf outside the channel slice and a GroupNorm input beyond valid_w never raise, and poll_range
     names exactly the layer;
  3. the input scale where it matters: |x| up to 1.2e5 at 2^-6, |x| ~ 2^-14 at 2^14 and the fused GroupNorm input at 2^-6 / 2^6,
     every output element against fp64 within the plan-space tolerance;
  4. plan changes and overflows reach the recorded module forwards, GraphedLines and restore_lines;
  5. two live layers whose tags are congruent modulo the slot count are both reported.
The last test prints the geometry x precision x check table, asserts that tests 1-3 saw every planner outcome and that every
negative control (a maximum without the last channel block, without the last sample, over the masked columns; an unscaled tiny
input) failed."""
import collections
import math
import warnings

import pytest
import torch

from oracle import conv_ref as R
from test_gpu_conv_plan_space import GEOMS, TOL, _cw, _epilogue, _guarded, _plan_str, _t, restore_cap  # noqa: F401 (fixture)

pytestmark = pytest.mark.gpu

SCALES = (1.0, 2.0 ** -3, 2.0 ** 5)
CAPS = (1, 7)
PRECS = ("f16x3", "bf16x3")
# |absmax - fp64| / fp64 of the fused GroupNorm input (__expf / __fdividef in the swish): 4x the worst of the first H100 run
TOL_GN_AMAX = 7.2e-7           # worst 1.78e-7

RECORDS = []                                   # dict(test, geom, prec, check, plan)
CONTROLS = collections.defaultdict(list)       # control -> [failed as it must]
NONFINITE = collections.defaultdict(list)      # (precision, planted value, activation) -> [output held Inf / NaN]
WORST = collections.defaultdict(float)
DONE = set()


def _dev():
    return torch.device("cuda:0")


def _prec(name):
    from marconet_b200 import ops
    return {"f16x3": ops.PREC_F16X3_TC, "bf16x3": ops.PREC_BF16X3_TC, "f16x1": ops.PREC_F16X1_TC}[name]


def _ids():
    return ["x".join(map(str, g[:3])) + f"_{g[3]}-{g[4]}_k{g[5]}" for g in GEOMS]


def _slice(src, fill):
    """src [N, H, W, C] copied into channels [32, 32 + C) of a wider buffer whose other channels hold ``fill``: (x, buffer)."""
    n, h, w, c = src.shape
    buf = torch.full((n, h, w, c + 64), fill, device=_dev())
    x = buf[..., 32:32 + c]
    x.copy_(src)
    return x, buf


def _conv(x, cw, k, prec, **kw):
    from marconet_b200 import ops
    plan = {}
    y = ops.conv2d(x, cw, k, k, pad=(k // 2, k // 2), precision=prec, plan=plan, **kw)
    torch.cuda.synchronize()
    return y, plan


def _note(test, gi, prec, check, plan):
    RECORDS.append(dict(test=test, geom=gi, prec=prec, check=check, plan=dict(plan)))


def _gn_fusable(plan):
    return plan["kernel"] == "tc2" and plan["TN"] == 1           # the halo tiling with one sample per pixel tile


def _calibrated(x, cw, k, prec, **kw):
    from marconet_b200 import ops
    with ops.calibration(_dev()) as cal:
        _, plan = _conv(x, cw, k, prec, **kw)
    return cal.results()[cw]["absmax"], plan


def _swish_gn64(x0, gn, vw=None):
    """|swish(GroupNorm(x))| in fp64, zero beyond valid_w (vw None: every column)."""
    mr, gamma, beta = (t.double() for t in gn)
    n, h, w, cin = x0.shape
    grp = torch.arange(cin, device=x0.device) // 32
    t = (x0.double() - mr[:, grp, 0][:, None, None, :]) * mr[:, grp, 1][:, None, None, :] * gamma[:cin] + beta[:cin]
    s = (t * torch.sigmoid(t)).abs()
    if vw is not None:
        s = s * (torch.arange(w, device=x0.device)[None, :] < vw.long()[:, None])[:, None, :, None]
    return s


# ---- 1. calibration maxima ---------------------------------------------------------------------------------------------------

def _run_absmax(gi, set_cap):
    n, h, w, cin, cout, k = GEOMS[gi]
    where = f"{GEOMS[gi]}"
    src = _t(n, h, w, cin, seed=1000 + gi, scale=1.5, shift=0.1)
    src[-1, h // 2, w // 2, cin - 7] = -100.0               # the unique maximum: last channel block of the last sample
    x, _ = _slice(src, 1e30)                                 # a read outside the slice would report 1e30
    want = float(src.abs().max())
    assert want == 100.0
    without = dict(last_channel_block=float(src[..., :cin - 64].abs().max()) if cin > 64 else 0.0,
                   last_sample=float(src[:-1].abs().max()) if n > 1 else 0.0)
    cw = _cw(cout, cin, k, 1100 + gi, f"range_guard.amax{gi}")
    plan0 = None
    for prec_name in PRECS:
        for s in SCALES:
            cw.x_scale = s
            got, plan = _calibrated(x, cw, k, _prec(prec_name))
            assert got == want, f"{where} {prec_name} x_scale {s:g}: calibration max {got!r}, max |x| {want!r}"
            _note("amax", gi, prec_name, f"amax xs={s:g}", plan)
            for name, v in without.items():
                CONTROLS["amax without " + name].append(v != got)
            plan0 = plan0 or plan
        cw.x_scale = 1.0
    try:
        for c in CAPS:
            set_cap(c)
            got, plan = _calibrated(x, cw, k, _prec("f16x3"))
            assert got == want, f"{where} cap {c}: calibration max {got!r}, max |x| {want!r}"
            _note("amax", gi, "f16x3", f"amax cap{c}", plan)
    finally:
        set_cap(0)
    if not _gn_fusable(plan0):
        return
    # the fused GroupNorm input: the maximum is taken after the transform, inside the image and each sample's valid window
    vw = _epilogue(gi, n, h, w, cout)["valid_w"]
    g_src = _t(n, h, w, cin, seed=1200 + gi, scale=1.5, shift=0.1)
    mr = R.groupnorm_stats64(g_src, valid_w=vw.tolist()).float()
    gn = (mr, _t(cin, seed=1300 + gi, scale=0.3, shift=1.0), _t(cin, seed=1400 + gi, scale=0.2))
    s_beyond = next((i for i in range(n) if int(vw[i]) < w), None)
    if s_beyond is not None:                                 # the transformed unique maximum, one column beyond the window
        g_src[s_beyond, h // 2, int(vw[s_beyond]), cin - 7] = 40.0 * float(mr[s_beyond, -1, 1]) ** -1 + float(mr[s_beyond, -1, 0])
    xg, _ = _slice(g_src, 1e30)
    ref = float(_swish_gn64(g_src, gn, vw).max())
    ref_all = float(_swish_gn64(g_src, gn).max())
    for prec_name in PRECS:
        for s in SCALES:
            cw.x_scale = s
            got, plan = _calibrated(xg, cw, k, _prec(prec_name), gn=gn, valid_w=vw)
            assert plan["gn_fused"], plan
            err = abs(got - ref) / ref
            WORST["gn absmax rel"] = max(WORST["gn absmax rel"], err)
            assert err <= TOL_GN_AMAX, f"{where} {prec_name} x_scale {s:g} gn: calibration max {got!r}, fp64 {ref!r}"
            _note("amax", gi, prec_name, f"amax gn xs={s:g}", plan)
            if s_beyond is not None:
                CONTROLS["gn amax over the masked columns"].append(abs(got - ref_all) / ref_all > TOL_GN_AMAX)
        cw.x_scale = 1.0


@pytest.mark.parametrize("gi", range(len(GEOMS)), ids=_ids())
def test_calibration_maxima_are_exact(restore_cap, gi):
    _run_absmax(gi, restore_cap)
    DONE.add(("amax", gi))


# ---- 2. the range flag at its boundary -----------------------------------------------------------------------------------

_F16_MAX = 65504.0
_F16_BELOW = float(torch.nextafter(torch.tensor(_F16_MAX), torch.tensor(0.0)))       # 65503.996: fp32's predecessor
# (precision, x_scale, planted |value|, raises)
FLAG_CASES = [("f16x3", 1.0, _F16_MAX, True), ("f16x3", 1.0, _F16_BELOW, False), ("f16x1", 1.0, _F16_MAX, True),
              ("f16x1", 1.0, _F16_BELOW, False), ("f16x3", 0.5, _F16_MAX, False), ("f16x3", 0.5, 2 * _F16_MAX, True),
              ("bf16x3", 1.0, 3e38, False), ("bf16x3", 1.0, math.inf, True), ("bf16x3", 1.0, math.nan, False)]
# planted values that really overflow their split: what the overflowed call's own output holds, per activation
OVERFLOWS = [("f16x3", 2 * _F16_MAX), ("f16x1", 2 * _F16_MAX), ("bf16x3", math.inf)]


def _expect_flag(cw, raised, where):
    from marconet_b200 import ops
    hits = ops.poll_range(_dev(), reroute=False)
    assert hits == ([cw] if raised else []), f"{where}: poll_range gave {[h.name for h in hits]}, expected {'[layer]' if raised else '[]'}"
    assert ops.poll_range(_dev(), reroute=False) == [], f"{where}: poll_range did not clear the flag"


def _run_flag(gi):
    from marconet_b200 import ops
    n, h, w, cin, cout, k = GEOMS[gi]
    base = _t(n, h, w, cin, seed=2000 + gi, scale=1.5).clamp(-4.0, 4.0)
    x, buf = _slice(base, 0.0)
    cw = _cw(cout, cin, k, 2100 + gi, f"range_guard.flag{gi}")
    ops.poll_range(_dev(), reroute=False)
    _, plan0 = _conv(x, cw, k, _prec("f16x3"))
    _expect_flag(cw, False, f"{GEOMS[gi]} benign input")
    positions = {"first": ((0, 0, 0, 0), 1.0), "last": ((n - 1, h - 1, w - 1, cin - 1), -1.0)}
    if plan0["splits"] > 1:                                  # the middle of the last k-slice
        positions["last k-slice"] = ((n // 2, h // 2, w // 2, cin - (cin // plan0["splits"]) // 2), 1.0)
    for pos_name, (pos, sign) in positions.items():
        for prec_name, xs, val, raises in FLAG_CASES:
            where = f"{GEOMS[gi]} {prec_name} x_scale {xs:g}: {sign * val!r} at {pos_name} {pos}"
            cw.x_scale = xs
            x[pos] = sign * val
            _, plan = _conv(x, cw, k, _prec(prec_name))
            x[pos] = base[pos]
            _expect_flag(cw, raises, where)
            _note("flag", gi, prec_name, f"flag {pos_name}", plan)
        cw.x_scale = 1.0
    # what an overflowed call's own output holds: the flag is the guarantee, the output is only sometimes visibly wrong
    for prec_name, val in OVERFLOWS:
        for act in (ops.ACT_NONE, ops.ACT_RELU, ops.ACT_LRELU02):
            x[0, 0, 0, 0] = val
            y, plan = _conv(x, cw, k, _prec(prec_name), act=act)
            x[0, 0, 0, 0] = base[0, 0, 0, 0]
            _expect_flag(cw, True, f"{GEOMS[gi]} {prec_name} {val!r} act {act}")
            NONFINITE[(prec_name, val, R.ACT_NAMES[act])].append(not bool(torch.isfinite(y).all()))
    # Inf in the channels beside the slice is never read: no flag at either precision
    for c in (31, 32 + cin):
        buf[n - 1, h - 1, w - 1, c] = math.inf
        buf[0, 0, 0, c] = -math.inf
    for prec_name in ("f16x3", "bf16x3"):
        _, plan = _conv(x, cw, k, _prec(prec_name))
        _expect_flag(cw, False, f"{GEOMS[gi]} {prec_name}: Inf outside the channel slice")
        _note("flag", gi, prec_name, "flag out-of-slice", plan)
    buf[..., :32] = 0.0
    buf[..., 32 + cin:] = 0.0
    if not _gn_fusable(plan0):
        return
    # the fused GroupNorm input: the guard sees the transformed value, and nothing beyond valid_w.  mean 0, rstd 1, gamma 100:
    # the benign |x| <= 4 stays below 400, a raw 1000 (inside fp16's range) becomes 1e5 after the transform
    vw = _epilogue(gi, n, h, w, cout)["valid_w"]
    mr = torch.stack([torch.zeros(n, cin // 32), torch.ones(n, cin // 32)], -1).to(_dev())
    gn = (mr, torch.full((cin,), 100.0, device=_dev()), torch.zeros(cin, device=_dev()))
    placements = [("inside", (0, 0, 0, 0), True)]
    s_beyond = next((i for i in range(n) if int(vw[i]) < w), None)
    if s_beyond is not None:
        placements.append(("beyond valid_w", (s_beyond, h - 1, int(vw[s_beyond]), cin - 1), False))
    for name, pos, raises in placements:
        x[pos] = 1000.0
        _, plan = _conv(x, cw, k, _prec("f16x3"), gn=gn, valid_w=vw)
        x[pos] = base[pos]
        assert plan["gn_fused"], plan
        _expect_flag(cw, raises, f"{GEOMS[gi]} gn: raw 1000 {name} {pos}")
        _note("flag", gi, "f16x3", f"flag gn {name}", plan)


@pytest.mark.parametrize("gi", range(len(GEOMS)), ids=_ids())
def test_range_flag_at_its_boundary(gi):
    _run_flag(gi)
    DONE.add(("flag", gi))


# ---- 3. the input scale where it matters ----------------------------------------------------------------------------------

def _check(got, ref, key, tol, where):
    r = R.ratio(got, ref[key], ref["bound" if key == "y" else "bound2"], tol)
    assert r <= 1.0, f"{where} {key}: error / tolerance {r:.3g}"
    return r


def _run_xscale(gi, prec_name):
    from marconet_b200 import ops
    n, h, w, cin, cout, k = GEOMS[gi]
    prec, tol = _prec(prec_name), TOL[_prec(prec_name)]
    cw = _cw(cout, cin, k, 3100 + gi, f"range_guard.xscale{gi}")
    epi = _epilogue(gi, n, h, w, cout)
    act, gain = epi.pop("act"), epi.pop("gain")
    y, y2 = _guarded(n, h, w, cout), _guarded(n, h, w, cout)
    ops.poll_range(_dev(), reroute=False)

    def run(src, xs, gn=None, mag=1.0):
        """The call at input scale xs; bias and residual scaled by ``mag`` so that the dot products dominate the bound."""
        x, _ = _slice(src, math.nan)
        opts = dict(epi, bias=epi["bias"] * mag, residual=epi["residual"] * mag)
        cw.x_scale = xs
        y.fill_(math.nan)
        y2.fill_(math.nan)
        plan = {}
        ops.conv2d(x, cw, k, k, pad=(k // 2, k // 2), out=y, out2=y2, precision=prec, plan=plan, act=act, gain=gain, gn=gn, **opts)
        torch.cuda.synchronize()
        cw.x_scale = 1.0
        ref = R.conv_ref_full(src, cw.w, k, k, (1, 1), (k // 2, k // 2), gn=gn, act=act, gain=gain, **opts)
        return plan, ref

    big = _t(n, h, w, cin, seed=3000 + gi, scale=2.5e4).clamp(-1.2e5, 1.2e5)
    big[0, 0, 0, 0] = 1.2e5                                # beyond fp16's range whatever the sample
    tiny = _t(n, h, w, cin, seed=3200 + gi, scale=2.0 ** -14)
    for name, src, xs, mag in (("|x| <= 1.2e5", big, 2.0 ** -6, 1.0), ("|x| ~ 2^-14", tiny, 2.0 ** 14, 2.0 ** -14)):
        where = f"{GEOMS[gi]} {prec_name} {name} x_scale {xs:g}"
        plan, ref = run(src, xs, mag=mag)
        _check(y, ref, "y", tol, where)
        _check(y2, ref, "y2", tol, where)
        _expect_flag(cw, False, where)
        _note("xscale", gi, prec_name, f"xscale {name}", plan)
    if prec_name == "f16x3":                                # the reason for the scale: unscaled, hi and lo fall into fp16 subnormals
        plan, ref = run(tiny, 1.0, mag=2.0 ** -14)
        CONTROLS["tiny input at x_scale 1"].append(R.ratio(y, ref["y"], ref["bound"], tol) > 1.0)
    if not _gn_fusable(plan):
        return
    g_src = _t(n, h, w, cin, seed=3300 + gi, scale=1.5, shift=0.1)
    mr = R.groupnorm_stats64(g_src, valid_w=epi["valid_w"].tolist()).float()
    gn = (mr, _t(cin, seed=3400 + gi, scale=0.3, shift=1.0), _t(cin, seed=3500 + gi, scale=0.2))
    for xs in (2.0 ** -6, 2.0 ** 6):
        where = f"{GEOMS[gi]} {prec_name} gn x_scale {xs:g}"
        plan, ref = run(g_src, xs, gn=gn)
        assert plan["gn_fused"], plan
        _check(y, ref, "y", tol, where)
        _check(y2, ref, "y2", tol, where)
        _expect_flag(cw, False, where)
        _note("xscale", gi, prec_name, f"xscale gn {xs:g}", plan)


@pytest.mark.parametrize("prec_name", PRECS)
@pytest.mark.parametrize("gi", range(len(GEOMS)), ids=_ids())
def test_input_scale_where_it_matters(gi, prec_name):
    _run_xscale(gi, prec_name)
    DONE.add(("xscale", gi, prec_name))


# ---- 4. plan changes and overflows through recorded forwards ---------------------------------------------------------------

@pytest.fixture
def fresh_plan():
    """An empty precision plan for fresh modules; the session's plan comes back afterwards (layer names are shared)."""
    from marconet_b200 import ops
    saved = dict(ops.PLAN)
    ops.PLAN.clear()
    try:
        yield
    finally:
        ops.poll_range(_dev(), reroute=False)
        ops.PLAN.clear()
        ops.PLAN.update(saved)


def _fresh(checkpoints, sd_encoder=None):
    from marconet_b200.models import networks
    out = {}
    for key, cls in (("tspgan", networks.TSPGAN), ("encoder", networks.TextContextEncoderV2), ("sr", networks.TSPSRNet)):
        m = cls()
        m.load_state_dict(sd_encoder if (key == "encoder" and sd_encoder is not None) else checkpoints[key], strict=True)
        out[key] = m.eval().to(_dev())
    return out


def _clone(res):
    return tuple(t.clone() for t in (res if isinstance(res, tuple) else (res,)))


def _same(a, b):
    return all(torch.equal(u, v) for u, v in zip(a, b))


def _tc_layer(call):
    """The deepest layer that one call launches on the tensor cores (a calibration sees exactly those)."""
    from marconet_b200 import ops
    with ops.calibration(_dev()) as cal:
        call()
    torch.cuda.synchronize()
    return list(cal.slots)[-1]


def test_plan_changes_reach_recorded_forwards(checkpoints, monkeypatch, fresh_plan):
    """Eager, recorded and replayed calls; then one layer's plan changes: every later call (eager, recorded, replayed under the new
    graph key) equals an eager call under that plan and differs from the first results; restoring the plan is a new recording that
    gives the first results' bytes again."""
    from marconet_b200 import ops
    from oracle import synth
    assert ops.MODULE_GRAPHS
    nets = _fresh(checkpoints)
    lq = synth.make_lq(1, 0).to(_dev())
    locs = synth.make_locs(1, 4, ragged=True, seed=2).to(_dev())
    _, _, w = nets["encoder"](lq)
    _, f64, f32_ = nets["tspgan"](styles=w.repeat(4, 1), labels=synth.make_labels(4, 3), noise=None)
    f64, f32_ = f64.clone(), f32_.clone()
    calls = {"encoder": (nets["encoder"], lambda: nets["encoder"](lq)), "sr": (nets["sr"], lambda: nets["sr"](lq, [f64], [f32_], locs))}
    for key, (module, call) in calls.items():
        first = [_clone(call()) for _ in range(3)]           # eager, records, replays
        assert all(_same(r, first[0]) for r in first[1:]), key
        layer = _tc_layer(call)
        for change in (dict(precision=ops.PREC_FP32_SIMT), dict(x_scale=2.0 ** -16)):
            where = f"{key}: {layer.name} {change}"
            layer.set_plan(**change)
            got = [_clone(call()) for _ in range(3)]
            assert any(k[1] == ops.graph_key() for k in module._mg), f"{where}: no recording under the new plan"
            monkeypatch.setattr(ops, "MODULE_GRAPHS", False)
            eager = _clone(call())
            monkeypatch.setattr(ops, "MODULE_GRAPHS", True)
            for i, g in enumerate(got):
                assert _same(g, eager), f"{where}: call {i + 1} differs from an eager call under the same plan"
            assert not _same(eager, first[0]), f"{where}: the plan change did not change the result"
            version = ops.PLAN_VERSION
            layer.set_plan(precision=ops.default_precision(), x_scale=1.0)
            assert ops.PLAN_VERSION > version
            back = [_clone(call()) for _ in range(3)]
            assert any(k[1] == ops.graph_key() for k in module._mg), f"{where}: restoring the plan made no new recording"
            for i, b in enumerate(back):
                assert _same(b, first[0]), f"{where}: call {i + 1} after restoring the plan differs from the first results"
        RECORDS.append(dict(test="modules", geom=None, prec=None, check=f"plan change {key}", plan=None))


def _rerouted_until_clean(call, attempts=16):
    """call() until a synchronised call leaves no flag (each call's module forwards re-route what the previous one flagged).  One
    overflow hides the next (its NaN becomes 0 after a ReLU), so a line x1000 takes several rounds."""
    from marconet_b200 import ops
    seen = []
    for i in range(attempts):
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            res = call()
        torch.cuda.synchronize()
        flags = ops.range_flags(_dev()).numpy()
        if not flags.any():
            return res, i + 1
        seen.append([(c.name, c.precision, c.x_scale) if c is not None else int(t)
                     for t in flags[flags != 0] for c in [ops.ConvWeight.from_tag(int(t))]])
    raise AssertionError(f"still flagged after {attempts} calls: {seen}")


def test_overflow_inside_a_replayed_forward_is_rerouted(checkpoints, monkeypatch, fresh_plan):
    """A recorded encoder forward replayed on a line x1000 (the BN-free ReLU ResNet is positively homogeneous, its tensor-core layers
    leave fp16's range): the flag rises, the next call re-routes the layers, a new recording follows, and its logits and w are
    finite and equal an eager call under the re-routed plan."""
    from marconet_b200 import ops
    from oracle import synth
    enc = _fresh(checkpoints)["encoder"]
    lq = synth.make_lq(1, 0).to(_dev())
    ops.poll_range(_dev(), reroute=False)
    for _ in range(3):
        enc(lq)
    torch.cuda.synchronize()
    assert ops.poll_range(_dev(), reroute=False) == []
    recorded = set(enc._mg)
    big = lq * 1000.0
    enc(big)                                                  # same signature: the recording replays
    torch.cuda.synchronize()
    assert set(enc._mg) == recorded
    flags = ops.range_flags(_dev()).numpy()
    raised = {ops.ConvWeight.from_tag(int(t)) for t in flags[flags != 0]}
    assert raised and all(c is not None and c.name.startswith("encoder.resnet") for c in raised), raised
    n_events = len(ops.RANGE_EVENTS)
    _, rounds = _rerouted_until_clean(lambda: enc(big))        # re-routes at its start, then runs eagerly under the new plan
    rerouted = {name for name, what in ops.RANGE_EVENTS[n_events:] if what == "rerouted to bf16x3"}
    assert {c.name for c in raised} <= rerouted, sorted({c.name for c in raised} - rerouted)
    res = [_clone(enc(big)) for _ in range(3)]                  # records, replays
    out = res[-1]
    assert len(set(enc._mg) - recorded) >= 1, "no new recording after the re-route"
    assert all(_same(r, res[0]) for r in res[1:]), "recorded / replayed calls under the re-routed plan differ"
    monkeypatch.setattr(ops, "MODULE_GRAPHS", False)
    eager = _clone(enc(big))
    torch.cuda.synchronize()
    logits, _, w = out
    assert torch.isfinite(logits).all() and torch.isfinite(w).all()
    assert _same(out, eager), "the re-routed replay differs from an eager call under the same plan"
    print(f"\nreplayed x1000 line: {len(raised)} layers flagged, {len(rerouted)} re-routed, clean after {rounds} round(s)")
    RECORDS.append(dict(test="modules", geom=None, prec=None, check=f"replay overflow rounds={rounds}", plan=None))


def test_graphed_lines_raise_after_an_overflowing_replay(checkpoints, fresh_plan):
    """GraphedLines bakes the plan in: check() raises FloatingPointError after a replay of the x1000 line, and a GraphedLines built
    afterwards (on the re-routed plan) is finite."""
    from marconet_b200 import ops
    from marconet_b200.graph import GraphedLines
    from oracle import synth
    nets = _fresh(checkpoints)
    lq, labels, locs = synth.make_lq(1, 0).to(_dev()), synth.make_labels(16, 0), synth.make_locs(1, 16).to(_dev())
    ops.poll_range(_dev(), reroute=False)
    g = GraphedLines(nets["encoder"], nets["tspgan"], nets["sr"], lines=1, chars=16)
    g(lq, labels, locs)
    g.check()
    g(lq * 1000.0, labels, locs)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        with pytest.raises(FloatingPointError):
            g.check()
    del g

    def rebuilt():
        g2 = GraphedLines(nets["encoder"], nets["tspgan"], nets["sr"], lines=1, chars=16)
        g2(lq * 1000.0, labels, locs)
        torch.cuda.synchronize()
        return g2

    g2, rounds = _rerouted_until_clean(rebuilt)
    g2.check()
    for key in ("sr", "logits", "w"):
        assert torch.isfinite(g2.outputs[key]).all(), key
    print(f"\nGraphedLines on the x1000 line: finite after {rounds} rebuild(s)")
    RECORDS.append(dict(test="modules", geom=None, prec=None, check=f"GraphedLines rebuilds={rounds}", plan=None))


@pytest.mark.parametrize("case", ["stem_x1000", "line_x1000"])
def test_restore_lines_out_of_range_needs_no_tuning(checkpoints, fresh_plan, case):
    """The x1000-stem checkpoint, and the regular one on a line x1000 (activations ~1e6), on a fresh plan:
    restore_lines(check_range=True) re-routes and re-runs until a run is clean, without pipeline.tune_precision.  The line x1000
    needs more re-runs than the three the loop once allowed: one overflow hides the next behind a ReLU."""
    from marconet_b200 import ops, pipeline
    from oracle import synth
    sd = None
    if case == "stem_x1000":
        sd = {k: v.clone() for k, v in checkpoints["encoder"].items()}
        sd["resnet.conv1.weight"] = sd["resnet.conv1.weight"] * 1000.0
    nets = _fresh(checkpoints, sd_encoder=sd)
    lq, labels, locs = synth.make_lq(1, 0).to(_dev()), [synth.make_labels(3, 0)], synth.make_locs(1, 3).to(_dev())
    if case == "line_x1000":
        lq = lq * 1000.0
    ops.poll_range(_dev(), reroute=False)
    n_events = len(ops.RANGE_EVENTS)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        out = pipeline.restore_lines(nets["encoder"], nets["tspgan"], nets["sr"], lq, labels, locs, check_range=True)
    events = ops.RANGE_EVENTS[n_events:]
    assert events, f"{case} raised no flag"
    for key in ("sr", "logits", "w"):
        assert torch.isfinite(out[key]).all(), f"{case}: {key} not finite after {len(events)} re-routes"
    # the returned result is the run of the final plan: a run under that plan raises no flag and gives the same bytes (a result
    # of a step in which a module's own poll re-routed an earlier layer would differ by far more)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        again = pipeline.restore_lines(nets["encoder"], nets["tspgan"], nets["sr"], lq, labels, locs, check_range=False)
    torch.cuda.synchronize()
    assert ops.poll_range(_dev(), reroute=False) == [], f"{case}: the returned plan still overflows"
    for key in ("sr", "logits", "w"):
        assert torch.equal(again[key], out[key]), f"{case}: {key} of the returned run differs from a run under the final plan"
    print(f"\nrestore_lines {case}: {len(events)} layers re-routed: {[name for name, _ in events]}")
    RECORDS.append(dict(test="modules", geom=None, prec=None, check=f"restore_lines {case} reroutes={len(events)}", plan=None))


# ---- 5. range slots ---------------------------------------------------------------------------------------------------------

def test_layers_with_congruent_tags_are_both_reported():
    """Two live layers whose tags are congruent modulo the slot count both overflow in one synchronised step: poll_range names
    both (with slots taken from tag % slots, the later writer hid the other, which stayed on the fp16 split)."""
    from marconet_b200 import ops
    a = _cw(64, 64, 3, 4000, "range_guard.slot_a")
    ops.ConvWeight._next_tag = a.tag + ops._RANGE_SLOTS
    b = _cw(64, 64, 3, 4001, "range_guard.slot_b")
    assert a.tag % ops._RANGE_SLOTS == b.tag % ops._RANGE_SLOTS
    x = _t(2, 16, 16, 64, seed=4002).clamp(-4.0, 4.0)
    x[1, 3, 5, 7] = 1e5
    ops.poll_range(_dev(), reroute=False)
    for cw in (a, b):
        ops.conv2d(x, cw, 3, 3, pad=(1, 1), precision=ops.PREC_F16X3_TC)
    torch.cuda.synchronize()
    hits = ops.poll_range(_dev(), reroute=False)
    assert sorted(c.name for c in hits) == [a.name, b.name], [c.name for c in hits]


# ---- 6. coverage --------------------------------------------------------------------------------------------------------------

def _outcomes(plan):
    out = {"tc1 per-tap" if plan["kernel"] == "tc1" else f"tc2 nt{plan['nt']}"}
    if plan["TN"] > 1:
        out.add("TN>1")
    if plan["splits"] > 1:
        out.add("split-K")
    if plan["cs"] == 2 and plan["m_tiles"] % 2 == 1:
        out.add("cs2 padding CTA")
    if plan["gn_fused"]:
        out.add("fused GN")
    return out


def test_coverage_and_negative_controls(restore_cap):
    """Runs whatever this session skipped, prints the table, asserts that each of tests 1-3 saw every planner outcome and that
    every negative control failed."""
    for gi in range(len(GEOMS)):
        if ("amax", gi) not in DONE:
            _run_absmax(gi, restore_cap)
            DONE.add(("amax", gi))
        if ("flag", gi) not in DONE:
            _run_flag(gi)
            DONE.add(("flag", gi))
        for p in PRECS:
            if ("xscale", gi, p) not in DONE:
                _run_xscale(gi, p)
                DONE.add(("xscale", gi, p))
    print("\ngeometry x precision: plan of the first call / checks passed (amax: calibration maxima, flag: range flag, "
          "xscale: input scale vs fp64)")
    by = collections.defaultdict(list)
    for r in RECORDS:
        if r["geom"] is not None:
            by[(r["geom"], r["prec"])].append(r)
    for (gi, p), rs in sorted(by.items()):
        checks = collections.Counter(r["check"].split(" ")[0] + (" gn" if " gn" in r["check"] else "") for r in rs)
        print(f"{str(GEOMS[gi]):28s} {p:7s} {_plan_str(rs[0]['plan']):52s} " + " ".join(f"{c}:{v}" for c, v in sorted(checks.items())))
    for r in RECORDS:
        if r["geom"] is None:
            print("modules:", r["check"])
    print("overflowed call's own output held Inf/NaN (geometries):",
          {f"{p} {v:g} {a}": f"{sum(f)}/{len(f)}" for (p, v, a), f in sorted(NONFINITE.items(), key=str)})
    print("worst:", dict(WORST))
    print("negative controls (failed as they must):", {k: f"{sum(v)}/{len(v)}" for k, v in sorted(CONTROLS.items())})
    need = {"tc1 per-tap", "tc2 nt64", "tc2 nt128", "TN>1", "split-K", "cs2 padding CTA", "fused GN"}
    for test in ("amax", "flag", "xscale"):
        seen = set()
        for r in RECORDS:
            if r["test"] == test:
                seen |= _outcomes(r["plan"])
        assert need <= seen, f"{test}: the reported plans missed {sorted(need - seen)}"
    for name in ("amax without last_channel_block", "amax without last_sample", "gn amax over the masked columns",
                 "tiny input at x_scale 1"):
        assert CONTROLS[name], f"control {name}: no geometry suited it"
        assert all(CONTROLS[name]), f"control {name} passed the comparison on {CONTROLS[name].count(False)} geometries"
    # an overflow without an activation is always visible in the output; ReLU's fmaxf may hide it (the flag does not)
    for (p, v, a), f in NONFINITE.items():
        if a == "none":
            assert all(f), f"{p} {v:g}: an overflowed call without activation gave a finite output"
