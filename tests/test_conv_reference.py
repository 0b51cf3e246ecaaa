"""The sampled fp64 convolution reference (oracle/conv_ref.py) against F.conv2d in fp64 with the epilogue written out by hand: every
epilogue feature, channel-sliced inputs, strides (1,1) (2,1) (2,2) (8,8).  CPU only: the GPU sweep (test_gpu_conv_sweep.py) trusts
this reference, so it is checked here first."""
import math

import pytest
import torch
import torch.nn.functional as F

from oracle import conv_ref as R


def _rand(*shape, seed):
    return torch.randn(*shape, generator=torch.Generator().manual_seed(seed))


def _hand_ref(x, w4, stride, pad, gn=None, valid_w=None, out_scale=None, bias=None, residual=None, res_broadcast=False, act=0,
              gain=1.0, y2_scale=None):
    """The whole op over every pixel, NCHW fp64, the straightforward way (no shared code with oracle/conv_ref.py)."""
    x = x.permute(0, 3, 1, 2).double()
    n, c, h, wd = x.shape
    if gn is not None:
        mr, gamma, beta = (t.double() for t in gn)
        xg = x.reshape(n, c // 32, 32, h, wd)
        xg = (xg - mr[:, :, 0, None, None, None]) * mr[:, :, 1, None, None, None]
        t = xg.reshape(n, c, h, wd) * gamma[None, :, None, None] + beta[None, :, None, None]
        x = t * torch.sigmoid(t)
        if valid_w is not None:
            for i in range(n):
                x[i, :, :, int(valid_w[i]):] = 0
    v = F.conv2d(x, w4.double(), stride=stride, padding=pad)
    if out_scale is not None:
        v = v * out_scale.double()[:, :, None, None]
    if bias is not None:
        v = v + bias.double()[None, :, None, None]
    if residual is not None:
        r = residual.permute(0, 3, 1, 2).double()
        v = v + (r.expand(n, -1, -1, -1) if res_broadcast else r)
    v = {0: lambda t: t, 1: F.relu, 2: lambda t: F.leaky_relu(t, 0.2), 3: torch.tanh, 4: F.gelu, 5: torch.sigmoid}[act](v) * gain
    if valid_w is not None:
        for i in range(n):
            v[i, :, :, int(valid_w[i]):] = 0
    v = v.permute(0, 2, 3, 1)
    return v, (None if y2_scale is None else v * y2_scale.double()[:, None, None, :])


def _close(a, b, scale):
    """|a - b| <= 1e-12 * scale everywhere (scale: the bound of a value, which two summation orders may differ by a multiple of
    2^-52 of; the value itself for the bound, a sum of magnitudes).  Zero scale demands equality."""
    return bool(((a - b).abs() <= 1e-12 * scale).all())


FEATURES = ["plain", "demod_bias_lrelu_y2", "residual_relu", "res_broadcast_tanh", "gelu", "sigmoid", "valid_w", "gn_swish_valid_w"]


@pytest.mark.parametrize("stride,k,pad", [((1, 1), 3, 1), ((2, 1), 3, 1), ((2, 2), 3, 1), ((8, 8), 8, 0), ((1, 1), 1, 0)])
@pytest.mark.parametrize("feature", FEATURES)
def test_sampled_reference_equals_fp64_conv(feature, stride, k, pad):
    n, h, w, cin, cout = 3, 16, 24, 64, 40
    buf = _rand(n, h, w, cin + 16, seed=1)
    x = buf[..., 8:8 + cin]                                  # a channel slice of a wider buffer
    w4 = _rand(cout, cin, k, k, seed=2) / math.sqrt(cin * k * k)
    oh, ow = (h + 2 * pad - k) // stride[0] + 1, (w + 2 * pad - k) // stride[1] + 1
    kw = {}
    if feature == "demod_bias_lrelu_y2":
        wide = _rand(n, 3 * cout, seed=3).abs() + 0.5          # column views with a row stride wider than Cout
        kw = dict(out_scale=wide[:, cout:2 * cout], bias=_rand(cout, seed=4), act=R.ACT_LRELU02, gain=2 ** 0.5,
                  y2_scale=wide[:, 2 * cout:])
    elif feature == "residual_relu":
        kw = dict(residual=_rand(n, oh, ow, cout + 8, seed=5)[..., 4:4 + cout], act=R.ACT_RELU, bias=_rand(cout, seed=6))
    elif feature == "res_broadcast_tanh":
        kw = dict(residual=_rand(1, oh, ow, cout, seed=7), res_broadcast=True, act=R.ACT_TANH)
    elif feature == "gelu":
        kw = dict(bias=_rand(cout, seed=8), act=R.ACT_GELU)
    elif feature == "sigmoid":
        kw = dict(act=R.ACT_SIGMOID, gain=0.5)
    elif feature == "valid_w":
        kw = dict(valid_w=torch.tensor([ow, max(1, ow // 2), 1]))
    elif feature == "gn_swish_valid_w":
        mr = torch.stack([_rand(n, cin // 32, seed=9) * 0.3, _rand(n, cin // 32, seed=10).abs() + 0.5], -1)
        kw = dict(gn=(mr, _rand(cin, seed=11) * 0.3 + 1, _rand(cin, seed=12) * 0.2), valid_w=torch.tensor([w, 7, 13]))
        if stride != (1, 1):
            kw["valid_w"] = None
    full, full2 = _hand_ref(x, w4, stride, pad, **kw)
    w2d = w4.permute(2, 3, 1, 0).reshape(k * k * cin, cout)
    pix = R.sample_pixels(n, oh, ow, th=4, tw=8, tn=2, m_tile=128, valid_w=kw.get("valid_w"), count=60, seed=3)
    g = {key: kw[key] for key in ("gn", "valid_w", "residual", "res_broadcast", "out_scale", "y2_scale", "bias") if kw.get(key) is not None}
    d = R.gather(x, k, k, stride, (pad, pad), pix, **g)
    ref = R.conv_ref(d, w2d, act=kw.get("act", 0), gain=kw.get("gain", 1.0))
    want = full[pix[:, 0], pix[:, 1], pix[:, 2]]
    assert torch.allclose(ref["y"], want, rtol=1e-12, atol=1e-12)
    if full2 is not None:
        assert torch.allclose(ref["y2"], full2[pix[:, 0], pix[:, 1], pix[:, 2]], rtol=1e-12, atol=1e-12)
    # the whole-tensor reference at the sampled pixels: the same values, bounds and masks as the sampled one
    whole = R.conv_ref_full(x, w2d, k, k, stride, (pad, pad), act=kw.get("act", 0), gain=kw.get("gain", 1.0), **g)
    assert whole["y"].shape == (n, oh, ow, cout) and _close(whole["y"], full, whole["bound"] + full.abs())
    at = lambda t: t[pix[:, 0], pix[:, 1], pix[:, 2]]          # noqa: E731
    assert torch.equal(at(whole["masked"]), ref["masked"])
    assert _close(at(whole["bound"]), ref["bound"], ref["bound"])
    assert _close(at(whole["y"]), ref["y"], ref["bound"] + ref["y"].abs())
    assert ("y2" in whole) == ("y2" in ref)
    if "y2" in ref:
        assert _close(at(whole["bound2"]), ref["bound2"], ref["bound2"])
        assert _close(at(whole["y2"]), ref["y2"], ref["bound2"] + ref["y2"].abs())
    # the bound dominates the exact error of an fp32 evaluation of the same numbers
    got = want.float()
    assert R.ratio(got, ref["y"], ref["bound"], 1e-6) <= 1.0
    if kw.get("valid_w") is not None:
        assert ref["masked"].any() and (ref["y"][ref["masked"]] == 0).all() and (ref["bound"][ref["masked"]] == 0).all()


def test_negative_controls_see_a_shifted_row_or_a_dropped_operand():
    n, h, w, cin, cout = 3, 8, 8, 64, 32
    x = _rand(n, h, w, cin, seed=20)
    w2d = _rand(9 * cin, cout, seed=21) / 24
    osc, y2s = _rand(n, cout, seed=22).abs() + 0.5, _rand(n, cout, seed=23)
    pix = R.sample_pixels(n, h, w, count=40)
    d = R.gather(x, 3, 3, (1, 1), (1, 1), pix, out_scale=osc, y2_scale=y2s, bias=_rand(cout, seed=24),
                 residual=_rand(n, h, w, cout, seed=25) * 0.1, valid_w=torch.tensor([8, 5, 3]))
    ref = R.conv_ref(d, w2d, act=R.ACT_LRELU02)
    got = ref["y"].float()
    assert R.ratio(got, ref["y"], ref["bound"], 1e-6) <= 1.0
    for kw in (dict(shift=1), dict(drop=("bias",)), dict(drop=("residual",))):
        bad = R.conv_ref(d, w2d, act=R.ACT_LRELU02, **kw)
        assert R.ratio(got, bad["y"], bad["bound"], 1e-4) > 1.0, kw
    assert R.ratio(ref["y2"].float(), R.conv_ref(d, w2d, act=R.ACT_LRELU02, shift=1)["y2"], ref["bound2"], 1e-4) > 1.0


def test_sampler_covers_tile_edges_valid_width_and_the_last_sample():
    pix = R.sample_pixels(5, 32, 64, th=8, tw=16, tn=2, valid_w=[64, 9, 64, 64, 30], count=10)
    s = {tuple(p) for p in pix.tolist()}
    assert any(p[0] == 4 for p in s) and any(p[0] == 0 for p in s)
    rows0 = {p[1] for p in s if p[0] == 0}
    cols1 = {p[2] for p in s if p[0] == 1}
    assert {0, 7, 8, 9, 15, 16, 17, 31} <= rows0
    assert {0, 15, 16, 17, 8, 9, 63} <= cols1
    assert len(pix) == len(s)


def test_linear_and_patch_embed_references():
    x = _rand(7, 128, seed=30)
    w = _rand(128, 48, seed=31) / 11
    b, r = _rand(48, seed=32), _rand(7, 48, seed=33)
    y, bound = R.linear_ref(x, w, b, act=R.ACT_GELU, residual=r)
    assert torch.allclose(y, F.gelu(F.linear(x.double(), w.double().t(), b.double()) + r.double()), rtol=1e-12, atol=1e-12)
    assert (bound > 0).all()
    feat = _rand(2, 8, 24, 16, seed=34)                        # B=2, T=3, C=16
    wp, bp, pe = _rand(8 * 8 * 16, 32, seed=35) / 32, _rand(32, seed=36), _rand(3, 32, seed=37)
    tok, _ = R.patch_embed_ref(feat, wp, bp, pe)
    conv = F.conv2d(feat.permute(0, 3, 1, 2).double(), wp.double().t().reshape(32, 8, 8, 16).permute(0, 3, 1, 2), bp.double(), stride=8)
    want = conv.flatten(2).transpose(1, 2).reshape(6, 32) + pe.double().repeat(2, 1)
    assert torch.allclose(tok, want, rtol=1e-12, atol=1e-12)


def test_groupnorm_stats64_matches_group_norm():
    y = _rand(2, 4, 10, 64, seed=40) * 3 + 5
    st = R.groupnorm_stats64(y, valid_w=[10, 6])
    for i, v in enumerate((10, 6)):
        t = y[i:i + 1, :, :v].permute(0, 3, 1, 2).double()
        ref = F.group_norm(t, 2, eps=1e-6)
        m = t.reshape(2, -1).mean(1)
        assert torch.allclose(st[i, :, 0], m)
        assert torch.allclose((t.reshape(2, -1) - m[:, None]) * st[i, :, 1:2], ref.reshape(2, -1), atol=1e-10)
