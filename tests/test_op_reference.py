"""The fp64 references of oracle/op_ref.py against torch's own fp64 operators (F.group_norm, F.interpolate, F.layer_norm, softmax
attention, F.conv2d for ToRGB) and restate._adain, with channel slices, valid widths and clipped windows.  CPU only: the GPU sweep
(test_gpu_op_sweep.py) trusts these references, so they are checked here first."""
import math

import pytest
import torch
import torch.nn.functional as F

from oracle import op_ref as R
from oracle import restate


def _rand(*shape, seed, scale=1.0, shift=0.0):
    return torch.randn(*shape, generator=torch.Generator().manual_seed(seed), dtype=torch.float64) * scale + shift


def _close(a, b, rel=1e-12):
    assert torch.allclose(a, b, rtol=rel, atol=rel * max(1.0, float(b.abs().max()))), float((a - b).abs().max())


@pytest.mark.parametrize("swish", [False, True])
@pytest.mark.parametrize("valid", [False, True])
def test_groupnorm_matches_group_norm(swish, valid):
    n, h, w, c = 3, 4, 7, 96
    buf = _rand(n, h, w, c + 32, seed=1, scale=2.0, shift=0.5)
    x = buf[..., 16:16 + c]                                     # a channel slice
    gamma, beta = _rand(c, seed=2), _rand(c, seed=3)
    vw = [w, 1, 4] if valid else None
    got, bound = R.groupnorm_swish_ref(x, gamma, beta, swish=swish, valid_w=vw)
    for i in range(n):
        v = w if vw is None else vw[i]
        want = F.group_norm(x[i:i + 1, :, :v].permute(0, 3, 1, 2), c // 32, gamma, beta, eps=1e-6).permute(0, 2, 3, 1)[0]
        if swish:
            want = want * torch.sigmoid(want)
        _close(got[i, :, :v], want)
        assert (got[i, :, v:] == 0).all() and (bound[i, :, v:] == 0).all()
        assert (bound[i, :, :v] >= got[i, :, :v].abs() * (0 if swish else 1) - 1e-12).all()


def test_affine_stats_recovers_the_applied_statistics():
    n, h, w, c = 2, 5, 6, 64
    x = _rand(n, h, w, c, seed=4, scale=0.01, shift=30.0)
    mr = R.groupnorm_stats64(x, valid_w=[w, 3])
    mr_off = mr.clone()
    mr_off[..., 0] += 1e-4
    mr_off[..., 1] *= 1 + 1e-5
    y, _ = R.groupnorm_apply_ref(x, mr_off, torch.ones(c), torch.zeros(c), swish=False, valid_w=[w, 3])
    got = R.affine_stats(x, y.float(), valid_w=[w, 3])
    assert R.stats_err(got, mr_off) < 1e-8
    assert R.stats_err(got, mr) > 1e-6


@pytest.mark.parametrize("shift_data", [0.0, 300.0])
def test_adain_concat_matches_restate_adain(shift_data):
    nc, h, wp, c, w = 3, 4, 8, 64, 20
    prior = _rand(nc, h, wp, c, seed=5, shift=shift_data)
    feat = _rand(2, h, w, c, seed=6, scale=0.5, shift=-shift_data)
    half = wp // 2
    # windows clipped at the left and right line edges (wv < wp, y1 != 0) and one full-width window
    wins = [(0, 0, 5, half - 5 // 2), (1, 17, 20, half - 3 // 2), (1, 6, 14, 0)]
    ref, bound, floor = R.adain_concat_ref(prior, feat, wins, wp)
    for i, (line, x1, x2, y1) in enumerate(wins):
        wv = x2 - x1
        p = prior[i, :, y1:y1 + wv].permute(2, 0, 1)[None]
        f = feat[line, :, x1:x2].permute(2, 0, 1)[None]
        want = restate._adain(p, f)[0].permute(1, 2, 0)
        _close(ref[i, :, :wv, :c], want)
        assert torch.equal(ref[i, :, :wv, c:], feat[line, :, x1:x2])
        assert (ref[i, :, wv:] == 0).all() and (bound[i, :, wv:] == 0).all() and (floor[i, :, wv:] == 0).all()
    bad, _, _ = R.adain_concat_ref(prior, feat, wins, wp, move=1)
    assert not torch.equal(bad, ref)


@pytest.mark.parametrize("h,w", [(1, 1), (1, 3), (4, 5), (7, 8)])
def test_bilinear_matches_interpolate(h, w):
    n, c = 2, 8
    x = _rand(n, h, w, c + 4, seed=7)[..., :c]
    s = _rand(n, c + 4, seed=8)[:, 4:]
    ref, bound = R.resample_ref(x, s)
    want = F.interpolate(x.permute(0, 3, 1, 2), scale_factor=2, mode="bilinear", align_corners=False).permute(0, 2, 3, 1)
    _close(ref, want * s[:, None, None, :])
    assert (bound >= ref.abs() - 1e-12).all()
    ref0, _ = R.resample_ref(x, s, up=False)
    _close(ref0, x * s[:, None, None, :])


def test_ragged_bilinear_is_each_sample_at_its_own_width():
    n, h, w, c = 3, 3, 9, 8
    x = _rand(n, h, w, c, seed=9)
    vw = [1, 5, 9]
    ref, bound = R.resample_ref(x, None, valid_w=vw)
    for i, v in enumerate(vw):
        want = F.interpolate(x[i:i + 1, :, :v].permute(0, 3, 1, 2), scale_factor=2, mode="bilinear", align_corners=False)
        _close(ref[i, :, :2 * v], want.permute(0, 2, 3, 1)[0])
        assert (ref[i, :, 2 * v:] == 0).all() and (bound[i, :, 2 * v:] == 0).all()


@pytest.mark.parametrize("with_skip", [False, True])
def test_torgb_matches_modulated_1x1_conv(with_skip):
    n, h, w, c = 2, 4, 6, 128
    x = _rand(n, h, w, c, seed=10)
    s = _rand(n, c + 64, seed=11)[:, 32:32 + c]
    wt, bias = _rand(3, c, seed=12, scale=0.1), _rand(3, seed=13)
    skip = _rand(n, h // 2, w // 2, 3, seed=14) if with_skip else None
    ref, bound = R.torgb_ref(x, s, wt, bias, skip)
    v = torch.stack([F.conv2d(x[i:i + 1].permute(0, 3, 1, 2), (wt * s[i])[:, :, None, None], bias) for i in range(n)])[:, 0]
    if with_skip:
        v = v + F.interpolate(skip.permute(0, 3, 1, 2), scale_factor=2, mode="bilinear", align_corners=False)
    _close(ref, torch.tanh(v).permute(0, 2, 3, 1))
    assert (bound >= 0).all()
    if with_skip:
        assert not torch.allclose(R.torgb_ref(x, s, wt, bias, skip, drop_skip=True)[0], ref)


def test_demod_and_pixelnorm():
    s = _rand(3, 40, seed=15)
    wsq = _rand(13, 70, seed=16).abs()
    ref, _ = R.demod_ref(s, wsq, s_off=7)
    _close(ref, 1 / torch.sqrt((s[:, 7:20] ** 2) @ wsq + 1e-8))
    z = _rand(5, 33, seed=17)
    _close(R.pixelnorm_ref(z)[0], z / torch.sqrt((z * z).mean(1, keepdim=True) + 1e-8))


def test_layernorm_and_token_mix():
    x = _rand(7, 50, seed=18, shift=2.0)
    g, b = _rand(50, seed=19), _rand(50, seed=20)
    _close(R.layernorm_ref(x, g, b)[0], F.layer_norm(x, (50,), g, b, eps=1e-5))
    bt, t, d, to = 2, 5, 70, 3
    x3 = _rand(bt, t, d, seed=21)
    gt, btok, w, bias = _rand(t, seed=22), _rand(t, seed=23), _rand(to, t, seed=24), _rand(to, seed=25)
    ln = F.layer_norm(x3.transpose(1, 2), (t,), gt, btok, eps=1e-5)                # [B, D, T]
    want = F.linear(ln, w, bias).transpose(1, 2)
    _close(R.token_mix_ref(x3, gt, btok, w, bias)[0], want)


@pytest.mark.parametrize("s", [1, 9, 33])
def test_attention_matches_softmax_attention(s):
    b, heads, dh = 2, 2, 64
    qkv = _rand(b, s, 3 * heads * dh, seed=26)
    ref, bound = R.attention_ref(qkv, heads, dh)
    q, k, v = (qkv[..., i * heads * dh:(i + 1) * heads * dh].reshape(b, s, heads, dh).transpose(1, 2) for i in range(3))
    want = F.scaled_dot_product_attention(q, k, v).transpose(1, 2).reshape(b, s, -1)
    _close(ref, want, rel=1e-10)
    assert (bound >= ref.abs() - 1e-12).all()


def test_statistics_kernels_build_without_spills(tmp_path):
    """ptxas -v for sm_90a: the GroupNorm and AdaIN statistics kernels (fp32 runs about a pivot, fp64 sums) keep everything in
    registers."""
    import os
    import re
    import subprocess
    from marconet_b200 import build
    src = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "marconet_b200", "csrc", "sr_ops.cu")
    r = subprocess.run([build.nvcc_path(), "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-DMN_BUILD", "-Xptxas", "-v",
                        "-cubin", src, "-o", str(tmp_path / "sr_ops.cubin")], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-2000:]
    props = re.findall(r"Function properties for (\S*(?:gn_stats|adain_stats)_kernel\S*)\n([^\n]*)", r.stderr)
    assert len(props) == 2, r.stderr[-2000:]
    for kernel, line in props:
        assert "0 bytes spill stores, 0 bytes spill loads" in line, f"{kernel}: {line}"


def test_ratio_floor_and_masked_zeros():
    t = lambda *v: torch.tensor(v, dtype=torch.float64)     # noqa: E731
    ref, bound = t(1.0, 0.0), t(1.0, 0.0)
    assert R.ratio(t(1.0 + 1e-6, 0.0), ref, bound, 1e-6) == pytest.approx(0.5)
    assert R.ratio(t(1.0, 1e-30), ref, bound, 1e-6) == math.inf
    assert R.ratio(t(1.0 + 3e-6, 0.0), ref, bound, 1e-6, floor=t(2e-6, 0.0)) == pytest.approx(0.5)
