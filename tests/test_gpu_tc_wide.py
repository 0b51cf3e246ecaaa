"""128-channel work items of the wgmma convolution (conv_tc2.cu, NT = 128) vs fp64 torch CPU convolution.  The plan takes NT = 128
when Cout % 128 == 0, at least 3 weight stages fit and halving the number of work items neither lengthens the persistent grid's
makespan on 132 SMs nor deepens split-K; every shape below is chosen so that it does."""
import math

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu


def _dev():
    return torch.device("cuda:0")


def _rand(*shape, seed=0, scale=1.0):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(*shape, generator=g) * scale


def _nhwc(x):
    return x.permute(0, 2, 3, 1).contiguous().to(_dev())


def _nchw(y):
    return y.permute(0, 3, 1, 2).cpu()


def _cw(w):
    from marconet_b200 import ops
    cout, cin, kh, kw = w.shape
    return ops.ConvWeight(w.permute(2, 3, 1, 0).reshape(kh * kw * cin, cout).contiguous().to(_dev()), kh * kw)


WIDE_CASES = [
    # N, H, W, Cin, Cout, k
    (4, 32, 64, 256, 256, 3),     # 36 k-blocks per item through a 3-stage weight ring, no split-K
    (4, 16, 128, 256, 256, 1),    # 1x1
    (65, 8, 16, 64, 256, 3),      # 65 pixel tiles: padding CTA in the last 2-CTA cluster
    (1, 12, 512, 128, 256, 3),    # H % 8 != 0: per-tap tiling (one shifted box per tap)
]
TOL = {"f16x3": 4e-5, "bf16x3": 2e-4, "f16x1": 4e-3}


@pytest.mark.parametrize("mode", ["f16x3", "bf16x3", "f16x1"])
@pytest.mark.parametrize("case", WIDE_CASES)
def test_conv_tc_wide_items_match_fp64(case, mode):
    from marconet_b200 import ops
    prec = {"f16x3": ops.PREC_F16X3_TC, "bf16x3": ops.PREC_BF16X3_TC, "f16x1": ops.PREC_F16X1_TC}[mode]
    n, h, w, cin, cout, k = case
    x = _rand(n, cin, h, w, seed=31) * 1.7 + 0.2
    wt = _rand(cout, cin, k, k, seed=32, scale=1.0 / math.sqrt(cin * k * k))
    ref = F.conv2d(x.double(), wt.double(), padding=k // 2).float()
    y = ops.conv2d(_nhwc(x), _cw(wt), k, k, pad=(k // 2, k // 2), precision=prec)
    torch.cuda.synchronize()
    err = (_nchw(y) - ref).abs().max().item()
    scale = ref.abs().max().item()
    print(f"{mode} {case}: max abs err {err:.3e} (ref max {scale:.2f})")
    assert err <= TOL[mode] * max(1.0, scale)


@pytest.mark.parametrize("ragged", [False, True])
def test_conv_tc_wide_items_fused_groupnorm_swish(ragged):
    """swish(GroupNorm(x)) built in the split stage of 128-channel work items, with ragged windows."""
    from marconet_b200 import ops
    d = _dev()
    n, h, w, cin, cout = 8, 32, 32, 128, 256
    x = _rand(n, cin, h, w, seed=40) * 2 + 0.3
    valid = [w, 17, 5, w - 1, 1, 32, 9, 30] if ragged else None
    if ragged:
        for i, v in enumerate(valid):
            x[i, :, :, v:] = 0
    wt = _rand(cout, cin, 3, 3, seed=41, scale=0.04)
    gamma, beta, bias = _rand(cin, seed=42) * 0.3 + 1, _rand(cin, seed=43) * 0.2, _rand(cout, seed=44)
    vw = torch.tensor(valid, dtype=torch.int32, device=d) if ragged else None
    xn = _nhwc(x)
    mr = ops.groupnorm_stats(xn, valid_w=vw)
    y = ops.conv2d(xn, _cw(wt), 3, 3, pad=(1, 1), bias=bias.to(d), valid_w=vw, gn=(mr, gamma.to(d), beta.to(d)), gn_fuse=True,
                   precision=ops.PREC_F16X3_TC)
    y = _nchw(y)
    for i in range(n):
        v = valid[i] if ragged else w
        xi = x[i:i + 1, :, :, :v].double()
        g = F.group_norm(xi, cin // 32, gamma.double(), beta.double(), eps=1e-6)
        g = g * torch.sigmoid(g)
        ref = F.conv2d(g, wt.double(), bias.double(), padding=1).float()
        err = (y[i:i + 1, :, :, :v] - ref).abs().max().item()
        assert err <= 3e-5 * max(1.0, ref.abs().max().item()), f"sample {i}: {err}"
        if v < w:
            assert y[i, :, :, v:].abs().max().item() == 0
