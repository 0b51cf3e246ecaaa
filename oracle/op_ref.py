"""fp64 references of the non-convolution kernels of ``ops``, each with a per-element error bound (as oracle/conv_ref.py).

Every reference takes the op's inputs as the op receives them (NHWC views, channel slices, per-sample vectors) and returns
``(ref, bound)`` in fp64 on the inputs' device.  ``bound`` is the magnitude of the terms the kernel adds up in fp32 -- e.g. for a
normalisation ``L * (|gamma| * rstd * (|x - mean| + |mean|) + |beta|)`` -- so that

    |got - ref| <= tol * (bound + |ref|) + floor

(``ratio``) sees an error in a small output that a bound scaled by the tensor's max would hide.  ``floor`` is an error the kernel
makes on purpose and exactly once: the fp32 rounding of a mean it hands on (``adain_concat_ref``).  Outputs that must be exact zeros
(beyond valid widths) have bound 0: any nonzero there is an infinite ratio.

The ops that are exact by construction (select_text, window_scatter, check_labels, the window integers, the layout conversions) are
compared bit for bit against fp32 torch / numpy expressions in the tests, not here.
"""
import math

import torch

from oracle.conv_ref import groupnorm_stats64

SWISH_LIPSCHITZ = 1.1     # max |d swish / du| = 1.0998 (at u = 2.40)
U32 = 2.0 ** -24          # fp32 unit roundoff


def ratio(got, ref, bound, tol, floor=None):
    """Worst (|got - ref| - floor) / (tol * (bound + |ref|)); a mismatch where the limit is exactly 0 is infinite, a NaN too."""
    got = got.double().to(ref.device)
    err = (got - ref).abs()
    if floor is not None:
        err = (err - floor).clamp_min(0)
    lim = tol * (bound + ref.abs())
    r = torch.where(lim > 0, err / lim.clamp_min(1e-300), torch.where(err > 0, torch.full_like(err, math.inf), torch.zeros_like(err)))
    r = torch.where(torch.isnan(got), torch.full_like(r, math.inf), r)
    return float(r.max()) if r.numel() else 0.0


def stats_err(got, ref):
    """GroupNorm statistics [..., 2] (mean, rstd) against fp64: max of |d mean| * rstd and |d rstd| / rstd.  The mean is handed on
    in fp32; its own rounding (up to 2^-24 |mean|) is not counted."""
    got = got.double().to(ref.device)
    em = (((got[..., 0] - ref[..., 0]).abs() - U32 * ref[..., 0].abs()).clamp_min(0) * ref[..., 1]).max().item()
    er = ((got[..., 1] - ref[..., 1]).abs() / ref[..., 1]).max().item()
    return max(em, er)


def _col_mask(n, w, valid_w, device):
    """[N, 1, W, 1] bool: column < valid_w[n] (all True without valid_w)."""
    if valid_w is None:
        return torch.ones(n, 1, w, 1, dtype=torch.bool, device=device)
    vw = torch.as_tensor([int(v) for v in valid_w], device=device)
    return (torch.arange(w, device=device)[None, :] < vw[:, None])[:, None, :, None]


# ---- GroupNorm ----------------------------------------------------------------------------------------------------------
def groupnorm_apply_ref(x, mr, gamma, beta, swish=True, valid_w=None, cpg=32, own_stats=False):
    """y = swish?((x - mean[n,g]) * rstd[n,g] * gamma + beta), 0 beyond valid_w[n].  ``mr`` [N, C/cpg, 2] as the op receives it
    (fp32 from the device), or the fp64 statistics when the op computes its own (``own_stats``: statistics accurate to a fraction
    of a std move the output by that fraction of |gamma|, a term of the bound)."""
    x = x.double()
    n, h, w, c = x.shape
    mr = mr.double().to(x.device)
    grp = torch.arange(c, device=x.device) // cpg
    mean = mr[:, grp, 0][:, None, None, :]
    rstd = mr[:, grp, 1][:, None, None, :]
    g, b = gamma.double().to(x.device)[:c], beta.double().to(x.device)[:c]
    u = (x - mean) * rstd * g + b
    bound = g.abs() * rstd.abs() * ((x - mean).abs() + mean.abs()) + b.abs()
    if own_stats:
        bound = bound + g.abs()
    if swish:
        u = u * torch.sigmoid(u)
        bound = SWISH_LIPSCHITZ * bound
    m = _col_mask(n, w, valid_w, x.device)
    return torch.where(m, u, torch.zeros_like(u)), torch.where(m, bound, torch.zeros_like(bound))


def groupnorm_swish_ref(x, gamma, beta, swish=True, valid_w=None, eps=1e-6, cpg=32):
    """Statistics (biased variance + eps, over each sample's first valid_w[n] columns) and apply, all in fp64."""
    return groupnorm_apply_ref(x, groupnorm_stats64(x, valid_w=valid_w, eps=eps, cpg=cpg), gamma, beta, swish, valid_w, cpg, own_stats=True)


def affine_stats(x, y, valid_w=None, cpg=32):
    """The (mean, rstd) [N, G, 2] an un-affine GroupNorm (gamma 1, beta 0, no swish) actually applied, recovered from its input x and
    output y = (x - mean) * rstd by a least-squares line per (sample, group) in fp64 (slope = rstd, mean = mean(x) - mean(y) / rstd).
    The fp32 rounding of y averages out: this sees the statistics the kernel computed to ~1e-9."""
    x, y = x.double(), y.double().to(x.device)
    n, h, w, c = x.shape
    out = torch.empty(n, c // cpg, 2, dtype=torch.float64, device=x.device)
    for i in range(n):
        v = w if valid_w is None else int(valid_w[i])
        xs = x[i, :, :v].reshape(-1, c // cpg, cpg).transpose(0, 1).reshape(c // cpg, -1)
        ys = y[i, :, :v].reshape(-1, c // cpg, cpg).transpose(0, 1).reshape(c // cpg, -1)
        xm, ym = xs.mean(1), ys.mean(1)
        slope = ((xs - xm[:, None]) * (ys - ym[:, None])).sum(1) / ((xs - xm[:, None]) ** 2).sum(1)
        out[i, :, 0] = xm - ym / slope
        out[i, :, 1] = slope
    return out


# ---- AdaIN + concat over per-character windows --------------------------------------------------------------------------
def _mean_std_unbiased(t):
    """[..., P, C] -> mean, sqrt(unbiased variance + 1e-5) over P (restate._adain)."""
    m = t.mean(-2, keepdim=True)
    var = ((t - m) ** 2).sum(-2, keepdim=True) / (t.shape[-2] - 1)
    return m, (var + 1e-5).sqrt()


def adain_concat_ref(prior, feat, wins, wp, shift=0, move=0):
    """out [Nc, H, wp, 2C]: for window i = (line, x1, x2, y1) of width wv = x2 - x1, the prior crop prior[i, :, y1:y1+wv] normalised
    to the statistics of the feature window feat[line, :, x1:x2] (unbiased variance + 1e-5, restate._adain) in the first C channels,
    the feature window itself in the last C; zeros from column wv on.  Returns (ref, bound, floor).
    Negative controls: ``shift`` = 1 takes the next window's prior crop, ``move`` = 1 moves every feature window one column right."""
    prior, feat = prior.double(), feat.double().to(prior.device)
    nc, h, _, c = prior.shape
    ref = torch.zeros(nc, h, wp, 2 * c, dtype=torch.float64, device=prior.device)
    bound, floor = torch.zeros_like(ref), torch.zeros_like(ref)
    for i, (line, x1, x2, y1) in enumerate(wins):
        wv = x2 - x1
        x1 = min(x1 + move, feat.shape[2] - wv)
        p = prior[(i + shift) % nc, :, y1:y1 + wv]
        f = feat[line, :, x1:x1 + wv]
        pm, ps = _mean_std_unbiased(p.reshape(1, -1, c))
        lm, ls = _mean_std_unbiased(f.reshape(1, -1, c))
        ref[i, :, :wv, :c] = (p - pm) / ps * ls + lm
        ref[i, :, :wv, c:] = f
        # statistics accurate to a fraction of a std move the output by that fraction of ls
        bound[i, :, :wv, :c] = ((p - pm).abs() / ps + 1) * ls
        floor[i, :, :wv, :c] = ((pm.float().double() - pm).abs() / ps * ls).expand(h, wv, c)     # the fp32 rounding of the prior mean
    return ref, bound, floor


# ---- bilinear x2 (+ per-sample channel scale) ---------------------------------------------------------------------------
def _bilin_taps(size_out, size_in, device):
    """align_corners=False, scale 2: src = (o + 0.5) / 2 - 0.5 clamped at 0 -> (i0, i1, l1) with i1 clamped to size_in - 1."""
    src = ((torch.arange(size_out, device=device, dtype=torch.float64) + 0.5) * 0.5 - 0.5).clamp_min(0)
    i0 = src.floor().long()
    i1 = torch.where(i0 < size_in - 1, i0 + 1, i0)
    return i0, i1, src - i0


def _up2_one(x, s=None):
    """fp64 bilinear x2 of one NHWC sample [H, W, C] and the same of |x| (the bound), times s [C]."""
    h, w, c = x.shape
    y0, y1, ly = _bilin_taps(2 * h, h, x.device)
    x0, x1, lx = _bilin_taps(2 * w, w, x.device)
    ly, lx = ly[:, None, None], lx[None, :, None]

    def up(t):
        top = t[y0][:, x0] * (1 - lx) + t[y0][:, x1] * lx
        bot = t[y1][:, x0] * (1 - lx) + t[y1][:, x1] * lx
        return top * (1 - ly) + bot * ly

    v, b = up(x), up(x.abs())
    if s is not None:
        v, b = v * s, b * s.abs()
    return v, b


def resample_ref(x, s=None, up=True, valid_w=None, shift=0):
    """ops.resample_modulate / ops.resample_up2_ragged: bilinear x2 (or a copy when ``up`` is False), times s[n, :C] per sample.
    ``valid_w``: sample n is its first valid_w[n] columns (the clamp at its own right edge) and the output is 0 from 2*valid_w[n]
    on.  ``shift`` = 1 takes the next sample's scale row (a negative control)."""
    x = x.double()
    n, h, w, c = x.shape
    s = None if s is None else s.double().to(x.device)
    oh, ow = (2 * h, 2 * w) if up else (h, w)
    ref = torch.zeros(n, oh, ow, c, dtype=torch.float64, device=x.device)
    bound = torch.zeros_like(ref)
    for i in range(n):
        sv = None if s is None else s[(i + shift) % n, :c]
        if not up:
            ref[i] = x[i] * (1 if sv is None else sv)
            bound[i] = ref[i].abs()
            continue
        v = w if valid_w is None else int(valid_w[i])
        ref[i, :, :2 * v], bound[i, :, :2 * v] = _up2_one(x[i, :, :v], sv)
    return ref, bound


# ---- ToRGB --------------------------------------------------------------------------------------------------------------
def torgb_ref(x, s, w, bias, skip=None, drop_skip=False, shift=0):
    """tanh(sum_c x[c] * w[o, c] * s[n, c] + bias[o] + up2(skip)[o]) -> [N, H, W, 3]; the bound is the sum of the magnitudes
    (tanh is 1-Lipschitz).  Negative controls: ``drop_skip``, ``shift`` = 1 (the next sample's style row)."""
    x = x.double()
    n, h, wd, c = x.shape
    s64 = s.double().to(x.device)[:, :c]
    s64 = s64[(torch.arange(n, device=x.device) + shift) % n]
    wm = w.double().to(x.device)[None, :, :c] * s64[:, None, :]           # [N, 3, C]
    acc = torch.einsum("nhwc,noc->nhwo", x, wm)
    mag = torch.einsum("nhwc,noc->nhwo", x.abs(), wm.abs())
    b = bias.double().to(x.device)
    acc, mag = acc + b, mag + b.abs()
    if skip is not None and not drop_skip:
        for i in range(n):
            v, bb = _up2_one(skip[i].double().to(x.device))
            acc[i] += v
            mag[i] += bb
    elif skip is not None:
        for i in range(n):
            mag[i] += _up2_one(skip[i].double().to(x.device))[1]
    return torch.tanh(acc), mag


# ---- demodulation -------------------------------------------------------------------------------------------------------
def demod_ref(s, wsq, s_off=0, shift=0):
    """rsqrt(s[n, s_off:s_off+cin]^2 @ wsq + 1e-8) [N, cout]: a sum of positive terms, so |ref| is the whole bound (bound 0)."""
    cin = wsq.shape[0]
    s64 = s.double()[:, s_off:s_off + cin]
    s64 = s64[(torch.arange(s64.shape[0], device=s64.device) + shift) % s64.shape[0]]
    ref = ((s64 * s64) @ wsq.double().to(s64.device) + 1e-8).rsqrt()
    return ref, torch.zeros_like(ref)


# ---- TextViT / mapping-network row ops ----------------------------------------------------------------------------------
def pixelnorm_ref(x):
    """x * rsqrt(mean(x^2) + 1e-8) per row: the bound is |ref|."""
    x = x.double()
    ref = x * ((x * x).mean(1, keepdim=True) + 1e-8).rsqrt()
    return ref, torch.zeros_like(ref)


def _ln(x, gamma, beta, eps, dim):
    """LayerNorm over ``dim`` (biased variance) -> (value, bound).  The kernels sum the row in fp32, so the error of their mean is
    a multiple of the rounding of mean(|x|): that is the bound's second term."""
    m = x.mean(dim, keepdim=True)
    rstd = (((x - m) ** 2).mean(dim, keepdim=True) + eps).rsqrt()
    return (x - m) * rstd * gamma + beta, gamma.abs() * rstd * ((x - m).abs() + x.abs().mean(dim, keepdim=True)) + beta.abs()


def layernorm_ref(x2d, gamma, beta, eps=1e-5):
    x = x2d.double()
    return _ln(x, gamma.double().to(x.device), beta.double().to(x.device), eps, 1)


def token_mix_ref(x, gamma, beta, w, bias, eps=1e-5):
    """x [B, T, D]: LayerNorm over the T tokens of each (b, d) (gamma, beta [T]), then out[b, to, d] = sum_t w[to, t] ln[b, t, d] +
    bias[to]."""
    x = x.double()
    dev = x.device
    ln, lnb = _ln(x, gamma.double().to(dev)[None, :, None], beta.double().to(dev)[None, :, None], eps, 1)
    w64, b64 = w.double().to(dev), bias.double().to(dev)
    ref = torch.einsum("ot,btd->bod", w64, ln) + b64[None, :, None]
    bound = torch.einsum("ot,btd->bod", w64.abs(), lnb) + b64.abs()[None, :, None]
    return ref, bound


def attention_ref(qkv, heads=8, dh=64, shift=0):
    """qkv [B, S, 3*heads*dh] -> softmax(q k^T * dh^-0.5) v [B, S, heads*dh].  Bound: sum_j P_ij |v_j| (1 + 2 A_ij), A_ij = the
    magnitude dh^-0.5 * sum |q k| of the score (an error e in a score moves the output by about P |v| e).  ``shift`` = 1 reads the
    next sample's keys and values (a negative control)."""
    x = qkv.double()
    b, s, _ = x.shape
    inner = heads * dh
    q = x[..., :inner].reshape(b, s, heads, dh).transpose(1, 2)
    k = x[..., inner:2 * inner].reshape(b, s, heads, dh).transpose(1, 2)
    v = x[..., 2 * inner:].reshape(b, s, heads, dh).transpose(1, 2)
    rot = (torch.arange(b, device=x.device) + shift) % b
    k, v = k[rot], v[rot]
    sc = dh ** -0.5
    p = torch.softmax(q @ k.transpose(-1, -2) * sc, -1)
    a = (q.abs() @ k.abs().transpose(-1, -2)) * sc
    ref = p @ v
    bound = (p * (1 + 2 * a)) @ v.abs()
    return ref.transpose(1, 2).reshape(b, s, inner), bound.transpose(1, 2).reshape(b, s, inner)
