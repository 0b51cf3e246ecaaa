"""fp64 reference of ``ops.conv2d`` / ``ops.linear`` / ``ops.patch_embed`` at sampled output pixels, with a per-element error bound.

A convolution is checked at a few hundred output pixels (n, oy, ox), all output channels: ``gather`` copies the im2col patches of
those pixels (and everything else the epilogue reads) in fp64 BEFORE the op runs -- the op may overwrite its own input or residual --
and ``conv_ref`` evaluates the whole epilogue in the kernels' order:

    x'  = swish((x - mean[n,g]) * rstd[n,g] * gamma[c] + beta[c])     (fused GroupNorm input; mean / rstd as the call received them)
          zero outside the image (and, with GroupNorm, beyond valid_w[n])
    v   = act(out_scale[n,o] * sum_k x'_k w[k,o] + bias[o] + residual) * gain,   0 where ox >= valid_w[n]
    y2  = v * y2_scale[n,o]

It also returns the magnitude A = sum_k |x'_k w[k,o]| of each dot product.  The comparison (``ratio``) bounds every element by

    |y - ref| <= tol * (gain * L_act * (|out_scale| * A + |bias| + |residual|) + |ref|)

where L_act is the activation's Lipschitz constant and the last term is the rounding of the stored value itself.  A bound per
element (rather than one scaled by the tensor's max) sees an error in a small output -- a row of the wrong sample's scale, a dropped
bias -- that a max-norm bound hides.

``conv_ref_full`` evaluates the same reference and bound for every output element (an fp64 ``F.conv2d`` on the input's device).
"""
import math

import torch

ACT_NONE, ACT_RELU, ACT_LRELU02, ACT_TANH, ACT_GELU, ACT_SIGMOID = range(6)
ACT_NAMES = {ACT_NONE: "none", ACT_RELU: "relu", ACT_LRELU02: "lrelu", ACT_TANH: "tanh", ACT_GELU: "gelu", ACT_SIGMOID: "sigmoid"}
# max |d act / dv|: GELU' = Phi(v) + v * phi(v) peaks at v = sqrt(2): 0.9214 + 0.2076 = 1.1289
LIPSCHITZ = {ACT_NONE: 1.0, ACT_RELU: 1.0, ACT_LRELU02: 1.0, ACT_TANH: 1.0, ACT_GELU: 1.13, ACT_SIGMOID: 0.25}


def act64(v, act):
    if act == ACT_NONE:
        return v
    if act == ACT_RELU:
        return v.clamp_min(0)
    if act == ACT_LRELU02:
        return torch.where(v > 0, v, 0.2 * v)
    if act == ACT_TANH:
        return torch.tanh(v)
    if act == ACT_GELU:
        return 0.5 * v * (1 + torch.erf(v / math.sqrt(2.0)))
    if act == ACT_SIGMOID:
        return torch.sigmoid(v)
    raise ValueError(f"activation {act}")


def _boundaries(size, step):
    """0, size-1 and every multiple of ``step`` inside (0, size) with its two neighbours."""
    out = {0, size - 1}
    if step and step < size:
        for b in range(step, size, step):
            out.update((b - 1, b, b + 1))
    return sorted(v for v in out if 0 <= v < size)


def sample_pixels(n, oh, ow, th=None, tw=None, tn=None, m_tile=None, valid_w=None, count=200, seed=0):
    """Output pixels [P, 3] (n, oy, ox) to check: the first and last sample; every sample at a boundary of a tile of ``tn`` samples;
    in those samples every row at an image border or a boundary of ``th``-row tiles (and +-1) and every such column of ``tw``-column
    tiles, plus valid_w - 1 and valid_w; the pixels on both sides of each boundary of ``m_tile`` flattened GEMM rows; ``count`` seeded
    random pixels over the whole output.  The last column of a stride-2 output is a border column."""
    g = torch.Generator().manual_seed(seed)
    rnd = lambda hi: int(torch.randint(hi, (1,), generator=g))     # noqa: E731
    pix = set()
    samples = set(_boundaries(n, tn or 0))
    vw = None if valid_w is None else [int(v) for v in valid_w]
    for s in samples:
        rows, cols = _boundaries(oh, th or 0), set(_boundaries(ow, tw or 0))
        if vw is not None:
            cols.update(v for v in (vw[s] - 1, vw[s]) if 0 <= v < ow)
        for oy in rows:
            pix.update(((s, oy, 0), (s, oy, ow - 1), (s, oy, rnd(ow))))
        for ox in cols:
            pix.update(((s, 0, ox), (s, oh - 1, ox), (s, rnd(oh), ox)))
    if m_tile:
        total = n * oh * ow
        for b in range(m_tile, total, m_tile):
            for m in (b - 1, b):
                pix.add((m // (oh * ow), (m // ow) % oh, m % ow))
    for _ in range(count):
        pix.add((rnd(n), rnd(oh), rnd(ow)))
    return torch.tensor(sorted(pix), dtype=torch.long)


def gather(x, kh, kw, stride, pad, pix, gn=None, valid_w=None, residual=None, res_broadcast=False, out_scale=None, y2_scale=None,
           bias=None):
    """Everything ``conv_ref`` needs, copied in fp64 on x's device (call it before the op runs).  ``x`` NHWC (a channel slice is fine),
    ``gn`` = (mean_rstd [N, Cin/32, 2], gamma, beta) as the op receives it.  Per-sample vectors are gathered by each pixel's sample."""
    n, h, w, cin = x.shape
    pix = pix.to(x.device)
    pn, oy, ox = pix[:, 0], pix[:, 1], pix[:, 2]
    ky = torch.arange(kh, device=x.device).repeat_interleave(kw)
    kx = torch.arange(kw, device=x.device).repeat(kh)
    iy = oy[:, None] * stride[0] - pad[0] + ky[None, :]                 # [P, taps]
    ix = ox[:, None] * stride[1] - pad[1] + kx[None, :]
    inside = (iy >= 0) & (iy < h) & (ix >= 0) & (ix < w)
    patches = x[pn[:, None], iy.clamp(0, h - 1), ix.clamp(0, w - 1)].double()     # [P, taps, Cin]
    d = dict(pix=pix, ksize=(kh, kw), patches=patches, inside=inside, ix=ix)
    if valid_w is not None:
        d["valid_w"] = valid_w.long().to(x.device)
    if gn is not None:
        d["gn"] = tuple(t.double() for t in gn)
    if residual is not None:
        rrow = torch.zeros_like(pn) if res_broadcast else pn
        d["residual"] = residual[rrow, oy, ox].double()
    if out_scale is not None:
        d["out_scale"] = out_scale.double()          # [N, >= Cout] (a column view of a wider buffer keeps its rows)
    if y2_scale is not None:
        d["y2_scale"] = y2_scale.double()
    if bias is not None:
        d["bias"] = bias.double()
    return d


def _row_vec(t, pn, cout, shift):
    """Rows of a per-sample [N, C] vector for each pixel; ``shift`` takes the NEXT sample's row (a negative control)."""
    if t is None:
        return None
    rows = (pn + shift) % t.shape[0]
    return t[rows, :cout]


def conv_ref(d, w, act=0, gain=1.0, drop=(), shift=0):
    """fp64 outputs at d["pix"]: dict(y=[P,Cout], y2 (when y2_scale was gathered), bound=[P,Cout] (the bracket of the tolerance,
    without ``tol``), masked=[P] bool).  ``w`` [KH*KW*Cin, Cout].  Negative controls: ``drop`` names operands to leave out
    ("bias", "residual"), ``shift`` = 1 reads out_scale / y2_scale / valid_w of the next sample."""
    pix, patches, inside = d["pix"], d["patches"], d["inside"].clone()
    pn = pix[:, 0]
    p, taps, cin = patches.shape
    w64 = w.double().to(patches.device).reshape(taps, cin, -1)
    cout = w64.shape[2]
    vw = d.get("valid_w")
    vw_rows = None if vw is None else vw[(pn + shift) % vw.shape[0]]
    xs = patches
    if "gn" in d:
        mr, gamma, beta = d["gn"]
        grp = torch.arange(cin, device=patches.device) // 32
        mean = mr[pn][:, grp, 0][:, None, :]
        rstd = mr[pn][:, grp, 1][:, None, :]
        t = (xs - mean) * rstd * gamma[:cin] + beta[:cin]
        xs = t * torch.sigmoid(t)
        if vw_rows is not None:
            inside &= d["ix"] < vw_rows[:, None]
    xs = xs * inside[:, :, None]
    acc = torch.einsum("ptc,tco->po", xs, w64)
    mag = torch.einsum("ptc,tco->po", xs.abs(), w64.abs())
    os_ = _row_vec(d.get("out_scale"), pn, cout, shift)
    if os_ is not None:
        acc = acc * os_
        mag = mag * os_.abs()
    if "bias" in d and "bias" not in drop:
        acc = acc + d["bias"][:cout]
    if "bias" in d:
        mag = mag + d["bias"][:cout].abs()
    if "residual" in d and "residual" not in drop:
        acc = acc + d["residual"][:, :cout]
    if "residual" in d:
        mag = mag + d["residual"][:, :cout].abs()
    v = act64(acc, act) * gain
    masked = torch.zeros(p, dtype=torch.bool, device=v.device) if vw_rows is None else pix[:, 2] >= vw_rows
    v = torch.where(masked[:, None], torch.zeros_like(v), v)
    bound = abs(gain) * LIPSCHITZ[act] * mag
    out = dict(y=v, bound=torch.where(masked[:, None], torch.zeros_like(bound), bound), masked=masked)
    y2s = _row_vec(d.get("y2_scale"), pn, cout, shift)
    if y2s is not None:
        out["y2"] = v * y2s
        out["bound2"] = out["bound"] * y2s.abs()
    return out


def conv_ref_full(x, w, kh, kw, stride, pad, gn=None, valid_w=None, residual=None, res_broadcast=False, out_scale=None, y2_scale=None,
                  bias=None, act=0, gain=1.0):
    """``conv_ref`` over every output element at once: an fp64 ``F.conv2d`` on x's device (on the GPU when x is there).  Arguments as
    ``gather`` and ``conv_ref`` take them (call it on copies made before the op runs); ``w`` [KH*KW*Cin, Cout].  Returns NHWC
    dict(y=[N,OH,OW,Cout], bound (the bracket of the tolerance, as ``conv_ref``), masked=[N,OH,OW] bool, and y2 / bound2 when
    ``y2_scale`` is given)."""
    import torch.nn.functional as F
    dev = x.device
    n, h, wd, cin = x.shape
    xs = x.permute(0, 3, 1, 2).double()
    w4 = w.double().to(dev).reshape(kh, kw, cin, -1).permute(3, 2, 0, 1)
    cout = w4.shape[0]
    vw = None if valid_w is None else valid_w.long().to(dev)
    if gn is not None:
        mr, gamma, beta = (t.double().to(dev) for t in gn)
        grp = torch.arange(cin, device=dev) // 32
        t = (xs - mr[:, grp, 0, None, None]) * mr[:, grp, 1, None, None] * gamma[None, :cin, None, None] + beta[None, :cin, None, None]
        xs = t * torch.sigmoid(t)
        if vw is not None:
            xs = xs * (torch.arange(wd, device=dev)[None, :] < vw[:, None])[:, None, None, :]
    acc = F.conv2d(xs, w4, stride=stride, padding=pad).permute(0, 2, 3, 1)
    mag = F.conv2d(xs.abs(), w4.abs(), stride=stride, padding=pad).permute(0, 2, 3, 1)
    if out_scale is not None:
        os_ = out_scale.double().to(dev)[:, None, None, :cout]
        acc = acc * os_
        mag = mag * os_.abs()
    if bias is not None:
        b = bias.double().to(dev)[:cout]
        acc = acc + b
        mag = mag + b.abs()
    if residual is not None:
        r = residual.double().to(dev)[..., :cout]
        if res_broadcast:
            r = r[:1]
        acc = acc + r
        mag = mag + r.abs()
    v = act64(acc, act) * gain
    oh, ow = v.shape[1], v.shape[2]
    masked = torch.zeros(n, oh, ow, dtype=torch.bool, device=dev)
    if vw is not None:
        masked = (torch.arange(ow, device=dev)[None, :] >= vw[:, None])[:, None, :].expand(n, oh, ow)
    v = torch.where(masked[..., None], torch.zeros_like(v), v)
    bound = abs(gain) * LIPSCHITZ[act] * mag
    out = dict(y=v, bound=torch.where(masked[..., None], torch.zeros_like(bound), bound), masked=masked)
    if y2_scale is not None:
        y2s = y2_scale.double().to(dev)[:, None, None, :cout]
        out["y2"] = v * y2s
        out["bound2"] = out["bound"] * y2s.abs()
    return out


def ratio(got, ref, bound, tol):
    """Worst |got - ref| / (tol * (bound + |ref|)); a mismatch where the bound is exactly 0 (a masked output) is infinite."""
    got = got.double().to(ref.device)
    err = (got - ref).abs()
    lim = tol * (bound + ref.abs())
    r = torch.where(lim > 0, err / lim.clamp_min(1e-300), torch.where(err > 0, torch.full_like(err, math.inf), torch.zeros_like(err)))
    r = torch.where(torch.isnan(got), torch.full_like(r, math.inf), r)
    return float(r.max()) if r.numel() else 0.0


def gather_out(y, pix):
    """Values of an NHWC output [N, OH, OW, C] at the sampled pixels, [P, C]."""
    pix = pix.to(y.device)
    return y[pix[:, 0], pix[:, 1], pix[:, 2]].double()


def linear_ref(x2d, w, bias=None, act=0, gain=1.0, residual=None):
    """fp64 ``x2d @ w + bias + residual`` -> act * gain, and its bound (as ``conv_ref``), on x2d's device."""
    x = x2d.double()
    w64 = w.double().to(x.device)
    acc = x @ w64
    mag = x.abs() @ w64.abs()
    if bias is not None:
        acc = acc + bias.double()
        mag = mag + bias.double().abs()
    if residual is not None:
        acc = acc + residual.double()
        mag = mag + residual.double().abs()
    return act64(acc, act) * gain, abs(gain) * LIPSCHITZ[act] * mag


def patch_tokens(feat):
    """TextViT patch rearrangement 'b (p1) (t p2) c -> (b t) (p1 p2 c)' of an NHWC [B, 8, 8T, C] map, fp64."""
    b, fh, fw, c = feat.shape
    t = fw // 8
    return feat.double().reshape(b, 8, t, 8, c).permute(0, 2, 1, 3, 4).reshape(b * t, 64 * c)


def patch_embed_ref(feat, w, bias, pe):
    b, t = feat.shape[0], feat.shape[2] // 8
    return linear_ref(patch_tokens(feat), w, bias, residual=pe.repeat(b, 1).to(feat.device))


def groupnorm_stats64(y, valid_w=None, eps=1e-6, cpg=32):
    """fp64 GroupNorm mean / rstd [N, C/cpg, 2] of an NHWC tensor over each sample's first valid_w[n] columns."""
    y = y.double()
    n, h, w, c = y.shape
    out = torch.empty(n, c // cpg, 2, dtype=torch.float64, device=y.device)
    for i in range(n):
        v = w if valid_w is None else int(valid_w[i])
        t = y[i, :, :v].reshape(-1, c // cpg, cpg).transpose(0, 1).reshape(c // cpg, -1)
        mean = t.mean(1)
        var = ((t - mean[:, None]) ** 2).mean(1)
        out[i, :, 0] = mean
        out[i, :, 1] = (var + eps).rsqrt()
    return out
