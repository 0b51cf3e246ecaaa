"""Print the plan of every ops.conv2d call of a fixed set of workloads, for comparing two builds call by call.

    MN_PRECISION=<p> python tools/dump_conv_plans.py [--out FILE]

Each call is run with ``plan={}`` and printed as: workload, layer name, input shape and strides, the call's options (tensors as
their shapes) and the plan (kernel, precision, nt, TN/TH/TW, split-K, gn_fused, gn_stats_out, x_scale).  After each workload
come the library launches it issued (ops.LAUNCHES), at the end the TC_FALLBACKS keys.  Module graphs are off, so every call is
eager.  Workloads: the bench.py step (1 line x 16 characters), the lines8 TSPSRNet case, a ragged whole-line TSPSRNet batch,
TSPGAN at 16 / 128 / 1024 characters and the direct shapes of tests/test_gpu_conv_sweep.py.  The output depends on the plans
only, not on the data or on the wording of fall-back reasons.
"""
import argparse
import math
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from marconet_b200 import ops  # noqa: E402
from marconet_b200.models import networks  # noqa: E402
from oracle import synth as ckpt  # noqa: E402

DEV = torch.device("cuda:0")
LINES = []


def _fmt(v):
    if isinstance(v, torch.Tensor):
        return f"T{tuple(v.shape)}"
    if isinstance(v, (tuple, list)):
        return "(" + ",".join(_fmt(t) for t in v) + ")"
    if isinstance(v, float):
        return f"{v:.6g}"
    return repr(v)


def _wrap(workload):
    """ops.conv2d, recording every call's plan under ``workload``."""
    orig = ops.conv2d

    def conv2d(x, w, kh, kw, **opts):
        plan = {}
        res = orig(x, w, kh, kw, plan=plan, **opts)
        name = w.name if isinstance(w, ops.ConvWeight) else "raw"
        o = " ".join(f"{k}={_fmt(v)}" for k, v in sorted(opts.items()))
        p = " ".join(f"{k}={_fmt(v)}" for k, v in sorted(plan.items()))
        LINES.append(f"{workload}\t{name}\tx={tuple(x.shape)}/{x.stride()} k={kh}x{kw}\t{o}\t{p}")
        return res
    return orig, conv2d


def _t(*shape, seed, scale=1.0, shift=0.0):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(*shape, generator=g) * scale + shift).to(DEV)


def _cw(cout, cin, k, seed, name):
    g = torch.Generator().manual_seed(seed)
    w4 = torch.randn(cout, cin, k, k, generator=g) / math.sqrt(cin * k * k)
    ops.PLAN.pop(name, None)
    return ops.ConvWeight(w4.permute(2, 3, 1, 0).reshape(k * k * cin, cout).contiguous().to(DEV), k * k, name=name)


def _priors(counts, seed):
    g = torch.Generator().manual_seed(seed)
    return ([torch.randn(c, 256, 64, 64, generator=g).to(DEV) for c in counts],
            [torch.randn(c, 512, 32, 32, generator=g).to(DEV) for c in counts])


def bench_step(nets):
    from marconet_b200.testing import synth
    chars = 16
    lq, labels, locs = synth.make_lq(1, 0).to(DEV), synth.make_labels(chars, 0), synth.make_locs(1, chars).to(DEV)
    _, _, w = nets["encoder"](lq)
    _, f64, f32_ = nets["tspgan"](styles=w.repeat_interleave(chars, dim=0), labels=labels, noise=None)
    nets["sr"](lq, [f64], [f32_], locs)


def lines8(nets):
    from oracle.make_golden2 import lines8_inputs
    inp = lines8_inputs()
    p64, p32 = _priors([l.shape[0] for l in inp["labels"]], 7)
    nets["sr"](inp["lq"].to(DEV), p64, p32, inp["locs"].to(DEV))


def sr_ragged(nets):
    widths, counts = (512, 700, 1264), (12, 20, 44)
    g = torch.Generator().manual_seed(3)
    lq = torch.rand(len(widths), 3, 32, max(widths), generator=g) * 2 - 1
    locs = torch.zeros(len(widths), 2 * max(counts))
    for b, (wb, n) in enumerate(zip(widths, counts)):
        locs[b, 0:2 * n:2] = torch.sort(torch.rand(n, generator=g) * 0.96 + 0.02).values
        locs[b, 1:2 * n:2] = 8.0 / wb
    p64, p32 = _priors(counts, 9)
    nets["sr"](lq.to(DEV), p64, p32, locs.to(DEV), widths=list(widths))


def tspgan(n):
    def run(nets):
        g = torch.Generator().manual_seed(100 + n)
        nets["tspgan"](styles=torch.randn(n, 512, generator=g).to(DEV), labels=torch.randint(0, 6735, (n, 1), generator=g), noise=None)
    return run


def direct(nets):
    """The shapes tests/test_gpu_conv_sweep.py calls ops.conv2d with directly."""
    f16 = ops.PREC_F16X3_TC
    for h, w in ((16, 8), (32, 4), (8, 8), (16, 16)):
        x = _t(3, h, w, 64, seed=1, scale=2.0, shift=0.3)
        vw = torch.tensor([w, max(1, w // 2), w - 1], dtype=torch.int32, device=DEV)
        ops.conv2d(x, _cw(64, 64, 3, 2, f"sweep.gn_{h}x{w}"), 3, 3, pad=(1, 1), bias=_t(64, seed=3), valid_w=vw,
                   gn=(ops.groupnorm_stats(x, valid_w=vw), _t(64, seed=4), _t(64, seed=5)), gn_stats=True, precision=f16)
    for h, w in ((4, 16), (2, 32), (1, 64)):
        x = _t(3, h, w, 64, seed=40)
        cw = _cw(64, 64, 3, 41, f"sweep.tile64_{h}x{w}")
        for feature in ("plain", "gn_stats_valid_w", "y2_ptrs"):
            kw = dict(pad=(1, 1), bias=_t(64, seed=42), out_scale=_t(3, 64, seed=43), act=ops.ACT_LRELU02, gain=2 ** 0.5,
                      out=torch.empty(3, h, w, 64, device=DEV), precision=f16)
            if feature == "gn_stats_valid_w":
                vw = torch.tensor([w, w // 2 + 1, 3], dtype=torch.int32, device=DEV)
                kw.update(valid_w=vw, gn=(ops.groupnorm_stats(x, valid_w=vw), _t(64, seed=44), _t(64, seed=45)), gn_stats=True)
            elif feature == "y2_ptrs":
                dst = [torch.empty(h * w * 64, device=DEV) for _ in range(3)]
                kw.update(out2_ptrs=torch.tensor([b.data_ptr() for b in dst], dtype=torch.int64, device=DEV), y2_scale=_t(3, 64, seed=46))
            ops.conv2d(x, cw, 3, 3, **kw)
    for n, h, w, cin, cout in ((4, 32, 32, 64, 128), (16, 64, 64, 64, 128), (5, 4, 4, 64, 64)):
        ops.conv2d(_t(n, h, w, cin, seed=10), _cw(cout, cin, 3, 11, f"sweep.act_tanh_{n}"), 3, 3, pad=(1, 1), bias=_t(cout, seed=12),
                   out_scale=_t(n, cout, seed=13), residual=_t(1, h, w, cout, seed=14), res_broadcast=True, act=ops.ACT_TANH,
                   gain=1.5, precision=f16)
    for h, w in ((6, 128), (12, 256)):
        buf = torch.zeros(3, h, w, 192, device=DEV)
        vw = torch.tensor([w, w // 2 + 3, 17], dtype=torch.int32, device=DEV)
        ops.conv2d(_t(3, h, w, 64, seed=20), _cw(128, 64, 3, 21, f"sweep.tc1_{h}"), 3, 3, pad=(1, 1), bias=_t(128, seed=22),
                   out_scale=_t(3, 256, seed=23)[:, 128:], residual=_t(3, h, w, 128, seed=24), act=ops.ACT_LRELU02, gain=2 ** 0.5,
                   out=buf[..., 32:160], out2=True, y2_scale=_t(3, 128, seed=25), valid_w=vw, precision=f16)
    ops.conv2d(_t(2, 32, 32, 128, seed=30), _cw(128, 128, 3, 31, "sweep.stats"), 3, 3, pad=(1, 1),
               bias=torch.full((128,), 30.0, device=DEV), gn_stats=True, precision=f16)


WORKLOADS = [("bench_step_1x16", bench_step), ("sr_lines8", lines8), ("sr_ragged_3", sr_ragged), ("tspgan_n16", tspgan(16)),
             ("tspgan_n128", tspgan(128)), ("tspgan_n1024", tspgan(1024)), ("direct", direct)]


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--out", help="write here instead of stdout")
    args = ap.parse_args()
    ops.MODULE_GRAPHS = False
    sds = ckpt.make_checkpoints(0)
    nets = {}
    for key, cls in (("tspgan", networks.TSPGAN), ("encoder", networks.TextContextEncoderV2), ("sr", networks.TSPSRNet)):
        m = cls()
        m.load_state_dict(sds[key], strict=True)
        nets[key] = m.eval().to(DEV)
    LINES.append(f"# default precision {ops.default_precision()}")
    for name, fn in WORKLOADS:
        orig, wrapped = _wrap(name)
        ops.conv2d = wrapped
        before = ops.LAUNCHES
        try:
            with torch.no_grad():
                fn(nets)
            torch.cuda.synchronize()
        finally:
            ops.conv2d = orig
        LINES.append(f"# {name}: {ops.LAUNCHES - before} library launches")
    LINES.append("# TC_FALLBACKS keys: " + " ".join(repr(k) for k in sorted(ops.TC_FALLBACKS)))
    text = "\n".join(LINES) + "\n"
    if args.out:
        with open(args.out, "w") as f:
            f.write(text)
    else:
        sys.stdout.write(text)


if __name__ == "__main__":
    main()
