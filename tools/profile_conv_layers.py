"""Per-layer timing of every mn_conv2d_nhwc call of one 16-character line (developer tool): CUDA events around each eager call,
warm caches, module graphs off.  Prints the layers sorted by time with their algorithmic TFLOP/s and, for the tensor-core layers, the
fraction of the tensor pipe (3 fp16 MMA passes per fp32-grade product, against MEASURED_PEAKS.json's bf16 burst peak when present,
else the H100 SXM data sheet's 989 TFLOP/s dense bf16, a 700 W figure).  The last column is the plan that ran: kernel / NT (the
tensor-core work-item width, 0 for the fp32 kernels) and, when split, ksS.

    MN_MODULE_GRAPHS=0 python tools/profile_conv_layers.py [--chars 16] [--iters 10]
"""
import argparse
import json
import os
import sys
from collections import defaultdict

os.environ.setdefault("MN_MODULE_GRAPHS", "0")
import torch  # noqa: E402

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--chars", type=int, default=16)
    ap.add_argument("--iters", type=int, default=10)
    args = ap.parse_args()
    from marconet_b200 import ops
    from marconet_b200.models import networks
    from marconet_b200.testing import synth
    dev = torch.device("cuda:0")
    sds = synth.make_checkpoints(0)
    nets = {}
    for key, cls in (("tspgan", networks.TSPGAN), ("encoder", networks.TextContextEncoderV2), ("sr", networks.TSPSRNet)):
        m = cls()
        m.load_state_dict(sds[key], strict=True)
        nets[key] = m.eval().to(dev)
    C = args.chars
    lq = synth.make_lq(1, 0).to(dev)
    labels = synth.make_labels(C, 0)
    locs = synth.make_locs(1, C).to(dev)
    enc, gen, sr = nets["encoder"], nets["tspgan"], nets["sr"]
    recs = defaultdict(list)
    plans = {}      # call index -> "kernel/NT [ksS]" of the plan that ran
    real = ops.conv2d
    seq = [0]

    def timed(x, w, kh, kw, *a, **k):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        if k.get("plan") is None:
            k["plan"] = {}
        plan = k["plan"]
        e0.record()
        out = real(x, w, kh, kw, *a, **k)
        e1.record()
        n, h, wd, cin, _ = ops.nhwc_info(x, "x")
        cout = (w.w if isinstance(w, ops.ConvWeight) else w).shape[1]
        y = out[0] if isinstance(out, tuple) else out
        oh, ow = (y.shape[1], y.shape[2]) if y is not None else (h, wd)
        name = getattr(w, "name", None) or "?"
        recs[(seq[0], name, n, h, wd, cin, cout, kh, oh, ow)].append((e0, e1))
        plans[seq[0]] = f"{plan['kernel']}/{plan['nt']}" + (f" ks{plan['splits']}" if plan["splits"] > 1 else "")
        seq[0] += 1
        return out

    ops.conv2d = timed
    networks.ops.conv2d = timed

    def one_pass():
        seq[0] = 0
        with torch.no_grad():
            _, _, w = enc(lq)
            _, f64, f32_ = gen(styles=w.repeat_interleave(C, dim=0), labels=labels, noise=None)
            return sr(lq, [f64], [f32_], locs)

    for _ in range(3):
        one_pass()
    torch.cuda.synchronize()
    recs.clear()
    for _ in range(args.iters):
        one_pass()
    torch.cuda.synchronize()
    peak = 989.0      # NVIDIA H100 SXM data sheet, dense bf16 (700 W card), as bench.py uses
    try:
        peak = json.load(open(os.path.join(os.path.dirname(__file__), "..", "MEASURED_PEAKS.json")))["bf16_tflops"]
    except Exception:
        pass
    rows = []
    for (s, name, n, h, wd, cin, cout, kh, oh, ow), evs in recs.items():
        ts = sorted(a.elapsed_time(b) * 1e3 for a, b in evs)
        us = ts[len(ts) // 2]
        flop = 2.0 * n * oh * ow * cout * cin * kh * kh
        rows.append((us, s, name, f"N{n} {h}x{wd} {cin}->{cout} k{kh}", flop / us * 1e-6, plans[s]))
    total = sum(r[0] for r in rows)
    print(f"{len(rows)} conv calls, {total:.0f} us per line in convs (eager, event-timed incl. launch gaps); tensor-pipe column assumes 3 MMA passes")
    for us, s, name, shape, tf, pl in sorted(rows, reverse=True):
        print(f"{us:8.1f} us {100 * us / total:5.1f}%  #{s:<3d} {name:<44s} {shape:<28s} {tf:7.1f} TF  pipe {3 * tf / peak:5.2f}  {pl}")


if __name__ == "__main__":
    main()
