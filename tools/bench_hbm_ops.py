"""Times the HBM-bound operators at the shapes of the bench step (1 line x 16 chars) with CUDA events, L2 flushed
between launches, and prints achieved GB/s against the algorithmic bytes (minimal fp32 read + write of the operands,
SURVEY 8d).  Usage (on the GPU box):  python tools/bench_hbm_ops.py [--iters 20] [--only NAME]
"""
import argparse
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from marconet_b200 import ops  # noqa: E402


def timeit(fn, iters, flush):
    st = torch.cuda.current_stream()
    tot = 0.0
    for i in range(iters + 3):
        flush.zero_()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(st)
        fn()
        e1.record(st)
        torch.cuda.synchronize()
        if i >= 3:
            tot += e0.elapsed_time(e1)
    return tot / iters * 1e3     # us


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--only", default="", help="time only the operators whose name contains this string (e.g. 'groupnorm_stats')")
    args = ap.parse_args()
    dev = torch.device("cuda:0")
    flush = torch.empty(64 << 20, dtype=torch.float32, device=dev)
    rows = []

    def add(name, fn, nbytes):
        if args.only not in name:
            return
        us = timeit(fn, args.iters, flush)
        rows.append({"op": name, "us": round(us, 1), "MB": round(nbytes / 1e6, 1), "GB/s": round(nbytes / us / 1e3, 0)})

    # bilinear x2 (+ style) : TSPGAN [16,H,W,C] and TSPSRNet [1,H,W,C]
    for n, h, w, c, styled in ((16, 64, 64, 256, True), (16, 32, 32, 512, True), (16, 16, 16, 512, True),
                               (1, 64, 1024, 128, False), (1, 32, 512, 256, False)):
        x = torch.randn(n, h, w, c, device=dev)
        s = torch.randn(n, c, device=dev) if styled else None
        y = torch.empty(n, 2 * h, 2 * w, c, device=dev)
        add(f"resample_modulate up [{n},{h},{w},{c}]", lambda: ops.resample_modulate(x, s, up=True, out=y), 5 * x.numel() * 4)
        del x, y
    # GroupNorm stats / apply+swish
    for n, h, w, c in ((1, 128, 2048, 64), (1, 64, 1024, 256), (16, 64, 64, 512), (16, 32, 32, 512)):
        x = torch.randn(n, h, w, c, device=dev)
        ga, be = torch.randn(c, device=dev), torch.randn(c, device=dev)
        y = torch.empty_like(x)
        mr = ops.groupnorm_stats(x)
        add(f"groupnorm_stats [{n},{h},{w},{c}]", lambda: ops.groupnorm_stats(x), x.numel() * 4)
        add(f"groupnorm_apply+swish [{n},{h},{w},{c}]", lambda: ops.groupnorm_apply(x, mr, ga, be, out=y), 2 * x.numel() * 4)
        del x, y
    # AdaIN + concat (statistics pass, then apply): 16 characters on a 512-wide line, windows 32 columns wide; bytes = prior crops and
    # feature windows read once, the [Nc, H, wp, 2C] output written once
    for nc, h, wp, c in ((16, 32, 32, 256), (16, 64, 64, 256)):
        prior = torch.randn(nc, h, wp, c, device=dev)
        feat = torch.randn(1, h, nc * wp, c, device=dev)
        win = torch.tensor([[0, i * wp, (i + 1) * wp, 0] for i in range(nc)], dtype=torch.int32, device=dev)
        add(f"adain_concat [{nc},{h},{wp},{c}]", lambda: ops.adain_concat(prior, feat, win, nc, wp), 4 * nc * h * wp * c * 4)
        del prior, feat
    # ToRGB
    for n, h, c in ((16, 128, 128), (16, 64, 256), (16, 32, 512)):
        x = torch.randn(n, h, h, c, device=dev)
        s = torch.randn(n, c, device=dev)
        wt, b = torch.randn(3, c, device=dev), torch.randn(3, device=dev)
        skip = torch.randn(n, h // 2, h // 2, 3, device=dev)
        add(f"torgb [{n},{h},{h},{c}]", lambda: ops.torgb(x, s, wt, b, skip), x.numel() * 4 + n * h * h * 3 * 4 * 1.25)
        del x
    # small-M linears (weight streaming): bytes = the weight matrix
    for m, k, n in ((16, 512, 512), (64, 512, 512), (64, 512, 1536), (64, 512, 1024), (64, 1024, 512), (64, 512, 6736), (16, 512, 7168)):
        x, w, b = torch.randn(m, k, device=dev), torch.randn(k, n, device=dev), torch.randn(n, device=dev)
        add(f"linear_small_m [{m}x{k}x{n}]", lambda: ops.linear(x, w, b), k * n * 4)
    feat = torch.randn(1, 8, 512, 512, device=dev)
    w, b, pe = torch.randn(32768, 512, device=dev), torch.randn(512, device=dev), torch.randn(64, 512, device=dev)
    add("patch_embed [64x32768x512]", lambda: ops.patch_embed(feat, w, b, pe), 32768 * 512 * 4)
    # NCHW <-> NHWC and the final 64->3 conv are covered by bench_conv.py
    for r in rows:
        print(json.dumps(r))


if __name__ == "__main__":
    main()
