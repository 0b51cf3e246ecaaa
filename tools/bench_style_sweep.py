"""BASELINE configs[4] / SURVEY 8d config 5: the data flow of the reference's test_w.py:95-108 scaled up -- two encoder
passes give w1, w2; labels = the 16 characters of image 1; priors are generated for `--steps` interpolated styles
w = w1*t + w2*(1-t), either one TSPGAN call per step (like the script) or one batched call of steps*16 (char, w) pairs.

    python tools/bench_style_sweep.py [--steps 256] [--chars 16] [--mode per_step|batched] [--chunk 128]
    python tools/bench_style_sweep.py --api [--steps 256] [--passes 3] [--api-chunks 16,128,512]

Prints one JSON line: prior characters per second (CUDA events, max of nothing: single GPU), the launch count per TSPGAN call and
the tensor-pipe share implied by the algorithmic 41.785 GFLOP per character (SURVEY 8d).  Not part of the product path.

--api times the whole user-facing path on test_w.py's two images (the content decodes 17 characters): host uint8 images in,
host uint8 strips out, one strip per style, --steps styles.  Arms: pipeline.interpolate_styles at each max_chars of --api-chunks,
and test_w.py's loop as tests/test_pipeline.py writes it out (host pre-processing, two encoder calls, host label decode, one
generator call per style with the style repeated, one copy back and a host strip per style).  The arms alternate pass by pass
after one warm-up pass each; each pass ends in a synchronisation.  One JSON line per arm: strip characters per second (median
pass), launches per call, torch.cuda.max_memory_reserved() of a pass, the largest grey-level difference from the loop's strips,
and the card's name and power limit read in the same run.
"""
import argparse
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

GFLOP_PER_CHAR = 41.785      # SURVEY 8d: TSPGAN, algorithmic


def _card():
    import subprocess
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True,
                       text=True)
    name, _, power = q.stdout.strip().partition(", ")
    return {"gpu": name or torch.cuda.get_device_name(0), "power_limit": power or None}


def api_main(args):
    import statistics
    import time

    import numpy as np
    from marconet_b200 import ops, pipeline
    from marconet_b200.models import networks
    from marconet_b200.testing import synth
    from oracle import image_ops
    from oracle.make_golden_script_w import input_arrays

    dev = torch.device("cuda:0")
    sds = synth.make_checkpoints(0)
    enc, gen = networks.TextContextEncoderV2(), networks.TSPGAN()
    enc.load_state_dict(sds["encoder"], strict=True)
    gen.load_state_dict(sds["tspgan"], strict=True)
    enc, gen = enc.eval().to(dev), gen.eval().to(dev)
    pair = tuple(np.ascontiguousarray(a[..., ::-1]) for a in input_arrays())      # the RGB arrays test_w.py holds
    scales = [i / (args.steps - 1) for i in range(args.steps)]

    def api(max_chars):
        return pipeline.interpolate_styles(enc, gen, [pair], scales=scales, max_chars=max_chars, to_host=True)[0]["strips"]

    def loop():                                                   # tests/test_pipeline.py::test_w_flow_on_gpu_matches_reference_script_pngs
        with torch.no_grad():
            lqs = [torch.from_numpy(image_ops.preprocess_lq(a)[0]).to(dev) for a in pair]
            logits1, _, w1 = enc(lqs[0])
            _, _, w2 = enc(lqs[1])
            labels = torch.tensor(pipeline.decode_labels(logits1[0]), dtype=torch.long).reshape(-1, 1)
            out = []
            for s in scales:
                prior, _, _ = gen(styles=(w1 * s + w2 * (1 - s)).repeat(labels.shape[0], 1), labels=labels, noise=None)
                row = np.hstack(list((prior * 0.5 + 0.5).permute(0, 2, 3, 1).cpu().numpy())) * 255.0
                out.append(np.clip(np.rint(row), 0, 255).astype(np.uint8))
            return np.stack(out)

    arms = [(f"interpolate_styles max_chars={c}", lambda c=c: api(c)) for c in args.api_chunks] + [("test_w.py loop", loop)]
    times, launches, mem, ref, diff = {}, {}, {}, None, {}
    for name, fn in arms:                                         # warm-up pass: every shape recorded, reference strips kept
        out = fn()
        if name == "test_w.py loop":
            ref = out
        diff[name] = out
    for name in diff:
        diff[name] = int(np.abs(diff[name].astype(np.int64) - ref.astype(np.int64)).max())
    for _ in range(args.passes):
        for name, fn in arms:
            torch.cuda.synchronize()
            torch.cuda.empty_cache()
            torch.cuda.reset_peak_memory_stats()
            l0 = ops.LAUNCHES
            t0 = time.perf_counter()
            fn()
            torch.cuda.synchronize()
            times.setdefault(name, []).append(time.perf_counter() - t0)
            launches[name] = ops.LAUNCHES - l0
            mem[name] = max(mem.get(name, 0), torch.cuda.max_memory_reserved())
    card = _card()
    n_chars = ref.shape[2] // 128
    for name, _ in arms:
        med = statistics.median(times[name])
        print(json.dumps({"workload": f"test_w.py style sweep, host images to host strips: {args.steps} styles x {n_chars} chars",
                          "arm": name, "strip_chars_per_sec": args.steps * n_chars / med, "sec_per_call_median": med,
                          "sec_per_call": times[name], "launches_per_call": launches[name], "max_memory_reserved_bytes": mem[name],
                          "max_grey_diff_vs_loop": diff[name], **card}), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=256, help="interpolation steps (test_w.py uses 11)")
    ap.add_argument("--chars", type=int, default=16)
    ap.add_argument("--mode", default="batched", choices=["per_step", "batched"])
    ap.add_argument("--chunk", type=int, default=128, help="(char, w) pairs per TSPGAN call in batched mode")
    ap.add_argument("--repeat", type=int, default=2)
    ap.add_argument("--api", action="store_true", help="time pipeline.interpolate_styles against test_w.py's loop, images to strips")
    ap.add_argument("--api-chunks", type=lambda v: [int(c) for c in v.split(",")], default=[16, 128, 512],
                    help="max_chars values of the --api arms")
    ap.add_argument("--passes", type=int, default=3, help="timed passes per arm in --api mode")
    args = ap.parse_args()
    if args.api:
        return api_main(args)
    from marconet_b200 import ops
    from marconet_b200.models import networks
    from marconet_b200.testing import synth

    dev = torch.device("cuda:0")
    sds = synth.make_checkpoints(0)
    enc, gen = networks.TextContextEncoderV2(), networks.TSPGAN()
    enc.load_state_dict(sds["encoder"], strict=True)
    gen.load_state_dict(sds["tspgan"], strict=True)
    enc, gen = enc.eval().to(dev), gen.eval().to(dev)
    labels = synth.make_labels(args.chars, 7).to(dev)
    with torch.no_grad():
        _, _, w1 = enc(synth.make_lq(1, 21).to(dev))
        _, _, w2 = enc(synth.make_lq(1, 22).to(dev))
        ts = torch.linspace(0, 1, args.steps, device=dev).view(-1, 1)
        w_steps = w1 * ts + w2 * (1 - ts)                                   # [steps, 512]   (test_w.py:101)

        def sweep():
            if args.mode == "per_step":
                for i in range(args.steps):
                    gen(styles=w_steps[i:i + 1].repeat(args.chars, 1), labels=labels, noise=None)
            else:
                styles = w_steps.repeat_interleave(args.chars, dim=0)      # [steps*chars, 512]
                labs = labels.repeat(args.steps, 1)
                for c0 in range(0, styles.shape[0], args.chunk):
                    gen(styles=styles[c0:c0 + args.chunk], labels=labs[c0:c0 + args.chunk], noise=None)

        sweep()
        torch.cuda.synchronize()
        l0 = ops.LAUNCHES
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(args.repeat):
            sweep()
        e1.record()
        torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / args.repeat
    total = args.steps * args.chars
    calls = args.steps if args.mode == "per_step" else -(-total // args.chunk)
    print(json.dumps({"workload": f"test_w.py sweep: {args.steps} styles x {args.chars} chars, {args.mode}", "prior_chars_per_sec": total / (ms / 1e3),
                      "ms_per_sweep": ms, "tspgan_calls": calls, "launches_per_call": (ops.LAUNCHES - l0) // (args.repeat * calls),
                      "algorithmic_tflops": total * GFLOP_PER_CHAR / ms, "chunk": args.chunk if args.mode == "batched" else args.chars}))


if __name__ == "__main__":
    main()
