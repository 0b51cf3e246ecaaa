"""Seeded forwards of the three modules that the per-call sweeps (tests/test_gpu_conv_sweep.py, tests/test_gpu_op_sweep.py) run
with their ops wrapped: every workload takes the dict of modules on cuda:0 ({"encoder", "tspgan", "sr"}) and runs one eager forward.
Between them they reach every kernel branch the modules use: batch 1 and 8 encoders, TSPGAN at 1 / 16 / 17 / 128 characters and
at two labels per character, TSPSRNet on the golden cases and on ragged-width batches."""
import torch


def _dev():
    return torch.device("cuda:0")


def encoder(gm, b):
    from marconet_b200.testing import synth
    gm["encoder"](synth.make_lq(b, 0).to(_dev()))


def tspgan(gm, n, l=1, labels_on_device=False):
    g = torch.Generator().manual_seed(100 + n)
    styles = torch.randn(n, 512, generator=g).to(_dev())
    labels = torch.randint(0, 6735, (n, l), generator=g)
    if labels_on_device:
        labels = labels.to(_dev())
    return gm["tspgan"](styles=styles, labels=labels, noise=None)


def priors(counts, seed):
    g = torch.Generator().manual_seed(seed)
    return ([torch.randn(c, 256, 64, 64, generator=g).to(_dev()) for c in counts],
            [torch.randn(c, 512, 32, 32, generator=g).to(_dev()) for c in counts])


def sr_case(gm, name):
    from oracle.make_golden import case_inputs
    from oracle.make_golden2 import lines8_inputs
    inp = case_inputs(name) if name != "lines8" else lines8_inputs()
    p64, p32 = priors([l.shape[0] for l in inp["labels"]], 7)
    gm["sr"](inp["lq"].to(_dev()), p64, p32, inp["locs"].to(_dev()))


def sr_ragged_inputs(widths, counts):
    """(lq [B, 3, 32, max(widths)], locs [B, 2 * max(counts)]) on the CPU: sorted centres, boxes 8 / width wide."""
    g = torch.Generator().manual_seed(3)
    lq = torch.rand(len(widths), 3, 32, max(widths), generator=g) * 2 - 1
    locs = torch.zeros(len(widths), 2 * max(counts))
    for b, (wb, n) in enumerate(zip(widths, counts)):
        locs[b, 0:2 * n:2] = torch.sort(torch.rand(n, generator=g) * 0.96 + 0.02).values
        locs[b, 1:2 * n:2] = 8.0 / wb
    return lq, locs


def sr_ragged(gm, widths, counts):
    lq, locs = sr_ragged_inputs(widths, counts)
    p64, p32 = priors(counts, 9)
    gm["sr"](lq.to(_dev()), p64, p32, locs.to(_dev()), widths=list(widths))


WORKLOADS = {
    "encoder_b1": lambda gm: encoder(gm, 1),
    "encoder_b8": lambda gm: encoder(gm, 8),
    "tspgan_n1": lambda gm: tspgan(gm, 1),
    "tspgan_n16": lambda gm: tspgan(gm, 16),
    "tspgan_n17": lambda gm: tspgan(gm, 17),
    "tspgan_n128": lambda gm: tspgan(gm, 128),
    "tspgan_n3_l2": lambda gm: tspgan(gm, 3, 2),
    "sr_config2": lambda gm: sr_case(gm, "config2"),
    "sr_lines8": lambda gm: sr_case(gm, "lines8"),
    "sr_ragged_3": lambda gm: sr_ragged(gm, (512, 700, 1264), (12, 20, 44)),
    "sr_ragged_2": lambda gm: sr_ragged(gm, (2048, 516), (70, 9)),
}
SUBSET = ["encoder_b1", "tspgan_n16", "tspgan_n3_l2", "sr_config2"]     # every module, split-K and TN > 1 of the convolution sweep
