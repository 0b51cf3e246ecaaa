"""Ragged-width SR decoder batches (mn_resample_modulate_ragged, mn_char_windows_ragged, TSPSRNet(..., widths=)) and lines decoded
in one piece (pipeline.restore_images(whole_lines=True)) on the GPU: each line of a ragged batch against the same module on that
line alone at its exact width and against the oracle, and the whole-line bytes against tests/golden/whole_line.npz (the
reference modules run on each whole line, oracle/make_golden_whole_line.py)."""
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
TOL = 1e-3          # the project's max-abs budget against the oracle
dev = torch.device("cuda:0")


def test_resample_ragged_equals_each_sample_alone_at_its_width():
    from marconet_b200 import ops
    g = torch.Generator().manual_seed(3)
    n, h, w, c = 4, 8, 45, 64
    x = torch.randn(n, h, w, c, generator=g).to(dev)
    s = torch.randn(n, c, generator=g).to(dev)
    valid = [45, 17, 4, 1]
    vw = torch.tensor(valid, dtype=torch.int32, device=dev)
    for sc in (None, s):
        out = torch.full((n, 2 * h, 2 * w, c), float("nan"), device=dev)
        ops.resample_up2_ragged(x, vw, s=sc, out=out)
        for b, v in enumerate(valid):
            ref = ops.resample_modulate(x[b:b + 1, :, :v].contiguous(), None if sc is None else sc[b:b + 1], up=True)
            assert torch.equal(out[b:b + 1, :, :2 * v], ref), b
            assert (out[b, :, 2 * v:] == 0).all()
    # a channel slice of a wider buffer (the trunk's concatenation buffers) as input and output
    big = torch.randn(n, h, w, 2 * c, generator=g).to(dev)
    dst = torch.full((n, 2 * h, 2 * w, 3 * c), float("nan"), device=dev)
    ops.resample_up2_ragged(big[..., c:], vw, out=dst[..., :c])
    for b, v in enumerate(valid):
        ref = ops.resample_modulate(big[b:b + 1, :, :v, c:].contiguous(), None, up=True)
        assert torch.equal(dst[b:b + 1, :, :2 * v, :c], ref)
        assert (dst[b, :, 2 * v:, :c] == 0).all()


def test_char_windows_ragged_equals_the_host_twin():
    from marconet_b200 import ops
    from marconet_b200.models.networks import TSPSRNet, _char_windows_np
    rng = np.random.default_rng(5)
    sr = TSPSRNet()
    for trial in range(30):
        b = int(rng.integers(1, 6))
        widths = [int(v) for v in rng.integers(1, 520, b) * 4]
        canvas = max(widths) + 4 * int(rng.integers(0, 3))
        half = (16, 32)[trial % 2]
        counts = [int(v) for v in rng.integers(1, 75, b)]
        locs = np.zeros((b, 2 * max(counts)), np.float32)
        for i, (wb, nc) in enumerate(zip(widths, counts)):
            locs[i, 0:2 * nc:2] = rng.choice([rng.uniform(0, 1), (wb - rng.integers(0, half + 2)) / wb, rng.uniform(0.97, 1.0)], size=nc)
        flag = torch.zeros(1, dtype=torch.int32, device=dev)
        lw = torch.tensor(widths, dtype=torch.int32, device=dev)
        win, valid, owner = ops.char_windows_ragged(torch.from_numpy(locs).to(dev), sr._line_first(counts, dev), lw, counts, canvas,
                                                    half, flag)
        try:
            hw, hv, ho = _char_windows_np(locs, counts, canvas, half, line_w=widths)
        except RuntimeError:
            assert int(flag.item()) & ops.ERR_WINDOW, trial
            continue
        assert int(flag.item()) == 0
        assert np.array_equal(win.cpu().numpy(), hw) and np.array_equal(valid.cpu().numpy(), hv)
        assert np.array_equal(owner.cpu().numpy(), ho)


def _ragged_inputs(gm, widths, counts, seed=0):
    """lq [B, 3, 32, max(widths)] (garbage beyond each line's width: the module must ignore it), TSPGAN priors, locs."""
    g = torch.Generator().manual_seed(seed)
    canvas = max(widths)
    lq = torch.rand(len(widths), 3, 32, canvas, generator=g) * 2 - 1
    locs = torch.zeros(len(widths), 2 * max(counts))
    for b, (wb, n) in enumerate(zip(widths, counts)):
        cen = torch.sort(torch.rand(n, generator=g) * 0.96 + 0.02).values
        locs[b, 0:2 * n:2] = cen
        locs[b, 1:2 * n:2] = 8.0 / wb
    styles = torch.randn(sum(counts), 512, generator=g).to(dev)
    labels = torch.randint(0, 6735, (sum(counts), 1), generator=g)
    _, f64, f32_ = gm["tspgan"](styles=styles, labels=labels, noise=None)
    p64, p32, o = [], [], 0
    for n in counts:
        p64.append(f64[o:o + n]); p32.append(f32_[o:o + n]); o += n
    return lq.to(dev), p64, p32, locs


def _alone(gm, lq, p64, p32, locs, widths, counts, b):
    wb = widths[b]
    return gm["sr"](lq[b:b + 1, :, :, :wb].contiguous(), [p64[b]], [p32[b]], locs[b:b + 1, :2 * counts[b]] * 1.0)


@pytest.mark.parametrize("widths,counts", [((512, 700, 1264), (12, 20, 44)), ((2048, 516), (70, 9))])
def test_ragged_tspsrnet_matches_each_line_alone_and_the_oracle(gpu_models, checkpoints, widths, counts):
    from oracle import restate
    gm = gpu_models
    lq, p64, p32, locs = _ragged_inputs(gm, list(widths), list(counts))
    outs = [gm["sr"](lq, p64, p32, locs, widths=list(widths)) for _ in range(3)]       # eager, then recorded and replayed
    torch.cuda.synchronize()
    for o in outs[1:]:
        assert (o - outs[0]).abs().max().item() <= 1e-5
    out = outs[0]
    assert tuple(out.shape) == (len(widths), 3, 128, 4 * max(widths))
    for b, wb in enumerate(widths):
        alone = _alone(gm, lq, p64, p32, locs, list(widths), list(counts), b)
        err = (out[b:b + 1, :, :, :4 * wb] - alone).abs().max().item()
        assert err <= 1e-4, (b, err)
        assert (out[b, :, :, 4 * wb:] == 0).all()
        # the fp32 CPU oracle on the line alone at its exact width
        ref = restate.tspsr_forward(checkpoints["sr"], lq[b:b + 1, :, :, :wb].cpu(), [p64[b].cpu()], [p32[b].cpu()],
                                    locs[b:b + 1, :2 * counts[b]])
        oerr = (out[b:b + 1, :, :, :4 * wb].cpu() - ref).abs().max().item()
        print(f"\nwidths {widths} line {b} (width {wb}, {counts[b]} chars): max-abs vs alone {err:.2e}, vs oracle {oerr:.2e}")
        assert oerr <= TOL, (b, oerr)


def test_equal_widths_take_the_unchanged_path_and_recordings_never_cross(gpu_models):
    from marconet_b200 import ops
    gm = gpu_models
    widths = [640, 640, 640]
    lq, p64, p32, locs = _ragged_inputs(gm, widths, [6, 9, 4], seed=1)
    prev = ops.MODULE_GRAPHS
    try:
        ops.MODULE_GRAPHS = False
        a = gm["sr"](lq, p64, p32, locs)
        b = gm["sr"](lq, p64, p32, locs, widths=widths)
        assert torch.equal(a, b)
        eager = {wd: gm["sr"](lq, p64, p32, locs, widths=list(wd)) for wd in ((640, 512, 320), (320, 640, 512))}
    finally:
        ops.MODULE_GRAPHS = prev
    got = {}
    for wd in ((640, 512, 320), (320, 640, 512), (640, 512, 320), (320, 640, 512), (640, 512, 320)):
        got[wd] = gm["sr"](lq, p64, p32, locs, widths=list(wd))       # the second sighting of each tuple records its own graph
        assert (got[wd] - eager[wd]).abs().max().item() <= 1e-5, wd
    assert (got[(640, 512, 320)] - got[(320, 640, 512)]).abs().max().item() > 0.1


def test_a_recording_outlives_the_eviction_of_its_width_table(gpu_models):
    """A graph recorded for one widths tuple keeps its device width table: after 70 other tuples have gone through the module's
    bounded cache (which drops the table) and fresh small allocations have taken the freed memory, replays still give the
    eager result."""
    from marconet_b200 import ops
    gm = gpu_models
    widths = [640, 320, 512]
    lq, p64, p32, locs = _ragged_inputs(gm, widths, [7, 3, 5], seed=2)
    prev = ops.MODULE_GRAPHS
    try:
        ops.MODULE_GRAPHS = False
        eager = gm["sr"](lq, p64, p32, locs, widths=widths)
    finally:
        ops.MODULE_GRAPHS = prev
    for _ in range(2):                                    # second sighting: recorded
        gm["sr"](lq, p64, p32, locs, widths=widths)
    for k in range(70):
        gm["sr"]._valid_widths((4 * (k + 1), 640, 4), dev)
    assert (tuple(widths), dev) not in gm["sr"]._widths_cache
    junk = [torch.full((5, 3), 1, dtype=torch.int32, device=dev) for _ in range(256)]
    got = gm["sr"](lq, p64, p32, locs, widths=widths)
    torch.cuda.synchronize()
    del junk
    assert (got - eager).abs().max().item() <= 1e-5


def _run(gm, images, **kw):
    from marconet_b200 import pipeline
    return pipeline.restore_images(gm["encoder"], gm["tspgan"], gm["sr"], [i[0] for i in images], [i[1] for i in images],
                                   [i[2] for i in images], **kw)


def _golden_lines():
    g = np.load(os.path.join(GOLDEN, "whole_line.npz"))
    return g, [(g[f"image{i}"], g[f"labels{i}"].tolist(), g[f"boxes{i}"].tolist()) for i in range(int(g["lines"]))]


def _within_one_level(got, ref, what):
    assert got.shape == ref.shape, (what, got.shape, ref.shape)
    diff = np.abs(got.astype(int) - ref.astype(int))
    assert diff.max() <= 1 and (diff != 0).mean() < 0.15, (what, int(diff.max()), float((diff != 0).mean()))


def test_whole_lines_match_the_reference_modules_on_the_whole_line(gpu_models):
    from marconet_b200 import ops
    g, lines = _golden_lines()
    stride = int(g["stride"])
    for ml in (1, 8):
        l0 = ops.LAUNCHES
        res = _run(gpu_models, lines, max_lines=ml, whole_lines=True, to_host=True)
        print(f"\nwhole_lines max_lines={ml}: {ops.LAUNCHES - l0} C-ABI launches")
        for i, r in enumerate(res):
            assert [list(s.crop) for s in r["segments"]] == g[f"crops{i}"].tolist()
            _within_one_level(r["sr_u8"][::stride, ::stride], g[f"sr_u8{i}"], (ml, i))


def test_mixed_batch_of_short_and_whole_lines(gpu_models):
    from marconet_b200 import pipeline
    gm = gpu_models
    rng = np.random.default_rng(11)
    short = [(rng.integers(0, 256, (40, 500, 3), dtype=np.uint8), [5, 17, 300, 4242], [[20 + 110 * i, 4, 100 + 110 * i, 36] for i in range(4)]),
             (rng.integers(0, 256, (24, 300, 3), dtype=np.uint8), [7, 8, 9], [[10, 2, 60, 22], [90, 2, 150, 22], [200, 2, 280, 22]])]
    _, wide = _golden_lines()
    images = [wide[0], short[0], wide[1], short[1]]
    alone_short = [pipeline.restore_image(gm["encoder"], gm["tspgan"], gm["sr"], *s)["sr_u8"].cpu().numpy() for s in short]
    alone_wide = [_run(gm, [w], max_lines=1, whole_lines=True, to_host=True)[0]["sr_u8"] for w in wide]
    for ml in (1, 8):
        res = _run(gm, images, max_lines=ml, whole_lines=True, to_host=True)
        for k, ref in ((1, alone_short[0]), (3, alone_short[1])):
            if ml == 1:             # a short line batched only with itself: restore_image's bytes
                assert np.array_equal(res[k]["sr_u8"], ref), k
            else:
                _within_one_level(res[k]["sr_u8"], ref, (ml, k))
        for k, ref in ((0, alone_wide[0]), (2, alone_wide[1])):
            _within_one_level(res[k]["sr_u8"], ref, (ml, k))
    # the default mode is untouched by the flag's existence: wide images still go crop by crop
    assert len(_run(gm, [wide[0]])[0]["segments"]) == 4
