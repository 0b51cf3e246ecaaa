"""Lines decoded in one piece (pipeline.restore_images(whole_lines=True), TSPSRNet's ``widths``) on the CPU: the oracle reproduces
tests/golden/whole_line.npz (oracle/make_golden_whole_line.py: the reference modules run on each whole line), the host window
integers of a ragged batch equal the ones the reference loop computed on each line alone, and the new kernels' C ABI."""
import os
import re

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "whole_line.npz")


def _line(g, i):
    return {k: g[f"{k}{i}"] for k in ("image", "boxes", "labels", "crops", "chars", "owner", "wc", "lq_w", "windows", "sr_samples",
                                      "sr_sum", "sr_u8")}


def test_whole_line_fixture_geometry():
    from marconet_b200 import pipeline
    from oracle import whole_line
    g = np.load(GOLDEN)
    wcs = []
    for i in range(int(g["lines"])):
        d = _line(g, i)
        h, w = d["image"].shape[:2]
        lq_w, wc = pipeline.whole_line_width(h, w)
        assert (lq_w, wc) == (int(d["lq_w"]), int(d["wc"])) == whole_line.whole_line_width(h, w)
        assert lq_w > 512 and wc % 4 == 0 and wc % 512 != 0 and wc - lq_w < 4
        segs = pipeline.plan_segments(h, w, d["boxes"].tolist(), labels=d["labels"].tolist())
        assert [list(s.crop) for s in segs] == d["crops"].tolist()
        assert [list(s.chars) for s in segs] == d["chars"].tolist()
        assert [k for k, s in enumerate(segs) for _ in range(*s.chars)] == d["owner"].tolist()
        wcs.append(wc)
    assert len(set(wcs)) == 2 and 1200 <= max(wcs) <= 1300 and 600 <= min(wcs) <= 800
    assert int(g["image0"].shape[0]) == 40 and 32 % int(g["image1"].shape[0]) != 0       # an integer and a non-integer LQ scale
    assert len(g["labels1"]) > 16                                                        # more characters than the encoder's 16


def test_oracle_reproduces_the_whole_line_fixture(checkpoints):
    """Encoder on the plan's crops, TSPGAN with each character's crop style, TSPSRNet on the whole line at Wc, all through the
    oracle (oracle/restate, oracle/image_ops, oracle/wide_line, oracle/whole_line): the fixture's bytes exactly, its fp32 samples and windows."""
    from marconet_b200 import pipeline
    from oracle import image_ops, restate, whole_line, wide_line
    g = np.load(GOLDEN)
    stride, (sy, sx) = int(g["stride"]), g["sample"].tolist()
    for i in range(int(g["lines"])):
        d = _line(g, i)
        img, boxes = d["image"], d["boxes"].tolist()
        h, w = img.shape[:2]
        styles = []
        for a, b in d["crops"].tolist():
            lq, _ = wide_line.preprocess_lq_crop(img, a, b)
            styles.append(restate.encoder_forward(checkpoints["encoder"], torch.from_numpy(lq))[2][:1])
        st = torch.cat([styles[k] for k in d["owner"].tolist()], dim=0)
        _, f64, f32_ = restate.tspgan_forward(checkpoints["tspgan"], st, torch.from_numpy(d["labels"]).reshape(-1, 1))
        lq, lq_w, wc = whole_line.preprocess_lq_whole_line(img)
        assert (lq_w, wc) == (int(d["lq_w"]), int(d["wc"]))
        locs = pipeline.boxes_to_locs(boxes, h, wc)
        sr, aux = restate.tspsr_forward(checkpoints["sr"], torch.from_numpy(lq), [f64], [f32_], locs, return_all=True)
        wins = [(32,) + r for r in aux["wins32"]] + [(64,) + r for r in aux["wins64"]]
        assert sorted(wins) == sorted(map(tuple, d["windows"].tolist()))
        np.testing.assert_allclose(sr[0, :, ::sy, ::sx].numpy(), d["sr_samples"], rtol=0, atol=1e-5)
        assert abs(sr.double().sum().item() - float(d["sr_sum"])) < 1e-2
        out = whole_line.whole_line_bytes(h, w, wc, image_ops.postprocess_sr(sr.numpy())[0])
        assert np.array_equal(out[::stride, ::stride], d["sr_u8"]), i


def _ragged_locs(g):
    from marconet_b200 import pipeline
    locs, counts, wcs = [], [], []
    for i in range(int(g["lines"])):
        d = _line(g, i)
        wc = int(d["wc"])
        locs.append(pipeline.boxes_to_locs(d["boxes"].tolist(), d["image"].shape[0], wc)[0])
        counts.append(len(d["boxes"]))
        wcs.append(wc)
    arr = np.zeros((len(locs), 2 * max(counts)), np.float32)
    for b, l in enumerate(locs):
        arr[b, :l.numel()] = l.numpy()
    return arr, counts, wcs


def test_host_ragged_windows_equal_the_reference_loop():
    """_char_windows_np on ONE ragged batch of both lines (canvas = the wider line) gives, per line, the window integers the
    unmodified reference loop computed on that line alone (sys.settrace, oracle/make_golden2.traced_sr)."""
    from marconet_b200.models.networks import _char_windows_np
    g = np.load(GOLDEN)
    arr, counts, wcs = _ragged_locs(g)
    canvas = max(wcs)
    for lvl, half, scale in ((32, 16, 1), (64, 32, 2)):
        wins, valid, owner = _char_windows_np(arr, counts, scale * canvas, half, line_w=[scale * v for v in wcs])
        o = 0
        for b, n in enumerate(counts):
            tr = g[f"windows{b}"]
            tr = tr[tr[:, 0] == lvl]
            assert tr.shape[0] == n
            got = wins[o:o + n]
            assert (got[:, 0] == b).all()
            assert np.array_equal(got[:, 1], tr[:, 3]) and np.array_equal(got[:, 2], tr[:, 4]) and np.array_equal(got[:, 3], tr[:, 5])
            assert np.array_equal(valid[o:o + n], tr[:, 4] - tr[:, 3])
            assert (owner[b, scale * wcs[b]:] == -1).all()
            o += n


def test_host_ragged_windows_adversarial_centres():
    """Centres at and around each line's own right edge: the host twin with per-line widths equals the reference arithmetic
    (oracle/restate.char_window, pinned to the reference loop) on each line at its own width, and raises where it would fail."""
    from marconet_b200.models.networks import _char_windows_np
    from oracle import restate
    rng = np.random.default_rng(7)
    widths = [512, 700, 1264, 2048]
    canvas = max(widths)
    for half in (16, 32):
        for _ in range(40):
            counts = [int(rng.integers(1, 30)) for _ in widths]
            arr = np.zeros((len(widths), 2 * max(counts)), np.float32)
            for b, (wb, n) in enumerate(zip(widths, counts)):
                cen = rng.choice([rng.uniform(0, 1), (wb - rng.integers(0, half + 2)) / wb, rng.uniform(0.98, 1.0)], size=n)
                arr[b, 0:2 * n:2] = cen.astype(np.float32)
            expect, empty = [], False
            for b, (wb, n) in enumerate(zip(widths, counts)):
                for c in range(n):
                    x1, x2, y1, _ = restate.char_window(torch.tensor(arr[b, 2 * c]), wb, half)
                    empty |= x2 - x1 <= 0 or x1 >= wb
                    expect.append((b, x1, x2, y1))
            if empty:
                with pytest.raises(RuntimeError, match="empty window"):
                    _char_windows_np(arr, counts, canvas, half, line_w=widths)
                continue
            wins, _, owner = _char_windows_np(arr, counts, canvas, half, line_w=widths)
            assert [tuple(r) for r in wins.tolist()] == expect
            for b, wb in enumerate(widths):
                assert (owner[b, wb:] == -1).all()


def test_ragged_kernel_symbols_match_the_header():
    from marconet_b200 import _lib
    header = open(os.path.join(ROOT, "include", "marconet_b200.h")).read()
    for name in ("mn_resample_modulate_ragged", "mn_char_windows_ragged"):
        decl = re.search(r"\bint " + name + r"\(([^;]*)\);", header)
        assert decl, name
        nargs = len([a for a in decl.group(1).split(",") if a.strip()])
        res, args = _lib.SYMBOLS[name]
        assert len(args) == nargs, (name, len(args), nargs)


def test_ragged_kernels_build_without_spills(tmp_path):
    """ptxas -v for sm_90a: both instantiations of the bilinear x2 kernel and the window kernel keep everything in registers."""
    import subprocess
    from marconet_b200 import build
    for src, kernels in (("generator_ops.cu", ("resample_up2_kernelILb1E", "resample_up2_kernelILb0E")),
                         ("sr_ops.cu", ("char_windows_kernel",))):
        path = os.path.join(ROOT, "marconet_b200", "csrc", src)
        r = subprocess.run([build.nvcc_path(), "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-DMN_BUILD", "-Xptxas", "-v",
                            "-cubin", path, "-o", str(tmp_path / (src + ".cubin"))], capture_output=True, text=True)
        assert r.returncode == 0, r.stderr[-2000:]
        for kernel in kernels:
            props = re.search(kernel + r"[^\n]*\n[^\n]*Function properties for [^\n]*" + kernel + r"[^\n]*\n([^\n]*)", r.stderr)
            assert props, f"no ptxas report for {kernel}"
            assert "0 bytes spill stores, 0 bytes spill loads" in props.group(1), props.group(1)


def test_recording_holds_its_width_table_past_cache_eviction(monkeypatch):
    """The bounded width-table cache of TSPSRNet may drop a table that a recorded graph's kernels still read: the recording keeps
    a reference of its own (the capture itself is stubbed here; the GPU test replays a real one)."""
    import gc
    import weakref
    from marconet_b200 import ops
    from marconet_b200.models import networks

    class _Graph:
        def replay(self):
            pass

    def fake_capture(sources, fn, fill):
        ent = networks._CapturedCall()
        ent.pinned = ent.h2d_done = ent.keep = None
        ent.graph, ent.inputs, ent.outputs, ent.flag = _Graph(), [None], (), None
        return ent

    monkeypatch.setattr(ops, "graphs_allowed", lambda: True)
    sr = networks.TSPSRNet()
    monkeypatch.setattr(sr, "_mg_capture", fake_capture)
    cpu = torch.device("cpu")
    table = sr._valid_widths((512, 700, 1264), cpu)
    ref = weakref.ref(table)
    for _ in range(2):                                    # eager on the first sighting, recorded on the second
        ent = sr._mg_run("k", [], None, fill=lambda st: None, keep=(table,))
    assert ent is not None and ent.keep[0] is table
    del table
    for k in range(70):
        sr._valid_widths((4 * (k + 1), 8), cpu)
    gc.collect()
    assert ((512, 700, 1264), cpu) not in sr._widths_cache         # the cache did drop it ...
    assert ref() is not None and ent.keep[0] is ref()               # ... the recording did not
    assert ref().tolist() == [[512, 700, 1264], [256, 350, 632], [128, 175, 316], [1024, 1400, 2528], [2048, 2800, 5056]]
    assert sr._mg_run("k", [], None, fill=lambda st: None) is ent   # replays keep the entry (and its table)
