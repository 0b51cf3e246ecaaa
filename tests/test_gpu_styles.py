"""Font-style interpolation on the device (pipeline.interpolate_styles, mn_decode_labels, mn_style_lerp, mn_prior_tiles_u8;
DESIGN.md section 7b) against the PNGs of the unmodified test_w.py (script_w.npz), the reference modules on a wide content line
(style_wide.npz) and the numpy twins."""
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def _script_pair():
    from oracle.make_golden_script_w import input_arrays
    return tuple(np.ascontiguousarray(a[..., ::-1]) for a in input_arrays())     # the RGB arrays test_w.py holds


def _wide_pair():
    from oracle.make_golden_style_wide import inputs
    return inputs()


def _grey(a, b):
    return int(np.abs(np.asarray(a, np.int64) - np.asarray(b, np.int64)).max())


def test_script_parity(gpu_models):
    """test_w.py's two images: 17 labels (T = 64 collapses to more than 16) and the 11 strips within one grey level of the PNGs
    the script wrote."""
    from marconet_b200 import pipeline
    g = np.load(os.path.join(GOLDEN, "script_w.npz"))
    sy, sx = int(g["sy"]), int(g["sx"])
    res = pipeline.interpolate_styles(gpu_models["encoder"], gpu_models["tspgan"], [_script_pair()], to_host=True)[0]
    assert len(res["labels"]) == 17 == int(g["width"]) // 128 and len(res["windows"]) == 1
    assert isinstance(res["strips"], np.ndarray) and res["strips"].shape == (11, 128, 17 * 128, 3)
    assert max(_grey(res["strips"][i][::sy, ::sx], g[f"png{i}"]) for i in range(11)) <= 1


def test_wide_parity(gpu_models):
    """A content line three detection windows wide: labels equal predict_characters' and the fixture's; each strip within one grey
    level of the reference modules' PNG."""
    from marconet_b200 import pipeline
    g = np.load(os.path.join(GOLDEN, "style_wide.npz"))
    content, donor = _wide_pair()
    res = pipeline.interpolate_styles(gpu_models["encoder"], gpu_models["tspgan"], [(content, donor)], scales=g["scales"].tolist())[0]
    pred = pipeline.predict_characters(gpu_models["encoder"], [content])[0]
    assert res["labels"] == pred["labels"] == g["labels"].tolist()
    assert len(res["windows"]) == 3
    strips = res["strips"].cpu().numpy()
    sy, sx = int(g["sy"]), int(g["sx"])
    for k in range(len(g["scales"])):
        assert _grey(strips[k][::sy, ::sx], g["strips"][k]) <= 1, k


def test_decode_labels_kernel_equals_clear_labels():
    """mn_decode_labels against restate.clear_labels on planted logits (ties, NaNs, repeats, blanks, 64 distinct timesteps giving 64
    labels); its first 16 labels equal mn_decode_predictions' decoded labels on the same rows."""
    from marconet_b200 import ops
    from oracle import predict, restate
    dev = torch.device("cuda:0")
    logits = np.concatenate([predict.planted_image(seed, 32, 3000)[0] for seed in range(5)])
    distinct = np.random.default_rng(9).standard_normal((1, 64, 6736), dtype=np.float32)
    distinct[0, np.arange(64), np.arange(64) * 100 + 7] += 10.0
    logits = np.concatenate([logits, distinct])
    n = logits.shape[0]
    with torch.cuda.device(dev):
        lg = torch.from_numpy(logits).to(dev)
        out = torch.empty(n * ops.label_dtype().itemsize, dtype=torch.uint8, device=dev)
        ops.decode_labels(lg, out, 0)
        table, pout = ops.prediction_table([(0.0, 512.0, float("-inf"), float("inf"))] * n, dev)
        ops.decode_predictions(lg, torch.zeros(n, 32, device=dev), table, 0)
        rec = out.cpu().numpy().view(ops.label_dtype())
        prd = pout.cpu().numpy().view(ops.pred_dtype())
    for r in range(n):
        ref = restate.clear_labels(torch.from_numpy(logits[r]))
        m = int(rec[r]["n"])
        assert rec[r]["label"][:m].tolist() == ref and (rec[r]["label"][m:] == -1).all(), r
        assert prd[r]["label"][:int(prd[r]["n_kept"])].tolist() == ref[:16], r
    assert int(rec[-1]["n"]) == 64


def test_style_lerp_kernel_equals_torch():
    from marconet_b200 import ops
    dev = torch.device("cuda:0")
    g = torch.Generator().manual_seed(4)
    w = (torch.randn(7, 512, generator=g) * 3).to(dev)
    scales = [i / 10 for i in range(11)] + [float(v) for v in np.random.default_rng(4).uniform(-2, 3, 50)]
    rows = [(int(a), int(b), s) for s in scales for a, b in ((0, 6), (3, 1), (5, 5))]
    with torch.cuda.device(dev):
        out = ops.style_lerp(w, torch.frombuffer(bytearray(ops.lerp_rows(rows, 7)), dtype=torch.uint8).to(dev), len(rows))
    for r, (a, b, s) in enumerate(rows):
        assert torch.equal(out[r], w[a] * s + w[b] * (1 - s)), (r, s)


def test_prior_tiles_kernel_equals_numpy_strip(gpu_models):
    """The tiles of one generator call (channels_last output, read in place) equal oracle.styles.strip of the same priors."""
    from marconet_b200 import ops
    from oracle import styles
    dev = torch.device("cuda:0")
    g = torch.Generator().manual_seed(5)
    with torch.no_grad(), torch.cuda.device(dev):
        img, _, _ = gpu_models["tspgan"](styles=torch.randn(6, 512, generator=g).to(dev) * 2,
                                         labels=torch.randint(0, 6735, (6, 1), generator=g), noise=None)
        img = img * 1.5                                 # values beyond [-1, 1]: the saturation
        strips = torch.zeros((2, 128, 3 * 128, 3), dtype=torch.uint8, device=dev)
        tab = torch.frombuffer(bytearray(ops.prior_tile_rows([(strips[j // 3], j % 3) for j in range(6)])), dtype=torch.uint8).to(dev)
        ops.prior_tiles(img, tab, 0)
        torch.cuda.synchronize()
    p = img.cpu().numpy()
    for k in range(2):
        assert np.array_equal(strips[k].cpu().numpy(), styles.strip(p[3 * k:3 * k + 3])), k


def _mixed_pairs():
    script, wide = _script_pair(), _wide_pair()
    return [script, wide, (np.load(os.path.join(GOLDEN, "predict.npz"))["fit_image"], wide[1])]


@pytest.mark.parametrize("max_chars", [1, 7, 128])
def test_batched_pairs_match_single_pair_calls(gpu_models, max_chars):
    """Fitting and wide content in one call at max_chars 1, 7 and 128 match each pair's own call within one grey level, and bit
    for bit with the same chunking (max_chars 1 and max_lines 1 on both sides)."""
    from marconet_b200 import pipeline
    enc, gen = gpu_models["encoder"], gpu_models["tspgan"]
    pairs, scales = _mixed_pairs(), (0.0, 0.45, 1.0)
    same = max_chars == 1                               # identical chunking: one encoder row and one character per launch
    both = pipeline.interpolate_styles(enc, gen, pairs, scales=scales, max_chars=max_chars, max_lines=1 if same else 3, to_host=True)
    for p, pair in enumerate(pairs):
        one = pipeline.interpolate_styles(enc, gen, [pair], scales=scales, max_chars=1 if same else 128, max_lines=1 if same else 8,
                                          to_host=True)[0]
        assert both[p]["labels"] == one["labels"] and both[p]["strips"].shape == one["strips"].shape, p
        if same:
            assert np.array_equal(both[p]["strips"], one["strips"]), p
        else:
            assert _grey(both[p]["strips"], one["strips"]) <= 1, p


def test_no_character_content_is_an_invalid_pair(gpu_models):
    """A content line the encoder reads no character on raises naming the pair, or becomes an error entry with skip_invalid."""
    from marconet_b200 import pipeline

    class Blank(torch.nn.Module):
        def __init__(self, enc):
            super().__init__()
            self.enc = enc

        def forward(self, lq):
            lg, lr, w = self.enc(lq)
            lg = torch.zeros_like(lg)
            lg[:, :, 6735] = 1.0
            return lg, lr, w

    enc = Blank(gpu_models["encoder"])
    pairs = _mixed_pairs()[:2]
    with pytest.raises(ValueError, match="pair 0: no character"):
        pipeline.interpolate_styles(enc, gpu_models["tspgan"], pairs[:1])
    out = pipeline.interpolate_styles(enc, gpu_models["tspgan"], pairs, skip_invalid=True)
    assert all(set(r) == {"error"} and "no character" in r["error"] for r in out)


def test_launches_syncs_and_no_module_graphs(gpu_models, monkeypatch):
    """ops.LAUNCHES per call is the stage plan's: per encoder batch one crop launch, the encoder and one decode launch per row kind
    present; one lerp launch; per chunk the generator (eager) and one tile launch.  The generator's module-graph cache gains no
    entry across calls with different totals."""
    from marconet_b200 import ops, pipeline
    enc, gen = gpu_models["encoder"], gpu_models["tspgan"]
    dev = torch.device("cuda:0")
    pairs, scales = _mixed_pairs(), (0.0, 1.0)
    pipeline.interpolate_styles(enc, gen, pairs, scales=scales, max_chars=40, max_lines=4)        # warm-up: encoder batches
    res = pipeline.interpolate_styles(enc, gen, pairs, scales=scales, max_chars=40, max_lines=4)
    n_rows = sum(len(r["windows"]) + 1 for r in res)
    kinds = ["fit"] * 2 + ["wide"] * 3 + ["donor"] * 3                   # pairs 0 and 2 fit, pair 1 is three windows wide
    assert n_rows == len(kinds)
    batches = [kinds[r0:r0 + 4] for r0 in range(0, n_rows, 4)]
    total = sum(len(r["labels"]) for r in res) * len(scales)
    chunks = [min(40, total - r0) for r0 in range(0, total, 40)]
    per_enc, per_gen = {}, {}
    flag = torch.zeros(1, dtype=torch.int32, device=dev)
    with torch.no_grad():
        for b in {len(bt) for bt in batches}:
            l0 = ops.LAUNCHES
            enc(torch.zeros(b, 3, 32, 512, device=dev))
            per_enc[b] = ops.LAUNCHES - l0
        for c in set(chunks):
            l0 = ops.LAUNCHES
            with ops.deferred_checks(flag):
                gen(styles=torch.zeros(c, 512, device=dev), labels=torch.zeros(c, 1, dtype=torch.long, device=dev), noise=None)
            per_gen[c] = ops.LAUNCHES - l0
    want = sum(1 + per_enc[len(bt)] + ("fit" in bt) + ("wide" in bt) for bt in batches) + 1 + sum(per_gen[c] + 1 for c in chunks)
    mg = dict(gen.TextGenerator._mg or {})
    hits = dict(gen.TextGenerator._mg_hits)
    syncs = []
    real_sync = torch.cuda.Stream.synchronize
    monkeypatch.setattr(torch.cuda.Stream, "synchronize", lambda self: (syncs.append(1), real_sync(self))[1])
    l0 = ops.LAUNCHES
    pipeline.interpolate_styles(enc, gen, pairs, scales=scales, max_chars=40, max_lines=4)
    assert ops.LAUNCHES - l0 == want
    assert len(syncs) == 1                                               # the read stage's copy back
    monkeypatch.undo()
    for sc, mc in (((0.0, 0.2, 1.0), 40), ((0.5,), 33), ((0.1, 0.9), 7)):
        out = pipeline.interpolate_styles(enc, gen, pairs[:2], scales=sc, max_chars=mc, to_host=True)
        assert all(isinstance(r["strips"], np.ndarray) for r in out)
    assert dict(gen.TextGenerator._mg or {}) == mg and dict(gen.TextGenerator._mg_hits) == hits
