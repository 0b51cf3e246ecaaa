"""Generates tests/golden/style_wide.npz: test_w.py's font-style interpolation (:95-114) for a content line wider than the
canvas, computed with the reference's UNMODIFIED modules (oracle/ref_harness.py, synthetic checkpoints seed 0) on the CPU.

  content  predict.npz's 40 x 1757 line (three detection windows, every logit margin >= 5e-3);
  donor    script_w's second image, as test_w.py holds it after cv2.cvtColor (the RGB array of w2.png);
  scales   (0.0, 0.3, 1.0).

Every window is cut by hand and encoded as test_w.py encodes an image (real cv2 cubic resize, IPP off; zero canvas; ToTensor /
Normalize).  Window k keeps the characters oracle/predict.py keeps (its decode and core test on the reference logits) and takes
the style w_k; per scale s its images are TSPGAN((w_k*s + w2*(1-s)).repeat(n_k, 1), labels_k), and the strip holds them in merged
(centre-sorted) order, 8-bit as cv2.imwrite(prior128 * 255.0) stores it (encoded and decoded by real cv2).  Stored: the merged
labels and owning windows, the reference's w rows and styles, samples of the priors ([::PY, ::PX]) and of the strips ([::SY, ::SX]).

Needs a reference checkout (MARCONET_REFERENCE=<path>):  python -m oracle.make_golden_style_wide
TEST INFRASTRUCTURE ONLY.
"""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OUT = os.path.join(ROOT, "tests", "golden", "style_wide.npz")
SCALES = (0.0, 0.3, 1.0)
SY, SX = 8, 16          # strip samples
PY, PX = 16, 32         # prior samples (a sub-grid of the strip samples)


def inputs():
    """(content, donor) uint8 [h, w, 3] arrays as interpolate_styles takes them."""
    from oracle.make_golden_script_w import input_arrays
    content = np.load(os.path.join(ROOT, "tests", "golden", "predict.npz"))["wide_image"]
    return content, np.ascontiguousarray(input_arrays()[1][..., ::-1])


def main():
    import cv2
    sys.path.insert(0, ROOT)
    cv2.ipp.setUseIPP(False)
    from marconet_b200.testing import synth
    from oracle import predict, ref_harness, styles
    from oracle.make_golden_predict import encode_crop
    torch.set_num_threads(os.cpu_count() or 1)
    models = ref_harness.build_reference_models(synth.make_checkpoints(0))
    enc, gen = models["encoder"], models["tspgan"]
    content, donor = inputs()
    h, w = content.shape[:2]
    g = np.load(os.path.join(ROOT, "tests", "golden", "predict.npz"))
    wins = predict.plan_windows(h, w)
    rows, w_rows = [], []
    with torch.no_grad():
        for k, ((a, b), (lo, hi)) in enumerate(wins):
            logits, locs, wk = enc(encode_crop(np.ascontiguousarray(content[:, a:b])))
            assert np.array_equal(logits[0].argmax(1).numpy(), g["wide_argmax"][k])
            rows.append(predict.decode_row(logits[0].numpy(), locs[0].numpy(), a, 16.0 * h, lo, hi)[:3])
            w_rows.append(wk)
        _, _, w2 = enc(encode_crop(donor))
        labels, owners = styles.merge_with_windows(h, w, rows)
        assert labels == g["wide_labels"].tolist()
        rec = dict(scales=np.asarray(SCALES), labels=np.asarray(labels, np.int64), owners=np.asarray(owners, np.int64),
                   w_rows=torch.cat(w_rows + [w2]).numpy(), sy=np.array(SY), sx=np.array(SX), py=np.array(PY), px=np.array(PX))
        st, pr, sp = [], [], []
        for s in SCALES:
            per_win, st_s = [], []
            for k, (labs, _, _) in enumerate(rows):
                new_w = w_rows[k] * s + w2 * (1 - s)
                st_s.append(new_w[0].numpy())
                if not labs:
                    per_win.append(np.zeros((0, 3, 128, 128), np.float32))
                    continue
                prior, _, _ = gen(styles=new_w.repeat(len(labs), 1), labels=torch.tensor(labs, dtype=torch.long).unsqueeze(1), noise=None)
                per_win.append(prior.numpy())
                print("scale", s, "window", k, "chars", len(labs), flush=True)
            merged = np.stack([per_win[k][j] for k, j in owners])
            row = np.hstack(list((torch.from_numpy(merged) * 0.5 + 0.5).permute(0, 2, 3, 1).numpy()))
            ok, enc_png = cv2.imencode(".png", row * 255.0)
            assert ok
            png = cv2.imdecode(enc_png, cv2.IMREAD_COLOR)
            assert png.shape == (128, 128 * len(labels), 3)
            st.append(np.stack(st_s))
            pr.append(merged[:, :, ::PY, ::PX])
            sp.append(png[::SY, ::SX])
        rec.update(styles=np.stack(st).astype(np.float32), priors=np.stack(pr).astype(np.float32), strips=np.stack(sp))
    np.savez_compressed(OUT, **rec)
    print("wrote", OUT, "chars", len(labels), os.path.getsize(OUT))


if __name__ == "__main__":
    main()
