"""Pin oracle/retinaface_oracle.py against the reference's GPEN RetinaFace-R50 detector and write
tests/golden/retinaface_vectors.npz and tests/golden/retinaface_checkpoint_layout.json.

Run in the BUILD container only (needs the reference checkout and torchvision):

    python oracle/make_golden_retinaface.py

The reference modules retinaface_detection.py, facemodels/{retinaface,net}.py, data/config.py,
layers/functions/prior_box.py and utils/{box_utils,nms/py_cpu_nms}.py are imported UNMODIFIED.  The seeded stand-in
checkpoint is written as <tmp>/weights/RetinaFace-R50.pth with a ``module.`` prefix and RetinaFaceDetection(tmp, 'cpu') loads
it (strict=False in the reference, so the script asserts that every key loaded).  On seeded structured images of 256 x 256
and 192 x 320 (and 200 x 180, reference side only) the script asserts oracle == reference (module outputs to 2e-5, decode
exact, detections equal), prints the detection statistics of the stand-in, and stores the reference's module outputs
sub-sampled, the full detections and landmarks.
"""
from __future__ import annotations

import json
import os
import sys
import tempfile

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
REF = "/root/reference"
OUT = os.path.join(ROOT, "tests", "golden", "retinaface_vectors.npz")
LAYOUT = os.path.join(ROOT, "tests", "golden", "retinaface_checkpoint_layout.json")
sys.path.insert(0, ROOT)

from oracle import golden_io  # noqa: E402
from oracle import retinaface_oracle as RO  # noqa: E402

TOL = 2e-5
SUB = 7                                                     # module outputs stored at every 7th prior
CASES = [("a", 256, 256, 21), ("b", 192, 320, 22)]          # tag, height, width, seed
REF_ONLY = ("c", 200, 180, 23)                              # not a multiple of 32: the reference side only
BINDING = ("a", dict(top_k=40, keep_top_k=3))               # a case where top_k and keep_top_k bind


def main():
    sys.path.insert(0, REF)
    import src.pretrained.gpen.face_detect.retinaface_detection as RD
    from src.pretrained.gpen.face_detect.layers.functions.prior_box import PriorBox
    from src.pretrained.gpen.face_detect.utils.box_utils import decode, decode_landm
    from src.pretrained.gpen.face_detect.utils.nms.py_cpu_nms import py_cpu_nms
    torch.set_grad_enabled(False)
    st = RO.synthetic_state()
    gold = {}
    with tempfile.TemporaryDirectory() as tmp:
        os.makedirs(os.path.join(tmp, "weights"))
        torch.save({"module." + k: v for k, v in st.items()}, os.path.join(tmp, "weights", "RetinaFace-R50.pth"))
        det = RD.RetinaFaceDetection(tmp, device="cpu")
    sd = det.net.state_dict()
    assert set(sd) == set(st) and all(torch.equal(sd[k], st[k]) for k in st), "the stand-in did not load completely"
    layout = {k: list(v.shape) for k, v in sd.items()}
    for tag, h, w, seed in CASES + [REF_ONLY]:
        img = RO.case_image(h, w, seed)
        xf = np.float32(img)
        xf -= (104, 117, 123)
        x = torch.from_numpy(xf.transpose(2, 0, 1).copy()).unsqueeze(0)
        loc, conf, landms = det.net(x)
        dets, lms = det.detect(img)
        priors = PriorBox(det.cfg, image_size=(h, w)).forward()
        assert torch.equal(priors, RO.prior_box(h, w)), tag
        assert torch.equal(decode(loc[0], priors, det.cfg["variance"]), RO.decode(loc[0], priors)), tag
        assert torch.equal(decode_landm(landms[0], priors, det.cfg["variance"]), RO.decode_landm(landms[0], priors)), tag
        scores = conf[0, :, 1].numpy()
        above = int((scores > 0.9).sum())
        print(f"  retina/{tag} {h}x{w}: {scores.size} priors, {above} ({above / scores.size:.2%}) above 0.9, "
              f"{len(dets)} kept after NMS", end="")
        if (tag, h, w, seed) == REF_ONLY:
            print(" (reference only)")
            continue
        branch = []
        o_loc, o_conf, o_lm = RO.forward(st, x, branch)
        errs = [float((a - b).abs().max() / b.abs().max()) for a, b in ((o_loc, loc), (o_conf, conf), (o_lm, landms))]
        o_dets, o_lms = RO.detect(st, img)
        same = o_dets.shape == dets.shape and np.array_equal(o_dets, dets) and np.array_equal(o_lms, lms)
        print(f"; oracle max-rel loc {errs[0]:.1e} conf {errs[1]:.1e} landms {errs[2]:.1e}, detections equal {same}; "
              f"||branch|| / ||identity|| {min(branch):.2f} .. {max(branch):.2f} (median {float(np.median(branch)):.2f})")
        assert max(errs) <= TOL and same, (tag, errs, same)
        assert len(dets) < above / 2, "NMS should suppress most of the stand-in's candidates"
        # the margin the GPU tests need: no score near the threshold
        gap = float(np.abs(scores - np.float32(0.9)).min())
        print(f"    closest score to 0.9: {gap:.2e}")
        gold[f"retina/{tag}/loc_sub"] = loc[0, ::SUB].numpy()
        gold[f"retina/{tag}/conf_sub"] = conf[0, ::SUB].numpy()
        gold[f"retina/{tag}/landms_sub"] = landms[0, ::SUB].numpy()
        gold[f"retina/{tag}/dets"] = dets
        gold[f"retina/{tag}/landms"] = lms
    tag, kw = BINDING
    h, w, seed = next((c[1], c[2], c[3]) for c in CASES if c[0] == tag)
    img = RO.case_image(h, w, seed)
    dets, lms = det.detect(img, **kw)
    o_dets, o_lms = RO.detect(st, img, **kw)
    assert np.array_equal(dets, o_dets) and np.array_equal(lms, o_lms) and len(dets) == kw["keep_top_k"], BINDING
    print(f"  retina/{tag} with {kw}: {len(dets)} kept, equal True")
    gold[f"retina/{tag}/dets_bound"] = dets
    gold[f"retina/{tag}/landms_bound"] = lms
    # the oracle's NMS is py_cpu_nms on tie-free input
    g = np.random.default_rng(5)
    xy = g.uniform(0, 200, (300, 2)).astype(np.float32)
    d = np.hstack([xy, xy + g.uniform(5, 60, (300, 2)).astype(np.float32), g.permutation(300)[:, None].astype(np.float32)])
    assert py_cpu_nms(d, 0.4) == RO.nms(d, 0.4)
    paths = golden_io.save(OUT, gold)
    with open(LAYOUT, "w") as f:
        json.dump(layout, f, indent=0, sort_keys=True)
        f.write("\n")
    print(f"wrote {len(gold)} arrays -> " + ", ".join(f"{p} ({os.path.getsize(p) / 1024:.0f} KiB)" for p in paths) +
          f"; {len(layout)} state-dict entries -> {LAYOUT}")


if __name__ == "__main__":
    main()
