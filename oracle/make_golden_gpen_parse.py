"""Pin oracle/gpen_parse_oracle.py against the reference's GPEN face parser and write tests/golden/gpen_parse_vectors.npz and
tests/golden/gpen_parse_checkpoint_layout.json.

Run in the BUILD container only (needs /root/reference):

    python oracle/make_golden_gpen_parse.py

The reference modules src/pretrained/gpen/face_parse/{blocks,parse_model,face_parsing}.py are imported UNMODIFIED.  The
seeded stand-in checkpoint (oracle/gpen_parse_oracle.py:synthetic_state) is written as <tmp>/weights/ParseNet-latest.pth, and
FaceParse(tmp, device="cpu") loads it with strict=True.  The network then runs on two seeded structured 512 x 512 uint8
images through process() and process_tensor(), and process_tensor() also on a 600 x 560 image (its nearest resize); the
script asserts that the oracle agrees with the reference (logits and out_img to 2e-5 relative, masks equal), that the stand-in
spreads the argmax (>= 5 classes at >= 1 % of the pixels, both mask values at >= 5 %), and stores the REFERENCE outputs:
logits and out_img sub-sampled every 8th pixel, the full 19-class labels and both masks.
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
OUT = os.path.join(ROOT, "tests", "golden", "gpen_parse_vectors.npz")
LAYOUT = os.path.join(ROOT, "tests", "golden", "gpen_parse_checkpoint_layout.json")
sys.path.insert(0, ROOT)

from oracle import golden_io  # noqa: E402
from oracle import gpen_parse_oracle as PO  # noqa: E402

TOL = 2e-5
SUB = 8                                                     # logits / out_img stored at every 8th pixel
CASES = [("a", 512, 512, 11), ("b", 512, 512, 12)]          # tag, height, width, seed
RESIZE_CASE = ("r600x560", 600, 560, 13)                    # process_tensor only


def main():
    sys.path.insert(0, REF)
    import src.pretrained.gpen.face_parse.face_parsing as FP
    torch.set_grad_enabled(False)
    st = PO.synthetic_state()
    gold = {}
    with tempfile.TemporaryDirectory() as tmp:
        os.makedirs(os.path.join(tmp, "weights"))
        torch.save(st, os.path.join(tmp, "weights", "ParseNet-latest.pth"))
        fp = FP.FaceParse(tmp, device="cpu")
    layout = {k: list(v.shape) for k, v in fp.faceparse.state_dict().items()}
    assert layout == {k: list(v) for k, v in PO.param_shapes().items()}, "param_shapes disagrees with the reference"
    for tag, h, w, seed in CASES:
        img = PO.case_image(h, w, seed)
        x = PO.process_input(img)
        branch = []
        lg_ref, im_ref = fp.faceparse(x)
        lg_ora, im_ora = PO.parsenet_forward(st, x, branch)
        e_lg = float((lg_ora - lg_ref).abs().max() / lg_ref.abs().max())
        e_im = float((im_ora - im_ref).abs().max() / im_ref.abs().max())
        m_ref, m_ora = fp.process(img), PO.process(st, img)
        same = len(m_ref) == 1 and m_ref[0].dtype == np.uint8 and np.array_equal(m_ref[0], m_ora[0])
        imt = PO.image_tensor(img)
        t_ref, t_ora = fp.process_tensor(imt), PO.process_tensor(st, imt)
        same_t = t_ref.dtype == torch.int64 and tuple(t_ref.shape) == (1, 1, 512, 512) and torch.equal(t_ref, t_ora)
        labels = lg_ref.argmax(1)[0]
        frac = torch.bincount(labels.flatten(), minlength=PO.NCLS).double() / labels.numel()
        zero = float((torch.from_numpy(m_ref[0]) == 0).double().mean())
        print(f"  parse/{tag}: logits max-rel {e_lg:.2e}, out_img max-rel {e_im:.2e}, process masks equal {same}, "
              f"process_tensor masks equal {same_t}; classes at >= 1 %: {int((frac >= 0.01).sum())} "
              f"({', '.join(f'{k}: {f:.1%}' for k, f in enumerate(frac.tolist()) if f >= 0.01)}), mask 0 / 255: "
              f"{zero:.1%} / {1 - zero:.1%}; ||branch|| / ||identity|| {min(branch):.2f} .. {max(branch):.2f} "
              f"(median {float(np.median(branch)):.2f}) over {len(branch)} blocks")
        assert e_lg <= TOL and e_im <= TOL and same and same_t, (tag, e_lg, e_im, same, same_t)
        assert int((frac >= 0.01).sum()) >= 5 and 0.05 <= zero <= 0.95, (tag, frac, zero)
        gold[f"parse/{tag}/logits_sub"] = lg_ref[0, :, ::SUB, ::SUB].numpy()
        gold[f"parse/{tag}/img_sub"] = im_ref[0, :, ::SUB, ::SUB].numpy()
        gold[f"parse/{tag}/labels"] = labels.to(torch.uint8).numpy()
        gold[f"parse/{tag}/mask"] = m_ref[0]
        gold[f"parse/{tag}/mask_tensor"] = t_ref[0, 0].to(torch.uint8).numpy()
    tag, h, w, seed = RESIZE_CASE
    imt = PO.image_tensor(PO.case_image(h, w, seed))
    t_ref, t_ora = fp.process_tensor(imt), PO.process_tensor(st, imt)
    assert torch.equal(t_ref, t_ora), tag
    print(f"  parse/{tag}: process_tensor masks equal True, mask 0: {float((t_ref == 0).double().mean()):.1%}")
    gold[f"parse/{tag}/mask_tensor"] = t_ref[0, 0].to(torch.uint8).numpy()
    paths = golden_io.save(OUT, gold)
    with open(LAYOUT, "w") as f:
        json.dump(layout, f, indent=0, sort_keys=True)
        f.write("\n")
    print(f"wrote {len(gold)} arrays -> " + ", ".join(f"{p} ({os.path.getsize(p) / 1024:.0f} KiB)" for p in paths) +
          f"; {len(layout)} state-dict entries -> {LAYOUT}")


if __name__ == "__main__":
    main()
