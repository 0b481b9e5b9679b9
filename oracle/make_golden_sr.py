"""Pin oracle/sr_oracle.py against the reference's RealESRNet x4 and write tests/golden/sr_vectors.npz and
tests/golden/sr_checkpoint_layout.json.

Run in the BUILD container only (needs /root/reference):

    python oracle/make_golden_sr.py

The reference modules src/pretrained/gpen/sr_model/{arch_util,rrdbnet_arch,real_esrnet}.py are imported UNMODIFIED.  The
seeded stand-in checkpoint (oracle/sr_oracle.py:synthetic_state) is written as <tmp>/weights/realesrnet_x4.pth under
"params_ema", and RealESRNet(tmp, "realesrnet", 4, device="cpu") loads it with strict=True.  The full 23-block network then
runs on seeded uint8 images (a square one and a non-square one whose sides are not multiples of the 8 x 16 pixel tile);
the script asserts that the oracle agrees with the reference (forward to 2e-5 relative, process() bytes equal) and stores
the REFERENCE outputs.
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
OUT = os.path.join(ROOT, "tests", "golden", "sr_vectors.npz")
LAYOUT = os.path.join(ROOT, "tests", "golden", "sr_checkpoint_layout.json")
sys.path.insert(0, ROOT)

from oracle import golden_io  # noqa: E402
from oracle import sr_oracle as SO  # noqa: E402

TOL = 2e-5
CASES = [("s32", 32, 32, 21), ("s20x44", 20, 44, 22)]     # tag, height, width, seed


def main():
    sys.path.insert(0, REF)
    import src.pretrained.gpen.sr_model.real_esrnet as RE
    torch.set_grad_enabled(False)
    st = SO.synthetic_state()
    gold = {}
    with tempfile.TemporaryDirectory() as tmp:
        os.makedirs(os.path.join(tmp, "weights"))
        torch.save({"params_ema": st}, os.path.join(tmp, "weights", "realesrnet_x4.pth"))
        sr = RE.RealESRNet(tmp, "realesrnet", 4, device="cpu")
    layout = {k: list(v.shape) for k, v in sr.srmodel.state_dict().items()}
    assert layout == {k: list(v) for k, v in SO.param_shapes().items()}, "sr_oracle.param_shapes disagrees with the reference"
    for tag, h, w, seed in CASES:
        img = SO.case_image(h, w, seed)
        x = SO.to_input(img)
        ref = sr.srmodel(x)
        ora = SO.rrdbnet_forward(st, x)
        e = float((ora - ref).abs().max() / ref.abs().max())
        out_ref = sr.process(img)
        out_ora = SO.process(st, img)
        same = out_ref is not None and out_ref.dtype == np.uint8 and np.array_equal(out_ref, out_ora)
        print(f"  sr/{tag}: forward max-rel {e:.2e}, process bytes equal {same}; output {tuple(ref.shape)}, "
              f"{float(((ref >= 0) & (ref <= 1)).double().mean()):.1%} inside [0, 1]")
        assert e <= TOL and same, (tag, e, same)
        assert out_ref.shape == (4 * h, 4 * w, 3)
        gold[f"sr/{tag}/image"] = img
        gold[f"sr/{tag}/forward"] = ref.numpy()
        gold[f"sr/{tag}/process"] = out_ref
    paths = golden_io.save(OUT, gold)
    with open(LAYOUT, "w") as f:
        json.dump(layout, f, indent=0, sort_keys=True)
        f.write("\n")
    print(f"wrote {len(gold)} arrays -> " + ", ".join(f"{p} ({os.path.getsize(p) / 1024:.0f} KiB)" for p in paths) +
          f"; {len(layout)} state-dict entries -> {LAYOUT}")


if __name__ == "__main__":
    main()
