"""Pin oracle/gpen_oracle.py against the reference's GPEN and write tests/golden/gpen_vectors.npz.

Run in the BUILD container only (needs /root/reference):

    python oracle/make_golden_gpen.py

The reference model (src/pretrained/gpen/face_model/gpen_model.py) runs on the CPU as shipped - its ops carry their
own CPU branches (op/fused_act.py:96, op/upfirdn2d.py:160-194) - so it is imported UNMODIFIED (only
torch.utils.cpp_extension.load is stubbed: the CUDA extensions cannot be JIT-built without a GPU), loaded with the seeded
synthetic state and run; the script asserts oracle == reference to fp32 rounding and stores the REFERENCE outputs.
"""
from __future__ import annotations

import os
import sys
import types

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
REF = "/root/reference"
OUT = os.path.join(ROOT, "tests", "golden", "gpen_vectors.npz")
sys.path.insert(0, ROOT)

from oracle import golden_io  # noqa: E402
from oracle import gpen_oracle as GO  # noqa: E402

TOL = 2e-5
CASES = [("g64", 64, 2, 7), ("g128", 128, 1, 8), ("g256", 256, 1, 9)]        # tag, size, batch, seed


def case_input(size: int, batch: int, seed: int) -> torch.Tensor:
    g = torch.Generator().manual_seed(seed)
    return torch.randn(batch, 3, size, size, generator=g)


def main():
    import torch.utils.cpp_extension as cpp
    cpp.load = lambda *a, **k: types.SimpleNamespace()
    sys.path.insert(0, REF)
    import src.pretrained.gpen.face_model.gpen_model as GM
    torch.set_grad_enabled(False)
    gold = {}
    for tag, size, batch, seed in CASES:
        model = GM.FullGenerator(size, 512, 8, channel_multiplier=2, narrow=1, device="cpu").eval()
        ref_shapes = {k: tuple(v.shape) for k, v in model.state_dict().items()}
        assert ref_shapes == GO.param_shapes(size), "oracle/gpen_oracle.py:param_shapes disagrees with the reference state_dict"
        st = GO.synthetic_state(size, salt=size)
        model.load_state_dict(st)
        x = case_input(size, batch, seed)
        ref, none = model(x)
        assert none is None
        ora = GO.full_generator_forward(st, x, size)
        e = float((ora - ref).abs().max() / ref.abs().max())
        print(f"  gpen/{tag}: ref-vs-oracle max-rel {e:.2e}  shape {tuple(ref.shape)}  |ref|max {float(ref.abs().max()):.3f}")
        assert e <= TOL, e
        # the encoder stack alone (its outputs are the generator's concatenated "noise")
        feats_ref, h = [], x
        for i in range(model.log_size - 1):
            h = getattr(model, model.names[i])(h)
            feats_ref.append(h)
        for i, (a, b) in enumerate(zip(feats_ref, GO.encode(st, x, size))):
            ee = float((a - b).abs().max() / a.abs().max())
            assert ee <= TOL, (i, ee)
        gold[f"gpen/{tag}/image"] = ref.numpy()
        gold[f"gpen/{tag}/ecd_last"] = feats_ref[-1].numpy()
        gold[f"gpen/{tag}/ecd1_sub"] = feats_ref[1][:, ::8, ::2, ::2].numpy()
    paths = golden_io.save(OUT, gold)
    print(f"wrote {len(gold)} arrays -> " + ", ".join(f"{p} ({os.path.getsize(p) / 1024:.0f} KiB)" for p in paths))


if __name__ == "__main__":
    main()
