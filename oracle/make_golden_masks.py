"""Pin oracle/mask_oracle.py against the reference and write tests/golden/mask_pipeline_vectors.npz.

Run in the BUILD container only (needs /root/reference):

    python oracle/make_golden_masks.py

Imports the reference's own functions - swap_head_mask_revisit_considerGlass (src/utils/swap_face_mask.py:33-83),
dilation / erosion (src/utils/morphology.py:23-197) - and runs the text of create_masks / swap_comp_style_vector
(scripts/face_swap.py:30-48, 117-146; the script module itself imports dlib-based alignment code that cannot be
imported here, so the two helper functions are exec'd from their source lines, unmodified).  Inputs: the
reference's example parsing masks (example/input/faceswap/{source,target}_mask.png converted 19 -> 12 classes,
already stored in reference_vectors.npz) plus seeded random label maps.  Every case asserts oracle == reference
EXACTLY and stores the REFERENCE outputs.
"""
from __future__ import annotations

import copy
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
REF = "/root/reference"
OUT = os.path.join(ROOT, "tests", "golden", "mask_pipeline_vectors.npz")
sys.path.insert(0, ROOT)

from oracle import golden_io  # noqa: E402
from oracle import mask_oracle as MO  # noqa: E402


def reference_functions():
    sys.path.insert(0, REF)
    from src.utils.swap_face_mask import swap_head_mask_revisit_considerGlass
    from src.utils.morphology import dilation, erosion
    lines = open(os.path.join(REF, "scripts", "face_swap.py")).read().split("\n")
    ns = {"copy": copy, "torch": torch, "dilation": dilation, "erosion": erosion}
    exec("\n".join(lines[29:48]), ns)           # def create_masks, scripts/face_swap.py:30-48
    exec("\n".join(lines[116:146]), ns)         # def swap_comp_style_vector, :117-146
    return swap_head_mask_revisit_considerGlass, dilation, erosion, ns["create_masks"], ns["swap_comp_style_vector"]


def synthetic_label_maps(seed: int, n: int, h: int, w: int):
    """Blocky random 12-class maps (every class present) - the tests regenerate them from the seed."""
    g = np.random.default_rng(seed)
    coarse = g.integers(0, 12, size=(n, max(1, h // 8), max(1, w // 8)))
    maps = np.kron(coarse, np.ones((8, 8), dtype=np.int64))[:, :h, :w]
    if maps.shape[1] < h or maps.shape[2] < w:
        maps = np.pad(maps, ((0, 0), (0, h - maps.shape[1]), (0, w - maps.shape[2])), mode="edge")
    noise = g.random(size=maps.shape) < 0.05
    maps = np.where(noise, g.integers(0, 12, size=maps.shape), maps)
    return maps.astype(np.uint8)


def main():
    swap_ref, dil_ref, ero_ref, create_ref, swap_sv_ref = reference_functions()
    base = golden_io.load(os.path.join(ROOT, "tests", "golden", "reference_vectors.npz"))
    src, tgt = base["mask/source_cls12"].astype(np.uint8), base["mask/target_cls12"].astype(np.uint8)
    gold = {}
    cases = {"example": (src, tgt), "example_rev": (tgt, src)}
    rnd = synthetic_label_maps(11, 4, 96, 72)
    cases["random_a"] = (rnd[0], rnd[1])
    cases["random_b"] = (rnd[2], rnd[3])
    for tag, (s, t) in cases.items():
        for hair_first in (True, False):
            r_res, r_hole = swap_ref(s.copy(), t.copy(), hair_first=hair_first)
            o_res, o_hole = MO.swap_head_mask(s, t, hair_first)
            assert np.array_equal(r_res, o_res) and np.array_equal(r_hole, o_hole), tag
            key = f"swap/{tag}/hair{int(hair_first)}"
            gold[key + "/res"], gold[key + "/hole"] = r_res.astype(np.uint8), r_hole.astype(np.uint8)
            print(f"  {key}: exact, {int((r_hole == 255).sum())} hole pixels, classes {sorted(set(r_res.ravel().tolist()))}")
        # foreground + blending masks exactly as scripts/face_swap.py:279-289 builds them
        res, hole = swap_ref(s.copy(), t.copy())
        swapped = torch.from_numpy(res.astype(np.int64))[None, None]
        mask_bg = torch.stack([swapped == c for c in [0, 11, 4]], dim=0).any(dim=0)       # logical_or_reduce, :50-51
        is_fg = torch.logical_not(mask_bg)
        is_fg[torch.from_numpy(hole == 255)[None][None]] = True
        fg = is_fg.float()
        assert np.array_equal(MO.foreground_mask(res, hole), fg[0, 0].numpy().astype(np.uint8)), tag
        gold[f"fg/{tag}"] = fg[0, 0].numpy().astype(np.uint8)
        for radius in (0, 1, 5):
            for op in ("dilation", "erosion", "expansion"):
                c_ref, b_ref, f_ref = create_ref(fg, outer_dilation=radius, operation=op)
                c_o, b_o, f_o = MO.create_masks(fg[0, 0].numpy().astype(np.uint8), radius, op)
                for name, a, b in (("content", c_ref, c_o), ("border", b_ref, b_o), ("full", f_ref, f_o)):
                    a = a[0, 0].numpy()
                    assert np.array_equal(a, a.round()) and np.array_equal(a.astype(np.uint8), b), (tag, radius, op, name)
                gold[f"masks/{tag}/r{radius}/{op}/border"] = b_ref[0, 0].numpy().astype(np.uint8)
                gold[f"masks/{tag}/r{radius}/{op}/full"] = f_ref[0, 0].numpy().astype(np.uint8)
        print(f"  masks/{tag}: dilation / erosion / expansion at r = 0, 1, 5 exact")
    # both engines of the reference agree on binary input (the oracle restates the arithmetic once)
    k = torch.ones(11, 11)
    x = torch.from_numpy(gold["fg/example"]).float()[None, None]
    assert torch.equal(dil_ref(x, k, engine="unfold"), dil_ref(x, k, engine="convolution"))
    assert torch.equal(ero_ref(x, k, engine="unfold"), ero_ref(x, k, engine="convolution"))
    # texture-vector swap
    g = torch.Generator().manual_seed(5)
    for tag, zero in (("plain", ()), ("no_ear", (7,)), ("no_teeth", (9,)), ("neither", (7, 9))):
        sv1, sv2 = torch.randn(1, 12, 64, generator=g), torch.randn(1, 12, 64, generator=g)
        for c in zero:
            sv2[:, c] = 0
        comp = sorted(set(range(12)) - {0, 4, 11, 10})                                   # scripts/face_swap.py:262
        for interp in (False, True):
            r = swap_sv_ref(sv1, sv2, comp, belowFace_interpolation=interp).numpy()
            o = MO.swap_comp_style_vector(sv1.numpy(), sv2.numpy(), comp, interp)
            assert np.array_equal(r, o), tag
            gold[f"stylevec/{tag}/interp{int(interp)}/sv1"] = sv1.numpy()
            gold[f"stylevec/{tag}/interp{int(interp)}/sv2"] = sv2.numpy()
            gold[f"stylevec/{tag}/interp{int(interp)}/out"] = r
    print("  stylevec: exact")
    np.savez_compressed(OUT, **gold)
    print(f"wrote {OUT}: {len(gold)} arrays, {os.path.getsize(OUT) / 1024:.0f} KiB")


if __name__ == "__main__":
    main()
