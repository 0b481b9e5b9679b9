"""Pin oracle/parser_oracle.py against the reference's BiSeNet face parser and write tests/golden/parser_vectors.npz.

Run in the BUILD container only (needs /root/reference):

    python oracle/make_golden_parser.py

The reference modules (src/pretrained/face_parsing/{resnet,model,face_parsing_demo}.py, src/datasets/dataset.py) are
imported UNMODIFIED.  Three things are stubbed around them, none of which changes what they compute:
  * torch.utils.model_zoo.load_url returns {} (Resnet18's constructor would fetch ImageNet weights, which the checkpoint load
    overwrites anyway) and torch.hub.load_state_dict_from_url raises: nothing reaches the network;
  * torch.Tensor.cuda is the identity while model.py is imported (its seg_mean / seg_std are moved to the GPU at import);
  * FaceParser runs with device="cpu" on a seeded checkpoint written to a temporary file, its BicubicDownSample filters
    as CPU tensors (downsample.cuda = "").
faceParsing_demo then runs end to end on seeded uint8 images; the script asserts that the oracle agrees with the reference
(logits and preprocess output to 2e-5 relative, labels exactly, state-dict layout equal) and stores the REFERENCE outputs.
"""
from __future__ import annotations

import os
import sys
import tempfile

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
REF = "/root/reference"
OUT = os.path.join(ROOT, "tests", "golden", "parser_vectors.npz")
sys.path.insert(0, ROOT)

from oracle import golden_io  # noqa: E402
from oracle import parser_oracle as PO  # noqa: E402

TOL = 2e-5
CASES = [("p1024", 1024, 11), ("p768", 768, 12)]        # tag, image side, seed (one image each)
SUB = 16                                                # stored logits: every SUB-th row and column


def _import_reference():
    import torch.hub
    import torch.utils.model_zoo as model_zoo

    def no_network(*a, **k):
        raise RuntimeError("make_golden_parser: a reference module tried to download weights")

    model_zoo.load_url = lambda *a, **k: {}
    torch.hub.load_state_dict_from_url = no_network
    sys.path.insert(0, REF)
    cuda = torch.Tensor.cuda
    torch.Tensor.cuda = lambda self, *a, **k: self
    try:
        import src.pretrained.face_parsing.model as BM
        import src.pretrained.face_parsing.face_parsing_demo as FD
        import src.datasets.dataset as D
    finally:
        torch.Tensor.cuda = cuda
    return BM, FD, D


def rel(a, b):
    return float((a - b).abs().max() / b.abs().max())


def main():
    from PIL import Image
    import torchvision
    BM, FD, D = _import_reference()
    torch.set_grad_enabled(False)
    ref_shapes = {k: tuple(v.shape) for k, v in BM.BiSeNet(n_classes=19).state_dict().items()}
    assert ref_shapes == PO.param_shapes(), "oracle/parser_oracle.py:param_shapes disagrees with the reference state_dict"
    st = PO.synthetic_state()
    gold = {}
    with tempfile.TemporaryDirectory() as tmp:
        ckpt = os.path.join(tmp, "bisenet_synthetic.pth")
        torch.save(st, ckpt)
        parser = FD.FaceParser(ckpt, size=1024, device="cpu")
        parser.downsample.cuda = ""
        parser.downsample_256.cuda = ""
        for tag, size, seed in CASES:
            img = PO.case_image(size, seed)
            pil = Image.fromarray(img)
            seg12 = FD.faceParsing_demo(parser, pil, convert_to_seg12=True)
            seg19 = FD.faceParsing_demo(parser, pil, convert_to_seg12=False)
            im_ref = parser.preprocess_img(pil)
            heads = parser.seg(im_ref)
            x = torchvision.transforms.ToTensor()(pil)[:3].unsqueeze(0)
            im_ora = PO.preprocess(x, 2)
            e_pre = rel(im_ora, im_ref)
            heads_ora = PO.bisenet_forward(st, im_ref)
            e_heads = [rel(a, b) for a, b in zip(heads_ora, heads)]
            lab_ora = PO.parse(st, x, 2)[0].numpy()
            same = bool((lab_ora == seg12).all())
            classes, counts = np.unique(seg12, return_counts=True)
            print(f"  parser/{tag}: preprocess max-rel {e_pre:.2e}, heads max-rel {', '.join(f'{e:.2e}' for e in e_heads)}, "
                  f"labels equal {same}; {len(classes)} classes, largest {counts.max() / seg12.size:.1%}")
            assert e_pre <= TOL and max(e_heads) <= TOL and same, (e_pre, e_heads, same)
            assert seg12.dtype == np.uint8 and seg12.shape == (size // 2, size // 2)
            gold[f"parser/{tag}/seg12"] = seg12
            gold[f"parser/{tag}/seg19"] = seg19
            gold[f"parser/{tag}/pre_sub"] = im_ref[:, :, ::8, ::8].numpy()
            for name, t in zip(("out", "out16", "out32"), heads):
                gold[f"parser/{tag}/{name}_sub"] = t[:, :, ::SUB, ::SUB].numpy()
        # the visualisation, on a 128 x 128 crop of the 1024 case's 19-class map and its image
        anno = gold["parser/p1024/seg19"][::4, ::4].copy()
        gold["parser/vis_anno"] = anno
        gold["parser/vis"] = FD.vis_parsing_maps(Image.fromarray(PO.case_image(1024, 11)), anno, stride=1)
    conv = getattr(D, "__ffhq_masks_to_faceParser_mask_detailed")
    gold["parser/ffhq_lut"] = conv(np.arange(256, dtype=np.uint8))
    assert (gold["parser/ffhq_lut"] == np.asarray(PO.FFHQ19_TO_12, dtype=np.uint8)).all()
    paths = golden_io.save(OUT, gold)
    print(f"wrote {len(gold)} arrays -> " + ", ".join(f"{p} ({os.path.getsize(p) / 1024:.0f} KiB)" for p in paths))


if __name__ == "__main__":
    main()
