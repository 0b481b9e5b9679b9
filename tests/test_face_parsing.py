"""BiSeNet face parser (e4s_b200.face_parsing): oracle and mirror against the reference's goldens on the CPU, the kernels'
end-to-end results on the GPU."""
import os
import subprocess
import sys
import tempfile

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from conftest import ROOT, REL_TOL, assert_close

from oracle import golden_io
from oracle import parser_oracle as PO

CASES = [("p1024", 1024, 11), ("p768", 768, 12)]
SUB = 16


@pytest.fixture(autouse=True)
def _no_grad():
    """Every test runs without autograd (the parser is forward-only); the setting is restored after it."""
    with torch.no_grad():
        yield


@pytest.fixture(scope="module")
def gold():
    return golden_io.load(os.path.join(ROOT, "tests", "golden", "parser_vectors.npz"))


def _image(size, seed):
    return torch.from_numpy(PO.case_image(size, seed)).permute(2, 0, 1)[None].float() / 255


def _pil(size, seed):
    from PIL import Image
    return Image.fromarray(PO.case_image(size, seed))


# ------------------------------------------------------------------------------------------------------------ CPU
@pytest.mark.parametrize("tag,size,seed", CASES)
def test_oracle_matches_reference_golden(gold, tag, size, seed):
    st = PO.synthetic_state()
    x = PO.preprocess(_image(size, seed), 2)
    e = float((x[:, :, ::8, ::8] - torch.from_numpy(gold[f"parser/{tag}/pre_sub"])).abs().max())
    assert e <= 2e-5, e
    for name, t in zip(("out", "out16", "out32"), PO.bisenet_forward(st, x)):
        ref = torch.from_numpy(gold[f"parser/{tag}/{name}_sub"])
        assert float((t[:, :, ::SUB, ::SUB] - ref).abs().max() / ref.abs().max()) <= 2e-5, name
    assert np.array_equal(PO.parse(st, _image(size, seed), 2)[0].numpy(), gold[f"parser/{tag}/seg12"])


def test_golden_label_maps_are_not_degenerate(gold):
    for tag, size, _ in CASES:
        seg = gold[f"parser/{tag}/seg12"]
        assert seg.shape == (size // 2, size // 2) and seg.dtype == np.uint8
        classes, counts = np.unique(seg, return_counts=True)
        assert len(classes) >= 6 and counts.max() <= 0.5 * seg.size, (tag, classes, counts / seg.size)


def test_mirror_state_dict_and_no_download(monkeypatch):
    import torch.hub
    import torch.utils.model_zoo as model_zoo

    def no_network(*a, **k):
        raise AssertionError("a download was attempted")

    monkeypatch.setattr(model_zoo, "load_url", no_network)
    monkeypatch.setattr(torch.hub, "load_state_dict_from_url", no_network)
    from e4s_b200.face_parsing.model import BiSeNet
    from e4s_b200.face_parsing.resnet import Resnet18
    Resnet18()
    net = BiSeNet(n_classes=19)
    assert {k: tuple(v.shape) for k, v in net.state_dict().items()} == PO.param_shapes()
    assert len(net.state_dict()) == 191


def test_ffhq_lut_and_stand_in_state(gold):
    from e4s_b200.masks import FFHQ19_TO_12
    from e4s_b200.synthetic import synthetic_parser_state
    assert np.array_equal(np.asarray(FFHQ19_TO_12, dtype=np.uint8), gold["parser/ffhq_lut"])
    ours = synthetic_parser_state(PO.param_shapes())
    theirs = PO.synthetic_state()
    assert sorted(ours) == sorted(theirs)
    for k in ours:
        assert ours[k].dtype == theirs[k].dtype and torch.equal(ours[k], theirs[k]), k


def test_vis_parsing_maps_golden(gold):
    from e4s_b200.face_parsing.face_parsing_demo import vis_parsing_maps
    out = vis_parsing_maps(_pil(1024, 11), gold["parser/vis_anno"], stride=1)
    assert out.dtype == np.uint8 and np.array_equal(out, gold["parser/vis"])


def test_dropin_resolves_face_parsing():
    code = ("import e4s_b200.dropin as d; d.install()\n"
            "from src.pretrained.face_parsing.face_parsing_demo import init_faceParsing_pretrained_model, faceParsing_demo, "
            "vis_parsing_maps\n"
            "from src.pretrained.face_parsing.model import BiSeNet\n"
            "from src.pretrained.face_parsing.resnet import Resnet18\n"
            "assert init_faceParsing_pretrained_model.__module__ == 'e4s_b200.face_parsing.face_parsing_demo'\n"
            "assert faceParsing_demo.__module__ == vis_parsing_maps.__module__ == 'e4s_b200.face_parsing.face_parsing_demo'\n"
            "assert BiSeNet.__module__ == 'e4s_b200.face_parsing.model'\n"
            "assert Resnet18.__module__ == 'e4s_b200.face_parsing.resnet'\n")
    r = subprocess.run([sys.executable, "-c", code], cwd=ROOT, capture_output=True, text=True,
                       env=dict(os.environ, PYTHONPATH=ROOT))
    assert r.returncode == 0, r.stderr


def _cpu_parser(tmp):
    from e4s_b200.face_parsing.face_parsing_demo import FaceParser
    ckpt = os.path.join(tmp, "bisenet.pth")
    torch.save(PO.synthetic_state(), ckpt)
    return FaceParser(ckpt, device="cpu")


def test_parse_rejects_bad_input_and_unsupported_paths():
    from e4s_b200.face_parsing import face_parsing_demo as FD
    from e4s_b200.face_parsing.model import BiSeNet
    with tempfile.TemporaryDirectory() as tmp:
        parser = _cpu_parser(tmp)
    with pytest.raises(ValueError):
        parser.parse(torch.rand(1, 3, 1024, 1024))                    # not on the GPU
    with pytest.raises(ValueError):
        parser.parse(np.zeros((1, 3, 1024, 1024), np.float32))
    with pytest.raises(NotImplementedError):
        FD.init_faceParsing_pretrained_model("segnext", "x.pth", "cfg.py")
    with pytest.raises(NotImplementedError):
        FD.faceParsing_demo(parser, None, model_name="segnext")
    with pytest.raises(NotImplementedError):
        BiSeNet(19).train()(torch.zeros(1, 3, 64, 64))


# ------------------------------------------------------------------------------------------------------------ float64 identities
def _f64(*shape, seed=0):
    return torch.randn(*shape, generator=torch.Generator().manual_seed(seed), dtype=torch.float64)


def test_bn_folding_identity():
    from e4s_b200.face_parsing.model import fold_bn
    bn = torch.nn.BatchNorm2d(8).eval().double()
    with torch.no_grad():
        bn.weight.copy_(1 + 0.1 * _f64(8, seed=1)), bn.bias.copy_(_f64(8, seed=2))
        bn.running_mean.copy_(_f64(8, seed=3)), bn.running_var.copy_(1 + _f64(8, seed=4).abs())
        w, x = _f64(8, 4, 3, 3, seed=5), _f64(2, 4, 9, 9, seed=6)
        ref = bn(F.conv2d(x, w, padding=1))
        # fold_bn rounds to fp32 once; the identity holds to that rounding
        wf, bf = fold_bn(w, bn)
        ours = F.conv2d(x, wf.double(), padding=1) + bf.double().reshape(1, -1, 1, 1)
    assert float((ours - ref).abs().max() / ref.abs().max()) < 1e-6


def test_operand_affine_and_up2_identities():
    x, a, b = _f64(2, 4, 6, 6, seed=7), torch.sigmoid(_f64(2, 4, seed=8)), _f64(2, 4, seed=9)
    w = _f64(5, 4, 3, 3, seed=10)
    aff = lambda t: t * a[:, :, None, None] + b[:, :, None, None]  # noqa: E731
    # ARM32(x) + avg, then nearest up2 and a padded convolution ...
    ref = F.conv2d(F.interpolate(aff(x), scale_factor=2, mode="nearest"), w, padding=1)
    # ... equals the kernel's order: up2 first, the affine on in-image pixels while staging (zero padding stays zero)
    up = F.interpolate(x, scale_factor=2, mode="nearest")
    assert torch.allclose(F.conv2d(aff(up), w, padding=1), ref, rtol=0, atol=1e-12)
    # the FFM's f * atten + f is the affine with scale 1 + atten, shift 0
    assert torch.allclose(x * a[:, :, None, None] + x, x * (1 + a)[:, :, None, None], rtol=0, atol=1e-12)
    # cat([feat8, feat_cp8]) through a 1x1 convolution = two 1x1 convolutions, summed
    y, w1 = _f64(2, 3, 6, 6, seed=11), _f64(5, 7, 1, 1, seed=12)
    assert torch.allclose(F.conv2d(torch.cat([x, y], 1), w1), F.conv2d(x, w1[:, :4]) + F.conv2d(y, w1[:, 4:]), rtol=0,
                          atol=1e-12)


def head_reference(low: torch.Tensor, out_h: int, out_w: int):
    """The head kernel's interpolation and argmax rule, restated: source coordinate fp32 scale (in - 1) / (out - 1) times
    the destination index, i0 = floor, i1 = min(i0 + 1, in - 1), weights s - i0; first index of the maximum."""
    h, w = low.shape[2:]
    sy = torch.tensor((h - 1) / (out_h - 1), dtype=torch.float32) * torch.arange(out_h, dtype=torch.float32)
    sx = torch.tensor((w - 1) / (out_w - 1), dtype=torch.float32) * torch.arange(out_w, dtype=torch.float32)
    y0, x0 = sy.long(), sx.long()
    y1, x1 = (y0 + 1).clamp(max=h - 1), (x0 + 1).clamp(max=w - 1)
    fy, fx = (sy - y0).to(low.dtype)[:, None], (sx - x0).to(low.dtype)[None, :]
    g = lambda yy, xx: low[:, :, yy][:, :, :, xx]  # noqa: E731
    up = (1 - fy) * ((1 - fx) * g(y0, x0) + fx * g(y0, x1)) + fy * ((1 - fx) * g(y1, x0) + fx * g(y1, x1))
    return up, up.argmax(1)


def test_head_index_rule_matches_interpolate():
    low = _f64(2, 19, 64, 64, seed=13)
    up, lab = head_reference(low, 512, 512)
    ref = F.interpolate(low, (512, 512), mode="bilinear", align_corners=True)
    # the fp32 source coordinate (as torch computes it for fp32 inputs) moves a sample by ~1e-6 of a low-res pixel
    d = float((up - ref).abs().max())
    assert d < 1e-5 * float(low.abs().max()), d
    margin = ref.topk(2, dim=1).values
    sure = (margin[:, 0] - margin[:, 1]) > 2 * d
    assert torch.equal(lab[sure], ref.argmax(1)[sure]) and float(sure.double().mean()) > 0.999
    # ties go to the first index
    tie = torch.zeros(1, 3, 2, 2, dtype=torch.float64)
    assert int(head_reference(tie, 4, 4)[1].max()) == 0


# ------------------------------------------------------------------------------------------------------------ GPU
def _gpu_parser(tmp):
    from e4s_b200.face_parsing.face_parsing_demo import FaceParser
    ckpt = os.path.join(tmp, "bisenet.pth")
    torch.save(PO.synthetic_state(), ckpt)
    return FaceParser(ckpt, device="cuda")


def margin_and_labels(logits64: torch.Tensor):
    """float64 logits [B, C, H, W] -> (top-1 minus top-2 margin, 19-class labels)."""
    top2 = logits64.topk(2, dim=1).values
    return top2[:, 0] - top2[:, 1], logits64.argmax(1)


@pytest.mark.gpu
@pytest.mark.parametrize("tag,size,seed", CASES)
def test_parser_against_reference_golden(gold, tag, size, seed):
    from e4s_b200.face_parsing.face_parsing_demo import faceParsing_demo
    with tempfile.TemporaryDirectory() as tmp:
        parser = _gpu_parser(tmp)
    img = _image(size, seed).cuda()
    x = parser.preprocess_img(_pil(size, seed))
    assert_close(x[:, :, ::8, ::8].cpu(), gold[f"parser/{tag}/pre_sub"], what="preprocess")
    heads = parser.seg(x)
    for name, t in zip(("out", "out16", "out32"), heads):
        assert_close(t[:, :, ::SUB, ::SUB].cpu(), gold[f"parser/{tag}/{name}_sub"], what=name)
    # labels: equal to the reference wherever the float64 oracle's top-1 / top-2 margin exceeds 2 E
    st64 = {k: v.double().cuda() if v.is_floating_point() else v for k, v in PO.synthetic_state().items()}
    l64 = PO.main_logits(st64, PO.preprocess(img.double(), 2))
    E = float((heads[0].double() - l64).abs().max())
    margin, _ = margin_and_labels(l64)
    sure = (margin > 2 * E)[0].cpu().numpy()
    assert 1 - sure.mean() < 1e-3, (E, 1 - sure.mean())
    ref = gold[f"parser/{tag}/seg12"]
    ours = parser.parse(img)[0].cpu().numpy()
    assert np.array_equal(ours[sure], ref[sure])
    demo = faceParsing_demo(parser, _pil(size, seed))
    assert demo.dtype == np.uint8 and demo.shape == ref.shape
    assert np.array_equal(demo[sure], ref[sure])
