"""GPEN's ParseNet (e4s_b200.gpen.face_parse): the oracle and the mirror against the reference's goldens on the CPU, the
padding identities the reflection-padded kernel relies on (float64), and on the GPU the network's logits, out_img and
masks against the goldens and one CUDA-graph capture of FaceParse.process_tensor.  The kernels against float64 at the
production batch are checked in tests/test_gpen_parse_at_scale.py."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from conftest import ROOT

from oracle import golden_io
from oracle import gpen_parse_oracle as PO

CASES = [("a", 512, 512, 11), ("b", 512, 512, 12)]
RESIZE_CASE = ("r600x560", 600, 560, 13)
SUB = 8


@pytest.fixture(scope="module")
def gold():
    return golden_io.load(os.path.join(ROOT, "tests", "golden", "gpen_parse_vectors.npz"))


# ------------------------------------------------------------------------------------------------------------ CPU
@pytest.mark.parametrize("tag,h,w,seed", CASES)
def test_oracle_matches_reference_golden(gold, tag, h, w, seed):
    st = PO.synthetic_state()
    img = PO.case_image(h, w, seed)
    with torch.no_grad():
        lg, im = PO.parsenet_forward(st, PO.process_input(img))
    ref = torch.from_numpy(gold[f"parse/{tag}/logits_sub"])
    assert float((lg[0, :, ::SUB, ::SUB] - ref).abs().max() / ref.abs().max()) <= 2e-5
    ref_im = torch.from_numpy(gold[f"parse/{tag}/img_sub"])
    assert float((im[0, :, ::SUB, ::SUB] - ref_im).abs().max() / ref_im.abs().max()) <= 2e-5
    assert np.array_equal(lg.argmax(1)[0].to(torch.uint8).numpy(), gold[f"parse/{tag}/labels"])
    assert np.array_equal(PO.process(st, img)[0], gold[f"parse/{tag}/mask"])
    t = PO.process_tensor(st, PO.image_tensor(img))
    assert t.dtype == torch.int64 and tuple(t.shape) == (1, 1, 512, 512)
    assert np.array_equal(t[0, 0].to(torch.uint8).numpy(), gold[f"parse/{tag}/mask_tensor"])


def test_golden_masks_are_not_degenerate(gold):
    """The stand-in head spreads the argmax: >= 5 classes at >= 1 % of the pixels, both mask values at >= 5 %."""
    for tag, *_ in CASES:
        lab = gold[f"parse/{tag}/labels"]
        frac = np.bincount(lab.ravel(), minlength=19) / lab.size
        assert (frac >= 0.01).sum() >= 5, (tag, frac)
        zero = float((gold[f"parse/{tag}/mask"] == 0).mean())
        assert 0.05 <= zero <= 0.95, (tag, zero)
        assert set(np.unique(gold[f"parse/{tag}/mask"])) == {0, 255}


def test_mirror_state_dict_layout():
    from e4s_b200.gpen.face_parse.parse_model import ParseNet, define_P
    with open(os.path.join(ROOT, "tests", "golden", "gpen_parse_checkpoint_layout.json")) as f:
        layout = json.load(f)
    assert len(layout) == 238
    net = ParseNet(512, 512, 32, 64, 19, norm_type='bn', relu_type='LeakyReLU', ch_range=[32, 256])
    assert {k: list(v.shape) for k, v in net.state_dict().items()} == layout
    net.load_state_dict(PO.synthetic_state(), strict=True)
    assert {k: list(v.shape) for k, v in define_P().state_dict().items()} == layout
    # other configurations build the reference's tree; their forward is not provided
    other = ParseNet(128, 128, 32, 64, 19, norm_type='bn', relu_type='prelu', ch_range=[32, 512])
    assert any(k.endswith("relu.func.weight") for k in other.state_dict())
    with pytest.raises(NotImplementedError), torch.no_grad():
        other(torch.zeros(1, 3, 128, 128))


def test_face_parse_loads_checkpoint_and_guards(tmp_path):
    from e4s_b200.gpen.face_parse.face_parsing import FaceParse
    os.makedirs(tmp_path / "weights")
    st = PO.synthetic_state()
    torch.save(st, tmp_path / "weights" / "ParseNet-latest.pth")
    fp = FaceParse(str(tmp_path), device="cpu")
    assert torch.equal(fp.faceparse.out_mask_conv.conv2d.bias, st["out_mask_conv.conv2d.bias"])
    assert not fp.faceparse.training and fp.MASK_COLORMAP == PO.MASK_COLORMAP
    with pytest.raises(ValueError), torch.no_grad():       # the kernels need a CUDA tensor
        fp.faceparse(torch.zeros(1, 3, 512, 512))
    with pytest.raises(ValueError):
        fp.process_tensor(torch.zeros(1, 3, 64, 64))
    fp.faceparse.train()
    with pytest.raises(NotImplementedError), torch.no_grad():
        fp.faceparse(torch.zeros(1, 3, 512, 512))


def test_process_input_is_the_reference_conversion():
    """FaceParse.process feeds the network exactly the reference's float64-normalised input."""
    from e4s_b200.gpen.face_parse.face_parsing import FaceParse
    import cv2
    img = PO.case_image(300, 280, 5)
    fp = FaceParse.__new__(FaceParse)
    fp.device, fp.size = "cpu", 512
    assert torch.equal(fp.img2tensor(cv2.resize(img, (512, 512))), PO.process_input(img))


def test_padding_identities_float64():
    """The three rules e4s_conv3x3_reflect_tcr_f32 relies on, in float64: (1) reflection pad 1 is the mirror rule; (2) nearest
    2x up-sampling then reflection pad 1 equals replicate padding at the source resolution; (3) reflection pad 1 then a 3x3
    stride-2 convolution equals the four taps {-1, 0}^2 over the space-to-depth operand with row / column -1 replicating
    row / column 0 (no padding read at the bottom or right for even sizes)."""
    g = torch.Generator().manual_seed(0)
    x = torch.randn(2, 4, 8, 10, generator=g, dtype=torch.float64)
    w = torch.randn(5, 4, 3, 3, generator=g, dtype=torch.float64)
    # (1)
    xp = F.pad(x, (1, 1, 1, 1), mode="reflect")
    assert torch.equal(xp[:, :, 0, 1:-1], x[:, :, 1]) and torch.equal(xp[:, :, -1, 1:-1], x[:, :, -2])
    assert torch.equal(xp[:, :, 1:-1, 0], x[:, :, :, 1]) and torch.equal(xp[:, :, 1:-1, -1], x[:, :, :, -2])
    # (2)
    ref = F.conv2d(F.pad(F.interpolate(x, scale_factor=2, mode="nearest"), (1, 1, 1, 1), mode="reflect"), w)
    rep = F.interpolate(F.pad(x, (1, 1, 1, 1), mode="replicate"), scale_factor=2, mode="nearest")[:, :, 1:-1, 1:-1]
    assert float((F.conv2d(rep, w) - ref).abs().max()) == 0.0
    # (3): the s2d channel order of e4s_space_to_depth_f32, (py, px, c)
    ref2 = F.conv2d(F.pad(x, (1, 1, 1, 1), mode="reflect"), w, stride=2)
    b, c, h, wd = x.shape
    s2d = x.reshape(b, c, h // 2, 2, wd // 2, 2).permute(0, 3, 5, 1, 2, 4).reshape(b, 4 * c, h // 2, wd // 2)
    s2d_p = F.pad(s2d, (1, 0, 1, 0), mode="replicate")
    w2 = torch.zeros(5, 4 * c, 2, 2, dtype=torch.float64)
    tap_of = {0: (0, 1), 1: (1, 0), 2: (1, 1)}             # k -> (tap index in {-1, 0} + 1, parity)
    for ky in range(3):
        ty, py = tap_of[ky]
        for kx in range(3):
            tx, px = tap_of[kx]
            w2[:, (py * 2 + px) * c:(py * 2 + px + 1) * c, ty, tx] = w[:, :, ky, kx]
    out2 = F.conv2d(s2d_p, w2)
    assert out2.shape == ref2.shape
    assert float((out2 - ref2).abs().max()) <= 1e-13


def test_dropin_resolves_face_parse():
    code = ("import e4s_b200.dropin as d; d.install()\n"
            "from src.pretrained.gpen.face_parse.blocks import ConvLayer, ResidualBlock, NormLayer, ReluLayer\n"
            "from src.pretrained.gpen.face_parse.parse_model import ParseNet\n"
            "from src.pretrained.gpen.face_parse.face_parsing import FaceParse\n"
            "assert ConvLayer.__module__ == ResidualBlock.__module__ == NormLayer.__module__ == ReluLayer.__module__ == "
            "'e4s_b200.gpen.face_parse.blocks'\n"
            "assert ParseNet.__module__ == 'e4s_b200.gpen.face_parse.parse_model'\n"
            "assert FaceParse.__module__ == 'e4s_b200.gpen.face_parse.face_parsing'\n")
    r = subprocess.run([sys.executable, "-c", code], cwd=ROOT, capture_output=True, text=True,
                       env=dict(os.environ, PYTHONPATH=ROOT))
    assert r.returncode == 0, r.stderr


# ------------------------------------------------------------------------------------------------------------ GPU
@pytest.fixture(scope="module")
def fp(tmp_path_factory):
    from e4s_b200.gpen.face_parse.face_parsing import FaceParse
    d = tmp_path_factory.mktemp("gpen_parse")
    os.makedirs(d / "weights")
    torch.save(PO.synthetic_state(), d / "weights" / "ParseNet-latest.pth")
    f = FaceParse(str(d), device="cuda")
    f.faceparse.requires_grad_(False)
    return f


def _logit_error(fp, gold):
    """Largest |ours - reference| of the logits over the stored pixels of both cases, and the forward outputs."""
    err, outs = 0.0, {}
    with torch.no_grad():
        for tag, h, w, seed in CASES:
            lg, im = fp.faceparse(PO.process_input(PO.case_image(h, w, seed)).cuda())
            ref = torch.from_numpy(gold[f"parse/{tag}/logits_sub"]).cuda()
            err = max(err, float((lg[0, :, ::SUB, ::SUB] - ref).abs().max()))
            outs[tag] = lg, im
    return err, outs


@pytest.mark.gpu
def test_forward_matches_reference_golden(fp, gold):
    _, outs = _logit_error(fp, gold)
    for tag, *_ in CASES:
        lg, im = outs[tag]
        assert tuple(lg.shape) == (1, 19, 512, 512) and tuple(im.shape) == (1, 3, 512, 512)
        for ours, key in ((lg, "logits_sub"), (im, "img_sub")):
            ref = torch.from_numpy(gold[f"parse/{tag}/{key}"]).cuda().double()
            d = ours[0, :, ::SUB, ::SUB].double() - ref
            e, r = float(d.abs().max() / ref.abs().max()), float(d.norm() / ref.norm())
            print(f"{tag} {key}: max-rel {e:.2e} rel-RMS {r:.2e}")
            assert e <= 1e-3 and r <= 1e-3, (tag, key, e, r)


@pytest.mark.gpu
def test_masks_match_reference_away_from_ties(fp, gold):
    """process() / process_tensor() masks equal the reference's at every pixel whose top-1 / top-2 logit margin (of our
    logits) exceeds twice the logit error measured on the stored pixels, times 2 for the pixels not stored."""
    err, outs = _logit_error(fp, gold)
    bar = 4.0 * err
    for tag, h, w, seed in CASES:
        img = PO.case_image(h, w, seed)
        lg = outs[tag][0][0]
        top2 = lg.topk(2, dim=0).values
        sure = ((top2[0] - top2[1]) > bar).cpu().numpy()
        m = fp.process(img)
        assert len(m) == 1 and m[0].dtype == np.uint8 and m[0].shape == (512, 512)
        t = fp.process_tensor(PO.image_tensor(img).cuda())
        assert t.dtype == torch.int64 and tuple(t.shape) == (1, 1, 512, 512)
        t = t[0, 0].cpu().numpy()
        ref_m, ref_t = gold[f"parse/{tag}/mask"], gold[f"parse/{tag}/mask_tensor"]
        print(f"{tag}: logit error {err:.2e}, pixels within the tie band {1 - sure.mean():.4%}; masks differing there: "
              f"process {int((m[0] != ref_m).sum())}, process_tensor {int((t != ref_t).sum())}")
        assert np.array_equal(m[0][sure], ref_m[sure]) and np.array_equal(t[sure], ref_t[sure]), tag
        assert (1 - sure.mean()) < 0.01, tag
    # process_tensor's nearest resize from a 600 x 560 image
    tag, h, w, seed = RESIZE_CASE
    t = fp.process_tensor(PO.image_tensor(PO.case_image(h, w, seed)).cuda())[0, 0].cpu().numpy()
    ref_t = gold[f"parse/{tag}/mask_tensor"]
    diff = float((t != ref_t).mean())
    print(f"{tag}: process_tensor masks differ at {diff:.4%} of the pixels")
    assert diff < 0.002, diff


@pytest.mark.gpu
def test_process_tensor_cuda_graph_equals_eager(fp):
    """One CUDA-graph capture of process_tensor on 16 faces, replayed on new inputs: equal to eager."""
    x = torch.stack([PO.image_tensor(PO.case_image(512, 512, 200 + i))[0] for i in range(16)]).cuda()
    x2 = torch.stack([PO.image_tensor(PO.case_image(512, 512, 300 + i))[0] for i in range(16)]).cuda()
    eager = fp.process_tensor(x)
    eager2 = fp.process_tensor(x2)
    static = x.clone()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        fp.process_tensor(static)                        # warm-up on the side stream (weights prepared, kernels loaded)
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        out = fp.process_tensor(static)
    g.replay()
    torch.cuda.synchronize()
    assert torch.equal(out, eager)
    static.copy_(x2)
    g.replay()
    torch.cuda.synchronize()
    assert torch.equal(out, eager2)
    assert tuple(out.shape) == (1, 16, 512, 512) and out.dtype == torch.int64


@pytest.mark.gpu
def test_forward_guards_autograd(fp):
    x = torch.zeros(1, 3, 512, 512, device="cuda", requires_grad=True)
    with pytest.raises(NotImplementedError):
        fp.faceparse(x)
    with pytest.raises(ValueError):
        with torch.no_grad():
            fp.faceparse(torch.zeros(1, 3, 256, 256, device="cuda"))
