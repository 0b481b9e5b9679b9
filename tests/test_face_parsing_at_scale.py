"""BiSeNet face-parser kernels against float64 at the production shape: 16 faces of 1024 x 1024 (the 512 x 512 network
input), each kernel on its own fp32 inputs, then the whole parse.  Tolerances are the measured errors (H100 80GB HBM3)
with headroom; each test prints what it measured."""
import os
import tempfile

import pytest
import torch
import torch.nn.functional as F

from conftest import REL_TOL, rel_err, rel_rms
from oracle import parser_oracle as PO

pytestmark = pytest.mark.gpu

B, SIZE = 16, 1024


def _check(ours, ref64, tol, what):
    e, r = rel_err(ours, ref64), rel_rms(ours, ref64)
    print(f"{what}: max-rel {e:.2e}  rel-RMS {r:.2e}")
    assert e <= tol and r <= tol, (what, e, r)
    return e


@pytest.fixture(autouse=True)
def _no_grad():
    """Every test runs without autograd (the parser is forward-only); the setting is restored after it."""
    with torch.no_grad():
        yield


@pytest.fixture(scope="module")
def parser():
    from e4s_b200.face_parsing.face_parsing_demo import FaceParser
    with tempfile.TemporaryDirectory() as tmp:
        ckpt = os.path.join(tmp, "bisenet.pth")
        torch.save(PO.synthetic_state(), ckpt)
        return FaceParser(ckpt, device="cuda")


@pytest.fixture(scope="module")
def images():
    return torch.stack([torch.from_numpy(PO.case_image(SIZE, 100 + i)).permute(2, 0, 1) for i in range(B)]).cuda().float() / 255


@pytest.fixture(scope="module")
def st64():
    return {k: v.double().cuda() if v.is_floating_point() else v for k, v in PO.synthetic_state().items()}


def _randn(*shape, seed, dev="cuda"):
    return torch.randn(*shape, generator=torch.Generator(device=dev).manual_seed(seed), device=dev)


@pytest.mark.parametrize("factor", [2, 4])
def test_preprocess(parser, images, factor):
    from e4s_b200 import kernels as K
    from e4s_b200.face_parsing.face_parsing_demo import BicubicDownSample
    mean, std, _, _ = parser._device_consts(images.device)
    ours = K.bicubic_down_norm(images, BicubicDownSample(factor).taps(images.device), factor, mean, std)
    _check(ours, PO.preprocess(images.double(), factor), 1e-5, f"preprocess f={factor}")


def test_stem(parser):
    from e4s_b200 import kernels as K
    x = _randn(B, 3, 512, 512, seed=1)
    w, b = parser.seg._prepared(x.device)["stem"]
    ours = K.parser_stem(x, w, b)
    ref = F.max_pool2d(F.relu(F.conv2d(x.double(), w.double(), stride=2, padding=3) + b.double()[None, :, None, None]), 3, 2, 1)
    _check(ours, ref.permute(0, 2, 3, 1), 1e-5, "stem + pool")


# (input side, Cin, Cout, kind): every convolution shape of the trunk at the 512 x 512 input
TRUNK = [(128, 64, 64, "plain"), (128, 64, 128, "s2d"), (128, 64, 128, "shortcut"), (64, 128, 128, "plain"),
         (64, 128, 256, "s2d"), (64, 128, 256, "shortcut"), (32, 256, 256, "plain"), (32, 256, 512, "s2d"),
         (32, 256, 512, "shortcut"), (16, 512, 512, "plain")]


@pytest.mark.parametrize("side,cin,cout,kind", TRUNK)
def test_bias_residual_conv(side, cin, cout, kind):
    from e4s_b200 import kernels as K
    from e4s_b200.encoders.psp_encoders import TAP_CENTRE, TAPS_S2D, _conv_planes, _conv_planes_s2d
    from e4s_b200.face_parsing.model import _shortcut_planes
    x = F.relu(_randn(B, side, side, cin, seed=side + cin))
    k = 1 if kind == "shortcut" else 3
    w = _randn(cout, cin, k, k, seed=cout, dev="cpu") * (2.0 / (cin * k * k)) ** 0.5
    bias = 0.1 * _randn(cout, seed=3)
    ref = F.conv2d(x.permute(0, 3, 1, 2).double(), w.double().cuda(), stride=1 if kind == "plain" else 2, padding=k // 2)
    ref = ref + bias.double()[None, :, None, None]
    if kind == "plain":
        res = _randn(B, side, side, cout, seed=5)
        ours = K.conv3x3_bias_tc(x, _conv_planes(w).cuda(), bias, residual=res, relu=True)
        ref = F.relu(ref + res.permute(0, 3, 1, 2).double())
    elif kind == "s2d":
        ours = K.conv3x3_bias_tc(K.space_to_depth(x), _conv_planes_s2d(w).cuda(), bias, relu=True, tap_mask=TAPS_S2D)
        ref = F.relu(ref)
    else:
        ours = K.conv3x3_bias_tc(K.space_to_depth(x), _shortcut_planes(w).cuda(), bias, tap_mask=TAP_CENTRE)
    _check(ours, ref.permute(0, 2, 3, 1), 5e-5, f"conv {kind} {side}^2 {cin}->{cout}")


@pytest.mark.parametrize("low,c", [(64, 256), (32, 64)])
def test_head(low, c):
    from e4s_b200 import kernels as K
    from e4s_b200.masks import FFHQ19_TO_12
    x = F.relu(_randn(B, low, low, c, seed=low))
    w = _randn(19, c, seed=c) / c ** 0.5
    lut = torch.tensor(FFHQ19_TO_12, dtype=torch.uint8, device="cuda")
    lab, lg = K.parse_head(x, w, 512, 512, labels=True, logits=True)
    lab12, none = K.parse_head(x, w, 512, 512, lut=lut)
    assert none is None
    ref = F.interpolate(torch.einsum("bhwc,kc->bkhw", x.double(), w.double()), (512, 512), mode="bilinear", align_corners=True)
    _check(lg, ref, 1e-5, f"head logits {low}^2 x {c}")
    E = float((lg.double() - ref).abs().max())
    top2 = ref.topk(2, dim=1).values
    sure = (top2[:, 0] - top2[:, 1]) > 2 * E
    assert float(sure.double().mean()) > 0.999
    assert torch.equal(lab[sure], ref.argmax(1)[sure].to(torch.uint8))
    assert torch.equal(lab12, lut[lab.long()])
    # labels equal to the argmax of the logits it wrote, ties to the first index
    assert torch.equal(lab, lg.argmax(1).to(torch.uint8))
    zero, _ = K.parse_head(torch.zeros_like(x), w, 512, 512)
    assert int(zero.max()) == 0


def test_forward_and_parse_against_float64(parser, images, st64):
    from e4s_b200 import kernels as K
    mean, std, lut, _ = parser._device_consts(images.device)
    xin = K.bicubic_down_norm(images, parser.downsample.taps(images.device), 2, mean, std)
    heads = parser.seg(xin)
    ref = PO.bisenet_forward(st64, xin.double())
    for name, a, b in zip(("out", "out16", "out32"), heads, ref):
        _check(a, b, REL_TOL, f"BiSeNet.forward {name}")
    E = float((heads[0].double() - ref[0]).abs().max())
    top2 = ref[0].topk(2, dim=1).values
    sure = (top2[:, 0] - top2[:, 1]) > 2 * E
    near = 1 - float(sure.double().mean())
    print(f"labels: E = {E:.2e}, near-tie pixels {near:.3%}")
    assert near < 1e-3
    lab = parser.parse(images)
    assert lab.dtype == torch.uint8 and tuple(lab.shape) == (B, 512, 512)
    ref12 = lut[ref[0].argmax(1)]
    assert torch.equal(lab[sure], ref12[sure])


def test_alone_equals_batch_and_graph_replay(parser, images):
    full = parser.parse(images)
    alone = parser.parse(images[5:6].contiguous())
    assert torch.equal(alone[0], full[5])
    # captured in a CUDA graph and replayed: bitwise the eager result
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        parser.parse(images)
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        out = parser.parse(images)
    g.replay()
    torch.cuda.synchronize()
    assert torch.equal(out, full)


def test_parse_feeds_the_swap_masks(parser, images):
    from e4s_b200 import masks as M
    lab = parser.parse(images)
    assert lab.dtype == torch.uint8 and tuple(lab.shape) == (B, 512, 512) and int(lab.max()) < 12
    half = B // 2
    swapped, hole, fg = M.swap_head_mask_with_foreground(lab[:half], lab[half:])
    onehot = M.labelMap2OneHot(swapped, 12)
    assert tuple(onehot.shape) == (half, 12, 512, 512)


def test_parse_rejects_bad_shapes(parser):
    with pytest.raises(ValueError):
        parser.parse(torch.zeros(1, 3, 1000, 1024, device="cuda"))
    with pytest.raises(ValueError):
        parser.parse(torch.zeros(1, 3, 384, 384, device="cuda"))        # narrower than 512
    with pytest.raises(ValueError):
        parser.parse(torch.zeros(1, 3, 1024, 1024, device="cuda", dtype=torch.float16))
