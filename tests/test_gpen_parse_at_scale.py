"""GPEN ParseNet kernels against float64 at the production batch: 16 faces of 512 x 512 (FaceParse on the face swap's restored
faces).  Each distinct layer form on its own fp32 inputs - the reflection-padded convolution at every (Cin, Cout, resolution)
class, the stride-2 pair of a down block, the up pair of an up block, a body block and the long skip, the 3 -> 64 input
convolution (with and without process_tensor's input conversion), the mask head's logits - then the whole forward.  The
float64 references are plain torch (F.pad reflect, F.conv2d, F.interpolate) on the GPU; at 512 x 512 they are computed for
faces 0 and 15 only (the kernels still run on all 16), elsewhere for all 16.  Tolerances are the measured errors (H100 80GB
HBM3) with headroom; each test prints what it measured."""
import pytest
import torch
import torch.nn.functional as F

from f64ref import Ledger, at_scale, nchw, pm, randn  # noqa: F401
from oracle import gpen_parse_oracle as PO

pytestmark = pytest.mark.gpu

B = 16
FACES_512 = [0, 15]
LAYER_TOL = 5e-5
FORWARD_TOL = 2e-4
LEDGER = Ledger(14)


def _weights(cout, cin, seed):
    w = randn(cout, cin, 3, 3, seed=seed) * (1.0 / (9 * cin)) ** 0.5
    return w, 0.1 * randn(cout, seed=seed + 1)


def _ref_conv(x64, w, b, scale="none"):
    """Float64 ConvLayer without norm: [up], reflection pad 1, conv (stride 2 for 'down'), + bias.  x64 NCHW float64."""
    if scale == "up":
        x64 = F.interpolate(x64, scale_factor=2, mode="nearest")
    return F.conv2d(F.pad(x64, (1, 1, 1, 1), mode="reflect"), w.double(), b.double(), stride=2 if scale == "down" else 1)


def _faces(res):
    return FACES_512 if res == 512 else list(range(B))


def _x64(x_pm, faces):
    return nchw(x_pm[faces]).double()


@pytest.mark.parametrize("cin,cout,res", [(64, 128, 512), (64, 64, 512), (128, 256, 256), (128, 128, 256), (256, 256, 128),
                                          (256, 256, 64), (256, 256, 32)])
def test_plain_reflect_conv(cin, cout, res):
    from e4s_b200 import kernels as K
    from e4s_b200.encoders.psp_encoders import _conv_planes
    x = randn(B, res, res, cin, seed=cin + res)
    w, b = _weights(cout, cin, seed=7 * cout + res)
    r0 = randn(B, res, res, cout, seed=3)
    y = K.conv3x3_reflect_tc(x, _conv_planes(w), b, lrelu=0.2)
    y2 = K.conv3x3_reflect_tc(x, _conv_planes(w), b, r0=r0)
    f = _faces(res)
    ref = _ref_conv(_x64(x, f), w, b)
    LEDGER.check(y[f], pm(F.leaky_relu(ref, 0.2)), LAYER_TOL, "conv+lrelu", f"{cin}->{cout}@{res}")
    LEDGER.check(y2[f], pm(ref) + r0[f].double(), LAYER_TOL, "conv+r0", f"{cin}->{cout}@{res}")


@pytest.mark.parametrize("cin,cout,res", [(64, 128, 512), (128, 256, 256), (256, 256, 128), (256, 256, 64)])
def test_down_block_stride2_pair(cin, cout, res):
    """A down block: the stride-2 shortcut and the stride-2 conv2 (adding the shortcut) over space-to-depth repacks."""
    from e4s_b200 import kernels as K
    from e4s_b200.encoders.psp_encoders import _conv_planes_s2d
    x = randn(B, res, res, cin, seed=11 + res)
    r = randn(B, res, res, cout, seed=12 + res)
    (ws, bs), (w2, b2) = _weights(cout, cin, seed=13), _weights(cout, cout, seed=17)
    idn = K.conv3x3_reflect_tc(K.space_to_depth(x), _conv_planes_s2d(ws), bs, scale="down")
    y = K.conv3x3_reflect_tc(K.space_to_depth(r), _conv_planes_s2d(w2), b2, r0=idn, scale="down")
    f = _faces(res)
    idn_ref = _ref_conv(_x64(x, f), ws, bs, "down")
    LEDGER.check(idn[f], pm(idn_ref), LAYER_TOL, "stride2", f"{cin}->{cout}@{res}")
    LEDGER.check(y[f], pm(_ref_conv(_x64(r, f), w2, b2, "down") + idn_ref), LAYER_TOL, "stride2+r0", f"{cin}->{cout}@{res}")


@pytest.mark.parametrize("cin,cout,res", [(256, 256, 32), (256, 256, 64), (256, 128, 128), (128, 64, 256)])
def test_up_block_pair(cin, cout, res):
    """An up block: the up-sampling shortcut (bias) and conv1 (LeakyReLU) read the same input, two launches."""
    from e4s_b200 import kernels as K
    from e4s_b200.encoders.psp_encoders import _conv_planes
    x = randn(B, res, res, cin, seed=21 + res)
    (ws, bs), (w1, b1) = _weights(cout, cin, seed=23), _weights(cout, cin, seed=29)
    idn = K.conv3x3_reflect_tc(x, _conv_planes(ws), bs, scale="up")
    r = K.conv3x3_reflect_tc(x, _conv_planes(w1), b1, scale="up", lrelu=0.2)
    f = _faces(2 * res)
    LEDGER.check(idn[f], pm(_ref_conv(_x64(x, f), ws, bs, "up")), LAYER_TOL, "up", f"{cin}->{cout}@{2 * res}")
    LEDGER.check(r[f], pm(F.leaky_relu(_ref_conv(_x64(x, f), w1, b1, "up"), 0.2)), LAYER_TOL, "up+lrelu",
                 f"{cin}->{cout}@{2 * res}")


def test_body_block_and_long_skip():
    from e4s_b200 import kernels as K
    from e4s_b200.encoders.psp_encoders import _conv_planes
    h = randn(B, 32, 32, 256, seed=31)
    feat = randn(B, 32, 32, 256, seed=37)
    (w1, b1), (w2, b2) = _weights(256, 256, seed=41), _weights(256, 256, seed=43)
    r = K.conv3x3_reflect_tc(h, _conv_planes(w1), b1, lrelu=0.2)
    y = K.conv3x3_reflect_tc(r, _conv_planes(w2), b2, r0=h)
    z = K.conv3x3_reflect_tc(r, _conv_planes(w2), b2, r0=h, r1=feat)
    h64 = nchw(h).double()
    r64 = F.leaky_relu(_ref_conv(h64, w1, b1), 0.2)
    y64 = _ref_conv(nchw(r).double(), w2, b2) + h64
    LEDGER.check(r, pm(r64), LAYER_TOL, "conv+lrelu", "body conv1")
    LEDGER.check(y, pm(y64), LAYER_TOL, "conv+r0", "body conv2")
    LEDGER.check(z, pm(y64) + feat.double(), LAYER_TOL, "conv+r0+r1", "long skip")


def test_input_conv_and_heads():
    from e4s_b200 import kernels as K
    x = randn(B, 3, 512, 512, seed=51).clamp(-1, 1)
    w, b = _weights(64, 3, seed=53)
    f = FACES_512
    y = K.conv3x3_rgb_reflect(x, w, b)
    LEDGER.check(y[f], pm(_ref_conv(x[f].double(), w, b)), LAYER_TOL, "rgb in", "encoder.0 3->64@512")
    # process_tensor's input: BGR in [0, 1] at 600 x 560, flipped, * 2 - 1, nearest-resized as encoder.0 reads it
    raw = randn(B, 3, 600, 560, seed=57).sigmoid()
    yp = K.conv3x3_rgb_reflect(raw, w, b, out_hw=(512, 512), prep=True)
    xin = F.interpolate(raw[f].flip(1) * 2 - 1, (512, 512))
    LEDGER.check(yp[f], pm(_ref_conv(xin.double(), w, b)), LAYER_TOL, "rgb in", "encoder.0 prep 600x560")
    feats = randn(B, 512, 512, 64, seed=59)
    wm, bm = _weights(19, 64, seed=61)
    lut = torch.tensor(PO.MASK_COLORMAP, dtype=torch.uint8, device="cuda")
    lg, mk = K.gpen_parse_head(feats, wm, bm, lut, logits=True, mask=torch.int64)
    lg64 = _ref_conv(_x64(feats, f), wm, bm)
    LEDGER.check(lg[f], lg64, LAYER_TOL, "head logits", "out_mask_conv 64->19@512")
    assert torch.equal(mk, PO.to_mask(lg))                       # the mask is the colormap of the logits' argmax
    _, mk8 = K.gpen_parse_head(feats, wm, bm, lut, mask=torch.uint8)
    assert torch.equal(mk8.long(), mk)
    wi, bi = _weights(3, 64, seed=67)
    im = K.conv3x3_rgb_reflect(feats, wi, bi)
    LEDGER.check(im[f], _ref_conv(_x64(feats, f), wi, bi), LAYER_TOL, "rgb out", "out_img_conv 64->3@512")


def test_whole_forward():
    """ParseNet.forward on 16 faces against the float64 oracle (faces 0 and 15), logits and out_img; and the masks of
    process_tensor against the float64 argmax away from ties."""
    from e4s_b200.gpen.face_parse.parse_model import ParseNet
    net = ParseNet(512, 512, 32, 64, 19, norm_type='bn', relu_type='LeakyReLU', ch_range=[32, 256])
    st = PO.synthetic_state()
    net.load_state_dict(st, strict=True)
    net = net.eval().requires_grad_(False).cuda()
    x = torch.cat([PO.process_input(PO.case_image(512, 512, 400 + i)) for i in range(B)]).cuda()
    lg, im = net(x)
    st64 = {k: v.cuda().double() if v.is_floating_point() else v for k, v in st.items()}
    f = FACES_512
    lg64, im64 = PO.parsenet_forward(st64, x[f].double())
    LEDGER.check(lg[f], lg64, FORWARD_TOL, "fwd logits", "ParseNet 16 faces", per_face=True)
    LEDGER.check(im[f], im64, FORWARD_TOL, "fwd out_img", "ParseNet 16 faces", per_face=True)
    err = float((lg[f].double() - lg64).abs().max())
    top2 = lg64.topk(2, dim=1).values
    sure = (top2[:, 0] - top2[:, 1]) > 2 * err
    _, _, mk = net._run(x, logits=False, img=False, mask=torch.int64)
    ref_mask = PO.to_mask(lg64)
    print(f"whole forward: logit error {err:.2e}, pixels within twice of a tie {1 - float(sure.double().mean()):.4%}")
    assert torch.equal(mk[f][sure], ref_mask[sure])
