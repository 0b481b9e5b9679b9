"""GPEN RetinaFace-R50 kernels against float64 at the face swap's batch: 16 images of 1024 x 1024 (RetinaFaceDetection on the
×4 super-resolved faces).  Each distinct layer form on its own fp32 inputs - every 1x1 shape of the network on the pointwise
kernel (stride 1 and 2, with the bottleneck residual r0, with FPN's up-sampled r_up), the zero-padded 3x3 convolutions at
stride 1 and 2, an SSH module writing its three branches into channel slices of one pitched buffer, the three head launches
into the flat head buffer, the stem - then the whole forward.  The float64 references are plain torch (F.conv2d, einsum,
F.max_pool2d, F.interpolate) on the GPU; at 256 x 256 and above they are computed for faces 0 and 15 only (the kernels
still run on all 16), below for all 16.  Tolerances are the measured errors (H100 80GB HBM3) with headroom; each test prints
what it measured."""
import pytest
import torch
import torch.nn.functional as F

from f64ref import Ledger, at_scale, nchw, pm, randn  # noqa: F401
from oracle import retinaface_oracle as RO

pytestmark = pytest.mark.gpu

B, S = 16, 1024
FACES = [0, 15]
LAYER_TOL = 2e-5          # 1x1, head, stem: <= 9e-6 measured
CONV3_TOL = 4e-5          # 3x3 (K = 9 Cin up to 4608): <= 2.0e-5 measured
FORWARD_TOL = 2e-4
LEDGER = Ledger(12)


def _faces(res):
    return FACES if res >= 256 else list(range(B))


def _pw_ref(x, w, b, faces, stride=1):
    """Float64 1x1 convolution + bias of pixel-major x [B, H, W, Cin] at (stride y, stride x): [F, h, w, Cout]."""
    return torch.einsum("bhwc,oc->bhwo", x[faces, ::stride, ::stride].double(), w.double()) + b.double()


# (cin, cout, output resolution, stride, epilogue term) of every 1x1 convolution of the network at 1024 x 1024:
# bottleneck conv1 (ReLU), conv3 (+ shortcut r0, ReLU), the shortcuts (no activation), FPN laterals (ReLU, + r_up)
POINTWISE = [
    (64, 64, 256, 1, None), (64, 256, 256, 1, "r0"), (64, 256, 256, 1, "shortcut"), (256, 64, 256, 1, None),
    (256, 128, 256, 1, None), (128, 512, 128, 1, "r0"), (256, 512, 128, 2, "shortcut"), (512, 128, 128, 1, None),
    (512, 256, 128, 1, None), (256, 1024, 64, 1, "r0"), (512, 1024, 64, 2, "shortcut"), (1024, 256, 64, 1, None),
    (1024, 512, 64, 1, None), (512, 2048, 32, 1, "r0"), (1024, 2048, 32, 2, "shortcut"), (2048, 512, 32, 1, None),
    (512, 256, 128, 1, "r_up"), (1024, 256, 64, 1, "r_up"), (2048, 256, 32, 1, None),
]


@pytest.mark.parametrize("cin,cout,res,stride,term", POINTWISE)
def test_pointwise(cin, cout, res, stride, term):
    from e4s_b200 import kernels as K
    x = randn(B, res * stride, res * stride, cin, seed=cin + res + stride)
    w = randn(cout, cin, seed=cout + 3) / cin ** 0.5
    b = 0.1 * randn(cout, seed=cout + 5)
    r0 = randn(B, res, res, cout, seed=7) if term == "r0" else None
    up = randn(B, res // 2, res // 2, cout, seed=11) if term == "r_up" else None
    slope = 1.0 if term == "shortcut" else 0.0
    y = K.conv1x1_tc(x, K.split_bf16(w), b, r0=r0, r_up=up, stride=stride, lrelu=slope)
    f = _faces(res)
    ref = _pw_ref(x, w, b, f, stride)
    if r0 is not None:
        ref = ref + r0[f].double()
    if slope == 0.0:
        ref = ref.clamp_min(0)
    if up is not None:
        ref = ref + up[f].double().repeat_interleave(2, 1).repeat_interleave(2, 2)
    LEDGER.check(y[f], ref, LAYER_TOL, f"1x1 {term or 'relu'}", f"{cin}->{cout}@{res}/{stride}")


@pytest.mark.parametrize("c,res,stride", [(64, 256, 1), (128, 128, 1), (256, 64, 1), (512, 32, 1), (256, 128, 1),
                                          (128, 128, 2), (256, 64, 2), (512, 32, 2)])
def test_conv3x3_zero_padded(c, res, stride):
    """Bottleneck conv2 and FPN merges (stride 1), the first conv2 of layer2-4 (stride 2 over space-to-depth)."""
    from e4s_b200 import kernels as K
    from e4s_b200.encoders.psp_encoders import _conv_planes, _conv_planes_s2d
    x = randn(B, res * stride, res * stride, c, seed=c + 17 * stride)
    w = randn(c, c, 3, 3, seed=c + 19) / (9 * c) ** 0.5
    b = 0.1 * randn(c, seed=23)
    if stride == 2:
        y = K.conv3x3_zero_tc(K.space_to_depth(x), _conv_planes_s2d(w), b, stride=2, lrelu=0.0)
    else:
        y = K.conv3x3_zero_tc(x, _conv_planes(w), b, lrelu=0.0)
    f = _faces(res * stride)
    ref = F.conv2d(nchw(x[f]).double(), w.double(), b.double(), stride=stride, padding=1).clamp_min(0)
    LEDGER.check(y[f], pm(ref), CONV3_TOL, f"3x3 /{stride}", f"{c}->{c}@{res}")


@pytest.mark.parametrize("res", [128, 64, 32])
def test_ssh_slices_and_heads(res):
    """An SSH module into one pitched [B, h, w, 256] buffer (conv3X3 -> channels 0-127, conv5X5_2 -> 128-191, conv7x7_3 ->
    192-255, each ReLU'd), then the level's head launch (256 -> 32, bias) into its view of the flat head buffer."""
    from e4s_b200 import kernels as K
    from e4s_b200.encoders.psp_encoders import _conv_planes
    x = randn(B, res, res, 256, seed=res + 29).clamp_min(0)
    ws = {k: (randn(co, ci, 3, 3, seed=31 + i) / (9 * ci) ** 0.5, 0.1 * randn(co, seed=37 + i))
          for i, (k, ci, co) in enumerate((("c3", 256, 128), ("c51", 256, 64), ("c52", 64, 64), ("c72", 64, 64),
                                           ("c73", 64, 64)))}
    P = {k: (_conv_planes(w), b) for k, (w, b) in ws.items()}
    cat = torch.empty(B, res, res, 256, device="cuda")
    K.conv3x3_zero_tc(x, *P["c3"], out=cat[..., :128], lrelu=0.0)
    t5 = K.conv3x3_zero_tc(x, *P["c51"], lrelu=0.0)
    K.conv3x3_zero_tc(t5, *P["c52"], out=cat[..., 128:192], lrelu=0.0)
    t7 = K.conv3x3_zero_tc(t5, *P["c72"], lrelu=0.0)
    K.conv3x3_zero_tc(t7, *P["c73"], out=cat[..., 192:], lrelu=0.0)
    f = _faces(res)
    conv = lambda t, k: F.conv2d(nchw(t[f]).double(), ws[k][0].double(), ws[k][1].double(), padding=1).clamp_min(0)  # noqa: E731
    for sl, inp, k in ((slice(0, 128), x, "c3"), (slice(128, 192), t5, "c52"), (slice(192, 256), t7, "c73")):
        LEDGER.check(cat[f][..., sl], pm(conv(inp, k)), CONV3_TOL, "ssh slice", f"{k}@{res}")
    LEDGER.check(t5[f], pm(conv(x, "c51")), CONV3_TOL, "ssh inner", f"c51@{res}")
    wh, bh = randn(32, 256, seed=41) / 16.0, 0.1 * randn(32, seed=43)
    heads = torch.full((B * 32 * (res * res + 4 * res * res),), float("nan"), device="cuda")
    off = B * 32 * 4 * res * res                           # this level after a preceding one of twice the size
    view = heads[off:off + B * 32 * res * res].view(B, res, res, 32)
    K.conv1x1_tc(cat, K.split_bf16(wh), bh, out=view)
    LEDGER.check(view[f], _pw_ref(cat, wh, bh, f), LAYER_TOL, "head", f"256->32@{res}")
    assert bool(heads[:off].isnan().all()), "the head launch wrote outside its level"


def test_stem():
    from e4s_b200 import kernels as K
    x = randn(B, 3, S, S, seed=47) * 60.0
    w = randn(64, 3, 7, 7, seed=53) / (147 ** 0.5)
    b = 0.1 * randn(64, seed=59)
    y = K.parser_stem(x, w, b)
    ref = F.max_pool2d(F.conv2d(x[FACES].double(), w.double(), b.double(), stride=2, padding=3).clamp_min(0), 3, 2, 1)
    LEDGER.check(y[FACES], pm(ref), LAYER_TOL, "stem", f"7x7/2+pool@{S}")


def test_whole_forward():
    """RetinaFace.forward on 16 seeded 1024 x 1024 images against the float64 restatement (faces 0 and 15), loc, conf and
    landms, each face against its own maximum."""
    from e4s_b200.gpen.face_detect.data import cfg_re50
    from e4s_b200.gpen.face_detect.facemodels.retinaface import RetinaFace
    st = RO.synthetic_state()
    net = RetinaFace(cfg=cfg_re50, phase='test')
    net.load_state_dict(st, strict=True)
    net = net.eval().requires_grad_(False).cuda()
    imgs = torch.stack([torch.from_numpy(RO.case_image(S, S, 200 + i).transpose(2, 0, 1).copy()) for i in range(B)]).cuda()
    from e4s_b200 import kernels as K
    x = K.retinaface_prep(imgs)
    loc, conf, landms = net(x)
    st64 = {k: v.cuda().double() if v.is_floating_point() else v.cuda() for k, v in st.items()}
    r_loc, r_conf, r_lm = RO.forward(st64, x[FACES].double())
    for name, ours, ref in (("fwd loc", loc, r_loc), ("fwd conf", conf, r_conf), ("fwd landms", landms, r_lm)):
        LEDGER.check(ours[FACES], ref, FORWARD_TOL, name, f"RetinaFace {B}x{S}", per_face=True)
