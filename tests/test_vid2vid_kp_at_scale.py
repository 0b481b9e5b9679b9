"""face-vid2vid's keypoint front end against float64 at the face swap's batch: KPDetector at B = 16 faces, HEEstimator at
2B = 32 (the sources and drivings of 16 pairs).  Each layer form on its own fp32 inputs - the five up blocks and the
keypoint head on the volumetric mode, the five down blocks (3x3 + ReLU + 2x2 average), the reshaping 1x1, HEEstimator's
stem, every bottleneck shape (width 256-2048, stride 1 and 2) and the five heads - then the whole forwards and the driven
keypoints against the oracle run in float64.  The float64 references are plain torch on the GPU, for faces 0 and 15 of
the large layers.  Tolerances are the measured errors (H100 80GB HBM3) with headroom; each test prints what it measured."""
import pytest
import torch
import torch.nn.functional as F

from f64ref import Ledger, at_scale, randn  # noqa: F401
from oracle import vid2vid_kp_oracle as O

pytestmark = pytest.mark.gpu

B = 16
FACES = [0, 15]
LAYER_TOL = 5e-5
VOL_TOL = 2e-4           # K = 27 Cin up to 27648: 9.5e-5 measured at up0
# the whole forwards: HEEstimator's heads read the pooled features' face-to-face deviation, ~0.12 of their magnitude,
# so the ~1e-5 per layer of 56 layers shows up ~8x larger in the bin logits (6.5e-4 measured)
FORWARD_TOL = 1e-3
KP_TOL = 1e-3            # absolute, keypoints in [-1, 1]
LEDGER = Ledger(14)

# (name, cin, cout, input slice side) of the volumetric layers; the keypoint head has no up-sampling and no ReLU
VOLUMETRIC = [("up0", 1024, 512, 2), ("up1", 512, 256, 4), ("up2", 256, 128, 8), ("up3", 128, 64, 16), ("up4", 64, 32, 32),
              ("kp", 32, 15, 64)]


@pytest.mark.parametrize("name,cin,cout,side", VOLUMETRIC)
def test_volumetric_layer(name, cin, cout, side):
    from e4s_b200 import kernels as K
    head = name == "kp"
    x = randn(B, side, side, 16, cin, seed=cin + side).relu()
    w = randn(cout, cin, 3, 3, 3, seed=cout + 1) / (27 * cin) ** 0.5
    b = 0.1 * randn(cout, seed=cout + 2)
    cp = 32 if head else cout
    wp = F.pad(w, (0, 0, 0, 0, 0, 0, 0, 0, 0, cp - cout))
    y = K.conv3d_tc(x, K.conv3d_planes(wp), F.pad(b, (0, cp - cout)).contiguous(), up=not head, relu=not head)
    xr = x[FACES].double().permute(0, 4, 3, 1, 2)                            # [F, C, D, H, W]
    if not head:
        xr = F.interpolate(xr, scale_factor=(1, 2, 2))
    ref = F.conv3d(xr, w.double(), b.double(), padding=1)
    if not head:
        ref = ref.relu()
    LEDGER.check(y[FACES][..., :cout].permute(0, 4, 3, 1, 2), ref, VOL_TOL, "volumetric", name)
    if head:
        assert torch.count_nonzero(y[..., cout:]) == 0


@pytest.mark.parametrize("i", range(5))
def test_down_block(i):
    from e4s_b200 import kernels as K
    cin, cout = O._down_io(i)
    side = 64 >> i
    cpad = 32 if cin == 3 else cin
    x = randn(B, side, side, cpad, seed=i + 40).relu()
    w = randn(cout, cin, 3, 3, seed=i + 41) / (9 * cin) ** 0.5
    b = 0.1 * randn(cout, seed=i + 42)
    wp = F.pad(w, (0, 0, 0, 0, 0, cpad - cin))
    y = K.avgpool2(K.conv3x3_zero_tc(x, K.split_bf16(wp.permute(2, 3, 0, 1).reshape(1, 9, cout, cpad).contiguous()), b,
                                     lrelu=0.0))
    ref = F.avg_pool2d(F.conv2d(x[..., :cin].double().permute(0, 3, 1, 2), w.double(), b.double(), padding=1).relu(), 2)
    LEDGER.check(y.permute(0, 3, 1, 2), ref, LAYER_TOL, "down block", f"down{i}")


def test_reshaping_pointwise():
    from e4s_b200 import kernels as K
    x = randn(B, 2, 2, 1024, seed=50).relu()
    w = randn(16384, 1024, seed=51) / 32
    b = 0.1 * randn(16384, seed=52)
    y = K.conv1x1_tc(x, K.split_bf16(w), b)
    ref = torch.einsum("bhwc,oc->bhwo", x.double(), w.double()) + b.double()
    LEDGER.check(y, ref, LAYER_TOL, "pointwise", "1024->16384 at 2x2")


def test_he_stem():
    from e4s_b200 import kernels as K
    x = torch.rand(2 * B, 3, 256, 256, device="cuda", generator=torch.Generator(device="cuda").manual_seed(60))
    w = randn(64, 3, 7, 7, seed=61) / 147 ** 0.5
    b = 0.1 * randn(64, seed=62)
    y = K.parser_stem(x, w, b)
    ref = F.max_pool2d(F.conv2d(x[FACES].double(), w.double(), b.double(), stride=2, padding=3).relu(), 3, 2, 1)
    LEDGER.check(y[FACES].permute(0, 3, 1, 2), ref, LAYER_TOL, "he stem", "7x7/2 + max-pool")


@pytest.fixture(scope="module")
def he_model():
    from e4s_b200.face_vid2vid.modules.keypoint_detector import HEEstimator
    he = HEEstimator(**O.HE_PARAMS)
    he.load_state_dict(O.he_synthetic_state(), strict=True)
    return he.eval().cuda()


# (module name, in_features, stride, input side) of every distinct bottleneck shape
BOTTLENECKS = [("block1.b1_0", 256, 1, 64), ("block2", 512, 2, 64), ("block3.b3_0", 512, 1, 32), ("block4", 1024, 2, 32),
               ("block5.b5_0", 1024, 1, 16), ("block6", 2048, 2, 16), ("block7.b7_0", 2048, 1, 8)]


@pytest.mark.parametrize("name,cin,stride,side", BOTTLENECKS)
def test_he_bottleneck(he_model, name, cin, stride, side):
    blocks = [d for kind, d in he_model._prepared(torch.device("cuda"))["trunk"] if kind == "res"]
    idx = [n for n, _, _ in O.HE_BLOCKS].index(name)
    x = randn(2 * B, side, side, cin, seed=cin + stride).relu()
    y = he_model._bottleneck(blocks[idx], x)
    st = {k: v.cuda().double() for k, v in O.he_synthetic_state().items() if k.startswith(name + ".")}
    ref = O._res(st, name + ".", x[FACES].double().permute(0, 3, 1, 2), stride)
    LEDGER.check(y[FACES].permute(0, 3, 1, 2), ref, LAYER_TOL, "bottleneck", f"{name} {cin} /{stride}")


def test_he_heads(he_model):
    from e4s_b200 import kernels as K
    pooled = randn(2 * B, 2048, seed=70).relu()
    wh, bh = he_model._prepared(torch.device("cuda"))["heads"]
    y = K.linear(pooled, wh, bh)
    ref = pooled.double() @ wh.double().t() + bh.double()
    LEDGER.check(y, ref, LAYER_TOL, "heads", "2048 -> 248")


@pytest.fixture(scope="module")
def pair_faces():
    return O.synthetic_faces(B, 80).cuda(), O.synthetic_faces(B, 81).cuda()


def test_forwards_and_keypoints(he_model, pair_faces):
    from e4s_b200.face_vid2vid.keypoints import drive_keypoints
    from e4s_b200.face_vid2vid.modules.keypoint_detector import KPDetector
    kp = KPDetector(**O.PARAMS)
    kp.load_state_dict(O.synthetic_state(), strict=True)
    kp = kp.eval().cuda()
    src, drv = pair_faces
    out = drive_keypoints(kp, he_model, src, drv)
    kst = {k: v.cuda().double() for k, v in O.synthetic_state().items()}
    hst = {k: v.cuda().double() for k, v in O.he_synthetic_state().items()}
    canon = torch.cat([O.kp_forward(kst, src[i:i + 4].double())["value"] for i in range(0, B, 4)])
    he = O.he_forward(hst, torch.cat([src, drv]).double())
    for k in ("yaw", "pitch", "roll", "t", "exp"):
        LEDGER.check(torch.cat([out["he_source"][k], out["he_driving"][k]]), he[k], FORWARD_TOL, "he forward", k)
    kerr = float((out["kp_canonical"]["value"].double() - canon).abs().max())
    ks = O.keypoint_transformation(canon, {k: v[:B] for k, v in he.items()})
    kd = O.keypoint_transformation(canon, {k: v[B:] for k, v in he.items()})
    serr = float((out["kp_source"].double() - ks).abs().max())
    derr = float((out["kp_driving"].double() - kd).abs().max())
    print(f"keypoints vs float64: canonical {kerr:.2e}, source {serr:.2e}, driving {derr:.2e} (bar {KP_TOL:.0e})")
    assert max(kerr, serr, derr) < KP_TOL
