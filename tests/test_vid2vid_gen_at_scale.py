"""face-vid2vid's SPADE generator against float64 at the face swap's batch of B = 16 pairs.  Each new kernel form on its own
fp32 inputs at the generator's shapes - the volumetric residual (resblocks_3d's conv2), the warp (deform_input), the
pointwise factor (fourth x occlusion), the mlp_shared GEMMs over the up-sampled seg map at 128^2 and 256^2, the fixed-order
instance-norm statistics, every SPADE gamma / beta GEMM with its epilogue (G_middle at 64^2, up_0 at 128^2, up_1 at 256^2,
x at half resolution in the up blocks) and both RGB convolutions - then the whole forward against the oracle run in
float64.  The float64 references are plain torch on the GPU, for pairs 0 and 15.  Tolerances: 2e-4 max-rel per layer,
1e-3 absolute on the prediction of the generator around its own dense motion (the float64 oracle fed the same mask,
deformation and occlusion map) and on the mask and occlusion map end to end; 3e-2 on the prediction end to end, where
the dense-motion network's fp32 deformation error (~6e-4 grid units) moves the stand-in's rough feature volume.  Each
test prints what it measured."""
import pytest
import torch
import torch.nn.functional as F

from f64ref import Ledger, at_scale, randn  # noqa: F401
from oracle import vid2vid_gen_oracle as O
from oracle import vid2vid_kp_oracle as KPO
from oracle import vid2vid_motion_oracle as MO

pytestmark = pytest.mark.gpu

B = 16
PAIRS = [0, 15]
LAYER_TOL = 2e-4
OUT_TOL = 1e-3           # absolute, on the prediction in [0, 1]
E2E_TOL = 3e-2           # absolute, the prediction end to end (see above)
LEDGER = Ledger(16)


def _pairs(t):
    return t[PAIRS]


def _planes(w):
    from e4s_b200 import kernels as K
    return K.split_bf16(w.float().permute(2, 3, 0, 1).reshape(1, 9, w.shape[0], w.shape[1]).contiguous())


def test_volume_layers():
    """resblocks_3d's conv2 with the residual, then deform_input's warp of the result."""
    from e4s_b200 import kernels as K
    x = randn(B, 64, 64, 16, 32, seed=1).relu()
    r = randn(B, 64, 64, 16, 32, seed=2)
    w = randn(32, 32, 3, 3, 3, seed=3) / (27 * 32) ** 0.5
    b = 0.1 * randn(32, seed=4)
    y = K.conv3d_residual_tc(x, K.conv3d_planes(w), b, r)
    ref = (F.conv3d(_pairs(x).double().permute(0, 4, 3, 1, 2), w.double(), b.double(), padding=1)
           + _pairs(r).double().permute(0, 4, 3, 1, 2))
    LEDGER.check(_pairs(y).permute(0, 4, 3, 1, 2), ref, LAYER_TOL, "volumetric", "resblock conv2 + residual")
    deform = torch.rand(B, 16, 64, 64, 3, device="cuda", generator=torch.Generator("cuda").manual_seed(5)) * 2.2 - 1.1
    warped = K.vid2vid_warp(y, deform).view(B, 64, 64, 16, 32)
    ref = F.grid_sample(_pairs(y).double().permute(0, 4, 3, 1, 2), _pairs(deform).double(), align_corners=False)
    LEDGER.check(_pairs(warped).permute(0, 4, 3, 1, 2), ref, LAYER_TOL, "warp", "deform_input")


def test_fourth_times_occlusion():
    from e4s_b200 import kernels as K
    x = randn(B, 64, 64, 256, seed=10).relu()
    w = randn(256, 256, seed=11) / 16.0
    b = 0.1 * randn(256, seed=12)
    occ = torch.sigmoid(randn(B, 1, 64, 64, seed=13))
    y = K.conv1x1_factor_tc(x, K.split_bf16(w), b, occ)
    ref = F.conv2d(_pairs(x).double().permute(0, 3, 1, 2), w.double().view(256, 256, 1, 1), b.double()) * _pairs(occ).double()
    LEDGER.check(_pairs(y).permute(0, 3, 1, 2), ref, LAYER_TOL, "pointwise", "fourth x occlusion")


@pytest.mark.parametrize("up", [2, 4])
def test_mlp_shared_over_the_upsampled_seg(up):
    from e4s_b200 import kernels as K
    seg = randn(B, 64, 64, 256, seed=20)
    w = randn(384, 256, 3, 3, seed=21) / (9 * 256) ** 0.5
    b = 0.1 * randn(384, seed=22)
    y = K.conv3x3_zero_up_tc(seg, _planes(w), b, up=up, lrelu=0.0)
    ref = F.relu(F.conv2d(F.interpolate(_pairs(seg).double().permute(0, 3, 1, 2), scale_factor=up), w.double(), b.double(),
                          padding=1))
    LEDGER.check(_pairs(y).permute(0, 3, 1, 2), ref, LAYER_TOL, "mlp_shared", f"{64 * up}^2")


# (name, output side, C, x at half resolution, slope, pitch of the mlp_shared buffer)
SPADES = [("G_middle.norm_0", 64, 512, False, 0.2, 1536), ("up_0.norm_s", 128, 512, True, 1.0, 384),
          ("up_0.norm_1", 128, 256, False, 0.2, 384), ("up_1.norm_0", 256, 256, True, 0.2, 384),
          ("up_1.norm_1", 256, 64, False, 0.2, 384)]


@pytest.mark.parametrize("name,side,c,half,slope,ld", SPADES)
def test_spade(name, side, c, half, slope, ld):
    """The statistics of x, then the gamma / beta GEMM over a 128-channel slice of the mlp_shared buffer with the SPADE
    epilogue, at the generator's shapes."""
    from e4s_b200 import kernels as K
    hx = side // 2 if half else side
    x = randn(B, hx, hx, c, seed=side + c) * 1.5 + 0.3
    buf = randn(B, side, side, ld, seed=side + 1).relu()
    actv = buf[..., 128:256]
    wg, wb = randn(c, 128, 3, 3, seed=c + 2) / 34.0, randn(c, 128, 3, 3, seed=c + 3) / 34.0
    bg, bb = 0.1 * randn(c, seed=c + 4), 0.1 * randn(c, seed=c + 5)
    scale, shift = K.instnorm_stats(x)
    xd = _pairs(x).double()
    var = xd.var((1, 2), unbiased=False)
    LEDGER.check(_pairs(scale), 1 / torch.sqrt(var + 1e-5), LAYER_TOL, "statistics", name + " scale")
    y = K.spade_tc(actv, K.spade_planes(wg, wb), torch.stack([bg, bb], 1).reshape(-1), x, scale, shift, slope)
    xd = xd.permute(0, 3, 1, 2)
    if half:
        xd = F.interpolate(xd, scale_factor=2)
    ad = _pairs(actv).double().permute(0, 3, 1, 2)
    gamma = F.conv2d(ad, wg.double(), bg.double(), padding=1)
    beta = F.conv2d(ad, wb.double(), bb.double(), padding=1)
    ref = F.leaky_relu(F.instance_norm(xd, eps=1e-5) * (1 + gamma) + beta, slope)
    LEDGER.check(_pairs(y).permute(0, 3, 1, 2), ref, LAYER_TOL, "SPADE", name)


def test_rgb_convolutions():
    from e4s_b200 import kernels as K
    img = torch.rand(B, 3, 256, 256, device="cuda", generator=torch.Generator("cuda").manual_seed(30))
    w, b = randn(64, 3, 3, 3, seed=31) / 5.0, 0.1 * randn(64, seed=32)
    y = K.conv3x3_rgb_act(img, w, b)
    LEDGER.check(_pairs(y).permute(0, 3, 1, 2), F.relu(F.conv2d(_pairs(img).double(), w.double(), b.double(), padding=1)),
                 LAYER_TOL, "RGB", "first")
    x = randn(B, 256, 256, 64, seed=33)
    w2, b2 = randn(3, 64, 3, 3, seed=34) / 24.0, 0.1 * randn(3, seed=35)
    y = K.conv3x3_rgb_act(x, w2, b2)
    ref = torch.sigmoid(F.conv2d(_pairs(x).double().permute(0, 3, 1, 2), w2.double(), b2.double(), padding=1))
    LEDGER.check(_pairs(y), ref, LAYER_TOL, "RGB", "conv_img")


def test_forward_against_float64_oracle():
    from e4s_b200.face_vid2vid.modules.generator import OcclusionAwareSPADEGenerator
    st = O.synthetic_state()
    net = OcclusionAwareSPADEGenerator(**O.PARAMS)
    net.load_state_dict(st, strict=True)
    net = net.eval().cuda()
    src = KPO.synthetic_faces(B, 120).cuda()
    kd, ks = (t.cuda() for t in MO.synthetic_keypoints(B, 121))
    from test_vid2vid_gen import run_with_motion
    out, motion = run_with_motion(net, src, kd, ks)
    with torch.no_grad():
        for f in PAIRS:
            args = (st, src[f:f + 1].double(), kd[f:f + 1].double(), ks[f:f + 1].double())
            own = O.forward(*args, motion={k: v[f:f + 1].double() for k, v in motion.items()})
            err = float((out["prediction"][f:f + 1].double() - own["prediction"]).abs().max())
            print(f"forward pair {f}: prediction around its own dense motion max abs {err:.2e} (bar {OUT_TOL:.0e})")
            LEDGER.note("forward prediction (own motion)", err, 0.0, f"pair {f}")
            assert err < OUT_TOL, (f, err)
            ref = O.forward(*args)
            for k in ref:
                bar = E2E_TOL if k == "prediction" else OUT_TOL
                err = float((out[k][f:f + 1].double() - ref[k]).abs().max())
                print(f"forward pair {f}: {k} end to end max abs {err:.2e} (bar {bar:.0e})")
                LEDGER.note("forward " + k, err, 0.0, f"pair {f}")
                assert err < bar, (f, k, err)
