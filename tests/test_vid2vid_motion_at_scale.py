"""face-vid2vid's dense-motion network against float64 at the face swap's batch of B = 16 pairs.  Each kernel on its own fp32
inputs - the front end (compress, then the sampled and heatmap channels), every hourglass layer form on the voxel-pitched
volumetric mode (the five down blocks' convolutions and (1, 2, 2) averages, the five up blocks, the decoder's last
convolution), the per-slice 7x7 GEMM and the combined mask logits - then the whole forward against the oracle run in
float64.  The float64 references are plain torch on the GPU, for pairs 0 and 15.  Tolerances are the measured errors
(H100 80GB HBM3) with headroom; each test prints what it measured."""
import pytest
import torch
import torch.nn.functional as F

from f64ref import Ledger, at_scale, randn  # noqa: F401
from oracle import vid2vid_motion_oracle as O

pytestmark = pytest.mark.gpu

B = 16
PAIRS = [0, 15]
FRONT_TOL = 1e-5
VOL_TOL = 2e-4
GEMM_TOL = 2e-4
OUT_TOL = 1e-3           # absolute: mask and occlusion in [0, 1], deformation in the [-1, 1] grid's units
LEDGER = Ledger(16)

# (name, cin (padded), cout (padded), input slice side, up) of the hourglass's volumetric layers
HOURGLASS = [("down0", 96, 64, 64, False), ("down1", 64, 128, 32, False), ("down2", 128, 256, 16, False),
             ("down3", 256, 512, 8, False), ("down4", 512, 1024, 4, False), ("up0", 1024, 512, 2, True),
             ("up1", 1024, 256, 4, True), ("up2", 512, 128, 8, True), ("up3", 256, 64, 16, True), ("up4", 128, 32, 32, True),
             ("decoder.conv", 128, 128, 64, False)]


def _pairs(t):
    return t[PAIRS]


@pytest.mark.parametrize("name,cin,cout,side,up", HOURGLASS)
def test_hourglass_layer(name, cin, cout, side, up):
    """The layer reads channel slice [cout, cout + cin) of a wider buffer and writes slice [0, cout) of another, as the
    concatenations do; a down block's (1, 2, 2) average follows on its output."""
    from e4s_b200 import kernels as K
    x = randn(B, side, side, 16, cin, seed=cin + side).relu()
    w = randn(cout, cin, 3, 3, 3, seed=cout + 1) / (27 * cin) ** 0.5
    b = 0.1 * randn(cout, seed=cout + 2)
    src = torch.zeros(B, side, side, 16, cout + cin, device="cuda")
    src[..., cout:] = x
    m = 2 if up else 1
    dst = torch.zeros(B, side * m, side * m, 16, 2 * cout, device="cuda")
    K.conv3d_pitched_tc(src[..., cout:], K.conv3d_planes(w), b, out=dst[..., :cout], up=up, relu=True)
    xd = _pairs(x).double().permute(0, 4, 3, 1, 2)
    if up:
        xd = F.interpolate(xd, scale_factor=(1, 2, 2))
    ref = F.relu(F.conv3d(xd, w.double(), b.double(), padding=1))
    got = _pairs(dst[..., :cout]).permute(0, 4, 3, 1, 2)
    LEDGER.check(got, ref, VOL_TOL, "volumetric", name)
    if name.startswith("down"):
        y = dst[..., :cout].contiguous()
        pool = K.avgpool2_vox(y)
        LEDGER.check(_pairs(pool).permute(0, 4, 3, 1, 2), F.avg_pool3d(_pairs(y).double().permute(0, 4, 3, 1, 2), (1, 2, 2)),
                     FRONT_TOL, "pool", name)


def test_front_end():
    from e4s_b200 import kernels as K
    feat = O.synthetic_feature(B, 100).cuda()
    kd, ks = (t.cuda() for t in O.synthetic_keypoints(B, 101))
    wc, bc = randn(4, 32, seed=102) / 32 ** 0.5, 0.1 * randn(4, seed=103)
    comp = K.vid2vid_compress(feat, torch.cat([wc.reshape(-1), bc]))
    ref_comp = F.relu(F.conv3d(_pairs(feat).double(), wc.double().view(4, 32, 1, 1, 1), bc.double()))
    LEDGER.check(_pairs(comp).permute(0, 4, 1, 2, 3), ref_comp, FRONT_TOL, "front end", "compress")
    buf = torch.zeros(B, 64, 64, 16, 128, device="cuda")
    K.vid2vid_motion_input(comp, kd, ks, buf[..., 32:])
    n = len(PAIRS)
    kdp, ksp = _pairs(kd).double(), _pairs(ks).double()
    rep = _pairs(comp).double().permute(0, 4, 1, 2, 3).unsqueeze(1).expand(n, 16, 4, 16, 64, 64).reshape(n * 16, 4, 16, 64, 64)
    deformed = F.grid_sample(rep, O.sparse_motions(kdp, ksp).reshape(n * 16, 16, 64, 64, 3), align_corners=False)
    ref = torch.cat([O.heatmaps(kdp, ksp).unsqueeze(2), deformed.view(n, 16, 4, 16, 64, 64)], 2).view(n, 80, 16, 64, 64)
    LEDGER.check(_pairs(buf[..., 32:112]).permute(0, 4, 3, 1, 2), ref, FRONT_TOL, "front end", "hourglass input")


def test_mask_gemm_and_logits():
    from e4s_b200 import kernels as K
    from e4s_b200.face_vid2vid.modules.dense_motion import gemm_weights
    pred = F.pad(randn(B, 64, 64, 16, 112, seed=110).relu(), (0, 16))
    wm = randn(16, 112, 7, 7, 7, seed=111) / (343 * 112) ** 0.5
    wo = randn(1, 1792, 7, 7, seed=112) / (49 * 1792) ** 0.5
    gw = gemm_weights(wm, wo)
    p = K.conv7x7_slices_tc(pred, K.split_bf16(gw))
    n = len(PAIRS)
    slices = _pairs(pred).double().permute(0, 3, 4, 1, 2).reshape(n * 16, 128, 64, 64)
    ref = F.conv2d(slices, gw.double().permute(1, 2, 0).reshape(128, 128, 7, 7), padding=3)
    LEDGER.check(_pairs(p).reshape(n * 16, 64, 64, 128).permute(0, 3, 1, 2), ref, GEMM_TOL, "7x7 GEMM", "mask / occlusion")
    mb, ob = torch.zeros(16, device="cuda"), torch.zeros(1, device="cuda")
    kd, ks = (t.cuda() for t in O.synthetic_keypoints(B, 113))
    mask, _, _ = K.vid2vid_motion_combine(p, mb, ob, kd, ks)
    pd = _pairs(pred).double().permute(0, 4, 3, 1, 2)[:, :112]
    logits = F.conv3d(pd, wm.double(), padding=3)
    # the mask's log recovers the logits up to a per-voxel constant: compare centred logits
    got = torch.log(_pairs(mask).double())
    LEDGER.check(got - got.mean(1, keepdim=True), logits - logits.mean(1, keepdim=True), GEMM_TOL, "logits", "mask logits")


def test_forward_against_float64_oracle():
    from e4s_b200.face_vid2vid.modules.dense_motion import DenseMotionNetwork
    st = O.synthetic_state()
    net = DenseMotionNetwork(**O.PARAMS)
    net.load_state_dict(st, strict=True)
    net = net.eval().cuda()
    feat = O.synthetic_feature(B, 120).cuda()
    kd, ks = (t.cuda() for t in O.synthetic_keypoints(B, 121))
    out = net(feat, {"value": kd}, {"value": ks})
    for f in PAIRS:
        ref = O.forward(st, feat[f:f + 1].double(), kd[f:f + 1].double(), ks[f:f + 1].double())
        for k in ref:
            err = float((out[k][f:f + 1].double() - ref[k]).abs().max())
            print(f"forward pair {f}: {k} max abs {err:.2e} (bar {OUT_TOL:.0e})")
            LEDGER.note("forward " + k, err, 0.0, f"pair {f}")
            assert err < OUT_TOL, (f, k, err)
