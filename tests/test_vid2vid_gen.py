"""face-vid2vid's occlusion-aware SPADE generator (e4s_b200.face_vid2vid.modules.generator): on the CPU the mirror's
state-dict layout against the reference's (the layout JSON), the oracle against the reference's goldens, the eval-mode
spectral-norm weight, the prepared operands' permutations and gamma / beta interleave, and the drop-in mapping; on the GPU
every new entry against float64 (the SPADE epilogue at both slopes with x at full and at half resolution, the fixed-order
statistics, the warp, the volumetric residual, the pointwise factor and both RGB instantiations), the forward against the
float64 oracle, ``reenact``, a pair's prediction bitwise alone / in a batch of 5 / graph-replayed, the one-device
DataParallel wrapper and bad inputs."""
import json
import os
import sys

import pytest
import torch
import torch.nn.functional as F

from conftest import ROOT

from oracle import golden_io
from oracle import vid2vid_gen_oracle as O
from oracle import vid2vid_kp_oracle as KPO
from oracle import vid2vid_motion_oracle as MO

GOLDEN = os.path.join(ROOT, "tests", "golden", "vid2vid_gen_vectors.npz")
LAYOUT = os.path.join(ROOT, "tests", "golden", "vid2vid_gen_checkpoint_layout.json")
FACE_SEED, KP_SEED = 41, 42
SUB = (slice(None), slice(None), slice(None, None, 4), slice(None, None, 4))


@pytest.fixture(scope="module")
def state():
    return O.synthetic_state()


def _net(state=None):
    from e4s_b200.face_vid2vid.modules.generator import OcclusionAwareSPADEGenerator
    net = OcclusionAwareSPADEGenerator(**O.PARAMS)
    if state is not None:
        net.load_state_dict(state, strict=True)
    return net.eval()


# ------------------------------------------------------------------------------------------------------------ CPU
def test_state_dict_layout_matches_reference(state):
    with open(LAYOUT) as f:
        layout = json.load(f)
    net = _net()
    assert {k: list(v.shape) for k, v in net.state_dict().items()} == layout
    assert {k: list(v.shape) for k, v in state.items()} == layout
    assert len(layout) == 386
    assert sum(k.startswith("dense_motion_network.") for k in layout) == 88
    assert sum(k.startswith("decoder.") for k in layout) == 182
    assert round(sum(p.numel() for p in net.parameters()) / 1e6, 1) == 101.0


def test_oracle_matches_reference_goldens(state):
    g = golden_io.load(GOLDEN)
    src = KPO.synthetic_faces(2, FACE_SEED)
    kd, ks = torch.from_numpy(g["kp_driving"]), torch.from_numpy(g["kp_source"])
    with torch.no_grad():
        out = O.forward(state, src, kd, ks)
    pred = out["prediction"][SUB]
    assert float((pred - torch.from_numpy(g["prediction"])).abs().max()) < 2e-5
    assert float((out["occlusion_map"] - torch.from_numpy(g["occlusion_map"])).abs().max()) < 2e-5


def test_spectral_norm_weight_is_the_eval_mode_weight(state):
    """The prepared weight is torch's eval-mode spectral-norm weight (stored u and v, no power iteration)."""
    from e4s_b200.face_vid2vid.modules.generator import _sn_weight
    net = _net(state)
    blk = net.decoder.up_0
    with torch.no_grad():
        blk.conv_s(torch.zeros(1, 512, 2, 2))                # eval-mode pre-hook sets .weight
        ref = blk.conv_s.weight.double()
    got = _sn_weight(blk.conv_s)
    assert float((got - ref).abs().max() / ref.abs().max()) < 1e-6
    sigma = float(ref.reshape(ref.shape[0], -1).norm() / got.reshape(got.shape[0], -1).norm())
    assert abs(sigma - 1.0) < 1e-6
    assert abs(float(torch.dot(blk.conv_s.weight_u.double(), blk.conv_s.weight_orig.double().reshape(256, -1)
                               @ blk.conv_s.weight_v.double())) - 1.0) > 0.1


def test_prepared_permutations_and_interleave():
    from e4s_b200 import kernels as K
    from e4s_b200.face_vid2vid.modules.generator import _depth_major
    g = torch.Generator().manual_seed(5)
    # second's rows: output channel d 32 + c of the permuted weights is the reference's c 16 + d
    perm = _depth_major(32, 16)
    x = torch.randn(2, 256, 3, 3, generator=g, dtype=torch.float64)
    w = torch.randn(512, 256, 1, 1, generator=g, dtype=torch.float64)
    ref = F.conv2d(x, w).view(2, 32, 16, 3, 3)                                # c, d
    got = F.conv2d(x, w[perm]).view(2, 16, 32, 3, 3)                          # d, c
    assert torch.equal(got.permute(0, 2, 1, 3, 4), ref)
    # third's input channels: the warped operand's channel d 32 + c reads the reference's c 16 + d
    vol = torch.randn(2, 32, 16, 5, 5, generator=g, dtype=torch.float64)
    w3 = torch.randn(8, 512, 3, 3, generator=g, dtype=torch.float64)
    ref = F.conv2d(vol.reshape(2, 512, 5, 5), w3, padding=1)
    got = F.conv2d(vol.permute(0, 2, 1, 3, 4).reshape(2, 512, 5, 5), w3[:, perm], padding=1)
    assert float((got - ref).abs().max()) < 1e-12
    # gamma / beta interleave: row 2 k is gamma k, row 2 k + 1 beta k
    wg, wb = torch.randn(64, 128, 3, 3, generator=g), torch.randn(64, 128, 3, 3, generator=g)
    planes = K.spade_planes(wg, wb).float()
    full = (planes[0] + planes[1])[0]                                          # [9, 128, 128]: tap, row, cin
    assert float((full[:, 0::2] - wg.permute(2, 3, 0, 1).reshape(9, 64, 128)).abs().max()) < 1e-5 * float(wg.abs().max())
    assert float((full[:, 1::2] - wb.permute(2, 3, 0, 1).reshape(9, 64, 128)).abs().max()) < 1e-5 * float(wb.abs().max())


def test_dropin_maps_the_generator_module():
    from e4s_b200 import dropin
    dropin.install()
    import e4s_b200.face_vid2vid.modules.generator as M
    assert sys.modules["src.pretrained.face_vid2vid.modules.generator"] is M
    assert M.OcclusionAwareSPADEGenerator and M.OcclusionAwareGenerator
    with pytest.raises(NotImplementedError):
        M.OcclusionAwareGenerator(**O.PARAMS)


# ------------------------------------------------------------------------------------------------------------ GPU
def _rel(a, b):
    return float((a.double() - b.double()).abs().max() / b.double().abs().max().clamp_min(1e-30))


def _planes(w):
    from e4s_b200 import kernels as K
    return K.split_bf16(w.float().permute(2, 3, 0, 1).reshape(1, 9, w.shape[0], w.shape[1]).contiguous()).cuda()


@pytest.mark.gpu
@pytest.mark.parametrize("b,h,c,half,slope", [(2, 16, 64, False, 0.2), (1, 32, 32, True, 0.2), (2, 16, 128, True, 1.0),
                                              (1, 8, 512, False, 1.0)])
def test_spade_epilogue_matches_float64(b, h, c, half, slope):
    """The gamma / beta GEMM over a 128-channel slice of a wider buffer, its epilogue applying the modulation to x (at
    full or half resolution, with its fixed-order statistics) and the activation, against float64."""
    from e4s_b200 import kernels as K
    g = torch.Generator().manual_seed(h * 7 + c)
    hx = h // 2 if half else h
    x = (torch.randn(b, hx, hx, c, generator=g) * 2.0 + 0.5).cuda()
    buf = torch.randn(b, h, h, 384, generator=g).relu().cuda()
    actv = buf[..., 128:256]
    wg = torch.randn(c, 128, 3, 3, generator=g) / (9 * 128) ** 0.5
    wb = torch.randn(c, 128, 3, 3, generator=g) / (9 * 128) ** 0.5
    bg, bb = 0.1 * torch.randn(c, generator=g), 0.1 * torch.randn(c, generator=g)
    scale, shift = K.instnorm_stats(x)
    out = K.spade_tc(actv, K.spade_planes(wg, wb).cuda(), torch.stack([bg, bb], 1).reshape(-1).cuda(), x, scale, shift, slope)
    xd = x.double().permute(0, 3, 1, 2)
    if half:
        xd = F.interpolate(xd, scale_factor=2)
    ad = actv.double().permute(0, 3, 1, 2)
    gamma = F.conv2d(ad, wg.double().cuda(), bg.double().cuda(), padding=1)
    beta = F.conv2d(ad, wb.double().cuda(), bb.double().cuda(), padding=1)
    ref = F.leaky_relu(F.instance_norm(xd, eps=1e-5) * (1 + gamma) + beta, slope)
    err = _rel(out.permute(0, 3, 1, 2), ref)
    print(f"spade b={b} {h}^2 c={c} half={half} slope={slope}: max-rel {err:.2e}")
    assert err < 2e-5


@pytest.mark.gpu
def test_instnorm_stats_fixed_order():
    """Statistics of a pitched slice against float64, and bit identical for a sample alone and inside a batch."""
    from e4s_b200 import kernels as K
    g = torch.Generator().manual_seed(3)
    buf = (torch.randn(3, 40, 72, 96, generator=g) * 3.0 + 2.0).cuda()
    x = buf[..., 16:80]
    scale, shift = K.instnorm_stats(x)
    xd = x.double()
    var = xd.var((1, 2), unbiased=False)
    rs = 1 / torch.sqrt(var + 1e-5)
    assert _rel(scale, rs) < 1e-6
    assert _rel(shift, -xd.mean((1, 2)) * rs) < 1e-6
    s1, t1 = K.instnorm_stats(x[1:2])
    assert torch.equal(s1[0], scale[1]) and torch.equal(t1[0], shift[1])


@pytest.mark.gpu
@pytest.mark.parametrize("b", [1, 2])
def test_warp_matches_float64(b):
    """deform_input against F.grid_sample in float64 (deformations reaching past +-1 put corners outside the volume)."""
    from e4s_b200 import kernels as K
    g = torch.Generator().manual_seed(20 + b)
    vol = torch.randn(b, 64, 64, 16, 32, generator=g)
    deform = torch.rand(b, 16, 64, 64, 3, generator=g) * 2.3 - 1.15
    got = K.vid2vid_warp(vol.cuda(), deform.cuda()).cpu().view(b, 64, 64, 16, 32)
    ref = F.grid_sample(vol.double().permute(0, 4, 3, 1, 2), deform.double(), align_corners=False)    # [B, 32, 16, 64, 64]
    err = _rel(got.permute(0, 4, 3, 1, 2), ref)
    print(f"warp B={b}: max-rel {err:.2e}")
    assert err < 1e-5


@pytest.mark.gpu
def test_conv3d_residual_matches_float64():
    from e4s_b200 import kernels as K
    g = torch.Generator().manual_seed(8)
    x = torch.randn(2, 16, 16, 16, 32, generator=g)
    r = torch.randn(2, 16, 16, 16, 32, generator=g)
    wt = torch.randn(32, 32, 3, 3, 3, generator=g) / (27 * 32) ** 0.5
    bias = 0.1 * torch.randn(32, generator=g)
    for relu in (False, True):
        y = K.conv3d_residual_tc(x.cuda(), K.conv3d_planes(wt).cuda(), bias.cuda(), r.cuda(), relu=relu).cpu()
        ref = F.conv3d(x.double().permute(0, 4, 3, 1, 2), wt.double(), bias.double(), padding=1) + r.double().permute(0, 4, 3, 1, 2)
        ref = F.relu(ref) if relu else ref
        err = _rel(y.permute(0, 4, 3, 1, 2), ref)
        print(f"conv3d residual relu={relu}: max-rel {err:.2e}")
        assert err < 2e-5


@pytest.mark.gpu
def test_conv1x1_factor_and_up_conv_match_float64():
    """The pointwise mode times a per-pixel factor over a pitched input, and the zero-padded plain mode over the nearest
    2x and 4x up-sampling of a pitched input."""
    from e4s_b200 import kernels as K
    g = torch.Generator().manual_seed(9)
    buf = torch.randn(2, 16, 16, 320, generator=g).cuda()
    x = buf[..., 32:288]
    w = torch.randn(64, 256, generator=g) / 16.0
    bias = 0.1 * torch.randn(64, generator=g)
    fac = torch.rand(2, 1, 16, 16, generator=g)
    y = K.conv1x1_factor_tc(x, K.split_bf16(w).cuda(), bias.cuda(), fac.cuda())
    ref = (F.conv2d(x.double().permute(0, 3, 1, 2), w.double().cuda().view(64, 256, 1, 1), bias.double().cuda())
           * fac.double().cuda())
    assert _rel(y.permute(0, 3, 1, 2), ref) < 2e-5
    wc = torch.randn(128, 256, 3, 3, generator=g) / (9 * 256) ** 0.5
    for up in (2, 4):
        y = K.conv3x3_zero_up_tc(x, _planes(wc), bias.repeat(2).cuda(), up=up, lrelu=0.0)
        ref = F.relu(F.conv2d(F.interpolate(x.double().permute(0, 3, 1, 2), scale_factor=up), wc.double().cuda(),
                              bias.repeat(2).double().cuda(), padding=1))
        err = _rel(y.permute(0, 3, 1, 2), ref)
        print(f"zero-padded conv over the {up}x up-sampling: max-rel {err:.2e}")
        assert err < 2e-5


@pytest.mark.gpu
def test_rgb_instantiations_match_float64():
    from e4s_b200 import kernels as K
    g = torch.Generator().manual_seed(10)
    img = torch.rand(2, 3, 40, 136, generator=g)
    w, b = torch.randn(64, 3, 3, 3, generator=g) / 5.0, 0.1 * torch.randn(64, generator=g)
    y = K.conv3x3_rgb_act(img.cuda(), w.cuda(), b.cuda())
    ref = F.relu(F.conv2d(img.double(), w.double(), b.double(), padding=1))
    assert _rel(y.cpu().permute(0, 3, 1, 2), ref) < 1e-6
    buf = torch.randn(2, 40, 136, 96, generator=g).cuda()
    w2, b2 = torch.randn(3, 64, 3, 3, generator=g) / 24.0, 0.1 * torch.randn(3, generator=g)
    y = K.conv3x3_rgb_act(buf[..., 8:72], w2.cuda(), b2.cuda())
    ref = torch.sigmoid(F.conv2d(buf[..., 8:72].double().permute(0, 3, 1, 2).cpu(), w2.double(), b2.double(), padding=1))
    assert _rel(y.cpu(), ref) < 1e-6


@pytest.fixture(scope="module")
def gpu_net(state):
    return _net(state).cuda()


def _inputs(b, seed):
    src = KPO.synthetic_faces(b, seed).cuda()
    kd, ks = (t.cuda() for t in MO.synthetic_keypoints(b, seed + 1))
    return src, kd, ks


def _run(net, src, kd, ks):
    with torch.no_grad():
        return net(src, {"value": kd}, {"value": ks})


def run_with_motion(net, src, kd, ks):
    """The forward's outputs and the dense-motion network's (captured by a hook)."""
    seen = {}
    h = net.dense_motion_network.register_forward_hook(lambda m, args, out: seen.update(out))
    try:
        out = _run(net, src, kd, ks)
    finally:
        h.remove()
    return out, seen


@pytest.mark.gpu
def test_forward_matches_float64_oracle(gpu_net, state):
    """The generator around its own dense motion against the float64 oracle around the same motion (bar 1e-3), the mask
    and occlusion map against the float64 oracle (1e-3), and the prediction end to end (3e-2: the stand-in's feature
    volume is rough, and the dense-motion network's fp32 deformation error of ~6e-4 grid units moves the warped
    features by ~3e-2)."""
    src, kd, ks = _inputs(2, FACE_SEED)
    out, motion = run_with_motion(gpu_net, src, kd, ks)
    with torch.no_grad():
        ref = O.forward(state, src.double(), kd.double(), ks.double())
        own = O.forward(state, src.double(), kd.double(), ks.double(), motion={k: v.double() for k, v in motion.items()})
    err = float((out["prediction"].double() - own["prediction"]).abs().max())
    print(f"forward prediction around its own dense motion: max-abs {err:.2e}")
    assert err < 1e-3
    for k, bar in (("mask", 1e-3), ("occlusion_map", 1e-3), ("prediction", 3e-2)):
        err = float((out[k].double() - ref[k]).abs().max())
        print(f"forward {k} end to end: max-abs {err:.2e}")
        assert tuple(out[k].shape) == tuple(ref[k].shape)
        assert err < bar, k


@pytest.mark.gpu
def test_prediction_bitwise_alone_batch_graph(gpu_net):
    src, kd, ks = _inputs(5, 60)
    batch = _run(gpu_net, src, kd, ks)["prediction"]
    alone = _run(gpu_net, src[2:3].contiguous(), kd[2:3].contiguous(), ks[2:3].contiguous())["prediction"]
    s, d, k = src[:1].clone(), kd[:1].clone(), ks[:1].clone()
    _run(gpu_net, s, d, k)                                                    # warm-up, prepares the weights
    graph = torch.cuda.CUDAGraph()
    with torch.no_grad(), torch.cuda.graph(graph):
        out = gpu_net(s, {"value": d}, {"value": k})["prediction"]
    s.copy_(src[2:3]), d.copy_(kd[2:3]), k.copy_(ks[2:3])
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(alone[0], batch[2])
    assert torch.equal(out[0], batch[2])


@pytest.mark.gpu
def test_data_parallel_one_device(gpu_net):
    src, kd, ks = _inputs(2, 70)
    ref = _run(gpu_net, src, kd, ks)
    out = _run(torch.nn.DataParallel(gpu_net, device_ids=[0]), src, kd, ks)
    for k in ref:
        assert torch.equal(out[k], ref[k]), k


@pytest.mark.gpu
def test_reenact_is_drive_keypoints_then_the_generator(gpu_net):
    from e4s_b200.face_vid2vid.keypoints import drive_keypoints, reenact
    from e4s_b200.face_vid2vid.modules.keypoint_detector import HEEstimator, KPDetector
    kp_detector = KPDetector(**KPO.PARAMS).cuda().eval()
    kp_detector.load_state_dict(KPO.synthetic_state(), strict=True)
    he_estimator = HEEstimator(**KPO.HE_PARAMS).cuda().eval()
    he_estimator.load_state_dict(KPO.he_synthetic_state(), strict=True)
    src, drv = KPO.synthetic_faces(2, 80).cuda(), KPO.synthetic_faces(2, 81).cuda()
    with torch.no_grad():
        pred = reenact(kp_detector, he_estimator, gpu_net, src, drv)
        kp = drive_keypoints(kp_detector, he_estimator, src, drv)
        ref = gpu_net(src, {"value": kp["kp_driving"]}, {"value": kp["kp_source"]})["prediction"]
    assert torch.equal(pred, ref)
    assert float(pred.min()) >= 0.0 and float(pred.max()) <= 1.0


@pytest.mark.gpu
def test_bad_inputs_raise(gpu_net, state):
    src, kd, ks = _inputs(1, 90)
    with pytest.raises(NotImplementedError):
        _run(gpu_net, src[..., :128, :128].contiguous(), kd, ks)
    with pytest.raises(NotImplementedError):
        _run(gpu_net, src.cpu(), kd, ks)
    with torch.no_grad(), pytest.raises(NotImplementedError):
        gpu_net(src, {"value": kd, "jacobian": torch.zeros(1, 15, 3, 3, device="cuda")}, {"value": ks})
    with pytest.raises(NotImplementedError):
        gpu_net(src.clone().requires_grad_(), {"value": kd}, {"value": ks})
    gpu_net.train()
    try:
        with pytest.raises(NotImplementedError):
            _run(gpu_net, src, kd, ks)
    finally:
        gpu_net.eval()
    from e4s_b200.face_vid2vid.modules.generator import OcclusionAwareSPADEGenerator
    other = OcclusionAwareSPADEGenerator(**dict(O.PARAMS, num_resblocks=2)).eval().cuda()
    with pytest.raises(NotImplementedError):
        _run(other, src, kd, ks)
