"""face-vid2vid's dense-motion network (e4s_b200.face_vid2vid.modules.dense_motion): on the CPU the mirror's state-dict
layout against the reference's (the layout JSON), the oracle against the reference's goldens, the prepared operands
re-contracted in float64 against F.conv3d / F.conv2d (the 80 -> 96 and 112 -> 128 padding, the (dz, o) / occlusion column
packing of the per-slice GEMM and the c 16 + d channel order) and the drop-in mapping; on the GPU every new entry against
float64 (depth edges, samples outside the volume, B = 1 and 2), a NaN-guarded direct call of each pitched write, the
forward against the goldens and the oracle, a pair's outputs bitwise alone / in a batch / graph-replayed, the one-device
DataParallel wrapper and bad inputs."""
import json
import os
import sys

import pytest
import torch
import torch.nn.functional as F

from conftest import ROOT

from oracle import golden_io
from oracle import vid2vid_motion_oracle as O

GOLDEN = os.path.join(ROOT, "tests", "golden", "vid2vid_motion_vectors.npz")
LAYOUT = os.path.join(ROOT, "tests", "golden", "vid2vid_motion_checkpoint_layout.json")
FEATURE_SEED, KP_SEED = 31, 32
SUB = (slice(None), slice(None), slice(None, None, 4), slice(None, None, 4), slice(None, None, 4))


@pytest.fixture(scope="module")
def gold():
    return golden_io.load(GOLDEN)


@pytest.fixture(scope="module")
def state():
    return O.synthetic_state()


def _net():
    from e4s_b200.face_vid2vid.modules.dense_motion import DenseMotionNetwork
    return DenseMotionNetwork(**O.PARAMS)


def _checksums(f):
    x = f.double().reshape(f.shape[0], -1)
    wgt = (torch.arange(x.shape[1], dtype=torch.float64) % 7) - 3
    return torch.stack([x.sum(1), (x * x).sum(1), (x * wgt).sum(1)], 1)


def _golden_inputs(g):
    feat = O.synthetic_feature(2, FEATURE_SEED)
    assert torch.allclose(_checksums(feat), torch.from_numpy(g["feature_checksums"]), rtol=1e-9, atol=1e-6)
    return feat, torch.from_numpy(g["kp_driving"]), torch.from_numpy(g["kp_source"])


# ------------------------------------------------------------------------------------------------------------ CPU
def test_state_dict_layout_matches_reference(state):
    with open(LAYOUT) as f:
        layout = json.load(f)
    net = _net()
    assert {k: list(v.shape) for k, v in net.state_dict().items()} == layout
    assert {k: list(v.shape) for k, v in state.items()} == layout
    net.load_state_dict(state, strict=True)
    assert len(layout) == 88
    assert round(sum(p.numel() for p in net.parameters()) / 1e6, 1) == 43.5


def test_oracle_matches_reference_golden(gold, state):
    feat, kd, ks = _golden_inputs(gold)
    with torch.no_grad():
        out = O.forward(state, feat, kd, ks)
    for name, got in (("mask_sub", out["mask"][SUB]), ("deformation_sub", out["deformation"][SUB[:4]]),
                      ("occlusion_map", out["occlusion_map"])):
        err = float((got - torch.from_numpy(gold[name])).abs().max())
        print(f"oracle vs reference {name}: max abs {err:.2e}")
        assert err < 2e-5, name


def test_prepared_operands_recontract_to_the_convolutions():
    """The per-slice GEMM weights and the padded volumetric planes, contracted in float64 as the kernels contract them,
    against the reference's convolutions on small tensors."""
    from e4s_b200 import kernels as K
    from e4s_b200.face_vid2vid.modules.dense_motion import gemm_weights
    g = torch.Generator().manual_seed(5)
    c, d, h, w = O.OUT_CH, 16, 5, 6
    pred = torch.randn(1, c, d, h, w, generator=g, dtype=torch.float64)
    wm = torch.randn(16, c, 7, 7, 7, generator=g, dtype=torch.float64)
    wo = torch.randn(1, c * d, 7, 7, generator=g, dtype=torch.float64)
    gw = gemm_weights(wm, wo)                                                  # [49, 128, 128]
    assert tuple(gw.shape) == (49, 128, 128) and not bool(gw[:, :, c:].any())
    x = F.pad(pred, (0, 0, 0, 0, 0, 0, 0, 128 - c))                            # channels 112 -> 128
    slices = x.permute(0, 2, 1, 3, 4).reshape(d, 128, h, w)                    # [D, C, h, w]
    p = F.conv2d(slices, gw.permute(1, 2, 0).reshape(128, 128, 7, 7), padding=3)   # [D, 128, h, w]
    logits = torch.zeros(16, d, h, w, dtype=torch.float64)
    for z in range(d):
        for dz in range(7):
            if 0 <= z + dz - 3 < d:
                logits[:, z] += p[z + dz - 3, 16 * dz:16 * dz + 16]
    ref = F.conv3d(pred, wm, padding=3)[0]
    assert float((logits - ref).abs().max() / ref.abs().max()) < 1e-12
    occ = sum(p[z, 112 + z] for z in range(d))
    ref = F.conv2d(pred.reshape(1, c * d, h, w), wo, padding=3)[0, 0]
    assert float((occ - ref).abs().max() / ref.abs().max()) < 1e-12
    # down0's weights zero-padded 80 -> 96 input channels: the planes hold the weights (hi + lo) and zeros
    w0 = torch.randn(64, O.IN_CH, 3, 3, 3, generator=g)
    planes = K.conv3d_planes(F.pad(w0, (0, 0, 0, 0, 0, 0, 0, 16))).float()
    full = (planes[0] + planes[1]).reshape(3, 3, 64, 3, 96)                   # ky, kx, o, kz, c
    assert float((full[..., :O.IN_CH].permute(2, 4, 3, 0, 1) - w0).abs().max()) < 1e-5 * float(w0.abs().max())
    assert not bool(full[..., O.IN_CH:].any())


def test_dropin_maps_the_dense_motion_module():
    from e4s_b200 import dropin
    dropin.install()
    import e4s_b200.face_vid2vid.modules.dense_motion as M
    assert sys.modules["src.pretrained.face_vid2vid.modules.dense_motion"] is M
    assert M.DenseMotionNetwork


# ------------------------------------------------------------------------------------------------------------ GPU
def _rel(a, b):
    return float((a.double() - b.double()).abs().max() / b.double().abs().max().clamp_min(1e-30))


def _nan_buffer(shape):
    return torch.full(shape, float("nan"), device="cuda")


@pytest.mark.gpu
@pytest.mark.parametrize("b", [1, 2])
def test_front_end_matches_float64(b):
    """compress, then the hourglass input written into channels 32..127 of a NaN-filled 128-channel buffer: channels 0..31
    stay NaN, the rest matches float64 (keypoints near and beyond +-1 put corners outside the volume)."""
    from e4s_b200 import kernels as K
    g = torch.Generator().manual_seed(40 + b)
    feat = O.synthetic_feature(b, 50 + b)
    kd, ks = O.synthetic_keypoints(b, 60 + b)
    wc = torch.randn(4, 32, generator=g) / 32 ** 0.5
    bc = 0.1 * torch.randn(4, generator=g)
    ref_comp = F.relu(F.conv3d(feat.double(), wc.double().view(4, 32, 1, 1, 1), bc.double()))
    comp = K.vid2vid_compress(feat.cuda(), torch.cat([wc.reshape(-1), bc]).cuda())
    assert _rel(comp.cpu().permute(0, 4, 1, 2, 3), ref_comp) < 1e-6
    buf = _nan_buffer((b, 64, 64, 16, 128))
    K.vid2vid_motion_input(comp, kd.cuda(), ks.cuda(), buf[..., 32:])
    torch.cuda.synchronize()
    assert bool(buf[..., :32].isnan().all())
    motions = O.sparse_motions(kd.double(), ks.double())
    rep = comp.cpu().double().permute(0, 4, 1, 2, 3).unsqueeze(1).expand(b, 16, 4, 16, 64, 64).reshape(b * 16, 4, 16, 64, 64)
    deformed = F.grid_sample(rep, motions.reshape(b * 16, 16, 64, 64, 3), align_corners=False).view(b, 16, 4, 16, 64, 64)
    ref = torch.cat([O.heatmaps(kd.double(), ks.double()).unsqueeze(2), deformed], 2).view(b, 80, 16, 64, 64)
    got = buf[..., 32:112].cpu().permute(0, 4, 3, 1, 2)
    err = _rel(got, ref)
    print(f"front end B={b}: max-rel {err:.2e}")
    assert err < 1e-5
    assert not bool(buf[..., 112:].cpu().any())


@pytest.mark.gpu
@pytest.mark.parametrize("b,side,cin,cout,up", [(1, 8, 96, 64, False), (2, 4, 64, 32, True), (2, 16, 128, 128, False)])
def test_pitched_conv3d_and_pool_match_float64(b, side, cin, cout, up):
    """The volumetric convolution from channel slice [16, 16 + cin) of a NaN-guarded buffer into slice [8, 8 + cout) of
    another, then the (1, 2, 2) average into a slice: neighbouring channels stay NaN, the values match float64."""
    from e4s_b200 import kernels as K
    g = torch.Generator().manual_seed(side * 7 + cin)
    x = torch.randn(b, side, side, 16, cin, generator=g)
    wt = torch.randn(cout, cin, 3, 3, 3, generator=g) / (27 * cin) ** 0.5
    bias = 0.1 * torch.randn(cout, generator=g)
    src = _nan_buffer((b, side, side, 16, cin + 32))
    src[..., 16:16 + cin] = x.cuda()
    m = 2 if up else 1
    dst = _nan_buffer((b, side * m, side * m, 16, cout + 16))
    K.conv3d_pitched_tc(src[..., 16:16 + cin], K.conv3d_planes(wt).cuda(), bias.cuda(), out=dst[..., 8:8 + cout], up=up, relu=True)
    xd = x.double().permute(0, 4, 3, 1, 2)
    if up:
        xd = F.interpolate(xd, scale_factor=(1, 2, 2))
    ref = F.relu(F.conv3d(xd, wt.double(), bias.double(), padding=1))
    got = dst.cpu()
    assert bool(got[..., :8].isnan().all()) and bool(got[..., 8 + cout:].isnan().all())
    err = _rel(got[..., 8:8 + cout].permute(0, 4, 3, 1, 2), ref)
    print(f"pitched conv3d b={b} side={side} {cin}->{cout} up={up}: max-rel {err:.2e}")
    assert err < 2e-4
    y = dst[..., 8:8 + cout].contiguous()
    pool = _nan_buffer((b, side * m // 2, side * m // 2, 16, cout + 8))
    K.avgpool2_vox(y, pool[..., 4:4 + cout])
    got = pool.cpu()
    assert bool(got[..., :4].isnan().all()) and bool(got[..., 4 + cout:].isnan().all())
    ref = F.avg_pool3d(y.cpu().double().permute(0, 4, 3, 1, 2), (1, 2, 2))
    assert _rel(got[..., 4:4 + cout].permute(0, 4, 3, 1, 2), ref) < 1e-6


@pytest.mark.gpu
@pytest.mark.parametrize("b,d,h,w,cin", [(1, 16, 8, 16, 32), (2, 5, 16, 32, 128), (1, 3, 64, 64, 64)])
def test_conv7x7_slices_matches_float64(b, d, h, w, cin):
    from e4s_b200 import kernels as K
    g = torch.Generator().manual_seed(d * 100 + h + cin)
    x = torch.randn(b, h, w, d, cin, generator=g)
    wt = torch.randn(49, 128, cin, generator=g) / (49 * cin) ** 0.5
    y = K.conv7x7_slices_tc(x.cuda(), K.split_bf16(wt).cuda()).cpu()
    slices = x.double().permute(0, 3, 4, 1, 2).reshape(b * d, cin, h, w)
    ref = F.conv2d(slices, wt.double().permute(1, 2, 0).reshape(128, cin, 7, 7), padding=3)
    err = _rel(y.reshape(b * d, h, w, 128).permute(0, 3, 1, 2), ref)
    print(f"7x7 slices b={b} d={d} {h}x{w} cin={cin}: max-rel {err:.2e}")
    assert err < 2e-4


@pytest.mark.gpu
@pytest.mark.parametrize("b", [1, 2])
def test_combine_matches_float64(b):
    from e4s_b200 import kernels as K
    g = torch.Generator().manual_seed(70 + b)
    p = torch.randn(b, 16, 64, 64, 128, generator=g) * 0.5
    mb, ob = torch.randn(16, generator=g), torch.randn(1, generator=g)
    kd, ks = O.synthetic_keypoints(b, 80 + b)
    mask, deform, occ = K.vid2vid_motion_combine(p.cuda(), mb.cuda(), ob.cuda(), kd.cuda(), ks.cuda())
    pd = p.double()
    logits = torch.zeros(b, 16, 16, 64, 64, dtype=torch.float64)
    for z in range(16):
        for dz in range(7):
            if 0 <= z + dz - 3 < 16:
                logits[:, :, z] += pd[:, z + dz - 3, :, :, 16 * dz:16 * dz + 16].permute(0, 3, 1, 2)
    ref_mask = torch.softmax(logits + mb.double().view(1, 16, 1, 1, 1), 1)
    motions = O.sparse_motions(kd.double(), ks.double())
    ref_def = (motions * ref_mask.unsqueeze(-1)).sum(1)
    ref_occ = torch.sigmoid(sum(pd[:, z, :, :, 112 + z] for z in range(16)) + ob.double()).unsqueeze(1)
    errs = [float((a.cpu().double() - r).abs().max()) for a, r in ((mask, ref_mask), (deform, ref_def), (occ, ref_occ))]
    print(f"combine B={b}: max abs mask {errs[0]:.2e} deformation {errs[1]:.2e} occlusion {errs[2]:.2e}")
    assert max(errs) < 1e-5


@pytest.fixture(scope="module")
def gpu_net(state):
    net = _net()
    net.load_state_dict(state, strict=True)
    return net.eval().cuda()


def _run(net, feat, kd, ks):
    with torch.no_grad():
        return net(feat, {"value": kd, "jacobian": None}, {"value": ks})


@pytest.mark.gpu
def test_forward_matches_golden_and_oracle(gpu_net, gold, state):
    feat, kd, ks = _golden_inputs(gold)
    out = _run(gpu_net, feat.cuda(), kd.cuda(), ks.cuda())
    assert tuple(out["mask"].shape) == (2, 16, 16, 64, 64) and out["mask"].is_contiguous()
    assert tuple(out["deformation"].shape) == (2, 16, 64, 64, 3) and out["deformation"].is_contiguous()
    assert tuple(out["occlusion_map"].shape) == (2, 1, 64, 64) and out["occlusion_map"].is_contiguous()
    for name, got in (("mask_sub", out["mask"][SUB]), ("deformation_sub", out["deformation"][SUB[:4]]),
                      ("occlusion_map", out["occlusion_map"])):
        err = float((got.cpu() - torch.from_numpy(gold[name])).abs().max())
        print(f"forward vs reference golden {name}: max abs {err:.2e}")
        assert err < 1e-3, name
    with torch.no_grad():
        ref = O.forward(state, feat[:1].double(), kd[:1].double(), ks[:1].double())
    for k in ref:
        err = float((out[k][:1].cpu().double() - ref[k]).abs().max())
        print(f"forward vs float64 oracle {k}: max abs {err:.2e}")
        assert err < 1e-3, k


@pytest.mark.gpu
def test_outputs_bitwise_alone_batch_graph(gpu_net):
    feat = O.synthetic_feature(3, 90).cuda()
    kd, ks = (t.cuda() for t in O.synthetic_keypoints(3, 91))
    batch = _run(gpu_net, feat, kd, ks)
    alone = _run(gpu_net, feat[1:2].contiguous(), kd[1:2].contiguous(), ks[1:2].contiguous())
    sf, sd, ss = feat[:2].clone(), kd[:2].clone(), ks[:2].clone()
    _run(gpu_net, sf, sd, ss)                                                  # warm-up, prepares the weights
    graph = torch.cuda.CUDAGraph()
    with torch.no_grad(), torch.cuda.graph(graph):
        out = gpu_net(sf, {"value": sd}, {"value": ss})
    sf.copy_(feat[1:3]), sd.copy_(kd[1:3]), ss.copy_(ks[1:3])
    graph.replay()
    torch.cuda.synchronize()
    for k in batch:
        assert torch.equal(alone[k][0], batch[k][1]), ("alone", k)
        assert torch.equal(out[k], batch[k][1:3]), ("graph", k)


@pytest.mark.gpu
def test_data_parallel_one_device(gpu_net):
    feat = O.synthetic_feature(2, 92).cuda()
    kd, ks = (t.cuda() for t in O.synthetic_keypoints(2, 93))
    ref = _run(gpu_net, feat, kd, ks)
    out = _run(torch.nn.DataParallel(gpu_net, device_ids=[0]), feat, kd, ks)
    for k in ref:
        assert torch.equal(out[k], ref[k]), k


@pytest.mark.gpu
def test_bad_inputs_raise(gpu_net):
    from e4s_b200 import kernels as K
    from e4s_b200.face_vid2vid.modules.dense_motion import DenseMotionNetwork
    feat = torch.zeros(1, 32, 16, 64, 64, device="cuda")
    kp = torch.zeros(1, 15, 3, device="cuda")
    with pytest.raises(NotImplementedError):
        _run(gpu_net, torch.zeros(1, 32, 16, 32, 32, device="cuda"), kp, kp)
    with pytest.raises(NotImplementedError):
        _run(gpu_net, feat.cpu(), kp.cpu(), kp.cpu())
    with pytest.raises(NotImplementedError):
        _run(gpu_net, feat, torch.zeros(2, 15, 3, device="cuda"), kp)
    with torch.no_grad(), pytest.raises(NotImplementedError):
        gpu_net(feat, {"value": kp, "jacobian": torch.zeros(1, 15, 3, 3, device="cuda")}, {"value": kp})
    with pytest.raises(NotImplementedError):
        gpu_net(feat.requires_grad_(), {"value": kp}, {"value": kp})
    gpu_net.train()
    try:
        with pytest.raises(NotImplementedError):
            _run(gpu_net, feat.detach(), kp, kp)
    finally:
        gpu_net.eval()
    other = DenseMotionNetwork(**dict(O.PARAMS, estimate_occlusion_map=False)).eval().cuda()
    with pytest.raises(NotImplementedError):
        _run(other, feat.detach(), kp, kp)
    with pytest.raises(RuntimeError):
        K.conv7x7_slices_tc(torch.zeros(1, 12, 16, 2, 32, device="cuda"),
                            torch.zeros(2, 49, 128, 32, dtype=torch.bfloat16, device="cuda"))
    with pytest.raises(RuntimeError):
        K.conv3d_pitched_tc(torch.zeros(1, 4, 4, 2, 64, device="cuda")[..., :32].transpose(1, 2),
                            torch.zeros(2, 9, 32, 96, dtype=torch.bfloat16, device="cuda"))
