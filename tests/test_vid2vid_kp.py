"""face-vid2vid's keypoint front end (e4s_b200.face_vid2vid): on the CPU both mirrors' state-dict layouts against the
reference's (the layout JSON), the oracle's KPDetector, HEEstimator and pose functions and the library's pose functions
against the reference's goldens, and the drop-in mapping; on the GPU the volumetric convolution mode against
float64 F.conv3d (depth edges, up-sampling, partial tiles, gutterless and mosaic tilings, several mosaic rows), the heatmap
head against float64 on a near-uniform and a one-hot heatmap, the input prep and the 2x2 average against float64, both
forwards and drive_keypoints against the oracle, a pair's keypoints bitwise alone / in a batch / graph-replayed, the
one-device DataParallel wrapper and bad inputs."""
import json
import os
import sys

import pytest
import torch
import torch.nn.functional as F

from conftest import ROOT

from oracle import golden_io
from oracle import vid2vid_kp_oracle as O

GOLDEN = os.path.join(ROOT, "tests", "golden", "vid2vid_kp_vectors.npz")
LAYOUT = os.path.join(ROOT, "tests", "golden", "vid2vid_kp_checkpoint_layout.json")


@pytest.fixture(scope="module")
def gold():
    return golden_io.load(GOLDEN)


def _he():
    from e4s_b200.face_vid2vid.modules.keypoint_detector import HEEstimator
    return HEEstimator(**O.HE_PARAMS)


def _faces(g):
    x = torch.from_numpy(g["x_u8"]).float() / 255
    d = torch.from_numpy(g["driving_u8"]).float() / 255
    return x, d


def _detector():
    from e4s_b200.face_vid2vid.modules.keypoint_detector import KPDetector
    p = dict(O.PARAMS)
    return KPDetector(**p)


def _rel(a, b):
    return float((a.double() - b.double()).abs().max() / b.double().abs().max().clamp_min(1e-30))


# ------------------------------------------------------------------------------------------------------------ CPU
def test_state_dict_layouts_match_reference():
    with open(LAYOUT) as f:
        layout = json.load(f)
    for name, mod, st in (("kp_detector", _detector(), O.synthetic_state()), ("he_estimator", _he(), O.he_synthetic_state())):
        got = {k: list(v.shape) for k, v in mod.state_dict().items()}
        assert got == layout[name], name
        assert {k: list(v.shape) for k, v in st.items()} == layout[name], name
        mod.load_state_dict(st, strict=True)
    assert len(layout["kp_detector"]) == 75 and len(layout["he_estimator"]) == 402


def test_oracle_matches_reference_golden(gold):
    x, d = _faces(gold)
    with torch.no_grad():
        v = O.kp_forward(O.synthetic_state(), x)["value"]
        he = O.he_forward(O.he_synthetic_state(), torch.cat([x, d]))
    assert (v - torch.from_numpy(gold["value"])).abs().max() < 2e-5
    for k in ("yaw", "pitch", "roll", "t", "exp"):
        want = torch.from_numpy(gold["he_" + k])
        assert (he[k] - want).abs().max() <= 2e-5 * want.abs().max(), k


@pytest.mark.parametrize("impl", ["oracle", "library"])
def test_pose_functions_match_reference_golden(gold, impl):
    from e4s_b200.face_vid2vid import keypoints as KP
    for tag, he, kp in (("net", {k: torch.from_numpy(gold["he_" + k]) for k in ("yaw", "pitch", "roll", "t", "exp")},
                         torch.from_numpy(gold["value"]).expand(3, 15, 3)),
                        ("seeded", {k: torch.from_numpy(gold["seeded_he_" + k]) for k in ("yaw", "pitch", "roll", "t", "exp")},
                         torch.from_numpy(gold["seeded_kp"]))):
        t_before = he["t"].clone()
        deg = {k: (O if impl == "oracle" else KP).headpose_pred_to_degree(he[k]) for k in ("yaw", "pitch", "roll")}
        for k in deg:
            assert (deg[k] - torch.from_numpy(gold[f"{tag}_deg_{k}"])).abs().max() < 1e-4, (tag, k)
        if impl == "oracle":
            rot = O.get_rotation_matrix(deg["yaw"], deg["pitch"], deg["roll"])
            kpt = O.keypoint_transformation(kp, he)
        else:
            rot = KP.get_rotation_matrix(deg["yaw"], deg["pitch"], deg["roll"])
            kpt = KP.keypoint_transformation({"value": kp}, he)["value"]
        assert (rot - torch.from_numpy(gold[f"{tag}_rot"])).abs().max() < 1e-5, tag
        assert (kpt - torch.from_numpy(gold[f"{tag}_kp_transformed"])).abs().max() < 1e-5, tag
        assert torch.equal(he["t"], t_before) and he["t"].dim() == 2               # not unsqueezed in place


def test_dropin_maps_the_keypoint_module():
    from e4s_b200 import dropin
    dropin.install()
    import e4s_b200.face_vid2vid.modules.keypoint_detector as M
    assert sys.modules["src.pretrained.face_vid2vid.modules.keypoint_detector"] is M
    assert M.KPDetector and M.HEEstimator


# ------------------------------------------------------------------------------------------------------------ GPU
CONV3D_CASES = [
    # b, d, h, w (input grid), cin, cout, up, relu
    (1, 16, 2, 2, 64, 64, True, True),        # 4 x 4 slices: mosaic with gutters, one mosaic row
    (2, 16, 4, 4, 32, 64, True, True),        # 8 x 8 slices, two mosaic rows
    (2, 5, 8, 8, 64, 32, True, False),        # 16 x 16 slices: gutterless stacked tiles, shallow depth
    (3, 7, 5, 7, 32, 32, False, True),        # 5 x 7 slices, 21 cells: partial mosaic row
    (1, 2, 8, 16, 32, 64, False, False),      # gutterless, depth 2: every chunk meets a depth edge
    (2, 3, 3, 20, 96, 32, True, True),        # 6 x 40 slices: partial tiles along x inside the mosaic
]


@pytest.mark.gpu
@pytest.mark.parametrize("b,d,h,w,cin,cout,up,relu", CONV3D_CASES)
def test_conv3d_matches_float64(b, d, h, w, cin, cout, up, relu):
    from e4s_b200 import kernels as K
    g = torch.Generator().manual_seed(b * 1000 + d * 100 + h * 10 + w)
    x = torch.randn(b, cin, d, h, w, generator=g)
    wt = torch.randn(cout, cin, 3, 3, 3, generator=g) / (27 * cin) ** 0.5
    bias = torch.randn(cout, generator=g) * 0.1
    xd = x.double()
    if up:
        xd = F.interpolate(xd, scale_factor=(1, 2, 2))
    ref = F.conv3d(xd, wt.double(), bias.double(), padding=1)
    if relu:
        ref = ref.relu()
    dev = torch.device("cuda")
    x_pm = x.permute(0, 3, 4, 2, 1).contiguous().to(dev)              # [B, H, W, D, C]
    y = K.conv3d_tc(x_pm, K.conv3d_planes(wt).to(dev), bias.to(dev), up=up, relu=relu)
    out = y.permute(0, 4, 3, 1, 2).cpu()                               # [B, C, D, H, W]
    err = _rel(out, ref)
    print(f"conv3d b{b} d{d} {h}x{w} {cin}->{cout} up={up} relu={relu}: rel err {err:.2e}, useful rows "
          f"{K.conv3d_useful_rows(b, d, h * (2 if up else 1), w * (2 if up else 1)):.3f}")
    assert err < 2e-5


@pytest.mark.gpu
def test_conv3d_useful_rows_of_the_kp_layers():
    from e4s_b200 import kernels as K
    f = [K.conv3d_useful_rows(16, 16, s, s) for s in (4, 8, 16, 32, 64)]
    assert abs(f[0] - 0.64) < 1e-9 and abs(f[1] - 4096 / 5184) < 1e-9 and f[2:] == [1.0, 1.0, 1.0]


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["near_uniform", "one_hot"])
def test_heatmap_matches_float64(kind):
    from e4s_b200 import kernels as K
    g = torch.Generator().manual_seed(5)
    b, k, d, h, w, c = 2, 15, 16, 64, 64, 32
    if kind == "near_uniform":
        lg = torch.randn(b, h, w, d, c, generator=g) * 1e-3
    else:
        lg = torch.randn(b, h, w, d, c, generator=g)
        idx = torch.randint(0, d * h * w, (b, k), generator=g)
        flat = lg.view(b, -1, c)
        for i in range(b):
            for j in range(k):
                flat[i, idx[i, j], j] = 1e3
    ref = O.heatmap_kp(lg.double().permute(0, 4, 3, 1, 2)[:, :k].contiguous(), 0.1)
    kp = K.vid2vid_heatmap(lg.cuda(), k, 0.1).cpu()
    err = float((kp.double() - ref).abs().max())
    print(f"heatmap {kind}: max abs err {err:.2e}")
    assert err < 2e-6


@pytest.mark.gpu
def test_prep_and_avgpool_match_float64():
    from e4s_b200 import kernels as K
    x = O.synthetic_faces(2, 3)
    filt = O.anti_alias_filter()
    ref = F.conv2d(F.pad(x.double(), (6, 6, 6, 6)), filt.double(), groups=3)[:, :, ::4, ::4]
    y = K.vid2vid_kp_prep(x.cuda(), filt.cuda()).cpu()
    assert _rel(y[..., :3].permute(0, 3, 1, 2), ref) < 1e-6
    assert torch.count_nonzero(y[..., 3:]) == 0
    z = torch.randn(2, 8, 6, 64)
    p = K.avgpool2(z.cuda()).cpu()
    assert _rel(p, F.avg_pool2d(z.double().permute(0, 3, 1, 2), 2).permute(0, 2, 3, 1)) < 1e-6


@pytest.fixture(scope="module")
def gpu_detector():
    det = _detector()
    det.load_state_dict(O.synthetic_state(), strict=True)
    return det.eval().cuda()


@pytest.mark.gpu
def test_forward_matches_oracle(gpu_detector):
    x = O.synthetic_faces(2, 11)
    with torch.no_grad():
        ref = O.kp_layers(O.synthetic_state(), x)
        out = gpu_detector(x.cuda())["value"].cpu()
    err = float((out - ref["value"]).abs().max())
    print(f"KPDetector forward: max abs keypoint err {err:.2e}")
    assert err < 5e-4


@pytest.mark.gpu
def test_keypoints_bitwise_alone_batch_graph(gpu_detector):
    x = O.synthetic_faces(5, 12).cuda()
    with torch.no_grad():
        batch = gpu_detector(x)["value"]
        alone = gpu_detector(x[2:3].contiguous())["value"]
        static = x[1:4].clone()
        gpu_detector(static)                                            # warm-up, prepares the weights
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            out = gpu_detector(static)["value"]
        static.copy_(x[1:4])
        graph.replay()
        torch.cuda.synchronize()
    assert torch.equal(alone[0], batch[2])
    assert torch.equal(out, batch[1:4])


@pytest.mark.gpu
def test_data_parallel_one_device(gpu_detector):
    x = O.synthetic_faces(2, 13).cuda()
    with torch.no_grad():
        ref = gpu_detector(x)["value"]
        out = torch.nn.DataParallel(gpu_detector, device_ids=[0])(x)["value"]
    assert torch.equal(out, ref)


@pytest.mark.gpu
def test_bad_inputs_raise(gpu_detector):
    from e4s_b200 import kernels as K
    with torch.no_grad():
        with pytest.raises(NotImplementedError):
            gpu_detector(torch.zeros(1, 3, 128, 128, device="cuda"))
        with pytest.raises(NotImplementedError):
            gpu_detector(torch.zeros(1, 3, 256, 256))
    with pytest.raises(NotImplementedError):
        gpu_detector(torch.zeros(1, 3, 256, 256, device="cuda", requires_grad=True))
    jac = KPDetector_with_jacobian()
    with torch.no_grad(), pytest.raises(NotImplementedError):
        jac(torch.zeros(1, 3, 256, 256, device="cuda"))
    with pytest.raises(RuntimeError):
        K.conv3d_tc(torch.zeros(1, 4, 4, 2, 48, device="cuda"), torch.zeros(2, 9, 32, 144, dtype=torch.bfloat16, device="cuda"))
    with pytest.raises(RuntimeError):
        K.conv3d_tc(torch.zeros(1, 4, 4, 2, 32, device="cuda"), torch.zeros(2, 9, 32, 64, dtype=torch.bfloat16, device="cuda"))


def KPDetector_with_jacobian():
    from e4s_b200.face_vid2vid.modules.keypoint_detector import KPDetector
    p = dict(O.PARAMS, estimate_jacobian=True)
    return KPDetector(**p).eval().cuda()


@pytest.fixture(scope="module")
def gpu_he():
    he = _he()
    he.load_state_dict(O.he_synthetic_state(), strict=True)
    return he.eval().cuda()


@pytest.mark.gpu
def test_he_forward_matches_oracle(gpu_he):
    x = O.synthetic_faces(3, 14)
    with torch.no_grad():
        ref = O.he_forward({k: v.double() for k, v in O.he_synthetic_state().items()}, x.double())
        out = gpu_he(x.cuda())
    for k in ("yaw", "pitch", "roll", "t", "exp"):
        err = _rel(out[k].cpu(), ref[k])
        print(f"HEEstimator {k}: rel err vs float64 {err:.2e}")
        assert err < 1e-3, k            # see FORWARD_TOL in test_vid2vid_kp_at_scale.py


@pytest.mark.gpu
def test_drive_keypoints_matches_oracle(gpu_detector, gpu_he, gold):
    from e4s_b200.face_vid2vid.keypoints import drive_keypoints
    x, d = _faces(gold)
    src, drv = torch.cat([x, d[:1]]), d
    with torch.no_grad():
        out = drive_keypoints(gpu_detector, gpu_he, src.cuda(), drv.cuda())
        canon = O.kp_forward(O.synthetic_state(), src)["value"]
        he = O.he_forward(O.he_synthetic_state(), torch.cat([src, drv]))
    ks = O.keypoint_transformation(canon, {k: v[:2] for k, v in he.items()})
    kd = O.keypoint_transformation(canon, {k: v[2:] for k, v in he.items()})
    es, ed = float((out["kp_source"].cpu() - ks).abs().max()), float((out["kp_driving"].cpu() - kd).abs().max())
    print(f"drive_keypoints: max abs err source {es:.2e}, driving {ed:.2e}")
    assert max(es, ed) < 1e-3
    assert out["kp_source"].shape == (2, 15, 3) and out["he_driving"]["yaw"].shape == (2, 66)


@pytest.mark.gpu
def test_drive_keypoints_bitwise_alone_batch_graph(gpu_detector, gpu_he):
    from e4s_b200.face_vid2vid.keypoints import drive_keypoints
    src, drv = O.synthetic_faces(4, 15).cuda(), O.synthetic_faces(4, 16).cuda()
    with torch.no_grad():
        batch = drive_keypoints(gpu_detector, gpu_he, src, drv)
        alone = drive_keypoints(gpu_detector, gpu_he, src[1:2].contiguous(), drv[1:2].contiguous())
        s_static, d_static = src[2:4].clone(), drv[2:4].clone()
        drive_keypoints(gpu_detector, gpu_he, s_static, d_static)
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            g_out = drive_keypoints(gpu_detector, gpu_he, s_static, d_static)
        s_static.copy_(src[2:4]), d_static.copy_(drv[2:4])
        graph.replay()
        torch.cuda.synchronize()
    for k in ("yaw", "pitch", "roll", "t", "exp"):
        assert torch.equal(alone["he_driving"][k][0], batch["he_driving"][k][1]), ("alone", k)
        assert torch.equal(g_out["he_driving"][k], batch["he_driving"][k][2:4]), ("graph", k)
    assert torch.equal(alone["kp_canonical"]["value"][0], batch["kp_canonical"]["value"][1])
    for key in ("kp_source", "kp_driving"):
        assert torch.equal(alone[key][0], batch[key][1]), ("alone", key)
        assert torch.equal(g_out[key], batch[key][2:4]), ("graph", key)


@pytest.mark.gpu
def test_he_data_parallel_and_bad_inputs(gpu_he):
    from e4s_b200.face_vid2vid.keypoints import drive_keypoints, keypoint_transformation
    x = O.synthetic_faces(2, 17).cuda()
    with torch.no_grad():
        ref = gpu_he(x)
        out = torch.nn.DataParallel(gpu_he, device_ids=[0])(x)
        for k in ref:
            assert torch.equal(out[k], ref[k]), k
        with pytest.raises(NotImplementedError):
            gpu_he(torch.zeros(1, 3, 128, 128, device="cuda"))
        with pytest.raises(ValueError):
            drive_keypoints(None, gpu_he, x, x[:1])
        with pytest.raises(NotImplementedError):
            keypoint_transformation({"value": torch.zeros(2, 15, 3, device="cuda")}, ref, estimate_jacobian=True)
    with pytest.raises(NotImplementedError):
        gpu_he(x.clone().requires_grad_())
