"""GPEN's RetinaFace-R50 detector (e4s_b200.gpen.face_detect): on the CPU the oracle against the reference's goldens, the
state-dict layout, the drop-in mapping and the oracle's decode / NMS restatements; on the GPU the kernel forward and
detect() against the goldens (with the margin that makes an equal detection list meaningful), the NMS kernel against the
oracle's py_cpu_nms on identical fp32 inputs, the decode kernel against torch's decode on the GPU, the pointwise convolution
against float64, detect_batch alone / in a batch / graph-replayed, and bad inputs."""
import json
import os
import sys

import numpy as np
import pytest
import torch

from conftest import ROOT

from oracle import golden_io
from oracle import retinaface_oracle as RO

CASES = [("a", 256, 256, 21), ("b", 192, 320, 22)]
SUB = 7


@pytest.fixture(scope="module")
def gold():
    return golden_io.load(os.path.join(ROOT, "tests", "golden", "retinaface_vectors.npz"))


@pytest.fixture(scope="module")
def state():
    return RO.synthetic_state()


# ------------------------------------------------------------------------------------------------------------ CPU
@pytest.mark.parametrize("tag,h,w,seed", CASES)
def test_oracle_matches_reference_golden(gold, state, tag, h, w, seed):
    img = RO.case_image(h, w, seed)
    with torch.no_grad():
        _, _, _, (loc, conf, landms) = RO.decoded(state, img)
        dets, lms = RO.detect(state, img)
    for name, t in (("loc", loc), ("conf", conf), ("landms", landms)):
        ref = torch.from_numpy(gold[f"retina/{tag}/{name}_sub"])
        assert float((t[0, ::SUB] - ref).abs().max() / ref.abs().max()) <= 2e-5, name
    assert np.array_equal(dets, gold[f"retina/{tag}/dets"]) and np.array_equal(lms, gold[f"retina/{tag}/landms"])
    assert len(dets) > 0


def test_golden_detections_exercise_the_tail(gold):
    """The stand-in's class head puts a few per cent of the priors above 0.9, and the fixture has a case where top_k and
    keep_top_k bind."""
    for tag, h, w, _ in CASES:
        n = RO.prior_box(h, w).shape[0]
        conf = gold[f"retina/{tag}/conf_sub"][:, 1]
        assert 0.005 <= float((conf > 0.9).mean()) <= 0.08, tag
        assert 0 < len(gold[f"retina/{tag}/dets"]) < n
    assert len(gold["retina/a/dets_bound"]) == 3


def test_mirror_state_dict_layout():
    from e4s_b200.gpen.face_detect.data import cfg_mnet, cfg_re50
    from e4s_b200.gpen.face_detect.facemodels.retinaface import RetinaFace
    from e4s_b200.synthetic import synthetic_retinaface_state
    with open(os.path.join(ROOT, "tests", "golden", "retinaface_checkpoint_layout.json")) as f:
        layout = json.load(f)
    net = RetinaFace(cfg=cfg_re50, phase='test')
    assert {k: list(v.shape) for k, v in net.state_dict().items()} == layout
    assert len(layout) == 456
    assert sum(v.numel() for k, v in net.state_dict().items() if not k.endswith("num_batches_tracked")) == 27_351_584
    st = synthetic_retinaface_state()
    net.load_state_dict(st, strict=True)
    RetinaFace(cfg=cfg_mnet, phase='test')          # the MobileNet tree builds


def test_detection_wrapper_loads_prefixed_checkpoint(tmp_path, state):
    from e4s_b200.gpen.face_detect.retinaface_detection import RetinaFaceDetection
    (tmp_path / "weights").mkdir()
    torch.save({"module." + k: v for k, v in state.items()}, tmp_path / "weights" / "RetinaFace-R50.pth")
    det = RetinaFaceDetection(str(tmp_path), device="cpu")
    sd = det.net.state_dict()
    assert all(torch.equal(sd[k], state[k]) for k in state)
    torch.set_grad_enabled(True)
    with pytest.raises(NotImplementedError):
        det.detect_tensor(torch.zeros(1, 3, 64, 64))


def test_dropin_maps_the_detector():
    from e4s_b200 import dropin
    dropin.install()
    import e4s_b200.gpen.face_detect.facemodels.net as N
    import e4s_b200.gpen.face_detect.facemodels.retinaface as R
    import e4s_b200.gpen.face_detect.retinaface_detection as D
    assert sys.modules["src.pretrained.gpen.face_detect.retinaface_detection"] is D
    assert sys.modules["src.pretrained.gpen.face_detect.facemodels.retinaface"] is R
    assert sys.modules["src.pretrained.gpen.face_detect.facemodels.net"] is N


def _py_cpu_nms(dets, thresh):
    """py_cpu_nms (utils/nms/py_cpu_nms.py) verbatim in behaviour: numpy's unstable descending argsort."""
    x1, y1, x2, y2, scores = (dets[:, i] for i in range(5))
    areas = (x2 - x1 + 1) * (y2 - y1 + 1)
    order = scores.argsort()[::-1]
    keep = []
    while order.size > 0:
        i = order[0]
        keep.append(int(i))
        xx1 = np.maximum(x1[i], x1[order[1:]])
        yy1 = np.maximum(y1[i], y1[order[1:]])
        xx2 = np.minimum(x2[i], x2[order[1:]])
        yy2 = np.minimum(y2[i], y2[order[1:]])
        w = np.maximum(0.0, xx2 - xx1 + 1)
        h = np.maximum(0.0, yy2 - yy1 + 1)
        inter = w * h
        ovr = inter / (areas[i] + areas[order[1:]] - inter)
        order = order[np.where(ovr <= thresh)[0] + 1]
    return keep


def _random_dets(n, seed):
    g = np.random.default_rng(seed)
    xy = g.uniform(0, 300, (n, 2)).astype(np.float32)
    wh = g.uniform(-5, 80, (n, 2)).astype(np.float32)            # zero and negative widths included
    wh[:5] = 0.0
    scores = (0.9 + 0.1 * g.permutation(n) / n).astype(np.float32)   # tie-free
    return np.hstack([xy, xy + wh, scores[:, None]]).astype(np.float32)


def test_oracle_nms_is_py_cpu_nms_without_ties():
    for seed in range(4):
        d = _random_dets(400, seed)
        assert RO.nms(d, 0.4) == _py_cpu_nms(d, 0.4)


def test_oracle_decode_is_box_utils_decode():
    """The restated decode keeps box_utils' operation order: against an independent float64 evaluation, and exact against
    the same ops spelled out."""
    g = torch.Generator().manual_seed(3)
    pri = RO.prior_box(64, 96)
    loc = torch.randn(pri.shape[0], 4, generator=g)
    pre = torch.randn(pri.shape[0], 10, generator=g)
    b = RO.decode(loc, pri)
    c = torch.cat((pri[:, :2] + loc[:, :2] * 0.1 * pri[:, 2:], pri[:, 2:] * torch.exp(loc[:, 2:] * 0.2)), 1)
    c[:, :2] -= c[:, 2:] / 2
    c[:, 2:] += c[:, :2]
    assert torch.equal(b, c)
    p64, l64 = pri.double(), loc.double()
    ctr = p64[:, :2] + l64[:, :2] * 0.1 * p64[:, 2:]
    wh = p64[:, 2:] * torch.exp(l64[:, 2:] * 0.2)
    assert torch.allclose(b.double(), torch.cat([ctr - wh / 2, ctr + wh / 2], 1), rtol=0, atol=1e-6)
    lm = RO.decode_landm(pre, pri)
    assert torch.allclose(lm.double()[:, 4:6], p64[:, :2] + pre.double()[:, 4:6] * 0.1 * p64[:, 2:], rtol=0, atol=1e-6)


# ------------------------------------------------------------------------------------------------------------ GPU
@pytest.fixture(scope="module")
def detector(tmp_path_factory, state):
    from e4s_b200.gpen.face_detect.retinaface_detection import RetinaFaceDetection
    d = tmp_path_factory.mktemp("retina")
    (d / "weights").mkdir()
    torch.save({"module." + k: v for k, v in state.items()}, d / "weights" / "RetinaFace-R50.pth")
    det = RetinaFaceDetection(str(d), device="cuda")
    torch.set_grad_enabled(True)            # the constructor turns autograd off globally, as the reference's does
    return det


def _planar(img):
    xf = np.float32(img)
    xf -= (104, 117, 123)
    return torch.from_numpy(xf.transpose(2, 0, 1).copy()).unsqueeze(0)


FWD_TOL = 1e-4


@pytest.mark.gpu
@pytest.mark.parametrize("tag,h,w,seed", CASES)
def test_forward_matches_oracle(detector, state, tag, h, w, seed):
    img = RO.case_image(h, w, seed)
    x = _planar(img)
    with torch.no_grad():
        loc, conf, landms = detector.net(x.cuda())
        r_loc, r_conf, r_lm = RO.forward(state, x)
    errs = [float((a.cpu() - b).abs().max() / b.abs().max()) for a, b in ((loc, r_loc), (conf, r_conf), (landms, r_lm))]
    print(f"retina/{tag}: forward max-rel loc {errs[0]:.2e} conf {errs[1]:.2e} landms {errs[2]:.2e}")
    assert max(errs) <= FWD_TOL, errs


@pytest.mark.gpu
@pytest.mark.parametrize("tag,h,w,seed", CASES)
def test_detect_matches_reference(detector, state, gold, tag, h, w, seed):
    """detect() keeps the reference's detections and order.  Margin condition first: with eps the measured error of the
    kernel's boxes and scores, every score is > 2 eps from the threshold and every overlap NMS evaluates is > 2 eps from
    0.4 - otherwise an equal list could not be expected and a weaker fixture would pass silently."""
    img = RO.case_image(h, w, seed)
    x = _planar(img)
    with torch.no_grad():
        boxes_r, lm_r, scores_r, _ = RO.decoded(state, img)
        (boxes, lms, keys), (_, conf, _) = _decode_all(detector, x.cuda(), 0.9)
    eps_s = float((conf[0, :, 1].cpu().double() - torch.from_numpy(scores_r).double()).abs().max())
    eps_b = float((boxes[0].cpu().double() - torch.from_numpy(boxes_r).double()).abs().max() / (1 + np.abs(boxes_r).max()))
    assert float(np.abs(scores_r.astype(np.float64) - np.float32(0.9)).min()) > 2 * eps_s, eps_s
    cand = boxes_r[scores_r > 0.9]
    ious = _all_ious(cand)
    assert ious.size == 0 or float(np.abs(ious - 0.4).min()) > 2 * max(eps_b * 4, eps_s), (eps_b, eps_s)
    dets, landms = detector.detect(img)
    print(f"retina/{tag}: score eps {eps_s:.1e}, box eps {eps_b:.1e}; {len(dets)} detections")
    ref_d, ref_l = gold[f"retina/{tag}/dets"], gold[f"retina/{tag}/landms"]
    assert dets.dtype == np.float32 and dets.shape == ref_d.shape and landms.shape == ref_l.shape
    np.testing.assert_allclose(dets, ref_d, rtol=0, atol=1e-3 * (1 + np.abs(ref_d).max()))
    np.testing.assert_allclose(landms, ref_l, rtol=0, atol=1e-3 * (1 + np.abs(ref_l).max()))
    d2, _ = detector.detect(img, top_k=40, keep_top_k=3) if tag == "a" else (None, None)
    if d2 is not None:
        np.testing.assert_allclose(d2, gold["retina/a/dets_bound"], rtol=0, atol=1e-3 * (1 + np.abs(ref_d).max()))


def _all_ious(b):
    x1, y1, x2, y2 = (b[:, i].astype(np.float64) for i in range(4))
    area = (x2 - x1 + 1) * (y2 - y1 + 1)
    w = np.maximum(0, np.minimum(x2[:, None], x2[None]) - np.maximum(x1[:, None], x1[None]) + 1)
    h = np.maximum(0, np.minimum(y2[:, None], y2[None]) - np.maximum(y1[:, None], y1[None]) + 1)
    inter = w * h
    iou = inter / (area[:, None] + area[None] - inter)
    return iou[np.triu_indices(len(b), 1)]


def _decode_all(detector, x, thr):
    from e4s_b200 import kernels as K
    heads = detector.net._heads(x)
    b, _, h, w = x.shape
    return K.retinaface_decode(heads, b, h, w, conf_thr=thr, module=True)


def _nms_kernel(dets, landms, thr=0.4, top_k=5000, keep_top_k=750, conf=0.9):
    """Run the NMS kernel on one image's fp32 [N, 5] dets (any order) and [N, 10] landmarks."""
    from e4s_b200 import kernels as K
    n = dets.shape[0]
    keys = torch.from_numpy(np.where(dets[:, 4] > np.float32(conf), dets[:, 4], -np.inf).astype(np.float32)).cuda()[None]
    ks, order = torch.sort(keys, dim=1, descending=True, stable=True)
    boxes = torch.from_numpy(np.ascontiguousarray(dets[:, :4])).cuda()[None]
    lm = torch.from_numpy(np.ascontiguousarray(landms)).cuda()[None]
    d, l, c = K.retinaface_nms(boxes, lm, ks, order, conf, thr, top_k, keep_top_k)
    k = int(c[0])
    return d[0, :k].cpu().numpy(), l[0, :k].cpu().numpy()


@pytest.mark.gpu
@pytest.mark.parametrize("case", ["random", "ties", "iou_exact", "degenerate", "none", "over_top_k", "over_keep_top_k"])
def test_nms_kernel_bit_exact(case):
    g = np.random.default_rng(7)
    d = _random_dets(3000, 1)
    thr, top_k, keep = 0.4, 5000, 750
    if case == "ties":
        d[::3, 4] = np.float32(0.95)
    elif case == "iou_exact":
        # py_cpu_nms's overlap of boxes 0 and 1 is exactly 0.4f: 5 x 7 boxes (with the + 1), offset by 3 rows, intersect in
        # 5 x 4 = 20, so ovr = 20 / (35 + 35 - 20) = 0.4f - not above the threshold, box 1 is kept.  Box 2 overlaps box 0
        # in 5 x 5 = 25, 25 / 45 > 0.4: suppressed
        d = np.array([[0, 0, 4, 6, 0.99], [0, 3, 4, 9, 0.98], [0, 2, 4, 8, 0.97]], np.float32)
        x1, y1, x2, y2 = (d[:2, i] for i in range(4))
        area = (x2 - x1 + 1) * (y2 - y1 + 1)
        inter = (np.minimum(x2[0], x2[1]) - np.maximum(x1[0], x1[1]) + 1) * (np.minimum(y2[0], y2[1]) - np.maximum(y1[0], y1[1]) + 1)
        assert inter / (area[0] + area[1] - inter) == np.float32(0.4)
    elif case == "degenerate":
        d[:, 2:4] = d[:, 0:2] - g.uniform(0, 3, (d.shape[0], 2)).astype(np.float32)
    elif case == "none":
        d[:, 4] = np.float32(0.5)
    elif case == "over_top_k":
        top_k = 100
    elif case == "over_keep_top_k":
        keep = 7
    lm = g.uniform(0, 300, (d.shape[0], 10)).astype(np.float32)
    ours_d, ours_l = _nms_kernel(d, lm, thr, top_k, keep)
    # the oracle's selection on the same fp32 inputs (ties: ascending index; numpy's py_cpu_nms on the tie-free cases)
    ref_d, ref_l = RO.select(d[:, :4], lm, d[:, 4], 0.9, thr, top_k, keep)
    if case not in ("ties",):
        cand = np.where(d[:, 4] > np.float32(0.9))[0]
        srt = cand[np.argsort(-d[cand, 4], kind="stable")][:top_k]
        keep_py = _py_cpu_nms(d[srt], thr)[:keep]
        assert np.array_equal(d[srt][keep_py], ref_d)
    print(f"nms/{case}: {len(ours_d)} kept")
    if case == "iou_exact":
        assert np.array_equal(ours_d[:, 4], np.float32([0.99, 0.98]))
    assert ours_d.tobytes() == ref_d.tobytes() and ours_l.tobytes() == ref_l.tobytes()


@pytest.mark.gpu
def test_decode_kernel_against_torch_decode_on_gpu(detector):
    x = _planar(RO.case_image(256, 256, 21)).cuda()
    with torch.no_grad():
        (boxes, lms, keys), (loc, conf, lr) = _decode_all(detector, x, 0.9)
    pri = RO.prior_box(256, 256).cuda()
    sc = torch.tensor([256.0, 256.0] * 2, device="cuda")
    ref_b = RO.decode(loc[0], pri) * sc / 1
    ref_l = RO.decode_landm(lr[0], pri) * torch.tensor([256.0] * 10, device="cuda") / 1
    ulp = lambda a, b: int((a.view(torch.int32).long() - b.view(torch.int32).long()).abs().max())  # noqa: E731
    ub, ul = ulp(boxes[0], ref_b), ulp(lms[0], ref_l)
    print(f"decode vs torch on the GPU: boxes {ub} ulp, landmarks {ul} ulp")
    assert ul == 0 and ub <= 1


@pytest.mark.gpu
@pytest.mark.parametrize("stride,res", [(1, "r0"), (2, None), (1, "r_up")])
def test_pointwise_conv_against_float64(stride, res):
    from e4s_b200 import kernels as K
    g = torch.Generator().manual_seed(11 + stride)
    b, h, w, cin, cout = 4, 32, 48, 256, 128
    x = torch.randn(b, h * stride, w * stride, cin + 32, generator=g)[..., :cin]
    wt = torch.randn(cout, cin, generator=g) / cin ** 0.5
    bias = torch.randn(cout, generator=g)
    r0 = torch.randn(b, h, w, cout, generator=g) if res == "r0" else None
    up = torch.randn(b, h // 2, w // 2, cout, generator=g) if res == "r_up" else None
    ours = K.conv1x1_tc(x.cuda(), K.split_bf16(wt.cuda()), bias.cuda(), r0=None if r0 is None else r0.cuda(),
                        r_up=None if up is None else up.cuda(), stride=stride, lrelu=0.0).cpu().double()
    ref = torch.einsum("bhwc,oc->bhwo", x[:, ::stride, ::stride].double(), wt.double()) + bias.double()
    if r0 is not None:
        ref = ref + r0.double()
    ref = ref.clamp_min(0)
    if up is not None:
        ref = ref + up.double().repeat_interleave(2, 1).repeat_interleave(2, 2)
    e = float((ours - ref).abs().max() / ref.abs().max())
    print(f"conv1x1 stride {stride} {res}: max-rel {e:.2e}")
    assert e <= 2e-5


@pytest.mark.gpu
def test_detect_batch_alone_batch_and_graph_bitwise(detector):
    from e4s_b200 import kernels as K
    imgs = torch.stack([torch.from_numpy(RO.case_image(256, 256, s).transpose(2, 0, 1).copy()) for s in (21, 31, 32)]).cuda()
    with torch.no_grad():
        batch = detector.detect_batch(imgs)
        batch_f = detector.detect_batch(imgs.float())
        # every convolution's N tile follows its channel count, never the batch: each image alone gives the same bits
        for i in range(imgs.shape[0]):
            alone = detector.detect_batch(imgs[i:i + 1])
            n = int(alone[2][0])
            assert n == int(batch[2][i]) and n > 0
            assert torch.equal(alone[0][0, :n], batch[0][i, :n]) and torch.equal(alone[1][0, :n], batch[1][i, :n]), i
        x = K.retinaface_prep(imgs)
        full = detector.net(x)
        for i in (0, 2):
            assert all(torch.equal(a[0], b[i]) for a, b in zip(detector.net(x[i:i + 1]), full)), i
        assert torch.equal(batch[2], batch_f[2])
        for i in range(imgs.shape[0]):                               # uint8 and float32 pixels: the same detections
            k = int(batch[2][i])
            assert torch.equal(batch[0][i, :k], batch_f[0][i, :k]) and torch.equal(batch[1][i, :k], batch_f[1][i, :k])
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            detector.detect_batch(imgs)
        torch.cuda.current_stream().wait_stream(s)
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            out = detector.detect_batch(imgs)
        graph.replay()
        torch.cuda.synchronize()
    assert torch.equal(out[2], batch[2])
    for i in range(imgs.shape[0]):
        k = int(batch[2][i])
        assert torch.equal(out[0][i, :k], batch[0][i, :k]) and torch.equal(out[1][i, :k], batch[1][i, :k])


@pytest.mark.gpu
def test_bad_inputs_raise(detector):
    from e4s_b200.gpen.face_detect.data import cfg_mnet
    from e4s_b200.gpen.face_detect.facemodels.retinaface import RetinaFace
    img = torch.zeros(1, 3, 64, 64, dtype=torch.uint8)
    with pytest.raises(ValueError):
        detector.detect_batch(img)                                   # CPU tensor
    with pytest.raises(ValueError):
        detector.detect_batch(img.cuda().to(torch.int32))            # wrong dtype
    with pytest.raises(NotImplementedError):
        detector.detect_batch(torch.zeros(1, 3, 64, 80, device="cuda"))
    with pytest.raises(NotImplementedError):
        detector.detect(np.zeros((100, 64, 3), np.uint8))
    with torch.no_grad(), pytest.raises(NotImplementedError):
        RetinaFace(cfg=cfg_mnet, phase='test').eval().cuda()(torch.zeros(1, 3, 64, 64, device="cuda"))
    with torch.no_grad(), pytest.raises(NotImplementedError):
        RetinaFace(cfg=detector.cfg, phase='train').eval().cuda()(torch.zeros(1, 3, 64, 64, device="cuda"))
    with torch.enable_grad(), pytest.raises(NotImplementedError):
        detector.net(torch.zeros(1, 3, 64, 64, device="cuda", requires_grad=True))
