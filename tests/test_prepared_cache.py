"""The kernel-ready weight cache of every network (e4s_b200/prepared.py), on the CPU: the operand builders are plain torch.

For each module that keeps prepared operands: an unchanged second call returns the same tensor objects; load_state_dict and
ordinary in-place ops are picked up without help; writes through ``.data`` (no version bump) are picked up after
``e4s_b200.invalidate_prepared`` on an enclosing module.  Values are compared against a fresh module holding the same weights.
"""
import types

import pytest
import torch
from torch import nn

import e4s_b200
from e4s_b200.stylegan2 import modconv_bwd as MB
from e4s_b200 import kernels as K

CPU = torch.device("cpu")
CONV_FIELDS = ("wt", "wsq", "wrgb", "w_hilo", "w_convt_hilo", "fir")


def _modconv():
    from e4s_b200.stylegan2.model import ModulatedConv2d
    return ModulatedConv2d(32, 32, 3, 64, upsample=True)


def _equal_linear():
    from e4s_b200.stylegan2.model import EqualLinear
    return EqualLinear(64, 32, lr_mul=0.01)


def _net3():
    from e4s_b200.networks import Net3
    return Net3(types.SimpleNamespace(fsencoder_type="psp", remaining_layer_idx=13, num_seg_cls=3, out_size=32,
                                      train_G=False, start_from_latent_avg=True, learn_in_w=False))


def _encoder():
    from e4s_b200.encoders.psp_encoders import FSEncoder_PSP
    return FSEncoder_PSP()


def _encoder_planes(m):
    return (m._prepared("in", m.input_layer[0].weight, pad_cin_to=32),
            m._prepared("0.c2s", m.body[0].res_layer[3].weight, s2d=True))


def _gpen_conv():
    from e4s_b200.gpen.gpen_model import ConvLayer
    return ConvLayer(16, 32, 3)


def _bisenet():
    from e4s_b200.face_parsing.model import BiSeNet
    return BiSeNet(n_classes=19)


def _parsenet():
    from e4s_b200.gpen.face_parse.parse_model import ParseNet
    return ParseNet(512, 512, 32, 64, 19, norm_type='bn', relu_type='LeakyReLU', ch_range=[32, 256])


def _rrdbnet():
    from e4s_b200.gpen.sr_model.rrdbnet_arch import RRDBNet
    return RRDBNet(num_in_ch=3, num_out_ch=3, num_feat=32, num_block=2, num_grow_ch=32, scale=4)


def _retinaface():
    from e4s_b200.gpen.face_detect.data import cfg_re50
    from e4s_b200.gpen.face_detect.facemodels.retinaface import RetinaFace
    return RetinaFace(cfg=cfg_re50, phase='test')


def _kp_detector():
    from e4s_b200.face_vid2vid.modules.keypoint_detector import KPDetector
    from oracle import vid2vid_kp_oracle as O
    return KPDetector(**O.PARAMS)


def _he_estimator():
    from e4s_b200.face_vid2vid.modules.keypoint_detector import HEEstimator
    from oracle import vid2vid_kp_oracle as O
    return HEEstimator(**O.HE_PARAMS)


def _dense_motion():
    from e4s_b200.face_vid2vid.modules.dense_motion import DenseMotionNetwork
    from oracle import vid2vid_motion_oracle as O
    return DenseMotionNetwork(**O.PARAMS)


def _spade_generator():
    from e4s_b200.face_vid2vid.modules.generator import OcclusionAwareSPADEGenerator
    from oracle import vid2vid_gen_oracle as O
    return OcclusionAwareSPADEGenerator(**O.PARAMS)


# (module factory, the call that returns its prepared operands)
CASES = {
    "ModulatedConv2d": (_modconv, lambda m: m.prepared()),
    "EqualLinear": (_equal_linear, lambda m: m._frozen()),
    "Net3": (_net3, lambda m: m._stacked_mlps()),
    "FSEncoder_PSP": (_encoder, _encoder_planes),
    "gpen.ConvLayer": (_gpen_conv, lambda m: m._prepared(m[0])),
    "BiSeNet": (_bisenet, lambda m: m._prepared(CPU)),
    "ParseNet": (_parsenet, lambda m: m._prepared(CPU)),
    "RRDBNet": (_rrdbnet, lambda m: m._prepared(CPU)),
    "RetinaFace": (_retinaface, lambda m: m._prepared(CPU)),
    "KPDetector": (_kp_detector, lambda m: m._prepared(CPU)),
    "HEEstimator": (_he_estimator, lambda m: m._prepared(CPU)),
    "DenseMotionNetwork": (_dense_motion, lambda m: m._prepared(CPU)),
    "OcclusionAwareSPADEGenerator": (_spade_generator, lambda m: m._prepared(CPU)),
}


def _leaves(x):
    """The prepared structure flattened to its tensors and plain values, in a fixed order."""
    if isinstance(x, dict):
        return [v for k in sorted(x) for v in _leaves(x[k])]
    if isinstance(x, (list, tuple)):
        return [v for e in x for v in _leaves(e)]
    if hasattr(x, "w_hilo"):                     # PreparedConv
        return [getattr(x, f) for f in CONV_FIELDS]
    return [x]


def _assert_same_values(got, want):
    assert len(got) == len(want)
    for g, w in zip(got, want):
        if isinstance(w, torch.Tensor):
            assert isinstance(g, torch.Tensor) and g.dtype == w.dtype and torch.equal(g, w)
        else:
            assert g == w


def _changed(got, old):
    return any(isinstance(g, torch.Tensor) and not torch.equal(g, o) for g, o in zip(got, old))


def _other_state(m, scale, shift):
    return {k: v * scale + shift if v.is_floating_point() else v.clone() for k, v in m.state_dict().items()}


def _fresh(make, call, state):
    """Operands of a new module of the same kind holding `state`."""
    f = make().eval()
    f.load_state_dict(state)
    return _leaves(call(f))


@pytest.mark.parametrize("case", list(CASES))
def test_prepared_cache(case):
    make, call = CASES[case]
    torch.manual_seed(0)
    m = make().eval()
    with torch.no_grad():
        first = _leaves(call(m))
        assert any(isinstance(t, torch.Tensor) for t in first)
        again = _leaves(call(m))
        assert all(a is b for a, b in zip(again, first)), "unchanged weights rebuilt"

        # load_state_dict: picked up by the version counters
        state = _other_state(m, 0.75, 0.02)
        m.load_state_dict(state)
        got = _leaves(call(m))
        assert _changed(got, first)
        _assert_same_values(got, _fresh(make, call, state))

        # an ordinary in-place op on the parameters
        for p in m.parameters():
            p.mul_(1.5)
        prev, got = got, _leaves(call(m))
        assert _changed(got, prev)
        _assert_same_values(got, _fresh(make, call, m.state_dict()))

        # a write through .data bumps no version: invalidate_prepared on an enclosing module drops the entry
        state = _other_state(m, 1.25, 0.01)
        versions = [t._version for t in m.state_dict().values()]
        for k, t in m.state_dict(keep_vars=True).items():
            t.data.copy_(state[k])
        assert [t._version for t in m.state_dict().values()] == versions
        e4s_b200.invalidate_prepared(nn.ModuleList([m]))
        got = _leaves(call(m))
        _assert_same_values(got, _fresh(make, call, state))


def test_invalidate_rebuilds_dgrad_planes():
    """The backward's flipped weights follow the forward operands through invalidate_prepared."""
    m = _modconv().eval()
    with torch.no_grad():
        MB._dgrad_planes(m.prepared())
        MB._dgrad_weights(m.prepared())
        w = torch.randn_like(m.weight)
        m.weight.data.copy_(w)
        e4s_b200.invalidate_prepared(nn.Sequential(m))
        new = _modconv().eval()
        new.weight.copy_(w)
        want = new.prepared().wt.flip(1)
        assert torch.equal(m.prepared().wt, new.prepared().wt)
        assert torch.equal(MB._dgrad_planes(m.prepared()), K.split_bf16(want.contiguous()))
        assert torch.equal(MB._dgrad_weights(m.prepared()), want.permute(0, 1, 3, 2).contiguous())
