"""torch restatement of face-vid2vid's OcclusionAwareSPADEGenerator on vox-256.yaml (src/pretrained/face_vid2vid/modules/
generator.py and the util.py blocks it uses), eval mode, no jacobian, plus a seeded stand-in checkpoint.

    layers(state, source, kp_driving, kp_source)    every intermediate; 'mask', 'occlusion_map', 'prediction' at the end
    forward(state, source, kp_driving, kp_source)   -> {'mask', 'occlusion_map', 'prediction'}

Either takes motion= {'mask', 'deformation', 'occlusion_map'} in place of the dense-motion network's outputs (the
generator around a given dense motion).

Runs in the dtype and on the device of `source` (float64 for the reference of the kernel tests).  The dense-motion network
is oracle/vid2vid_motion_oracle.py.  The stand-in (386 keys) is not degenerate: its BatchNorm running statistics are those
of seeded faces, its spectral-norm u and v come from three power iterations (so u . W v is near, not at, the largest
singular value, and far from 1), its SPADE gamma / beta convolutions are scaled to a spread of 0.3 around zero (the
modulation moves every block), and conv_img to logits of spread 1.2 (the prediction is not saturated).
oracle/make_golden_vid2vid_gen.py pins this file to the unmodified reference.
"""
from __future__ import annotations

import math

import torch
import torch.nn.functional as F

from oracle import vid2vid_kp_oracle as KPO
from oracle import vid2vid_motion_oracle as MO

PARAMS = dict(image_channel=3, feature_channel=32, num_kp=15, block_expansion=64, max_features=512, num_down_blocks=2,
              reshape_channel=32, reshape_depth=16, num_resblocks=6, estimate_occlusion_map=True,
              dense_motion_params=dict(block_expansion=32, max_features=1024, num_blocks=5, reshape_depth=16, compress=4),
              estimate_jacobian=False)
EPS = 1e-5
# SPADEResnetBlock (fin, fout) of the decoder
BLOCKS = [(f"G_middle_{i}", 512, 512) for i in range(6)] + [("up_0", 512, 256), ("up_1", 256, 64)]
GAMMA_SPREAD, LOGIT_SPREAD = 0.3, 1.2


def _bn(x, st, p, calibrate=False):
    if calibrate:
        dims = [0] + list(range(2, x.dim()))
        st[p + "running_mean"] = x.mean(dims).float()
        st[p + "running_var"] = x.var(dims).float()
    c = lambda k: st[p + k].to(x)  # noqa: E731
    return F.batch_norm(x, c("running_mean"), c("running_var"), c("weight"), c("bias"), False, 0.0, EPS)


def sn_weight(st, p, like):
    """Eval-mode spectral-norm weight: weight_orig / (u . W v), with the stored u and v."""
    w = st[p + "weight_orig"].to(like)
    sigma = torch.dot(st[p + "weight_u"].to(like), torch.mv(w.reshape(w.shape[0], -1), st[p + "weight_v"].to(like)))
    return w / sigma


def spade(st, p, x, seg, out, name, calibrate=False):
    c = lambda k: st[p + k].to(x)  # noqa: E731
    normalized = F.instance_norm(x, eps=EPS)
    segmap = F.interpolate(seg, size=x.shape[2:], mode='nearest')
    actv = F.relu(F.conv2d(segmap, c("mlp_shared.0.weight"), c("mlp_shared.0.bias"), padding=1))
    if calibrate:
        for k in ("mlp_gamma.", "mlp_beta."):
            raw = F.conv2d(actv, c(k + "weight"), padding=1)
            s = GAMMA_SPREAD / float(raw.std())
            st[p + k + "weight"] = (st[p + k + "weight"] * s).float()
            st[p + k + "bias"] = (st[p + k + "bias"] * GAMMA_SPREAD - raw.mean((0, 2, 3)) * s).float()
    gamma = F.conv2d(actv, c("mlp_gamma.weight"), c("mlp_gamma.bias"), padding=1)
    beta = F.conv2d(actv, c("mlp_beta.weight"), c("mlp_beta.bias"), padding=1)
    out[name + ".gamma"], out[name + ".beta"] = gamma, beta
    o = normalized * (1 + gamma) + beta
    out[name] = o
    return o


def spade_block(st, p, x, seg, out, calibrate=False):
    c = lambda k: st[p + k].to(x)  # noqa: E731
    x_s = x
    if p + "conv_s.weight_orig" in st:
        x_s = F.conv2d(spade(st, p + "norm_s.", x, seg, out, p + "norm_s", calibrate), sn_weight(st, p + "conv_s.", x))
        out[p + "conv_s"] = x_s
    dx = F.conv2d(F.leaky_relu(spade(st, p + "norm_0.", x, seg, out, p + "norm_0", calibrate), 2e-1),
                  sn_weight(st, p + "conv_0.", x), c("conv_0.bias"), padding=1)
    out[p + "conv_0"] = dx
    dx = F.conv2d(F.leaky_relu(spade(st, p + "norm_1.", dx, seg, out, p + "norm_1", calibrate), 2e-1),
                  sn_weight(st, p + "conv_1.", x), c("conv_1.bias"), padding=1)
    o = x_s + dx
    out[p + "out"] = o
    return o


def layers(st: dict, source, kd, ks, calibrate: bool = False, motion: dict = None) -> dict:
    """Every intermediate of the forward.  calibrate: set the BatchNorm statistics, the gamma / beta and conv_img scales
    on the way (the stand-in's construction).  motion: the dense-motion outputs to use instead of the network's."""
    c = lambda k: st[k].to(source)  # noqa: E731
    out = {}
    x = F.relu(_bn(F.conv2d(source, c("first.conv.weight"), c("first.conv.bias"), padding=1), st, "first.norm.", calibrate))
    out["first"] = x
    for i in range(PARAMS["num_down_blocks"]):
        p = f"down_blocks.{i}."
        x = F.avg_pool2d(F.relu(_bn(F.conv2d(x, c(p + "conv.weight"), c(p + "conv.bias"), padding=1), st, p + "norm.",
                                    calibrate)), (2, 2))
        out[f"down{i}"] = x
    x = F.conv2d(x, c("second.weight"), c("second.bias"))
    out["second"] = x
    bs, _, h, w = x.shape
    f = x.view(bs, PARAMS["reshape_channel"], PARAMS["reshape_depth"], h, w)
    for i in range(PARAMS["num_resblocks"]):
        p = f"resblocks_3d.3dr{i}."
        a = F.relu(_bn(f, st, p + "norm1.", calibrate))
        a = F.relu(_bn(F.conv3d(a, c(p + "conv1.weight"), c(p + "conv1.bias"), padding=1), st, p + "norm2.", calibrate))
        f = F.conv3d(a, c(p + "conv2.weight"), c(p + "conv2.bias"), padding=1) + f
        out[f"res3d{i}"] = f
    dm_st = {k[len("dense_motion_network."):]: v for k, v in st.items() if k.startswith("dense_motion_network.")}
    dm = {k: v.to(f) for k, v in motion.items()} if motion is not None else MO.layers(dm_st, f, kd, ks, calibrate=calibrate)
    if calibrate:
        st.update({"dense_motion_network." + k: v for k, v in dm_st.items()})
    out["mask"], out["occlusion_map"], out["deformation"] = dm["mask"], dm["occlusion_map"], dm["deformation"]
    warped = F.grid_sample(f, dm["deformation"], align_corners=False)
    out["warped"] = warped
    x = warped.reshape(bs, -1, h, w)
    x = F.leaky_relu(_bn(F.conv2d(x, c("third.conv.weight"), c("third.conv.bias"), padding=1), st, "third.norm.", calibrate))
    out["third"] = x
    seg = F.conv2d(x, c("fourth.weight"), c("fourth.bias")) * dm["occlusion_map"]
    out["fourth"] = seg
    x = F.conv2d(seg, c("decoder.fc.weight"), c("decoder.fc.bias"), padding=1)
    out["fc"] = x
    for name, _, _ in BLOCKS:
        if name.startswith("up"):
            x = F.interpolate(x, scale_factor=2)
        x = spade_block(st, f"decoder.{name}.", x, seg, out, calibrate)
    x = F.conv2d(F.leaky_relu(x, 2e-1), c("decoder.conv_img.weight"), c("decoder.conv_img.bias"), padding=1)
    if calibrate:
        s = LOGIT_SPREAD / float(x.std())
        st["decoder.conv_img.weight"] = (st["decoder.conv_img.weight"] * s).float()
        st["decoder.conv_img.bias"] = (st["decoder.conv_img.bias"] * s - x.mean((0, 2, 3)) * s).float()
        x = (x - x.mean((0, 2, 3), keepdim=True)) * s
    out["logits"] = x
    out["prediction"] = torch.sigmoid(x)
    return out


def forward(st: dict, source, kd, ks, motion: dict = None) -> dict:
    o = layers(st, source, kd, ks, motion=motion)
    return {k: o[k] for k in ("mask", "occlusion_map", "prediction")}


def synthetic_state(seed: int = 0) -> dict:
    """Seeded stand-in for checkpoint['generator'] (386 keys)."""
    g = torch.Generator().manual_seed(seed)
    st = {"dense_motion_network." + k: v for k, v in MO.synthetic_state(seed).items()}

    def conv(prefix, shape, bias=True, gain=1.0):
        st[prefix + "weight"] = torch.randn(shape, generator=g) * (gain / math.sqrt(math.prod(shape[1:])))
        if bias:
            st[prefix + "bias"] = torch.randn(shape[0], generator=g) * 0.1

    def bn(prefix, ch):
        st[prefix + "weight"] = 1.0 + 0.3 * torch.randn(ch, generator=g)
        st[prefix + "bias"] = 0.2 * torch.randn(ch, generator=g)
        st[prefix + "running_mean"] = torch.zeros(ch)
        st[prefix + "running_var"] = torch.ones(ch)
        st[prefix + "num_batches_tracked"] = torch.tensor(1000, dtype=torch.int64)

    def sn_conv(prefix, shape, bias=True):
        w = torch.randn(shape, generator=g) * (1.5 / math.sqrt(math.prod(shape[1:])))
        wm = w.reshape(shape[0], -1).double()
        u = F.normalize(torch.randn(shape[0], generator=g, dtype=torch.float64), dim=0)
        for _ in range(3):
            v = F.normalize(torch.mv(wm.t(), u), dim=0)
            u = F.normalize(torch.mv(wm, v), dim=0)
        st[prefix + "weight_orig"] = w
        if bias:
            st[prefix + "bias"] = torch.randn(shape[0], generator=g) * 0.1
        st[prefix + "weight_u"], st[prefix + "weight_v"] = u.float(), v.float()

    conv("first.conv.", (64, 3, 3, 3))
    bn("first.norm.", 64)
    for i, (ci, co) in enumerate(((64, 128), (128, 256))):
        conv(f"down_blocks.{i}.conv.", (co, ci, 3, 3))
        bn(f"down_blocks.{i}.norm.", co)
    conv("second.", (512, 256, 1, 1))
    for i in range(PARAMS["num_resblocks"]):
        p = f"resblocks_3d.3dr{i}."
        conv(p + "conv1.", (32, 32, 3, 3, 3))
        conv(p + "conv2.", (32, 32, 3, 3, 3), gain=0.5)
        bn(p + "norm1.", 32)
        bn(p + "norm2.", 32)
    conv("third.conv.", (256, 512, 3, 3))
    bn("third.norm.", 256)
    conv("fourth.", (256, 256, 1, 1))
    conv("decoder.fc.", (512, 256, 3, 3))
    for name, fin, fout in BLOCKS:
        p = f"decoder.{name}."
        fmid = min(fin, fout)
        sn_conv(p + "conv_0.", (fmid, fin, 3, 3))
        sn_conv(p + "conv_1.", (fout, fmid, 3, 3))
        norms = [("norm_0.", fin), ("norm_1.", fmid)]
        if fin != fout:
            sn_conv(p + "conv_s.", (fout, fin, 1, 1), bias=False)
            norms.append(("norm_s.", fin))
        for n, ch in norms:
            conv(p + n + "mlp_shared.0.", (128, 256, 3, 3))
            conv(p + n + "mlp_gamma.", (ch, 128, 3, 3))
            conv(p + n + "mlp_beta.", (ch, 128, 3, 3))
    conv("decoder.conv_img.", (3, 64, 3, 3))
    kd, ks = MO.synthetic_keypoints(2, seed + 1)
    with torch.no_grad():
        layers(st, KPO.synthetic_faces(2, seed + 1), kd, ks, calibrate=True)
    return st
