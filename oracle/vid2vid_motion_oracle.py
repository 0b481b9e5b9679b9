"""CPU torch restatement of face-vid2vid's DenseMotionNetwork on vox-256.yaml (src/pretrained/face_vid2vid/modules/
dense_motion.py and the util.py blocks it uses), eval mode, no jacobian, plus a seeded stand-in checkpoint and inputs.

    layers(state, feature, kp_driving, kp_source)   every intermediate; 'mask', 'deformation', 'occlusion_map' at the end
    forward(state, feature, kp_driving, kp_source)  -> {'mask', 'deformation', 'occlusion_map'}

Runs in the dtype and on the device of `feature` (float64 for the reference of the kernel tests).  The stand-in's BatchNorm running
statistics are those of a seeded feature, and its mask and occlusion weights are scaled so that the softmax is neither
one-hot nor uniform and the occlusion map spreads over (0, 1).  oracle/make_golden_vid2vid_motion.py pins this file to
the unmodified reference.
"""
from __future__ import annotations

import math

import torch
import torch.nn.functional as F

PARAMS = dict(block_expansion=32, num_blocks=5, max_features=1024, num_kp=15, feature_channel=32, reshape_depth=16,
              compress=4, estimate_occlusion_map=True)
D, H, W = 16, 64, 64
NK = PARAMS["num_kp"] + 1
IN_CH = NK * (PARAMS["compress"] + 1)          # 80
OUT_CH = PARAMS["block_expansion"] + IN_CH     # 112
EPS = 1e-5


def _down_io(i):
    e, mx = PARAMS["block_expansion"], PARAMS["max_features"]
    return (IN_CH if i == 0 else min(mx, e * 2 ** i)), min(mx, e * 2 ** (i + 1))


def _up_io(j):
    """Decoder up block j (the reference's order: the deepest first)."""
    e, mx, n = PARAMS["block_expansion"], PARAMS["max_features"], PARAMS["num_blocks"]
    i = n - 1 - j
    return (1 if i == n - 1 else 2) * min(mx, e * 2 ** (i + 1)), min(mx, e * 2 ** i)


def make_coordinate_grid(d, h, w, dtype=torch.float32) -> torch.Tensor:
    """[d, h, w, 3]: (x, y, z), each 2 (i / (n - 1)) - 1."""
    ax = lambda n: 2 * (torch.arange(n, dtype=dtype) / (n - 1)) - 1  # noqa: E731
    x, y, z = ax(w), ax(h), ax(d)
    return torch.stack([x.view(1, 1, -1).expand(d, h, w), y.view(1, -1, 1).expand(d, h, w), z.view(-1, 1, 1).expand(d, h, w)], 3)


def _bn(x, st, p, calibrate=False):
    if calibrate:
        st[p + "running_mean"] = x.mean((0, 2, 3, 4)).float()
        st[p + "running_var"] = x.var((0, 2, 3, 4)).float()
    c = lambda k: st[p + k].to(x)  # noqa: E731
    return F.batch_norm(x, c("running_mean"), c("running_var"), c("weight"), c("bias"), False, 0.0, EPS)


def sparse_motions(kd, ks, d=D, h=H, w=W) -> torch.Tensor:
    """[B, 16, d, h, w, 3]: the identity grid, then grid - kp_driving[k] + kp_source[k]."""
    b = kd.shape[0]
    grid = make_coordinate_grid(d, h, w, kd.dtype).to(kd).view(1, 1, d, h, w, 3)
    moved = grid - kd.view(b, -1, 1, 1, 1, 3) + ks.view(b, -1, 1, 1, 1, 3)
    return torch.cat([grid.expand(b, 1, d, h, w, 3), moved], 1)


def heatmaps(kd, ks, d=D, h=H, w=W) -> torch.Tensor:
    """[B, 16, d, h, w]: 0, then exp(-0.5 |g - kd|^2 / 0.01) - exp(-0.5 |g - ks|^2 / 0.01)."""
    grid = make_coordinate_grid(d, h, w, kd.dtype).to(kd).view(1, 1, d, h, w, 3)
    g = lambda kp: torch.exp(-0.5 * ((grid - kp.view(*kp.shape[:2], 1, 1, 1, 3)) ** 2).sum(-1) / 0.01)  # noqa: E731
    hm = g(kd) - g(ks)
    return torch.cat([torch.zeros_like(hm[:, :1]), hm], 1)


def layers(st: dict, feature, kd, ks, calibrate: bool = False) -> dict:
    """Every intermediate of the forward.  calibrate: set every BatchNorm's running statistics to those of its input on
    the way (the stand-in's construction)."""
    c = lambda k: st[k].to(feature)  # noqa: E731
    kd, ks = kd.to(feature), ks.to(feature)
    out = {}
    b, _, d, h, w = feature.shape
    comp = F.relu(_bn(F.conv3d(feature, c("compress.weight"), c("compress.bias")), st, "norm.", calibrate))
    out["comp"] = comp
    motions = sparse_motions(kd, ks, d, h, w)
    out["motions"] = motions
    rep = comp.unsqueeze(1).expand(b, NK, *comp.shape[1:]).reshape(b * NK, -1, d, h, w)
    deformed = F.grid_sample(rep, motions.reshape(b * NK, d, h, w, 3), align_corners=False).view(b, NK, -1, d, h, w)
    x = torch.cat([heatmaps(kd, ks, d, h, w).unsqueeze(2), deformed], 2).view(b, -1, d, h, w)
    out["input"] = x
    skips = [x]
    for i in range(PARAMS["num_blocks"]):
        p = f"hourglass.encoder.down_blocks.{i}."
        y = F.relu(_bn(F.conv3d(skips[-1], c(p + "conv.weight"), c(p + "conv.bias"), padding=1), st, p + "norm.", calibrate))
        out[f"down{i}_conv"] = y
        skips.append(F.avg_pool3d(y, (1, 2, 2)))
        out[f"down{i}"] = skips[-1]
    y = skips.pop()
    for j in range(PARAMS["num_blocks"]):
        p = f"hourglass.decoder.up_blocks.{j}."
        y = F.interpolate(y, scale_factor=(1, 2, 2))
        y = F.relu(_bn(F.conv3d(y, c(p + "conv.weight"), c(p + "conv.bias"), padding=1), st, p + "norm.", calibrate))
        out[f"up{j}"] = y
        y = torch.cat([y, skips.pop()], 1)
    p = "hourglass.decoder."
    pred = F.relu(_bn(F.conv3d(y, c(p + "conv.weight"), c(p + "conv.bias"), padding=1), st, p + "norm.", calibrate))
    out["prediction"] = pred
    logits = F.conv3d(pred, c("mask.weight"), c("mask.bias"), padding=3)
    out["mask_logits"] = logits
    mask = F.softmax(logits, dim=1)
    out["mask"] = mask
    out["deformation"] = (motions.permute(0, 1, 5, 2, 3, 4) * mask.unsqueeze(2)).sum(1).permute(0, 2, 3, 4, 1)
    occ_logits = F.conv2d(pred.reshape(b, -1, h, w), c("occlusion.weight"), c("occlusion.bias"), padding=3)
    out["occlusion_logits"] = occ_logits
    out["occlusion_map"] = torch.sigmoid(occ_logits)
    return out


def forward(st: dict, feature, kd, ks) -> dict:
    o = layers(st, feature, kd, ks)
    return {k: o[k] for k in ("mask", "deformation", "occlusion_map")}


def synthetic_feature(b: int, seed: int) -> torch.Tensor:
    """Seeded smooth fp32 stand-in for the generator's 3D feature, [b, 32, 16, 64, 64]."""
    g = torch.Generator().manual_seed(seed)
    low = torch.randn((b, PARAMS["feature_channel"], 4, 8, 8), generator=g)
    x = F.interpolate(low, size=(D, H, W), mode="trilinear", align_corners=False)
    return (x + 0.1 * torch.randn((b, PARAMS["feature_channel"], D, H, W), generator=g)).contiguous()


def synthetic_keypoints(b: int, seed: int):
    """Seeded (kp_driving, kp_source) values [b, 15, 3]: keypoints over [-1, 1] and a few near and beyond +-1 (sparse
    motions that leave the volume), the source a displaced driving."""
    g = torch.Generator().manual_seed(seed)
    kd = torch.rand((b, PARAMS["num_kp"], 3), generator=g) * 1.8 - 0.9
    kd[:, 0] = torch.tensor([1.05, -0.98, 0.99])
    kd[:, 1] = torch.tensor([-1.1, 1.02, -1.03])
    ks = kd + 0.25 * torch.randn((b, PARAMS["num_kp"], 3), generator=g)
    ks[:, 2] = torch.tensor([0.97, 1.08, -1.06])
    return kd.contiguous(), ks.contiguous()


def synthetic_state(seed: int = 0) -> dict:
    """Seeded stand-in for the generator checkpoint's dense_motion_network.* entries (88 keys, prefix stripped)."""
    g = torch.Generator().manual_seed(seed)
    st = {}

    def conv(prefix, shape, gain=1.0):
        st[prefix + "weight"] = torch.randn(shape, generator=g) * (gain / math.sqrt(math.prod(shape[1:])))
        st[prefix + "bias"] = torch.randn(shape[0], generator=g) * 0.1

    def bn(prefix, ch):
        st[prefix + "weight"] = 1.0 + 0.3 * torch.randn(ch, generator=g)
        st[prefix + "bias"] = 0.2 * torch.randn(ch, generator=g)
        st[prefix + "running_mean"] = torch.zeros(ch)
        st[prefix + "running_var"] = torch.ones(ch)
        st[prefix + "num_batches_tracked"] = torch.tensor(1000, dtype=torch.int64)

    for i in range(PARAMS["num_blocks"]):
        cin, cout = _down_io(i)
        conv(f"hourglass.encoder.down_blocks.{i}.conv.", (cout, cin, 3, 3, 3))
        bn(f"hourglass.encoder.down_blocks.{i}.norm.", cout)
    for j in range(PARAMS["num_blocks"]):
        cin, cout = _up_io(j)
        conv(f"hourglass.decoder.up_blocks.{j}.conv.", (cout, cin, 3, 3, 3))
        bn(f"hourglass.decoder.up_blocks.{j}.norm.", cout)
    conv("hourglass.decoder.conv.", (OUT_CH, OUT_CH, 3, 3, 3))
    bn("hourglass.decoder.norm.", OUT_CH)
    conv("mask.", (NK, OUT_CH, 7, 7, 7))
    conv("compress.", (PARAMS["compress"], PARAMS["feature_channel"], 1, 1, 1))
    bn("norm.", PARAMS["compress"])
    conv("occlusion.", (1, OUT_CH * PARAMS["reshape_depth"], 7, 7))
    # BatchNorm statistics of a seeded pair, then the heads scaled: mask logits with a spread of 1.75 around their
    # per-channel means (the fp32 forward's mask and deformation errors grow with that spread), occlusion logits with a
    # spread of 1.5 around 0
    kd, ks = synthetic_keypoints(1, seed + 1)
    lay = layers(st, synthetic_feature(1, seed + 1), kd, ks, calibrate=True)
    ml = lay["mask_logits"] - st["mask.bias"].view(1, -1, 1, 1, 1)
    s = 1.75 / float(ml.std())
    st["mask.weight"] = st["mask.weight"] * s
    st["mask.bias"] = 0.5 * torch.randn(NK, generator=g) - ml.mean((0, 2, 3, 4)) * s
    ol = lay["occlusion_logits"] - st["occlusion.bias"]
    s = 1.5 / float(ol.std())
    st["occlusion.weight"] = st["occlusion.weight"] * s
    st["occlusion.bias"] = -ol.mean().reshape(1) * s
    return st
