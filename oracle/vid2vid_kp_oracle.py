"""CPU torch restatement of face-vid2vid's KPDetector and HEEstimator on vox-256.yaml (src/pretrained/face_vid2vid/
modules/keypoint_detector.py and the util.py blocks they use), eval mode, estimate_jacobian False, and of driven_demo.py's
pose arithmetic, plus seeded stand-in checkpoints.

    kp_forward(state, x)     x [B, 3, 256, 256] in [0, 1] -> {'value': [B, 15, 3]}
    he_forward(he_state, x)  -> {'yaw', 'pitch', 'roll': [B, 66], 't': [B, 3], 'exp': [B, 45]}
    keypoint_transformation(kp, he) -> [B, 15, 3]

The stand-in is scaled so that the tests see something: every keypoint's heatmap is peaked (softmax at T = 0.1 of logits
with a spread of a few units), so the keypoints spread over [-1, 1], and the BatchNorm running statistics are far from
(0, 1).  oracle/make_golden_vid2vid_kp.py pins this file to the unmodified reference.
"""
from __future__ import annotations

import math

import torch
import torch.nn.functional as F

PARAMS = dict(block_expansion=32, max_features=1024, num_blocks=5, reshape_channel=16384, reshape_depth=16, num_kp=15,
              temperature=0.1, estimate_jacobian=False, scale_factor=0.25, feature_channel=32, image_channel=3)
SIZE = 256
EPS = 1e-5


def _down_io(i):
    e, mx = PARAMS["block_expansion"], PARAMS["max_features"]
    return (PARAMS["image_channel"] if i == 0 else min(mx, e * 2 ** i)), min(mx, e * 2 ** (i + 1))


def _up_io(i):
    e, mx, n = PARAMS["block_expansion"], PARAMS["max_features"], PARAMS["num_blocks"]
    return min(mx, e * 2 ** (n - i)), min(mx, e * 2 ** (n - i - 1))


def anti_alias_filter(channels=3, scale=0.25) -> torch.Tensor:
    """AntiAliasInterpolation2d's buffer: [channels, 1, k, k], a normalised Gaussian (sigma (1 / scale - 1) / 2)."""
    sigma = (1 / scale - 1) / 2
    k = 2 * round(sigma * 4) + 1
    g = torch.arange(k, dtype=torch.float32)
    g1 = torch.exp(-(g - (k - 1) / 2) ** 2 / (2 * sigma ** 2))
    ker = g1.view(-1, 1) * g1.view(1, -1)
    ker = ker / ker.sum()
    return ker.view(1, 1, k, k).repeat(channels, 1, 1, 1)


def synthetic_state(seed: int = 0) -> dict:
    """Seeded stand-in for checkpoint['kp_detector'] with the reference's 75 keys and shapes."""
    g = torch.Generator().manual_seed(seed)
    st = {}

    def add_conv(prefix, shape, gain):
        fan = math.prod(shape[1:])
        st[prefix + "weight"] = torch.randn(shape, generator=g) * (gain / math.sqrt(fan))
        st[prefix + "bias"] = torch.randn(shape[0], generator=g) * 0.1

    def add_bn(prefix, c):
        st[prefix + "weight"] = 1.0 + 0.3 * torch.randn(c, generator=g)
        st[prefix + "bias"] = 0.2 * torch.randn(c, generator=g)
        st[prefix + "running_mean"] = 0.3 * torch.randn(c, generator=g)
        st[prefix + "running_var"] = 0.5 + torch.rand(c, generator=g) * 1.5
        st[prefix + "num_batches_tracked"] = torch.tensor(1000, dtype=torch.int64)

    for i in range(PARAMS["num_blocks"]):
        cin, cout = _down_io(i)
        add_conv(f"predictor.down_blocks.down{i}.conv.", (cout, cin, 3, 3), 2.0)
        add_bn(f"predictor.down_blocks.down{i}.norm.", cout)
    add_conv("predictor.conv.", (PARAMS["reshape_channel"], _down_io(PARAMS["num_blocks"] - 1)[1], 1, 1), 1.5)
    for i in range(PARAMS["num_blocks"]):
        cin, cout = _up_io(i)
        add_conv(f"predictor.up_blocks.up{i}.conv.", (cout, cin, 3, 3, 3), 2.0)
        add_bn(f"predictor.up_blocks.up{i}.norm.", cout)
    add_conv("kp.", (PARAMS["num_kp"], _up_io(PARAMS["num_blocks"] - 1)[1], 3, 3, 3), 0.08)
    st["down.weight"] = anti_alias_filter(PARAMS["image_channel"], PARAMS["scale_factor"])
    return st


def _bn(x, st, p):
    return F.batch_norm(x, st[p + "running_mean"], st[p + "running_var"], st[p + "weight"], st[p + "bias"], False, 0.0, EPS)


def make_coordinate_grid(d, h, w) -> torch.Tensor:
    """[d, h, w, 3]: (x, y, z), each 2 (i / (n - 1)) - 1."""
    x = 2 * (torch.arange(w, dtype=torch.float32) / (w - 1)) - 1
    y = 2 * (torch.arange(h, dtype=torch.float32) / (h - 1)) - 1
    z = 2 * (torch.arange(d, dtype=torch.float32) / (d - 1)) - 1
    return torch.stack([x.view(1, 1, -1).expand(d, h, w), y.view(1, -1, 1).expand(d, h, w), z.view(-1, 1, 1).expand(d, h, w)], 3)


def heatmap_kp(prediction: torch.Tensor, temperature: float) -> torch.Tensor:
    """prediction [B, K, D, H, W] -> [B, K, 3]: softmax(prediction / T) over the voxels, expectation of the grid."""
    b, k, d, h, w = prediction.shape
    heat = F.softmax(prediction.reshape(b, k, -1) / temperature, dim=2).view(b, k, d, h, w, 1)
    return (heat * make_coordinate_grid(d, h, w).to(prediction)).sum(dim=(2, 3, 4))


def kp_layers(st: dict, x: torch.Tensor) -> dict:
    """Every intermediate of the forward (the down blocks' pooled outputs, the 3D operand, the up blocks, the kp logits)."""
    out = {}
    filt = st["down.weight"]
    ka = filt.shape[-1] // 2
    h = F.conv2d(F.pad(x, (ka, ka, ka, ka)), filt, groups=x.shape[1])[:, :, ::4, ::4]
    out["down"] = h
    for i in range(PARAMS["num_blocks"]):
        p = f"predictor.down_blocks.down{i}."
        h = F.conv2d(h, st[p + "conv.weight"], st[p + "conv.bias"], padding=1)
        h = F.avg_pool2d(F.relu(_bn(h, st, p + "norm.")), 2)
        out[f"down{i}"] = h
    h = F.conv2d(h, st["predictor.conv.weight"], st["predictor.conv.bias"])
    b, c, hh, ww = h.shape
    h = h.view(b, c // PARAMS["reshape_depth"], PARAMS["reshape_depth"], hh, ww)
    out["reshape"] = h
    for i in range(PARAMS["num_blocks"]):
        p = f"predictor.up_blocks.up{i}."
        h = F.interpolate(h, scale_factor=(1, 2, 2))
        h = F.relu(_bn(F.conv3d(h, st[p + "conv.weight"], st[p + "conv.bias"], padding=1), st, p + "norm."))
        out[f"up{i}"] = h
    out["kp"] = F.conv3d(h, st["kp.weight"], st["kp.bias"], padding=1)
    out["value"] = heatmap_kp(out["kp"], PARAMS["temperature"])
    return out


def kp_forward(st: dict, x: torch.Tensor) -> dict:
    return {"value": kp_layers(st, x)["value"]}


def synthetic_faces(b: int, seed: int) -> torch.Tensor:
    """Seeded smooth images in [0, 1], [b, 3, 256, 256]."""
    g = torch.Generator().manual_seed(seed)
    low = torch.rand((b, 3, 16, 16), generator=g)
    img = F.interpolate(low, size=(SIZE, SIZE), mode="bicubic", align_corners=False)
    return (img + 0.05 * torch.rand((b, 3, SIZE, SIZE), generator=g)).clamp(0, 1)


# ---------------------------------------------------------------------------------------------------------- HEEstimator
HE_PARAMS = dict(block_expansion=64, max_features=2048, num_bins=66, feature_channel=32, num_kp=15, image_channel=3,
                 estimate_jacobian=False)
# (module name, in_features, stride) of every ResBottleneck, in order; the 1x1 + BN + ReLU convs come before blocks 1, 2, 4, 6
HE_BLOCKS = ([(f"block1.b1_{i}", 256, 1) for i in range(3)] + [("block2", 512, 2)] +
             [(f"block3.b3_{i}", 512, 1) for i in range(3)] + [("block4", 1024, 2)] +
             [(f"block5.b5_{i}", 1024, 1) for i in range(5)] + [("block6", 2048, 2)] +
             [(f"block7.b7_{i}", 2048, 1) for i in range(2)])
HE_CONVS = {"block1.b1_0": ("conv2", 64, 256), "block2": ("conv3", 256, 512), "block4": ("conv4", 512, 1024),
            "block6": ("conv5", 1024, 2048)}
HE_HEADS = (("fc_roll", 66), ("fc_pitch", 66), ("fc_yaw", 66), ("fc_t", 3), ("fc_exp", 45))


def he_synthetic_state(seed: int = 1) -> dict:
    """Seeded stand-in for checkpoint['he_estimator'] (402 keys).  The BatchNorm running statistics are those of seeded
    faces and the bin heads are scaled so that the softmax over the 66 bins picks angles tens of degrees apart from face
    to face."""
    g = torch.Generator().manual_seed(seed)
    st = {}

    def conv(prefix, shape, gain):
        st[prefix + "weight"] = torch.randn(shape, generator=g) * (gain / math.sqrt(math.prod(shape[1:])))
        st[prefix + "bias"] = torch.randn(shape[0], generator=g) * 0.1

    def bn(prefix, c, scale=1.0):
        st[prefix + "weight"] = scale * (1.0 + 0.3 * torch.randn(c, generator=g))
        st[prefix + "bias"] = 0.2 * torch.randn(c, generator=g)
        st[prefix + "running_mean"] = 0.3 * torch.randn(c, generator=g)
        st[prefix + "running_var"] = 0.5 + torch.rand(c, generator=g) * 1.5
        st[prefix + "num_batches_tracked"] = torch.tensor(1000, dtype=torch.int64)

    conv("conv1.", (64, 3, 7, 7), 2.0)
    bn("norm1.", 64)
    for name, cin, stride in HE_BLOCKS:
        if name in HE_CONVS:
            cname, ci, co = HE_CONVS[name]
            conv(cname + ".", (co, ci, 1, 1), 2.0)
            bn("norm" + cname[-1] + ".", co)
        mid = cin // 4
        conv(name + ".conv1.", (mid, cin, 1, 1), 2.0)
        conv(name + ".conv2.", (mid, mid, 3, 3), 2.0)
        conv(name + ".conv3.", (cin, mid, 1, 1), 1.0)
        bn(name + ".norm1.", mid)
        bn(name + ".norm2.", mid)
        bn(name + ".norm3.", cin, 0.5)
        if stride != 1:
            conv(name + ".skip.", (cin, cin, 1, 1), 1.0)
            bn(name + ".norm4.", cin)
    # BatchNorm statistics of seeded faces, as a trained network has them, keep the features face-dependent through the
    # 16 bottlenecks; the heads read the pooled features' deviation from their mean over those faces, scaled to bin
    # logits of spread ~1.5 and t / exp of spread ~0.1 / ~0.05
    pooled = he_layers(st, synthetic_faces(8, 99), heads=False, calibrate=True)["pooled"]
    mean, spread = pooled.mean(0), float((pooled - pooled.mean(0)).pow(2).mean().sqrt())
    for name, n in HE_HEADS:
        w = torch.randn((n, 2048), generator=g) * ({"fc_t": 0.1, "fc_exp": 0.05}.get(name, 1.5) / math.sqrt(2048)) / spread
        st[name + ".weight"] = w
        st[name + ".bias"] = -(w.double() @ mean.double()).float()
    return st


def _calibrating_bn(x, st, p):
    """_bn after setting the running statistics to x's own (per channel over batch and pixels)."""
    st[p + "running_mean"] = x.mean((0, 2, 3))
    st[p + "running_var"] = x.var((0, 2, 3))
    return _bn(x, st, p)


def _res(st, p, x, stride, bn=_bn):
    out = F.relu(bn(F.conv2d(x, st[p + "conv1.weight"], st[p + "conv1.bias"]), st, p + "norm1."))
    out = F.relu(bn(F.conv2d(out, st[p + "conv2.weight"], st[p + "conv2.bias"], padding=1, stride=stride), st, p + "norm2."))
    out = bn(F.conv2d(out, st[p + "conv3.weight"], st[p + "conv3.bias"]), st, p + "norm3.")
    if stride != 1:
        x = bn(F.conv2d(x, st[p + "skip.weight"], st[p + "skip.bias"], stride=stride), st, p + "norm4.")
    return F.relu(out + x)


def he_layers(st: dict, x: torch.Tensor, heads: bool = True, calibrate: bool = False) -> dict:
    """Every intermediate of HEEstimator's forward (the stem, each 1x1 + BN + ReLU, each bottleneck, the pooled features)
    and its output dict under 'out' ('yaw' is fc_roll's output and 'roll' fc_yaw's, as in the reference).  calibrate:
    set every BatchNorm's running statistics to those of x on the way (the stand-in's construction)."""
    out = {}
    bn = _calibrating_bn if calibrate else _bn
    h = F.relu(bn(F.conv2d(x, st["conv1.weight"], st["conv1.bias"], padding=3, stride=2), st, "norm1."))
    h = F.max_pool2d(h, 3, 2, 1)
    out["stem"] = h
    for name, _, stride in HE_BLOCKS:
        if name in HE_CONVS:
            cname = HE_CONVS[name][0]
            h = F.relu(bn(F.conv2d(h, st[cname + ".weight"], st[cname + ".bias"]), st, "norm" + cname[-1] + "."))
            out[cname] = h
        h = _res(st, name + ".", h, stride, bn)
        out[name] = h
    pooled = F.adaptive_avg_pool2d(h, 1).flatten(1)
    out["pooled"] = pooled
    if not heads:
        return out
    fc = {n: F.linear(pooled, st[n + ".weight"], st[n + ".bias"]) for n, _ in HE_HEADS}
    out["out"] = {"yaw": fc["fc_roll"], "pitch": fc["fc_pitch"], "roll": fc["fc_yaw"], "t": fc["fc_t"], "exp": fc["fc_exp"]}
    return out


def he_forward(st: dict, x: torch.Tensor) -> dict:
    return he_layers(st, x)["out"]


def headpose_pred_to_degree(pred):
    p = F.softmax(pred, dim=1)
    return (p * torch.arange(66, dtype=pred.dtype, device=pred.device)).sum(1) * 3 - 99


def get_rotation_matrix(yaw, pitch, roll):
    """pitch (about x) @ yaw (about y) @ roll (about z), degrees converted with / 180 * 3.14."""
    def rot(a, i, j):
        a = a / 180 * 3.14
        m = torch.eye(3, dtype=a.dtype, device=a.device).repeat(a.shape[0], 1, 1)
        c, s = torch.cos(a), torch.sin(a)
        m[:, i, i], m[:, j, j], m[:, i, j], m[:, j, i] = c, c, -s, s
        return m
    return rot(pitch, 1, 2) @ rot(yaw, 2, 0) @ rot(roll, 0, 1)


def keypoint_transformation(kp: torch.Tensor, he: dict) -> torch.Tensor:
    """Canonical kp [B, K, 3] -> R kp + t + exp."""
    r = get_rotation_matrix(headpose_pred_to_degree(he["yaw"]), headpose_pred_to_degree(he["pitch"]),
                            headpose_pred_to_degree(he["roll"]))
    return torch.einsum("bmp,bkp->bkm", r, kp) + he["t"][:, None, :] + he["exp"].reshape(kp.shape[0], -1, 3)
