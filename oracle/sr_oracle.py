"""Torch-CPU restatement of GPEN's RealESRNet x4 super-resolution (src/pretrained/gpen/sr_model/): RRDBNet.forward
(rrdbnet_arch.py:31-38, 58-62, 104-117) and RealESRNet.process (real_esrnet.py:26-59) at scale 4, written from the state
dict with torch.nn.functional, in whatever dtype / device the state and input are given in.  Also the seeded stand-in
checkpoint (no realesrnet_x4.pth can be downloaded).  Pinned against the unmodified reference by oracle/make_golden_sr.py."""
from __future__ import annotations

import math
from typing import Dict

import numpy as np
import torch
import torch.nn.functional as F

NUM_FEAT, NUM_BLOCK, NUM_GROW = 32, 23, 32        # RealESRNet.load_srmodel (real_esrnet.py:16)


# ------------------------------------------------------------------------------------------------------------ state
def param_shapes(num_in_ch: int = 3, num_out_ch: int = 3, num_feat: int = NUM_FEAT, num_block: int = NUM_BLOCK,
                 num_grow_ch: int = NUM_GROW) -> Dict[str, tuple]:
    """State-dict keys and shapes of RRDBNet(num_in_ch, num_out_ch, scale=4, num_feat, num_block, num_grow_ch)."""
    s = {}

    def conv(p, cin, cout):
        s[p + ".weight"] = (cout, cin, 3, 3)
        s[p + ".bias"] = (cout,)

    conv("conv_first", num_in_ch, num_feat)
    for i in range(num_block):
        for r in range(1, 4):
            p = f"body.{i}.rdb{r}."
            for j in range(1, 5):
                conv(p + f"conv{j}", num_feat + (j - 1) * num_grow_ch, num_grow_ch)
            conv(p + "conv5", num_feat + 4 * num_grow_ch, num_feat)
    for name in ("conv_body", "conv_up1", "conv_up2", "conv_hr"):
        conv(name, num_feat, num_feat)
    conv("conv_last", num_feat, num_out_ch)
    return s


def _key_seed(key: str) -> int:
    h = 2166136261                     # FNV-1a, 32 bit
    for ch in key.encode():
        h = ((h ^ ch) * 16777619) & 0xFFFFFFFF
    return h


def synthetic_state(seed: int = 0) -> Dict[str, torch.Tensor]:
    """Seeded stand-in for realesrnet_x4.pth's params_ema: one generator per tensor, seeded by a hash of its key and `seed`.
    Convolution weights ~ N(0, 2 / fan_in) (He initialisation without the reference's 0.1 damping, so that the dense
    branches contribute: ||0.2 x5|| / ||x|| is 0.19 .. 0.43, median 0.28, over the 69 blocks on a 32 x 32 case image),
    conv_last's ~ N(0, 2e-5 / fan_in); biases 0.1 n, conv_last's 0.5 + 0.05 n, so that ~94 % of the image lands inside
    [0, 1] and process()'s clamp and rounding both matter."""
    out = {}
    shapes = param_shapes()
    for key in sorted(shapes):
        shape = shapes[key]
        g = torch.Generator().manual_seed(_key_seed(key) ^ seed)
        t = torch.randn(shape, generator=g, dtype=torch.float32)
        last = key.startswith("conv_last.")
        if len(shape) == 4:
            t = t * math.sqrt((2e-5 if last else 2.0) / (shape[1] * 9))
        else:
            t = 0.5 + 0.05 * t if last else 0.1 * t
        out[key] = t
    return out


# ------------------------------------------------------------------------------------------------------------ network
def _conv(st, name, x):
    return F.conv2d(x, st[name + ".weight"].to(x), st[name + ".bias"].to(x), padding=1)


def rdb_forward(st, p, x):
    """ResidualDenseBlock.forward (rrdbnet_arch.py:31-38)."""
    x1 = F.leaky_relu(_conv(st, p + "conv1", x), 0.2)
    x2 = F.leaky_relu(_conv(st, p + "conv2", torch.cat((x, x1), 1)), 0.2)
    x3 = F.leaky_relu(_conv(st, p + "conv3", torch.cat((x, x1, x2), 1)), 0.2)
    x4 = F.leaky_relu(_conv(st, p + "conv4", torch.cat((x, x1, x2, x3), 1)), 0.2)
    x5 = _conv(st, p + "conv5", torch.cat((x, x1, x2, x3, x4), 1))
    return x5 * 0.2 + x


def rrdb_forward(st, p, x):
    """RRDB.forward (rrdbnet_arch.py:58-62)."""
    out = rdb_forward(st, p + "rdb1.", x)
    out = rdb_forward(st, p + "rdb2.", out)
    out = rdb_forward(st, p + "rdb3.", out)
    return out * 0.2 + x


def num_blocks(st) -> int:
    return 1 + max(int(k.split(".")[1]) for k in st if k.startswith("body."))


def rrdbnet_forward(st, x):
    """RRDBNet.forward at scale 4 (rrdbnet_arch.py:104-117): planar [B, 3, H, W] -> [B, 3, 4H, 4W]."""
    feat = _conv(st, "conv_first", x)
    body = feat
    for i in range(num_blocks(st)):
        body = rrdb_forward(st, f"body.{i}.", body)
    feat = feat + _conv(st, "conv_body", body)
    feat = F.leaky_relu(_conv(st, "conv_up1", F.interpolate(feat, scale_factor=2, mode="nearest")), 0.2)
    feat = F.leaky_relu(_conv(st, "conv_up2", F.interpolate(feat, scale_factor=2, mode="nearest")), 0.2)
    return _conv(st, "conv_last", F.leaky_relu(_conv(st, "conv_hr", feat), 0.2))


def to_input(img: np.ndarray) -> torch.Tensor:
    """process()'s input conversion (real_esrnet.py:27-29): uint8 BGR [H, W, 3] -> float RGB [1, 3, H, W] in [0, 1]."""
    img = img.astype(np.float32) / 255.
    return torch.from_numpy(np.transpose(img[:, :, [2, 1, 0]], (2, 0, 1))).float().unsqueeze(0)


def to_image(out: torch.Tensor) -> np.ndarray:
    """process()'s output conversion (real_esrnet.py:54-56): one float RGB [3, H, W] -> uint8 BGR [H, W, 3]."""
    out = out.float().cpu().clamp_(0, 1).numpy()
    return (np.transpose(out[[2, 1, 0], :, :], (1, 2, 0)) * 255.0).round().astype(np.uint8)


def process(st, img: np.ndarray, device="cpu") -> np.ndarray:
    """RealESRNet.process at scale 4 (no padding: mod_scale is None)."""
    with torch.no_grad():
        return to_image(rrdbnet_forward(st, to_input(img).to(device))[0])


def case_image(h: int, w: int, seed: int) -> np.ndarray:
    """Seeded uint8 BGR test image [h, w, 3]: a smooth colour field plus noise (face-crop-like statistics, every value used)."""
    g = torch.Generator().manual_seed(seed)
    yy, xx = torch.meshgrid(torch.linspace(0, 1, h), torch.linspace(0, 1, w), indexing="ij")
    phase = torch.rand(3, 2, generator=g) * 6.0
    base = torch.stack([0.5 + 0.35 * torch.sin(phase[c, 0] + 3 * yy) * torch.cos(phase[c, 1] + 4 * xx) for c in range(3)], -1)
    img = base + 0.08 * torch.randn(h, w, 3, generator=g)
    return (img.clamp(0, 1) * 255).round().to(torch.uint8).numpy()
