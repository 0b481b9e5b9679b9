"""Torch-CPU restatement of GPEN's face parser (src/pretrained/gpen/face_parse/): ParseNet.forward (parse_model.py:69-75,
blocks.py:92-125) in FaceParse's configuration and FaceParse.process / process_tensor (face_parsing.py:39-79), written from
the state dict with torch.nn.functional, in whatever dtype / device the state and input are given in.  Also the seeded
stand-in checkpoint (no ParseNet-latest.pth can be downloaded).  Pinned against the unmodified reference by
oracle/make_golden_gpen_parse.py."""
from __future__ import annotations

import math
from typing import Dict

import numpy as np
import torch
import torch.nn.functional as F

SIZE, NCLS, DEPTH = 512, 19, 10
MASK_COLORMAP = [0, 255, 255, 255, 255, 255, 255, 255, 255, 255, 255, 255, 255, 255, 0, 255, 255, 255, 0]
DOWN = [(64, 128), (128, 256), (256, 256), (256, 256)]     # (cin, cout) of encoder.1 .. 4
UP = [(256, 256), (256, 256), (256, 128), (128, 64)]       # decoder.0 .. 3
BODY_CH = 256


# ------------------------------------------------------------------------------------------------------------ state
def param_shapes() -> Dict[str, tuple]:
    """State-dict keys and shapes of ParseNet(512, 512, 32, 64, 19, norm_type='bn', relu_type='LeakyReLU', ch_range=[32, 256])."""
    s = {}

    def conv(p, cin, cout, bn):
        s[p + ".conv2d.weight"] = (cout, cin, 3, 3)
        if bn:
            for k in ("weight", "bias", "running_mean", "running_var"):
                s[p + ".norm.norm." + k] = (cout,)
            s[p + ".norm.norm.num_batches_tracked"] = ()
        else:
            s[p + ".conv2d.bias"] = (cout,)

    def block(p, cin, cout, shortcut):
        if shortcut:
            conv(p + ".shortcut_func", cin, cout, False)
        conv(p + ".conv1", cin, cout, True)
        conv(p + ".conv2", cout, cout, True)

    conv("encoder.0", 3, 64, False)
    for i, (ci, co) in enumerate(DOWN):
        block(f"encoder.{i + 1}", ci, co, True)
    for i in range(DEPTH):
        block(f"body.{i}", BODY_CH, BODY_CH, False)
    for i, (ci, co) in enumerate(UP):
        block(f"decoder.{i}", ci, co, True)
    conv("out_img_conv", 64, 3, False)
    conv("out_mask_conv", 64, NCLS, False)
    return s


def _key_seed(key: str) -> int:
    h = 2166136261                     # FNV-1a, 32 bit
    for ch in key.encode():
        h = ((h ^ ch) * 16777619) & 0xFFFFFFFF
    return h


# out_mask_conv bias offsets: the background (0) and the two classes that map to mask value 0 (14, 18) and a few others are
# raised so that the argmax spreads over several classes and both mask values
_HEAD_BIAS = {0: 1.2, 1: 0.9, 13: 0.9, 14: 0.9, 18: 0.7, 2: 0.5, 10: 0.5}


def synthetic_state(seed: int = 0) -> Dict[str, torch.Tensor]:
    """Seeded stand-in for ParseNet-latest.pth: one generator per tensor, seeded by a hash of its key and `seed`.
    Convolution weights ~ N(0, 1 / fan_in) (out_mask_conv's N(0, 0.36 / fan_in)); BatchNorm weight 1 + 0.1 n, bias 0.1 n,
    running_mean 0.05 n, running_var 0.5 + U(0, 1) (not the identity, so the fold matters); conv2 of every block has its
    BN weight scaled by 0.5 so that the residual branches stay comparable to the identity (||branch|| / ||identity|| is
    recorded by make_golden_gpen_parse.py); convolution biases 0.1 n, out_mask_conv's 0.3 n plus the _HEAD_BIAS offsets."""
    out = {}
    shapes = param_shapes()
    for key in sorted(shapes):
        shape = shapes[key]
        g = torch.Generator().manual_seed(_key_seed(key) ^ seed)
        if key.endswith("num_batches_tracked"):
            out[key] = torch.tensor(1000, dtype=torch.int64)
            continue
        if key.endswith("running_var"):
            out[key] = 0.5 + torch.rand(shape, generator=g, dtype=torch.float32)
            continue
        t = torch.randn(shape, generator=g, dtype=torch.float32)
        head = key.startswith("out_mask_conv.")
        if len(shape) == 4:
            t = t * math.sqrt((0.36 if head else 1.0) / (shape[1] * 9))
        elif key.endswith("norm.norm.weight"):
            t = (1.0 + 0.1 * t) * (0.5 if ".conv2." in key else 1.0)
        elif key.endswith("running_mean"):
            t = 0.05 * t
        elif head:
            t = 0.3 * t + torch.tensor([_HEAD_BIAS.get(k, 0.0) for k in range(NCLS)])
        else:
            t = 0.1 * t
        out[key] = t
    return out


# ------------------------------------------------------------------------------------------------------------ network
def conv_layer(st, p, x, scale="none", act=False):
    """ConvLayer.forward (blocks.py:92-99): nearest 2x ('up'), reflection pad 1, 3x3 conv (stride 2 for 'down'), BN (eval)
    when the layer has one, LeakyReLU(0.2) when `act`."""
    if scale == "up":
        x = F.interpolate(x, scale_factor=2, mode="nearest")
    x = F.pad(x, (1, 1, 1, 1), mode="reflect")
    b = st.get(p + ".conv2d.bias")
    x = F.conv2d(x, st[p + ".conv2d.weight"].to(x), None if b is None else b.to(x), stride=2 if scale == "down" else 1)
    if p + ".norm.norm.weight" in st:
        n = p + ".norm.norm."
        x = F.batch_norm(x, st[n + "running_mean"].to(x), st[n + "running_var"].to(x), st[n + "weight"].to(x),
                         st[n + "bias"].to(x), False, 0.0, 1e-5)
    return F.leaky_relu(x, 0.2) if act else x


def residual_block(st, p, x, scale="none", branch=None):
    """ResidualBlock.forward (blocks.py:120-125).  `branch`: a list that receives ||res|| / ||identity|| per sample."""
    identity = x if scale == "none" else conv_layer(st, p + ".shortcut_func", x, scale)
    res = conv_layer(st, p + ".conv1", x, "up" if scale == "up" else "none", act=True)
    res = conv_layer(st, p + ".conv2", res, "down" if scale == "down" else "none")
    if branch is not None:
        branch.extend((res.flatten(1).norm(dim=1) / identity.flatten(1).norm(dim=1)).tolist())
    return identity + res


def parsenet_forward(st, x, branch=None):
    """ParseNet.forward (parse_model.py:69-75): planar [B, 3, 512, 512] -> (out_mask [B, 19, 512, 512], out_img)."""
    feat = conv_layer(st, "encoder.0", x)
    for i in range(len(DOWN)):
        feat = residual_block(st, f"encoder.{i + 1}", feat, "down", branch)
    body = feat
    for i in range(DEPTH):
        body = residual_block(st, f"body.{i}", body, "none", branch)
    y = feat + body
    for i in range(len(UP)):
        y = residual_block(st, f"decoder.{i}", y, "up", branch)
    return conv_layer(st, "out_mask_conv", y), conv_layer(st, "out_img_conv", y)


def to_mask(logits: torch.Tensor) -> torch.Tensor:
    """First-index argmax over the classes, then MASK_COLORMAP: [B, 19, H, W] -> int64 [B, H, W]."""
    return torch.tensor(MASK_COLORMAP, dtype=torch.int64, device=logits.device)[logits.argmax(dim=1)]


def process_input(img: np.ndarray) -> torch.Tensor:
    """process()'s input conversion (face_parsing.py:40, 59-63): cv2.resize to 512 x 512, BGR -> RGB, float64 / 255 * 2 - 1,
    then fp32 [1, 3, 512, 512]."""
    import cv2
    img = cv2.resize(img, (SIZE, SIZE))[..., ::-1]
    img = img / 255. * 2 - 1
    return torch.from_numpy(img.transpose(2, 0, 1)).unsqueeze(0).float()


def process(st, img: np.ndarray) -> list:
    """FaceParse.process: uint8 BGR image -> [uint8 mask [512, 512]] with values 0 / 255."""
    with torch.no_grad():
        return [m.numpy().astype(np.uint8) for m in to_mask(parsenet_forward(st, process_input(img))[0])]


def tensor_input(imt: torch.Tensor) -> torch.Tensor:
    """process_tensor()'s input conversion (face_parsing.py:48): BGR [B, 3, H, W] in [0, 1] -> nearest-resized RGB in [-1, 1]."""
    return F.interpolate(imt.flip(1) * 2 - 1, (SIZE, SIZE))


def process_tensor(st, imt: torch.Tensor) -> torch.Tensor:
    """FaceParse.process_tensor: BGR [B, 3, H, W] in [0, 1] -> int64 [1, B, 512, 512] with values 0 / 255."""
    with torch.no_grad():
        return to_mask(parsenet_forward(st, tensor_input(imt))[0]).unsqueeze(0)


def case_image(h: int, w: int, seed: int) -> np.ndarray:
    """Seeded uint8 BGR test image [h, w, 3]: a face-like layout (a bright ellipse on a darker background, two dark eye
    spots, a mouth bar) over a smooth colour field plus noise."""
    g = torch.Generator().manual_seed(seed)
    yy, xx = torch.meshgrid(torch.linspace(-1, 1, h), torch.linspace(-1, 1, w), indexing="ij")
    phase = torch.rand(3, 2, generator=g) * 6.0
    img = torch.stack([0.35 + 0.2 * torch.sin(phase[c, 0] + 3 * yy) * torch.cos(phase[c, 1] + 4 * xx) for c in range(3)], -1)
    cy, cx = (torch.rand(2, generator=g) - 0.5) * 0.3
    face = (((yy - cy) / 0.75) ** 2 + ((xx - cx) / 0.55) ** 2) < 1
    img[face] = img[face] * 0.5 + torch.tensor([0.45, 0.55, 0.75])
    for ex in (-0.22, 0.22):
        eye = (((yy - cy + 0.15) / 0.06) ** 2 + ((xx - cx - ex) / 0.1) ** 2) < 1
        img[eye] = 0.1
    mouth = ((yy - cy - 0.35).abs() < 0.04) & ((xx - cx).abs() < 0.2)
    img[mouth] = torch.tensor([0.3, 0.2, 0.7])
    img = img + 0.05 * torch.randn(h, w, 3, generator=g)
    return (img.clamp(0, 1) * 255).round().to(torch.uint8).numpy()


def image_tensor(img: np.ndarray) -> torch.Tensor:
    """uint8 BGR [H, W, 3] -> process_tensor's input, fp32 BGR [1, 3, H, W] in [0, 1]."""
    return (torch.from_numpy(img).permute(2, 0, 1).float() / 255.).unsqueeze(0).contiguous()
