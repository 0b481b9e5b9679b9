"""Torch-CPU restatement of the reference's face parser (src/pretrained/face_parsing/): FaceParser.preprocess_img,
BiSeNet.forward (model.py:236-260, resnet.py:58-80), the argmax and the 19 -> 12 conversion
(src/datasets/dataset.py:60-108), written from the state dict with torch.nn.functional.  Pinned against the unmodified
reference by oracle/make_golden_parser.py."""
from __future__ import annotations

import math
from typing import Dict, Sequence

import torch
import torch.nn.functional as F

MEAN = (0.485, 0.456, 0.406)
STD = (0.229, 0.224, 0.225)
# 19 parser classes -> 12 classes of the mask stage
FFHQ19_TO_12 = [0, 6, 2, 2, 3, 3, 10, 7, 7, 11, 5, 9, 1, 1, 8, 0, 0, 4, 0] + [0] * (256 - 19)
N_CLASSES = 19


# ------------------------------------------------------------------------------------------------------------ state
def param_shapes(n_classes: int = N_CLASSES) -> Dict[str, tuple]:
    """State-dict keys and shapes of BiSeNet(n_classes)."""
    s = {}

    def bn(p, c):
        s.update({p + ".weight": (c,), p + ".bias": (c,), p + ".running_mean": (c,), p + ".running_var": (c,),
                  p + ".num_batches_tracked": ()})

    def cbr(p, cin, cout, k):
        s[p + ".conv.weight"] = (cout, cin, k, k)
        bn(p + ".bn", cout)

    r = "cp.resnet."
    s[r + "conv1.weight"] = (64, 3, 7, 7)
    bn(r + "bn1", 64)
    cin = 64
    for li, cout in enumerate((64, 128, 256, 512), start=1):
        for bi in range(2):
            p = f"{r}layer{li}.{bi}."
            c_in = cin if bi == 0 else cout
            s[p + "conv1.weight"] = (cout, c_in, 3, 3)
            bn(p + "bn1", cout)
            s[p + "conv2.weight"] = (cout, cout, 3, 3)
            bn(p + "bn2", cout)
            if bi == 0 and (c_in != cout or li > 1):
                s[p + "downsample.0.weight"] = (cout, c_in, 1, 1)
                bn(p + "downsample.1", cout)
        cin = cout
    for arm, c in (("arm16", 256), ("arm32", 512)):
        cbr(f"cp.{arm}.conv", c, 128, 3)
        s[f"cp.{arm}.conv_atten.weight"] = (128, 128, 1, 1)
        bn(f"cp.{arm}.bn_atten", 128)
    cbr("cp.conv_head32", 128, 128, 3)
    cbr("cp.conv_head16", 128, 128, 3)
    cbr("cp.conv_avg", 512, 128, 1)
    cbr("ffm.convblk", 256, 256, 1)
    s["ffm.conv1.weight"] = (64, 256, 1, 1)
    s["ffm.conv2.weight"] = (256, 64, 1, 1)
    for head, cin_h, mid in (("conv_out", 256, 256), ("conv_out16", 128, 64), ("conv_out32", 128, 64)):
        cbr(head + ".conv", cin_h, mid, 3)
        s[head + ".conv_out.weight"] = (n_classes, mid, 1, 1)
    return s


def _key_seed(key: str) -> int:
    h = 2166136261                     # FNV-1a, 32 bit
    for ch in key.encode():
        h = ((h ^ ch) * 16777619) & 0xFFFFFFFF
    return h


def synthetic_state(shapes: Dict[str, Sequence[int]] | None = None, salt: int = 0) -> Dict[str, torch.Tensor]:
    """The seeded stand-in checkpoint (same recipe as e4s_b200/synthetic.py:synthetic_parser_state)."""
    shapes = param_shapes() if shapes is None else shapes
    out = {}
    for key in sorted(shapes):
        shape = tuple(shapes[key])
        if key.endswith("num_batches_tracked"):
            out[key] = torch.zeros(shape, dtype=torch.int64)
            continue
        g = torch.Generator().manual_seed(_key_seed(key) ^ salt)
        t = torch.randn(shape, generator=g, dtype=torch.float32)
        if len(shape) == 4:
            t = t * math.sqrt(2.0 / (shape[1] * shape[2] * shape[3]))
        elif key.endswith("running_var"):
            t = 3.0 * (1.0 + 0.1 * t.abs())
        elif key.endswith("running_mean"):
            t = 0.1 * t
        elif key.endswith(".bias"):
            t = torch.zeros(shape, dtype=torch.float32)
        else:
            t = 1.0 + 0.1 * t
            if key.endswith("bn2.weight") or key.endswith("downsample.1.weight"):
                t = t * (1.0 / math.sqrt(2.0))
        out[key] = t
    return out


def case_image(size: int, seed: int):
    """A seeded uint8 RGB test image [size, size, 3] (numpy): smooth colour fields (bicubic from 8 x 8) plus noise."""
    g = torch.Generator().manual_seed(seed)
    low = torch.rand(1, 3, 8, 8, generator=g)
    img = F.interpolate(low, size=(size, size), mode="bicubic", align_corners=False)
    img = img + 0.05 * torch.randn(1, 3, size, size, generator=g)
    return (img.clamp(0, 1) * 255).round().to(torch.uint8)[0].permute(1, 2, 0).contiguous().numpy()


# ------------------------------------------------------------------------------------------------------------ step 1
def bicubic_taps(factor: int, a: float = -0.5) -> torch.Tensor:
    """4 f taps of the cubic convolution kernel at (i - 2 f + 0.5) / f, normalised to sum 1 (fp32)."""
    x = ((torch.arange(4 * factor, dtype=torch.float32) - 2 * factor + 0.5) / factor).abs()
    k = torch.where(x <= 1.0, (a + 2.0) * x ** 3 - (a + 3.0) * x ** 2 + 1.0,
                    torch.where(x < 2.0, a * x ** 3 - 5.0 * a * x ** 2 + 8.0 * a * x - 4.0 * a, torch.zeros_like(x)))
    return k / k.sum()


def bicubic_down(x: torch.Tensor, factor: int) -> torch.Tensor:
    """[B, 3, H, W] -> [B, 3, H/f, W/f]: reflect pad 3f // 2 before / the rest after, vertical pass, horizontal pass."""
    k = bicubic_taps(factor).to(x)
    pad = 3 * factor
    x = F.pad(x, (0, 0, pad // 2, pad - pad // 2), mode="reflect")
    x = F.conv2d(x, k.reshape(1, 1, -1, 1).repeat(3, 1, 1, 1), stride=(factor, 1), groups=3)
    x = F.pad(x, (pad // 2, pad - pad // 2, 0, 0), mode="reflect")
    return F.conv2d(x, k.reshape(1, 1, 1, -1).repeat(3, 1, 1, 1), stride=(1, factor), groups=3)


def normalize(x: torch.Tensor) -> torch.Tensor:
    mean = torch.tensor(MEAN, dtype=torch.float32).reshape(1, 3, 1, 1).to(x)
    std = torch.tensor(STD, dtype=torch.float32).reshape(1, 3, 1, 1).to(x)
    return (x.clamp(0, 1) - mean) / std


def preprocess(images: torch.Tensor, factor: int) -> torch.Tensor:
    """images [B, 3, H, W] in [0, 1] (H, W >= 512) -> the normalised network input [B, 3, H/f, W/f]."""
    return normalize(bicubic_down(images, factor))


# ------------------------------------------------------------------------------------------------------------ step 2
def _bn(st, p, x):
    return F.batch_norm(x, st[p + ".running_mean"].to(x), st[p + ".running_var"].to(x), st[p + ".weight"].to(x),
                        st[p + ".bias"].to(x), False, 0.0, 1e-5)


def _conv(st, key, x, stride=1):
    w = st[key].to(x)
    return F.conv2d(x, w, stride=stride, padding=w.shape[-1] // 2)


def _cbr(st, p, x):
    return F.relu(_bn(st, p + ".bn", _conv(st, p + ".conv.weight", x)))


def _arm(st, p, x):
    feat = _cbr(st, p + ".conv", x)
    atten = torch.sigmoid(_bn(st, p + ".bn_atten", _conv(st, p + ".conv_atten.weight", feat.mean((2, 3), keepdim=True))))
    return feat * atten


def resnet18(st, x):
    r = "cp.resnet."
    x = F.max_pool2d(F.relu(_bn(st, r + "bn1", _conv(st, r + "conv1.weight", x, 2))), 3, 2, 1)
    feats = []
    for li in range(1, 5):
        for bi in range(2):
            p = f"{r}layer{li}.{bi}."
            stride = 2 if (li > 1 and bi == 0) else 1
            res = F.relu(_bn(st, p + "bn1", _conv(st, p + "conv1.weight", x, stride)))
            res = _bn(st, p + "bn2", _conv(st, p + "conv2.weight", res))
            sc = _bn(st, p + "downsample.1", _conv(st, p + "downsample.0.weight", x, stride)) if p + "downsample.0.weight" in st else x
            x = F.relu(sc + res)
        feats.append(x)
    return feats[1], feats[2], feats[3]


def features(st, x):
    """-> (FFM output, feat_cp8, feat_cp16)."""
    feat8, feat16, feat32 = resnet18(st, x)
    avg = _cbr(st, "cp.conv_avg", feat32.mean((2, 3), keepdim=True))
    up = lambda t: F.interpolate(t, scale_factor=2, mode="nearest")  # noqa: E731
    feat32_up = _cbr(st, "cp.conv_head32", up(_arm(st, "cp.arm32", feat32) + avg))
    feat16_up = _cbr(st, "cp.conv_head16", up(_arm(st, "cp.arm16", feat16) + feat32_up))
    feat = _cbr(st, "ffm.convblk", torch.cat([feat8, feat16_up], dim=1))
    atten = feat.mean((2, 3), keepdim=True)
    atten = torch.sigmoid(_conv(st, "ffm.conv2.weight", F.relu(_conv(st, "ffm.conv1.weight", atten))))
    return feat * atten + feat, feat16_up, feat32_up


def _head(st, p, x, hw):
    y = _conv(st, p + ".conv_out.weight", _cbr(st, p + ".conv", x))
    return F.interpolate(y, hw, mode="bilinear", align_corners=True)


def bisenet_forward(st, x):
    """Normalised x [B, 3, H, W] -> the three heads' logits [B, 19, H, W], in the dtype and on the device of x (fp32, or
    float64 references)."""
    fuse, cp8, cp16 = features(st, x)
    hw = tuple(x.shape[2:])
    return _head(st, "conv_out", fuse, hw), _head(st, "conv_out16", cp8, hw), _head(st, "conv_out32", cp16, hw)


def main_logits(st, x):
    """The first head only (what the labels need)."""
    return _head(st, "conv_out", features(st, x)[0], tuple(x.shape[2:]))


# ------------------------------------------------------------------------------------------------------------ steps 3-4
def labels(logits: torch.Tensor, seg12: bool = True) -> torch.Tensor:
    """First-index argmax over the classes, then the 19 -> 12 table: uint8 [B, H, W]."""
    lab = logits.argmax(1)
    if seg12:
        lab = torch.tensor(FFHQ19_TO_12, dtype=torch.uint8, device=lab.device)[lab]
    return lab.to(torch.uint8)


def parse(st, images: torch.Tensor, factor: int, seg12: bool = True) -> torch.Tensor:
    """images [B, 3, H, W] in [0, 1] -> uint8 label maps [B, H/f, W/f]."""
    return labels(main_logits(st, preprocess(images, factor)), seg12)
