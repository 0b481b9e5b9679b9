"""Seeded stand-in parameters for benchmarks and demos: none of the E4S / StyleGAN2 / GPEN checkpoints ships with the
reference or can be downloaded here (SURVEY.md section 8c), so throughput is measured on random-init weights of the real
architectures.

`synthetic_state(shapes)` draws every tensor from its own generator seeded by a hash of its state-dict key, so a model gets
the same parameters wherever and in whatever order it is built.  Conventions follow the reference's initialisers (randn
weights, modulation bias 1) except that parameters the reference zero-initialises (noise.weight, activate.bias, ToRGB
bias) get small non-zero values, so that those code paths do work.  The test oracle has its own copy of this recipe
(oracle/e4s_oracle.py:synthetic_state - the golden vectors were generated with it); tests/test_host_logic.py asserts that
the two produce bit-identical tensors.
"""
from __future__ import annotations

import math
from typing import Dict, Sequence

import torch


def _key_seed(key: str) -> int:
    h = 2166136261                     # FNV-1a, 32 bit
    for ch in key.encode():
        h = ((h ^ ch) * 16777619) & 0xFFFFFFFF
    return h


def _fir_1331(gain: float) -> torch.Tensor:
    t = torch.tensor([1.0, 3.0, 3.0, 1.0], dtype=torch.float64)
    k2 = torch.outer(t, t)
    return (k2 / k2.sum() * gain).to(torch.float32)


def synthetic_state(shapes: Dict[str, Sequence[int]], salt: int = 0) -> Dict[str, torch.Tensor]:
    out = {}
    for key in sorted(shapes):
        shape = tuple(shapes[key])
        g = torch.Generator().manual_seed(_key_seed(key) ^ salt)
        t = torch.randn(shape, generator=g, dtype=torch.float32)
        if key.endswith("modulation.bias"):
            t = 1.0 + 0.1 * t
        elif key.endswith("noise.weight") or key.endswith("activate.bias") or key.endswith(".bias"):
            t = 0.1 * t
        elif key.endswith("blur.kernel") or key.endswith("upsample.kernel"):
            t = _fir_1331(4.0)
        elif "encoder." in key and key.endswith(".weight") and len(shape) == 4:
            t = t * (1.0 / math.sqrt(shape[1] * shape[2] * shape[3]))   # keep the conv stack O(1)
        elif "encoder." in key and key.endswith(".weight") and len(shape) == 1:
            t = 0.25 + 0.05 * t                                          # PReLU slopes
        out[key] = t
    return out


def load_synthetic(module: torch.nn.Module, salt: int = 0, parameters_only: bool = False) -> None:
    """Load seeded stand-in values into `module`.  parameters_only keeps the module's registered buffers (FIR kernels)."""
    src = dict(module.named_parameters()) if parameters_only else module.state_dict()
    state = synthetic_state({k: tuple(v.shape) for k, v in src.items()}, salt)
    module.load_state_dict(state, strict=not parameters_only)


def synthetic_loss_state(module: torch.nn.Module, salt: int = 0) -> Dict[str, torch.Tensor]:
    """Seeded stand-in for the loss networks' checkpoints (e4s_b200.criteria: AlexNet + LPIPS linear layers and IR-SE50 cannot
    be downloaded; only the parsing UNet ships with the reference).  Conv / linear weights ~ N(0, 2 / fan_in) (ReLU networks)
    or N(0, 1 / fan_in) with the last BatchNorm of every residual branch at 0.25 (IR-SE50: a stand-in has to be as well
    conditioned as a trained network), BatchNorm otherwise weight 1 + 0.1 n, bias 0.1 n, running_mean 0.1 n, running_var
    1 + 0.1 |n|, PReLU slopes 0.25 + 0.05 n, LPIPS linear weights |n| / C; one generator per tensor, seeded by a hash of its key.  The test oracle has its own copy of this recipe
    (oracle/loss_oracle.py:synthetic_loss_state); tests/test_losses.py asserts that the two produce bit-identical tensors."""
    prelu = {name + ".weight" for name, m in module.named_modules() if isinstance(m, torch.nn.PReLU)}
    out = {}
    for key, ref in sorted(module.state_dict().items()):
        shape = tuple(ref.shape)
        g = torch.Generator().manual_seed(_key_seed(key) ^ salt)
        if key.endswith("num_batches_tracked"):
            out[key] = torch.zeros(shape, dtype=torch.int64)
            continue
        if key.endswith("net.mean") or key.endswith("net.std"):
            out[key] = ref.detach().clone().cpu()
            continue
        t = torch.randn(shape, generator=g, dtype=torch.float32)
        if key.endswith("running_var"):
            t = 1.0 + 0.1 * t.abs()
        elif key.endswith("running_mean"):
            t = 0.1 * t
        elif key.startswith("lin.") or ".lin." in key:
            t = t.abs() / shape[1]
        elif len(shape) >= 2:
            fan_in = 1
            for d in shape[1:]:
                fan_in *= d
            t = t * math.sqrt((1.0 if key.startswith("facenet.") else 2.0) / fan_in)
        elif key.endswith(".bias"):
            t = 0.1 * t
        elif key in prelu:
            t = 0.25 + 0.05 * t
        elif key.endswith("res_layer.4.weight"):
            t = 0.25 * (1.0 + 0.1 * t)
        elif key.endswith(".weight") and len(shape) == 1:
            t = 1.0 + 0.1 * t
        out[key] = t
    return out


def synthetic_parser_state(shapes: Dict[str, Sequence[int]], salt: int = 0) -> Dict[str, torch.Tensor]:
    """Seeded stand-in for the BiSeNet face parser's checkpoint (79999_iter.pth cannot be downloaded): convolution weights
    ~ N(0, 2 / fan_in) (a ReLU network), BatchNorm weight 1 + 0.1 n, bias 0, running_mean 0.1 n, running_var
    3 (1 + 0.1 |n|), with the second BatchNorm of every residual block (and of its shortcut) scaled by 1 / sqrt(2) so that
    the activations stay O(1) through the residual stages.  (With bias 0.1 n and running_var 1 + 0.1 |n| the per-channel
    offsets build up through the trunk and one class takes ~95 % of the pixels; this recipe gives seeded test images 7 of
    the 12 classes, none above 41 %.)  One generator per tensor, seeded by a hash of its key.  The test
    oracle has its own copy of this recipe (oracle/parser_oracle.py:synthetic_state); tests/test_face_parsing.py asserts that
    the two produce bit-identical tensors."""
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
        else:                                                            # BatchNorm weight
            t = 1.0 + 0.1 * t
            if key.endswith("bn2.weight") or key.endswith("downsample.1.weight"):
                t = t * (1.0 / math.sqrt(2.0))
        out[key] = t
    return out


def synthetic_sr_state(seed: int = 0) -> Dict[str, torch.Tensor]:
    """Seeded stand-in for GPEN's realesrnet_x4.pth ``params_ema`` (RRDBNet num_feat 32, 23 blocks, num_grow_ch 32; it cannot
    be downloaded).  Convolution weights ~ N(0, 2 / fan_in) - He initialisation without the reference's 0.1 damping of the
    dense blocks, so that their branches contribute (||0.2 x5|| / ||x|| is 0.19 .. 0.43, median 0.28, over the 69 residual
    dense blocks on a 32 x 32 face-like image) - and conv_last's ~ N(0, 2e-5 / fan_in); biases 0.1 n, conv_last's
    0.5 + 0.05 n, so that most of the image lies inside [0, 1].  One generator per tensor, seeded by a hash of its key and
    `seed`.  The test oracle has its own copy of this recipe (oracle/sr_oracle.py:synthetic_state); tests/test_sr.py asserts
    that the two produce bit-identical tensors."""
    from .gpen.sr_model.rrdbnet_arch import RRDBNet
    with torch.device("meta"):
        shapes = {k: tuple(v.shape) for k, v in RRDBNet(3, 3, scale=4, num_feat=32, num_block=23, num_grow_ch=32).state_dict().items()}
    out = {}
    for key in sorted(shapes):
        shape = shapes[key]
        g = torch.Generator().manual_seed(_key_seed(key) ^ seed)
        t = torch.randn(shape, generator=g, dtype=torch.float32)
        last = key.startswith("conv_last.")
        if len(shape) == 4:
            t = t * math.sqrt((2e-5 if last else 2.0) / (shape[1] * shape[2] * shape[3]))
        else:
            t = 0.5 + 0.05 * t if last else 0.1 * t
        out[key] = t
    return out


def load_synthetic_losses(criterion: torch.nn.Module, salt: int = 0) -> None:
    """Seeded weights for the three loss networks of an e4s_b200.criteria.InversionLoss (salts as oracle/loss_oracle.py:loss_states)."""
    for off, name in enumerate(("lpips_loss", "id_loss", "face_parsing_loss")):
        sub = getattr(criterion, name, None)
        if sub is not None:
            sub.load_state_dict(synthetic_loss_state(sub, salt + off), strict=True)


def synthetic_retinaface_state(seed: int = 0, face_bias: float = 0.6, class_gain: float = 2.0,
                               box_size: float = 4.0) -> Dict[str, torch.Tensor]:
    """Seeded stand-in for GPEN's RetinaFace-R50.pth (cfg_re50; it cannot be downloaded), unprefixed keys.  Convolution
    weights ~ N(0, 2 / fan_in); BatchNorm weight 1 + 0.1 n (0.5 (1 + 0.1 n) at every bottleneck's bn3 and shortcut BN, so
    that the 16 residual stages stay O(1) while each branch still counts), bias 0.1 n, running_mean 0.1 n, running_var
    3 (1 + 0.1 |n|).  Heads: class weights ~ N(0, class_gain^2 / fan_in) with bias (0, face_bias) per anchor (background,
    face), so that a few per cent of the priors score above 0.9; bbox and landmark weights ~ N(0, 0.5 / fan_in), bias
    0.1 n, plus box_size on the bbox head's two log-size outputs (boxes ~2.2x their anchor), so that neighbouring candidates
    overlap and NMS suppresses most of them.  One generator per tensor, seeded by a hash of its key and `seed`."""
    from .gpen.face_detect.data import cfg_re50
    from .gpen.face_detect.facemodels.retinaface import RetinaFace
    with torch.device("meta"):
        shapes = {k: tuple(v.shape) for k, v in RetinaFace(cfg=cfg_re50, phase='test').state_dict().items()}
    out = {}
    for key in sorted(shapes):
        shape = shapes[key]
        if key.endswith("num_batches_tracked"):
            out[key] = torch.zeros(shape, dtype=torch.int64)
            continue
        g = torch.Generator().manual_seed(_key_seed(key) ^ seed)
        t = torch.randn(shape, generator=g, dtype=torch.float32)
        head = key.startswith(("ClassHead", "BboxHead", "LandmarkHead"))
        if len(shape) == 4:
            fan = shape[1] * shape[2] * shape[3]
            gain = class_gain ** 2 if key.startswith("ClassHead") else 0.5 if head else 2.0
            t = t * math.sqrt(gain / fan)
        elif head:                                                       # head biases
            if key.startswith("ClassHead"):
                t = torch.tensor([0.0, face_bias] * (shape[0] // 2), dtype=torch.float32)
            else:
                t = 0.1 * t
                if key.startswith("BboxHead"):
                    t[2::4] += box_size                                  # log-size offsets: boxes exp(0.2 box_size)
                    t[3::4] += box_size                                  # times their anchor, so neighbours overlap
        elif key.endswith("running_var"):
            t = 3.0 * (1.0 + 0.1 * t.abs())
        elif key.endswith(("running_mean", ".bias")):
            t = 0.1 * t
        else:                                                            # BatchNorm weight
            t = 1.0 + 0.1 * t
            if key.endswith("bn3.weight") or key.endswith("downsample.1.weight"):
                t = 0.5 * t
        out[key] = t
    return out
