"""The reference's OWN GPU formulation of the synthesis forward, restated on torch/cuDNN - the stronger baseline of
BASELINE.md section 4 / SURVEY.md section 8d, timed by bench.py's `gpu_baseline` leg on the same GPU.  CHECKER SIDE: test
infrastructure like the rest of oracle/, never imported by e4s_b200/.

What the reference executes per masked layer (src/models/stylegan2/model.py):
  * one full ModulatedConv2d per region (:395-398), each with per-sample modulated + demodulated weights materialised
    (:277-285) and ONE grouped convolution over the whole batch, groups = B (:312-318; conv_transpose2d :287-300), i.e. cuDNN;
  * Blur / Upsample = upfirdn2d (its own CUDA kernel in the reference; here the equivalent depthwise torch convolution,
    which is cuDNN / ATen - a library kernel either way), fused bias + leaky ReLU (an elementwise kernel);
  * mask multiply and accumulate per region (:397-398), noise add, ToRGB with the same per-region loop (:434-437).
This module reproduces exactly that structure (oracle/e4s_oracle.py keeps a per-sample loop instead of groups = B because
it targets the CPU).  Numerics equal the oracle's: tests/test_oracle_golden.py::test_gpu_baseline_structure_equals_oracle
(CPU, small case).
"""
from __future__ import annotations

import math
from typing import Dict, List

import torch
import torch.nn.functional as F

from . import e4s_oracle as O

Tensor = torch.Tensor


def modulated_conv2d_grouped(x: Tensor, style: Tensor, weight: Tensor, mod_weight: Tensor, mod_bias: Tensor,
                             demodulate: bool = True, upsample: bool = False) -> Tensor:
    """ModulatedConv2d.forward, fused branch with groups = batch: model.py:276-320."""
    b, cin, h, w = x.shape
    _, cout, _, k, _ = weight.shape
    s = O.equal_linear(style, mod_weight, mod_bias)                                        # :276
    wmod = (1.0 / math.sqrt(cin * k * k)) * weight * s.reshape(b, 1, cin, 1, 1)              # :277
    if demodulate:
        d = torch.rsqrt(wmod.pow(2).sum([2, 3, 4]) + 1e-8)                                   # :280
        wmod = wmod * d.reshape(b, cout, 1, 1, 1)                                            # :281
    if upsample:
        xin = x.reshape(1, b * cin, h, w)                                                    # :288
        wt = wmod.transpose(1, 2).reshape(b * cin, cout, k, k)                               # :289-294
        out = F.conv_transpose2d(xin, wt, padding=0, stride=2, groups=b)                     # :295-297
        out = out.reshape(b, cout, out.shape[2], out.shape[3])
        fir = O.make_fir((1, 3, 3, 1), gain=4.0, dtype=x.dtype).to(x.device)
        return O.upfirdn2d(out, fir, pad=(1, 1))                                             # :300 (Blur)
    xin = x.reshape(1, b * cin, h, w)                                                        # :313
    out = F.conv2d(xin, wmod.reshape(b * cout, cin, k, k), padding=k // 2, groups=b)          # :314-316
    return out.reshape(b, cout, out.shape[2], out.shape[3])


def _styled(x, style, mask, noise, p, prefix, upsample, mask_op):
    wk = dict(weight=p[prefix + "conv.weight"], mod_weight=p[prefix + "conv.modulation.weight"], mod_bias=p[prefix + "conv.modulation.bias"])
    if not mask_op:
        out = modulated_conv2d_grouped(x, style, upsample=upsample, **wk)
    else:
        seg = O.nearest_resize(mask, x.shape[2] * (2 if upsample else 1))                   # :391
        out = None
        for c in range(style.shape[1]):                                                      # :395-398
            oc = modulated_conv2d_grouped(x, style[:, c], upsample=upsample, **wk) * seg[:, c:c + 1]
            out = oc if out is None else out + oc
    out = out + p[prefix + "noise.weight"] * noise
    return O.fused_leaky_relu(out, p[prefix + "activate.bias"])


def _to_rgb(x, style, mask, skip, p, prefix, mask_op):
    wk = dict(weight=p[prefix + "conv.weight"], mod_weight=p[prefix + "conv.modulation.weight"], mod_bias=p[prefix + "conv.modulation.bias"],
              demodulate=False)
    if not mask_op:
        out = modulated_conv2d_grouped(x, style, **wk)
    else:
        seg = O.nearest_resize(mask, x.shape[2])
        out = None
        for c in range(style.shape[1]):                                                      # :434-437
            oc = modulated_conv2d_grouped(x, style[:, c], **wk) * seg[:, c:c + 1]
            out = oc if out is None else out + oc
    out = out + p[prefix + "bias"]
    if skip is not None:
        fir = O.make_fir((1, 3, 3, 1), gain=4.0, dtype=x.dtype).to(x.device)
        out = out + O.upfirdn2d(skip, fir, up=2, pad=(2, 1))
    return out


def generator_forward(p: Dict[str, Tensor], codes: Tensor, mask: Tensor, noise: List[Tensor], size: int,
                      remaining_layer_idx: int = 13, split_layer_idx: int = 5, prefix: str = ""):
    """Generator.forward (model.py:576-667) in the reference's execution structure; same schedule as O.generator_forward."""
    K = remaining_layer_idx
    log_size, conv_mask, rgb_mask = O.generator_layer_plan(size, K)
    b = codes.shape[0]
    out = p[prefix + "input.input"].repeat(b, 1, 1, 1)
    out = _styled(out, codes[:, :, 0], mask, noise[0], p, prefix + "conv1.", False, True)
    skip = _to_rgb(out, codes[:, :, 1], mask, None, p, prefix + "to_rgb1.", True)
    feats = None
    i = 1
    for r in range(log_size - 2):
        c1, c2, tr = f"{prefix}convs.{2 * r}.", f"{prefix}convs.{2 * r + 1}.", f"{prefix}to_rgbs.{r}."
        n1, n2 = noise[1 + 2 * r], noise[2 + 2 * r]
        if i < K:
            out = _styled(out, codes[:, :, i] if conv_mask[r] else codes[:, 0, i], mask, n1, p, c1, True, conv_mask[r])
            if i + 2 == split_layer_idx:
                feats = out
            out = _styled(out, codes[:, :, i + 1] if conv_mask[r] else codes[:, 0, i + 1], mask, n2, p, c2, False, conv_mask[r])
            st = codes[:, :, i + 2] if (K == 17 or i + 2 != K) else codes[:, 0, i + 2]
            skip = _to_rgb(out, st, mask, skip, p, tr, rgb_mask[r])
        else:
            out = _styled(out, codes[:, 0, i], mask, n1, p, c1, True, conv_mask[r])
            out = _styled(out, codes[:, 0, i + 1], mask, n2, p, c2, False, conv_mask[r])
            skip = _to_rgb(out, codes[:, 0, i + 2], mask, skip, p, tr, rgb_mask[r])
        i += 2
    return skip, feats
