"""Fused bias + leaky ReLU on the sm_90a kernel.

Mirror of src/models/stylegan2/op/fused_act.py: ``FusedLeakyReLU`` (:72-81, owns ``bias``),
``fused_leaky_relu`` (:84-85) and the autograd construction of :18-69 (gradient masks on the saved
forward OUTPUT, bias gradient = sum over non-channel axes, second order reuses the same kernel).
"""
from __future__ import annotations

import torch
from torch import nn
from torch.autograd import Function

from ... import kernels as K


class _FusedLeakyReLUGrad(Function):
    @staticmethod
    def forward(ctx, grad_output, out, negative_slope, scale):
        ctx.save_for_backward(out)
        ctx.cfg = (negative_slope, scale)
        gx = K.bias_act_bwd(grad_output, out, negative_slope, scale)
        return gx, K.bias_grad(gx)

    @staticmethod
    def backward(ctx, gg_input, gg_bias):
        (out,) = ctx.saved_tensors
        negative_slope, scale = ctx.cfg
        gg = gg_input
        if gg_bias is not None:
            gg = gg + gg_bias.reshape([1, -1] + [1] * (gg_input.ndim - 2))
        return K.bias_act_bwd(gg, out, negative_slope, scale), None, None, None


class _FusedLeakyReLU(Function):
    @staticmethod
    def forward(ctx, input, bias, negative_slope, scale):
        out = K.bias_act_fwd(input, bias, negative_slope, scale)
        ctx.save_for_backward(out)
        ctx.cfg = (negative_slope, scale, bias is not None)
        return out

    @staticmethod
    def backward(ctx, grad_output):
        (out,) = ctx.saved_tensors
        negative_slope, scale, has_bias = ctx.cfg
        gx, gb = _FusedLeakyReLUGrad.apply(grad_output, out, negative_slope, scale)
        return gx, (gb if has_bias else None), None, None


def fused_leaky_relu(input, bias, negative_slope=0.2, scale=2 ** 0.5):
    if not input.is_cuda:
        raise RuntimeError("input must be a CUDA tensor")
    return _FusedLeakyReLU.apply(input, bias, negative_slope, scale)


class FusedLeakyReLU(nn.Module):
    def __init__(self, channel, negative_slope=0.2, scale=2 ** 0.5):
        super().__init__()
        self.bias = nn.Parameter(torch.zeros(channel))
        self.negative_slope = negative_slope
        self.scale = scale

    def forward(self, input):
        return fused_leaky_relu(input, self.bias, self.negative_slope, self.scale)
