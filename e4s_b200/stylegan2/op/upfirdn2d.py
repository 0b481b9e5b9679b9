"""upfirdn2d with first- and second-order gradients, on the sm_90a kernel.

Mirror of src/models/stylegan2/op/upfirdn2d.py: same call signature as ``upfirdn2d`` (:142-147) and the
same gradient construction (the adjoint of upfirdn is upfirdn with the flipped FIR, up<->down swapped
and the padding of :108-113; the adjoint of that is the forward op again, :61-82).  The native layer is
the C ABI ``e4s_upfirdn2d_f32`` instead of a pybind module JIT-built at import (:8-14).
"""
from __future__ import annotations

import torch
from torch.autograd import Function

from ... import kernels as K


def _plan(in_h, in_w, kh, kw, up, down, pad):
    up_x, up_y = up
    down_x, down_y = down
    px0, px1, py0, py1 = pad
    out_h = (in_h * up_y + py0 + py1 - kh) // down_y + 1
    out_w = (in_w * up_x + px0 + px1 - kw) // down_x + 1
    g_pad = (kw - px0 - 1, in_w * up_x - out_w * down_x + px0 - up_x + 1,
             kh - py0 - 1, in_h * up_y - out_h * down_y + py0 - up_y + 1)
    return (out_h, out_w), g_pad


class _UpFirDn2dAdjoint(Function):
    @staticmethod
    def forward(ctx, grad_output, fir, fir_flipped, up, down, pad, g_pad, in_size):
        ctx.save_for_backward(fir)
        ctx.cfg = (up, down, pad)
        gx = K.upfirdn2d_raw(grad_output, fir_flipped, down[0], down[1], up[0], up[1], *g_pad)
        assert gx.shape[2:] == tuple(in_size[2:]), (gx.shape, in_size)
        return gx

    @staticmethod
    def backward(ctx, gg_input):
        (fir,) = ctx.saved_tensors
        up, down, pad = ctx.cfg
        gg_out = K.upfirdn2d_raw(gg_input, fir, up[0], up[1], down[0], down[1], *pad)
        return gg_out, None, None, None, None, None, None, None


class _UpFirDn2d(Function):
    @staticmethod
    def forward(ctx, input, fir, up, down, pad):
        kh, kw = fir.shape
        _, _, in_h, in_w = input.shape
        _, g_pad = _plan(in_h, in_w, kh, kw, up, down, pad)
        ctx.save_for_backward(fir, torch.flip(fir, [0, 1]))
        ctx.cfg = (up, down, pad, g_pad, tuple(input.shape))
        return K.upfirdn2d_raw(input, fir, up[0], up[1], down[0], down[1], *pad)

    @staticmethod
    def backward(ctx, grad_output):
        fir, fir_flipped = ctx.saved_tensors
        up, down, pad, g_pad, in_size = ctx.cfg
        gx = _UpFirDn2dAdjoint.apply(grad_output, fir, fir_flipped, up, down, pad, g_pad, in_size)
        return gx, None, None, None, None


def upfirdn2d(input, kernel, up=1, down=1, pad=(0, 0)):
    """out = decimate(conv(pad(zero_stuff(input, up)), kernel), down); input [N, C, H, W], kernel [kh, kw]."""
    if not input.is_cuda:
        raise RuntimeError("input must be a CUDA tensor")
    dtype = input.dtype
    out = _UpFirDn2d.apply(input, kernel.to(device=input.device), (up, up), (down, down),
                           (pad[0], pad[1], pad[0], pad[1]))
    return out if dtype == torch.float32 else out.to(dtype)
