"""Backward of the fused StyledConv / ToRGB ops: input-, style- (and noise-) gradients; weights are frozen.

Math and kernels: csrc/modconv_bwd.cu.  What the reference does instead: autograd through per-region
F.conv2d / F.conv_transpose2d with per-sample modulated weights (model.py:277-316) - a cuDNN dgrad and wgrad
per region per layer - plus the elementwise chain of mask-multiply, noise, bias-act.
"""
from __future__ import annotations

import torch

from .. import kernels as K
from .op.upfirdn2d import _plan

SQRT2 = 2 ** 0.5


def _dgrad_weights(prep):
    """[nphase, 9, Cin, Cout] forward weights -> [nphase, 9, Cout, Cin] with the taps spatially flipped."""
    if prep.wd is None:
        prep.wd = prep.wt.flip(1).permute(0, 1, 3, 2).contiguous()
    return prep.wd


BWD_MODE_DEFAULT = "auto"        # tensor-core dgrad whenever the channel counts allow it (multiples of 32); "simt" = exact fp32


def _dgrad_planes(prep):
    """bf16 hi/lo operand planes of the dgrad: [2, nphase, 9, Cin, Cout] (taps flipped, K-major over Cout)."""
    if prep.wd_hilo is None:
        prep.wd_hilo = K.split_bf16(prep.wt.flip(1).contiguous())
    return prep.wd_hilo


def _use_tc_bwd(prep, gy) -> bool:
    import os
    mode = os.environ.get("E4S_B200_BWD", BWD_MODE_DEFAULT)
    cin, cout = prep.wt.shape[2], prep.wt.shape[3]
    if mode == "simt" or cin % 32 or cout % 32:
        return False
    return True          # auto == tc: even one 4x4 tile per CTA beats the SIMT dgrad (2.2 ms per 512->512 layer at one face)


def save_for_styled_backward(ctx, x_pm, s, dm, noise, noise_w, bias, label, prep, up, demodulate, act, y):
    ctx.save_for_backward(x_pm, s, dm, noise, noise_w, bias, label, y)
    ctx.cfg = (prep, up, demodulate, act)


def styled_backward(ctx, gy):
    x_pm, s, dm, noise, noise_w, bias, label, y = ctx.saved_tensors
    prep, up, demodulate, act = ctx.cfg
    none11 = [None] * 11
    if gy is None:
        return tuple(none11)
    need_gx, need_gs, need_gn = ctx.needs_input_grad[0], ctx.needs_input_grad[1], ctx.needs_input_grad[2]
    gy = gy.contiguous().float()
    s = s.contiguous()
    gx = gs = None
    if need_gx or need_gs:
        if _use_tc_bwd(prep, gy):
            gx, gs = K.modconv3x3_bwd_tc(gy, y if act else None, x_pm if need_gs else None, _dgrad_planes(prep), s, dm, label,
                                         up, act, need_gx, need_gs)
        else:
            gx, gs = K.modconv3x3_bwd(gy, y if act else None, x_pm if need_gs else None, _dgrad_weights(prep), s, dm, label,
                                      up, act, need_gx, need_gs)
    if need_gs and demodulate:
        # demodulation path: d = rsqrt(s^2 Wsq^T + eps)  ->  d(loss)/ds_i -= s_i * sum_o gdu[o] d[o]^2 Wsq[o,i]
        gdu = K.class_reduce(gy, y, label, noise, noise_w, bias, s.shape[1], act)
        gs = gs - s * torch.matmul(gdu * dm * dm, prep.wsq)
    gn = None
    if need_gn and noise is not None:
        gv = gy * torch.where(y > 0, SQRT2, 0.2 * SQRT2) if act else gy
        gn = (gv.sum(-1) * noise_w).unsqueeze(1)
        if noise.shape[0] == 1 and gn.shape[0] != 1:
            gn = gn.sum(0, keepdim=True)
    none11[0], none11[1], none11[2] = gx, gs, gn
    return tuple(none11)


def save_for_torgb_backward(ctx, x_pm, s, skip, label, prep, fir):
    ctx.save_for_backward(x_pm, s, label, fir)
    ctx.cfg = (prep, None if skip is None else tuple(skip.shape))


def torgb_backward(ctx, g):
    x_pm, s, label, fir = ctx.saved_tensors
    prep, skip_shape = ctx.cfg
    out = [None] * 7
    if g is None:
        return tuple(out)
    g = g.contiguous().float()
    need_gx, need_gs, need_gskip = ctx.needs_input_grad[0], ctx.needs_input_grad[1], ctx.needs_input_grad[2]
    if need_gx or need_gs:
        out[0], out[1] = K.torgb_bwd(g, x_pm, prep.wrgb, s.contiguous(), label, need_gx, need_gs)
    if need_gskip and skip_shape is not None:
        # adjoint of Upsample (upfirdn2d up=2, pad=(2,1), model.py:34-53): flipped FIR, down=2, padding of upfirdn2d.py:108-113
        _, g_pad = _plan(skip_shape[2], skip_shape[3], 4, 4, (2, 2), (1, 1), (2, 1, 2, 1))
        out[2] = K.upfirdn2d_raw(g, torch.flip(fir, [0, 1]), 1, 1, 2, 2, *g_pad)
    return tuple(out)
