"""Tensor-level wrappers over the C ABI (no autograd here; see stylegan2/op and stylegan2/model).

Conventions: "planar" tensors are ordinary contiguous NCHW; "pixel-major" tensors are contiguous
[B, H, W, C] (returned to users as ``.permute(0, 3, 1, 2)`` views, i.e. NCHW tensors with
channels_last strides).  Every function checks device/dtype/contiguity and raises RuntimeError.
"""
from __future__ import annotations

from typing import Optional

import ctypes

import torch

from . import _lib
from ._lib import check, ptr, stream_ptr

Tensor = torch.Tensor


class LaunchStats:
    """Counts kernel launches made through the C ABI and, when `timing` is on, brackets every launch with
    CUDA events on the launching stream (bench.py reads per-kernel device time from here)."""
    launches = 0
    timing = False
    records = []          # (name, work, start_event, end_event); work = algorithmic FLOPs or bytes of the launch

    @classmethod
    def reset(cls, timing=False):
        cls.launches, cls.timing, cls.records = 0, timing, []

    @classmethod
    def summary(cls):
        """name -> (launches, total_ms, total_work).  Call after torch.cuda.synchronize()."""
        out = {}
        for name, work, e0, e1 in cls.records:
            n, ms, w = out.get(name, (0, 0.0, 0.0))
            out[name] = (n + 1, ms + e0.elapsed_time(e1), w + work)
        return out


def _call(name, fn, *args, work=0.0):
    LaunchStats.launches += 1
    if LaunchStats.timing:
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        rc = fn(*args)
        e1.record()
        LaunchStats.records.append((name, work, e0, e1))
    else:
        rc = fn(*args)
    check(rc, name)


def _f32c(t: Tensor, what: str) -> Tensor:
    _lib.require_cuda(t, what)
    if t.dtype != torch.float32:
        t = t.float()
    return t.contiguous()


def to_pixel_major(x: Tensor) -> Tensor:
    """Logical NCHW tensor -> contiguous [B, H, W, C] storage (free if x is already channels_last)."""
    _lib.require_cuda(x)
    xp = x.permute(0, 2, 3, 1)
    if xp.is_contiguous() and x.dtype == torch.float32:
        return xp
    if x.requires_grad and torch.is_grad_enabled():
        return xp.float().contiguous()             # module-boundary path: let autograd track the layout change
    x = _f32c(x, "input")
    b, c, h, w = x.shape
    y = torch.empty((b, h, w, c), device=x.device, dtype=torch.float32)
    with torch.cuda.device(x.device):
        _call("e4s_planar_to_pixel_f32", _lib.load().e4s_planar_to_pixel_f32, ptr(x), ptr(y), b, c, h, w, stream_ptr())
    return y


def to_planar(x_pm: Tensor) -> Tensor:
    """Contiguous [B, H, W, C] -> contiguous NCHW."""
    b, h, w, c = x_pm.shape
    y = torch.empty((b, c, h, w), device=x_pm.device, dtype=torch.float32)
    with torch.cuda.device(x_pm.device):
        _call("e4s_pixel_to_planar_f32", _lib.load().e4s_pixel_to_planar_f32, ptr(x_pm), ptr(y), b, c, h, w, stream_ptr())
    return y


def upfirdn2d_raw(x: Tensor, fir: Tensor, up_x: int, up_y: int, down_x: int, down_y: int, pad_x0: int, pad_x1: int,
                  pad_y0: int, pad_y1: int) -> Tensor:
    """x: planar [N, C, H, W] fp32 CUDA.  Mirrors the pybind op upfirdn2d.cpp:12-19 (NCHW instead of
    the reference's [major, H, W, 1] view)."""
    x = _f32c(x, "input")
    fir = _f32c(fir, "kernel")
    _lib.ensure_device(x)
    n, c, h, w = x.shape
    kh, kw = fir.shape
    out_h = (h * up_y + pad_y0 + pad_y1 - kh) // down_y + 1
    out_w = (w * up_x + pad_x0 + pad_x1 - kw) // down_x + 1
    if out_h <= 0 or out_w <= 0:
        raise RuntimeError(f"upfirdn2d: empty output ({out_h}x{out_w})")
    y = torch.empty((n, c, out_h, out_w), device=x.device, dtype=torch.float32)
    if n * c == 0:
        return y
    with torch.cuda.device(x.device):
        _call("e4s_upfirdn2d_f32", _lib.load().e4s_upfirdn2d_f32, ptr(x), ptr(y), ptr(fir), n * c, h, w, out_h, out_w, kh, kw, up_x, up_y,
                                            down_x, down_y, pad_x0, pad_x1, pad_y0, pad_y1, stream_ptr(),
              work=4.0 * n * c * (h * w + out_h * out_w))
    return y


def bias_act_fwd(x: Tensor, bias: Optional[Tensor], alpha: float, scale: float) -> Tensor:
    """scale*lrelu(x + bias[channel]); channel axis is dim 1 of the LOGICAL tensor.  Works on both planar
    and channels_last storage without a copy."""
    _lib.require_cuda(x, "input")
    if bias is not None:
        _lib.require_cuda(bias, "bias")
        bias = bias.float().contiguous()
    if x.dtype != torch.float32:
        x = x.float()
    _lib.ensure_device(x)
    size_b = x.shape[1] if x.ndim > 1 else 1
    if x.ndim == 4 and not x.is_contiguous() and x.permute(0, 2, 3, 1).is_contiguous():
        step_b = 1                                    # pixel-major storage: channel is the fastest axis
        y = torch.empty_like(x)                       # preserves channels_last strides
    else:
        x = x.contiguous()
        step_b = 1
        for d in x.shape[2:]:
            step_b *= d
        y = torch.empty_like(x)
    n = x.numel()
    if n:
        with torch.cuda.device(x.device):
            _call("e4s_bias_act_fwd_f32", _lib.load().e4s_bias_act_fwd_f32, ptr(x), ptr(bias), ptr(y), n, step_b, size_b, alpha, scale, stream_ptr())
    return y


def _same_storage_order(a: Tensor, like: Tensor) -> Tensor:
    if a.dtype != torch.float32:
        a = a.float()
    if a.stride() == like.stride() and a.shape == like.shape:
        return a
    out = torch.empty_like(like)
    out.copy_(a)
    return out


def bias_act_bwd(grad: Tensor, out: Tensor, alpha: float, scale: float) -> Tensor:
    """gx = scale * (out > 0 ? g : alpha*g); `out` is the forward output (fused_act.py:27-29)."""
    grad = _same_storage_order(grad, out)
    gx = torch.empty_like(out)
    n = out.numel()
    if n:
        with torch.cuda.device(out.device):
            _call("e4s_bias_act_bwd_f32", _lib.load().e4s_bias_act_bwd_f32, ptr(grad), ptr(out), ptr(gx), n, alpha, scale, stream_ptr())
    return gx


def bias_grad(gx: Tensor) -> Tensor:
    """Sum over every axis but the channel axis (dim 1)."""
    c = gx.shape[1]
    gb = torch.empty((c,), device=gx.device, dtype=torch.float32)
    if gx.ndim == 4 and not gx.is_contiguous() and gx.permute(0, 2, 3, 1).is_contiguous():
        outer, step = gx.numel() // c, 1
    else:
        gx = gx.contiguous()
        step = 1
        for d in gx.shape[2:]:
            step *= d
        outer = gx.shape[0]
    with torch.cuda.device(gx.device):
        _call("e4s_bias_grad_f32", _lib.load().e4s_bias_grad_f32, ptr(gx), ptr(gb), outer, c, step, stream_ptr())
    return gb


# ------------------------------------------------------------------------------ mask ops
def onehot_to_label(onehot: Tensor):
    """[B, ncls, H, W] float one-hot -> ([B, H, W] uint8, device int flag: 1 if not one-hot)."""
    onehot = _f32c(onehot, "mask")
    _lib.ensure_device(onehot)
    b, ncls, h, w = onehot.shape
    label = torch.empty((b, h, w), device=onehot.device, dtype=torch.uint8)
    flag = torch.zeros((1,), device=onehot.device, dtype=torch.int32)
    with torch.cuda.device(onehot.device):
        _call("e4s_onehot_to_label_u8", _lib.load().e4s_onehot_to_label_u8, ptr(onehot), ptr(label), ptr(flag), b, ncls, h, w, stream_ptr())
    return label, flag


def label_to_onehot(label: Tensor, ncls: int) -> Tensor:
    """labelMap2OneHot (src/utils/torch_utils.py:166-172).  label: [B,1,H,W] or [B,H,W] integer tensor."""
    _lib.require_cuda(label, "label")
    if label.ndim == 4:
        label = label[:, 0]
    lab = label.to(torch.uint8).contiguous()
    b, h, w = lab.shape
    out = torch.empty((b, ncls, h, w), device=lab.device, dtype=torch.float32)
    with torch.cuda.device(lab.device):
        _call("e4s_label_to_onehot_f32", _lib.load().e4s_label_to_onehot_f32, ptr(lab), ptr(out), b, ncls, h, w, stream_ptr())
    return out


def label_resize_nearest(label: Tensor, out_h: int, out_w: int) -> Tensor:
    label = label.contiguous()
    b, h, w = label.shape
    if (h, w) == (out_h, out_w):
        return label
    out = torch.empty((b, out_h, out_w), device=label.device, dtype=torch.uint8)
    with torch.cuda.device(label.device):
        _call("e4s_label_resize_nearest_u8", _lib.load().e4s_label_resize_nearest_u8, ptr(label), ptr(out), b, h, w, out_h, out_w, stream_ptr())
    return out


def label_remap(label: Tensor, lut: Tensor) -> Tensor:
    label = label.contiguous()
    lut = lut.to(device=label.device, dtype=torch.uint8).contiguous()
    assert lut.numel() == 256
    out = torch.empty_like(label)
    with torch.cuda.device(label.device):
        _call("e4s_label_remap_u8", _lib.load().e4s_label_remap_u8, ptr(label), ptr(out), ptr(lut), label.numel(), stream_ptr())
    return out


def _u8c(t: Tensor, what: str) -> Tensor:
    _lib.require_cuda(t, what)
    if t.dtype != torch.uint8:
        t = t.to(torch.uint8)
    return t.contiguous()


def swap_head_mask(source: Tensor, target: Tensor, hair_first: bool = True):
    """Two 12-class label maps of equal shape -> (swapped labels, hole map in {0, 255}, foreground in {0, 1}), uint8."""
    source, target = _u8c(source, "source"), _u8c(target, "target")
    if source.shape != target.shape:
        raise RuntimeError(f"source {tuple(source.shape)} and target {tuple(target.shape)} label maps differ in shape")
    res, hole, fg = torch.empty_like(target), torch.empty_like(target), torch.empty_like(target)
    if target.numel() == 0:
        return res, hole, fg
    with torch.cuda.device(target.device):
        _call("e4s_swap_head_mask_u8", _lib.load().e4s_swap_head_mask_u8, ptr(source), ptr(target), ptr(res), ptr(hole), ptr(fg),
              target.numel(), int(bool(hair_first)), stream_ptr(), work=5.0 * target.numel())
    return res, hole, fg


def mask_box_morph(mask: Tensor, radius: int, erode: bool, max_val: float = 1e4) -> Tensor:
    """uint8 or fp32 images [..., H, W] -> flat (2r+1)^2 box dilation / erosion with the geodesic border."""
    _lib.require_cuda(mask, "mask")
    if mask.dtype not in (torch.uint8, torch.float32):
        mask = mask.float()
    mask = mask.contiguous()
    if mask.dim() < 2:
        raise RuntimeError("mask must have at least 2 dimensions")
    h, w = mask.shape[-2:]
    out = torch.empty_like(mask)
    if mask.numel() == 0:
        return out
    planes = mask.numel() // (h * w)
    with torch.cuda.device(mask.device):
        if mask.dtype == torch.uint8:
            _call("e4s_mask_box_morph_u8", _lib.load().e4s_mask_box_morph_u8, ptr(mask), ptr(out), planes, h, w, int(radius),
                  int(bool(erode)), stream_ptr(), work=2.0 * mask.numel())
        else:
            _call("e4s_box_morph_f32", _lib.load().e4s_box_morph_f32, ptr(mask), ptr(out), planes, h, w, int(radius),
                  int(bool(erode)), float(max_val), stream_ptr(), work=8.0 * mask.numel())
    return out


def region_mean(feats_pm: Tensor, label: Tensor, ncls: int):
    """feats_pm: [B, H, W, C] contiguous; label: [B, H, W] uint8 -> ([B, ncls, C], area [B, ncls] int32)."""
    b, h, w, c = feats_pm.shape
    out = torch.empty((b, ncls, c), device=feats_pm.device, dtype=torch.float32)
    area = torch.empty((b, ncls), device=feats_pm.device, dtype=torch.int32)
    with torch.cuda.device(feats_pm.device):
        _call("e4s_region_mean_f32", _lib.load().e4s_region_mean_f32, ptr(feats_pm), ptr(label), ptr(out), ptr(area), b, ncls, h, w, c, stream_ptr())
    return out, area


# ------------------------------------------------------------------------------ conv ops
def demod(s: Tensor, wsq: Tensor, eps: float = 1e-8) -> Tensor:
    """s: [..., Cin]; wsq: [Cout, Cin] -> [..., Cout] = rsqrt(s^2 @ wsq^T + eps)."""
    s2 = s.reshape(-1, s.shape[-1]).contiguous()
    rows, cin = s2.shape
    cout = wsq.shape[0]
    out = torch.empty((rows, cout), device=s.device, dtype=torch.float32)
    with torch.cuda.device(s.device):
        if cin % 4 == 0 and cout % 4 == 0:             # tiled GEMM form (csrc/linear.cu)
            ws = _workspace(1, rows, cout, cin, s.device)
            _call("e4s_demod_gemm_f32", _lib.load().e4s_demod_gemm_f32, ptr(s2), ptr(wsq), ptr(out), rows, cin, cout, eps, ptr(ws), stream_ptr())
        else:                                           # warp-per-output form
            _call("e4s_demod_f32", _lib.load().e4s_demod_f32, ptr(s2), ptr(wsq), ptr(out), rows, cin, cout, eps, stream_ptr())
    return out.reshape(*s.shape[:-1], cout)


def _workspace(groups: int, m: int, n: int, k: int, device) -> Optional[Tensor]:
    """K-split scratch of the small-GEMM kernels (None when the shape needs none)."""
    need = int(_lib.load().e4s_linear_workspace_floats(groups, m, n, k))
    return torch.empty(need, device=device, dtype=torch.float32) if need else None


def modconv3x3_fwd(x_pm: Tensor, wt: Tensor, s: Tensor, dm: Optional[Tensor], label: Optional[Tensor],
                   noise: Optional[Tensor], noise_w: Optional[Tensor], bias: Optional[Tensor], up: bool, act: bool) -> Tensor:
    """x_pm [B,H,W,Cin]; wt [nphase,9,Cin,Cout]; s [B,ncls,Cin]; dm [B,ncls,Cout]|None; label [B,Ho,Wo] u8|None;
    noise [B|1, Ho, Wo]|None -> y_pm [B,Ho,Wo,Cout]."""
    b, h, w, cin = x_pm.shape
    cout = wt.shape[-1]
    ncls = s.shape[1]
    m = 2 if up else 1
    y = torch.empty((b, h * m, w * m, cout), device=x_pm.device, dtype=torch.float32)
    nb = noise.shape[0] if noise is not None else 1
    with torch.cuda.device(x_pm.device):
        _call("e4s_modconv3x3_fwd_f32", _lib.load().e4s_modconv3x3_fwd_f32, ptr(x_pm), ptr(wt), ptr(s), ptr(dm), ptr(label), ptr(noise), ptr(noise_w),
                                                 ptr(bias), ptr(y), b, h, w, cin, cout, ncls, int(up), nb, int(act),
                                                 stream_ptr(), work=2.0 * 9 * cin * cout * b * h * w)
    return y


def tc_eligible(cin: int, cout: int) -> bool:
    """Shapes the tensor-core kernel takes (K steps of 32 channels, N tiles of 32 or 64 channels)."""
    return cin % 32 == 0 and cout % 32 == 0


def modconv3x3_tcr_fwd(x_pm: Tensor, w_hilo: Tensor, s: Tensor, dm: Optional[Tensor], label: Optional[Tensor],
                       noise: Optional[Tensor], noise_w: Optional[Tensor], bias: Optional[Tensor], up: bool, act: bool) -> Tensor:
    """Tensor-core path; w_hilo: bf16 [2, nphase, 9, Cout, Cin].  Same contract as modconv3x3_fwd."""
    b, h, w, cin = x_pm.shape
    cout = w_hilo.shape[3]
    ncls = s.shape[1]
    m = 2 if up else 1
    y = torch.empty((b, h * m, w * m, cout), device=x_pm.device, dtype=torch.float32)
    nb = noise.shape[0] if noise is not None else 1
    with torch.cuda.device(x_pm.device):
        _call("e4s_modconv3x3_tcr_fwd", _lib.load().e4s_modconv3x3_tcr_fwd, ptr(x_pm), ptr(w_hilo), ptr(s), ptr(dm), ptr(label),
              ptr(noise), ptr(noise_w), ptr(bias), ptr(y), b, h, w, cin, cout, ncls, int(up), nb, int(act), stream_ptr(),
              work=2.0 * 9 * cin * cout * b * h * w)
    return y


def modconv3x3_up_tcr_fwd(x_pm: Tensor, wt_hilo: Tensor, fir: Tensor, s: Tensor, dm: Optional[Tensor], noise: Optional[Tensor],
                          noise_w: Optional[Tensor], bias: Optional[Tensor], act: bool) -> Tensor:
    """Unmasked up-sampling layer as transposed-convolution GEMM + blur pass; wt_hilo: bf16 [2, 1, 9, 4 Cout, Cin] class-stacked
    planes, fir [4, 4].  Same result as modconv3x3_tcr_fwd with label None and up True."""
    b, h, w, cin = x_pm.shape
    cout = wt_hilo.shape[3] // 4
    t = torch.empty((b, h + 1, w + 1, 4 * cout), device=x_pm.device, dtype=torch.float32)
    y = torch.empty((b, 2 * h, 2 * w, cout), device=x_pm.device, dtype=torch.float32)
    nb = noise.shape[0] if noise is not None else 1
    with torch.cuda.device(x_pm.device):
        _call("e4s_modconv3x3_up_tcr_fwd", _lib.load().e4s_modconv3x3_up_tcr_fwd, ptr(x_pm), ptr(wt_hilo), ptr(fir), ptr(s), ptr(dm),
              ptr(noise), ptr(noise_w), ptr(bias), ptr(t), ptr(y), b, h, w, cin, cout, nb, int(act), stream_ptr(),
              work=2.0 * 9 * cin * cout * b * h * w)
    return y


def convt_masked_cap(h: int, w: int) -> int:
    """(T' pixel, region) rows reserved per sample by modconv3x3_up_masked_tcr_fwd for an H x W input: three per T' pixel.
    Past that the gathered GEMM would do more multiply-accumulates than the folded kernel (36 per input pixel against 9
    per row), so a sample with more rows runs on the folded kernel instead."""
    return 3 * (h + 1) * (w + 1)


def modconv3x3_up_masked_tcr_fwd(x_pm: Tensor, wt_hilo: Tensor, w_hilo: Tensor, fir: Tensor, s: Tensor, dm: Optional[Tensor],
                                 label: Tensor, noise: Optional[Tensor], noise_w: Optional[Tensor], bias: Optional[Tensor],
                                 act: bool) -> Tensor:
    """Masked up-sampling layer as a transposed-convolution GEMM over the (T' pixel, region) pairs the blur reads, plus a
    region-aware blur pass; samples with more than ``convt_masked_cap`` rows fall back to the folded kernel on the device.
    wt_hilo: bf16 [2, 1, 9, 4 Cout, Cin] class-stacked planes, w_hilo: the folded planes [2, 4, 9, Cout, Cin], fir [4, 4].
    Same result as modconv3x3_tcr_fwd with up True."""
    b, h, w, cin = x_pm.shape
    cout = wt_hilo.shape[3] // 4
    ncls = s.shape[1]
    cap = convt_masked_cap(h, w)
    dev = x_pm.device
    need = torch.empty((b, h + 1, w + 1), device=dev, dtype=torch.int32)
    base = torch.empty((b, h + 1, w + 1), device=dev, dtype=torch.int32)
    count = torch.empty((b,), device=dev, dtype=torch.int32)
    rows = torch.empty((b, cap), device=dev, dtype=torch.int32)
    t = torch.empty((b, cap, 4 * cout), device=dev, dtype=torch.float32)
    y = torch.empty((b, 2 * h, 2 * w, cout), device=dev, dtype=torch.float32)
    nb = noise.shape[0] if noise is not None else 1
    with torch.cuda.device(dev):
        _call("e4s_modconv3x3_up_masked_tcr_fwd", _lib.load().e4s_modconv3x3_up_masked_tcr_fwd, ptr(x_pm), ptr(wt_hilo), ptr(w_hilo),
              ptr(fir), ptr(s), ptr(dm), ptr(label), ptr(noise), ptr(noise_w), ptr(bias), ptr(need), ptr(base), ptr(count),
              ptr(rows), ptr(t), ptr(y), b, h, w, cin, cout, ncls, cap, nb, int(act), stream_ptr(),
              work=2.0 * 9 * cin * cout * b * h * w)
    return y


def torgb_fwd(x_pm: Tensor, wrgb: Tensor, s: Tensor, label: Optional[Tensor], bias: Optional[Tensor],
              skip: Optional[Tensor], fir: Optional[Tensor]) -> Tensor:
    """x_pm [B,H,W,Cin]; wrgb [3,Cin]; s [B,ncls,Cin]; skip planar [B,3,H/2,W/2]|None -> planar [B,3,H,W]."""
    b, h, w, cin = x_pm.shape
    out = torch.empty((b, 3, h, w), device=x_pm.device, dtype=torch.float32)
    with torch.cuda.device(x_pm.device):
        _call("e4s_torgb_fwd_f32", _lib.load().e4s_torgb_fwd_f32, ptr(x_pm), ptr(wrgb), ptr(s), ptr(label), ptr(bias), ptr(skip), ptr(fir), ptr(out),
                                            b, h, w, cin, s.shape[1], stream_ptr(), work=4.0 * b * h * w * (cin + 3))
    return out


# ------------------------------------------------------------------------------ backward
def modconv3x3_bwd(gy: Tensor, y: Optional[Tensor], x_pm: Optional[Tensor], wd: Tensor, s: Tensor, dm: Optional[Tensor],
                   label: Optional[Tensor], up: bool, act: bool, need_gx: bool, need_gs: bool):
    """Returns (gx [B,H,W,Cin] | None, gs_conv [B,ncls,Cin] | None)."""
    b, ho, wo, cout = gy.shape
    m = 2 if up else 1
    h, w = ho // m, wo // m
    cin = wd.shape[-1]
    ncls = s.shape[1]
    gx = torch.empty((b, h, w, cin), device=gy.device, dtype=torch.float32) if need_gx else None
    gs = torch.zeros((b, ncls, cin), device=gy.device, dtype=torch.float32) if need_gs else None
    with torch.cuda.device(gy.device):
        _call("e4s_modconv3x3_bwd_f32", _lib.load().e4s_modconv3x3_bwd_f32, ptr(gy), ptr(y), ptr(x_pm), ptr(wd), ptr(s),
              ptr(dm), ptr(label), ptr(gx), ptr(gs), b, h, w, cin, cout, ncls, int(up), int(act), stream_ptr(),
              work=2.0 * 9 * cin * cout * b * h * w)
    return gx, gs


def modconv3x3_bwd_tc(gy: Tensor, y: Optional[Tensor], x_pm: Optional[Tensor], wd_hilo: Tensor, s: Tensor, dm: Optional[Tensor],
                      label: Optional[Tensor], up: bool, act: bool, need_gx: bool, need_gs: bool):
    """Tensor-core backward; wd_hilo bf16 [2, nphase, 9, Cin, Cout].  Returns (gx | None, gs_conv | None)."""
    b, ho, wo, cout = gy.shape
    m = 2 if up else 1
    h, w = ho // m, wo // m
    cin = wd_hilo.shape[3]
    ncls = s.shape[1]
    gx = torch.empty((b, h, w, cin), device=gy.device, dtype=torch.float32) if need_gx else None
    gs = torch.zeros((b, ncls, cin), device=gy.device, dtype=torch.float32) if need_gs else None
    with torch.cuda.device(gy.device):
        _call("e4s_modconv3x3_bwd_tc", _lib.load().e4s_modconv3x3_bwd_tc, ptr(gy), ptr(y), ptr(x_pm), ptr(wd_hilo), ptr(s),
              ptr(dm), ptr(label), ptr(gx), ptr(gs), b, h, w, cin, cout, ncls, int(up), int(act), stream_ptr(),
              work=2.0 * 9 * cin * cout * b * h * w)
    return gx, gs


def class_reduce(gy: Tensor, y: Tensor, label: Optional[Tensor], noise: Optional[Tensor], noise_w: Optional[Tensor],
                 bias: Optional[Tensor], ncls: int, act: bool) -> Tensor:
    b, ho, wo, cout = gy.shape
    gdu = torch.zeros((b, ncls, cout), device=gy.device, dtype=torch.float32)
    nb = noise.shape[0] if noise is not None else 1
    with torch.cuda.device(gy.device):
        _call("e4s_class_reduce_f32", _lib.load().e4s_class_reduce_f32, ptr(gy), ptr(y), ptr(label), ptr(noise), ptr(noise_w),
              ptr(bias), ptr(gdu), b, ncls, ho, wo, cout, nb, int(act), stream_ptr(), work=8.0 * gy.numel())
    return gdu


def torgb_bwd(g: Tensor, x_pm: Tensor, wrgb: Tensor, s: Tensor, label: Optional[Tensor], need_gx: bool, need_gs: bool):
    b, h, w, cin = x_pm.shape
    ncls = s.shape[1]
    gx = torch.empty_like(x_pm) if need_gx else None
    gs = torch.zeros((b, ncls, cin), device=g.device, dtype=torch.float32) if need_gs else None
    with torch.cuda.device(g.device):
        _call("e4s_torgb_bwd_f32", _lib.load().e4s_torgb_bwd_f32, ptr(g), ptr(x_pm), ptr(wrgb), ptr(s), ptr(label), ptr(gx),
              ptr(gs), b, h, w, cin, ncls, stream_ptr(), work=4.0 * b * h * w * (2 * cin + 3))
    return gx, gs


# ------------------------------------------------------------------------------ encoder conv stack
def split_bf16(w: Tensor) -> Tensor:
    """fp32 -> stacked (hi, lo) bf16 planes with hi + lo == w to ~2^-17 relative."""
    hi = w.to(torch.bfloat16)
    lo = (w - hi.float()).to(torch.bfloat16)
    return torch.stack([hi, lo]).contiguous()


def conv3x3_tc(x_pm: Tensor, w_hilo: Tensor, scale: Optional[Tensor] = None, shift: Optional[Tensor] = None,
               prelu: Optional[Tensor] = None, out_stride: int = 1, tap_mask: int = 0) -> Tensor:
    """x_pm [B,H,W,Cin]; w_hilo bf16 [2,1,9,Cout,Cin]; scale/shift [B,Cin]; prelu [Cout].  out_stride 1: [B,H,W,Cout]; 2: the even
    pixels [B,H/2,W/2,Cout]; 4: space-to-depth store [B,H/2,W/2,4*Cout] (channel = (y & 1, x & 1, c)).  tap_mask: the 3x3 taps
    (bit = row-major index) whose weights are not identically zero; 0 = all."""
    b, h, w, cin = x_pm.shape
    cout = w_hilo.shape[3]
    shape = (b, h, w, cout) if out_stride == 1 else (b, h // 2, w // 2, cout if out_stride == 2 else 4 * cout)
    y = torch.empty(shape, device=x_pm.device, dtype=torch.float32)
    ntaps = bin(tap_mask).count("1") if tap_mask else 9
    with torch.cuda.device(x_pm.device):
        _call("e4s_conv3x3_tcr_f32", _lib.load().e4s_conv3x3_tcr_f32, ptr(x_pm), ptr(w_hilo), ptr(scale), ptr(shift), ptr(prelu),
              ptr(y), b, h, w, cin, cout, out_stride, tap_mask, stream_ptr(), work=2.0 * ntaps * cin * cout * b * h * w)
    return y


def conv3x3_bias_tc(x_pm: Tensor, w_hilo: Tensor, bias: Optional[Tensor] = None, residual: Optional[Tensor] = None,
                    relu: bool = False, scale: Optional[Tensor] = None, shift: Optional[Tensor] = None, out_stride: int = 1,
                    tap_mask: int = 0) -> Tensor:
    """conv3x3_tc with the epilogue relu?(acc + bias[o] + residual): bias [Cout]; residual shaped like the output."""
    b, h, w, cin = x_pm.shape
    cout = w_hilo.shape[3]
    shape = (b, h, w, cout) if out_stride == 1 else (b, h // 2, w // 2, cout if out_stride == 2 else 4 * cout)
    if residual is not None and tuple(residual.shape) != shape:
        raise RuntimeError(f"residual {tuple(residual.shape)} does not match the output {shape}")
    y = torch.empty(shape, device=x_pm.device, dtype=torch.float32)
    ntaps = bin(tap_mask).count("1") if tap_mask else 9
    with torch.cuda.device(x_pm.device):
        _call("e4s_conv3x3_bias_tcr_f32", _lib.load().e4s_conv3x3_bias_tcr_f32, ptr(x_pm), ptr(w_hilo), ptr(scale), ptr(shift),
              ptr(bias), ptr(residual), ptr(y), b, h, w, cin, cout, out_stride, tap_mask, int(bool(relu)), stream_ptr(),
              work=2.0 * ntaps * cin * cout * b * h * w)
    return y


def pixel_pitch(t: Tensor, what: str) -> int:
    """Pixel stride (floats) of a pixel-PITCHED fp32 CUDA tensor [B, H, W, C]: a channel slice t = buf[..., c0:c1] of a
    contiguous [B, H, W, Cbuf] buffer, or a contiguous tensor itself (pitch C)."""
    _lib.require_cuda(t, what)
    if t.dtype != torch.float32 or t.dim() != 4:
        raise RuntimeError(f"{what} must be an fp32 [B, H, W, C] tensor, got {t.dtype} {tuple(t.shape)}")
    b, h, w, c = t.shape
    ld = t.stride(2)
    if t.stride(3) != 1 or ld < c or t.stride(1) != w * ld or (b > 1 and t.stride(0) != h * w * ld):
        raise RuntimeError(f"{what}: strides {t.stride()} are not a channel slice of a contiguous [B, H, W, C'] buffer")
    return ld


def conv3x3_dense_tc(x: Tensor, w_hilo: Tensor, bias: Optional[Tensor] = None, out: Optional[Tensor] = None,
                     alpha: float = 1.0, r0: Optional[Tensor] = None, beta: float = 1.0, r1: Optional[Tensor] = None,
                     up: bool = False, lrelu: float = 1.0) -> Tensor:
    """Plain 3x3 convolution on the tensor-core kernel over pixel-pitched operands (``pixel_pitch``): x [B, H, W, Cin] ->
    out [B, Ho, Wo, Cout] (Ho = 2H with ``up``: nearest 2x up-sampling of x first), out = lrelu_slope((((acc + bias) * alpha)
    + r0) * beta + r1), each residual optional and shaped and pitched like out.  ``out`` may be a channel slice of the buffer
    x is a slice of, when the two channel ranges do not overlap.  w_hilo bf16 [2, 1, 9, Cout, Cin]."""
    b, h, w, cin = x.shape
    cout = w_hilo.shape[3]
    m = 2 if up else 1
    shape = (b, h * m, w * m, cout)
    if out is None:
        out = torch.empty(shape, device=x.device, dtype=torch.float32)
    if tuple(out.shape) != shape:
        raise RuntimeError(f"out {tuple(out.shape)} does not match the output {shape}")
    x_ld, y_ld = pixel_pitch(x, "input"), pixel_pitch(out, "out")
    for r, name in ((r0, "r0"), (r1, "r1")):
        if r is not None and (tuple(r.shape) != shape or pixel_pitch(r, name) != y_ld):
            raise RuntimeError(f"{name} {tuple(r.shape)} / {r.stride()} is not shaped and pitched like the output")
    with torch.cuda.device(x.device):
        _call("e4s_conv3x3_dense_tcr_f32", _lib.load().e4s_conv3x3_dense_tcr_f32, ptr(x), x_ld, ptr(w_hilo), ptr(bias),
              float(alpha), ptr(r0), float(beta), ptr(r1), ptr(out), y_ld, b, h, w, cin, cout, int(bool(up)), float(lrelu),
              stream_ptr(), work=2.0 * 9 * cin * cout * b * h * w * m * m)
    return out


def conv3x3_rgb(x: Tensor, w: Tensor, bias: Tensor, out: Optional[Tensor] = None) -> Tensor:
    """RRDBNet's RGB-side convolutions (3x3, padding 1, + bias), w [Cout, Cin, 3, 3]: conv_first, planar x [B, 3, H, W] ->
    pixel-pitched out [B, H, W, 32] (a channel slice of a wider buffer, or allocated); conv_last, pixel-pitched x
    [B, H, W, 32] -> planar [B, 3, H, W]."""
    cout, cin = w.shape[:2]
    if cin == 3:
        b, _, h, wd = x.shape
        if out is None:
            out = torch.empty((b, h, wd, cout), device=x.device, dtype=torch.float32)
        x_ld, y_ld = 0, pixel_pitch(out, "out")
        if tuple(out.shape) != (b, h, wd, cout) or not x.is_contiguous():
            raise RuntimeError(f"conv3x3_rgb: input {tuple(x.shape)} / out {tuple(out.shape)} do not fit")
    else:
        b, h, wd, _ = x.shape
        x_ld, y_ld = pixel_pitch(x, "input"), 0
        out = torch.empty((b, cout, h, wd), device=x.device, dtype=torch.float32)
    with torch.cuda.device(x.device):
        _call("e4s_conv3x3_rgb_f32", _lib.load().e4s_conv3x3_rgb_f32, ptr(x), x_ld, ptr(w), ptr(bias), ptr(out), y_ld, b, h, wd,
              cin, cout, stream_ptr(), work=2.0 * 9 * cin * cout * b * h * wd)
    return out


def space_to_depth(x_pm: Tensor) -> Tensor:
    """[B, H, W, C] -> [B, H/2, W/2, 4C], channel (y & 1, x & 1, c)."""
    b, h, w, c = x_pm.shape
    y = torch.empty((b, h // 2, w // 2, 4 * c), device=x_pm.device, dtype=torch.float32)
    with torch.cuda.device(x_pm.device):
        _call("e4s_space_to_depth_f32", _lib.load().e4s_space_to_depth_f32, ptr(x_pm), ptr(y), b, h, w, c, stream_ptr(),
              work=8.0 * x_pm.numel())
    return y


def channel_mean(x_pm: Tensor) -> Tensor:
    """Spatial mean of pixel-major [B, H, W, C] -> [B, C]."""
    b, h, w, c = x_pm.shape
    y = torch.empty((b, c), device=x_pm.device, dtype=torch.float32)
    with torch.cuda.device(x_pm.device):
        _call("e4s_channel_mean_f32", _lib.load().e4s_channel_mean_f32, ptr(x_pm), ptr(y), b, h * w, c, stream_ptr(),
              work=4.0 * x_pm.numel())
    return y


def bicubic_down_norm(x: Tensor, taps: Tensor, factor: int, mean: Optional[Tensor] = None,
                      std: Optional[Tensor] = None) -> Tensor:
    """planar [B, 3, H, W] -> [B, 3, H/f, W/f]: BicubicDownSample's separable filter (taps [4f] on x's device), then, with
    mean / std ([3] on the device), clamp(0, 1) and (v - mean) / std."""
    b, c, h, w = x.shape
    y = torch.empty((b, 3, h // factor, w // factor), device=x.device, dtype=torch.float32)
    with torch.cuda.device(x.device):
        _call("e4s_bicubic_down_norm_f32", _lib.load().e4s_bicubic_down_norm_f32, ptr(x), ptr(taps), ptr(mean), ptr(std), ptr(y),
              b, h, w, int(factor), stream_ptr(), work=4.0 * (x.numel() + y.numel()))
    return y


def parser_stem(x: Tensor, w7x7: Tensor, bias: Tensor) -> Tensor:
    """planar [B, 3, H, W] -> maxpool3x3/2(relu(conv7x7/2(x) + bias)) pixel-major [B, H/4, W/4, 64]."""
    b, c, h, w = x.shape
    y = torch.empty((b, h // 4, w // 4, 64), device=x.device, dtype=torch.float32)
    with torch.cuda.device(x.device):
        _call("e4s_parser_stem_f32", _lib.load().e4s_parser_stem_f32, ptr(x), ptr(w7x7), ptr(bias), ptr(y), b, h, w, stream_ptr(),
              work=2.0 * 147 * 64 * b * (h // 2) * (w // 2))
    return y


def parse_head(x_pm: Tensor, w1x1: Tensor, out_h: int, out_w: int, lut: Optional[Tensor] = None, labels: bool = True,
               logits: bool = False):
    """x_pm [B, h, w, C], w1x1 [ncls, C] -> (labels uint8 [B, out_h, out_w] | None, logits planar [B, ncls, out_h, out_w] | None):
    1x1 convolution, bilinear align_corners up-sampling, first-index argmax (through lut [256] uint8 when given)."""
    b, h, w, c = x_pm.shape
    ncls = w1x1.shape[0]
    dev = x_pm.device
    lab = torch.empty((b, out_h, out_w), device=dev, dtype=torch.uint8) if labels else None
    lg = torch.empty((b, ncls, out_h, out_w), device=dev, dtype=torch.float32) if logits else None
    with torch.cuda.device(dev):
        _call("e4s_parse_head_u8", _lib.load().e4s_parse_head_u8, ptr(x_pm), ptr(w1x1), ptr(lut), ptr(lab), ptr(lg), b, h, w, c,
              ncls, out_h, out_w, stream_ptr(), work=4.0 * x_pm.numel() + b * out_h * out_w * (1.0 + (4.0 * ncls if logits else 0.0)))
    return lab, lg


def instnorm_affine(x_pm: Tensor, eps: float = 1e-5):
    """InstanceNorm2d statistics of x_pm [B,H,W,C] as (scale, shift), each [B, C]."""
    b, h, w, c = x_pm.shape
    ws = torch.empty((b, c, 2), device=x_pm.device, dtype=torch.float32)
    scale = torch.empty((b, c), device=x_pm.device, dtype=torch.float32)
    shift = torch.empty((b, c), device=x_pm.device, dtype=torch.float32)
    with torch.cuda.device(x_pm.device):
        _call("e4s_instnorm_affine_f32", _lib.load().e4s_instnorm_affine_f32, ptr(x_pm), ptr(ws), ptr(scale), ptr(shift), b, h, w,
              c, eps, stream_ptr(), work=4.0 * x_pm.numel())
    return scale, shift


def norm_residual(y: Tensor, y_scale: Tensor, y_shift: Tensor, alpha: float, shortcut: Optional[Tensor] = None,
                  sc_scale: Optional[Tensor] = None, sc_shift: Optional[Tensor] = None, sc_stride: int = 1,
                  prelu: Optional[Tensor] = None) -> Tensor:
    b, h, w, c = y.shape
    out = torch.empty_like(y)
    with torch.cuda.device(y.device):
        _call("e4s_norm_residual_f32", _lib.load().e4s_norm_residual_f32, ptr(y), ptr(y_scale), ptr(y_shift), float(alpha),
              ptr(shortcut), ptr(sc_scale), ptr(sc_shift), int(sc_stride), ptr(prelu), ptr(out), b, h, w, c, stream_ptr(),
              work=12.0 * y.numel())
    return out


# ------------------------------------------------------------------------------ loss-network inputs
def avgpool_pyramid(x: Tensor):
    """planar x [N, C, H, W] -> (2x2 block means [N, C, H/2, W/2], 4x4 block means [N, C, H/4, W/4]) in one pass."""
    x = _f32c(x, "input")
    _lib.ensure_device(x)
    n, c, h, w = x.shape
    y2 = torch.empty((n, c, h // 2, w // 2), device=x.device, dtype=torch.float32)
    y4 = torch.empty((n, c, h // 4, w // 4), device=x.device, dtype=torch.float32)
    with torch.cuda.device(x.device):
        _call("e4s_avgpool_pyramid_f32", _lib.load().e4s_avgpool_pyramid_f32, ptr(x), ptr(y2), ptr(y4), n * c, h, w, stream_ptr(),
              work=4.0 * x.numel() * (1 + 0.25 + 0.0625))
    return y2, y4


def avgpool_pyramid_bwd(g1: Optional[Tensor], g2: Optional[Tensor], g4: Optional[Tensor], shape) -> Tensor:
    """gx [N, C, H, W] = g1 + up2(g2) / 4 + up4(g4) / 16."""
    n, c, h, w = shape
    ref = next(g for g in (g1, g2, g4) if g is not None)
    g1, g2, g4 = (None if g is None else _f32c(g, "grad") for g in (g1, g2, g4))
    gx = torch.empty((n, c, h, w), device=ref.device, dtype=torch.float32)
    with torch.cuda.device(ref.device):
        _call("e4s_avgpool_pyramid_bwd_f32", _lib.load().e4s_avgpool_pyramid_bwd_f32, ptr(g1), ptr(g2), ptr(g4), ptr(gx), n * c, h, w,
              stream_ptr(), work=4.0 * gx.numel() * (2 + 0.25 + 0.0625))
    return gx


# ------------------------------------------------------------------------------ small GEMMs (style modulation, LocalMLP)
def linear(x: Tensor, w: Tensor, bias: Optional[Tensor] = None, act_slope: float = 1.0, w_is_kn: bool = False) -> Tensor:
    """Grouped small fp32 GEMM on the library's own kernel (csrc/linear.cu).

    x: [G, M, K] or [M, K]; w: [G, N, K] / [N, K] (nn.Linear layout) or, with w_is_kn, [G, K, N] / [K, N]; bias [G, N] / [N].
    A 2-D operand is shared by every group.  Returns [G, M, N] (or [M, N] when nothing is grouped)."""
    x, w = _f32c(x, "input"), _f32c(w, "weight")
    _lib.ensure_device(x)
    groups = max(x.shape[0] if x.ndim == 3 else 1, w.shape[0] if w.ndim == 3 else 1)
    m, k = x.shape[-2], x.shape[-1]
    n = w.shape[-1] if w_is_kn else w.shape[-2]
    assert (w.shape[-2] if w_is_kn else w.shape[-1]) == k, (tuple(x.shape), tuple(w.shape))
    if bias is not None:
        bias = _f32c(bias, "bias")
    grouped = x.ndim == 3 or w.ndim == 3
    y = torch.empty((groups, m, n) if grouped else (m, n), device=x.device, dtype=torch.float32)
    with torch.cuda.device(x.device):
        ws = _workspace(groups, m, n, k, x.device)
        _call("e4s_linear_f32", _lib.load().e4s_linear_f32, ptr(x), ptr(w), ptr(bias), ptr(y), groups, m, n, k,
              m * k if x.ndim == 3 else 0, n * k if w.ndim == 3 else 0, (n if (bias is not None and bias.ndim == 2) else 0), m * n,
              int(w_is_kn), float(act_slope), ptr(ws), stream_ptr(), work=2.0 * groups * m * n * k)
    return y


def linear_multi(problems) -> None:
    """Many small products in one launch per 48 (e4s_linear_multi_f32): problems = [(x_ptr, ldx, w, bias | None, y, m, rsqrt_eps)]
    with x_ptr an int device address of [m, k] fp32 rows ldx floats apart, w [n, k], y [m, n] contiguous fp32 tensors;
    rsqrt_eps < 0: y = x w^T + bias, >= 0: y = rsqrt((x * x) w^T + eps)."""
    arr = (_lib.LinearProblem * len(problems))()
    work = 0.0
    for q, (x_ptr, ldx, w, bias, y, m, eps) in zip(arr, problems):
        n, k = w.shape
        assert w.is_contiguous() and y.is_contiguous() and y.numel() == m * n and w.dtype == y.dtype == torch.float32
        q.x, q.w, q.bias, q.y = x_ptr, w.data_ptr(), (0 if bias is None else bias.data_ptr()), y.data_ptr()
        q.m, q.n, q.k, q.ldx, q.rsqrt_eps = m, n, k, ldx, eps
        work += 2.0 * m * n * k
    dev = problems[0][4].device
    with torch.cuda.device(dev):
        _call("e4s_linear_multi_f32", _lib.load().e4s_linear_multi_f32, ctypes.cast(arr, ctypes.c_void_p), len(problems), stream_ptr(), work=work)
