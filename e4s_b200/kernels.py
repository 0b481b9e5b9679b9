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


REFLECT_MODES = {"none": 0, "up": 1, "down": 2}


def conv3x3_reflect_tc(x: Tensor, w_hilo: Tensor, bias: Optional[Tensor] = None, out: Optional[Tensor] = None,
                       alpha: float = 1.0, r0: Optional[Tensor] = None, beta: float = 1.0, r1: Optional[Tensor] = None,
                       scale: str = "none", lrelu: float = 1.0) -> Tensor:
    """``conv3x3_dense_tc`` with reflection padding 1 (ParseNet's ``ConvLayer``).  scale "none": x [B, H, W, Cin] -> [B, H, W,
    Cout]; "up": nearest 2x up-sampling first, -> [B, 2H, 2W, Cout]; "down": x is ``space_to_depth`` of the [B, 2H, 2W, Cin / 4]
    input and w_hilo its stride-2 weights (``_conv_planes_s2d``), -> [B, H, W, Cout]."""
    b, h, w, cin = x.shape
    cout = w_hilo.shape[3]
    mode = REFLECT_MODES[scale]
    m = 2 if mode == 1 else 1
    shape = (b, h * m, w * m, cout)
    if out is None:
        out = torch.empty(shape, device=x.device, dtype=torch.float32)
    if tuple(out.shape) != shape:
        raise RuntimeError(f"out {tuple(out.shape)} does not match the output {shape}")
    x_ld, y_ld = pixel_pitch(x, "input"), pixel_pitch(out, "out")
    for r, name in ((r0, "r0"), (r1, "r1")):
        if r is not None and (tuple(r.shape) != shape or pixel_pitch(r, name) != y_ld):
            raise RuntimeError(f"{name} {tuple(r.shape)} / {r.stride()} is not shaped and pitched like the output")
    taps = 4 if mode == 2 else 9
    with torch.cuda.device(x.device):
        _call("e4s_conv3x3_reflect_tcr_f32", _lib.load().e4s_conv3x3_reflect_tcr_f32, ptr(x), x_ld, ptr(w_hilo), ptr(bias),
              float(alpha), ptr(r0), float(beta), ptr(r1), ptr(out), y_ld, b, h, w, cin, cout, mode, float(lrelu),
              stream_ptr(), work=2.0 * taps * cin * cout * b * h * w * m * m)
    return out


def conv3x3_rgb_reflect(x: Tensor, w: Tensor, bias: Tensor, out_hw=None, prep: bool = False) -> Tensor:
    """ParseNet's RGB-side convolutions (3x3, reflection padding 1, + bias), w [Cout, Cin, 3, 3]: encoder.0, planar x
    [B, 3, H, W] -> pixel-major [B, H, W, 64] (``prep``: x is BGR in [0, 1] of any size, the network input is
    F.interpolate(x.flip(1) * 2 - 1, out_hw) with mode 'nearest'); out_img_conv, pixel-pitched x [B, H, W, 64] -> planar
    [B, 3, H, W]."""
    cout, cin = w.shape[:2]
    if cin == 3:
        b, _, hs, ws = x.shape
        h, wd = out_hw if prep else (hs, ws)
        if not x.is_contiguous() or x.dtype != torch.float32:
            raise RuntimeError(f"conv3x3_rgb_reflect: input must be contiguous fp32, got {x.dtype} {tuple(x.shape)}")
        out = torch.empty((b, h, wd, cout), device=x.device, dtype=torch.float32)
        x_ld, y_ld = 0, cout
    else:
        b, h, wd, _ = x.shape
        hs, ws = h, wd
        x_ld, y_ld = pixel_pitch(x, "input"), 0
        out = torch.empty((b, cout, h, wd), device=x.device, dtype=torch.float32)
    with torch.cuda.device(x.device):
        _call("e4s_conv3x3_rgb_reflect_f32", _lib.load().e4s_conv3x3_rgb_reflect_f32, ptr(x), x_ld, hs, ws, int(bool(prep)),
              ptr(w), ptr(bias), ptr(out), y_ld, b, h, wd, cin, cout, stream_ptr(), work=2.0 * 9 * cin * cout * b * h * wd)
    return out


def gpen_parse_head(x: Tensor, w: Tensor, bias: Tensor, lut: Tensor, logits: bool = False, mask: Optional[torch.dtype] = None):
    """ParseNet's out_mask_conv (3x3, reflection padding 1, + bias, w [19, 64, 3, 3]) over pixel-pitched x [B, H, W, 64], then
    lut[first-index argmax] per pixel (lut uint8 [19] on x's device) -> (logits planar [B, 19, H, W] | None, mask [B, H, W] of
    dtype ``mask`` (torch.uint8 or torch.int64) | None)."""
    b, h, wd, cin = x.shape
    ncls = w.shape[0]
    dev = x.device
    lg = torch.empty((b, ncls, h, wd), device=dev, dtype=torch.float32) if logits else None
    mk = torch.empty((b, h, wd), device=dev, dtype=mask) if mask is not None else None
    if mask not in (None, torch.uint8, torch.int64):
        raise RuntimeError(f"gpen_parse_head: mask dtype {mask} is not uint8 or int64")
    with torch.cuda.device(dev):
        _call("e4s_gpen_parse_head_u8", _lib.load().e4s_gpen_parse_head_u8, ptr(x), pixel_pitch(x, "input"), ptr(w), ptr(bias),
              ptr(lut), ptr(lg), ptr(mk if mask == torch.uint8 else None), ptr(mk if mask == torch.int64 else None), b, h, wd,
              cin, ncls, stream_ptr(), work=2.0 * 9 * cin * ncls * b * h * wd)
    return lg, mk


def conv1x1_tc(x: Tensor, w_hilo: Tensor, bias: Optional[Tensor] = None, out: Optional[Tensor] = None, alpha: float = 1.0,
               r0: Optional[Tensor] = None, r_up: Optional[Tensor] = None, stride: int = 1, lrelu: float = 1.0) -> Tensor:
    """1x1 convolution on the tensor-core kernel's pointwise mode over pixel-pitched operands: x [B, s H, s W, Cin] read at
    (s y, s x), s = ``stride`` (1 or 2) -> out [B, H, W, Cout], out = lrelu_slope((acc + bias) * alpha + r0) + r_up, r0 shaped
    and pitched like out, r_up [B, H / 2, W / 2, Cout] pixel-pitched, read at (y >> 1, x >> 1).  w_hilo bf16 [2, Cout, Cin]."""
    b, hi, wi, cin = x.shape
    cout = w_hilo.shape[1]
    if stride not in (1, 2) or hi % stride or wi % stride or tuple(w_hilo.shape) != (2, cout, cin):
        raise RuntimeError(f"conv1x1_tc: input {tuple(x.shape)}, weights {tuple(w_hilo.shape)}, stride {stride} do not fit")
    shape = (b, hi // stride, wi // stride, cout)
    if out is None:
        out = torch.empty(shape, device=x.device, dtype=torch.float32)
    if tuple(out.shape) != shape:
        raise RuntimeError(f"out {tuple(out.shape)} does not match the output {shape}")
    x_ld, y_ld = pixel_pitch(x, "input"), pixel_pitch(out, "out")
    if r0 is not None and (tuple(r0.shape) != shape or pixel_pitch(r0, "r0") != y_ld):
        raise RuntimeError(f"r0 {tuple(r0.shape)} / {r0.stride()} is not shaped and pitched like the output")
    up_ld = 0
    if r_up is not None:
        if tuple(r_up.shape) != (b, shape[1] // 2, shape[2] // 2, cout) or shape[1] % 2 or shape[2] % 2:
            raise RuntimeError(f"r_up {tuple(r_up.shape)} is not the half-resolution map of the output {shape}")
        up_ld = pixel_pitch(r_up, "r_up")
    with torch.cuda.device(x.device):
        _call("e4s_conv1x1_tcr_f32", _lib.load().e4s_conv1x1_tcr_f32, ptr(x), x_ld, ptr(w_hilo), ptr(bias), float(alpha), ptr(r0),
              ptr(r_up), up_ld, ptr(out), y_ld, b, shape[1], shape[2], cin, cout, int(stride), float(lrelu), stream_ptr(),
              work=2.0 * cin * cout * b * shape[1] * shape[2])
    return out


def conv3x3_zero_tc(x: Tensor, w_hilo: Tensor, bias: Optional[Tensor] = None, out: Optional[Tensor] = None,
                    alpha: float = 1.0, r0: Optional[Tensor] = None, beta: float = 1.0, r1: Optional[Tensor] = None,
                    stride: int = 1, lrelu: float = 1.0) -> Tensor:
    """``conv3x3_dense_tc`` (zero padding 1) with the N tile fixed by Cout, so that a sample's output does not depend on the
    batch.  stride 1: x [B, H, W, Cin] -> out [B, H, W, Cout]; stride 2: x is ``space_to_depth`` of the [B, 2H, 2W, Cin / 4]
    input and w_hilo its stride-2 weights (``_conv_planes_s2d``) -> out [B, H, W, Cout]."""
    b, h, w, cin = x.shape
    cout = w_hilo.shape[3]
    shape = (b, h, w, cout)
    if out is None:
        out = torch.empty(shape, device=x.device, dtype=torch.float32)
    if tuple(out.shape) != shape:
        raise RuntimeError(f"out {tuple(out.shape)} does not match the output {shape}")
    x_ld, y_ld = pixel_pitch(x, "input"), pixel_pitch(out, "out")
    for r, name in ((r0, "r0"), (r1, "r1")):
        if r is not None and (tuple(r.shape) != shape or pixel_pitch(r, name) != y_ld):
            raise RuntimeError(f"{name} {tuple(r.shape)} / {r.stride()} is not shaped and pitched like the output")
    k = 9 * cin if stride == 1 else 9 * (cin // 4)
    with torch.cuda.device(x.device):
        _call("e4s_conv3x3_zero_tcr_f32", _lib.load().e4s_conv3x3_zero_tcr_f32, ptr(x), x_ld, ptr(w_hilo), ptr(bias), float(alpha),
              ptr(r0), float(beta), ptr(r1), ptr(out), y_ld, b, h, w, cin, cout, int(stride), float(lrelu), stream_ptr(),
              work=2.0 * k * cout * b * h * w)
    return out


def conv3d_tc(x: Tensor, w_hilo: Tensor, bias: Optional[Tensor] = None, up: bool = False, relu: bool = False) -> Tensor:
    """3x3x3 convolution (padding 1) on the tensor-core kernel's volumetric mode: contiguous x [B, H, W, D, Cin] -> [B, Ho, Wo,
    D, Cout] (Ho, Wo = 2H, 2W with ``up``: nearest up-sampling by (1, 2, 2) first), relu?(acc + bias).  w_hilo bf16 [2, 9,
    Cout, 3 Cin] (``conv3d_planes``)."""
    _lib.require_cuda(x, "input")
    if x.dtype != torch.float32 or x.dim() != 5 or not x.is_contiguous():
        raise RuntimeError(f"conv3d_tc: contiguous fp32 [B, H, W, D, C] input expected, got {x.dtype} {tuple(x.shape)}")
    b, h, w, d, cin = x.shape
    cout = w_hilo.shape[2]
    if tuple(w_hilo.shape) != (2, 9, cout, 3 * cin):
        raise RuntimeError(f"conv3d_tc: weights {tuple(w_hilo.shape)} do not fit the input {tuple(x.shape)}")
    m = 2 if up else 1
    y = torch.empty((b, h * m, w * m, d, cout), device=x.device, dtype=torch.float32)
    with torch.cuda.device(x.device):
        _call("e4s_conv3d_tcr_f32", _lib.load().e4s_conv3d_tcr_f32, ptr(x), ptr(w_hilo), ptr(bias), ptr(y), b, d, h, w, cin, cout,
              int(bool(up)), int(bool(relu)), stream_ptr(), work=2.0 * 27 * cin * cout * b * d * h * w * m * m)
    return y


def voxel_pitch(t: Tensor, what: str) -> int:
    """Voxel stride (floats) of a voxel-PITCHED fp32 CUDA tensor [B, H, W, D, C]: a channel slice t = buf[..., c0:c1] of a
    contiguous [B, H, W, D, Cbuf] buffer, or a contiguous tensor itself (pitch C)."""
    _lib.require_cuda(t, what)
    if t.dtype != torch.float32 or t.dim() != 5:
        raise RuntimeError(f"{what} must be an fp32 [B, H, W, D, C] tensor, got {t.dtype} {tuple(t.shape)}")
    b, h, w, d, c = t.shape
    vp = t.stride(3)
    if t.stride(4) != 1 or vp < c or t.stride(2) != d * vp or t.stride(1) != w * d * vp or (b > 1 and t.stride(0) != h * w * d * vp):
        raise RuntimeError(f"{what}: strides {t.stride()} are not a channel slice of a contiguous [B, H, W, D, C'] buffer")
    return vp


def conv3d_pitched_tc(x: Tensor, w_hilo: Tensor, bias: Optional[Tensor] = None, out: Optional[Tensor] = None, up: bool = False,
                      relu: bool = False) -> Tensor:
    """``conv3d_tc`` over voxel-pitched operands (``voxel_pitch``): x [B, H, W, D, Cin] -> out [B, Ho, Wo, D, Cout], either a
    channel slice of a wider buffer (the hourglass's skip concatenations) or allocated."""
    b, h, w, d, cin = x.shape
    cout = w_hilo.shape[2]
    if tuple(w_hilo.shape) != (2, 9, cout, 3 * cin):
        raise RuntimeError(f"conv3d_pitched_tc: weights {tuple(w_hilo.shape)} do not fit the input {tuple(x.shape)}")
    m = 2 if up else 1
    shape = (b, h * m, w * m, d, cout)
    if out is None:
        out = torch.empty(shape, device=x.device, dtype=torch.float32)
    if tuple(out.shape) != shape:
        raise RuntimeError(f"out {tuple(out.shape)} does not match the output {shape}")
    x_vp, y_vp = voxel_pitch(x, "input"), voxel_pitch(out, "out")
    with torch.cuda.device(x.device):
        _call("e4s_conv3d_pitched_tcr_f32", _lib.load().e4s_conv3d_pitched_tcr_f32, ptr(x), x_vp, ptr(w_hilo), ptr(bias), ptr(out),
              y_vp, b, d, h, w, cin, cout, int(bool(up)), int(bool(relu)), stream_ptr(),
              work=2.0 * 27 * cin * cout * b * d * h * w * m * m)
    return out


def avgpool2_vox(x: Tensor, out: Optional[Tensor] = None) -> Tensor:
    """AvgPool3d((1, 2, 2)) of contiguous x [B, H, W, D, C] -> out [B, H / 2, W / 2, D, C], voxel-pitched (a channel slice of
    a wider buffer) or allocated."""
    _lib.require_cuda(x, "input")
    if x.dtype != torch.float32 or x.dim() != 5 or not x.is_contiguous():
        raise RuntimeError(f"avgpool2_vox: contiguous fp32 [B, H, W, D, C] input expected, got {x.dtype} {tuple(x.shape)}")
    b, h, w, d, c = x.shape
    shape = (b, h // 2, w // 2, d, c)
    if out is None:
        out = torch.empty(shape, device=x.device, dtype=torch.float32)
    if tuple(out.shape) != shape:
        raise RuntimeError(f"out {tuple(out.shape)} does not match the output {shape}")
    with torch.cuda.device(x.device):
        _call("e4s_avgpool2_vox_f32", _lib.load().e4s_avgpool2_vox_f32, ptr(x), ptr(out), voxel_pitch(out, "out"), b, h, w, d, c,
              stream_ptr(), work=5.0 * out.numel())
    return out


def conv7x7_slices_tc(x: Tensor, w_hilo: Tensor) -> Tensor:
    """7x7 convolution (zero padding 3) of every depth slice of contiguous x [B, H, W, D, Cin] with w_hilo bf16 [2, 49, 128,
    Cin] (tap 7 ky + kx) -> [B, D, H, W, 128]."""
    _lib.require_cuda(x, "input")
    if x.dtype != torch.float32 or x.dim() != 5 or not x.is_contiguous():
        raise RuntimeError(f"conv7x7_slices_tc: contiguous fp32 [B, H, W, D, C] input expected, got {x.dtype} {tuple(x.shape)}")
    b, h, w, d, cin = x.shape
    if tuple(w_hilo.shape) != (2, 49, 128, cin) or w_hilo.dtype != torch.bfloat16 or not w_hilo.is_contiguous():
        raise RuntimeError(f"conv7x7_slices_tc: weights {tuple(w_hilo.shape)} do not fit the input {tuple(x.shape)}")
    y = torch.empty((b, d, h, w, 128), device=x.device, dtype=torch.float32)
    with torch.cuda.device(x.device):
        _call("e4s_conv7x7_slices_tcr_f32", _lib.load().e4s_conv7x7_slices_tcr_f32, ptr(x), ptr(w_hilo), ptr(y), b, d, h, w, cin,
              stream_ptr(), work=2.0 * 49 * cin * 128 * b * d * h * w)
    return y


def vid2vid_compress(feature: Tensor, wb: Tensor) -> Tensor:
    """DenseMotionNetwork's compress + folded BatchNorm + ReLU: contiguous fp32 NCDHW feature [B, 32, D, H, W], wb [132]
    (the folded [4, 32] weights, then the 4 biases) -> [B, D, H, W, 4]."""
    _lib.require_cuda(feature, "feature")
    if feature.dtype != torch.float32 or feature.dim() != 5 or feature.shape[1] != 32 or not feature.is_contiguous():
        raise RuntimeError(f"vid2vid_compress: contiguous fp32 [B, 32, D, H, W] feature expected, got {feature.dtype} "
                           f"{tuple(feature.shape)}")
    wb = _f32c(wb, "weights")
    if wb.numel() != 132:
        raise RuntimeError(f"vid2vid_compress: weights {tuple(wb.shape)} are not the 132 folded values")
    b, _, d, h, w = feature.shape
    y = torch.empty((b, d, h, w, 4), device=feature.device, dtype=torch.float32)
    with torch.cuda.device(feature.device):
        _call("e4s_vid2vid_compress_f32", _lib.load().e4s_vid2vid_compress_f32, ptr(feature), ptr(wb), ptr(y), b, d, h, w,
              stream_ptr(), work=2.0 * 32 * 4 * b * d * h * w)
    return y


def _keypoints(kp: Tensor, b: int, what: str) -> Tensor:
    kp = _f32c(kp, what)
    if tuple(kp.shape) != (b, 15, 3):
        raise RuntimeError(f"{what} {tuple(kp.shape)} is not [{b}, 15, 3]")
    return kp


def vid2vid_motion_input(comp: Tensor, kp_driving: Tensor, kp_source: Tensor, out: Tensor) -> Tensor:
    """The hourglass input of DenseMotionNetwork from comp [B, D, H, W, 4] (``vid2vid_compress``) and the keypoints
    [B, 15, 3] into out [B, H, W, D, 96], voxel-pitched: channel 5 k + j is the heatmap difference (j = 0) or compressed
    channel j - 1 sampled at sparse motion k; channels 80..95 zero."""
    _lib.require_cuda(comp, "comp")
    if comp.dtype != torch.float32 or comp.dim() != 5 or comp.shape[4] != 4 or not comp.is_contiguous():
        raise RuntimeError(f"vid2vid_motion_input: contiguous fp32 [B, D, H, W, 4] volume expected, got {tuple(comp.shape)}")
    b, d, h, w, _ = comp.shape
    kd, ks = _keypoints(kp_driving, b, "kp_driving"), _keypoints(kp_source, b, "kp_source")
    if tuple(out.shape) != (b, h, w, d, 96):
        raise RuntimeError(f"out {tuple(out.shape)} is not [{b}, {h}, {w}, {d}, 96]")
    with torch.cuda.device(comp.device):
        _call("e4s_vid2vid_motion_input_f32", _lib.load().e4s_vid2vid_motion_input_f32, ptr(comp), ptr(kd), ptr(ks), ptr(out),
              voxel_pitch(out, "out"), b, d, h, w, stream_ptr(), work=16.0 * 40 * b * d * h * w)
    return out


def vid2vid_motion_combine(p: Tensor, mask_bias: Tensor, occ_bias: Tensor, kp_driving: Tensor, kp_source: Tensor):
    """DenseMotionNetwork's outputs from the per-slice GEMM p [B, D, H, W, 128] (``conv7x7_slices_tc``): (mask [B, 16, D, H, W],
    deformation [B, D, H, W, 3], occlusion_map [B, 1, H, W])."""
    _lib.require_cuda(p, "p")
    if p.dtype != torch.float32 or p.dim() != 5 or p.shape[4] != 128 or not p.is_contiguous():
        raise RuntimeError(f"vid2vid_motion_combine: contiguous fp32 [B, D, H, W, 128] expected, got {tuple(p.shape)}")
    b, d, h, w, _ = p.shape
    kd, ks = _keypoints(kp_driving, b, "kp_driving"), _keypoints(kp_source, b, "kp_source")
    mb, ob = _f32c(mask_bias, "mask_bias"), _f32c(occ_bias, "occ_bias")
    if mb.numel() != 16 or ob.numel() != 1:
        raise RuntimeError(f"vid2vid_motion_combine: biases {tuple(mb.shape)}, {tuple(ob.shape)} are not [16], [1]")
    dev = p.device
    mask = torch.empty((b, 16, d, h, w), device=dev, dtype=torch.float32)
    deformation = torch.empty((b, d, h, w, 3), device=dev, dtype=torch.float32)
    occlusion = torch.empty((b, 1, h, w), device=dev, dtype=torch.float32)
    with torch.cuda.device(dev):
        _call("e4s_vid2vid_motion_combine_f32", _lib.load().e4s_vid2vid_motion_combine_f32, ptr(p), ptr(mb), ptr(ob), ptr(kd),
              ptr(ks), ptr(mask), ptr(deformation), ptr(occlusion), b, d, h, w, stream_ptr(), work=200.0 * b * d * h * w)
    return mask, deformation, occlusion


def conv3d_planes(w: Tensor) -> Tensor:
    """Conv3d weight [Cout, Cin, 3, 3, 3] -> the volumetric mode's bf16 hi / lo planes [2, 9, Cout, 3 Cin]: tap 3 ky + kx,
    K index kz Cin + c."""
    cout, cin = w.shape[:2]
    return split_bf16(w.float().permute(3, 4, 0, 2, 1).reshape(9, cout, 3 * cin).contiguous())


def conv3d_useful_rows(b: int, d: int, ho: int, wo: int) -> float:
    """Fraction of the pixel rows of the volumetric mode's tiles that hold an output voxel, for B x D slices of ho x wo."""
    mh, mw = ctypes.c_int(), ctypes.c_int()
    check(_lib.load().e4s_conv3d_tcr_plan(b, d, ho, wo, ctypes.byref(mh), ctypes.byref(mw)), "e4s_conv3d_tcr_plan")
    tiles = -(-mh.value // 8) * -(-mw.value // 16)
    return b * d * ho * wo / (tiles * 128.0)


def vid2vid_kp_prep(x: Tensor, filt: Tensor) -> Tensor:
    """KPDetector's AntiAliasInterpolation2d (scale 1/4) of planar fp32 x [B, 3, H, W] with the filter buffer [3, 1, 13, 13]
    -> pixel-major [B, H / 4, W / 4, 32], channels 3..31 zero."""
    _lib.require_cuda(x, "input")
    if x.dtype != torch.float32 or x.dim() != 4 or x.shape[1] != 3 or not x.is_contiguous():
        raise RuntimeError(f"vid2vid_kp_prep: contiguous fp32 [B, 3, H, W] input expected, got {x.dtype} {tuple(x.shape)}")
    filt = _f32c(filt, "filter")
    if filt.numel() != 3 * 13 * 13:
        raise RuntimeError(f"vid2vid_kp_prep: filter {tuple(filt.shape)} is not [3, 1, 13, 13]")
    b, _, h, w = x.shape
    y = torch.empty((b, h // 4, w // 4, 32), device=x.device, dtype=torch.float32)
    with torch.cuda.device(x.device):
        _call("e4s_vid2vid_kp_prep_f32", _lib.load().e4s_vid2vid_kp_prep_f32, ptr(x), ptr(filt), ptr(y), b, h, w, stream_ptr(),
              work=2.0 * 3 * 169 * b * (h // 4) * (w // 4))
    return y


def avgpool2(x_pm: Tensor) -> Tensor:
    """AvgPool2d(2) of contiguous pixel-major [B, H, W, C] -> [B, H / 2, W / 2, C]."""
    _lib.require_cuda(x_pm, "input")
    if x_pm.dtype != torch.float32 or x_pm.dim() != 4 or not x_pm.is_contiguous():
        raise RuntimeError(f"avgpool2: contiguous fp32 [B, H, W, C] input expected, got {x_pm.dtype} {tuple(x_pm.shape)}")
    b, h, w, c = x_pm.shape
    y = torch.empty((b, h // 2, w // 2, c), device=x_pm.device, dtype=torch.float32)
    with torch.cuda.device(x_pm.device):
        _call("e4s_avgpool2_f32", _lib.load().e4s_avgpool2_f32, ptr(x_pm), ptr(y), b, h, w, c, stream_ptr(), work=5.0 * y.numel())
    return y


def vid2vid_heatmap(logits: Tensor, num_kp: int, temperature: float) -> Tensor:
    """Keypoints [B, num_kp, 3] of contiguous logits [B, H, W, D, C] (keypoint k at channel k): per keypoint softmax(logits /
    temperature) over the voxels and the expectation of make_coordinate_grid's (x, y, z)."""
    _lib.require_cuda(logits, "logits")
    if logits.dtype != torch.float32 or logits.dim() != 5 or not logits.is_contiguous():
        raise RuntimeError(f"vid2vid_heatmap: contiguous fp32 [B, H, W, D, C] logits expected, got {tuple(logits.shape)}")
    b, h, w, d, c = logits.shape
    kp = torch.empty((b, num_kp, 3), device=logits.device, dtype=torch.float32)
    with torch.cuda.device(logits.device):
        _call("e4s_vid2vid_heatmap_f32", _lib.load().e4s_vid2vid_heatmap_f32, ptr(logits), c, float(temperature), ptr(kp), b, num_kp,
              d, h, w, stream_ptr(), work=12.0 * b * num_kp * d * h * w)
    return kp


# ------------------------------------------------------------------------------ face-vid2vid's SPADE generator
def conv3d_residual_tc(x: Tensor, w_hilo: Tensor, bias: Tensor, residual: Tensor, relu: bool = False) -> Tensor:
    """``conv3d_tc`` (no up-sampling) plus a residual after the bias, before the ReLU: relu?(acc + bias + residual), residual
    contiguous and shaped like the output [B, H, W, D, Cout]."""
    _lib.require_cuda(x, "input")
    if x.dtype != torch.float32 or x.dim() != 5 or not x.is_contiguous():
        raise RuntimeError(f"conv3d_residual_tc: contiguous fp32 [B, H, W, D, C] input expected, got {x.dtype} {tuple(x.shape)}")
    b, h, w, d, cin = x.shape
    cout = w_hilo.shape[2]
    if tuple(w_hilo.shape) != (2, 9, cout, 3 * cin):
        raise RuntimeError(f"conv3d_residual_tc: weights {tuple(w_hilo.shape)} do not fit the input {tuple(x.shape)}")
    shape = (b, h, w, d, cout)
    residual = _f32c(residual, "residual")
    if tuple(residual.shape) != shape:
        raise RuntimeError(f"residual {tuple(residual.shape)} does not match the output {shape}")
    y = torch.empty(shape, device=x.device, dtype=torch.float32)
    with torch.cuda.device(x.device):
        _call("e4s_conv3d_residual_tcr_f32", _lib.load().e4s_conv3d_residual_tcr_f32, ptr(x), ptr(w_hilo), ptr(bias),
              ptr(residual), ptr(y), b, d, h, w, cin, cout, int(bool(relu)), stream_ptr(),
              work=2.0 * 27 * cin * cout * b * d * h * w)
    return y


def conv3x3_zero_up_tc(x: Tensor, w_hilo: Tensor, bias: Optional[Tensor] = None, up: int = 2, lrelu: float = 1.0) -> Tensor:
    """``conv3x3_zero_tc`` over the nearest up-sampling of pixel-pitched x [B, H, W, Cin] by ``up`` (2 or 4), read through
    the halo copy (never written) -> [B, up H, up W, Cout] = lrelu_slope(acc + bias).  The N tile follows Cout only."""
    b, h, w, cin = x.shape
    cout = w_hilo.shape[3]
    if up not in (2, 4) or tuple(w_hilo.shape) != (2, 1, 9, cout, cin):
        raise RuntimeError(f"conv3x3_zero_up_tc: input {tuple(x.shape)}, weights {tuple(w_hilo.shape)}, up {up} do not fit")
    out = torch.empty((b, h * up, w * up, cout), device=x.device, dtype=torch.float32)
    with torch.cuda.device(x.device):
        _call("e4s_conv3x3_zero_up_tcr_f32", _lib.load().e4s_conv3x3_zero_up_tcr_f32, ptr(x), pixel_pitch(x, "input"), ptr(w_hilo),
              ptr(bias), ptr(out), cout, b, h, w, cin, cout, up.bit_length() - 1, float(lrelu), stream_ptr(),
              work=2.0 * 9 * cin * cout * b * h * w * up * up)
    return out


def instnorm_stats(x: Tensor, eps: float = 1e-5):
    """InstanceNorm2d statistics of pixel-pitched x [B, H, W, C] as (scale, shift), each [B, C]: scale = 1 / sqrt(var + eps)
    (biased variance), shift = -mean scale, summed in double in an order fixed by H, W and C (bit identical at any batch;
    ``instnorm_affine`` splits by the batch and sums with atomics)."""
    b, h, w, c = x.shape
    ld = pixel_pitch(x, "input")
    ws = torch.empty((b, -(-h * w // 1024), c, 2), device=x.device, dtype=torch.float64)
    scale = torch.empty((b, c), device=x.device, dtype=torch.float32)
    shift = torch.empty((b, c), device=x.device, dtype=torch.float32)
    with torch.cuda.device(x.device):
        _call("e4s_instnorm_stats_fixed_f32", _lib.load().e4s_instnorm_stats_fixed_f32, ptr(x), ld, ptr(ws), ptr(scale), ptr(shift),
              b, h, w, c, float(eps), stream_ptr(), work=4.0 * b * h * w * c)
    return scale, shift


def spade_tc(actv: Tensor, w_hilo: Tensor, bias: Tensor, x: Tensor, scale: Tensor, shift: Tensor, slope: float = 1.0) -> Tensor:
    """SPADE: the 3x3 gamma / beta convolutions of pixel-pitched actv [B, H, W, Cin] as one GEMM of interleaved columns
    (``spade_planes``), whose epilogue writes lrelu_slope((x scale + shift) (1 + gamma) + beta) -> [B, H, W, C]; x
    pixel-pitched [B, H, W, C], or [B, H / 2, W / 2, C] read at (y >> 1, x >> 1) (its nearest up-sampling); scale, shift
    [B, C] (``instnorm_stats`` of x)."""
    b, h, w, cin = actv.shape
    c2 = w_hilo.shape[3]
    c = c2 // 2
    if tuple(w_hilo.shape) != (2, 1, 9, c2, cin) or tuple(bias.shape) != (c2,):
        raise RuntimeError(f"spade_tc: weights {tuple(w_hilo.shape)} / bias {tuple(bias.shape)} do not fit {tuple(actv.shape)}")
    if x.shape[0] != b or x.shape[3] != c or tuple(x.shape[1:3]) not in ((h, w), (h // 2, w // 2)):
        raise RuntimeError(f"spade_tc: x {tuple(x.shape)} is neither [{b}, {h}, {w}, {c}] nor at half resolution")
    half = int(tuple(x.shape[1:3]) != (h, w))
    for t, name in ((scale, "scale"), (shift, "shift")):
        if tuple(t.shape) != (b, c) or t.dtype != torch.float32 or not t.is_contiguous():
            raise RuntimeError(f"spade_tc: {name} {tuple(t.shape)} is not a contiguous fp32 [{b}, {c}]")
    out = torch.empty((b, h, w, c), device=actv.device, dtype=torch.float32)
    with torch.cuda.device(actv.device):
        _call("e4s_spade_tcr_f32", _lib.load().e4s_spade_tcr_f32, ptr(actv), pixel_pitch(actv, "actv"), ptr(w_hilo), ptr(bias),
              ptr(x), pixel_pitch(x, "x"), half, ptr(scale), ptr(shift), ptr(out), c, b, h, w, cin, c, float(slope),
              stream_ptr(), work=2.0 * 9 * cin * c2 * b * h * w)
    return out


def spade_planes(w_gamma: Tensor, w_beta: Tensor) -> Tensor:
    """mlp_gamma / mlp_beta weights [C, Cin, 3, 3] -> ``spade_tc``'s bf16 planes [2, 1, 9, 2 C, Cin], row 2 k gamma k and
    row 2 k + 1 beta k."""
    w = torch.stack([w_gamma.float(), w_beta.float()], 1).reshape(-1, *w_gamma.shape[1:])
    return split_bf16(w.permute(2, 3, 0, 1).reshape(1, 9, w.shape[0], w.shape[1]).contiguous())


def conv1x1_factor_tc(x: Tensor, w_hilo: Tensor, bias: Tensor, factor: Tensor) -> Tensor:
    """``conv1x1_tc`` times a per-pixel factor: pixel-pitched x [B, H, W, Cin] -> [B, H, W, Cout] = (acc + bias)
    factor[b, y, x], factor [B, H, W] (or [B, 1, H, W])."""
    b, h, w, cin = x.shape
    cout = w_hilo.shape[1]
    if tuple(w_hilo.shape) != (2, cout, cin):
        raise RuntimeError(f"conv1x1_factor_tc: weights {tuple(w_hilo.shape)} do not fit the input {tuple(x.shape)}")
    factor = _f32c(factor, "factor")
    if factor.numel() != b * h * w:
        raise RuntimeError(f"conv1x1_factor_tc: factor {tuple(factor.shape)} is not [{b}, {h}, {w}]")
    out = torch.empty((b, h, w, cout), device=x.device, dtype=torch.float32)
    with torch.cuda.device(x.device):
        _call("e4s_conv1x1_factor_tcr_f32", _lib.load().e4s_conv1x1_factor_tcr_f32, ptr(x), pixel_pitch(x, "input"), ptr(w_hilo),
              ptr(bias), ptr(factor), ptr(out), cout, b, h, w, cin, cout, stream_ptr(), work=2.0 * cin * cout * b * h * w)
    return out


def vid2vid_warp(vol: Tensor, deformation: Tensor) -> Tensor:
    """deform_input: F.grid_sample (trilinear, zero padding, align_corners=False) of contiguous vol [B, H, W, D, 32] at
    deformation [B, D, H, W, 3] -> [B, H, W, D 32], channel z 32 + c."""
    _lib.require_cuda(vol, "vol")
    if vol.dtype != torch.float32 or vol.dim() != 5 or vol.shape[4] != 32 or not vol.is_contiguous():
        raise RuntimeError(f"vid2vid_warp: contiguous fp32 [B, H, W, D, 32] volume expected, got {vol.dtype} {tuple(vol.shape)}")
    b, h, w, d, _ = vol.shape
    deformation = _f32c(deformation, "deformation")
    if tuple(deformation.shape) != (b, d, h, w, 3):
        raise RuntimeError(f"vid2vid_warp: deformation {tuple(deformation.shape)} is not [{b}, {d}, {h}, {w}, 3]")
    y = torch.empty((b, h, w, d * 32), device=vol.device, dtype=torch.float32)
    with torch.cuda.device(vol.device):
        _call("e4s_vid2vid_warp_f32", _lib.load().e4s_vid2vid_warp_f32, ptr(vol), ptr(deformation), ptr(y), b, d, h, w,
              stream_ptr(), work=16.0 * 32 * b * d * h * w)
    return y


def conv3x3_rgb_act(x: Tensor, w: Tensor, bias: Tensor) -> Tensor:
    """The SPADE generator's RGB-side convolutions (3x3, zero padding 1, + bias), w [Cout, Cin, 3, 3]: ``first``, planar x
    [B, 3, H, W] -> pixel-major [B, H, W, 64], then ReLU; ``conv_img``, pixel-pitched x [B, H, W, 64] -> planar
    [B, 3, H, W], then the sigmoid."""
    cout, cin = w.shape[:2]
    w, bias = _f32c(w, "weights"), _f32c(bias, "bias")
    if cin == 3:
        x = _f32c(x, "input")
        b, _, h, wd = x.shape
        out = torch.empty((b, h, wd, cout), device=x.device, dtype=torch.float32)
        x_ld, y_ld, act = 0, cout, 1
    else:
        b, h, wd, _ = x.shape
        x_ld, y_ld, act = pixel_pitch(x, "input"), 0, 2
        out = torch.empty((b, cout, h, wd), device=x.device, dtype=torch.float32)
    with torch.cuda.device(x.device):
        _call("e4s_conv3x3_rgb_act_f32", _lib.load().e4s_conv3x3_rgb_act_f32, ptr(x), x_ld, ptr(w), ptr(bias), ptr(out), y_ld, b, h,
              wd, cin, cout, act, stream_ptr(), work=2.0 * 9 * cin * cout * b * h * wd)
    return out


def retinaface_prep(x: Tensor) -> Tensor:
    """Planar BGR [B, 3, H, W] pixel values (uint8 or fp32, CUDA) -> fp32 x - (104, 117, 123)."""
    if x.dtype not in (torch.uint8, torch.float32) or not x.is_contiguous():
        raise RuntimeError(f"retinaface_prep: contiguous uint8 / fp32 input expected, got {x.dtype}")
    b, c, h, w = x.shape
    y = torch.empty((b, 3, h, w), device=x.device, dtype=torch.float32)
    with torch.cuda.device(x.device):
        _call("e4s_retinaface_prep_f32", _lib.load().e4s_retinaface_prep_f32, ptr(x), int(x.dtype == torch.uint8), ptr(y), b, h, w,
              stream_ptr(), work=4.0 * y.numel())
    return y


def retinaface_num_priors(h: int, w: int) -> int:
    return 2 * sum((h // s) * (w // s) for s in (8, 16, 32))


def retinaface_decode(heads: Tensor, batch: int, h: int, w: int, resize: float = 1.0, conf_thr: float = 0.0, boxes=True,
                      keys=True, module=False):
    """The detector's per-prior tail over the three levels' head maps (``heads``: flat fp32, level after level, each
    [B, h / s, w / s, 32]).  Returns (boxes [B, P, 4], landms [B, P, 10], keys [B, P]) when ``boxes`` (keys: the score where
    > conf_thr, else -inf), and / or (loc [B, P, 4], conf [B, P, 2], landm [B, P, 10]) when ``module``."""
    n = retinaface_num_priors(h, w)
    dev = heads.device
    e = lambda *s: torch.empty(s, device=dev, dtype=torch.float32)  # noqa: E731
    bx, lm = (e(batch, n, 4), e(batch, n, 10)) if boxes else (None, None)
    ky = e(batch, n) if keys else None
    lc, cf, lr = (e(batch, n, 4), e(batch, n, 2), e(batch, n, 10)) if module else (None, None, None)
    with torch.cuda.device(dev):
        _call("e4s_retinaface_decode_f32", _lib.load().e4s_retinaface_decode_f32, ptr(heads), batch, h, w, float(resize),
              float(conf_thr), ptr(bx), ptr(lm), ptr(ky), ptr(lc), ptr(cf), ptr(lr), stream_ptr(), work=4.0 * 32 * batch * n / 2)
    return (bx, lm, ky), (lc, cf, lr)


def retinaface_nms(boxes: Tensor, landms: Tensor, keys_sorted: Tensor, order: Tensor, conf_thr: float, nms_thr: float,
                   top_k: int, keep_top_k: int):
    """Selection and greedy NMS per image (see e4s_retinaface_nms_f32): -> (dets [B, keep_top_k, 5], landms [B, keep_top_k,
    10] in x1..x5, y1..y5 order, count [B] int32); slots past count are unspecified."""
    b, n = keys_sorted.shape
    dev = boxes.device
    if order.dtype != torch.int64 or not (boxes.is_contiguous() and landms.is_contiguous() and keys_sorted.is_contiguous()
                                           and order.is_contiguous()):
        raise RuntimeError("retinaface_nms: contiguous operands and int64 order expected")
    dets = torch.empty((b, keep_top_k, 5), device=dev, dtype=torch.float32)
    lm = torch.empty((b, keep_top_k, 10), device=dev, dtype=torch.float32)
    count = torch.empty((b,), device=dev, dtype=torch.int32)
    with torch.cuda.device(dev):
        _call("e4s_retinaface_nms_f32", _lib.load().e4s_retinaface_nms_f32, ptr(boxes), ptr(landms), ptr(keys_sorted), ptr(order),
              b, n, float(conf_thr), float(nms_thr), int(top_k), int(keep_top_k), ptr(dets if keep_top_k else None),
              ptr(lm if keep_top_k else None), ptr(count), stream_ptr(), work=4.0 * b * min(top_k, n))
    return dets, lm, count


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
