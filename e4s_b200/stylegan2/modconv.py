"""Host side of the region-selected modulated convolutions (label pyramid, weight preparation, autograd).

Reference behaviour being replaced: StyledConv / ToRGB run ``ModulatedConv2d`` once per region and
mask-sum the results (src/models/stylegan2/model.py:395-398, 434-437).  Here a float one-hot mask
becomes a uint8 label map once per forward (``LabelPyramid``), each layer selects the style of every
output pixel's own region inside the kernel, and the modulated weights are never materialised
(shared-weight form, model.py:245-274).
"""
from __future__ import annotations

import math
import os
import warnings
import weakref
from typing import Dict, Optional, Tuple

import torch
from torch.autograd import Function
from torch.autograd.function import once_differentiable

from .. import kernels as K

Tensor = torch.Tensor


# =============================================================================== label pyramid
class LabelPyramid:
    """uint8 class map of a one-hot region mask plus its nearest-resized copies.

    ``at(h, w)`` equals ``argmax_c F.interpolate(mask, (h, w), mode='nearest')`` (model.py:391, :430):
    every level is resampled from the ORIGINAL mask, like the reference does, never from another level.
    """

    # one-hot validation is remembered per mask TENSOR OBJECT (weak reference) and version: an address-keyed cache could be hit
    # by a different, freshly allocated mask that recycles a freed tensor's address (round-1 review)
    _validated: Dict[int, Tuple] = {}                 # id(mask) -> (weakref to the mask, its version when validated)

    def __init__(self, label: Tensor, ncls: int):
        assert label.dtype == torch.uint8 and label.ndim == 3
        self.base = label.contiguous()
        self.ncls = int(ncls)
        self._levels: Dict[Tuple[int, int], Tensor] = {tuple(label.shape[1:]): self.base}

    @classmethod
    def from_mask(cls, mask) -> "LabelPyramid":
        if isinstance(mask, LabelPyramid):
            return mask
        if mask.ndim != 4:
            raise RuntimeError(f"mask must be [B, ncls, H, W], got {tuple(mask.shape)}")
        if not mask.is_cuda:
            raise RuntimeError("mask must be a CUDA tensor")
        label, flag = K.onehot_to_label(mask)
        if os.environ.get("E4S_B200_CHECK_MASK", "1") != "0":
            hit = cls._validated.get(id(mask))
            if hit is None or hit[0]() is not mask or hit[1] != mask._version:
                if int(flag.item()) != 0:   # one host sync per distinct mask tensor (and version)
                    raise RuntimeError(
                        "e4s_b200: the region mask is not one-hot (exactly one 1.0 per pixel). The region-selected "
                        "kernels implement the reference's mask-sum (model.py:395-398) for one-hot masks only.")
                key = id(mask)
                cls._validated[key] = (weakref.ref(mask, lambda _r, k=key: cls._validated.pop(k, None)), mask._version)
        return cls(label, mask.shape[1])

    def at(self, h: int, w: int) -> Tensor:
        key = (int(h), int(w))
        if key not in self._levels:
            self._levels[key] = K.label_resize_nearest(self.base, key[0], key[1])
        return self._levels[key]


# =========================================================================== weight preparation
def fold_upsample_kernels(weight: Tensor, blur: Tensor) -> Tensor:
    """Fold conv_transpose2d(stride 2, 3x3) + upfirdn2d(blur 4x4, pad (1,1)) (model.py:287-300) into four
    3x3 kernels, one per output parity (py, px), acting on the INPUT grid with zero padding 1:

        out[2m+py, 2n+px] = sum_{dy,dx} Weff[py,px][:, :, dy, dx] * x[m+dy-1, n+dx-1]
        Weff[py,px][dy,dx] = sum_{ky,kx} W[ky,kx] * blur_flipped[2(dy-1)+ky+1-py, 2(dx-1)+kx+1-px]

    (indices outside 0..3 contribute nothing).  weight: [Cout, Cin, 3, 3]; returns [4, Cout, Cin, 3, 3].
    """
    assert weight.shape[-1] == 3 and tuple(blur.shape) == (4, 4)
    bf = torch.flip(blur.to(torch.float64), [0, 1])
    w64 = weight.to(torch.float64)
    out = torch.zeros((4,) + tuple(weight.shape), dtype=torch.float64, device=weight.device)
    for py in range(2):
        for px in range(2):
            for dy in range(3):
                for dx in range(3):
                    for ky in range(3):
                        a = 2 * (dy - 1) + ky + 1 - py
                        if a < 0 or a > 3:
                            continue
                        for kx in range(3):
                            c = 2 * (dx - 1) + kx + 1 - px
                            if c < 0 or c > 3:
                                continue
                            out[py * 2 + px, :, :, dy, dx] += w64[:, :, ky, kx] * bf[a, c]
    return out.to(torch.float32)


# weight row ky that output parity a takes from source row m - 1 + dy (conv_transpose2d: u[2m + a] = sum_i x[i] w[2m + a - 2i])
CONVT_ROW = {(0, 0): 2, (0, 1): 0, (1, 1): 1}


def convt_class_kernels(weight: Tensor) -> Tensor:
    """The stride-2 conv_transpose2d of model.py:287-300 as a stride-1 convolution on the input grid, padded by one pixel
    before: T'[m, n, (a, c)] = u[2m + a, 2n + c] = sum_{dy,dx in {0,1}} Wc[(a, c), 3 dy + dx] x[m - 1 + dy, n - 1 + dx].
    weight: [Cout, Cin, 3, 3]; returns [9, 4 Cout, Cin] (rows (a, c, o); taps outside {0, 1, 3, 4} and the pairs a parity
    does not use are zero), the operand of e4s_modconv3x3_up_tcr_fwd."""
    cout, cin = weight.shape[:2]
    out = torch.zeros((9, 4, cout, cin), dtype=weight.dtype, device=weight.device)
    for (a, dy), ky in CONVT_ROW.items():
        for (c, dx), kx in CONVT_ROW.items():
            out[3 * dy + dx, 2 * a + c] = weight[:, :, ky, kx]
    return out.reshape(9, 4 * cout, cin)


class PreparedConv:
    """Kernel-ready views of one ModulatedConv2d's frozen parameters, rebuilt when the parameter changes."""

    def __init__(self):
        self.key = None
        self.wt = None      # [nphase, 9, Cin, Cout] (3x3) - scaled by 1/sqrt(fan_in)
        self.wsq = None     # [Cout, Cin] sum_k (scale*W)^2
        self.wrgb = None    # [Cout, Cin] for 1x1 convs
        self.w_hilo = None  # bf16 [2 (hi, lo), nphase, 9, Cout, Cin] operand planes of the tensor-core kernel
        self.w_convt_hilo = None   # up-sampling: bf16 [2, 1, 9, 4 Cout, Cin] transposed-convolution planes
        self.fir = None     # up-sampling: the blur FIR [4, 4] that follows the transposed convolution

    def invalidate(self) -> None:
        """Forget the prepared tensors.  The cache key is (address, autograd version): in-place writes through ``.data``
        (``param.data.copy_()``, EMA ``accumulate`` loops) bump no version - call this (or ``e4s_b200.invalidate_prepared(model)``)
        after them.  ``load_state_dict`` and ordinary in-place ops are picked up automatically."""
        self.key = None

    def get(self, weight: Tensor, upsample: bool, blur: Optional[Tensor]):
        key = (weight.data_ptr(), weight._version, str(weight.device),
               None if blur is None else (blur.data_ptr(), blur._version))
        if key == self.key:
            return self
        with torch.no_grad():
            w = weight.detach().float()[0]                      # [Cout, Cin, k, k]
            cout, cin, k, _ = w.shape
            ws = w * (1.0 / math.sqrt(cin * k * k))             # model.py:223-224
            self.wsq = ws.pow(2).sum((2, 3)).contiguous()
            if k == 1:
                self.wrgb = ws[:, :, 0, 0].contiguous()
                self.wt = None
            else:
                if upsample:
                    wk = fold_upsample_kernels(ws, blur.detach().float())     # [4, Cout, Cin, 3, 3]
                else:
                    wk = ws.unsqueeze(0)
                # -> [nphase, tap, Cin, Cout]
                self.wt = wk.permute(0, 3, 4, 2, 1).reshape(wk.shape[0], 9, cin, cout).contiguous()
                self.wrgb = None
                if K.tc_eligible(cin, cout):
                    wk_k = wk.permute(0, 3, 4, 1, 2).reshape(wk.shape[0], 9, cout, cin)     # K-major rows [.., Cout, Cin]
                    hi = wk_k.to(torch.bfloat16)
                    lo = (wk_k - hi.float()).to(torch.bfloat16)
                    self.w_hilo = torch.stack([hi, lo]).contiguous()
                    self.w_convt_hilo = K.split_bf16(convt_class_kernels(ws)[None]) if upsample else None
                    self.fir = blur.detach().float().contiguous() if upsample else None
                else:
                    self.w_hilo = self.w_convt_hilo = self.fir = None
        self.key = key
        return self


_warned_weight_grad = False


def warn_frozen(*params: Optional[Tensor]):
    """The fused kernels produce gradients for the activations, styles and noise maps only.  Any PARAMETER of the layer that
    requires grad under grad mode (conv weight, NoiseInjection.weight, FusedLeakyReLU bias, ToRGB bias) gets none: say so once."""
    global _warned_weight_grad
    if _warned_weight_grad or not torch.is_grad_enabled():
        return
    if any(p is not None and p.requires_grad for p in params):
        warnings.warn("e4s_b200: synthesis-network weights are treated as frozen (as Net3 does for inference and "
                      "inversion, networks.py:69-71); no gradient is produced for them.")
        _warned_weight_grad = True


def conv_path(prep: "PreparedConv", x_pm: Tensor) -> str:
    """Kernel choice for one layer: 'tcr' (the tensor-core kernel) or 'simt' (exact fp32).  E4S_B200_CONV=auto|tcr|simt.
    auto: the tensor-core kernel for every layer whose channel counts are multiples of 32 (even a single mostly-halo 4x4
    tile per CTA beats the SIMT kernel's latency)."""
    mode = os.environ.get("E4S_B200_CONV", "auto")
    if prep.w_hilo is None or mode == "simt":
        return "simt"
    return "tcr"


# ================================================================================== autograd
class PrecomputedStyle:
    """Modulation output s = EqualLinear(style) [B, R, Cin] (and, for demodulated convs, demod [B, R, Cout]) computed ahead of
    the layer: ``Generator.forward`` runs the modulations of ALL its layers as one launch and the demodulations as a second
    (``kernels.linear_multi``) when no gradient is wanted, and hands each StyledConv / ToRGB one of these instead of a style."""
    __slots__ = ("s", "dm")

    def __init__(self, s: Tensor, dm: Optional[Tensor] = None):
        self.s, self.dm = s, dm


class LinearFn(Function):
    """y = leaky_relu(x @ w^T + bias, slope) on the library's small-GEMM kernel (csrc/linear.cu); w, bias are frozen prepared
    tensors (scale / lr_mul folded in), grouped [G, N, K] or shared [N, K] (kernels.linear).  Differentiable wrt x."""

    @staticmethod
    def forward(ctx, x, w, bias, slope):
        y = K.linear(x, w, bias, slope)
        ctx.slope = float(slope)
        ctx.save_for_backward(w, y if slope != 1.0 else None)
        return y

    @staticmethod
    def backward(ctx, gy):
        w, y = ctx.saved_tensors
        if ctx.slope != 1.0:
            gy = gy * torch.where(y > 0, 1.0, ctx.slope)
        return K.linear(gy.contiguous(), w, None, 1.0, w_is_kn=True), None, None, None


# Smallest output side at which a masked up-sampling layer runs as the gathered transposed convolution.  At 8 x 8 a face
# mask needs ~6 rows per input pixel, more than kernels.convt_masked_cap reserves, so every sample falls back to the
# folded kernel and the row list and the idle launches only add time.
MASKED_CONVT_MIN_RES = 16


class StyledConvFn(Function):
    """y = act(demod * conv(x*s) + noise_w*noise + bias) on pixel-major tensors; differentiable wrt x, s, noise."""

    @staticmethod
    def forward(ctx, x_pm, s, noise, noise_w, bias, label, prep, up, demodulate, act, dm_pre=None):
        dm = (dm_pre if dm_pre is not None else K.demod(s, prep.wsq)) if demodulate else None
        path = conv_path(prep, x_pm)
        if path == "tcr" and up and label is None:
            # one style per sample: the transposed convolution is region-free, so it runs at its own cost (9 MACs per input
            # pixel) and the blur follows as a streaming pass, instead of the four folded parity kernels (36)
            y = K.modconv3x3_up_tcr_fwd(x_pm, prep.w_convt_hilo, prep.fir, s.contiguous(), dm, noise, noise_w, bias, act)
        elif path == "tcr" and up and min(x_pm.shape[1], x_pm.shape[2]) * 2 >= MASKED_CONVT_MIN_RES:
            # masked up-sampling layer from MASKED_CONVT_MIN_RES on: the transposed convolution over (pixel, region) rows
            y = K.modconv3x3_up_masked_tcr_fwd(x_pm, prep.w_convt_hilo, prep.w_hilo, prep.fir, s.contiguous(), dm, label,
                                               noise, noise_w, bias, act)
        elif path == "tcr":
            y = K.modconv3x3_tcr_fwd(x_pm, prep.w_hilo, s.contiguous(), dm, label, noise, noise_w, bias, up, act)
        else:
            y = K.modconv3x3_fwd(x_pm, prep.wt, s.contiguous(), dm, label, noise, noise_w, bias, up, act)
        ctx.set_materialize_grads(False)
        if any(ctx.needs_input_grad[:3]):
            from . import modconv_bwd
            modconv_bwd.save_for_styled_backward(ctx, x_pm, s, dm, noise, noise_w, bias, label, prep, up, demodulate, act, y)
        return y

    @staticmethod
    @once_differentiable            # first-order only: a double backward (R1 / path-length regularisation) raises instead of being wrong
    def backward(ctx, gy):
        from . import modconv_bwd
        return modconv_bwd.styled_backward(ctx, gy)


class ToRGBFn(Function):
    """rgb = conv1x1(x*s) + bias + upsample(skip); differentiable wrt x, s, skip."""

    @staticmethod
    def forward(ctx, x_pm, s, skip, bias, label, prep, fir):
        out = K.torgb_fwd(x_pm, prep.wrgb, s.contiguous(), label, bias, skip, fir)
        ctx.set_materialize_grads(False)
        if any(ctx.needs_input_grad[:3]):
            from . import modconv_bwd
            modconv_bwd.save_for_torgb_backward(ctx, x_pm, s, skip, label, prep, fir)
        return out

    @staticmethod
    @once_differentiable
    def backward(ctx, g):
        from . import modconv_bwd
        return modconv_bwd.torgb_backward(ctx, g)
