"""GPEN's generator (blind face restoration, stage 2 of scripts/face_swap.py:208) on the e4s_b200 kernels.

Host-side mirror of the inference half of src/pretrained/gpen/face_model/gpen_model.py: same class names, constructor
arguments (the `device=` argument the reference threads through to pick its CPU op branches is accepted and ignored),
parameter / buffer names and shapes (GPEN-BFR checkpoints load), same `forward` signatures.  GPEN is built from the three
ops of the E4S synthesis path - modulated convolution (:187-284), upfirdn2d, fused bias + leaky ReLU - with three
differences, all handled here on the host side, none needing a new kernel:

* no region mask: every layer is the single-region case of the region-selected kernels;
* "noise" is the encoder's feature map of the same resolution, CONCATENATED on the channel axis (NoiseInjection :287-302,
  isconcat=True), so the activation sees 2 x Cout channels.  FusedLeakyReLU is per channel, hence
  act(cat(conv, w * noise) + bias) = cat(act(conv + bias[:C]), act(w * noise + bias[C:])): the first half is the conv
  kernel's fused epilogue, the second a bias-act pass over the noise; the concatenation is a channels_last copy;
* the encoder is a stack of [Blur pad (2,2)] -> 3x3 stride-2 conv WITHOUT padding -> FusedLeakyReLU (ConvLayer :558-605).
  The tensor-core conv kernel computes padding-1 convolutions and takes stride 2 by keeping even pixels; blurring with
  one more leading pad row/column (pad (3,2)) shifts the blurred image by one pixel, the padded stride-2 convolution of
  that image then equals the reference's at every output but the first row/column, which is dropped.

The discriminator and training-only pieces of the reference file (:690-817) are out of scope.
"""
from __future__ import annotations

import itertools
import math
import random

import torch
from torch import nn

from .. import kernels as K
from ..encoders.psp_encoders import _conv_planes
from ..prepared import cached
from ..stylegan2.model import (Blur, ConstantInput, Downsample, EqualConv2d, EqualLinear, ModulatedConv2d,  # noqa: F401
                               PixelNorm, ScaledLeakyReLU, Upsample, make_kernel, _as_nchw_view)
from ..stylegan2.model import ToRGB as _MaskedToRGB
from ..stylegan2.op import FusedLeakyReLU, fused_leaky_relu, upfirdn2d


def _channels(narrow, channel_multiplier):
    cm = channel_multiplier
    return {4: int(512 * narrow), 8: int(512 * narrow), 16: int(512 * narrow), 32: int(512 * narrow),
            64: int(256 * cm * narrow), 128: int(128 * cm * narrow), 256: int(64 * cm * narrow),
            512: int(32 * cm * narrow), 1024: int(16 * cm * narrow), 2048: int(8 * cm * narrow)}


class NoiseInjection(nn.Module):
    def __init__(self, isconcat=True):
        super().__init__()
        self.isconcat = isconcat
        self.weight = nn.Parameter(torch.zeros(1))

    def forward(self, image, noise=None):
        if noise is None:
            noise = torch.empty_like(image).normal_()
        if self.isconcat:
            return torch.cat((image, self.weight * noise), dim=1)
        return image + self.weight * noise


class StyledConv(nn.Module):
    def __init__(self, in_channel, out_channel, kernel_size, style_dim, upsample=False, blur_kernel=[1, 3, 3, 1],
                 demodulate=True, isconcat=True, device="cpu"):
        super().__init__()
        self.conv = ModulatedConv2d(in_channel, out_channel, kernel_size, style_dim, upsample=upsample,
                                    blur_kernel=blur_kernel, demodulate=demodulate)
        self.noise = NoiseInjection(isconcat)
        self.activate = FusedLeakyReLU(out_channel * (2 if isconcat else 1))

    def forward(self, input, style, noise=None):
        x_pm = K.to_pixel_major(input)
        cout = self.conv.out_channel
        standard_act = self.activate.negative_slope == 0.2 and abs(self.activate.scale - 2 ** 0.5) < 1e-12
        if not (self.noise.isconcat and standard_act):
            y = _as_nchw_view(self.conv.forward_regions(x_pm, style.unsqueeze(1), None))
            return self.activate(self.noise(y, noise=noise))
        # conv half: bias + activation in the kernel's epilogue
        y = self.conv.forward_regions(x_pm, style.unsqueeze(1), None, bias=self.activate.bias[:cout], act=True)
        y = _as_nchw_view(y)
        if noise is None:
            noise = torch.empty_like(y).normal_()
        n = fused_leaky_relu(self.noise.weight * noise, self.activate.bias[cout:], self.activate.negative_slope,
                             self.activate.scale)
        b, _, h, w = y.shape
        out = torch.empty((b, h, w, 2 * cout), device=y.device, dtype=torch.float32)          # pixel-major storage
        out[..., :cout] = y.permute(0, 2, 3, 1)
        out[..., cout:] = n.permute(0, 2, 3, 1)
        return _as_nchw_view(out)


class ToRGB(_MaskedToRGB):
    def __init__(self, in_channel, style_dim, upsample=True, blur_kernel=[1, 3, 3, 1], device="cpu"):
        super().__init__(in_channel, style_dim, upsample=upsample, blur_kernel=blur_kernel, mask_op=False)

    def forward(self, input, style, skip=None):
        return super().forward(input, style, None, skip)


class Generator(nn.Module):
    """gpen_model.py:381-555."""

    def __init__(self, size, style_dim, n_mlp, channel_multiplier=2, blur_kernel=[1, 3, 3, 1], lr_mlp=0.01, isconcat=True,
                 narrow=1, device="cpu"):
        super().__init__()
        self.size = size
        self.n_mlp = n_mlp
        self.style_dim = style_dim
        self.feat_multiplier = 2 if isconcat else 1
        layers = [PixelNorm()]
        layers += [EqualLinear(style_dim, style_dim, lr_mul=lr_mlp, activation="fused_lrelu") for _ in range(n_mlp)]
        self.style = nn.Sequential(*layers)
        self.channels = _channels(narrow, channel_multiplier)
        fm = self.feat_multiplier
        self.input = ConstantInput(self.channels[4])
        self.conv1 = StyledConv(self.channels[4], self.channels[4], 3, style_dim, blur_kernel=blur_kernel, isconcat=isconcat)
        self.to_rgb1 = ToRGB(self.channels[4] * fm, style_dim, upsample=False)
        self.log_size = int(math.log(size, 2))
        self.convs = nn.ModuleList()
        self.upsamples = nn.ModuleList()
        self.to_rgbs = nn.ModuleList()
        in_channel = self.channels[4]
        for i in range(3, self.log_size + 1):
            out_channel = self.channels[2 ** i]
            self.convs.append(StyledConv(in_channel * fm, out_channel, 3, style_dim, upsample=True, blur_kernel=blur_kernel,
                                         isconcat=isconcat))
            self.convs.append(StyledConv(out_channel * fm, out_channel, 3, style_dim, blur_kernel=blur_kernel, isconcat=isconcat))
            self.to_rgbs.append(ToRGB(out_channel * fm, style_dim))
            in_channel = out_channel
        self.n_latent = self.log_size * 2 - 2

    def make_noise(self):
        device = self.input.input.device
        noises = [torch.randn(1, 1, 2 ** 2, 2 ** 2, device=device)]
        for i in range(3, self.log_size + 1):
            for _ in range(2):
                noises.append(torch.randn(1, 1, 2 ** i, 2 ** i, device=device))
        return noises

    def mean_latent(self, n_latent):
        latent_in = torch.randn(n_latent, self.style_dim, device=self.input.input.device)
        return self.style(latent_in).mean(0, keepdim=True)

    def get_latent(self, input):
        return self.style(input)

    def forward(self, styles, return_latents=False, inject_index=None, truncation=1, truncation_latent=None,
                input_is_latent=False, noise=None):
        if not input_is_latent:
            styles = [self.style(s) for s in styles]
        if noise is None:                                               # :508-516 (note: it stops at n_mlp + 1 maps, as the reference)
            batch = styles[0].shape[0]
            noise = []
            for i in range(self.n_mlp + 1):
                size = 2 ** (i + 2)
                noise.append(torch.randn(batch, self.channels[size], size, size, device=styles[0].device))
        if truncation < 1:
            styles = [truncation_latent + truncation * (s - truncation_latent) for s in styles]
        if len(styles) < 2:
            inject_index = self.n_latent
            latent = styles[0].unsqueeze(1).repeat(1, inject_index, 1)
        else:
            if inject_index is None:
                inject_index = random.randint(1, self.n_latent - 1)
            latent = styles[0].unsqueeze(1).repeat(1, inject_index, 1)
            latent2 = styles[1].unsqueeze(1).repeat(1, self.n_latent - inject_index, 1)
            latent = torch.cat([latent, latent2], 1)
        out = self.input(latent)
        out = self.conv1(out, latent[:, 0], noise=noise[0])
        skip = self.to_rgb1(out, latent[:, 1])
        i = 1
        for conv1, conv2, noise1, noise2, to_rgb in zip(self.convs[::2], self.convs[1::2], noise[1::2], noise[2::2], self.to_rgbs):
            out = conv1(out, latent[:, i], noise=noise1)
            out = conv2(out, latent[:, i + 1], noise=noise2)
            skip = to_rgb(out, latent[:, i + 2], skip)
            i += 2
        image = skip
        return (image, latent) if return_latents else (image, None)


class ConvLayer(nn.Sequential):
    """gpen_model.py:558-605; forward runs on the tensor-core conv kernel (see the module docstring)."""

    def __init__(self, in_channel, out_channel, kernel_size, downsample=False, blur_kernel=[1, 3, 3, 1], bias=True,
                 activate=True, device="cpu"):
        layers = []
        if downsample:
            factor = 2
            p = (len(blur_kernel) - factor) + (kernel_size - 1)
            layers.append(Blur(blur_kernel, pad=((p + 1) // 2, p // 2)))
            stride, self.padding = 2, 0
        else:
            stride, self.padding = 1, kernel_size // 2
        layers.append(EqualConv2d(in_channel, out_channel, kernel_size, padding=self.padding, stride=stride,
                                  bias=bias and not activate))
        if activate:
            layers.append(FusedLeakyReLU(out_channel) if bias else ScaledLeakyReLU(0.2))
        super().__init__(*layers)
        self._downsample = downsample

    def _prepared(self, conv):
        return cached(self, "conv", (conv.weight,), conv.weight.device,
                      lambda: _conv_planes(conv.weight * conv.scale, pad_cin_to=32 if conv.weight.shape[1] < 32 else 0))

    def forward(self, input):
        if torch.is_grad_enabled() and (input.requires_grad or any(p.requires_grad for p in self.parameters())):
            raise NotImplementedError("e4s_b200: GPEN's encoder kernels are forward-only (the reference runs GPEN under "
                                      "torch.no_grad(), gpen_demo.py:40); wrap the call in torch.no_grad().")
        mods = list(self)
        conv = mods[1] if self._downsample else mods[0]
        act = mods[-1] if len(mods) > (2 if self._downsample else 1) else None
        k = conv.weight.shape[2]
        cout, cin = conv.weight.shape[:2]
        if cout % 32 or (cin % 32 and cin > 32) or k not in (1, 3):
            raise NotImplementedError(f"ConvLayer {cin}->{cout} k={k}: the conv kernel takes 1x1 / 3x3 and channel counts in multiples of 32")
        planes = self._prepared(conv)
        if self._downsample:
            if k != 3 or input.shape[2] % 2 or input.shape[3] % 2:
                raise NotImplementedError("down-sampling ConvLayer: 3x3 kernels on even-sized inputs")
            blur = mods[0]
            z = upfirdn2d(input, blur.kernel, pad=(blur.pad[0] + 1, blur.pad[1]))              # [B, C, H+2, W+2]
            y = K.conv3x3_tc(K.to_pixel_major(z), planes, out_stride=2)[:, 1:, 1:, :].contiguous()
        else:
            x_pm = K.to_pixel_major(input)
            if cin < 32:                                                                        # RGB input: one 32-channel K chunk
                xp = x_pm.new_zeros(x_pm.shape[:3] + (32,))
                xp[..., :cin] = x_pm
                x_pm = xp
            y = K.conv3x3_tc(x_pm, planes)
        y = _as_nchw_view(y)
        if conv.bias is not None:
            y = y + conv.bias.view(1, -1, 1, 1)
        return act(y) if act is not None else y


class FullGenerator(nn.Module):
    """gpen_model.py:621-688: conv encoder -> latent + per-resolution feature maps -> Generator."""

    def __init__(self, size, style_dim, n_mlp, channel_multiplier=2, blur_kernel=[1, 3, 3, 1], lr_mlp=0.01, isconcat=True,
                 narrow=1, device="cpu"):
        super().__init__()
        channels = _channels(narrow, channel_multiplier)
        self.log_size = int(math.log(size, 2))
        self.generator = Generator(size, style_dim, n_mlp, channel_multiplier=channel_multiplier, blur_kernel=blur_kernel,
                                   lr_mlp=lr_mlp, isconcat=isconcat, narrow=narrow)
        self.ecd0 = nn.Sequential(ConvLayer(3, channels[size], 1))
        in_channel = channels[size]
        self.names = ["ecd%d" % i for i in range(self.log_size - 1)]
        for i in range(self.log_size, 2, -1):
            out_channel = channels[2 ** (i - 1)]
            setattr(self, self.names[self.log_size - i + 1], nn.Sequential(ConvLayer(in_channel, out_channel, 3, downsample=True)))
            in_channel = out_channel
        self.final_linear = nn.Sequential(EqualLinear(channels[4] * 4 * 4, style_dim, activation="fused_lrelu"))

    def forward(self, inputs, return_latents=False, inject_index=None, truncation=1, truncation_latent=None,
                input_is_latent=False):
        noise = []
        for i in range(self.log_size - 1):
            inputs = getattr(self, self.names[i])(inputs)
            noise.append(inputs)
        # the reference flattens a planar [B, C, 4, 4] tensor: channel-major order
        inputs = inputs.contiguous().view(inputs.shape[0], -1)
        outs = self.final_linear(inputs)
        noise = list(itertools.chain.from_iterable(itertools.repeat(x, 2) for x in noise))[::-1]
        return self.generator([outs], return_latents, inject_index, truncation, truncation_latent, input_is_latent,
                              noise=noise[1:])
