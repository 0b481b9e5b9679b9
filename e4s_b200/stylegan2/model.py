"""Mask-guided StyleGAN2 synthesis network on the e4s_b200 kernels.

Host-side mirror of the generator half of src/models/stylegan2/model.py: same class names, constructor
arguments, parameter / buffer names and shapes (checkpoint drop-in, SURVEY.md section 5) and the same
``forward`` signatures, so ``Net3`` (src/models/networks.py) and the reference scripts run on it
unchanged.  What differs is the execution:

* every StyledConv / ToRGB is ONE kernel launch for all regions (the reference loops over regions,
  model.py:395-398 / :434-437), with noise, bias and activation fused into the conv epilogue;
* activations travel between layers in pixel-major storage (NCHW tensors with channels_last strides);
* region masks travel as a uint8 label pyramid built once per forward.

Outputs equal the reference's for one-hot masks (tests/test_parity_gpu.py).  The discriminator half of the reference
file (model.py:670-799: ConvLayer, ResBlock, Discriminator) is mirrored at the end of this file on this package's
upfirdn2d / fused-act ops (SURVEY.md section 8 f4: the module, forward and autograd; the training loop of
src/training/coach.py stays out of scope).
"""
from __future__ import annotations

import math
import os
import random

import torch
from torch import nn
from torch.nn import functional as F

from .op import FusedLeakyReLU, fused_leaky_relu, upfirdn2d, conv2d_gradfix
from . import modconv as MC
from .. import kernels as K
from ..prepared import cached


class PixelNorm(nn.Module):
    def forward(self, input):
        return input * torch.rsqrt(input.pow(2).mean(dim=1, keepdim=True) + 1e-8)


def make_kernel(k):
    """1-D taps -> normalised 2-D FIR (reference make_kernel, model.py:23-31)."""
    k = torch.as_tensor(k, dtype=torch.float32)
    if k.ndim == 1:
        k = torch.outer(k, k)
    return k / k.sum()


class Upsample(nn.Module):
    def __init__(self, kernel, factor=2):
        super().__init__()
        self.factor = factor
        self.register_buffer("kernel", make_kernel(kernel) * (factor ** 2))
        p = self.kernel.shape[0] - factor
        self.pad = ((p + 1) // 2 + factor - 1, p // 2)

    def forward(self, input):
        return upfirdn2d(input, self.kernel, up=self.factor, down=1, pad=self.pad)


class Downsample(nn.Module):
    def __init__(self, kernel, factor=2):
        super().__init__()
        self.factor = factor
        self.register_buffer("kernel", make_kernel(kernel))
        p = self.kernel.shape[0] - factor
        self.pad = ((p + 1) // 2, p // 2)

    def forward(self, input):
        return upfirdn2d(input, self.kernel, up=1, down=self.factor, pad=self.pad)


class Blur(nn.Module):
    def __init__(self, kernel, pad, upsample_factor=1):
        super().__init__()
        kernel = make_kernel(kernel)
        if upsample_factor > 1:
            kernel = kernel * (upsample_factor ** 2)
        self.register_buffer("kernel", kernel)
        self.pad = pad

    def forward(self, input):
        return upfirdn2d(input, self.kernel, pad=self.pad)


class EqualConv2d(nn.Module):
    """Plain conv with equalised learning rate (model.py:97-132); used outside the synthesis hot path."""

    def __init__(self, in_channel, out_channel, kernel_size, stride=1, padding=0, bias=True):
        super().__init__()
        self.weight = nn.Parameter(torch.randn(out_channel, in_channel, kernel_size, kernel_size))
        self.scale = 1 / math.sqrt(in_channel * kernel_size ** 2)
        self.stride = stride
        self.padding = padding
        self.bias = nn.Parameter(torch.zeros(out_channel)) if bias else None

    def forward(self, input):
        return conv2d_gradfix.conv2d(input, self.weight * self.scale, bias=self.bias, stride=self.stride,
                                     padding=self.padding)

    def __repr__(self):
        return (f"{self.__class__.__name__}({self.weight.shape[1]}, {self.weight.shape[0]},"
                f" {self.weight.shape[2]}, stride={self.stride}, padding={self.padding})")


class EqualLinear(nn.Module):
    def __init__(self, in_dim, out_dim, bias=True, bias_init=0, lr_mul=1, activation=None):
        super().__init__()
        self.weight = nn.Parameter(torch.randn(out_dim, in_dim).div_(lr_mul))
        self.bias = nn.Parameter(torch.zeros(out_dim).fill_(bias_init)) if bias else None
        self.activation = activation
        self.scale = (1 / math.sqrt(in_dim)) * lr_mul
        self.lr_mul = lr_mul

    def _frozen(self):
        """(weight * scale, bias * lr_mul) of the frozen parameters, cached per parameter version."""
        def build():
            with torch.no_grad():
                return ((self.weight * self.scale).float().contiguous(),
                        None if self.bias is None else (self.bias * self.lr_mul).float().contiguous())
        return cached(self, "frozen", (self.weight, self.bias), self.weight.device, build)

    def forward(self, input):
        trainable = torch.is_grad_enabled() and (self.weight.requires_grad or (self.bias is not None and self.bias.requires_grad))
        if (input.is_cuda and not self.activation and not trainable and input.dtype == torch.float32
                and self.weight.shape[0] % 4 == 0 and self.weight.shape[1] % 4 == 0):
            # the style modulations of the synthesis path (model.py:276): own small-GEMM kernel, no library GEMM
            w, b = self._frozen()
            lead = input.shape[:-1]
            y = MC.LinearFn.apply(input.reshape(-1, input.shape[-1]).contiguous(), w, b, 1.0)
            return y.reshape(*lead, w.shape[0])
        w = self.weight * self.scale
        if self.activation:
            return fused_leaky_relu(F.linear(input, w), self.bias * self.lr_mul)
        return F.linear(input, w, bias=None if self.bias is None else self.bias * self.lr_mul)

    def __repr__(self):
        return f"{self.__class__.__name__}({self.weight.shape[1]}, {self.weight.shape[0]})"


class ScaledLeakyReLU(nn.Module):
    def __init__(self, negative_slope=0.2):
        super().__init__()
        self.negative_slope = negative_slope

    def forward(self, input):
        return F.leaky_relu(input, negative_slope=self.negative_slope) * math.sqrt(2)


def _as_nchw_view(y_pm):
    return y_pm.permute(0, 3, 1, 2)


class ModulatedConv2d(nn.Module):
    """Modulated (and optionally demodulated / up-sampling) convolution, reference model.py:184-320.

    ``forward(input, style)`` takes ONE style per sample ([B, style_dim]) like the reference.  The
    region-selected entry point used by StyledConv / ToRGB is ``forward_regions``.
    """

    def __init__(self, in_channel, out_channel, kernel_size, style_dim, demodulate=True, upsample=False,
                 downsample=False, blur_kernel=[1, 3, 3, 1], fused=True):
        super().__init__()
        if downsample:
            raise NotImplementedError("downsample=True is only used by the discriminator (out of scope)")
        if kernel_size not in (1, 3):
            raise NotImplementedError("e4s_b200 kernels cover the 3x3 and 1x1 modulated convs of the generator")
        self.eps = 1e-8
        self.kernel_size = kernel_size
        self.in_channel = in_channel
        self.out_channel = out_channel
        self.upsample = upsample
        self.downsample = downsample
        if upsample:
            factor = 2
            p = (len(blur_kernel) - factor) - (kernel_size - 1)
            self.blur = Blur(blur_kernel, pad=((p + 1) // 2 + factor - 1, p // 2 + 1), upsample_factor=factor)
        self.scale = 1 / math.sqrt(in_channel * kernel_size ** 2)
        self.padding = kernel_size // 2
        self.weight = nn.Parameter(torch.randn(1, out_channel, in_channel, kernel_size, kernel_size))
        self.modulation = EqualLinear(style_dim, in_channel, bias_init=1)
        self.demodulate = demodulate
        self.fused = fused

    def __repr__(self):
        return (f"{self.__class__.__name__}({self.in_channel}, {self.out_channel}, {self.kernel_size}, "
                f"upsample={self.upsample}, downsample={self.downsample})")

    def prepared(self):
        weight, blur = self.weight, (self.blur.kernel if self.upsample else None)
        MC.warn_frozen(weight)
        return cached(self, "conv", (weight, blur), weight.device,
                      lambda: MC.PreparedConv().get(weight, self.upsample, blur))

    def forward_regions(self, x_pm, styles, label, noise=None, noise_w=None, bias=None, act=False):
        """x_pm [B,H,W,Cin] pixel-major; styles [B, R, style_dim]; label [B,Ho,Wo] uint8 or None (R == 1)."""
        MC.warn_frozen(noise_w, bias)
        if isinstance(styles, MC.PrecomputedStyle):                    # modulations of the whole network ran as one launch
            return MC.StyledConvFn.apply(x_pm, styles.s, noise, noise_w, bias, label, self.prepared(), self.upsample,
                                         self.demodulate, act, styles.dm)
        s = self.modulation(styles)                                    # [B, R, Cin]   (model.py:276)
        return MC.StyledConvFn.apply(x_pm, s, noise, noise_w, bias, label, self.prepared(), self.upsample,
                                     self.demodulate, act)

    def forward(self, input, style):
        x_pm = K.to_pixel_major(input)
        if self.kernel_size == 1:
            if self.out_channel != 3 or self.demodulate:
                raise NotImplementedError("the 1x1 modulated conv is provided in its ToRGB form (3 outputs, no demod)")
            s = self.modulation(style).unsqueeze(1)
            return MC.ToRGBFn.apply(x_pm, s, None, None, None, self.prepared(), None)
        return _as_nchw_view(self.forward_regions(x_pm, style.unsqueeze(1), None))


class NoiseInjection(nn.Module):
    def __init__(self):
        super().__init__()
        self.weight = nn.Parameter(torch.zeros(1))

    def forward(self, image, noise=None):
        if noise is None:
            b, _, h, w = image.shape
            noise = image.new_empty(b, 1, h, w).normal_()
        return image + self.weight * noise


class ConstantInput(nn.Module):
    def __init__(self, channel, size=4):
        super().__init__()
        self.input = nn.Parameter(torch.randn(1, channel, size, size))

    def forward(self, input):
        return self.input.repeat(input.shape[0], 1, 1, 1)


def _fusable_noise(noise, b, h, w):
    return (noise.ndim == 4 and noise.shape[1] == 1 and noise.shape[0] in (1, b)
            and tuple(noise.shape[2:]) == (h, w))


class StyledConv(nn.Module):
    def __init__(self, in_channel, out_channel, kernel_size, style_dim, upsample=False, blur_kernel=[1, 3, 3, 1],
                 demodulate=True, mask_op=False):
        super().__init__()
        self.conv = ModulatedConv2d(in_channel, out_channel, kernel_size, style_dim, upsample=upsample,
                                    blur_kernel=blur_kernel, demodulate=demodulate)
        self.noise = NoiseInjection()
        self.activate = FusedLeakyReLU(out_channel)
        self.mask_op = mask_op

    def forward(self, input, style, mask, noise=None):
        """input [B,Cin,H,W]; style [B,ncls,512] if mask_op else [B,512]; mask one-hot [B,ncls,Hm,Wm] (or a
        LabelPyramid); noise [B|1,1,Ho,Wo] or None (fresh N(0,1), reference model.py:333)."""
        x_pm = K.to_pixel_major(input)
        b, h, w, _ = x_pm.shape
        ho, wo = (2 * h, 2 * w) if self.conv.upsample else (h, w)
        pre = isinstance(style, MC.PrecomputedStyle)
        if self.mask_op:
            label = MC.LabelPyramid.from_mask(mask).at(ho, wo)
            styles = style
        else:
            label, styles = None, (style if pre else style.unsqueeze(1))
        if noise is None:
            noise = x_pm.new_empty(b, 1, ho, wo).normal_()
        standard_act = (self.activate.negative_slope == 0.2 and abs(self.activate.scale - 2 ** 0.5) < 1e-12)
        if _fusable_noise(noise, b, ho, wo) and standard_act:
            y = self.conv.forward_regions(x_pm, styles, label, noise=noise.contiguous().float(),
                                          noise_w=self.noise.weight, bias=self.activate.bias, act=True)
            return _as_nchw_view(y)
        # unusual noise shapes (e.g. per-channel noise): conv kernel, then the op-level pieces
        y = _as_nchw_view(self.conv.forward_regions(x_pm, styles, label))
        return self.activate(self.noise(y, noise=noise))


class ToRGB(nn.Module):
    def __init__(self, in_channel, style_dim, upsample=True, blur_kernel=[1, 3, 3, 1], mask_op=False):
        super().__init__()
        if upsample:
            self.upsample = Upsample(blur_kernel)
        self.conv = ModulatedConv2d(in_channel, 3, 1, style_dim, demodulate=False)
        self.bias = nn.Parameter(torch.zeros(1, 3, 1, 1))
        self.mask_op = mask_op

    def forward(self, input, style, mask, skip=None):
        x_pm = K.to_pixel_major(input)
        b, h, w, _ = x_pm.shape
        pre = isinstance(style, MC.PrecomputedStyle)
        if self.mask_op:
            label = MC.LabelPyramid.from_mask(mask).at(h, w)
            styles = style
        else:
            label, styles = None, (style if pre else style.unsqueeze(1))
        MC.warn_frozen(self.bias)
        s = styles.s if pre else self.conv.modulation(styles)
        prep = self.conv.prepared()
        fuse_skip = (skip is not None and tuple(skip.shape[2:]) == (h // 2, w // 2) and h % 2 == 0 and w % 2 == 0
                     and tuple(self.upsample.kernel.shape) == (4, 4) and self.upsample.pad == (2, 1))
        if skip is None or fuse_skip:
            sk = None if skip is None else skip.contiguous().float()
            fir = None if skip is None else self.upsample.kernel
            return MC.ToRGBFn.apply(x_pm, s, sk, self.bias.reshape(3), label, prep, fir)
        out = MC.ToRGBFn.apply(x_pm, s, None, self.bias.reshape(3), label, prep, None)
        return out + self.upsample(skip)


class Generator(nn.Module):
    """Mask-guided synthesis network (reference Generator, model.py:451-667).

    ``forward`` keeps the reference signature and returns ``(image, latent | None, intermediate_feats)``.
    Layer i < remaining_layer_idx takes per-region latents ``latent[:, :, i]``; later layers take the
    global latent ``latent[:, 0, i]`` (model.py:639-657).
    """

    def __init__(self, size, style_dim, n_mlp, channel_multiplier=2, blur_kernel=[1, 3, 3, 1], lr_mlp=0.01,
                 split_layer_idx=7, remaining_layer_idx=18):
        super().__init__()
        self.split_layer_idx = split_layer_idx
        self.remaining_layer_idx = remaining_layer_idx
        self.size = size
        self.style_dim = style_dim

        mapping = [PixelNorm()]
        mapping += [EqualLinear(style_dim, style_dim, lr_mul=lr_mlp, activation="fused_lrelu") for _ in range(n_mlp)]
        self.style = nn.Sequential(*mapping)

        cm = channel_multiplier
        self.channels = {4: 512, 8: 512, 16: 512, 32: 512, 64: 256 * cm, 128: 128 * cm, 256: 64 * cm, 512: 32 * cm,
                         1024: 16 * cm}
        self.log_size = int(math.log(size, 2))
        self.num_layers = (self.log_size - 2) * 2 + 1
        self.n_latent = self.log_size * 2 - 2
        K_ = remaining_layer_idx
        last_masked_res = 2 + K_ // 2                         # log2 of the last resolution with masked convs

        self.input = ConstantInput(self.channels[4])
        self.conv1 = StyledConv(self.channels[4], self.channels[4], 3, style_dim, blur_kernel=blur_kernel, mask_op=True)
        self.to_rgb1 = ToRGB(self.channels[4], style_dim, upsample=False, mask_op=True)

        self.convs = nn.ModuleList()
        self.upsamples = nn.ModuleList()
        self.to_rgbs = nn.ModuleList()
        self.noises = nn.Module()
        for layer_idx in range(self.num_layers):
            res = 2 ** ((layer_idx + 5) // 2)
            self.noises.register_buffer(f"noise_{layer_idx}", torch.randn(1, 1, res, res))

        cin = self.channels[4]
        for i in range(3, self.log_size + 1):
            cout = self.channels[2 ** i]
            masked = i <= last_masked_res
            self.convs.append(StyledConv(cin, cout, 3, style_dim, upsample=True, blur_kernel=blur_kernel, mask_op=masked))
            self.convs.append(StyledConv(cout, cout, 3, style_dim, blur_kernel=blur_kernel, mask_op=masked))
            self.to_rgbs.append(ToRGB(cout, style_dim, mask_op=(K_ == 17 or i < last_masked_res)))
            cin = cout

    def make_noise(self):
        device = self.input.input.device
        noises = [torch.randn(1, 1, 4, 4, device=device)]
        for i in range(3, self.log_size + 1):
            noises += [torch.randn(1, 1, 2 ** i, 2 ** i, device=device) for _ in range(2)]
        return noises

    def mean_latent(self, n_latent):
        z = torch.randn(n_latent, self.style_dim, device=self.input.input.device)
        return self.style(z).mean(0, keepdim=True)

    def get_latent(self, input):
        return self.style(input)

    def _assemble_latent(self, styles, inject_index):
        if len(styles) < 2:
            if styles[0].ndim < 4:
                return styles[0].unsqueeze(1).repeat(1, self.n_latent, 1)
            return styles[0]
        if inject_index is None:
            inject_index = random.randint(1, self.n_latent - 1)
        first = styles[0].unsqueeze(1).repeat(1, inject_index, 1)
        second = styles[1].unsqueeze(1).repeat(1, self.n_latent - inject_index, 1)
        return torch.cat([first, second], 1)

    def _schedule(self):
        """[(module, latent index, per-region style?)] in execution order: which latent each layer of ``forward`` consumes
        (reference model.py:639-657).  Per-region layers take latent[:, :, i] ([B, ncls, 512]), the others latent[:, 0, i]."""
        K_ = self.remaining_layer_idx
        sched = [(self.conv1, 0, True), (self.to_rgb1, 1, True)]
        i = 1
        for r, to_rgb in enumerate(self.to_rgbs):
            up_conv, conv = self.convs[2 * r], self.convs[2 * r + 1]
            if i < K_:
                sched += [(up_conv, i, up_conv.mask_op), (conv, i + 1, conv.mask_op),
                          (to_rgb, i + 2, to_rgb.mask_op if (K_ == 17 or i + 2 != K_) else False)]
            else:
                sched += [(up_conv, i, False), (conv, i + 1, False), (to_rgb, i + 2, False)]
            i += 2
        return sched

    def _layer_styles(self, latent, sched):
        """What each scheduled layer receives as its style.  Under grad mode with a latent that requires grad (inversion), or
        with trainable modulations: the latent slices themselves (each layer runs its own differentiable EqualLinear).
        Otherwise: every layer's modulation s = EqualLinear(style) in ONE launch and every demodulation rsqrt(s^2 Wsq^T + eps)
        in a second (kernels.linear_multi reads the latent slices in place) instead of ~85 launches of 6-8 us."""
        slices = [latent[:, :, idx] if per_region else latent[:, 0, idx] for _, idx, per_region in sched]
        mods = [m.conv.modulation for m, _, _ in sched]
        wants_grad = torch.is_grad_enabled() and (latent.requires_grad or any(p.requires_grad for m in mods for p in m.parameters()))
        if (wants_grad or not latent.is_cuda or latent.dtype != torch.float32 or not latent.is_contiguous()
                or os.environ.get("E4S_B200_STYLE_BATCH", "1") == "0"
                or any(m.conv.in_channel % 4 or m.conv.out_channel % 4 for m, _, _ in sched if m.conv.kernel_size == 3)
                or any(m.conv.in_channel % 4 for m, _, _ in sched)):
            return slices
        bsz, ncls, nlat, dim = latent.shape
        rows = [bsz * ncls if per_region else bsz for _, _, per_region in sched]
        cins = [m.conv.in_channel for m, _, _ in sched]
        demods = [m.conv.out_channel if (m.conv.demodulate and m.conv.kernel_size == 3) else 0 for m, _, _ in sched]
        s_all = latent.new_empty(sum(r * c for r, c in zip(rows, cins)))
        d_all = latent.new_empty(sum(r * c for r, c in zip(rows, demods)))
        base, esz = latent.data_ptr(), latent.element_size()
        lin, dem, styles, so, do = [], [], [], 0, 0
        for (m, idx, per_region), r, cin, cout in zip(sched, rows, cins, demods):
            w, b = m.conv.modulation._frozen()
            s = s_all[so:so + r * cin].view(bsz, r // bsz, cin)
            so += r * cin
            ldx = nlat * dim if per_region else ncls * nlat * dim
            lin.append((base + idx * dim * esz, ldx, w, b, s, r, -1.0))
            dm = None
            if cout:
                dm = d_all[do:do + r * cout].view(bsz, r // bsz, cout)
                do += r * cout
                dem.append((s.data_ptr(), cin, m.conv.prepared().wsq, None, dm, r, m.conv.eps))
            styles.append(MC.PrecomputedStyle(s, dm))
        K.linear_multi(lin)
        if dem:
            K.linear_multi(dem)
        return styles

    def forward(self, styles, structure_feats, mask, return_latents=False, inject_index=None, truncation=1,
                truncation_latent=None, input_is_latent=False, noise=None, randomize_noise=True,
                use_structure_code=False):
        if not input_is_latent:
            styles = [self.style(s) for s in styles]
        if noise is None:
            if randomize_noise:
                noise = [None] * self.num_layers
            else:
                noise = [getattr(self.noises, f"noise_{i}") for i in range(self.num_layers)]
        if truncation < 1:
            styles = [truncation_latent + truncation * (s - truncation_latent) for s in styles]
        latent = self._assemble_latent(styles, inject_index)
        if latent.ndim != 4:
            raise RuntimeError("the mask-guided generator expects a per-region latent [B, ncls, n_latent, style_dim]")

        K_ = self.remaining_layer_idx
        regions = MC.LabelPyramid.from_mask(mask)            # one argmax + validation per forward
        sched = self._schedule()
        st = iter(self._layer_styles(latent, sched))
        out = self.input(latent)
        out = self.conv1(out, next(st), regions, noise=noise[0])
        skip = self.to_rgb1(out, next(st), regions)
        intermediate_feats = None

        i = 1
        for r, to_rgb in enumerate(self.to_rgbs):
            up_conv, conv = self.convs[2 * r], self.convs[2 * r + 1]
            n_up, n_conv = noise[1 + 2 * r], noise[2 + 2 * r]
            out = up_conv(out, next(st), regions, noise=n_up)
            if i < K_ and i + 2 == self.split_layer_idx:
                if use_structure_code:
                    out = structure_feats
                intermediate_feats = out
            out = conv(out, next(st), regions, noise=n_conv)
            skip = to_rgb(out, next(st), regions, skip)
            i += 2

        image = skip
        return image, (latent if return_latents else None), intermediate_feats


# ================================================================================ discriminator half (model.py:670-799)
class ConvLayer(nn.Sequential):
    """Blur (when down-sampling) -> EqualConv2d -> FusedLeakyReLU / ScaledLeakyReLU, reference model.py:670-716.  The blur and
    the activation run on this package's kernels (upfirdn2d, fused bias + leaky ReLU, both with first- and second-order
    autograd, which R1 regularisation needs); the convolution is the plain library convolution the reference uses."""

    def __init__(self, in_channel, out_channel, kernel_size, downsample=False, blur_kernel=[1, 3, 3, 1], bias=True, activate=True):
        layers = []
        if downsample:
            factor = 2
            p = (len(blur_kernel) - factor) + (kernel_size - 1)
            layers.append(Blur(blur_kernel, pad=((p + 1) // 2, p // 2)))
            stride = 2
            self.padding = 0
        else:
            stride = 1
            self.padding = kernel_size // 2
        layers.append(EqualConv2d(in_channel, out_channel, kernel_size, padding=self.padding, stride=stride,
                                  bias=bias and not activate))
        if activate:
            layers.append(FusedLeakyReLU(out_channel) if bias else ScaledLeakyReLU(0.2))
        super().__init__(*layers)


class ResBlock(nn.Module):
    def __init__(self, in_channel, out_channel, blur_kernel=[1, 3, 3, 1]):
        super().__init__()
        self.conv1 = ConvLayer(in_channel, in_channel, 3)
        self.conv2 = ConvLayer(in_channel, out_channel, 3, downsample=True)
        self.skip = ConvLayer(in_channel, out_channel, 1, downsample=True, activate=False, bias=False)

    def forward(self, input):
        out = self.conv2(self.conv1(input))
        return (out + self.skip(input)) / math.sqrt(2)


class Discriminator(nn.Module):
    """StyleGAN2 discriminator with minibatch standard deviation, reference model.py:740-799 (same module tree and state-dict
    keys: ``convs.N.*``, ``final_conv.*``, ``final_linear.{0,1}.*``)."""

    def __init__(self, size, channel_multiplier=2, blur_kernel=[1, 3, 3, 1]):
        super().__init__()
        cm = channel_multiplier
        channels = {4: 512, 8: 512, 16: 512, 32: 512, 64: 256 * cm, 128: 128 * cm, 256: 64 * cm, 512: 32 * cm, 1024: 16 * cm}
        convs = [ConvLayer(3, channels[size], 1)]
        log_size = int(math.log(size, 2))
        in_channel = channels[size]
        for i in range(log_size, 2, -1):
            out_channel = channels[2 ** (i - 1)]
            convs.append(ResBlock(in_channel, out_channel, blur_kernel))
            in_channel = out_channel
        self.convs = nn.Sequential(*convs)
        self.stddev_group = 4
        self.stddev_feat = 1
        self.final_conv = ConvLayer(in_channel + 1, channels[4], 3)
        self.final_linear = nn.Sequential(EqualLinear(channels[4] * 4 * 4, channels[4], activation="fused_lrelu"),
                                          EqualLinear(channels[4], 1))

    def forward(self, input):
        out = self.convs(input)
        batch, channel, height, width = out.shape
        group = min(batch, self.stddev_group)
        stddev = out.reshape(group, -1, self.stddev_feat, channel // self.stddev_feat, height, width)
        stddev = torch.sqrt(stddev.var(0, unbiased=False) + 1e-8)
        stddev = stddev.mean([2, 3, 4], keepdims=True).squeeze(2)
        stddev = stddev.repeat(group, 1, height, width)
        out = torch.cat([out, stddev], 1)
        out = self.final_conv(out)
        return self.final_linear(out.reshape(batch, -1))
