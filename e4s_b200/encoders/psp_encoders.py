"""RGI (region-wise) encoder: mirror of FSEncoder_PSP, src/models/encoders/psp_encoders.py:238-309.

The module tree (``input_layer``, ``body.N.{shortcut_layer,res_layer}``) and its parameter names are the
reference's, so E4S checkpoints load.  ``forward`` does not run those torch modules: the whole conv stack executes
on the e4s_b200 kernels -

* every 3x3 convolution (and the 1x1 stride-2 shortcut convolutions, as centre-tap 3x3 kernels) on the
  tensor-core kernel ``e4s_conv3x3_tcr_f32`` (split-bf16 x3, fp32 accumulate); a stride-2 convolution runs as four taps over the
  space-to-depth output of the convolution before it, a 1x1 shortcut as the centre tap alone (tap mask);
* InstanceNorm as per-(sample, channel) statistics (``e4s_instnorm_affine_f32``) folded onto the operand of the
  following convolution, PReLU in the convolution epilogue;
* the unit tail ``0.5 * IN(conv2) + shortcut`` in one pass (``e4s_norm_residual_f32``); 0.5 is the SE gate - the
  squeeze input is an InstanceNorm output (zero spatial mean) and the SE convolutions have no bias, so
  sigmoid(fc2(relu(fc1(0)))) = 0.5 for any weights (helpers.py:56-72, 136-137);
* per-region pooling ``get_per_comp_styleCode`` (:264-283; a B x ncls Python loop with a host sync and a
  masked_select per region in the reference) as ONE kernel over a uint8 label map (``e4s_region_mean_f32``).

Gradients through the encoder are training-only (scripts call it under ``torch.no_grad()``,
scripts/optimization.py:178-180, scripts/face_swap.py:149) and are not provided.
"""
import os

import torch
from torch import nn

from .helpers import get_block, bottleneck_IR_SE_Ours
from .. import kernels as K
from ..prepared import cached
from ..stylegan2.modconv import LabelPyramid


def _conv_planes(weight: torch.Tensor, pad_cin_to: int = 0) -> torch.Tensor:
    """nn.Conv2d weight [Cout, Cin, k, k] (k = 3, or 1 -> centre tap) -> bf16 operand planes [2, 1, 9, Cout, Cin']."""
    w = weight.detach().float()
    cout, cin, k, _ = w.shape
    if k == 1:
        w3 = w.new_zeros(cout, cin, 3, 3)
        w3[:, :, 1, 1] = w[:, :, 0, 0]
        w = w3
    if pad_cin_to and cin < pad_cin_to:
        w = torch.cat([w, w.new_zeros(cout, pad_cin_to - cin, 3, 3)], 1)
    return K.split_bf16(w.permute(2, 3, 0, 1).reshape(1, 9, cout, w.shape[1]))


TAP_UNITS = (6, 20, 23)  # body units whose outputs are pooled into the 256 + 512 + 512 wide code (the last of blocks 2-4)
TAPS_S2D = 0x1B          # taps (dy, dx) in {-1, 0}^2 of a 3x3 kernel: bits 0, 1, 3, 4
TAP_CENTRE = 0x10


def _conv_planes_s2d(weight: torch.Tensor) -> torch.Tensor:
    """Stride-2 3x3 convolution (padding 1) as a stride-1 kernel on the space-to-depth tensor x4[y, x, (py, px, c)] =
    x[2y + py, 2x + px, c]: input row 2y + ky - 1 is (dy, py) = (-1, 1), (0, 0), (0, 1) for ky = 0, 1, 2 (same for columns), so
    only the taps (dy, dx) in {-1, 0}^2 carry weights: W4[dy, dx][:, (py, px, c)] = W[:, c, ky, kx].  [Cout, Cin, 3, 3] ->
    bf16 operand planes [2, 1, 9, Cout, 4 Cin]; the other five taps are zero and are skipped through the kernel's tap mask."""
    w = weight.detach().float()
    cout, cin, k, _ = w.shape
    assert k == 3
    w4 = w.new_zeros(9, cout, 4, cin)
    tap_of = {0: (-1, 1), 1: (0, 0), 2: (0, 1)}           # k -> (d, parity)
    for ky in range(3):
        dy, py = tap_of[ky]
        for kx in range(3):
            dx, px = tap_of[kx]
            w4[(dy + 1) * 3 + (dx + 1), :, py * 2 + px, :] = w[:, :, ky, kx]
    return K.split_bf16(w4.reshape(1, 9, cout, 4 * cin))


class FSEncoder_PSP(nn.Module):
    def __init__(self, mode="ir_se", opts=None):
        super().__init__()
        assert mode in ["ir_se"], "the E4S RGI encoder is the ir_se variant (networks.py:48)"
        blocks = [get_block(64, 128, 3), get_block(128, 256, 4), get_block(256, 512, 14), get_block(512, 512, 3)]
        self.n_styles = 11
        self.input_layer = nn.Sequential(nn.Conv2d(3, 64, (3, 3), 1, 1, bias=False), nn.InstanceNorm2d(64), nn.PReLU(64))
        self.body = nn.Sequential(*[bottleneck_IR_SE_Ours(u.in_channel, u.depth, u.stride) for blk in blocks for u in blk])

    # ------------------------------------------------------------------------------------------ weights
    def _prepared(self, name: str, weight: torch.Tensor, pad_cin_to: int = 0, s2d: bool = False) -> torch.Tensor:
        return cached(self, name, (weight,), weight.device,
                      lambda: _conv_planes_s2d(weight) if s2d else _conv_planes(weight, pad_cin_to))

    # ------------------------------------------------------------------------------------------ pooling
    def get_per_comp_styleCode(self, style_feats, segmap):
        """style_feats [B,C,h,w] (or pixel-major [B,h,w,C] storage); segmap one-hot [B,ncls,H,W] -> [B,ncls,C]."""
        regions = LabelPyramid.from_mask(segmap)
        h, w = style_feats.shape[2:]
        codes, _area = K.region_mean(K.to_pixel_major(style_feats), regions.at(h, w), regions.ncls)
        return codes

    # ------------------------------------------------------------------------------------------ conv stack
    def _input_layer(self, x: torch.Tensor) -> torch.Tensor:
        """input_layer (conv 3 -> 64, InstanceNorm, PReLU) on planar x [B,3,H,W] -> pixel-major [B,H,W,64]."""
        b, c, h, w = x.shape
        xp = x.new_zeros((b, h, w, 32), dtype=torch.float32)             # 3 -> 32 channels (one 64-byte K chunk)
        xp[..., :c] = x.permute(0, 2, 3, 1)
        conv0, prelu0 = self.input_layer[0], self.input_layer[2]
        y = K.conv3x3_tc(xp, self._prepared("in", conv0.weight, pad_cin_to=32))
        s0, t0 = K.instnorm_affine(y)
        return K.norm_residual(y, s0, t0, 1.0, prelu=prelu0.weight)      # PReLU(IN(conv))

    def _unit(self, idx: int, unit: bottleneck_IR_SE_Ours, x: torch.Tensor) -> torch.Tensor:
        """One bottleneck_IR_SE_Ours on pixel-major x [B,H,W,Cin] (helpers.py:122-144)."""
        conv1, prelu, conv2 = unit.res_layer[1], unit.res_layer[2], unit.res_layer[3]
        stride = conv2.stride[0]
        sx, tx = K.instnorm_affine(x)                                                     # res_layer[0]
        if stride == 2 and x.shape[1] % 2 == 0 and x.shape[2] % 2 == 0 and os.environ.get("E4S_B200_ENC_S2D", "1") != "0":
            # true stride 2: conv1 stores its output space-to-depth, conv2 is then four taps over 4 C channels at the OUTPUT
            # resolution (16 C Cout MACs per output instead of the 36 C Cout of "every pixel, keep the even ones")
            r = K.conv3x3_tc(x, self._prepared(f"{idx}.c1", conv1.weight), sx, tx, prelu.weight, out_stride=4)
            r = K.conv3x3_tc(r, self._prepared(f"{idx}.c2s", conv2.weight, s2d=True), tap_mask=TAPS_S2D)
        else:
            r = K.conv3x3_tc(x, self._prepared(f"{idx}.c1", conv1.weight), sx, tx, prelu.weight)   # conv + PReLU
            r = K.conv3x3_tc(r, self._prepared(f"{idx}.c2", conv2.weight), out_stride=stride)
        s2, t2 = K.instnorm_affine(r)                                                     # res_layer[4]
        if isinstance(unit.shortcut_layer, nn.MaxPool2d):                                 # MaxPool2d(1, stride) == subsample
            return K.norm_residual(r, s2, t2, 0.5, shortcut=x, sc_stride=stride)
        # 1x1 stride-2 shortcut (helpers.py:125-131): sub-sample FIRST (a quarter of the pixels), then the centre-tap kernel at
        # the output resolution (the other eight taps are masked: neither loaded nor multiplied)
        xs = x[:, ::stride, ::stride, :].contiguous() if stride > 1 else x
        sc = K.conv3x3_tc(xs, self._prepared(f"{idx}.sc", unit.shortcut_layer[0].weight), tap_mask=TAP_CENTRE)
        ss, ts = K.instnorm_affine(sc)
        return K.norm_residual(r, s2, t2, 0.5, shortcut=sc, sc_scale=ss, sc_shift=ts, sc_stride=1)

    def forward(self, x, segmap):
        """x [B,3,256,256]; segmap one-hot [B,ncls,Hm,Wm] -> ([B,ncls,1280], zeros [B,512,16,16])."""
        if torch.is_grad_enabled() and (x.requires_grad or any(p.requires_grad for p in self.parameters())):
            raise NotImplementedError("e4s_b200: the RGI encoder kernels are forward-only (the reference runs the encoder "
                                      "under torch.no_grad() on this path); wrap the call in torch.no_grad().")
        h, w = x.shape[2:]
        if h % 16 or w % 16:
            # four stride-2 units: every one of them needs an even input side (Net3 always feeds 256 x 256)
            raise ValueError(f"e4s_b200: the RGI encoder needs both input sides to be multiples of 16, got {h}x{w}")
        if not x.is_cuda:
            raise RuntimeError("input must be a CUDA tensor")
        regions = LabelPyramid.from_mask(segmap)
        x = self._input_layer(x)
        taps = {}
        for i, unit in enumerate(self.body):
            x = self._unit(i, unit, x)
            if i in TAP_UNITS:
                taps[i] = x
        codes = []
        for i in TAP_UNITS:
            f = taps[i]
            codes.append(K.region_mean(f, regions.at(f.shape[1], f.shape[2]), regions.ncls)[0])
        out = torch.cat(codes, dim=2)
        bb, hh, ww, cc = x.shape
        return out, x.new_zeros((bb, cc, hh, ww))
