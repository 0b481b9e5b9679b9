"""ESRGAN's RRDBNet: mirror of src/pretrained/gpen/sr_model/rrdbnet_arch.py (ResidualDenseBlock, RRDB, RRDBNet).

The module tree, constructor arguments and parameter names and shapes are the reference's, so a ``realesrnet_x4.pth``
``params_ema`` dict loads with strict=True.  ``RRDBNet.forward`` does not run those torch modules: at scale 4 the network
executes on the e4s_b200 kernels, forward only -

* every 3x3 convolution of the trunk and the up-sampling tail on the tensor-core kernel's plain mode
  (``e4s_conv3x3_dense_tcr_f32``) over pixel-major, pixel-pitched operands;
* a residual dense block in one [B, H, W, num_feat + 4 num_grow_ch] buffer: x at channel 0, x1 .. x4 after it; conv k reads
  the channel prefix of the buffer and writes its output behind it, so no ``torch.cat`` is made;
* conv5's ``x5 * 0.2 + x`` - and on a block's third residual dense block also the RRDB's ``out * 0.2 + x`` - in its epilogue,
  ``feat + conv_body(...)`` in conv_body's, each ``lrelu`` in the epilogue of the convolution it follows;
* ``F.interpolate(scale_factor=2, mode="nearest")`` inside conv_up1 / conv_up2's halo copy (the up-sampled tensors are never
  written);
* conv_first (3 -> num_feat, planar image in) and conv_last (num_feat -> 3, planar image out) on a small fp32 kernel of
  their own (``e4s_conv3x3_rgb_f32``; num_feat 32, the configuration RealESRNet uses).

Kernel-ready weights (bf16 hi / lo operand planes) are prepared once per parameter version.  Scales 1 and 2 (pixel-unshuffled
input) build the reference's module tree; their forward raises NotImplementedError (the face-swap pipeline uses scale 4).
"""
import itertools

import torch
from torch import nn

from ... import kernels as K
from ...encoders.psp_encoders import _conv_planes
from ...prepared import cached


class ResidualDenseBlock(nn.Module):
    """Residual Dense Block of ESRGAN (run by RRDBNet.forward)."""

    def __init__(self, num_feat=64, num_grow_ch=32):
        super(ResidualDenseBlock, self).__init__()
        self.conv1 = nn.Conv2d(num_feat, num_grow_ch, 3, 1, 1)
        self.conv2 = nn.Conv2d(num_feat + num_grow_ch, num_grow_ch, 3, 1, 1)
        self.conv3 = nn.Conv2d(num_feat + 2 * num_grow_ch, num_grow_ch, 3, 1, 1)
        self.conv4 = nn.Conv2d(num_feat + 3 * num_grow_ch, num_grow_ch, 3, 1, 1)
        self.conv5 = nn.Conv2d(num_feat + 4 * num_grow_ch, num_feat, 3, 1, 1)
        self.lrelu = nn.LeakyReLU(negative_slope=0.2, inplace=True)


class RRDB(nn.Module):
    """Residual in Residual Dense Block (run by RRDBNet.forward)."""

    def __init__(self, num_feat, num_grow_ch=32):
        super(RRDB, self).__init__()
        self.rdb1 = ResidualDenseBlock(num_feat, num_grow_ch)
        self.rdb2 = ResidualDenseBlock(num_feat, num_grow_ch)
        self.rdb3 = ResidualDenseBlock(num_feat, num_grow_ch)


class RRDBNet(nn.Module):
    def __init__(self, num_in_ch, num_out_ch, scale=4, num_feat=64, num_block=23, num_grow_ch=32):
        super(RRDBNet, self).__init__()
        self.scale = scale
        self.num_feat, self.num_grow_ch = num_feat, num_grow_ch
        self._out_ch = num_out_ch
        if scale == 2:
            num_in_ch = num_in_ch * 4
        elif scale == 1:
            num_in_ch = num_in_ch * 16
        self._in_ch = num_in_ch
        self.conv_first = nn.Conv2d(num_in_ch, num_feat, 3, 1, 1)
        self.body = nn.Sequential(*[RRDB(num_feat=num_feat, num_grow_ch=num_grow_ch) for _ in range(num_block)])
        self.conv_body = nn.Conv2d(num_feat, num_feat, 3, 1, 1)
        # upsample
        self.conv_up1 = nn.Conv2d(num_feat, num_feat, 3, 1, 1)
        self.conv_up2 = nn.Conv2d(num_feat, num_feat, 3, 1, 1)
        self.conv_hr = nn.Conv2d(num_feat, num_feat, 3, 1, 1)
        self.conv_last = nn.Conv2d(num_feat, num_out_ch, 3, 1, 1)
        self.lrelu = nn.LeakyReLU(negative_slope=0.2, inplace=True)

    # ------------------------------------------------------------------------------------------ weights
    def _prepared(self, device) -> dict:
        """Kernel operands on `device`, rebuilt when any parameter changes (pointer or version)."""
        return cached(self, "prepared", self.parameters(), device, lambda: self._build_prepared(device))

    def _build_prepared(self, device) -> dict:
        def planes(conv):
            return _conv_planes(conv.weight).to(device), conv.bias.detach().float().contiguous().to(device)

        def plain(conv):
            return conv.weight.detach().float().contiguous().to(device), conv.bias.detach().float().contiguous().to(device)

        P = {"conv_first": plain(self.conv_first), "conv_last": plain(self.conv_last)}
        for name in ("conv_body", "conv_up1", "conv_up2", "conv_hr"):
            P[name] = planes(getattr(self, name))
        P["body"] = [[[planes(getattr(rdb, f"conv{j}")) for j in range(1, 6)] for rdb in (blk.rdb1, blk.rdb2, blk.rdb3)]
                     for blk in self.body]
        return P

    # ------------------------------------------------------------------------------------------ network
    def _check(self, x: torch.Tensor) -> None:
        if self.scale != 4:
            raise NotImplementedError(f"e4s_b200: RRDBNet runs scale 4 only (pixel-unshuffled scale {self.scale} is not "
                                      "provided)")
        if self._in_ch != 3 or self._out_ch != 3 or self.num_feat != 32 or self.num_grow_ch % 32:
            raise NotImplementedError("e4s_b200: RRDBNet runs 3 -> 3 channels with num_feat 32 and num_grow_ch a multiple "
                                      "of 32 (RealESRNet's configuration)")
        if torch.is_grad_enabled() and (x.requires_grad or any(p.requires_grad for p in self.parameters())):
            raise NotImplementedError("e4s_b200: the RRDBNet kernels are forward-only; wrap the call in torch.no_grad() or "
                                      "freeze the parameters")
        if not (x.is_cuda and x.dtype == torch.float32 and x.dim() == 4 and x.shape[1] == 3):
            raise ValueError(f"e4s_b200: RRDBNet takes a CUDA fp32 [B, 3, H, W] tensor, got {x.dtype} {tuple(x.shape)} "
                             f"on {x.device}")

    def forward(self, x):
        """Planar x [B, 3, H, W] (CUDA fp32, any H and W) -> [B, 3, 4H, 4W].  No host synchronisation (graph-capturable)."""
        self._check(x)
        P = self._prepared(x.device)
        b, _, h, w = x.shape
        nf, gc = self.num_feat, self.num_grow_ch
        width = nf + 4 * gc

        def buffer():
            return torch.empty((b, h, w, width), device=x.device, dtype=torch.float32)

        # first: conv_first's output at channel 0 (the trunk's input, kept for the long skip), then the dense slots of the
        # first block's rdb1.  A block's output goes to channel 0 of bufs[0], its rdb2 / rdb3 run in bufs[1] / bufs[2].
        first, bufs = buffer(), [buffer() for _ in range(3)]
        K.conv3x3_rgb(x.contiguous(), *P["conv_first"], out=first[..., :nf])
        src = first
        for rdbs in P["body"]:
            ins = (src, bufs[1], bufs[2])
            for r, convs in enumerate(rdbs):
                buf = ins[r]
                for j in range(4):
                    c0 = nf + j * gc
                    K.conv3x3_dense_tc(buf[..., :c0], *convs[j], out=buf[..., c0:c0 + gc], lrelu=0.2)
                if r < 2:            # x5 * 0.2 + x
                    K.conv3x3_dense_tc(buf, *convs[4], out=ins[r + 1][..., :nf], alpha=0.2, r0=buf[..., :nf])
                else:                # (x5 * 0.2 + x) * 0.2 + (the block's input)
                    K.conv3x3_dense_tc(buf, *convs[4], out=bufs[0][..., :nf], alpha=0.2, r0=buf[..., :nf], beta=0.2,
                                       r1=src[..., :nf])
            src = bufs[0]
        trunk = K.conv3x3_dense_tc(src[..., :nf], *P["conv_body"], out=bufs[1][..., :nf], r0=first[..., :nf])
        feat = K.conv3x3_dense_tc(trunk, *P["conv_up1"], up=True, lrelu=0.2)
        del first, bufs, src, trunk
        feat = K.conv3x3_dense_tc(feat, *P["conv_up2"], up=True, lrelu=0.2)
        feat = K.conv3x3_dense_tc(feat, *P["conv_hr"], lrelu=0.2)
        return K.conv3x3_rgb(feat, *P["conv_last"])
