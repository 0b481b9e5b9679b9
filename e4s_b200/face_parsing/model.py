"""BiSeNet face parser: mirror of src/pretrained/face_parsing/model.py (BiSeNet, ContextPath, FeatureFusionModule, ...).

The module tree, constructor arguments and parameter / buffer names are the reference's, so ``79999_iter.pth`` loads.
``BiSeNet.forward`` does not run those torch modules: the network executes on the e4s_b200 kernels, eval mode only -

* BatchNorm folded into every convolution's weights and bias (in float64, once per parameter version);
* the stem (7x7 / 2 convolution + ReLU + 3x3 / 2 max-pool) in one kernel (``e4s_parser_stem_f32``);
* every other convolution on the tensor-core kernel with a bias / residual / ReLU epilogue (``e4s_conv3x3_bias_tcr_f32``):
  a stride-2 3x3 convolution as four taps over the space-to-depth repack of its input, a 1x1 convolution as the centre
  tap, the 1x1 / 2 shortcut as the centre tap over the same repack with weights on the even-pixel channels only;
* the attention vectors as channel means (``e4s_channel_mean_f32``) and small GEMMs (``e4s_linear_f32``), then applied
  for free as the per-(sample, channel) operand affine of the NEXT convolution: ``ARM32(x) + avg`` is
  ``conv * atten + avg`` and the FFM's ``f * atten + f`` is ``f * (1 + atten)``; nearest up-sampling commutes with it;
* the FFM's ``cat(feat8, feat_cp8)`` 1x1 convolution as two 1x1 convolutions, the second adding the first as its residual;
* each head's 1x1 classifier, bilinear (align_corners) up-sampling and argmax in one kernel (``e4s_parse_head_u8``).

Torch glue is limited to the context path's data movement on maps of at most 32 x 32 pixels: the nearest 2x up-sampling of
the two attention sums and the ARM16 sum ``feat16 * atten16 + feat32_up`` (DESIGN.md section 1).
"""
import itertools

import torch
import torch.nn as nn

from .resnet import Resnet18
from .. import kernels as K
from ..encoders.psp_encoders import TAP_CENTRE, TAPS_S2D, _conv_planes, _conv_planes_s2d

seg_mean = torch.tensor([[0.485, 0.456, 0.406]], dtype=torch.float32).reshape(1, 3, 1, 1)
seg_std = torch.tensor([[0.229, 0.224, 0.225]], dtype=torch.float32).reshape(1, 3, 1, 1)
seg_criterion = nn.CrossEntropyLoss()


class ConvBNReLU(nn.Module):
    def __init__(self, in_chan, out_chan, ks=3, stride=1, padding=1, *args, **kwargs):
        super().__init__()
        self.conv = nn.Conv2d(in_chan, out_chan, kernel_size=ks, stride=stride, padding=padding, bias=False)
        self.bn = nn.BatchNorm2d(out_chan)


class BiSeNetOutput(nn.Module):
    def __init__(self, in_chan, mid_chan, n_classes, *args, **kwargs):
        super().__init__()
        self.conv = ConvBNReLU(in_chan, mid_chan, ks=3, stride=1, padding=1)
        self.conv_out = nn.Conv2d(mid_chan, n_classes, kernel_size=1, bias=False)


class AttentionRefinementModule(nn.Module):
    def __init__(self, in_chan, out_chan, *args, **kwargs):
        super().__init__()
        self.conv = ConvBNReLU(in_chan, out_chan, ks=3, stride=1, padding=1)
        self.conv_atten = nn.Conv2d(out_chan, out_chan, kernel_size=1, bias=False)
        self.bn_atten = nn.BatchNorm2d(out_chan)
        self.sigmoid_atten = nn.Sigmoid()


class ContextPath(nn.Module):
    def __init__(self, *args, **kwargs):
        super().__init__()
        self.resnet = Resnet18()
        self.arm16 = AttentionRefinementModule(256, 128)
        self.arm32 = AttentionRefinementModule(512, 128)
        self.conv_head32 = ConvBNReLU(128, 128, ks=3, stride=1, padding=1)
        self.conv_head16 = ConvBNReLU(128, 128, ks=3, stride=1, padding=1)
        self.conv_avg = ConvBNReLU(512, 128, ks=1, stride=1, padding=0)


class FeatureFusionModule(nn.Module):
    def __init__(self, in_chan, out_chan, *args, **kwargs):
        super().__init__()
        self.convblk = ConvBNReLU(in_chan, out_chan, ks=1, stride=1, padding=0)
        self.conv1 = nn.Conv2d(out_chan, out_chan // 4, kernel_size=1, stride=1, padding=0, bias=False)
        self.conv2 = nn.Conv2d(out_chan // 4, out_chan, kernel_size=1, stride=1, padding=0, bias=False)
        self.relu = nn.ReLU(inplace=True)
        self.sigmoid = nn.Sigmoid()


def fold_bn(weight: torch.Tensor, bn: nn.BatchNorm2d):
    """(conv weight, eval-mode BatchNorm) -> (weight * g / sqrt(var + eps), beta - mean * g / sqrt(var + eps)), computed in
    float64 and rounded once to fp32."""
    s = bn.weight.detach().double() / torch.sqrt(bn.running_var.detach().double() + bn.eps)
    w = weight.detach().double() * s.reshape(-1, *([1] * (weight.dim() - 1)))
    b = bn.bias.detach().double() - bn.running_mean.detach().double() * s
    return w.float(), b.float().contiguous()


def _shortcut_planes(weight: torch.Tensor) -> torch.Tensor:
    """1x1 / 2 convolution [Cout, Cin, 1, 1] as the centre tap over the space-to-depth input: only the channels of the even
    pixels, (0, 0, c), carry weights."""
    cout, cin = weight.shape[:2]
    w4 = weight.new_zeros(cout, 4 * cin, 1, 1)
    w4[:, :cin] = weight
    return _conv_planes(w4)


def _up2(x_pm: torch.Tensor) -> torch.Tensor:
    """Nearest 2x up-sampling of a pixel-major map (the context path's F.interpolate(mode='nearest'))."""
    b, h, w, c = x_pm.shape
    return x_pm[:, :, None, :, None, :].expand(b, h, 2, w, 2, c).reshape(b, 2 * h, 2 * w, c)


class BiSeNet(nn.Module):
    def __init__(self, n_classes, *args, **kwargs):
        super().__init__()
        self.cp = ContextPath()
        self.ffm = FeatureFusionModule(256, 256)
        self.conv_out = BiSeNetOutput(256, 256, n_classes)
        self.conv_out16 = BiSeNetOutput(128, 64, n_classes)
        self.conv_out32 = BiSeNetOutput(128, 64, n_classes)
        self._prep = None

    # ------------------------------------------------------------------------------------------ weights
    def _prepared(self, device) -> dict:
        """Folded kernel operands on `device`, rebuilt when any parameter or buffer changes (pointer or version)."""
        key = (str(device),) + tuple((t.data_ptr(), t._version) for t in itertools.chain(self.parameters(), self.buffers()))
        if self._prep is not None and self._prep[0] == key:
            return self._prep[1]
        P = {}

        def conv(name, cbr: ConvBNReLU, s2d=False):
            w, b = fold_bn(cbr.conv.weight, cbr.bn)
            P[name] = (_conv_planes_s2d(w) if s2d else _conv_planes(w)).to(device), b.to(device)

        net = self.cp.resnet
        w, b = fold_bn(net.conv1.weight, net.bn1)
        P["stem"] = w.contiguous().to(device), b.to(device)
        for li in range(1, 5):
            for bi, blk in enumerate(getattr(net, f"layer{li}")):
                name = f"layer{li}.{bi}"
                stride = blk.conv1.stride[0]
                w1, b1 = fold_bn(blk.conv1.weight, blk.bn1)
                P[name + ".conv1"] = (_conv_planes_s2d(w1) if stride == 2 else _conv_planes(w1)).to(device), b1.to(device)
                w2, b2 = fold_bn(blk.conv2.weight, blk.bn2)
                P[name + ".conv2"] = _conv_planes(w2).to(device), b2.to(device)
                if blk.downsample is not None:
                    assert stride == 2, "Resnet18: only the first block of stages 2-4 has a shortcut convolution"
                    ws, bs = fold_bn(blk.downsample[0].weight, blk.downsample[1])
                    P[name + ".downsample"] = _shortcut_planes(ws).to(device), bs.to(device)
        cp = self.cp
        wa, ba = fold_bn(cp.conv_avg.conv.weight, cp.conv_avg.bn)
        P["conv_avg"] = wa.flatten(1).contiguous().to(device), ba.to(device)
        for arm in ("arm16", "arm32"):
            m = getattr(cp, arm)
            conv(arm, m.conv)
            wt, bt = fold_bn(m.conv_atten.weight, m.bn_atten)
            P[arm + ".atten"] = wt.flatten(1).contiguous().to(device), bt.to(device)
        conv("conv_head32", cp.conv_head32)
        conv("conv_head16", cp.conv_head16)
        wf, bf = fold_bn(self.ffm.convblk.conv.weight, self.ffm.convblk.bn)
        half = wf.shape[1] // 2                           # cat([feat8, feat_cp8]): the first half multiplies feat8
        P["ffm.sp"] = _conv_planes(wf[:, :half].contiguous()).to(device)
        P["ffm.cp"] = _conv_planes(wf[:, half:].contiguous()).to(device), bf.to(device)
        P["ffm.conv1"] = self.ffm.conv1.weight.detach().float().flatten(1).contiguous().to(device)
        P["ffm.conv2"] = self.ffm.conv2.weight.detach().float().flatten(1).contiguous().to(device)
        for head in ("conv_out", "conv_out16", "conv_out32"):
            m = getattr(self, head)
            conv(head, m.conv)
            P[head + ".cls"] = m.conv_out.weight.detach().float().flatten(1).contiguous().to(device)
        self._prep = (key, P)
        return P

    # ------------------------------------------------------------------------------------------ network
    def _check(self, x: torch.Tensor) -> None:
        if self.training:
            raise NotImplementedError("e4s_b200: the BiSeNet kernels are inference-only; call .eval() first")
        if torch.is_grad_enabled() and (x.requires_grad or any(p.requires_grad for p in self.parameters())):
            raise NotImplementedError("e4s_b200: the BiSeNet kernels are forward-only; wrap the call in torch.no_grad() or "
                                      "freeze the parameters")
        if not (x.is_cuda and x.dtype == torch.float32 and x.dim() == 4 and x.shape[1] == 3):
            raise ValueError(f"e4s_b200: BiSeNet takes a CUDA fp32 [B, 3, H, W] tensor, got {x.dtype} {tuple(x.shape)} "
                             f"on {x.device}")
        if x.shape[2] % 32 or x.shape[3] % 32:
            raise ValueError(f"e4s_b200: BiSeNet needs both input sides to be multiples of 32, got {x.shape[2]}x{x.shape[3]}")

    @staticmethod
    def _block(P, name, x):
        c1, c2, sc = P[name + ".conv1"], P[name + ".conv2"], P.get(name + ".downsample")
        if sc is None:
            r = K.conv3x3_bias_tc(x, *c1, relu=True)
            return K.conv3x3_bias_tc(r, *c2, residual=x, relu=True)
        x4 = K.space_to_depth(x)
        r = K.conv3x3_bias_tc(x4, *c1, relu=True, tap_mask=TAPS_S2D)
        s = K.conv3x3_bias_tc(x4, *sc, tap_mask=TAP_CENTRE)
        return K.conv3x3_bias_tc(r, *c2, residual=s, relu=True)

    @staticmethod
    def _atten(P, name, feat):
        """sigmoid(BN(conv1x1(mean(feat)))) [B, C] of an AttentionRefinementModule."""
        return torch.sigmoid(K.linear(K.channel_mean(feat), *P[name + ".atten"]))

    def _features(self, x):
        """Normalised planar x [B, 3, H, W] -> (FFM output [B, H/8, W/8, 256], its operand scale 1 + atten [B, 256],
        feat_cp8 [B, H/8, W/8, 128], feat_cp16 [B, H/16, W/16, 128]), pixel-major."""
        P = self._prepared(x.device)
        f = K.parser_stem(x.contiguous(), *P["stem"])
        feats = []
        for li in range(1, 5):
            for bi in range(2):
                f = self._block(P, f"layer{li}.{bi}", f)
            feats.append(f)
        feat8, feat16, feat32 = feats[1:]
        avg = K.linear(K.channel_mean(feat32), *P["conv_avg"], act_slope=0.0)
        f32 = K.conv3x3_bias_tc(feat32, *P["arm32"], relu=True)
        feat32_up = K.conv3x3_bias_tc(_up2(f32), *P["conv_head32"], relu=True, scale=self._atten(P, "arm32", f32), shift=avg)
        f16 = K.conv3x3_bias_tc(feat16, *P["arm16"], relu=True)
        s16 = torch.addcmul(feat32_up, f16, self._atten(P, "arm16", f16)[:, None, None, :])
        feat_cp8 = K.conv3x3_bias_tc(_up2(s16), *P["conv_head16"], relu=True)
        y8 = K.conv3x3_bias_tc(feat8, P["ffm.sp"], tap_mask=TAP_CENTRE)
        fuse = K.conv3x3_bias_tc(feat_cp8, *P["ffm.cp"], residual=y8, relu=True, tap_mask=TAP_CENTRE)
        att = torch.sigmoid(K.linear(K.linear(K.channel_mean(fuse), P["ffm.conv1"], act_slope=0.0), P["ffm.conv2"]))
        return fuse, 1.0 + att, feat_cp8, feat32_up

    def _head(self, P, name, feat, scale, out_hw, lut=None, logits=False):
        r = K.conv3x3_bias_tc(feat, *P[name], relu=True, scale=scale)
        return K.parse_head(r, P[name + ".cls"], out_hw[0], out_hw[1], lut=lut, labels=not logits, logits=logits)

    def forward(self, x):
        """Normalised x [B, 3, H, W] (CUDA fp32) -> the three heads' logits, each planar [B, n_classes, H, W]."""
        self._check(x)
        P = self._prepared(x.device)
        hw = tuple(x.shape[2:])
        fuse, scale, feat_cp8, feat_cp16 = self._features(x)
        out = self._head(P, "conv_out", fuse, scale, hw, logits=True)[1]
        out16 = self._head(P, "conv_out16", feat_cp8, None, hw, logits=True)[1]
        out32 = self._head(P, "conv_out32", feat_cp16, None, hw, logits=True)[1]
        return out, out16, out32

    def labels(self, x, lut=None):
        """Normalised x [B, 3, H, W] -> uint8 [B, H, W]: first-index argmax of the first head (through lut [256] uint8 on the
        device when given).  No logits are written and the auxiliary heads are not computed."""
        self._check(x)
        P = self._prepared(x.device)
        fuse, scale, _, _ = self._features(x)
        return self._head(P, "conv_out", fuse, scale, tuple(x.shape[2:]), lut=lut)[0]
