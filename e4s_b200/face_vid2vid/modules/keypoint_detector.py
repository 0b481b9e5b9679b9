"""face-vid2vid's canonical-keypoint detector and head-pose / expression estimator: mirror of KPDetector and HEEstimator in
src/pretrained/face_vid2vid/modules/keypoint_detector.py (with the util.py blocks they are built from: KPHourglass,
DownBlock2d, UpBlock3d, AntiAliasInterpolation2d, ResBottleneck).

The module tree, constructor arguments and state-dict keys are the reference's (75 entries on vox-256.yaml, BatchNorm
buffers and the anti-alias filter ``down.weight`` included), so ``checkpoint['kp_detector']`` loads with strict=True.  On
vox-256.yaml's kp_detector_params (estimate_jacobian False) at 256 x 256, ``forward`` does not run those torch modules:
the network executes on the e4s_b200 kernels, inference only, BatchNorm (eval-mode running statistics) folded into the
weights and bias in float64 -

* the anti-alias filter from the loaded buffer, to the pixel-major [B, 64, 64, 32] operand of down0 (channels 3..31 zero;
  down0's weights are zero-padded to 32 input channels): ``e4s_vid2vid_kp_prep_f32``;
* the down blocks' 3x3 convolutions (+ ReLU) on the plain mode with zero padding, each followed by the 2x2 average pass;
* the 1x1 convolution 1024 -> 16384 on the pointwise mode with its weight rows permuted (row d * 1024 + c <- c * 16 + d),
  so that its [B, 2, 2, 16384] output *is* the [B, H, W, D = 16, C = 1024] operand of the 3D blocks, without a copy;
* the five UpBlock3d ((1, 2, 2) nearest up-sampling, 3x3x3 convolution, ReLU) and the kp head (Cout 15 padded to 32 with
  zero weights) on the volumetric mode (``e4s_conv3d_tcr_f32``);
* softmax(logits / temperature) and the expectation of the coordinate grid on ``e4s_vid2vid_heatmap_f32``.

HEEstimator (402 state-dict entries, ``checkpoint['he_estimator']``) runs on existing entries, BatchNorm folded the same
way: the 7x7 / 2 stem + ReLU + 3x3 / 2 max-pool on ``e4s_parser_stem_f32``; every 1x1 on the pointwise mode (a
bottleneck's conv3 adds the identity or the stride-2 skip, read strided, before its ReLU); the 3x3s on the plain mode with
zero padding, at stride 2 over ``e4s_space_to_depth_f32``; ``e4s_channel_mean_f32``; the five heads as one 2048 -> 248
product on ``e4s_linear_f32`` (rows roll | pitch | yaw | t | exp, two zero rows), in launches of at most 32 faces, where
its K split does not depend on the row count.  As in the reference, 'yaw' is fc_roll's output and 'roll' fc_yaw's.

Every output's sum order is fixed by the channel counts alone: a face's keypoints and head pose are bit identical alone,
inside any batch and graph-replayed, and the forwards make no host synchronisation.  The jacobian, other sizes or
configurations, training mode and autograd raise NotImplementedError.
"""
import torch
import torch.nn.functional as F
from torch import nn

from ... import kernels as K
from ...encoders.psp_encoders import _conv_planes, _conv_planes_s2d
from ...prepared import cached

SIZE = 256


def _fold(conv: nn.Module, bn: nn.Module):
    """(conv with bias, eval-mode BatchNorm) -> (weight * g / sqrt(var + eps), (bias - mean) * g / sqrt(var + eps) + beta),
    computed in float64 and rounded once to fp32."""
    s = bn.weight.detach().double() / torch.sqrt(bn.running_var.detach().double() + bn.eps)
    w = conv.weight.detach().double() * s.reshape(-1, *([1] * (conv.weight.dim() - 1)))
    b = (conv.bias.detach().double() - bn.running_mean.detach().double()) * s + bn.bias.detach().double()
    return w.float(), b.float().contiguous()


def _check_input(name: str, module: nn.Module, x: torch.Tensor) -> None:
    if module.training:
        raise NotImplementedError(f"e4s_b200 {name}: inference only (call .eval())")
    if torch.is_grad_enabled() and (x.requires_grad or any(p.requires_grad for p in module.parameters())):
        raise NotImplementedError(f"e4s_b200 {name}: no autograd; run under torch.no_grad()")
    if not x.is_cuda or x.dim() != 4 or tuple(x.shape[1:]) != (3, SIZE, SIZE):
        raise NotImplementedError(f"e4s_b200 {name}: CUDA input [B, 3, {SIZE}, {SIZE}] expected, got {x.device} "
                                  f"{tuple(x.shape)}")


def make_coordinate_grid(spatial_size, type):
    """[D, H, W, 3] grid of (x, y, z), each 2 (i / (n - 1)) - 1 along W, H and D, of tensor type `type`."""
    d, h, w = spatial_size
    axis = lambda n: 2 * (torch.arange(n).type(type) / (n - 1)) - 1  # noqa: E731
    x, y, z = axis(w), axis(h), axis(d)
    return torch.stack([x.view(1, 1, w).expand(d, h, w), y.view(1, h, 1).expand(d, h, w), z.view(d, 1, 1).expand(d, h, w)], 3)


class DownBlock2d(nn.Module):
    def __init__(self, in_features, out_features, kernel_size=3, padding=1, groups=1):
        super().__init__()
        self.conv = nn.Conv2d(in_features, out_features, kernel_size=kernel_size, padding=padding, groups=groups)
        self.norm = nn.BatchNorm2d(out_features, affine=True)
        self.pool = nn.AvgPool2d(kernel_size=(2, 2))


class UpBlock3d(nn.Module):
    def __init__(self, in_features, out_features, kernel_size=3, padding=1, groups=1):
        super().__init__()
        self.conv = nn.Conv3d(in_features, out_features, kernel_size=kernel_size, padding=padding, groups=groups)
        self.norm = nn.BatchNorm3d(out_features, affine=True)


class KPHourglass(nn.Module):
    def __init__(self, block_expansion, in_features, reshape_features, reshape_depth, num_blocks=3, max_features=256):
        super().__init__()
        self.down_blocks = nn.Sequential()
        for i in range(num_blocks):
            self.down_blocks.add_module('down' + str(i), DownBlock2d(
                in_features if i == 0 else min(max_features, block_expansion * (2 ** i)),
                min(max_features, block_expansion * (2 ** (i + 1))), kernel_size=3, padding=1))
        in_filters = min(max_features, block_expansion * (2 ** num_blocks))
        self.conv = nn.Conv2d(in_channels=in_filters, out_channels=reshape_features, kernel_size=1)
        self.up_blocks = nn.Sequential()
        for i in range(num_blocks):
            in_filters = min(max_features, block_expansion * (2 ** (num_blocks - i)))
            out_filters = min(max_features, block_expansion * (2 ** (num_blocks - i - 1)))
            self.up_blocks.add_module('up' + str(i), UpBlock3d(in_filters, out_filters, kernel_size=3, padding=1))
        self.reshape_depth = reshape_depth
        self.out_filters = out_filters


class AntiAliasInterpolation2d(nn.Module):
    """Holds the band-limiting filter buffer ``weight`` [channels, 1, k, k]: a normalised Gaussian with sigma
    (1 / scale - 1) / 2 and k = 2 round(4 sigma) + 1 (13 at scale 1/4); the checkpoint's copy replaces it on load."""

    def __init__(self, channels, scale):
        super().__init__()
        sigma = (1 / scale - 1) / 2
        k = 2 * round(sigma * 4) + 1
        self.ka = k // 2
        self.kb = self.ka - 1 if k % 2 == 0 else self.ka
        r = torch.arange(k, dtype=torch.float32)
        g = torch.exp(-(r - (k - 1) / 2) ** 2 / (2 * sigma ** 2))
        ker = g.view(k, 1) * g.view(1, k)
        self.register_buffer('weight', (ker / ker.sum()).view(1, 1, k, k).repeat(channels, 1, 1, 1))
        self.groups = channels
        self.scale = scale
        self.int_inv_scale = int(1 / scale)


class KPDetector(nn.Module):
    """Detecting canonical keypoints: forward(x [B, 3, 256, 256] CUDA in [0, 1]) -> {'value': [B, num_kp, 3]}."""

    def __init__(self, block_expansion, feature_channel, num_kp, image_channel, max_features, reshape_channel, reshape_depth,
                 num_blocks, temperature, estimate_jacobian=False, scale_factor=1, single_jacobian_map=False):
        super().__init__()
        self.predictor = KPHourglass(block_expansion, in_features=image_channel, max_features=max_features,
                                     reshape_features=reshape_channel, reshape_depth=reshape_depth, num_blocks=num_blocks)
        self.kp = nn.Conv3d(in_channels=self.predictor.out_filters, out_channels=num_kp, kernel_size=3, padding=1)
        if estimate_jacobian:
            self.num_jacobian_maps = 1 if single_jacobian_map else num_kp
            self.jacobian = nn.Conv3d(in_channels=self.predictor.out_filters, out_channels=9 * self.num_jacobian_maps,
                                      kernel_size=3, padding=1)
            self.jacobian.weight.data.zero_()
            self.jacobian.bias.data.copy_(torch.tensor([1, 0, 0, 0, 1, 0, 0, 0, 1] * self.num_jacobian_maps, dtype=torch.float))
        else:
            self.jacobian = None
        self.temperature = temperature
        self.scale_factor = scale_factor
        if self.scale_factor != 1:
            self.down = AntiAliasInterpolation2d(image_channel, self.scale_factor)
        self._config = dict(block_expansion=block_expansion, num_kp=num_kp, image_channel=image_channel,
                            max_features=max_features, reshape_channel=reshape_channel, reshape_depth=reshape_depth,
                            num_blocks=num_blocks, scale_factor=scale_factor)

    def gaussian2kp(self, heatmap):
        shape = heatmap.shape
        heatmap = heatmap.unsqueeze(-1)
        grid = make_coordinate_grid(shape[2:], heatmap.type()).unsqueeze_(0).unsqueeze_(0)
        return {'value': (heatmap * grid).sum(dim=(2, 3, 4))}

    def _supported(self) -> bool:
        return self._config == dict(block_expansion=32, num_kp=15, image_channel=3, max_features=1024, reshape_channel=16384,
                                    reshape_depth=16, num_blocks=5, scale_factor=0.25) and self.jacobian is None

    # ------------------------------------------------------------------------------------------ weights
    def _prepared(self, device) -> dict:
        """Folded kernel operands on `device`, rebuilt when any parameter or buffer changes (pointer or version)."""
        return cached(self, "prepared", (*self.parameters(), *self.buffers()), device, lambda: self._build_prepared(device))

    def _build_prepared(self, device) -> dict:
        pr = self.predictor
        down = []
        for i, blk in enumerate(pr.down_blocks):
            w, b = _fold(blk.conv, blk.norm)
            if w.shape[1] % 32:                                       # down0: 3 input channels -> the prep's 32
                w = F.pad(w, (0, 0, 0, 0, 0, 32 - w.shape[1] % 32))
            down.append((K.split_bf16(w.permute(2, 3, 0, 1).reshape(1, 9, w.shape[0], w.shape[1]).contiguous()).to(device),
                         b.to(device)))
        c, d = pr.conv.out_channels // pr.reshape_depth, pr.reshape_depth
        perm = torch.arange(c * d).view(c, d).t().reshape(-1)          # row d * C + c <- c * D + d
        w1 = pr.conv.weight.detach().float().reshape(c * d, -1)[perm].contiguous()
        b1 = pr.conv.bias.detach().float()[perm].contiguous()
        up = []
        for blk in pr.up_blocks:
            w, b = _fold(blk.conv, blk.norm)
            up.append((K.conv3d_planes(w).to(device), b.to(device)))
        nkp = self.kp.out_channels
        wk = F.pad(self.kp.weight.detach().float(), (0, 0, 0, 0, 0, 0, 0, 0, 0, 32 - nkp))
        bk = F.pad(self.kp.bias.detach().float(), (0, 32 - nkp))
        prep = dict(filt=self.down.weight.detach().float().contiguous().to(device), down=down,
                    conv=(K.split_bf16(w1).to(device), b1.to(device)), up=up,
                    kp=(K.conv3d_planes(wk).to(device), bk.contiguous().to(device)))
        return prep

    def forward(self, x):
        if not self._supported():
            raise NotImplementedError("e4s_b200 KPDetector: only vox-256.yaml's kp_detector_params with estimate_jacobian "
                                      "False are implemented")
        _check_input("KPDetector", self, x)
        P = self._prepared(x.device)
        h = K.vid2vid_kp_prep(x.float().contiguous(), P["filt"])
        for w, b in P["down"]:
            h = K.avgpool2(K.conv3x3_zero_tc(h, w, b, lrelu=0.0))
        h = K.conv1x1_tc(h, *P["conv"])
        bsz, hh, ww, _ = h.shape
        h = h.view(bsz, hh, ww, self.predictor.reshape_depth, -1)
        for w, b in P["up"]:
            h = K.conv3d_tc(h, w, b, up=True, relu=True)
        logits = K.conv3d_tc(h, *P["kp"])
        return {'value': K.vid2vid_heatmap(logits, self.kp.out_channels, self.temperature)}


class ResBottleneck(nn.Module):
    def __init__(self, in_features, stride):
        super().__init__()
        mid = in_features // 4
        self.conv1 = nn.Conv2d(in_channels=in_features, out_channels=mid, kernel_size=1)
        self.conv2 = nn.Conv2d(in_channels=mid, out_channels=mid, kernel_size=3, padding=1, stride=stride)
        self.conv3 = nn.Conv2d(in_channels=mid, out_channels=in_features, kernel_size=1)
        self.norm1 = nn.BatchNorm2d(mid, affine=True)
        self.norm2 = nn.BatchNorm2d(mid, affine=True)
        self.norm3 = nn.BatchNorm2d(in_features, affine=True)
        self.stride = stride
        if self.stride != 1:
            self.skip = nn.Conv2d(in_channels=in_features, out_channels=in_features, kernel_size=1, stride=stride)
            self.norm4 = nn.BatchNorm2d(in_features, affine=True)


# HEEstimator's trunk after the stem: (name, kind) with kind "pw" (1x1 + BN + ReLU) or "res" (ResBottleneck / a Sequential
# of them)
_HE_TRUNK = ("conv2", "block1", "conv3", "block2", "block3", "conv4", "block4", "block5", "conv5", "block6", "block7")
HEAD_ROWS = 248                     # roll 66 | pitch 66 | yaw 66 | t 3 | exp 45, two zero rows (a multiple of 4)


class HEEstimator(nn.Module):
    """Estimating head pose and expression: forward(x [B, 3, 256, 256] CUDA in [0, 1]) -> {'yaw', 'pitch', 'roll':
    [B, num_bins] bin logits, 't': [B, 3], 'exp': [B, 3 num_kp]} (views of one [B, 248] head output)."""

    def __init__(self, block_expansion, feature_channel, num_kp, image_channel, max_features, num_bins=66,
                 estimate_jacobian=True):
        super().__init__()
        self.conv1 = nn.Conv2d(in_channels=image_channel, out_channels=block_expansion, kernel_size=7, padding=3, stride=2)
        self.norm1 = nn.BatchNorm2d(block_expansion, affine=True)
        self.maxpool = nn.MaxPool2d(kernel_size=3, stride=2, padding=1)
        self.conv2 = nn.Conv2d(in_channels=block_expansion, out_channels=256, kernel_size=1)
        self.norm2 = nn.BatchNorm2d(256, affine=True)
        self.block1 = nn.Sequential()
        for i in range(3):
            self.block1.add_module('b1_' + str(i), ResBottleneck(in_features=256, stride=1))
        self.conv3 = nn.Conv2d(in_channels=256, out_channels=512, kernel_size=1)
        self.norm3 = nn.BatchNorm2d(512, affine=True)
        self.block2 = ResBottleneck(in_features=512, stride=2)
        self.block3 = nn.Sequential()
        for i in range(3):
            self.block3.add_module('b3_' + str(i), ResBottleneck(in_features=512, stride=1))
        self.conv4 = nn.Conv2d(in_channels=512, out_channels=1024, kernel_size=1)
        self.norm4 = nn.BatchNorm2d(1024, affine=True)
        self.block4 = ResBottleneck(in_features=1024, stride=2)
        self.block5 = nn.Sequential()
        for i in range(5):
            self.block5.add_module('b5_' + str(i), ResBottleneck(in_features=1024, stride=1))
        self.conv5 = nn.Conv2d(in_channels=1024, out_channels=2048, kernel_size=1)
        self.norm5 = nn.BatchNorm2d(2048, affine=True)
        self.block6 = ResBottleneck(in_features=2048, stride=2)
        self.block7 = nn.Sequential()
        for i in range(2):
            self.block7.add_module('b7_' + str(i), ResBottleneck(in_features=2048, stride=1))
        self.fc_roll = nn.Linear(2048, num_bins)
        self.fc_pitch = nn.Linear(2048, num_bins)
        self.fc_yaw = nn.Linear(2048, num_bins)
        self.fc_t = nn.Linear(2048, 3)
        self.fc_exp = nn.Linear(2048, 3 * num_kp)
        self._config = dict(block_expansion=block_expansion, num_kp=num_kp, image_channel=image_channel, num_bins=num_bins)

    def _supported(self) -> bool:
        return self._config == dict(block_expansion=64, num_kp=15, image_channel=3, num_bins=66)

    def _prepared(self, device) -> dict:
        return cached(self, "prepared", (*self.parameters(), *self.buffers()), device, lambda: self._build_prepared(device))

    def _build_prepared(self, device) -> dict:
        def pw(conv, bn):
            w, b = _fold(conv, bn)
            return K.split_bf16(w.reshape(w.shape[0], w.shape[1]).contiguous()).to(device), b.to(device)

        def res(blk):
            w2, b2 = _fold(blk.conv2, blk.norm2)
            d = {"stride": blk.stride, "conv1": pw(blk.conv1, blk.norm1),
                 "conv2": ((_conv_planes_s2d(w2) if blk.stride == 2 else _conv_planes(w2)).to(device), b2.to(device)),
                 "conv3": pw(blk.conv3, blk.norm3)}
            if blk.stride != 1:
                d["skip"] = pw(blk.skip, blk.norm4)
            return d

        w7, b7 = _fold(self.conv1, self.norm1)
        trunk = []
        for name in _HE_TRUNK:
            m = getattr(self, name)
            if isinstance(m, nn.Conv2d):
                trunk.append(("pw", pw(m, getattr(self, "norm" + name[-1]))))
            else:
                for blk in (m if isinstance(m, nn.Sequential) else [m]):
                    trunk.append(("res", res(blk)))
        fcs = (self.fc_roll, self.fc_pitch, self.fc_yaw, self.fc_t, self.fc_exp)
        wh = torch.cat([f.weight.detach().float() for f in fcs], 0)
        bh = torch.cat([f.bias.detach().float() for f in fcs], 0)
        wh = torch.nn.functional.pad(wh, (0, 0, 0, HEAD_ROWS - wh.shape[0])).contiguous()
        bh = torch.nn.functional.pad(bh, (0, HEAD_ROWS - bh.shape[0])).contiguous()
        P = {"stem": (w7.contiguous().to(device), b7.to(device)), "trunk": trunk, "heads": (wh.to(device), bh.to(device))}
        return P

    @staticmethod
    def _bottleneck(d: dict, x: torch.Tensor) -> torch.Tensor:
        r = K.conv1x1_tc(x, *d["conv1"], lrelu=0.0)
        if d["stride"] == 2:
            r = K.conv3x3_zero_tc(K.space_to_depth(r), *d["conv2"], stride=2, lrelu=0.0)
        else:
            r = K.conv3x3_zero_tc(r, *d["conv2"], lrelu=0.0)
        idn = K.conv1x1_tc(x, *d["skip"], stride=2) if "skip" in d else x
        return K.conv1x1_tc(r, *d["conv3"], r0=idn, lrelu=0.0)

    def features(self, x: torch.Tensor) -> torch.Tensor:
        """The pooled 2048-channel features [B, 2048] the heads read."""
        P = self._prepared(x.device)
        f = K.parser_stem(x.float().contiguous(), *P["stem"])
        for kind, d in P["trunk"]:
            f = K.conv1x1_tc(f, *d, lrelu=0.0) if kind == "pw" else self._bottleneck(d, f)
        return K.channel_mean(f)

    def forward(self, x):
        if not self._supported():
            raise NotImplementedError("e4s_b200 HEEstimator: only vox-256.yaml's he_estimator_params are implemented")
        _check_input("HEEstimator", self, x)
        P = self._prepared(x.device)
        pooled = self.features(x)
        out = torch.empty((x.shape[0], HEAD_ROWS), device=x.device, dtype=torch.float32)
        for i in range(0, x.shape[0], 32):
            out[i:i + 32] = K.linear(pooled[i:i + 32], *P["heads"])
        nb = self.fc_roll.out_features
        return {'yaw': out[:, :nb], 'pitch': out[:, nb:2 * nb], 'roll': out[:, 2 * nb:3 * nb],
                't': out[:, 3 * nb:3 * nb + 3], 'exp': out[:, 3 * nb + 3:3 * nb + 3 + self.fc_exp.out_features]}
