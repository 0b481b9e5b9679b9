"""face-vid2vid's dense-motion network: mirror of DenseMotionNetwork in src/pretrained/face_vid2vid/modules/dense_motion.py
(with the util.py blocks it is built from: Hourglass, Encoder, Decoder, DownBlock3d, UpBlock3d).

The module tree, constructor arguments and state-dict keys are the reference's (88 entries on vox-256.yaml), so the
generator checkpoint's ``dense_motion_network.*`` entries, with that prefix stripped, load with strict=True.  On
vox-256.yaml's dense_motion_params and a [B, 32, 16, 64, 64] feature, ``forward`` does not run those torch modules: the
network executes on the e4s_b200 kernels, inference only, every BatchNorm (eval-mode running statistics) folded into its
convolution in float64 -

* compress (1x1x1, 32 -> 4) + BatchNorm + ReLU, one float4 per voxel: ``e4s_vid2vid_compress_f32``;
* the 16 sparse motions (the identity grid, then grid - kp_driving + kp_source), F.grid_sample of the compressed volume
  at them (trilinear, zero padding, align_corners=False) and the heatmap differences, as the hourglass's 80 input
  channels (5 k + j) and 16 zeros, written into their slice of the level-0 concatenation: ``e4s_vid2vid_motion_input_f32``;
* the hourglass on the volumetric mode (``e4s_conv3d_pitched_tcr_f32``) over [B, H, W, D, C] buffers: every skip
  concatenation [up-block output | skip] is one buffer whose producers write their own channel range of it (down block:
  convolution + ReLU, then AvgPool3d((1, 2, 2)) into the next level's skip slice, ``e4s_avgpool2_vox_f32``; up block:
  (1, 2, 2) nearest up-sampling, convolution + ReLU into the level's first slice).  down0 reads 96 channels and the
  decoder's last convolution 128 in and out, the padding zero weights;
* ``mask`` (7x7x7, 112 -> 16) and ``occlusion`` (7x7 over the 112 x 16 channels c 16 + d) as one 7x7 GEMM per depth slice
  with N = 128 columns, the (dz, o) mask weights and one occlusion column per depth (``e4s_conv7x7_slices_tcr_f32``),
  then the depth sums, the softmax, the deformation and the sigmoid (``e4s_vid2vid_motion_combine_f32``).

Every output's sum order is fixed by the channel counts alone: a pair's outputs are bit identical alone, inside any
batch and graph-replayed, and the forward makes no host synchronisation.  The jacobian, other sizes or configurations,
training mode and autograd raise NotImplementedError.
"""
import torch
import torch.nn.functional as F
from torch import nn

from ... import kernels as K
from ...prepared import cached
from .keypoint_detector import UpBlock3d, _fold

FEATURE = (32, 16, 64, 64)                # (C, D, H, W) of the generator's 3D feature on vox-256.yaml
IN_PAD, OUT_PAD = 96, 128                 # hourglass input 80 -> 96 channels, decoder output 112 -> 128


class DownBlock3d(nn.Module):
    def __init__(self, in_features, out_features, kernel_size=3, padding=1, groups=1):
        super().__init__()
        self.conv = nn.Conv3d(in_features, out_features, kernel_size=kernel_size, padding=padding, groups=groups)
        self.norm = nn.BatchNorm3d(out_features, affine=True)
        self.pool = nn.AvgPool3d(kernel_size=(1, 2, 2))


class Encoder(nn.Module):
    def __init__(self, block_expansion, in_features, num_blocks=3, max_features=256):
        super().__init__()
        self.down_blocks = nn.ModuleList([
            DownBlock3d(in_features if i == 0 else min(max_features, block_expansion * (2 ** i)),
                        min(max_features, block_expansion * (2 ** (i + 1))), kernel_size=3, padding=1)
            for i in range(num_blocks)])


class Decoder(nn.Module):
    def __init__(self, block_expansion, in_features, num_blocks=3, max_features=256):
        super().__init__()
        up_blocks = []
        for i in range(num_blocks)[::-1]:
            in_filters = (1 if i == num_blocks - 1 else 2) * min(max_features, block_expansion * (2 ** (i + 1)))
            out_filters = min(max_features, block_expansion * (2 ** i))
            up_blocks.append(UpBlock3d(in_filters, out_filters, kernel_size=3, padding=1))
        self.up_blocks = nn.ModuleList(up_blocks)
        self.out_filters = block_expansion + in_features
        self.conv = nn.Conv3d(in_channels=self.out_filters, out_channels=self.out_filters, kernel_size=3, padding=1)
        self.norm = nn.BatchNorm3d(self.out_filters, affine=True)


class Hourglass(nn.Module):
    def __init__(self, block_expansion, in_features, num_blocks=3, max_features=256):
        super().__init__()
        self.encoder = Encoder(block_expansion, in_features, num_blocks, max_features)
        self.decoder = Decoder(block_expansion, in_features, num_blocks, max_features)
        self.out_filters = self.decoder.out_filters


class DenseMotionNetwork(nn.Module):
    """Dense motion from the sparse keypoint motions: forward(feature [B, 32, 16, 64, 64] CUDA, kp_driving, kp_source
    ({'value': [B, 15, 3]})) -> {'mask': [B, 16, 16, 64, 64], 'deformation': [B, 16, 64, 64, 3], 'occlusion_map':
    [B, 1, 64, 64]}."""

    def __init__(self, block_expansion, num_blocks, max_features, num_kp, feature_channel, reshape_depth, compress,
                 estimate_occlusion_map=False):
        super().__init__()
        self.hourglass = Hourglass(block_expansion=block_expansion, in_features=(num_kp + 1) * (compress + 1),
                                   max_features=max_features, num_blocks=num_blocks)
        self.mask = nn.Conv3d(self.hourglass.out_filters, num_kp + 1, kernel_size=7, padding=3)
        self.compress = nn.Conv3d(feature_channel, compress, kernel_size=1)
        self.norm = nn.BatchNorm3d(compress, affine=True)
        if estimate_occlusion_map:
            self.occlusion = nn.Conv2d(self.hourglass.out_filters * reshape_depth, 1, kernel_size=7, padding=3)
        else:
            self.occlusion = None
        self.num_kp = num_kp
        self._config = dict(block_expansion=block_expansion, num_blocks=num_blocks, max_features=max_features, num_kp=num_kp,
                            feature_channel=feature_channel, reshape_depth=reshape_depth, compress=compress,
                            estimate_occlusion_map=estimate_occlusion_map)

    def _supported(self) -> bool:
        return self._config == dict(block_expansion=32, num_blocks=5, max_features=1024, num_kp=15, feature_channel=32,
                                    reshape_depth=16, compress=4, estimate_occlusion_map=True)

    # ------------------------------------------------------------------------------------------ weights
    def _prepared(self, device) -> dict:
        """Folded kernel operands on `device`, rebuilt when any parameter or buffer changes (pointer or version)."""
        return cached(self, "prepared", (*self.parameters(), *self.buffers()), device, lambda: self._build_prepared(device))

    def _build_prepared(self, device) -> dict:
        wc, bc = _fold(self.compress, self.norm)
        down = []
        for blk in self.hourglass.encoder.down_blocks:
            w, b = _fold(blk.conv, blk.norm)
            if w.shape[1] % 32:                                        # down0: 80 input channels -> 96
                w = F.pad(w, (0, 0, 0, 0, 0, 0, 0, IN_PAD - w.shape[1]))
            down.append((K.conv3d_planes(w).to(device), b.to(device)))
        dec = self.hourglass.decoder
        up = []
        for blk in dec.up_blocks:
            w, b = _fold(blk.conv, blk.norm)
            up.append((K.conv3d_planes(w).to(device), b.to(device)))
        w, b = _fold(dec.conv, dec.norm)
        nf = dec.out_filters
        w = F.pad(w, (0, 0, 0, 0, 0, 0, 0, OUT_PAD - nf, 0, OUT_PAD - nf))
        b = F.pad(b, (0, OUT_PAD - nf))
        P = dict(compress=torch.cat([wc.reshape(-1), bc]).contiguous().to(device), down=down, up=up,
                 last=(K.conv3d_planes(w).to(device), b.contiguous().to(device)),
                 gemm=K.split_bf16(gemm_weights(self.mask.weight.detach().float(),
                                                self.occlusion.weight.detach().float())).to(device),
                 mask_bias=self.mask.bias.detach().float().contiguous().to(device),
                 occ_bias=self.occlusion.bias.detach().float().contiguous().to(device))
        return P

    def _check(self, feature, kp_driving, kp_source):
        if not self._supported():
            raise NotImplementedError("e4s_b200 DenseMotionNetwork: only vox-256.yaml's dense_motion_params are implemented")
        if self.training:
            raise NotImplementedError("e4s_b200 DenseMotionNetwork: inference only (call .eval())")
        if torch.is_grad_enabled() and (feature.requires_grad or any(p.requires_grad for p in self.parameters()) or
                                        any(kp['value'].requires_grad for kp in (kp_driving, kp_source))):
            raise NotImplementedError("e4s_b200 DenseMotionNetwork: no autograd; run under torch.no_grad()")
        if not feature.is_cuda or feature.dim() != 5 or tuple(feature.shape[1:]) != FEATURE:
            raise NotImplementedError(f"e4s_b200 DenseMotionNetwork: CUDA feature [B, {', '.join(map(str, FEATURE))}] "
                                      f"expected, got {feature.device} {tuple(feature.shape)}")
        for name, kp in (("kp_driving", kp_driving), ("kp_source", kp_source)):
            if kp.get('jacobian') is not None:
                raise NotImplementedError(f"e4s_b200 DenseMotionNetwork: {name}['jacobian'] is not implemented")
            v = kp['value']
            if v.device != feature.device or tuple(v.shape) != (feature.shape[0], self.num_kp, 3):
                raise NotImplementedError(f"e4s_b200 DenseMotionNetwork: {name}['value'] [B, {self.num_kp}, 3] on "
                                          f"{feature.device} expected, got {v.device} {tuple(v.shape)}")

    def forward(self, feature, kp_driving, kp_source):
        self._check(feature, kp_driving, kp_source)
        P = self._prepared(feature.device)
        kd, ks = kp_driving['value'].float().contiguous(), kp_source['value'].float().contiguous()
        feature = feature.float().contiguous()
        bs, _, d, h, w = feature.shape
        comp = K.vid2vid_compress(feature, P["compress"])
        # level l (resolution 64 / 2^l): [up-block output | skip]; level 0's skip is the 96-channel hourglass input
        ups = [blk.conv.out_channels for blk in self.hourglass.decoder.up_blocks][::-1]       # 32, 64, .. 512
        skips = [IN_PAD] + [blk.conv.out_channels for blk in self.hourglass.encoder.down_blocks][:-1]
        dev = feature.device
        levels = [torch.empty((bs, h >> i, w >> i, d, ups[i] + skips[i]), device=dev, dtype=torch.float32)
                  for i in range(len(ups))]
        K.vid2vid_motion_input(comp, kd, ks, levels[0][..., ups[0]:])
        x = None
        for i, (wt, b) in enumerate(P["down"]):
            y = K.conv3d_pitched_tc(levels[i][..., ups[i]:], wt, b, relu=True)
            x = K.avgpool2_vox(y, levels[i + 1][..., ups[i + 1]:] if i + 1 < len(levels) else None)
        for j, (wt, b) in enumerate(P["up"]):
            i = len(levels) - 1 - j
            K.conv3d_pitched_tc(x, wt, b, out=levels[i][..., :ups[i]], up=True, relu=True)
            x = levels[i]
        pred = K.conv3d_pitched_tc(x, *P["last"], relu=True)
        mask, deformation, occlusion = K.vid2vid_motion_combine(K.conv7x7_slices_tc(pred, P["gemm"]), P["mask_bias"],
                                                                P["occ_bias"], kd, ks)
        return {'mask': mask, 'deformation': deformation, 'occlusion_map': occlusion}


def gemm_weights(wm: torch.Tensor, wo: torch.Tensor) -> torch.Tensor:
    """mask weight [16, C, 7, 7, 7] and occlusion weight [1, C D, 7, 7] (input channel c D + d) -> the per-slice GEMM's
    [49, 128, 128] (tap 7 ky + kx, column, channel): columns 16 dz + o the mask weights of kernel depth dz, columns
    7 16 + d the occlusion weights of input depth d; channels past C zero."""
    nk, c = wm.shape[:2]
    d = wo.shape[1] // c
    m = wm.permute(3, 4, 2, 0, 1).reshape(49, 7 * nk, c)
    o = wo.reshape(c, d, 7, 7).permute(2, 3, 1, 0).reshape(49, d, c)
    return F.pad(torch.cat([m, o], 1), (0, OUT_PAD - c)).contiguous()
