"""face-vid2vid's occlusion-aware SPADE generator: mirror of OcclusionAwareSPADEGenerator and SPADEDecoder in
src/pretrained/face_vid2vid/modules/generator.py (with the util.py blocks they are built from: SameBlock2d, DownBlock2d,
ResBlock3d, SPADE, SPADEResnetBlock).

The module tree, constructor arguments and state-dict keys are the reference's (386 entries on vox-256.yaml: 88 under
``dense_motion_network.``, 182 under ``decoder.``), so ``checkpoint['generator']`` loads with strict=True; conv_0, conv_1
and conv_s carry torch's spectral norm (``weight_orig``, ``weight_u``, ``weight_v``).  On vox-256.yaml's generator_params
and 256 x 256 sources, ``forward`` does not run those torch modules: the network executes on the e4s_b200 kernels,
inference only, every BatchNorm (eval-mode running statistics) folded into its convolution and every spectral norm
applied (weight_orig / (u . W v) with the stored u and v, as torch does in eval mode) in float64 -

* ``first`` (3x3, 3 -> 64, ReLU) on the fp32 RGB kernel (``e4s_conv3x3_rgb_act_f32``), the down blocks on the plain mode
  with the 2x2 average pass, ``second`` (1x1, 256 -> 512) on the pointwise mode with its weight rows permuted (row
  d 32 + c <- c 16 + d), so that its output is the [B, 64, 64, 16, 32] operand of the volumetric mode;
* ``resblocks_3d``: per block the BatchNorm + ReLU pre-activation through ``e4s_norm_residual_f32`` (zero PReLU slopes,
  the volume viewed as [B, 64, 64 16, 32]), conv1 with norm2 folded (+ ReLU) and conv2 with the block input added in its
  epilogue (``e4s_conv3d_residual_tcr_f32``);
* the dense-motion network (``DenseMotionNetwork``, unchanged), handed the NCDHW feature of its public forward through one
  permute copy;
* ``deform_input`` (trilinear grid_sample at the deformation) written as ``third``'s [B, 64, 64, 512] operand, channel
  d 32 + c, ``third``'s input channels permuted to match (``e4s_vid2vid_warp_f32``);
* ``third`` (3x3, 512 -> 256, LeakyReLU 0.01) on the plain mode, ``fourth`` (1x1) times the occlusion map on the pointwise
  mode (``e4s_conv1x1_factor_tcr_f32``);
* the decoder: ``fc`` on the plain mode; the SPADE blocks' ``mlp_shared`` (+ ReLU) as one GEMM per resolution over the
  64 x 64 seg map - the twelve of G_middle_0..5 at 64^2 (N = 1536), the three of up_0 at 128^2 and the three of up_1 at
  256^2, the last two reading the 64^2 map through the halo copy's nearest up-sampling (``e4s_conv3x3_zero_up_tcr_f32``;
  no up-sampled seg map is written); each SPADE's gamma / beta convolutions as one GEMM of interleaved columns over its
  128-channel slice, whose epilogue applies the modulation (and LeakyReLU 0.2 for norm_0 / norm_1) to the
  instance-normalised input (``e4s_spade_tcr_f32``) - up_0 and up_1 read their input at half resolution with its own
  statistics (``e4s_instnorm_stats_fixed_f32``), so nn.Upsample's output, the normalised tensors and the gamma / beta maps
  are never written; conv_0, conv_1 (+ the shortcut) and conv_s on the plain and pointwise modes, up_1.conv_1 with
  ``conv_img``'s LeakyReLU 0.2 in its epilogue;
* ``conv_img`` (3x3, 64 -> 3) + sigmoid on the RGB kernel, planar out.

Every output's sum order is fixed by the channel counts and image size alone: a pair's prediction is bit identical alone,
inside any batch and graph-replayed, and the forward makes no host synchronisation.  The jacobian, other sizes or
configurations, training mode and autograd raise NotImplementedError; so does OcclusionAwareGenerator (E4S builds only
the SPADE generator).
"""
import torch
from torch import nn
from torch.nn.utils import spectral_norm

from ... import kernels as K
from ...prepared import cached
from .dense_motion import DenseMotionNetwork
from .keypoint_detector import SIZE, DownBlock2d, _fold

VOX256 = dict(image_channel=3, feature_channel=32, num_kp=15, block_expansion=64, max_features=512, num_down_blocks=2,
              reshape_channel=32, reshape_depth=16, num_resblocks=6, estimate_occlusion_map=True,
              dense_motion_params=dict(block_expansion=32, max_features=1024, num_blocks=5, reshape_depth=16, compress=4),
              estimate_jacobian=False)


class SameBlock2d(nn.Module):
    def __init__(self, in_features, out_features, groups=1, kernel_size=3, padding=1, lrelu=False):
        super().__init__()
        self.conv = nn.Conv2d(in_channels=in_features, out_channels=out_features, kernel_size=kernel_size, padding=padding,
                              groups=groups)
        self.norm = nn.BatchNorm2d(out_features, affine=True)
        self.ac = nn.LeakyReLU() if lrelu else nn.ReLU()


class ResBlock3d(nn.Module):
    def __init__(self, in_features, kernel_size, padding):
        super().__init__()
        self.conv1 = nn.Conv3d(in_channels=in_features, out_channels=in_features, kernel_size=kernel_size, padding=padding)
        self.conv2 = nn.Conv3d(in_channels=in_features, out_channels=in_features, kernel_size=kernel_size, padding=padding)
        self.norm1 = nn.BatchNorm3d(in_features, affine=True)
        self.norm2 = nn.BatchNorm3d(in_features, affine=True)


class SPADE(nn.Module):
    def __init__(self, norm_nc, label_nc):
        super().__init__()
        self.param_free_norm = nn.InstanceNorm2d(norm_nc, affine=False)
        nhidden = 128
        self.mlp_shared = nn.Sequential(nn.Conv2d(label_nc, nhidden, kernel_size=3, padding=1), nn.ReLU())
        self.mlp_gamma = nn.Conv2d(nhidden, norm_nc, kernel_size=3, padding=1)
        self.mlp_beta = nn.Conv2d(nhidden, norm_nc, kernel_size=3, padding=1)


class SPADEResnetBlock(nn.Module):
    def __init__(self, fin, fout, norm_G, label_nc, use_se=False, dilation=1):
        super().__init__()
        self.learned_shortcut = (fin != fout)
        fmiddle = min(fin, fout)
        self.use_se = use_se
        self.conv_0 = nn.Conv2d(fin, fmiddle, kernel_size=3, padding=dilation, dilation=dilation)
        self.conv_1 = nn.Conv2d(fmiddle, fout, kernel_size=3, padding=dilation, dilation=dilation)
        if self.learned_shortcut:
            self.conv_s = nn.Conv2d(fin, fout, kernel_size=1, bias=False)
        if 'spectral' in norm_G:
            self.conv_0 = spectral_norm(self.conv_0)
            self.conv_1 = spectral_norm(self.conv_1)
            if self.learned_shortcut:
                self.conv_s = spectral_norm(self.conv_s)
        self.norm_0 = SPADE(fin, label_nc)
        self.norm_1 = SPADE(fmiddle, label_nc)
        if self.learned_shortcut:
            self.norm_s = SPADE(fin, label_nc)


class SPADEDecoder(nn.Module):
    def __init__(self):
        super().__init__()
        ic, oc, norm_G, label_nc = 256, 64, 'spadespectralinstance', 256
        self.fc = nn.Conv2d(ic, 2 * ic, 3, padding=1)
        for i in range(6):
            setattr(self, f"G_middle_{i}", SPADEResnetBlock(2 * ic, 2 * ic, norm_G, label_nc))
        self.up_0 = SPADEResnetBlock(2 * ic, ic, norm_G, label_nc)
        self.up_1 = SPADEResnetBlock(ic, oc, norm_G, label_nc)
        self.conv_img = nn.Conv2d(oc, 3, 3, padding=1)
        self.up = nn.Upsample(scale_factor=2)


class OcclusionAwareGenerator(nn.Module):
    """The reference's non-SPADE generator: not implemented (E4S builds the SPADE generator, driven_demo's gen="spade")."""

    def __init__(self, *args, **kwargs):
        raise NotImplementedError("e4s_b200 OcclusionAwareGenerator: only OcclusionAwareSPADEGenerator (gen='spade') is "
                                  "implemented")


def _sn_weight(conv: nn.Module) -> torch.Tensor:
    """Eval-mode spectral-norm weight of `conv`: weight_orig / (u . W v), W = weight_orig as [out, -1], with the stored u
    and v (no power iteration), in float64."""
    w = conv.weight_orig.detach().double()
    sigma = torch.dot(conv.weight_u.detach().double(), torch.mv(w.reshape(w.shape[0], -1), conv.weight_v.detach().double()))
    return w / sigma


def _planes(w: torch.Tensor) -> torch.Tensor:
    """[Cout, Cin, 3, 3] -> the plain mode's bf16 planes [2, 1, 9, Cout, Cin]."""
    w = w.float()
    return K.split_bf16(w.permute(2, 3, 0, 1).reshape(1, 9, w.shape[0], w.shape[1]).contiguous())


def _depth_major(c: int, d: int) -> torch.Tensor:
    """Index map of the channel order d C + c (depth-major, the volumetric operand) onto the reference's c D + d."""
    return torch.arange(c * d).view(c, d).t().reshape(-1)


class OcclusionAwareSPADEGenerator(nn.Module):
    """Re-enacted face: forward(source_image [B, 3, 256, 256] CUDA in [0, 1], kp_driving, kp_source ({'value':
    [B, 15, 3]})) -> {'mask': [B, 16, 16, 64, 64], 'occlusion_map': [B, 1, 64, 64], 'prediction': [B, 3, 256, 256]}."""

    def __init__(self, image_channel, feature_channel, num_kp, block_expansion, max_features, num_down_blocks, reshape_channel,
                 reshape_depth, num_resblocks, estimate_occlusion_map=False, dense_motion_params=None, estimate_jacobian=False):
        super().__init__()
        if dense_motion_params is not None:
            self.dense_motion_network = DenseMotionNetwork(num_kp=num_kp, feature_channel=feature_channel,
                                                           estimate_occlusion_map=estimate_occlusion_map, **dense_motion_params)
        else:
            self.dense_motion_network = None
        self.first = SameBlock2d(image_channel, block_expansion, kernel_size=(3, 3), padding=(1, 1))
        down_blocks = []
        for i in range(num_down_blocks):
            in_features = min(max_features, block_expansion * (2 ** i))
            out_features = min(max_features, block_expansion * (2 ** (i + 1)))
            down_blocks.append(DownBlock2d(in_features, out_features, kernel_size=(3, 3), padding=(1, 1)))
        self.down_blocks = nn.ModuleList(down_blocks)
        self.second = nn.Conv2d(in_channels=out_features, out_channels=max_features, kernel_size=1, stride=1)
        self.reshape_channel = reshape_channel
        self.reshape_depth = reshape_depth
        self.resblocks_3d = torch.nn.Sequential()
        for i in range(num_resblocks):
            self.resblocks_3d.add_module('3dr' + str(i), ResBlock3d(reshape_channel, kernel_size=3, padding=1))
        out_features = block_expansion * (2 ** (num_down_blocks))
        self.third = SameBlock2d(max_features, out_features, kernel_size=(3, 3), padding=(1, 1), lrelu=True)
        self.fourth = nn.Conv2d(in_channels=out_features, out_channels=out_features, kernel_size=1, stride=1)
        self.estimate_occlusion_map = estimate_occlusion_map
        self.image_channel = image_channel
        self.decoder = SPADEDecoder()
        self._config = dict(image_channel=image_channel, feature_channel=feature_channel, num_kp=num_kp,
                            block_expansion=block_expansion, max_features=max_features, num_down_blocks=num_down_blocks,
                            reshape_channel=reshape_channel, reshape_depth=reshape_depth, num_resblocks=num_resblocks,
                            estimate_occlusion_map=estimate_occlusion_map, dense_motion_params=dense_motion_params,
                            estimate_jacobian=estimate_jacobian)

    def _supported(self) -> bool:
        return self._config == VOX256

    # ------------------------------------------------------------------------------------------ weights
    def _prepared(self, device) -> dict:
        """Folded kernel operands on `device`, rebuilt when any parameter or buffer changes (pointer or version)."""
        return cached(self, "prepared", (*self.parameters(), *self.buffers()), device, lambda: self._build_prepared(device))

    def _build_prepared(self, device) -> dict:
        dev = lambda t: t.contiguous().to(device)  # noqa: E731
        wf, bf = _fold(self.first.conv, self.first.norm)
        down = []
        for blk in self.down_blocks:
            w, b = _fold(blk.conv, blk.norm)
            down.append((dev(_planes(w)), dev(b)))
        perm = _depth_major(self.reshape_channel, self.reshape_depth)
        w2 = self.second.weight.detach().float().reshape(self.second.out_channels, -1)[perm]
        res3d = []
        for blk in self.resblocks_3d:
            n1 = blk.norm1
            s = n1.weight.detach().double() / torch.sqrt(n1.running_var.detach().double() + n1.eps)
            t = n1.bias.detach().double() - n1.running_mean.detach().double() * s
            w1, b1 = _fold(blk.conv1, blk.norm2)
            res3d.append(dict(scale=dev(s.float()), shift=dev(t.float()), conv1=(dev(K.conv3d_planes(w1)), dev(b1)),
                              conv2=(dev(K.conv3d_planes(blk.conv2.weight.detach())), dev(blk.conv2.bias.detach().float()))))
        w3, b3 = _fold(self.third.conv, self.third.norm)
        dec = self.decoder

        def spade(norm):
            bias = torch.stack([norm.mlp_gamma.bias.detach().float(), norm.mlp_beta.bias.detach().float()], 1).reshape(-1)
            return dev(K.spade_planes(norm.mlp_gamma.weight.detach(), norm.mlp_beta.weight.detach())), dev(bias)

        def shared(norms):
            w = torch.cat([n.mlp_shared[0].weight.detach().float() for n in norms])
            return dev(_planes(w)), dev(torch.cat([n.mlp_shared[0].bias.detach().float() for n in norms]))

        def block(blk):
            d = dict(norm_0=spade(blk.norm_0), norm_1=spade(blk.norm_1),
                     conv_0=(dev(_planes(_sn_weight(blk.conv_0))), dev(blk.conv_0.bias.detach().float())),
                     conv_1=(dev(_planes(_sn_weight(blk.conv_1))), dev(blk.conv_1.bias.detach().float())))
            if blk.learned_shortcut:
                ws = _sn_weight(blk.conv_s).float()
                d["norm_s"] = spade(blk.norm_s)
                d["conv_s"] = dev(K.split_bf16(ws.reshape(ws.shape[0], ws.shape[1])))
            return d

        mids = [getattr(dec, f"G_middle_{i}") for i in range(6)]
        P = dict(first=(dev(wf), dev(bf)), down=down,
                 second=(dev(K.split_bf16(w2)), dev(self.second.bias.detach().float()[perm])), res3d=res3d,
                 slopes=torch.zeros(self.reshape_channel, device=device),
                 third=(dev(_planes(w3[:, perm])), dev(b3)),
                 fourth=(dev(K.split_bf16(self.fourth.weight.detach().float().reshape(self.fourth.out_channels, -1))),
                         dev(self.fourth.bias.detach().float())),
                 fc=(dev(_planes(dec.fc.weight.detach())), dev(dec.fc.bias.detach().float())),
                 shared_mid=shared([n for m in mids for n in (m.norm_0, m.norm_1)]),
                 shared_up=[shared([u.norm_0, u.norm_1, u.norm_s]) for u in (dec.up_0, dec.up_1)],
                 mids=[block(m) for m in mids], ups=[block(dec.up_0), block(dec.up_1)],
                 conv_img=(dev(dec.conv_img.weight.detach().float()), dev(dec.conv_img.bias.detach().float())))
        return P

    def _check(self, source_image, kp_driving, kp_source):
        if not self._supported():
            raise NotImplementedError("e4s_b200 OcclusionAwareSPADEGenerator: only vox-256.yaml's generator_params are "
                                      "implemented")
        if self.training:
            raise NotImplementedError("e4s_b200 OcclusionAwareSPADEGenerator: inference only (call .eval())")
        if torch.is_grad_enabled() and (source_image.requires_grad or any(p.requires_grad for p in self.parameters()) or
                                        any(kp['value'].requires_grad for kp in (kp_driving, kp_source))):
            raise NotImplementedError("e4s_b200 OcclusionAwareSPADEGenerator: no autograd; run under torch.no_grad()")
        x = source_image
        if not x.is_cuda or x.dim() != 4 or tuple(x.shape[1:]) != (3, SIZE, SIZE):
            raise NotImplementedError(f"e4s_b200 OcclusionAwareSPADEGenerator: CUDA source [B, 3, {SIZE}, {SIZE}] expected, "
                                      f"got {x.device} {tuple(x.shape)}")
        for name, kp in (("kp_driving", kp_driving), ("kp_source", kp_source)):
            if kp.get('jacobian') is not None:
                raise NotImplementedError(f"e4s_b200 OcclusionAwareSPADEGenerator: {name}['jacobian'] is not implemented")

    @staticmethod
    def _spade_block(d: dict, x, actv, last: bool):
        """One SPADEResnetBlock from its input x (pixel-major; at half the output resolution when x_half) and its
        mlp_shared outputs actv (the 128-channel slices norm_0, norm_1 (, norm_s))."""
        scale, shift = K.instnorm_stats(x)
        shortcut = x
        if "norm_s" in d:
            shortcut = K.conv1x1_tc(K.spade_tc(actv[..., 256:384], *d["norm_s"], x, scale, shift), d["conv_s"])
        h = K.spade_tc(actv[..., :128], *d["norm_0"], x, scale, shift, 0.2)
        dx = K.conv3x3_zero_tc(h, *d["conv_0"])
        h = K.spade_tc(actv[..., 128:256], *d["norm_1"], dx, *K.instnorm_stats(dx), 0.2)
        return K.conv3x3_zero_tc(h, *d["conv_1"], r0=shortcut, lrelu=0.2 if last else 1.0)

    def forward(self, source_image, kp_driving, kp_source):
        self._check(source_image, kp_driving, kp_source)
        P = self._prepared(source_image.device)
        bs = source_image.shape[0]
        x = K.conv3x3_rgb_act(source_image.float().contiguous(), *P["first"])
        for w, b in P["down"]:
            x = K.avgpool2(K.conv3x3_zero_tc(x, w, b, lrelu=0.0))
        f = K.conv1x1_tc(x, *P["second"])
        _, h, w, _ = f.shape
        c, d = self.reshape_channel, self.reshape_depth
        vol = f.view(bs, h, w, d, c)
        for blk in P["res3d"]:
            a = K.norm_residual(vol.view(bs, h, w * d, c), blk["scale"].expand(bs, c).contiguous(),
                                blk["shift"].expand(bs, c).contiguous(), 1.0, prelu=P["slopes"])
            a = K.conv3d_tc(a.view(bs, h, w, d, c), *blk["conv1"], relu=True)
            vol = K.conv3d_residual_tc(a, *blk["conv2"], residual=vol)
        dense_motion = self.dense_motion_network(feature=vol.permute(0, 4, 3, 1, 2).contiguous(), kp_driving=kp_driving,
                                                 kp_source=kp_source)
        occlusion_map = dense_motion['occlusion_map']
        out = K.conv3x3_zero_tc(K.vid2vid_warp(vol, dense_motion['deformation']), *P["third"], lrelu=0.01)
        seg = K.conv1x1_factor_tc(out, *P["fourth"], occlusion_map)
        x = K.conv3x3_zero_tc(seg, *P["fc"])
        actv = K.conv3x3_zero_tc(seg, *P["shared_mid"], lrelu=0.0)
        for i, d in enumerate(P["mids"]):
            x = self._spade_block(d, x, actv[..., 256 * i:256 * (i + 1)], False)
        for j, d in enumerate(P["ups"]):
            actv = K.conv3x3_zero_up_tc(seg, *P["shared_up"][j], up=2 << j, lrelu=0.0)
            x = self._spade_block(d, x, actv, j == 1)
        return {'mask': dense_motion['mask'], 'occlusion_map': occlusion_map,
                'prediction': K.conv3x3_rgb_act(x, *P["conv_img"])}
