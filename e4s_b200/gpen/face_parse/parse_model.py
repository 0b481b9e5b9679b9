"""GPEN's face parser: mirror of src/pretrained/gpen/face_parse/parse_model.py (define_P, ParseNet).

The module tree, constructor arguments and state-dict keys are the reference's, so ``ParseNet-latest.pth`` loads with
strict=True.  ``ParseNet.forward`` does not run those torch modules: in FaceParse's configuration (512 x 512, min_feat_size 32,
base_ch 64, 19 classes, 10 body blocks, BatchNorm, LeakyReLU, ch_range [32, 256]) the network executes on the e4s_b200
kernels, forward only -

* every 3x3 convolution of the encoder blocks, the body and the decoder on the tensor-core kernel's plain mode with
  reflection padding (``e4s_conv3x3_reflect_tcr_f32``) over pixel-major operands, eval-mode BatchNorm folded into the
  weights and bias (in float64, rounded once), LeakyReLU(0.2) and the residual adds in the epilogue: conv2 of a block adds
  the block's identity, the last body block also the long skip ``feat + body(feat)``;
* a down block's stride-2 shortcut and conv2 as four taps over the space-to-depth repack of their input
  (``e4s_space_to_depth_f32``), the reflection padding then being row / column -1 replicating row / column 0;
* an up block's ``F.interpolate(scale_factor=2, mode='nearest')`` inside its shortcut's and conv1's halo copy (the up-sampled
  tensors are never written; reflection padding of the up-sampled grid is replicate padding);
* encoder.0 (3 -> 64, planar image in), out_img_conv (64 -> 3, planar image out) and out_mask_conv (64 -> 19) on fp32
  kernels of their own (``e4s_conv3x3_rgb_reflect_f32``, ``e4s_gpen_parse_head_u8``); the mask head can also give the
  MASK_COLORMAP value of the first-index argmax class per pixel without writing the logits (FaceParse.process_tensor).

Kernel-ready weights are prepared once per parameter version.  Other configurations build the reference's module tree; their
forward raises NotImplementedError.
"""
import numpy as np
import torch
from torch import nn

from ... import kernels as K
from ...encoders.psp_encoders import _conv_planes, _conv_planes_s2d
from ...face_parsing.model import fold_bn
from ...prepared import cached
from .blocks import ConvLayer, ResidualBlock

# the configuration FaceParse.load_model builds (face_parsing.py:34)
_RUN_CONFIG = dict(in_size=512, out_size=512, min_feat_size=32, base_ch=64, parsing_ch=19, res_depth=10, relu_type='leakyrelu',
                   norm_type='bn', ch_range=(32, 256))


def define_P(in_size=512, out_size=512, min_feat_size=32, relu_type='LeakyReLU', isTrain=False, weight_path=None):
    net = ParseNet(in_size, out_size, min_feat_size, 64, 19, norm_type='bn', relu_type=relu_type, ch_range=[32, 256])
    if not isTrain:
        net.eval()
    if weight_path is not None:
        net.load_state_dict(torch.load(weight_path))
    return net


class ParseNet(nn.Module):
    def __init__(self,
                 in_size=128,
                 out_size=128,
                 min_feat_size=32,
                 base_ch=64,
                 parsing_ch=19,
                 res_depth=10,
                 relu_type='prelu',
                 norm_type='bn',
                 ch_range=[32, 512],
                 ):
        super().__init__()
        self.res_depth = res_depth
        act_args = {'norm_type': norm_type, 'relu_type': relu_type}
        min_ch, max_ch = ch_range
        self._config = dict(in_size=in_size, out_size=out_size, min_feat_size=min_feat_size, base_ch=base_ch,
                            parsing_ch=parsing_ch, res_depth=res_depth, relu_type=relu_type.lower(), norm_type=norm_type,
                            ch_range=tuple(ch_range))

        ch_clip = lambda x: max(min_ch, min(x, max_ch))  # noqa: E731
        min_feat_size = min(in_size, min_feat_size)

        down_steps = int(np.log2(in_size // min_feat_size))
        up_steps = int(np.log2(out_size // min_feat_size))

        # =============== define encoder-body-decoder ====================
        self.encoder = []
        self.encoder.append(ConvLayer(3, base_ch, 3, 1))
        head_ch = base_ch
        for i in range(down_steps):
            cin, cout = ch_clip(head_ch), ch_clip(head_ch * 2)
            self.encoder.append(ResidualBlock(cin, cout, scale='down', **act_args))
            head_ch = head_ch * 2

        self.body = []
        for i in range(res_depth):
            self.body.append(ResidualBlock(ch_clip(head_ch), ch_clip(head_ch), **act_args))

        self.decoder = []
        for i in range(up_steps):
            cin, cout = ch_clip(head_ch), ch_clip(head_ch // 2)
            self.decoder.append(ResidualBlock(cin, cout, scale='up', **act_args))
            head_ch = head_ch // 2

        self.encoder = nn.Sequential(*self.encoder)
        self.body = nn.Sequential(*self.body)
        self.decoder = nn.Sequential(*self.decoder)
        self.out_img_conv = ConvLayer(ch_clip(head_ch), 3)
        self.out_mask_conv = ConvLayer(ch_clip(head_ch), parsing_ch)

    # ------------------------------------------------------------------------------------------ weights
    def _prepared(self, device) -> dict:
        """Folded kernel operands on `device`, rebuilt when any parameter or buffer changes (pointer or version)."""
        return cached(self, "prepared", (*self.parameters(), *self.buffers()), device, lambda: self._build_prepared(device))

    def _build_prepared(self, device) -> dict:
        def plain(layer: ConvLayer):
            conv = layer.conv2d
            return conv.weight.detach().float().contiguous().to(device), conv.bias.detach().float().contiguous().to(device)

        def planes(layer: ConvLayer, s2d=False):
            if layer.norm_type == 'bn':
                w, b = fold_bn(layer.conv2d.weight, layer.norm.norm)
            else:
                w, b = layer.conv2d.weight.detach().float(), layer.conv2d.bias.detach().float().contiguous()
            return (_conv_planes_s2d(w) if s2d else _conv_planes(w)).to(device), b.to(device)

        P = {"in": plain(self.encoder[0]), "img": plain(self.out_img_conv), "mask": plain(self.out_mask_conv)}
        P["down"] = [(planes(blk.shortcut_func, True), planes(blk.conv1), planes(blk.conv2, True)) for blk in self.encoder[1:]]
        P["body"] = [(planes(blk.conv1), planes(blk.conv2)) for blk in self.body]
        P["up"] = [(planes(blk.shortcut_func), planes(blk.conv1), planes(blk.conv2)) for blk in self.decoder]
        P["lut"] = torch.tensor(MASK_COLORMAP, dtype=torch.uint8, device=device)
        return P

    # ------------------------------------------------------------------------------------------ network
    def _check(self, x: torch.Tensor, prep: bool) -> None:
        if self._config != _RUN_CONFIG:
            raise NotImplementedError("e4s_b200: ParseNet runs FaceParse's configuration only (ParseNet(512, 512, 32, 64, 19, "
                                      "norm_type='bn', relu_type='LeakyReLU', ch_range=[32, 256]))")
        if self.training:
            raise NotImplementedError("e4s_b200: the ParseNet kernels are inference-only; call .eval() first")
        if torch.is_grad_enabled() and (x.requires_grad or any(p.requires_grad for p in self.parameters())):
            raise NotImplementedError("e4s_b200: the ParseNet kernels are forward-only; wrap the call in torch.no_grad() or "
                                      "freeze the parameters")
        size = self._config["in_size"]
        if not (x.is_cuda and x.dtype == torch.float32 and x.dim() == 4 and x.shape[1] == 3 and
                (prep or tuple(x.shape[2:]) == (size, size))):
            raise ValueError(f"e4s_b200: ParseNet takes a CUDA fp32 [B, 3, {size}, {size}] tensor, got {x.dtype} "
                             f"{tuple(x.shape)} on {x.device}")

    def _run(self, x: torch.Tensor, prep: bool = False, logits: bool = True, img: bool = True, mask=None):
        """The network on the kernels: (logits | None, out_img | None, mask of dtype `mask` | None).  prep: x is
        process_tensor's BGR [B, 3, H, W] in [0, 1], resized (nearest) to the network's size on the way in."""
        self._check(x, prep)
        size = self._config["in_size"]
        P = self._prepared(x.device)
        h = K.conv3x3_rgb_reflect(x.contiguous(), *P["in"], out_hw=(size, size), prep=prep)
        for sc, c1, c2 in P["down"]:
            idn = K.conv3x3_reflect_tc(K.space_to_depth(h), *sc, scale="down")
            r = K.conv3x3_reflect_tc(h, *c1, lrelu=0.2)
            h = K.conv3x3_reflect_tc(K.space_to_depth(r), *c2, r0=idn, scale="down")
        feat = h
        for i, (c1, c2) in enumerate(P["body"]):
            r = K.conv3x3_reflect_tc(h, *c1, lrelu=0.2)
            h = K.conv3x3_reflect_tc(r, *c2, r0=h, r1=feat if i == len(P["body"]) - 1 else None)
        for sc, c1, c2 in P["up"]:
            idn = K.conv3x3_reflect_tc(h, *sc, scale="up")
            r = K.conv3x3_reflect_tc(h, *c1, scale="up", lrelu=0.2)
            h = K.conv3x3_reflect_tc(r, *c2, r0=idn)
        out_mask, m = (K.gpen_parse_head(h, *P["mask"], P["lut"], logits=logits, mask=mask) if logits or mask is not None
                       else (None, None))
        out_img = K.conv3x3_rgb_reflect(h, *P["img"]) if img else None
        return out_mask, out_img, m

    def forward(self, x):
        """Planar x [B, 3, 512, 512] (CUDA fp32) -> (out_mask [B, 19, 512, 512], out_img [B, 3, 512, 512]).  No host
        synchronisation (graph-capturable)."""
        out_mask, out_img, _ = self._run(x)
        return out_mask, out_img


# FaceParse.MASK_COLORMAP (face_parsing.py:30): class -> mask value
MASK_COLORMAP = [0, 255, 255, 255, 255, 255, 255, 255, 255, 255, 255, 255, 255, 255, 0, 255, 255, 255, 0]
