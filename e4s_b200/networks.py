"""E4S model facade: mirror of src/models/networks.py (LocalMLP :15-39, Net3 :41-183).

Same constructor (an ``opts`` object with num_seg_cls, remaining_layer_idx, out_size, train_G,
start_from_latent_avg, learn_in_w, fsencoder_type), same attribute/parameter names, same methods
(``forward``, ``get_style_vectors``, ``cal_style_codes``, ``gen_img``), so the reference scripts
(scripts/face_swap.py:372-376, scripts/optimization.py:63-70) can construct and call it unchanged.
"""
import torch
import torch.nn as nn
import torch.nn.functional as F

from .stylegan2.model import EqualLinear, Generator
from .encoders.psp_encoders import FSEncoder_PSP
from .prepared import cached


class LocalMLP(nn.Module):
    """Per-region map from a 1280-d texture vector to `num_w_layers` W+ codes."""

    def __init__(self, dim_component=512, dim_style=512, num_w_layers=18, latent_squeeze_ratio=1):
        super().__init__()
        self.dim_component = dim_component
        self.dim_style = dim_style
        self.num_w_layers = num_w_layers
        hidden = dim_style // latent_squeeze_ratio
        self.mlp = nn.Sequential(EqualLinear(dim_component, hidden, lr_mul=1), nn.LeakyReLU(),
                                 EqualLinear(hidden, dim_style * num_w_layers, lr_mul=1))

    def forward(self, x):
        return self.mlp(x).view(-1, self.num_w_layers, self.dim_style)


class Net3(nn.Module):
    """Multi-scale region style extraction + mask-guided StyleGAN2."""

    def __init__(self, opts):
        super().__init__()
        self.opts = opts
        assert self.opts.fsencoder_type in ["psp"]
        self.encoder = FSEncoder_PSP(mode="ir_se", opts=self.opts)
        dim_s_code = 256 + 512 + 512
        self.split_layer_idx = 5
        self.remaining_layer_idx = self.opts.remaining_layer_idx
        K = self.remaining_layer_idx
        self.MLPs = nn.ModuleList([LocalMLP(dim_component=dim_s_code, dim_style=512, num_w_layers=K if K != 17 else 18)
                                   for _ in range(self.opts.num_seg_cls)])
        self.G = Generator(size=self.opts.out_size, style_dim=512, n_mlp=8, split_layer_idx=self.split_layer_idx,
                           remaining_layer_idx=K)
        # which parts are frozen, networks.py:68-82
        frozen = self.G.style.parameters() if self.opts.train_G else self.G.parameters()
        for p in frozen:
            p.requires_grad = False
        if K != 17:
            for p in self.G.convs[-(17 - K):].parameters():
                p.requires_grad = False
            for p in self.G.to_rgbs[-(17 - K) // 2 - 1:].parameters():
                p.requires_grad = False

    # ------------------------------------------------------------------ texture vectors -> W+ codes
    def _stacked_mlps(self):
        params = [p for m in self.MLPs for p in m.parameters()]

        def build():
            with torch.no_grad():
                l0 = [m.mlp[0] for m in self.MLPs]
                l2 = [m.mlp[2] for m in self.MLPs]
                w0 = torch.stack([l.weight * l.scale for l in l0]).float().contiguous()    # [ncls, 512, 1280]  (nn.Linear layout)
                b0 = torch.stack([l.bias * l.lr_mul for l in l0]).float().contiguous()     # [ncls, 512]
                w2 = torch.stack([l.weight * l.scale for l in l2]).float().contiguous()    # [ncls, K*512, 512]
                b2 = torch.stack([l.bias * l.lr_mul for l in l2]).float().contiguous()
            return w0, b0, w2, b2
        return cached(self, "mlps", params, params[0].device, build)

    def _region_codes(self, style_vectors):
        """[B, ncls, 1280] -> [B, ncls, K, 512]: the ncls LocalMLPs (networks.py:15-39) as two grouped GEMMs on the library's own
        small-GEMM kernel (csrc/linear.cu), leaky ReLU 0.01 fused into the first."""
        bs, ncls = style_vectors.shape[:2]
        trainable = torch.is_grad_enabled() and any(p.requires_grad for p in self.MLPs.parameters())
        if trainable:   # keep the parameter graph (training is outside the hot path)
            return torch.stack([self.MLPs[i](style_vectors[:, i, :]) for i in range(ncls)], dim=1)
        w0, b0, w2, b2 = self._stacked_mlps()
        if not style_vectors.is_cuda:
            raise RuntimeError("input must be a CUDA tensor")
        from .stylegan2.modconv import LinearFn
        x = style_vectors.float().transpose(0, 1).contiguous()              # [ncls, B, 1280]
        h = LinearFn.apply(x, w0, b0, 0.01)                           # [ncls, B, 512]   EqualLinear + LeakyReLU(0.01)
        o = LinearFn.apply(h, w2, b2, 1.0)                            # [ncls, B, K*512]
        return o.transpose(0, 1).reshape(bs, ncls, -1, 512)

    def _add_latent_avg(self, codes):
        bs, ncls = codes.shape[:2]
        K = self.remaining_layer_idx
        if not self.opts.start_from_latent_avg:
            return codes
        if self.opts.learn_in_w:
            codes = codes + self.latent_avg[:K, :].repeat(bs, ncls, 1)
            rest = self.latent_avg[K:, :].repeat(bs, ncls, 1)
            return torch.cat([codes, rest], dim=2)
        if K != 17:
            codes = codes + self.latent_avg[:K, :].reshape(1, 1, K, -1)
            rest = self.latent_avg[K:, :].reshape(1, 1, -1, codes.shape[-1]).expand(bs, ncls, -1, -1)
            return torch.cat([codes, rest], dim=2)
        return codes + self.latent_avg.reshape(1, 1, *self.latent_avg.shape)

    def cal_style_codes(self, style_vectors):
        """Per-region texture vectors [B, ncls, 1280] -> style codes [B, ncls, 18, 512]."""
        return self._add_latent_avg(self._region_codes(style_vectors))

    # ------------------------------------------------------------------------------ encoder
    def get_style_vectors(self, img, mask):
        """img [B,3,H,W], mask one-hot [B,ncls,Hm,Wm] -> ([B,ncls,1280], zeros [B,512,16,16])."""
        return self.encoder(F.interpolate(img, (256, 256), mode="bilinear"), mask)

    # ---------------------------------------------------------------------------- synthesis
    def gen_img(self, struc_codes, style_codes, mask, randomize_noise=True, noise=None, return_latents=False):
        images, result_latent, structure_feats = self.G([style_codes], struc_codes, mask, input_is_latent=True,
                                                        randomize_noise=randomize_noise, noise=noise,
                                                        return_latents=return_latents, use_structure_code=False)
        if return_latents:
            return images, result_latent, structure_feats
        return images, -1, structure_feats

    def forward(self, img, mask, resize=False, randomize_noise=True, return_latents=False):
        style_vectors, structure_feats = self.get_style_vectors(img, mask)
        codes = self.cal_style_codes(style_vectors)
        images, result_latent, feats = self.G([codes], structure_feats, mask, input_is_latent=True,
                                              randomize_noise=randomize_noise, return_latents=return_latents,
                                              use_structure_code=False)
        if return_latents:
            return images, feats, result_latent
        return images, feats
