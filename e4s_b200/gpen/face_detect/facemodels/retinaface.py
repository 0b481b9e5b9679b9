"""GPEN's face detector: mirror of src/pretrained/gpen/face_detect/facemodels/retinaface.py (ClassHead, BboxHead,
LandmarkHead, RetinaFace).

The module tree, constructor arguments and state-dict keys are the reference's (the body is torchvision's resnet50 under
IntermediateLayerGetter), so ``RetinaFace-R50.pth`` loads unchanged.  On cfg_re50 with phase 'test', ``RetinaFace.forward``
does not run those torch modules: the network executes on the e4s_b200 kernels, forward only, BatchNorm folded into the
weights and bias in float64 (every activation is ReLU: out_channel 256 > 64 gives the FPN and SSH LeakyReLUs slope 0) -

* the stem (7x7 / 2 conv, BN, ReLU, 3x3 / 2 max-pool) on ``e4s_parser_stem_f32``, the same stem as BiSeNet's ResNet-18;
* every 1x1 convolution (bottleneck conv1 / conv3, the stride-1 and stride-2 downsample shortcuts, the FPN laterals, the
  heads) on the tensor-core kernel's pointwise mode (``e4s_conv1x1_tcr_f32``): conv3 adds the shortcut before its ReLU, an
  FPN lateral adds the nearest-up-sampled coarser level after its ReLU, so neither sum is a separate pass;
* the 3x3 convolutions on the plain mode with zero padding (``e4s_conv3x3_zero_tcr_f32``); each SSH branch writes its
  ReLU'd output into its channel slice of one [B, h, w, 256] buffer (no torch.cat, no separate ReLU); the stride-2 ones
  (the first conv2 of layer2-4) as four taps over the space-to-depth repack of their input (``e4s_space_to_depth_f32``);
* every convolution's N tile follows its channel count, never the batch: an image's detections are bit identical alone,
  inside any batch and graph-replayed;
* the three heads of a level as one 1x1 launch, 256 -> 32 = class 4 | bbox 8 | landmark 20;
* softmax, priors, box and landmark decode on ``e4s_retinaface_decode_f32``; for detection, a stable descending sort of
  the scores and the greedy NMS kernel ``e4s_retinaface_nms_f32`` (RetinaFace.detect_batch).

Other configurations, phase 'train', autograd and sizes that are not multiples of 32 build the module tree and raise
NotImplementedError in forward.
"""
import torch
import torchvision.models as models
import torchvision.models._utils as _utils
from torch import nn

from .... import kernels as K
from ....encoders.psp_encoders import _conv_planes, _conv_planes_s2d
from ....face_parsing.model import fold_bn
from ....prepared import cached
from .net import FPN, SSH, MobileNetV1


class ClassHead(nn.Module):
    def __init__(self, inchannels=512, num_anchors=3):
        super().__init__()
        self.num_anchors = num_anchors
        self.conv1x1 = nn.Conv2d(inchannels, self.num_anchors * 2, kernel_size=(1, 1), stride=1, padding=0)

    def forward(self, x):
        out = self.conv1x1(x).permute(0, 2, 3, 1).contiguous()
        return out.view(out.shape[0], -1, 2)


class BboxHead(nn.Module):
    def __init__(self, inchannels=512, num_anchors=3):
        super().__init__()
        self.conv1x1 = nn.Conv2d(inchannels, num_anchors * 4, kernel_size=(1, 1), stride=1, padding=0)

    def forward(self, x):
        out = self.conv1x1(x).permute(0, 2, 3, 1).contiguous()
        return out.view(out.shape[0], -1, 4)


class LandmarkHead(nn.Module):
    def __init__(self, inchannels=512, num_anchors=3):
        super().__init__()
        self.conv1x1 = nn.Conv2d(inchannels, num_anchors * 10, kernel_size=(1, 1), stride=1, padding=0)

    def forward(self, x):
        out = self.conv1x1(x).permute(0, 2, 3, 1).contiguous()
        return out.view(out.shape[0], -1, 10)


def _pw_planes(w: torch.Tensor) -> torch.Tensor:
    """1x1 weight [Cout, Cin(, 1, 1)] -> bf16 hi / lo planes [2, Cout, Cin] of the pointwise kernel."""
    return K.split_bf16(w.reshape(w.shape[0], w.shape[1]).float().contiguous())


class RetinaFace(nn.Module):
    def __init__(self, cfg=None, phase='train'):
        super().__init__()
        self.phase = phase
        self._cfg_name = cfg['name']
        backbone = None
        if cfg['name'] == 'mobilenet0.25':
            backbone = MobileNetV1()
            if cfg['pretrain']:
                raise NotImplementedError("e4s_b200: the MobileNet-0.25 ImageNet checkpoint is not loaded here; load the "
                                          "detector's state dict instead")
        elif cfg['name'] == 'Resnet50':
            backbone = models.resnet50(weights=models.ResNet50_Weights.IMAGENET1K_V1 if cfg['pretrain'] else None)
        self.body = _utils.IntermediateLayerGetter(backbone, cfg['return_layers'])
        in_channels_stage2 = cfg['in_channel']
        in_channels_list = [in_channels_stage2 * 2, in_channels_stage2 * 4, in_channels_stage2 * 8]
        out_channels = cfg['out_channel']
        self.fpn = FPN(in_channels_list, out_channels)
        self.ssh1 = SSH(out_channels, out_channels)
        self.ssh2 = SSH(out_channels, out_channels)
        self.ssh3 = SSH(out_channels, out_channels)
        self.ClassHead = self._make_class_head(fpn_num=3, inchannels=cfg['out_channel'])
        self.BboxHead = self._make_bbox_head(fpn_num=3, inchannels=cfg['out_channel'])
        self.LandmarkHead = self._make_landmark_head(fpn_num=3, inchannels=cfg['out_channel'])

    def _make_class_head(self, fpn_num=3, inchannels=64, anchor_num=2):
        return nn.ModuleList([ClassHead(inchannels, anchor_num) for _ in range(fpn_num)])

    def _make_bbox_head(self, fpn_num=3, inchannels=64, anchor_num=2):
        return nn.ModuleList([BboxHead(inchannels, anchor_num) for _ in range(fpn_num)])

    def _make_landmark_head(self, fpn_num=3, inchannels=64, anchor_num=2):
        return nn.ModuleList([LandmarkHead(inchannels, anchor_num) for _ in range(fpn_num)])

    # ------------------------------------------------------------------------------------------ weights
    def _prepared(self, device) -> dict:
        """Folded kernel operands on `device`, rebuilt when any parameter or buffer changes (pointer or version)."""
        return cached(self, "prepared", (*self.parameters(), *self.buffers()), device, lambda: self._build_prepared(device))

    def _build_prepared(self, device) -> dict:
        def pw(conv, bn):
            w, b = fold_bn(conv.weight, bn)
            return _pw_planes(w).to(device), b.to(device)

        def c3(conv, bn, s2d=False):
            w, b = fold_bn(conv.weight, bn)
            return (_conv_planes_s2d(w) if s2d else _conv_planes(w)).to(device), b.to(device)

        body = self.body
        w7, b7 = fold_bn(body.conv1.weight, body.bn1)
        P = {"stem": (w7.contiguous().to(device), b7.to(device)), "layers": []}
        for name in ("layer1", "layer2", "layer3", "layer4"):
            blocks = []
            for blk in getattr(body, name):
                stride = blk.conv2.stride[0]
                d = {"stride": stride, "conv1": pw(blk.conv1, blk.bn1), "conv2": c3(blk.conv2, blk.bn2, stride == 2),
                     "conv3": pw(blk.conv3, blk.bn3)}
                if blk.downsample is not None:
                    d["down"] = pw(blk.downsample[0], blk.downsample[1])
                blocks.append(d)
            P["layers"].append(blocks)
        f = self.fpn
        P["lateral"] = [pw(m[0], m[1]) for m in (f.output1, f.output2, f.output3)]
        P["merge"] = [c3(m[0], m[1]) for m in (f.merge1, f.merge2)]
        P["ssh"] = [{k: c3(getattr(s, k)[0], getattr(s, k)[1]) for k in ("conv3X3", "conv5X5_1", "conv5X5_2", "conv7X7_2",
                                                                         "conv7x7_3")} for s in (self.ssh1, self.ssh2, self.ssh3)]
        heads = []
        for i in range(3):
            convs = [self.ClassHead[i].conv1x1, self.BboxHead[i].conv1x1, self.LandmarkHead[i].conv1x1]
            w = torch.cat([c.weight.detach().float() for c in convs], 0)
            b = torch.cat([c.bias.detach().float() for c in convs], 0).contiguous()
            heads.append((_pw_planes(w).to(device), b.to(device)))
        P["heads"] = heads
        return P

    # ------------------------------------------------------------------------------------------ network
    def _check(self, x: torch.Tensor) -> None:
        if self._cfg_name != 'Resnet50':
            raise NotImplementedError("e4s_b200: RetinaFace runs cfg_re50 (ResNet-50) only; the MobileNet-0.25 "
                                      "configuration is not implemented on the kernels")
        if self.phase != 'test':
            raise NotImplementedError("e4s_b200: the RetinaFace kernels run phase='test' only")
        if self.training:
            raise NotImplementedError("e4s_b200: the RetinaFace kernels are inference-only; call .eval() first")
        if torch.is_grad_enabled() and (x.requires_grad or any(p.requires_grad for p in self.parameters())):
            raise NotImplementedError("e4s_b200: the RetinaFace kernels are forward-only; wrap the call in torch.no_grad() "
                                      "or freeze the parameters")
        if not (x.is_cuda and x.dtype == torch.float32 and x.dim() == 4 and x.shape[1] == 3):
            raise ValueError(f"e4s_b200: RetinaFace takes a CUDA fp32 [B, 3, H, W] tensor, got {x.dtype} {tuple(x.shape)} "
                             f"on {x.device}")
        if x.shape[2] % 32 or x.shape[3] % 32:
            raise NotImplementedError(f"e4s_b200: RetinaFace runs image sizes that are multiples of 32 (every stride-2 "
                                      f"stage needs even sizes); got {tuple(x.shape[2:])}")

    @staticmethod
    def _bottleneck(d: dict, x: torch.Tensor) -> torch.Tensor:
        r = K.conv1x1_tc(x, *d["conv1"], lrelu=0.0)
        if d["stride"] == 2:
            r = K.conv3x3_zero_tc(K.space_to_depth(r), *d["conv2"], stride=2, lrelu=0.0)
        else:
            r = K.conv3x3_zero_tc(r, *d["conv2"], lrelu=0.0)
        idn = K.conv1x1_tc(x, *d["down"], stride=d["stride"]) if "down" in d else x
        return K.conv1x1_tc(r, *d["conv3"], r0=idn, lrelu=0.0)

    def _heads(self, x: torch.Tensor) -> torch.Tensor:
        """Mean-subtracted planar x [B, 3, H, W] -> the three levels' head maps, flat, level l as [B, H / s_l, W / s_l, 32]."""
        self._check(x)
        P = self._prepared(x.device)
        b, _, h, w = x.shape
        f = K.parser_stem(x.contiguous(), *P["stem"])
        feats = []
        for li, layer in enumerate(P["layers"]):
            for d in layer:
                f = self._bottleneck(d, f)
            if li:
                feats.append(f)
        lat = P["lateral"]
        o3 = K.conv1x1_tc(feats[2], *lat[2], lrelu=0.0)
        o2 = K.conv3x3_zero_tc(K.conv1x1_tc(feats[1], *lat[1], r_up=o3, lrelu=0.0), *P["merge"][1], lrelu=0.0)
        o1 = K.conv3x3_zero_tc(K.conv1x1_tc(feats[0], *lat[0], r_up=o2, lrelu=0.0), *P["merge"][0], lrelu=0.0)
        sizes = [(h // s, w // s) for s in (8, 16, 32)]
        heads = torch.empty(b * 32 * sum(a * c for a, c in sizes), device=x.device, dtype=torch.float32)
        off = 0
        for lvl, (feat, (lh, lw)) in enumerate(zip((o1, o2, o3), sizes)):
            S = P["ssh"][lvl]
            cat = torch.empty((b, lh, lw, 256), device=x.device, dtype=torch.float32)
            K.conv3x3_zero_tc(feat, *S["conv3X3"], out=cat[..., :128], lrelu=0.0)
            t5 = K.conv3x3_zero_tc(feat, *S["conv5X5_1"], lrelu=0.0)
            K.conv3x3_zero_tc(t5, *S["conv5X5_2"], out=cat[..., 128:192], lrelu=0.0)
            t7 = K.conv3x3_zero_tc(t5, *S["conv7X7_2"], lrelu=0.0)
            K.conv3x3_zero_tc(t7, *S["conv7x7_3"], out=cat[..., 192:], lrelu=0.0)
            n = b * lh * lw * 32
            K.conv1x1_tc(cat, *P["heads"][lvl], out=heads[off:off + n].view(b, lh, lw, 32))
            off += n
        return heads

    def forward(self, inputs):
        """Planar CUDA [B, 3, H, W] (BGR minus (104, 117, 123); H, W multiples of 32) -> (loc [B, P, 4], softmax conf
        [B, P, 2], landms [B, P, 10]) in the reference's prior order.  No host synchronisation (graph-capturable)."""
        heads = self._heads(inputs)
        b, _, h, w = inputs.shape
        _, module = K.retinaface_decode(heads, b, h, w, boxes=False, keys=False, module=True)
        return module

    def detect_batch(self, x, resize=1, confidence_threshold=0.9, nms_threshold=0.4, top_k=5000, keep_top_k=750):
        """Mean-subtracted planar x [B, 3, H, W] -> (dets [B, keep_top_k, 5], landms [B, keep_top_k, 10], count [B] int32),
        RetinaFaceDetection.detect's selection per image.  Ties in score are ordered by ascending prior index."""
        if top_k < 0 or keep_top_k < 0:
            raise ValueError("e4s_b200: top_k and keep_top_k must be >= 0")
        heads = self._heads(x)
        b, _, h, w = x.shape
        (boxes, landms, keys), _ = K.retinaface_decode(heads, b, h, w, resize=resize, conf_thr=confidence_threshold)
        keys_sorted, order = torch.sort(keys, dim=1, descending=True, stable=True)
        return K.retinaface_nms(boxes, landms, keys_sorted, order, confidence_threshold, nms_threshold, top_k, keep_top_k)
