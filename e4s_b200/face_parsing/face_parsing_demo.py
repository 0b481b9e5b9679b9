"""Face parsing entry points: mirror of src/pretrained/face_parsing/face_parsing_demo.py.

``init_faceParsing_pretrained_model`` / ``faceParsing_demo`` keep the reference's signatures and return types (a PIL image
in, a numpy uint8 label map out).  ``FaceParser.parse`` is the batched device path the reference lacks: CUDA images in,
uint8 12-class label maps out, with no host synchronisation and no logits written, so it can be captured in a CUDA graph
and its output fed to ``e4s_b200.face_swap.swap_faces`` as it is.

The "segnext" parser needs mmseg and is not provided.
"""
import numpy as np
import torch
import torchvision
from PIL import Image
from torch import nn

import cv2

from .. import kernels as K
from ..masks import FFHQ19_TO_12
from .model import BiSeNet, seg_mean, seg_std


def _bicubic_taps(factor: int, a: float = -0.5) -> torch.Tensor:
    """BicubicDownSample's filter: 4 f taps of the cubic convolution kernel (parameter a) at (i - 2 f + 0.5) / f, normalised
    to sum 1, fp32."""
    x = ((torch.arange(4 * factor, dtype=torch.float32) - 2 * factor + 0.5) / factor).abs()
    near = (a + 2.0) * x ** 3 - (a + 3.0) * x ** 2 + 1.0
    far = a * x ** 3 - 5.0 * a * x ** 2 + 8.0 * a * x - 4.0 * a
    k = torch.where(x <= 1.0, near, torch.where(x < 2.0, far, torch.zeros_like(x)))
    return k / k.sum()


class BicubicDownSample(nn.Module):
    """Separable bicubic down-sampling by `factor` with reflect padding (the vertical pass first), on the library's kernel.
    ``k1`` / ``k2`` are the reference's per-channel [3, 1, 4f, 1] / [3, 1, 1, 4f] filters."""

    def __init__(self, factor=4, cuda=True, padding="reflect"):
        super().__init__()
        self.factor = factor
        k = _bicubic_taps(factor)
        self.k1 = k.reshape(1, 1, -1, 1).repeat(3, 1, 1, 1)
        self.k2 = k.reshape(1, 1, 1, -1).repeat(3, 1, 1, 1)
        self.cuda = ".cuda" if cuda else ""
        self.padding = padding
        self._taps = {}

    def taps(self, device) -> torch.Tensor:
        """The filter [4f] on `device` (copied once per device)."""
        key = str(device)
        if key not in self._taps:
            self._taps[key] = self.k1[0, 0, :, 0].contiguous().to(device)
        return self._taps[key]

    def forward(self, x, nhwc=False, clip_round=False, byte_output=False):
        if nhwc or clip_round or byte_output or self.padding != "reflect":
            raise NotImplementedError("e4s_b200: BicubicDownSample implements the planar fp32 reflect-padded case only")
        if not (x.is_cuda and x.dtype == torch.float32 and x.dim() == 4 and x.shape[1] == 3):
            raise ValueError(f"e4s_b200: BicubicDownSample takes a CUDA fp32 [B, 3, H, W] tensor, got {x.dtype} "
                             f"{tuple(x.shape)} on {x.device}")
        return K.bicubic_down_norm(x.contiguous(), self.taps(x.device), self.factor)


# 24 part colours (RGB); class 0 (background) is drawn white
_PART_COLORS = np.array([[255, 0, 0], [255, 85, 0], [255, 170, 0], [255, 0, 85], [255, 0, 170], [0, 255, 0], [85, 255, 0],
                         [170, 255, 0], [0, 255, 85], [0, 255, 170], [0, 0, 255], [85, 0, 255], [170, 0, 255], [0, 85, 255],
                         [0, 170, 255], [255, 255, 0], [255, 255, 85], [255, 255, 170], [255, 0, 255], [255, 85, 255],
                         [255, 170, 255], [0, 255, 255], [85, 255, 255], [170, 255, 255]], dtype=np.uint8)


def vis_parsing_maps(image, parsing_anno, stride=1):
    """Overlay of a label map on its image, as a BGR uint8 array (cv2 order): 0.4 x the image, resized bilinearly to
    (parsing_anno.shape[0], parsing_anno.shape[1]) as (width, height), plus 0.6 x the class colours, the labels enlarged
    `stride` times by nearest neighbour."""
    im = np.array(image.resize((parsing_anno.shape[0], parsing_anno.shape[1]), Image.BILINEAR)).astype(np.uint8)
    anno = cv2.resize(parsing_anno.astype(np.uint8), None, fx=stride, fy=stride, interpolation=cv2.INTER_NEAREST)
    palette = _PART_COLORS.copy()
    palette[0] = 255
    colour = palette[anno]
    return cv2.addWeighted(cv2.cvtColor(im, cv2.COLOR_RGB2BGR), 0.4, colour, 0.6, 0)


class FaceParser(nn.Module):
    """BiSeNet with its preprocessing.  ``size``: the image side the parser is built for; images at least 512 wide are
    down-sampled by f = size // 512 (2 for 1024 x 1024 faces), narrower ones are resized to 512 x 512 on the host."""

    def __init__(self, seg_ckpt, size=1024, device="cuda"):
        super().__init__()
        self.seg_ckpt = seg_ckpt
        self.size = size
        self.device = device
        self.load_segmentation_network()
        self.load_downsampling()
        self._consts = {}

    def load_downsampling(self):
        self.downsample = BicubicDownSample(factor=self.size // 512)
        self.downsample_256 = BicubicDownSample(factor=self.size // 256)

    def load_segmentation_network(self):
        self.seg = BiSeNet(n_classes=19)
        self.seg.to(self.device)
        self.seg.load_state_dict(torch.load(self.seg_ckpt, map_location="cpu"))
        for param in self.seg.parameters():
            param.requires_grad = False
        self.seg.eval()

    def _device_consts(self, device):
        """(mean [3], std [3], 19 -> 12 table [256] uint8, one-tap filter) on `device`, copied once per device."""
        key = str(device)
        if key not in self._consts:
            self._consts[key] = (seg_mean.flatten().to(device), seg_std.flatten().to(device),
                                 torch.tensor(FFHQ19_TO_12, dtype=torch.uint8).to(device),
                                 torch.tensor([0.0, 1.0, 0.0, 0.0]).to(device))
        return self._consts[key]

    def parse(self, images, convert_to_seg12=True):
        """images: CUDA fp32 planar [B, 3, H, W] in [0, 1], H and W multiples of 32 f and W >= 512 -> uint8 [B, H/f, W/f]:
        the 12-class maps of the mask stage (convert_to_seg12) or the parser's 19 classes.  Enqueued on the current stream
        without a host synchronisation."""
        f = self.downsample.factor
        if not (isinstance(images, torch.Tensor) and images.is_cuda and images.dtype == torch.float32 and images.dim() == 4
                and images.shape[1] == 3):
            raise ValueError("FaceParser.parse takes CUDA fp32 images [B, 3, H, W], got "
                             + (f"{images.dtype} {tuple(images.shape)} on {images.device}" if isinstance(images, torch.Tensor)
                                else type(images).__name__))
        h, w = images.shape[2:]
        if h % (32 * f) or w % (32 * f) or w < 512:
            raise ValueError(f"FaceParser.parse: image sides must be multiples of {32 * f} (32 x the down-sampling factor "
                             f"{f}) and at least 512 wide, got {h}x{w}")
        mean, std, lut, _ = self._device_consts(images.device)
        with torch.no_grad():
            x = K.bicubic_down_norm(images.contiguous(), self.downsample.taps(images.device), f, mean, std)
            return self.seg.labels(x, lut if convert_to_seg12 else None)

    def preprocess_img(self, img):
        """PIL image -> the normalised network input [1, 3, h, w] on the parser's device."""
        mean, std, _, one_tap = self._device_consts(torch.device(self.device))
        if img.size[0] >= 512:
            im = torchvision.transforms.ToTensor()(img)[:3].unsqueeze(0).to(self.device)
            return K.bicubic_down_norm(im.contiguous(), self.downsample.taps(im.device), self.downsample.factor, mean, std)
        im = img.resize((512, 512), Image.BILINEAR)
        im = torchvision.transforms.ToTensor()(im)[:3].unsqueeze(0).to(self.device)
        # the filter (0, 1, 0, 0) at factor 1 passes every pixel through: clamp and normalisation only
        return K.bicubic_down_norm(im.contiguous(), one_tap, 1, mean, std)

    def forward(self, img):
        """PIL image -> the 19-class label map [h, w] (int64, on the device), as the reference returns it."""
        if img.size[0] >= 512:
            im = torchvision.transforms.ToTensor()(img)[:3].unsqueeze(0).to(self.device)
            return self.parse(im, convert_to_seg12=False)[0].long()
        with torch.no_grad():
            return self.seg.labels(self.preprocess_img(img))[0].long()


# ===============================================
def init_faceParsing_pretrained_model(faceParser_name, ckpt_path, config_path=""):
    if faceParser_name == "default":
        return FaceParser(seg_ckpt=ckpt_path)
    if faceParser_name == "segnext":
        raise NotImplementedError("e4s_b200: the SegNeXt parser needs mmseg and is not provided; use 'default' (BiSeNet)")
    raise ValueError(f"unknown face parser {faceParser_name!r}")


def faceParsing_demo(model, img, convert_to_seg12=True, model_name="default"):
    """PIL image -> numpy uint8 label map [h, w]: the 12 classes of the mask stage (convert_to_seg12) or the parser's 19."""
    if model_name == "segnext":
        raise NotImplementedError("e4s_b200: the SegNeXt parser needs mmseg and is not provided")
    if model_name != "default":
        raise ValueError(f"unknown face parser {model_name!r}")
    with torch.no_grad():
        seg = model(img).cpu().numpy().astype(np.uint8)
    if convert_to_seg12:
        seg = np.asarray(FFHQ19_TO_12, dtype=np.uint8)[seg]
    return seg
