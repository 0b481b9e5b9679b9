"""GPEN's face-parse wrapper: mirror of src/pretrained/gpen/face_parse/face_parsing.py (FaceParse).

``process`` keeps the reference's host-side contract (numpy BGR uint8 image in, list of {0, 255} uint8 masks out; the same
cv2.resize and float64 normalisation, so the network input is bit-equal to the reference's).  ``process_tensor`` is the
batched device path: BGR [B, 3, H, W] in [0, 1] -> int64 [1, B, 512, 512], with the flip, normalisation and nearest resize
done as encoder.0 reads its input and the mask head writing the MASK_COLORMAP values directly (no logits written, no host
synchronisation: capturable in a CUDA graph).
"""
import os

import numpy as np
import torch

from .parse_model import MASK_COLORMAP, ParseNet


class FaceParse(object):
    def __init__(self, base_dir='./', model='ParseNet-latest', device='cuda'):
        self.mfile = os.path.join(base_dir, 'weights', model + '.pth')
        self.size = 512
        self.device = device
        self.MASK_COLORMAP = list(MASK_COLORMAP)
        self.load_model()

    def load_model(self):
        self.faceparse = ParseNet(self.size, self.size, 32, 64, 19, norm_type='bn', relu_type='LeakyReLU', ch_range=[32, 256])
        self.faceparse.load_state_dict(torch.load(self.mfile, map_location=torch.device('cpu')))
        self.faceparse.to(self.device)
        self.faceparse.eval()

    def _masks(self, imt, prep, dtype):
        if self.MASK_COLORMAP != MASK_COLORMAP:
            raise NotImplementedError("e4s_b200: FaceParse runs the reference's MASK_COLORMAP only")
        with torch.no_grad():
            return self.faceparse._run(imt, prep=prep, logits=False, img=False, mask=dtype)[2]

    def process(self, im):
        import cv2
        im = cv2.resize(im, (self.size, self.size))
        imt = self.img2tensor(im)
        mask = self._masks(imt, False, torch.uint8)
        return list(mask.cpu().numpy())

    def process_tensor(self, imt):
        if not (imt.is_cuda and imt.dtype == torch.float32 and imt.dim() == 4 and imt.shape[1] == 3):
            raise ValueError(f"e4s_b200: FaceParse.process_tensor takes a CUDA fp32 [B, 3, H, W] tensor, got {imt.dtype} "
                             f"{tuple(imt.shape)} on {imt.device}")
        return self._masks(imt.contiguous(), True, torch.int64).unsqueeze(0)

    def img2tensor(self, img):
        img = img[..., ::-1]
        img = img / 255. * 2 - 1
        img_tensor = torch.from_numpy(img.transpose(2, 0, 1)).unsqueeze(0).to(self.device)
        return img_tensor.float()
