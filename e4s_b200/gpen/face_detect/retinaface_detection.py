"""GPEN's face detection wrapper: mirror of src/pretrained/gpen/face_detect/retinaface_detection.py (RetinaFaceDetection).

Same constructor, load_model / check_keys / remove_prefix (a ``module.`` prefix is stripped; strict=False as in the
reference), and ``detect()``'s numpy contract: the host steps are the reference's (float32, the resize of images longer
than 1500 px, mean subtraction, exact for integer pixel values), then the forward, decode, selection and NMS run on the
device (RetinaFace.detect_batch) and one device-to-host copy returns (dets / ss, landms / ss), landms as [N, 10] ordered
x1..x5, y1..y5.  ``detect_batch`` is the batched device path: no host synchronisation, graph-capturable.

The kernels run image sizes that are multiples of 32 (the face swap detects on 1024 x 1024).  ``detect_tensor`` always
rescales to a longest side of 1000, which never is one, so it raises NotImplementedError; so does ``detect()`` on an image
longer than 1500 px (after the reference's resize to 1000).
"""
import os

import cv2
import numpy as np
import torch
import torch.backends.cudnn as cudnn

from ... import kernels as K
from .data import cfg_re50
from .facemodels.retinaface import RetinaFace


class RetinaFaceDetection(object):
    def __init__(self, base_dir, device='cuda', network='RetinaFace-R50'):
        torch.set_grad_enabled(False)
        cudnn.benchmark = True
        self.pretrained_path = os.path.join(base_dir, 'weights', network + '.pth')
        self.device = device
        self.cfg = cfg_re50
        self.net = RetinaFace(cfg=self.cfg, phase='test')
        self.load_model()
        self.net = self.net.to(device)
        self.mean = torch.tensor([[[[104]], [[117]], [[123]]]]).to(device)

    def check_keys(self, pretrained_state_dict):
        ckpt_keys = set(pretrained_state_dict.keys())
        model_keys = set(self.net.state_dict().keys())
        used_pretrained_keys = model_keys & ckpt_keys
        assert len(used_pretrained_keys) > 0, 'load NONE from pretrained checkpoint'
        return True

    def remove_prefix(self, state_dict, prefix):
        """Old style model is stored with all names of parameters sharing common prefix 'module.'"""
        f = lambda x: x.split(prefix, 1)[-1] if x.startswith(prefix) else x  # noqa: E731
        return {f(key): value for key, value in state_dict.items()}

    def load_model(self, load_to_cpu=False):
        pretrained_dict = torch.load(self.pretrained_path, map_location=torch.device('cpu'))
        if "state_dict" in pretrained_dict.keys():
            pretrained_dict = self.remove_prefix(pretrained_dict['state_dict'], 'module.')
        else:
            pretrained_dict = self.remove_prefix(pretrained_dict, 'module.')
        self.check_keys(pretrained_dict)
        self.net.load_state_dict(pretrained_dict, strict=False)
        self.net.eval()

    def detect(self, img_raw, resize=1, confidence_threshold=0.9, nms_threshold=0.4, top_k=5000, keep_top_k=750,
               save_image=False):
        img = np.float32(img_raw)
        im_height, im_width = img.shape[:2]
        ss = 1.0
        if max(im_height, im_width) > 1500:
            ss = 1000.0 / max(im_height, im_width)
            img = cv2.resize(img, (0, 0), fx=ss, fy=ss)
        img -= (104, 117, 123)
        x = torch.from_numpy(np.ascontiguousarray(img.transpose(2, 0, 1))).unsqueeze(0).to(self.device)
        with torch.no_grad():
            dets, landms, count = self.net.detect_batch(x, resize, confidence_threshold, nms_threshold, top_k, keep_top_k)
            k = dets.shape[1]
            host = torch.cat([count.float(), dets[0].flatten(), landms[0].flatten()]).cpu().numpy()    # one copy
        n = int(host[0])
        dets = host[1:1 + 5 * k].reshape(k, 5)[:n]
        landms = host[1 + 5 * k:].reshape(k, 10)[:n]
        return dets / ss, landms / ss

    def detect_batch(self, imgs, resize=1, confidence_threshold=0.9, nms_threshold=0.4, top_k=5000, keep_top_k=750):
        """CUDA planar BGR [B, 3, H, W] with 0-255 values (uint8 or float32; H, W multiples of 32) -> (dets [B, keep_top_k, 5],
        landms [B, keep_top_k, 10] (x1..x5, y1..y5), count [B] int32), all on the device; slots past count are
        unspecified.  detect()'s selection per image, with no host synchronisation (graph-capturable)."""
        if not (isinstance(imgs, torch.Tensor) and imgs.is_cuda and imgs.dtype in (torch.uint8, torch.float32) and
                imgs.dim() == 4 and imgs.shape[1] == 3):
            raise ValueError("e4s_b200: detect_batch takes a CUDA uint8 / float32 [B, 3, H, W] tensor, got "
                             f"{getattr(imgs, 'dtype', type(imgs))} {tuple(getattr(imgs, 'shape', ()))}")
        if imgs.shape[2] % 32 or imgs.shape[3] % 32:
            raise NotImplementedError(f"e4s_b200: RetinaFace runs image sizes that are multiples of 32; got "
                                      f"{tuple(imgs.shape[2:])}")
        with torch.no_grad():
            x = K.retinaface_prep(imgs.contiguous())
            return self.net.detect_batch(x, resize, confidence_threshold, nms_threshold, top_k, keep_top_k)

    def detect_tensor(self, img, resize=1, confidence_threshold=0.9, nms_threshold=0.4, top_k=5000, keep_top_k=750,
                      save_image=False):
        raise NotImplementedError("e4s_b200: detect_tensor rescales to a longest side of 1000 pixels, which is not a multiple "
                                  "of 32; use detect_batch on the 1024 x 1024 images instead")
