"""GPEN's super-resolution front end: mirror of src/pretrained/gpen/sr_model/real_esrnet.py.

``RealESRNet(base_dir, model, scale, device)`` loads ``<base_dir>/weights/<model>_x<scale>.pth`` (``realesrnet_x2.pth`` when
model is None) into the mirror's RRDBNet with strict=True, as the reference does.  ``process(img)`` keeps the reference's
contract - a numpy uint8 BGR [H, W, 3] image in, the uint8 BGR [4H, 4W, 3] image out, None (with a message) when the
network fails at run time - and runs RRDBNet.forward on the library's kernels, with the uint8 <-> float conversions on the
device.  Only scale 4 runs (the face swap's configuration); the other scales raise NotImplementedError.
"""
import os

import numpy as np
import torch

from .rrdbnet_arch import RRDBNet


class RealESRNet(object):
    def __init__(self, base_dir='./', model=None, scale=2, device='cuda'):
        self.base_dir = base_dir
        self.scale = scale
        self.device = device
        self.load_srmodel(base_dir, model)

    def load_srmodel(self, base_dir, model):
        self.srmodel = RRDBNet(num_in_ch=3, num_out_ch=3, num_feat=32, num_block=23, num_grow_ch=32, scale=self.scale)
        if model is None:
            loadnet = torch.load(os.path.join(self.base_dir, 'weights', 'realesrnet_x2.pth'), map_location="cpu")
        else:
            loadnet = torch.load(os.path.join(self.base_dir, 'weights', model + '_x%d.pth' % self.scale), map_location="cpu")
        self.srmodel.load_state_dict(loadnet['params_ema'], strict=True)
        self.srmodel.eval()
        self.srmodel = self.srmodel.to(self.device)

    def process(self, img):
        """uint8 BGR [H, W, 3] -> uint8 BGR [4H, 4W, 3]: img / 255 in RGB, RRDBNet, clamp(0, 1), * 255, round half to even -
        the reference's float32 arithmetic, so the bytes are its bytes up to the network's own rounding."""
        if self.scale != 4:
            raise NotImplementedError(f"e4s_b200: RealESRNet runs scale 4 only, not {self.scale}")
        x = torch.from_numpy(np.ascontiguousarray(img)).to(self.device)
        x = (x[:, :, [2, 1, 0]].permute(2, 0, 1).float() / 255.).unsqueeze(0).contiguous()
        try:
            with torch.no_grad():
                output = self.srmodel(x)
        except RuntimeError as e:           # the reference returns None when the network fails (face_enhancement.py:64)
            print('sr failed:', e)
            return None
        output = (output[0].clamp_(0, 1)[[2, 1, 0]].permute(1, 2, 0) * 255.0).round().to(torch.uint8)
        return output.cpu().numpy()
