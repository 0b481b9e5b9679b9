"""CPU torch restatement of GPEN's RetinaFace-R50 detector (src/pretrained/gpen/face_detect/: facemodels/{retinaface,net}.py
on cfg_re50, layers/functions/prior_box.py, utils/box_utils.py decode / decode_landm, utils/nms/py_cpu_nms.py and
RetinaFaceDetection.detect), pinned against the unmodified reference by oracle/make_golden_retinaface.py.

The forward is written with F ops over a state dict (conv, eval-mode BatchNorm, ReLU, max-pool, nearest interpolate, cat,
softmax).  NMS orders candidates by descending score with ties in ascending prior index (the reference's two unstable numpy
argsorts leave that order to the implementation); on inputs without exact score ties it is py_cpu_nms.
"""
from __future__ import annotations

import numpy as np
import torch
import torch.nn.functional as F

MIN_SIZES = [[16, 32], [64, 128], [256, 512]]
STEPS = [8, 16, 32]
VARIANCE = [0.1, 0.2]
LAYERS = [("layer1", 3), ("layer2", 4), ("layer3", 6), ("layer4", 3)]


def synthetic_state() -> dict:
    from e4s_b200.synthetic import synthetic_retinaface_state
    return synthetic_retinaface_state()


def _bn(st, p, x):
    return F.batch_norm(x, st[p + ".running_mean"], st[p + ".running_var"], st[p + ".weight"], st[p + ".bias"], False, 0.0, 1e-5)


def _conv_bn(st, p, x, stride=1, relu=True):
    """nn.Sequential(Conv2d(bias=False), BatchNorm2d[, ReLU]) at prefix p (p.0, p.1)."""
    w = st[p + ".0.weight"]
    y = _bn(st, p + ".1", F.conv2d(x, w, None, stride, w.shape[-1] // 2))
    return F.relu(y) if relu else y


def forward(st: dict, x: torch.Tensor, branch: list | None = None):
    """Planar [B, 3, H, W] (BGR minus the mean) -> (loc [B, P, 4], conf [B, P, 2] (softmax), landms [B, P, 10]).
    branch: receives ||residual branch|| / ||identity|| of every bottleneck."""
    y = F.relu(_bn(st, "body.bn1", F.conv2d(x, st["body.conv1.weight"], None, 2, 3)))
    y = F.max_pool2d(y, 3, 2, 1)
    feats = []
    for name, n in LAYERS:
        for i in range(n):
            p = f"body.{name}.{i}"
            stride = 2 if (i == 0 and name != "layer1") else 1
            r = F.relu(_bn(st, p + ".bn1", F.conv2d(y, st[p + ".conv1.weight"])))
            r = F.relu(_bn(st, p + ".bn2", F.conv2d(r, st[p + ".conv2.weight"], None, stride, 1)))
            r = _bn(st, p + ".bn3", F.conv2d(r, st[p + ".conv3.weight"]))
            idn = _bn(st, p + ".downsample.1", F.conv2d(y, st[p + ".downsample.0.weight"], None, stride)) if i == 0 else y
            if branch is not None:
                branch.append(float(r.norm() / idn.norm()))
            y = F.relu(r + idn)
        if name != "layer1":
            feats.append(y)
    o1, o2, o3 = (_conv_bn(st, f"fpn.output{k + 1}", f) for k, f in enumerate(feats))
    o2 = _conv_bn(st, "fpn.merge2", o2 + F.interpolate(o3, size=[o2.size(2), o2.size(3)], mode="nearest"))
    o1 = _conv_bn(st, "fpn.merge1", o1 + F.interpolate(o2, size=[o1.size(2), o1.size(3)], mode="nearest"))
    outs = {"loc": [], "conf": [], "landms": []}
    for k, f in enumerate((o1, o2, o3)):
        p = f"ssh{k + 1}"
        c5 = _conv_bn(st, p + ".conv5X5_1", f)
        s = F.relu(torch.cat([_conv_bn(st, p + ".conv3X3", f, relu=False), _conv_bn(st, p + ".conv5X5_2", c5, relu=False),
                              _conv_bn(st, p + ".conv7x7_3", _conv_bn(st, p + ".conv7X7_2", c5), relu=False)], 1))
        for key, head, d in (("loc", "BboxHead", 4), ("conf", "ClassHead", 2), ("landms", "LandmarkHead", 10)):
            h = F.conv2d(s, st[f"{head}.{k}.conv1x1.weight"], st[f"{head}.{k}.conv1x1.bias"])
            outs[key].append(h.permute(0, 2, 3, 1).reshape(h.shape[0], -1, d))
    loc, conf, landms = (torch.cat(outs[k], 1) for k in ("loc", "conf", "landms"))
    return loc, F.softmax(conf, dim=-1), landms


def prior_box(h: int, w: int) -> torch.Tensor:
    """PriorBox(cfg_re50, (h, w)).forward(): [P, 4] (cx, cy, s_kx, s_ky), Python floats rounded to float32."""
    anchors = []
    for k, step in enumerate(STEPS):
        fh, fw = -(-h // step), -(-w // step)
        for i in range(fh):
            for j in range(fw):
                for ms in MIN_SIZES[k]:
                    anchors += [(j + 0.5) * step / w, (i + 0.5) * step / h, ms / w, ms / h]
    return torch.tensor(anchors, dtype=torch.float32).view(-1, 4)


def decode(loc: torch.Tensor, priors: torch.Tensor) -> torch.Tensor:
    v0, v1 = VARIANCE
    boxes = torch.cat((priors[:, :2] + loc[:, :2] * v0 * priors[:, 2:], priors[:, 2:] * torch.exp(loc[:, 2:] * v1)), 1)
    boxes[:, :2] -= boxes[:, 2:] / 2
    boxes[:, 2:] += boxes[:, :2]
    return boxes


def decode_landm(pre: torch.Tensor, priors: torch.Tensor) -> torch.Tensor:
    v0 = VARIANCE[0]
    return torch.cat([priors[:, :2] + pre[:, 2 * k:2 * k + 2] * v0 * priors[:, 2:] for k in range(5)], dim=1)


def nms(dets: np.ndarray, thresh: float) -> list:
    """py_cpu_nms on float32 dets [N, 5] with the order fixed: descending score, ties in ascending row index."""
    x1, y1, x2, y2, scores = (dets[:, i] for i in range(5))
    areas = (x2 - x1 + 1) * (y2 - y1 + 1)
    order = np.argsort(-scores, kind="stable")
    keep = []
    while order.size > 0:
        i = order[0]
        keep.append(int(i))
        xx1 = np.maximum(x1[i], x1[order[1:]])
        yy1 = np.maximum(y1[i], y1[order[1:]])
        xx2 = np.minimum(x2[i], x2[order[1:]])
        yy2 = np.minimum(y2[i], y2[order[1:]])
        ww = np.maximum(0.0, xx2 - xx1 + 1)
        hh = np.maximum(0.0, yy2 - yy1 + 1)
        inter = ww * hh
        ovr = inter / (areas[i] + areas[order[1:]] - inter)
        order = order[np.where(ovr <= thresh)[0] + 1]
    return keep


def select(boxes: np.ndarray, landms: np.ndarray, scores: np.ndarray, confidence_threshold=0.9, nms_threshold=0.4,
           top_k=5000, keep_top_k=750):
    """RetinaFaceDetection.detect after the decode: threshold, sort (stable), top_k, NMS, keep_top_k, landmark reorder."""
    inds = np.where(scores > confidence_threshold)[0]
    boxes, landms, scores = boxes[inds], landms[inds], scores[inds]
    order = np.argsort(-scores, kind="stable")[:top_k]
    boxes, landms, scores = boxes[order], landms[order], scores[order]
    dets = np.hstack((boxes, scores[:, np.newaxis])).astype(np.float32, copy=False)
    keep = nms(dets, nms_threshold)
    dets, landms = dets[keep, :][:keep_top_k, :], landms[keep][:keep_top_k, :]
    landms = landms.reshape((-1, 5, 2)).transpose((0, 2, 1)).reshape(-1, 10)
    return dets, landms


def decoded(st: dict, img_raw: np.ndarray, resize=1):
    """detect()'s host steps, forward and decode for an image whose longest side is <= 1500: (boxes, landms, scores) numpy
    and the module outputs."""
    img = np.float32(img_raw)
    h, w = img.shape[:2]
    img -= (104, 117, 123)
    x = torch.from_numpy(img.transpose(2, 0, 1).copy()).unsqueeze(0)
    loc, conf, landms = forward(st, x)
    priors = prior_box(h, w)
    scale = torch.tensor([w, h, w, h], dtype=torch.float32)
    boxes = (decode(loc[0], priors) * scale / resize).numpy()
    lm = (decode_landm(landms[0], priors) * torch.tensor([w, h] * 5, dtype=torch.float32) / resize).numpy()
    return boxes, lm, conf[0, :, 1].numpy(), (loc, conf, landms)


def detect(st: dict, img_raw: np.ndarray, resize=1, confidence_threshold=0.9, nms_threshold=0.4, top_k=5000, keep_top_k=750):
    boxes, lm, scores, _ = decoded(st, img_raw, resize)
    return select(boxes, lm, scores, confidence_threshold, nms_threshold, top_k, keep_top_k)


def case_image(h: int, w: int, seed: int) -> np.ndarray:
    """Seeded structured uint8 BGR image [h, w, 3]: smooth blobs on a gradient, with noise."""
    g = np.random.default_rng(seed)
    yy, xx = np.mgrid[0:h, 0:w].astype(np.float64)
    img = np.zeros((h, w, 3))
    for c in range(3):
        img[..., c] = 60 + 80 * (xx / w) * (c + 1) / 3 + 40 * (yy / h)
    for _ in range(6):
        cy, cx, r = g.uniform(0, h), g.uniform(0, w), g.uniform(0.05, 0.25) * min(h, w)
        col = g.uniform(0, 255, 3)
        m = np.exp(-((yy - cy) ** 2 + (xx - cx) ** 2) / (2 * r * r))[..., None]
        img = img * (1 - m) + col * m
    img += g.normal(0, 6, img.shape)
    return np.clip(np.rint(img), 0, 255).astype(np.uint8)
