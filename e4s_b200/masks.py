"""Region-mask utilities on the GPU, bit-exact (SURVEY.md section 8a last row, section 8f.3).

Second half of the file: the mask stage of scripts/face_swap.py (shape swapping, foreground mask, blending masks) -
`swap_head_mask_revisit_considerGlass`, `dilation`, `erosion`, `create_masks`, `swap_comp_style_vector` keep the
reference's names and signatures.

`labelMap2OneHot` mirrors src/utils/torch_utils.py:166-172.  The 19 -> 12 class conversion of
CelebAMask-HQ labels mirrors __celebAHQ_masks_to_faceParser_mask_detailed, src/datasets/dataset.py:153-209,
which is a pure per-pixel table lookup; the table below restates it.
"""
import torch

from . import kernels as K

# index = CelebAMask-HQ label (0 background, 1 skin, 2 nose, 3 eye_g, 4 l_eye, 5 r_eye, 6 l_brow, 7 r_brow,
# 8 l_ear, 9 r_ear, 10 mouth, 11 u_lip, 12 l_lip, 13 hair, 14 hat, 15 ear_r, 16 neck_l, 17 neck, 18 cloth)
# value = 12-class label (0 background, 1 lip, 2 eyebrows, 3 eyes, 4 hair, 5 nose, 6 skin, 7 ears,
# 8 belowface, 9 mouth, 10 eye_glass, 11 ear_rings)
CELEBA19_TO_12 = [0, 6, 5, 10, 3, 3, 2, 2, 7, 7, 9, 1, 1, 4, 0, 11, 0, 8, 0] + [0] * (256 - 19)
# The same for the 19 classes of the BiSeNet face parser (face-parsing.PyTorch order: 0 background, 1 skin, 2 l_brow,
# 3 r_brow, 4 l_eye, 5 r_eye, 6 eye_g, 7 l_ear, 8 r_ear, 9 ear_r, 10 nose, 11 mouth, 12 u_lip, 13 l_lip, 14 neck,
# 15 neck_l, 16 cloth, 17 hair, 18 hat): __ffhq_masks_to_faceParser_mask_detailed, src/datasets/dataset.py:60-108.
FFHQ19_TO_12 = [0, 6, 2, 2, 3, 3, 10, 7, 7, 11, 5, 9, 1, 1, 8, 0, 0, 4, 0] + [0] * (256 - 19)


def labelMap2OneHot(label, num_cls):
    """[B, 1, H, W] integer label map -> [B, num_cls, H, W] float one-hot."""
    return K.label_to_onehot(label, num_cls)


def celeba19_to_12(label_u8: torch.Tensor) -> torch.Tensor:
    lut = torch.tensor(CELEBA19_TO_12, dtype=torch.uint8, device=label_u8.device)
    return K.label_remap(label_u8.to(torch.uint8), lut)


def ffhq19_to_12(label_u8: torch.Tensor) -> torch.Tensor:
    lut = torch.tensor(FFHQ19_TO_12, dtype=torch.uint8, device=label_u8.device)
    return K.label_remap(label_u8.to(torch.uint8), lut)


# ------------------------------------------------------------------------------------------------------------------
# Mask stage of the face-swapping pipeline (scripts/face_swap.py steps 4 and 6) on the GPU, bit-exact.
def swap_head_mask_revisit_considerGlass(source, target, hair_first=True):
    """Drop-in for src/utils/swap_face_mask.py:33-83.  `source` / `target`: 12-class label maps, numpy arrays (as the
    reference passes them; the result comes back as numpy arrays of the target's dtype) or CUDA tensors (results stay on
    the device as uint8).  Returns (swapped label map, hole map in {0, 255})."""
    res, hole, _ = _swap(source, target, hair_first)
    return res, hole


def swap_head_mask_with_foreground(source, target, hair_first=True):
    """The same launch also yields the foreground mask scripts/face_swap.py:280-284 derives from the two results
    (labels outside {0, 11, 4}, plus every hole), as 0/1."""
    return _swap(source, target, hair_first)


def _swap(source, target, hair_first):
    import numpy as np
    as_numpy = isinstance(target, np.ndarray)
    if as_numpy:
        dev = torch.device("cuda", torch.cuda.current_device())
        s = torch.from_numpy(np.ascontiguousarray(source).astype(np.uint8)).to(dev)
        t = torch.from_numpy(np.ascontiguousarray(target).astype(np.uint8)).to(dev)
    else:
        s, t = source, target
    res, hole, fg = K.swap_head_mask(s, t, hair_first)
    if as_numpy:
        return tuple(x.cpu().numpy().astype(target.dtype) for x in (res, hole, fg))
    return res, hole, fg


def _flat_box_radius(kernel: torch.Tensor, structuring_element, origin, border_type, what: str) -> int:
    # the reference's general grey-scale morphology (src/utils/morphology.py) is only ever called with a full square
    # of ones, the default origin and the geodesic border (scripts/face_swap.py:34-42): that is what the kernel does
    if not isinstance(kernel, torch.Tensor):
        raise TypeError(f"Kernel type is not a torch.Tensor. Got {type(kernel)}")
    if len(kernel.shape) != 2:
        raise ValueError(f"Kernel size must have 2 dimensions. Got {kernel.dim()}")
    kh, kw = kernel.shape
    if kh != kw or kh % 2 == 0 or structuring_element is not None or origin is not None or border_type != "geodesic":
        raise NotImplementedError(f"{what}: only a flat odd square structuring element with the default origin and the "
                                  "geodesic border is implemented")
    if not bool((kernel != 0).all()):
        raise NotImplementedError(f"{what}: the structuring element must be all ones")
    return kh // 2


def dilation(tensor, kernel, structuring_element=None, origin=None, border_type="geodesic", border_value=0.0,
             max_val=1e4, engine="unfold"):
    """src/utils/morphology.py:23-106 for [B, C, H, W] float (or uint8) images and a flat box element; both engines of the
    reference compute the same values, so `engine` is accepted and ignored."""
    if not isinstance(tensor, torch.Tensor):
        raise TypeError(f"Input type is not a torch.Tensor. Got {type(tensor)}")
    if len(tensor.shape) != 4:
        raise ValueError(f"Input size must have 4 dimensions. Got {tensor.dim()}")
    r = _flat_box_radius(kernel, structuring_element, origin, border_type, "dilation")
    return K.mask_box_morph(tensor, r, erode=False, max_val=max_val).view_as(tensor)


def erosion(tensor, kernel, structuring_element=None, origin=None, border_type="geodesic", border_value=0.0,
            max_val=1e4, engine="unfold"):
    """src/utils/morphology.py:109-197, same restrictions as `dilation`."""
    if not isinstance(tensor, torch.Tensor):
        raise TypeError(f"Input type is not a torch.Tensor. Got {type(tensor)}")
    if len(tensor.shape) != 4:
        raise ValueError(f"Input size must have 4 dimensions. Got {tensor.dim()}")
    r = _flat_box_radius(kernel, structuring_element, origin, border_type, "erosion")
    return K.mask_box_morph(tensor, r, erode=True, max_val=max_val).view_as(tensor)


def create_masks(mask, outer_dilation=0, operation="dilation"):
    """scripts/face_swap.py:30-48: (content, border, full) blending masks of a [B, 1, H, W] 0/1 mask."""
    radius = outer_dilation
    ones = torch.ones(2 * radius + 1, 2 * radius + 1, device=mask.device)
    if operation == "dilation":
        full_mask = dilation(mask, ones, engine="convolution")
        border_mask = full_mask - mask
    elif operation == "erosion":
        full_mask = erosion(mask, ones, engine="convolution")
        border_mask = mask - full_mask
    elif operation == "expansion":          # a boundary that expands to both sides
        full_mask = dilation(mask, ones, engine="convolution")
        border_mask = full_mask - erosion(mask, ones, engine="convolution")
    else:
        raise ValueError(f"unknown operation {operation!r}: 'dilation', 'erosion' or 'expansion'")
    return mask, border_mask.clip(0, 1), full_mask


def swap_comp_style_vector(style_vectors1, style_vectors2, comp_indices=(), belowFace_interpolation=False):
    """scripts/face_swap.py:117-146 for a BATCH of faces and without the two host synchronisations of its
    `if torch.sum(...) == 0` tests: the empty-region decisions (no ear / no teeth region in the source) are taken per
    sample on the device with `torch.where`.  For one face ([1, ncls, C], the reference's case) the result is identical."""
    assert comp_indices is not None
    out = style_vectors1.clone()
    idx = list(comp_indices)
    if idx:
        out[:, idx, :] = style_vectors2[:, idx, :]
    no_ear = style_vectors2[:, 7, :].sum(dim=-1, keepdim=True) == 0
    out[:, 7, :] = torch.where(no_ear, (style_vectors1[:, 7, :] + style_vectors2[:, 7, :]) / 2, out[:, 7, :])
    no_teeth = style_vectors2[:, 9, :].sum(dim=-1, keepdim=True) == 0
    out[:, 9, :] = torch.where(no_teeth, style_vectors1[:, 9, :], out[:, 9, :])
    if belowFace_interpolation:
        out[:, 8, :] = (style_vectors1[:, 8, :] + style_vectors2[:, 8, :]) / 2
    return out
