"""ctypes binding of libe4s_b200.so (the C ABI declared in include/e4s_b200.h).

There is NO fallback: if the shared library is missing or the device is not an sm_90 (H100-class) GPU the
import / call fails loudly.  Build with ``python -m e4s_b200.build`` (or ``__graft_entry__.build()``).
"""
from __future__ import annotations

import ctypes
import os
from ctypes import c_char_p, c_float, c_int, c_int64, c_void_p

import torch

_PKG = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("E4S_B200_LIB") or os.path.join(_PKG, "libe4s_b200.so")   # env: an alternative build of the library

_ERR = {-1: "E4S_ERR_ARG (null pointer / bad size)", -2: "E4S_ERR_SHAPE (unsupported shape)",
        -3: "E4S_ERR_ALIGN (pointer not 16-byte aligned)", -4: "E4S_ERR_NOT_ONEHOT", -5: "E4S_ERR_ARCH (device is not sm_90)"}

# name -> argtypes; every function returns int.  Kept in one table so tests can check that the
# library exports exactly what include/e4s_b200.h declares.
P = c_void_p
SIGNATURES = {
    "e4s_upfirdn2d_f32": [P, P, P] + [c_int] * 15 + [P],
    "e4s_bias_act_fwd_f32": [P, P, P, c_int64, c_int, c_int, c_float, c_float, P],
    "e4s_bias_act_bwd_f32": [P, P, P, c_int64, c_float, c_float, P],
    "e4s_bias_grad_f32": [P, P, c_int64, c_int, c_int, P],
    "e4s_onehot_to_label_u8": [P, P, P, c_int, c_int, c_int, c_int, P],
    "e4s_label_to_onehot_f32": [P, P, c_int, c_int, c_int, c_int, P],
    "e4s_label_resize_nearest_u8": [P, P, c_int, c_int, c_int, c_int, c_int, P],
    "e4s_label_remap_u8": [P, P, P, c_int64, P],
    "e4s_swap_head_mask_u8": [P, P, P, P, P, c_int64, c_int, P],
    "e4s_mask_box_morph_u8": [P, P, c_int, c_int, c_int, c_int, c_int, P],
    "e4s_box_morph_f32": [P, P, c_int, c_int, c_int, c_int, c_int, c_float, P],
    "e4s_region_mean_f32": [P, P, P, P, c_int, c_int, c_int, c_int, c_int, P],
    "e4s_demod_f32": [P, P, P, c_int, c_int, c_int, c_float, P],
    "e4s_demod_gemm_f32": [P, P, P, c_int, c_int, c_int, c_float, P, P],
    "e4s_modconv3x3_fwd_f32": [P] * 9 + [c_int] * 9 + [P],
    "e4s_modconv3x3_tcr_fwd": [P] * 9 + [c_int] * 9 + [P],
    "e4s_modconv3x3_up_tcr_fwd": [P] * 10 + [c_int] * 7 + [P],
    "e4s_modconv3x3_up_masked_tcr_fwd": [P] * 16 + [c_int] * 9 + [P],
    "e4s_conv3x3_tcr_f32": [P] * 6 + [c_int] * 7 + [P],
    "e4s_conv3x3_bias_tcr_f32": [P] * 7 + [c_int] * 8 + [P],
    "e4s_conv3x3_dense_tcr_f32": [P, c_int, P, P, c_float, P, c_float, P, P] + [c_int] * 7 + [c_float, P],
    "e4s_conv3x3_rgb_f32": [P, c_int, P, P, P] + [c_int] * 6 + [P],
    "e4s_bicubic_down_norm_f32": [P] * 5 + [c_int] * 4 + [P],
    "e4s_parser_stem_f32": [P] * 4 + [c_int] * 3 + [P],
    "e4s_parse_head_u8": [P] * 5 + [c_int] * 7 + [P],
    "e4s_channel_mean_f32": [P, P, c_int, c_int, c_int, P],
    "e4s_space_to_depth_f32": [P, P] + [c_int] * 4 + [P],
    "e4s_set_deterministic": [c_int],
    "e4s_instnorm_affine_f32": [P] * 4 + [c_int] * 4 + [c_float, P],
    "e4s_norm_residual_f32": [P, P, P, c_float, P, P, P, c_int, P, P] + [c_int] * 4 + [P],
    "e4s_modconv3x3_bwd_f32": [P] * 9 + [c_int] * 8 + [P],
    "e4s_modconv3x3_bwd_tc": [P] * 9 + [c_int] * 8 + [P],
    "e4s_modconv3x3_bwd_tc_plan": [c_int] * 6 + [P, P, P],
    "e4s_modconv3x3_tcr_fwd_plan": [c_int] * 4 + [P],
    "e4s_class_reduce_f32": [P] * 7 + [c_int] * 7 + [P],
    "e4s_torgb_bwd_f32": [P] * 7 + [c_int] * 5 + [P],
    "e4s_torgb_fwd_f32": [P] * 8 + [c_int] * 5 + [P],
    "e4s_linear_f32": [P, P, P, P, c_int, c_int, c_int, c_int, c_int64, c_int64, c_int64, c_int64, c_int, c_float, P, P],
    "e4s_linear_multi_f32": [P, c_int, P],
    "e4s_avgpool_pyramid_f32": [P, P, P, c_int64, c_int, c_int, P],
    "e4s_avgpool_pyramid_bwd_f32": [P, P, P, P, c_int64, c_int, c_int, P],
    "e4s_planar_to_pixel_f32": [P, P, c_int, c_int, c_int, c_int, P],
    "e4s_pixel_to_planar_f32": [P, P, c_int, c_int, c_int, c_int, P],
}
PLAIN = {"e4s_linear_workspace_floats": ([c_int, c_int, c_int, c_int], c_int64), "e4s_get_deterministic": ([], c_int), "e4s_version": ([], c_int), "e4s_build_arch": ([], c_char_p), "e4s_device_ok": ([], c_int)}



class LinearProblem(ctypes.Structure):
    """E4sLinearProblem of include/e4s_b200.h."""
    _fields_ = [("x", c_void_p), ("w", c_void_p), ("bias", c_void_p), ("y", c_void_p), ("m", c_int), ("n", c_int), ("k", c_int),
                ("ldx", c_int), ("rsqrt_eps", c_float), ("reserved", c_int)]


_lib = None


def load() -> ctypes.CDLL:
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise ImportError(
            f"{LIB_PATH} is missing: the e4s_b200 CUDA extension is not built. Run `python -m e4s_b200.build` "
            "(needs nvcc; cross-compiles for sm_90a without a GPU). There is no CPU/PyTorch fallback.")
    lib = ctypes.CDLL(LIB_PATH)
    for name, args in SIGNATURES.items():
        fn = getattr(lib, name)
        fn.argtypes, fn.restype = args, c_int
    for name, (args, res) in PLAIN.items():
        fn = getattr(lib, name)
        fn.argtypes, fn.restype = args, res
    _lib = lib
    return lib


def exported_symbols():
    return sorted(list(SIGNATURES) + list(PLAIN))


def check(rc: int, name: str) -> None:
    if rc == 0:
        return
    if rc < 0:
        raise RuntimeError(f"{name} failed: {_ERR.get(rc, rc)}")
    raise RuntimeError(f"{name} failed: CUDA error {rc}")


def stream_ptr() -> c_void_p:
    return c_void_p(torch.cuda.current_stream().cuda_stream)


def ptr(t):
    """Device pointer of a tensor (or NULL for None)."""
    return c_void_p(0) if t is None else c_void_p(t.data_ptr())


def require_cuda(t: torch.Tensor, what: str = "input") -> None:
    # same failure the reference's pybind layer produces (fused_bias_act.cpp:13, upfirdn2d.cpp:15)
    if not t.is_cuda:
        raise RuntimeError(f"{what} must be a CUDA tensor")


_device_checked = set()


def ensure_device(t: torch.Tensor) -> None:
    idx = t.device.index if t.device.index is not None else torch.cuda.current_device()
    if idx in _device_checked:
        return
    with torch.cuda.device(idx):
        check(load().e4s_device_ok(), "e4s_device_ok")
    _device_checked.add(idx)
