"""ctypes binding of libgh_raster.so (C ABI: include/gh_rasterizer.h).

The library handle, the signature of every symbol, `check()` for its status codes, and the three helpers every
caller uses to hand torch tensors to it: `_f32` (argument check), `_ptr` (device pointer or NULL) and `_stream`
(the current CUDA stream).  Device memory is allocated by the callers.  The library must have been built
(python -m gaussianhaircut_b200.build); a missing library is a hard error, there is no fallback path.
"""
from __future__ import annotations

import ctypes as C
import os
from typing import Optional

import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "lib", "libgh_raster.so")

GH_OK = 0
GH_E_INVALID_ARG = 1
GH_E_NO_COLORS = 2
GH_E_CUDA = 3
GH_E_PREFILTERED = 4

ABI_VERSION = 6

_p = C.c_void_p
_i = C.c_int
_f = C.c_float
_d = C.c_double
_ll = C.c_longlong
_sz = C.c_size_t

# the leading arguments shared by gh_project_forward, gh_project_forward_binned and gh_project_backward
_PROJ_ARGS = [
    _i, _i, _i,                              # P width height
    _p, _p, _p, _p,                          # xyz scaling rotation dirs
    _p, _p,                                  # features_dc features_rest
    _p, _p, _p,                              # opacity label orient_conf
    _p, _p, _p,                              # viewmatrix projmatrix campos
    _f, _f, _f, _i, C.c_uint, _f]            # tan_fovx tan_fovy scale_modifier sh_degree flags det_eps

# the same for the capturable variants: one device pointer to tan(fov / 2) (x, y) instead of the two host floats
_PROJ_ARGS_CAPTURABLE = _PROJ_ARGS[:15] + [_p] + _PROJ_ARGS[17:]

# name -> (restype, argtypes); every symbol declared in include/gh_rasterizer.h
SIGNATURES = {
    "gh_abi_version": (_i, []),
    "gh_num_channels": (_i, []),
    "gh_last_error": (C.c_char_p, []),
    "gh_kernel_launch_count": (C.c_ulonglong, []),
    "gh_stage_timing_enable": (None, [_i]),
    "gh_stage_timing_read": (_i, [C.POINTER(C.c_double), C.POINTER(C.c_ulonglong), _i]),
    "gh_forward_workspace_sizes": (_i, [_i, _i, _i, C.POINTER(_sz), C.POINTER(_sz)]),
    "gh_binning_workspace_size": (_i, [_ll, C.POINTER(_sz)]),
    "gh_backward_det_workspace_size": (_i, [_i, _ll, C.POINTER(_sz)]),
    "gh_forward_preprocess": (_i, [
        _i, _i, _i, _i, _i,                  # P D M width height
        _p, _p, _p, _p, _p,                  # means3D means2D_precomp shs colors_precomp opacities
        _p, _f, _p,                          # scales scale_modifier rotations
        _p, _p,                              # cov3D_precomp conic_precomp
        _p, _p, _p,                          # viewmatrix projmatrix cam_pos
        _f, _f, _i,                          # tan_fovx tan_fovy prefiltered
        _p,                                  # radii
        _p, _p,                              # geom_buffer img_buffer
        _p, _ll,                             # binning_buffer binning_capacity (records)
        C.POINTER(_i), C.POINTER(_i), C.POINTER(_i),   # num_rendered max_tile_len emitted
        _i, _p]),                            # debug stream
    "gh_forward_render": (_i, [
        _i, _i, _i, _p, _p, _p, _p, _p, _p, _i, _i, _i, _p, _i, _p]),     # ... num_rendered max_tile_len emitted ...
    "gh_backward": (_i, [
        _i, _i, _i, _i, _i, _i,              # P D M R width height
        _p,                                  # background
        _p, _p, _p,                          # means3D shs colors_precomp
        _p, _f, _p,                          # scales scale_modifier rotations
        _p, _p,                              # cov3D_precomp conic_precomp
        _p, _p, _p,                          # viewmatrix projmatrix campos
        _f, _f,                              # tan_fovx tan_fovy
        _p,                                  # radii
        _p, _p, _p,                          # geom binning img
        _p,                                  # dL_dpix
        _p, _p, _p, _p,                      # dL_dmean2D dL_dconic dL_dopacity dL_dcolor
        _p, _p, _p, _p, _p,                  # dL_dmean3D dL_dcov3D dL_dsh dL_dscale dL_drot
        _i, _p,                              # debug stream
        _p, _sz]),                           # det_buffer det_bytes (NULL, 0: the fast path)
    "gh_mark_visible": (_i, [_i, _p, _p, _p, _p, _p]),
    "gh_adam_step": (_i, [_i, _p, _p, _p, _p, _p, _p, _d, _d, _f, _i, _p, _p, _p, _p]),
    "gh_image_loss_workspace_size": (_i, [_i, _i, C.POINTER(C.c_size_t)]),
    "gh_allreduce_p2p": (_i, [_p, _p, C.c_ulonglong, _i, _i, C.c_size_t, C.c_size_t, C.c_uint, _p, _p, _p]),
    "gh_image_loss": (_i, [_i, _i, _p, _p, _p, _p, _p, _f, _f, _f, _f, _p, _p, _p, _p, _i]),
    "gh_image_loss_stage": (_i, [_i, _i, _i, C.c_uint, _p, _p, _p, _p, _p, _f, _f, _f, _f, _p, _p, _p, _p, _i]),
    "gh_render_maps": (_i, [_i, _i, _p, _p, _p, _p, _p, _p, _p, _p, _p, _p]),   # W H out_color angle conf_masked render hair head orient orient_vis conf_vis stream
    "gh_eval_metrics_workspace_size": (_i, [_i, _i, C.POINTER(_sz)]),
    "gh_eval_metrics": (_i, [_i, _i, _i, _p, _p, _p, _p, _p, _p, _sz, _p, _p]),   # W H stage out_color gt_image gt_mask gt_angle gt_conf workspace bytes row stream
    "gh_eval_ssim_workspace_size": (_i, [_i, _i, _i, C.POINTER(_sz)]),   # B W H bytes
    "gh_eval_ssim": (_i, [_i, _i, _i, _p, _i, _ll, _p, _i, _ll, _p, _ll, C.c_uint, _p, _ll, _p, _ll, _p, _sz, _i, _p]),
    # B W H img1 dtype1 stride1 img2 dtype2 stride2 mask mask_stride flags ssim ssim_stride psnr psnr_stride workspace bytes debug stream
    "gh_project_workspace_size": (_i, [_i, C.POINTER(C.c_size_t)]),
    "gh_project_forward": (_i, _PROJ_ARGS + [
        _p, _p, _p, _p, _p, _p,              # means2D colors opacities conic cov3D visible
        _p]),                                # stream
    "gh_project_forward_binned": (_i, _PROJ_ARGS + [
        _p, _p, _p, _p, _p, _p,              # means2D colors opacities conic cov3D visible
        _p, _p, _p, _p, _ll,                 # radii geom_buffer img_buffer binning_buffer binning_capacity
        C.POINTER(C.c_int), C.POINTER(C.c_int), C.POINTER(C.c_int),   # num_rendered max_tile_len emitted
        _p]),
    "gh_project_backward": (_i, _PROJ_ARGS + [
        _p,                                  # visible
        _p,                                  # geom_buffer
        _p, _p, _p, _p,                      # dL_dmeans2D dL_dconic dL_dcolors dL_dopacity
        _p, _p, _p, _p, _p, _p,              # d_xyz d_scaling d_rotation d_dirs d_features_dc d_features_rest
        _p, _p, _p, _p, _p,                  # d_opacity d_label d_orient_conf d_means2D d_camera
        _p, _p, _p]),                        # nan_flag workspace stream
    "gh_project_forward_binned_capturable": (_i, _PROJ_ARGS_CAPTURABLE + [
        _p, _p, _p, _p, _p,                  # means2D colors opacities conic visible
        _p, _p, _p, _p, _ll,                 # radii geom_buffer img_buffer binning_buffer capacity
        _p, _p, _i, _p]),                    # status num_rendered debug stream
    "gh_forward_render_capturable": (_i, [_i, _i, _i, _ll, _p, _p, _p, _p, _p, _p, _i, _p]),
    "gh_backward_capturable": (_i, [_i, _i, _i, _ll, _p, _p, _p, _p, _p, _p, _p, _i, _p, _p, _sz]),
    "gh_project_backward_capturable": (_i, _PROJ_ARGS_CAPTURABLE + [
        _p, _p,                              # visible geom_buffer
        _p, _p, _p, _p,                      # dL_dmeans2D dL_dconic dL_dcolors dL_dopacity
        _p, _p, _p, _p, _p, _p,              # d_xyz d_scaling d_rotation d_dirs d_features_dc d_features_rest
        _p, _p, _p, _p, _p,                  # d_opacity d_label d_orient_conf d_means2D d_camera
        _p, _p, _i, _p]),                    # nan_flag workspace debug stream
    "gh_adam_step_capturable": (_i, [_i, _p, _p, _p, _p, _p, _p, _d, _d, _f, _p, _p, _p, _i, _p]),
    "gh_hair_strands_forward_binned_capturable": (_i, [
        _i, _i, _i, _i, _i,                  # n_head S L width height
        _p, _p, _p, _p, _p, _p,              # head: xyz scaling rotation features_dc features_rest opacity
        C.c_uint, _f,                        # head_flags head_det_eps
        _p, _p, _p, _p, _p, _p,              # origins dirs scale features_dc features_rest orient_conf
        C.c_uint, _f,                        # flags det_eps
        _p, _p, _p, _p, _f, _i,              # viewmatrix projmatrix campos tan_fov scale_modifier sh_degree
        _p,                                  # midpoints
        _p, _p, _p, _p, _p,                  # means2D colors opacities conic visible
        _p, _p, _p, _p, _ll,                 # radii geom_buffer img_buffer binning_buffer capacity
        _p, _p, _i, _p]),                    # status num_rendered debug stream
    "gh_hair_strands_backward_capturable": (_i, [
        _i, _i, _i, _i, _i,                  # n_head S L width height
        _p, _p, _p, _p, _p, _p,              # midpoints dirs scale features_dc features_rest orient_conf
        C.c_uint, _f,                        # flags det_eps
        _p, _p, _p, _p, _f, _i,              # viewmatrix projmatrix campos tan_fov scale_modifier sh_degree
        _p, _p,                              # visible geom_buffer
        _p, _p, _p, _p, _p,                  # d_xyz d_dirs d_features_dc d_features_rest d_orient_conf
        _p, _i, _p]),                        # nan_flag debug stream
    "gh_hair_segments_forward_binned_capturable": (_i, [
        _i, _i, _i, _i,                      # n_head N width height
        _p, _p, _p, _p, _p, _p,              # head: xyz scaling rotation features_dc features_rest opacity
        C.c_uint, _f,                        # head_flags head_det_eps
        _p, _p, _p, _p, _p, _p,              # xyz dirs scale features_dc features_rest orient_conf
        C.c_uint, _f,                        # flags det_eps
        _p, _p, _p, _p, _f, _i,              # viewmatrix projmatrix campos tan_fov scale_modifier sh_degree
        _p, _p, _p, _p, _p,                  # means2D colors opacities conic visible
        _p, _p, _p, _p, _ll,                 # radii geom_buffer img_buffer binning_buffer capacity
        _p, _p, _i, _p]),                    # status num_rendered debug stream
    "gh_hair_segments_backward_capturable": (_i, [
        _i, _i, _i, _i,                      # n_head N width height
        _p, _p, _p, _p, _p, _p,              # xyz dirs scale features_dc features_rest orient_conf
        C.c_uint, _f,                        # flags det_eps
        _p, _p, _p, _p, _f, _i,              # viewmatrix projmatrix campos tan_fov scale_modifier sh_degree
        _p, _p,                              # visible geom_buffer
        _p, _p, _p, _p, _p,                  # d_xyz d_dirs d_features_dc d_features_rest d_orient_conf
        _p, _i, _p]),                        # nan_flag debug stream
    "gh_strand_midpoints": (_i, [_i, _i, _p, _p, _p, _p]),          # S L origins dirs xyz stream
    "gh_strand_backward": (_i, [_i, _i, _p, _p, _p, _p]),           # S L d_xyz d_dirs nan_flag stream
    "gh_densify_classify": (_i, [_i, _p, _p, _p, _p, _f, _f, _f, _f, _p, _p]),
    "gh_densify_scatter": (_i, [_i, _i, _p, _p, _p, _p, _p, _p, _p, _i, _i, _i, _p, _p, _i, _i, _i, _p, _i, _p]),
    "gh_debug_export": (_i, [_i, _i, _i, _ll, _p, _p, _p, _p, _p, _p, _p, _p, _p, _p, _p, _p]),
    "gh_knn_workspace_size": (_i, [_ll, C.POINTER(_sz)]),
    "gh_knn_morton": (_i, [_ll, _p, _p, _p, _sz, _p]),                # P points codes workspace bytes stream
    "gh_knn_mean_dist3": (_i, [_ll, _p, _p, _p, _p, _sz, _p]),        # P points order out workspace bytes stream
    "gh_orient_workspace_size": (_i, [_i, _i, _i, _i, _i, C.POINTER(_sz)]),   # H W N K num_filters bytes
    "gh_orient_dog": (_i, [_i, _i, _i, _p, _p, _i, _p, _i, _p, _p, _sz, _p]),  # H W C image w_low r_low w_high r_high dog ws bytes stream
    "gh_orient_gabor": (_i, [_i, _i, _p, _i, _i, _i, _p, _p, _p, _p, _sz, _p]),  # H W bank N K nf thetas orients var ws bytes stream
    "gh_camera_forward": (_i, [_i, _p, _p, _p, _p, _p, _p, _p, _p, _i, _p]),   # n residuals base index view proj campos tan status debug stream
    "gh_camera_backward": (_i, [_i, _p, _p, _p, _i, _p, _p, _p, _p, _p, _i, _p]),   # n residuals base index intrinsics d_camera grad touched nan status debug stream
    "gh_camera_adam_step": (_i, [_i, _i, _p, _p, _p, _p, _p, _p, _p, _d, _d, _f, _p, _p, _i, _p]),   # n intrinsics r grad touched m v steps lrs b1 b2 eps nan skip debug stream
}

_lib = None


class GhError(RuntimeError):
    """Raised for any non-zero status of the native library (the reference raises RuntimeError from
    AT_ERROR / std::runtime_error at the same places)."""

    def __init__(self, code: int, message: str):
        super().__init__(message)
        self.code = code


def load() -> C.CDLL:
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.isfile(LIB_PATH):
        raise RuntimeError(
            f"gaussianhaircut_b200: native library not found at {LIB_PATH}. "
            "Build it with `python -m gaussianhaircut_b200.build` (needs nvcc; there is no CPU fallback).")
    lib = C.CDLL(LIB_PATH)
    for name, (res, args) in SIGNATURES.items():
        fn = getattr(lib, name)  # AttributeError if the symbol is missing: fail loudly
        fn.restype = res
        fn.argtypes = args
    if lib.gh_abi_version() != ABI_VERSION:
        raise RuntimeError(f"libgh_raster.so ABI {lib.gh_abi_version()} != binding ABI {ABI_VERSION}; rebuild")
    _lib = lib
    return lib


STAGE_NAMES = ("preprocess", "tile_scan", "emit", "tile_sort", "blend_forward", "blend_backward",
               "preprocess_backward")


def stage_timing_read():
    """{stage: (total_ms, calls)} accumulated since gh_stage_timing_enable(1)."""
    lib = load()
    n = len(STAGE_NAMES)
    ms = (C.c_double * n)()
    calls = (C.c_ulonglong * n)()
    lib.gh_stage_timing_read(ms, calls, n)
    return {STAGE_NAMES[i]: (ms[i], int(calls[i])) for i in range(n)}


def check(status: int) -> None:
    if status != GH_OK:
        msg = load().gh_last_error().decode("utf-8", "replace")
        raise GhError(status, msg or f"libgh_raster error {status}")


def _ptr(t: Optional[torch.Tensor]):
    """Device pointer of `t`, or NULL for an absent argument: None or an empty tensor (reference __init__.py:210-222)."""
    if t is None or t.numel() == 0:
        return None
    return C.c_void_p(t.data_ptr())


def _stream(device: torch.device):
    return C.c_void_p(torch.cuda.current_stream(device).cuda_stream)


def _f32(t: Optional[torch.Tensor], name: str, device: torch.device, align: int = 4) -> Optional[torch.Tensor]:
    """`t` as a detached contiguous float32 tensor on `device` whose data pointer is `align`-byte aligned (cloned if it
    is not), like `.contiguous().data<float>()` in the reference binding.  An absent argument (None or an empty tensor,
    on any device) is returned as it is."""
    if t is None or t.numel() == 0:
        return t
    if not t.is_cuda:
        raise RuntimeError(f"gaussianhaircut_b200: '{name}' must be a CUDA tensor (there is no CPU path)")
    if t.dtype != torch.float32:
        raise RuntimeError(f"expected scalar type Float but found {t.dtype} for argument '{name}'")
    if t.device != device:
        raise RuntimeError(f"argument '{name}' is on {t.device}, expected {device}")
    if t.requires_grad:
        t = t.detach()
    t = t.contiguous()
    if t.data_ptr() % align:
        t = t.clone()
    return t
