"""Exact 3-nearest-neighbour mean squared distance of a point cloud: what `GaussianModel.create_from_pcd`
(src/scene/gaussian_model.py:409) gets from `simple_knn._C.distCUDA2` to size the initial Gaussians.

`mean_dist3(points)[i]` = mean of the three smallest float32 squared distances from point i to the other finite points
(contract: include/gh_rasterizer.h, DESIGN §14).  The Morton order the search walks in comes from `torch.sort` of the
codes that `gh_knn_morton` writes; everything else is csrc/gh_knn.cu.  Nothing here loads the native library or touches
CUDA until the function is called.
"""
from __future__ import annotations

import ctypes as C

import torch

from . import _capi
from ._capi import _ptr, _stream


def mean_dist3(points: torch.Tensor) -> torch.Tensor:
    """(P,3) float32 CUDA tensor -> (P,) float32 on the same device, produced on the current stream without a host
    synchronisation.  +inf where a point has fewer than three finite neighbours, NaN for a point with a non-finite
    coordinate; bit-reproducible."""
    if points.dim() != 2 or points.shape[1] != 3:
        raise RuntimeError(f"distCUDA2: 'points' must have shape (P, 3), got {tuple(points.shape)}")
    if points.dtype != torch.float32:
        raise RuntimeError(f"expected scalar type Float but found {points.dtype} for argument 'points'")
    if not points.is_cuda:
        raise RuntimeError("distCUDA2: 'points' must be a CUDA tensor (there is no CPU path)")
    dev, P = points.device, int(points.shape[0])
    out = torch.empty(P, dtype=torch.float32, device=dev)
    if P == 0:
        return out
    lib = _capi.load()
    pts = points.detach().contiguous()
    nbytes = C.c_size_t()
    _capi.check(lib.gh_knn_workspace_size(P, C.byref(nbytes)))
    with torch.cuda.device(dev):
        ws = torch.empty(nbytes.value, dtype=torch.uint8, device=dev)
        codes = torch.empty(P, dtype=torch.int64, device=dev)
        stream = _stream(dev)
        _capi.check(lib.gh_knn_morton(P, _ptr(pts), _ptr(codes), _ptr(ws), nbytes.value, stream))
        order = torch.sort(codes, stable=True).indices
        _capi.check(lib.gh_knn_mean_dist3(P, _ptr(pts), _ptr(order), _ptr(out), _ptr(ws), nbytes.value, stream))
    return out
