"""Signed distance of points to a triangle mesh on the device, and the FLAME-intersection filter built on it: what
`src/preprocessing/filter_flame_intersections.py` gets from `pysdf.SDF` (DESIGN §23).

`MeshSDF(verts, faces)(points)` = +d inside, -d outside, d the distance to the closest point of the mesh and the side
decided by the generalized winding number (contract: include/gh_rasterizer.h; kernels: csrc/gh_sdf.cu).
`flame_filter_keep` is lines 88 and 104-119 of the script: the mask of Gaussians that `prune_points` keeps, built on
the device with no host copy.  Nothing here loads the native library or touches CUDA until it is called.
"""
from __future__ import annotations

import ctypes as C
import math

import torch

from . import _capi
from ._capi import _ptr, _stream

GH_STATUS_SDF_FACE_INDEX = 4        # include/gh_rasterizer.h


class MeshSDF:
    """A triangle mesh prepared once for signed-distance queries.

    verts (V,3) float32 and faces (F,3) int32 CUDA tensors on one device.  The constructor writes one record per face
    into a workspace it keeps, and checks the face indices once (one host synchronisation): an index outside [0, V)
    raises.  The mesh tensors are not kept; changing them later does not change the prepared mesh."""

    def __init__(self, verts: torch.Tensor, faces: torch.Tensor):
        if verts.dim() != 2 or verts.shape[1] != 3 or faces.dim() != 2 or faces.shape[1] != 3:
            raise RuntimeError(f"MeshSDF: verts and faces must be (V, 3) and (F, 3), got {tuple(verts.shape)} and "
                               f"{tuple(faces.shape)}")
        if verts.dtype != torch.float32:
            raise RuntimeError(f"expected scalar type Float but found {verts.dtype} for argument 'verts'")
        if faces.dtype != torch.int32:
            raise RuntimeError(f"expected scalar type Int but found {faces.dtype} for argument 'faces'")
        if not (verts.is_cuda and faces.is_cuda):
            raise RuntimeError("MeshSDF: verts and faces must be CUDA tensors (there is no CPU path)")
        if verts.device != faces.device:
            raise RuntimeError(f"MeshSDF: verts on {verts.device}, faces on {faces.device}")
        self.device = verts.device
        self.num_verts, self.num_faces = int(verts.shape[0]), int(faces.shape[0])
        lib = _capi.load()
        nbytes = C.c_size_t()
        _capi.check(lib.gh_sdf_workspace_size(self.num_faces, C.byref(nbytes)))
        v, f = verts.detach().contiguous(), faces.contiguous()
        with torch.cuda.device(self.device):
            self._records = torch.empty(nbytes.value, dtype=torch.uint8, device=self.device)
            status = torch.zeros(1, dtype=torch.int32, device=self.device)
            _capi.check(lib.gh_sdf_prepare(self.num_verts, self.num_faces, _ptr(v), _ptr(f), _ptr(self._records),
                                           nbytes.value, _ptr(status), 0, _stream(self.device)))
            if int(status.item()) & GH_STATUS_SDF_FACE_INDEX:
                raise RuntimeError(f"MeshSDF: a face index lies outside [0, {self.num_verts})")

    def __call__(self, points: torch.Tensor, return_parts: bool = False):
        """(N,3) float32 on the mesh's device -> sdf (N,) float32, produced on the current stream without a host
        synchronisation; with `return_parts`, (sdf, d, w): the distance and the winding number as well.  NaN for a
        point with a non-finite coordinate; bit-reproducible, and a point's result does not depend on the batch."""
        if points.dim() != 2 or points.shape[1] != 3:
            raise RuntimeError(f"MeshSDF: 'points' must have shape (N, 3), got {tuple(points.shape)}")
        if points.dtype != torch.float32:
            raise RuntimeError(f"expected scalar type Float but found {points.dtype} for argument 'points'")
        if points.device != self.device:
            raise RuntimeError(f"MeshSDF: 'points' is on {points.device}, the mesh on {self.device}")
        n = int(points.shape[0])
        p = points.detach().contiguous()
        new = lambda: torch.empty(n, dtype=torch.float32, device=self.device)  # noqa: E731
        sdf = new()
        d, w = (new(), new()) if return_parts else (None, None)
        lib = _capi.load()
        with torch.cuda.device(self.device):
            _capi.check(lib.gh_sdf_query(n, _ptr(p), self.num_faces, _ptr(self._records), self._records.numel(),
                                         _ptr(sdf), _ptr(d), _ptr(w), 0, _stream(self.device)))
        return (sdf, d, w) if return_parts else sdf


def _build_rotation(r: torch.Tensor) -> torch.Tensor:
    """build_rotation (src/utils/general_utils.py:79-109): the quaternion normalised, then R (column layout as there)."""
    norm = torch.sqrt(r[:, 0] * r[:, 0] + r[:, 1] * r[:, 1] + r[:, 2] * r[:, 2] + r[:, 3] * r[:, 3])
    q = r / norm[:, None]
    R = torch.zeros((q.size(0), 3, 3), device=r.device)
    r, x, y, z = q[:, 0], q[:, 1], q[:, 2], q[:, 3]
    R[:, 0, 0] = 1 - 2 * (y * y + z * z)
    R[:, 1, 0] = 2 * (x * y - r * z)
    R[:, 2, 0] = 2 * (x * z + r * y)
    R[:, 0, 1] = 2 * (x * y + r * z)
    R[:, 1, 1] = 1 - 2 * (x * x + z * z)
    R[:, 2, 1] = 2 * (y * z - r * x)
    R[:, 0, 2] = 2 * (x * z - r * y)
    R[:, 1, 2] = 2 * (y * z + r * x)
    R[:, 2, 2] = 1 - 2 * (x * x + y * y)
    return R


def _build_scaling_rotation(s: torch.Tensor, r: torch.Tensor) -> torch.Tensor:
    """build_scaling_rotation (src/utils/general_utils.py:111-120): M = S @ R."""
    S = torch.zeros((s.shape[0], 3, 3), dtype=torch.float, device=s.device)
    S[:, 0, 0] = s[:, 0]
    S[:, 1, 1] = s[:, 1]
    S[:, 2, 2] = s[:, 2]
    return S @ _build_rotation(r)


def icosahedron(device=None) -> torch.Tensor:
    """(12,3) float32: the level-0 icosphere, the vertices (+-1, +-t, 0), (0, +-1, +-t), (+-t, 0, +-1) normalised,
    t the golden ratio.  Their order does not matter to the filter (it reduces with .all over the 12 corners)."""
    t = (1.0 + math.sqrt(5.0)) / 2.0
    v = torch.tensor([[-1, t, 0], [1, t, 0], [-1, -t, 0], [1, -t, 0], [0, -1, t], [0, 1, t], [0, -1, -t], [0, 1, -t],
                      [t, 0, -1], [t, 0, 1], [-t, 0, -1], [-t, 0, 1]], dtype=torch.float64)
    return (v / v.norm(dim=1, keepdim=True)).to(device=device, dtype=torch.float32)


def flame_corners(xyz: torch.Tensor, scaling: torch.Tensor, rotation: torch.Tensor) -> torch.Tensor:
    """(P*12, 3): the icosahedron's vertices on each Gaussian's 3-sigma ellipsoid, with the script's own expressions
    (filter_flame_intersections.py:88, 108): M = build_scaling_rotation(scaling * 3, rotation), v @ M + xyz."""
    M = _build_scaling_rotation(scaling * 3, rotation)
    verts = icosahedron(xyz.device)
    return ((verts[None, :, None, :] @ M[:, None, :, :])[:, :, 0, :] + xyz[:, None]).view(-1, 3)


def flame_filter_keep(xyz: torch.Tensor, scaling: torch.Tensor, rotation: torch.Tensor, label: torch.Tensor,
                      sdf: MeshSDF) -> torch.Tensor:
    """filter_flame_intersections.py:88, 104-119 on the device: -> bool (P,), True for a Gaussian the script keeps --
    all 12 corners outside the mesh (sdf < 0), or label <= 0.5.  xyz, scaling, label: the model's activated get_xyz,
    get_scaling and get_label; rotation: its raw _rotation (the script passes it to build_scaling_rotation as it is).
    Runs on the current stream with no host synchronisation."""
    corners = flame_corners(xyz.detach(), scaling.detach(), rotation.detach())
    outside = (sdf(corners).view(xyz.shape[0], 12) < 0).all(dim=1)
    return torch.logical_or(outside, label.detach().squeeze() <= 0.5)
