"""Signed distance of points to a triangle mesh on the device, and the FLAME-intersection filter built on it: what
`src/preprocessing/filter_flame_intersections.py` gets from `pysdf.SDF` (DESIGN §23).

`MeshSDF(verts, faces)(points)` = +d inside, -d outside, d the distance to the closest point of the mesh and the side
decided by the generalized winding number (contract: include/gh_rasterizer.h; kernels: csrc/gh_sdf.cu).
`flame_filter_keep` is lines 88 and 104-119 of the script: the mask of Gaussians that `prune_points` keeps, built on
the device with no host copy.

The head mesh rasterized per view, what `src/preprocessing/extract_non_visible_head_scalp.py` gets from pytorch3d's
`MeshRasterizer` (DESIGN §24): `rasterize_faces` (a z-buffered `pix_to_face`), `head_masks` (the script's dilated
hair/body masks) and `scalp_visibility` (its `check_visiblity_of_faces`).  Kernels: csrc/gh_mesh_raster.cu.

Nothing here loads the native library or touches CUDA until it is called.
"""
from __future__ import annotations

import ctypes as C
import math
import warnings

import torch
import torch.nn.functional as Fn

from . import _capi
from ._capi import _ptr, _stream

GH_STATUS_SDF_FACE_INDEX = 4        # include/gh_rasterizer.h
GH_STATUS_RASTER_NEAR = 8
RASTER_ZBUF_BYTES = 1 << 30          # the z-buffer share of rasterize_faces' workspace: it sets the views per chunk


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


def _raster_args(verts, faces, K, R, t, H, W):
    if verts.dim() != 2 or verts.shape[1] != 3 or faces.dim() != 2 or faces.shape[1] != 3:
        raise RuntimeError(f"mesh raster: verts and faces must be (V, 3) and (F, 3), got {tuple(verts.shape)} and "
                           f"{tuple(faces.shape)}")
    if faces.dtype != torch.int32:
        raise RuntimeError(f"expected scalar type Int but found {faces.dtype} for argument 'faces'")
    if verts.shape[0] < 1 or faces.shape[0] < 1:
        raise RuntimeError("mesh raster: the mesh needs at least one vertex and one face")
    B = K.shape[0] if K.dim() == 3 else -1
    for name, x, shape in (("K", K, (B, 3, 3)), ("R", R, (B, 3, 3)), ("t", t, (B, 3))):
        if tuple(x.shape) != shape or B < 1:
            raise RuntimeError(f"mesh raster: '{name}' must have shape (B, {', '.join(map(str, shape[1:]))}) with one "
                               f"B >= 1 for K, R and t, got {tuple(x.shape)}")
    if not (1 <= int(H) <= 8192 and 1 <= int(W) <= 8192):
        raise RuntimeError(f"mesh raster: H and W must lie in [1, 8192], got {H} x {W}")
    if not (verts.is_cuda and faces.is_cuda):
        raise RuntimeError("mesh raster: verts and faces must be CUDA tensors (there is no CPU path)")
    dev = verts.device
    if faces.device != dev:
        raise RuntimeError(f"mesh raster: verts on {dev}, faces on {faces.device}")
    f32 = [_capi._f32(x, n, dev) for x, n in ((verts, "verts"), (K, "K"), (R, "R"), (t, "t"))]
    return dev, B, f32, faces.contiguous()


def _raster(verts, faces, K, R, t, H, W, chunk, head=None, pix_to_face=None, vis_head=None, counts=None):
    """One gh_mesh_raster sweep on the current stream; -> the device status word (not read here)."""
    dev, B, (v, k, r, tt), f = _raster_args(verts, faces, K, R, t, H, W)
    nv, nf = int(v.shape[0]), int(f.shape[0])
    lib = _capi.load()
    nbytes = C.c_size_t()
    _capi.check(lib.gh_mesh_raster_workspace_size(nv, nf, int(H), int(W), int(chunk), C.byref(nbytes)))
    with torch.cuda.device(dev):
        ws = torch.empty(nbytes.value, dtype=torch.uint8, device=dev)
        status = torch.zeros(1, dtype=torch.int32, device=dev)
        c0, c1 = counts if counts is not None else (None, None)
        _capi.check(lib.gh_mesh_raster(nv, nf, _ptr(v), _ptr(f), B, _ptr(k), _ptr(r), _ptr(tt), int(H), int(W),
                                       _ptr(head), _ptr(pix_to_face), _ptr(vis_head), _ptr(c0), _ptr(c1), int(chunk),
                                       _ptr(ws), nbytes.value, _ptr(status), 0, _stream(dev)))
    return status


def _check_status(status: torch.Tensor, who: str, V: int) -> None:
    s = int(status.item())
    if s & GH_STATUS_SDF_FACE_INDEX:
        raise RuntimeError(f"{who}: a face index lies outside [0, {V})")
    if s & GH_STATUS_RASTER_NEAR:
        warnings.warn(f"{who}: a face crosses a camera's z = 0 plane and was skipped (pytorch3d would draw its "
                      "visible part)", RuntimeWarning, stacklevel=3)


def rasterize_faces(verts: torch.Tensor, faces: torch.Tensor, K: torch.Tensor, R: torch.Tensor, t: torch.Tensor,
                    H: int, W: int) -> torch.Tensor:
    """pytorch3d's `MeshRasterizer(...)(mesh, cameras=cameras_from_opencv_projection(R, t, K, (H, W))).pix_to_face`
    with faces_per_pixel = 1 and blur_radius = 0, for B views at once: -> (B, H, W) int32, the covered face of smallest
    perspective-correct depth at each pixel centre (the smallest index on equal depth), -1 where none is.

    verts (V,3) float32, faces (F,3) int32, K (B,3,3), R (B,3,3), t (B,3) float32, all CUDA tensors on one device; the
    OpenCV world-to-camera convention, x_cam = R X + t.  The kernels run on the current stream; the status word is
    read once at the end (one host synchronisation): a face index outside [0, V) raises, and a face that crosses a
    camera's z = 0 plane -- skipped, where pytorch3d would draw its visible part -- warns."""
    _raster_args(verts, faces, K, R, t, H, W)
    B = K.shape[0]
    chunk = max(1, min(B, RASTER_ZBUF_BYTES // (8 * int(H) * int(W))))
    out = torch.empty((B, int(H), int(W)), dtype=torch.int32, device=verts.device)
    status = _raster(verts, faces, K, R, t, H, W, chunk, pix_to_face=out)
    _check_status(status, "rasterize_faces", int(verts.shape[0]))
    return out


def head_masks(hair: torch.Tensor, body: torch.Tensor) -> torch.Tensor:
    """extract_non_visible_head_scalp.py:112-115 and 81 on the device: -> bool (B, H, W), True where the dilated body
    mask is set and the dilated hair mask is not.

    hair, body: uint8 (B, H, W) or (B, H, W, C) images as `cv2.imread` gives them (channel 0 is used, as the script
    uses it).  `cv2.dilate(m, np.ones((5, 5)))` is a 5x5 max filter that ignores pixels beyond the border: here
    `max_pool2d` with its -inf padding, exact on integer images.  `dilate / 255. >= 0.5` is `dilate >= 128`, and
    `clip(body - hair, 0, 1) >= 0.5` is `body and not hair`."""
    def dilated(m, name):
        if m.dtype != torch.uint8 or m.dim() not in (3, 4):
            raise RuntimeError(f"head_masks: '{name}' must be uint8 (B, H, W) or (B, H, W, C), got {m.dtype} "
                               f"{tuple(m.shape)}")
        m = m[..., 0] if m.dim() == 4 else m
        return Fn.max_pool2d(m[:, None].float(), kernel_size=5, stride=1, padding=2)[:, 0] >= 128
    h, b = dilated(hair, "hair"), dilated(body, "body")
    if h.shape != b.shape:
        raise RuntimeError(f"head_masks: hair {tuple(h.shape)} and body {tuple(b.shape)} differ in shape")
    return b & ~h


def scalp_visibility(verts: torch.Tensor, faces: torch.Tensor, K: torch.Tensor, R: torch.Tensor, t: torch.Tensor,
                     head_masks: torch.Tensor, chunk: int = 16, vis_out: torch.Tensor | None = None):
    """`check_visiblity_of_faces` (extract_non_visible_head_scalp.py:51-93) for B views: -> (vis_mask bool (V,),
    vis_maps float32 (V,), vis_maps_head float32 (V,)).

    vis_maps[v] counts the views whose `pix_to_face.unique()[1:]` holds a face of vertex v, vis_maps_head those whose
    `where(head_mask, pix_to_face, -1).unique()[1:]` does (the kernels count them); then the script's expressions,
    `prob_hair = 1 - vis_maps_head / vis_maps` and `vis_mask = (prob_hair > 0.5) | (vis_maps / B < 0.1)`, so a vertex
    no view sees is NaN there and True in vis_mask.  head_masks: bool (B, H, W), one image size for every view, as
    the script rasterizes every view at one size.  Views run `chunk` at a time (a chunk * H * W * 8-byte z-buffer).
    vis_out: an optional bool (B, H, W) CUDA tensor that receives the script's per-view images
    `where(head_mask, pix_to_face, -1) >= 0` from the same pass.  One host synchronisation (the status word)."""
    if head_masks.dtype != torch.bool or head_masks.dim() != 3:
        raise RuntimeError(f"scalp_visibility: head_masks must be bool (B, H, W), got {head_masks.dtype} "
                           f"{tuple(head_masks.shape)}")
    B, H, W = head_masks.shape
    if K.dim() != 3 or K.shape[0] != B:
        raise RuntimeError(f"scalp_visibility: {B} head masks for K of shape {tuple(K.shape)}")
    if head_masks.device != verts.device:
        raise RuntimeError(f"scalp_visibility: head_masks on {head_masks.device}, verts on {verts.device}")
    if vis_out is not None and (vis_out.dtype != torch.bool or tuple(vis_out.shape) != (B, H, W)
                                or vis_out.device != verts.device or not vis_out.is_contiguous()):
        raise RuntimeError(f"scalp_visibility: vis_out must be a contiguous bool {(B, H, W)} tensor on {verts.device}")
    V = int(verts.shape[0])
    counts = torch.empty((2, V), dtype=torch.int32, device=verts.device)
    status = _raster(verts, faces, K, R, t, H, W, min(int(chunk), B) if chunk >= 1 else chunk,
                     head=head_masks.contiguous(), vis_head=vis_out, counts=(counts[0], counts[1]))
    _check_status(status, "scalp_visibility", V)
    vis_maps, vis_maps_head = counts[0].float(), counts[1].float()
    prob_vis_head = vis_maps_head / vis_maps
    prob_hair = 1 - prob_vis_head
    vis_mask = torch.logical_or(prob_hair > 0.5, vis_maps / B < 0.1)
    return vis_mask, vis_maps, vis_maps_head
