"""Trainable cameras on the device (DESIGN §17): the reference's BARF camera model and its camera Adam.

The reference trains, for every training view, a se(3) pose residual and a field-of-view residual
(src/scene/cameras.py:95-152 with trainable_cameras = trainable_intrinsics = use_barf = True) with its own
torch.optim.Adam (src/train_gaussians.py:45-63, 183-196).  Its `Camera` properties rebuild the whole model in PyTorch
on every access.  Here a `CameraRig` holds all cameras in four device tables and each view is ONE autograd node whose
forward and backward are the kernels gh_camera_forward / gh_camera_backward (include/gh_rasterizer.h); `CameraAdam`
steps the visited cameras with gh_camera_adam_step.  The kernels never synchronise with the host and every call can be
captured (graphs.CapturedTrainStep(..., cameras=rig, camera_optimizer=CameraAdam(...)): the captured iteration has no
host synchronisation besides its one read of the status word and the losses).  Eagerly, the fused renderer reads a
view's tan(FoV / 2) back to the host once per render (renderer._static: the non-capturable projection takes tan fov as
host arguments), and CameraAdam.step() stages the learning rates through pinned memory without a synchronisation.

    rig = CameraRig.from_cameras(scene.getTrainCameras())       # the reference's Camera objects
    cam_opt = CameraAdam(rig, opt.cam_rotation_lr, opt.cam_translation_lr_init * scale, opt.cam_fov_lr)
    view = rig.view(i)                 # world_view_transform, full_proj_transform, camera_center, tan_fov, ...
    out = renderer.render(view, gaussians, pipe, bg)  ... loss.backward(); cam_opt.step(); cam_opt.zero_grad()
    rig.write_back(scene.getTrainCameras())             # the trained residuals back into the Camera parameters

Only the BARF parameterisation (use_barf=True) is supported.
"""
from __future__ import annotations

from typing import Dict, List, Optional, Sequence

import torch

from . import _capi
from ._capi import _ptr, _stream

__all__ = ["CameraRig", "CameraView", "CameraAdam", "STATUS_CAMERA_INDEX"]

STATUS_CAMERA_INDEX = 2          # GH_STATUS_CAMERA_INDEX
BASE, ROW, DCAMERA = 18, 8, 37   # GH_CAM_BASE, GH_CAM_ROW, GH_CAM_DCAMERA


def _check_barf(cam, intrinsics: bool) -> None:
    name = getattr(cam, "image_name", "?")
    if getattr(cam, "use_barf", True) is False:
        raise ValueError(f"CameraRig: camera '{name}' uses the 6-D ortho2rotation residual (use_barf=False); only the "
                         "BARF se(3) parameterisation (use_barf=True) is supported")
    rot = getattr(cam, "_rotation_res", None)
    if rot is None or getattr(cam, "trainable_cameras", True) is False:
        raise ValueError(f"CameraRig: camera '{name}' has no trainable pose (_rotation_res); trainable intrinsics without "
                         "trainable cameras are not supported (the reference never steps that optimizer)")
    if rot.numel() != 3 or cam._translation_res.numel() != 3:
        raise ValueError(f"CameraRig: camera '{name}': _rotation_res and _translation_res must have 3 elements (use_barf=True)")
    fov = getattr(cam, "_fov_res", None)
    if intrinsics and (fov is None or fov.numel() != 2):
        raise ValueError(f"CameraRig: camera '{name}' has no 2-element _fov_res; pass intrinsics=False")
    if not intrinsics and fov is not None and (getattr(cam, "trainable_intrinsics", False) or bool(fov.detach().any())):
        # the rig would render with the base FoV, the reference Camera with FoV + _fov_res
        raise ValueError(f"CameraRig: camera '{name}' has a trainable or non-zero _fov_res; intrinsics=False would drop "
                         "it (pass intrinsics=True)")


class CameraRig:
    """N trainable cameras on one device.  Tables (device, float32 unless noted):
    `base` (N, 18) = the float32 _colmap_transform (row-major), FoVx, FoVy; `residuals` (N, 8) = _rotation_res,
    _translation_res, _fov_res (the last two stay 0 without `intrinsics`); `grad` (N, 8) = dL/dresiduals accumulated by
    the views' backward; `touched` (N,) int32 = rows with a gradient since the last CameraAdam step.  Also `nan_flag`
    and `status` (int32 (1,) each): the camera NaN verdict and the GH_STATUS_CAMERA_INDEX bit."""

    def __init__(self, base: torch.Tensor, residuals: torch.Tensor, names: Sequence[str], sizes: Sequence[tuple],
                 intrinsics: bool = True):
        n = int(base.shape[0])
        if n <= 0 or base.shape != (n, BASE) or residuals.shape != (n, ROW) or len(names) != n or len(sizes) != n:
            raise ValueError(f"CameraRig: base must be (N, {BASE}), residuals (N, {ROW}), names and sizes N long")
        dev = base.device
        f = dict(dtype=torch.float32, device=dev)
        self.n, self.device, self.intrinsics = n, dev, bool(intrinsics)
        self.names, self.sizes = list(names), [(int(w), int(h)) for w, h in sizes]
        self.base = base.detach().to(**f).contiguous().clone()
        self.residuals = residuals.detach().to(**f).contiguous().clone()
        if not self.intrinsics:
            self.residuals[:, 6:] = 0
        # a leaf that requires grad so that autograd runs the views' backward; its own .grad is never written
        self.residuals.requires_grad_(True)
        self.grad = torch.zeros(n, ROW, **f)
        self.touched = torch.zeros(n, dtype=torch.int32, device=dev)
        self.nan_flag = torch.zeros(1, dtype=torch.int32, device=dev)
        self.status = torch.zeros(1, dtype=torch.int32, device=dev)
        self.indices = torch.arange(n, dtype=torch.int32, device=dev)   # the device index of view i is indices[i]

    @classmethod
    def from_cameras(cls, cameras, intrinsics: bool = True) -> "CameraRig":
        """From the reference's `Camera` objects (cameras.py:21, trainable_cameras and use_barf set) or anything with
        `_colmap_transform`, `_FoVx`, `_FoVy`, `image_width`, `image_height`, `image_name`, `_rotation_res`,
        `_translation_res` and, with `intrinsics`, `_fov_res`."""
        cameras = list(cameras)
        if not cameras:
            raise ValueError("CameraRig.from_cameras: no cameras")
        base, res = [], []
        for cam in cameras:
            _check_barf(cam, intrinsics)
            C = cam._colmap_transform.detach().float().reshape(16)
            fx = torch.as_tensor(cam._FoVx).detach().float().reshape(-1)[:1].to(C.device)
            fy = torch.as_tensor(cam._FoVy).detach().float().reshape(-1)[:1].to(C.device)
            base.append(torch.cat([C, fx, fy]))
            f = cam._fov_res.detach().float().reshape(2) if intrinsics else torch.zeros(2, device=C.device)
            res.append(torch.cat([cam._rotation_res.detach().float().reshape(3), cam._translation_res.detach().float().reshape(3),
                                  f.to(C.device)]))
        return cls(torch.stack(base), torch.stack(res), [c.image_name for c in cameras],
                   [(c.image_width, c.image_height) for c in cameras], intrinsics)

    # ------------------------------------------------------------------------------------------ views
    def view(self, i: int, requires_grad: bool = True) -> "CameraView":
        """Camera i as the reference renderer reads it.  `requires_grad=False`: the frozen form (stages 2 and 3,
        evaluation).  A view evaluates the residuals once, on first use: take a new view after an optimizer step."""
        i = int(i)
        if not 0 <= i < self.n:
            raise IndexError(f"CameraRig.view: index {i} outside [0, {self.n})")
        return CameraView(self, i, requires_grad)

    def _lib(self):
        if not self.device.type == "cuda":
            raise RuntimeError("CameraRig: the camera kernels need the rig's tables on a CUDA device (there is no CPU path)")
        return _capi.load()

    def forward(self, index: torch.Tensor, out: Optional[torch.Tensor] = None, status: Optional[torch.Tensor] = None):
        """gh_camera_forward for the camera at the device int32 `index` (1,) -> the (37,) output buffer `out` (allocated
        when None): viewmatrix (16), projmatrix (16), campos (3), tan_fov (2)."""
        if out is None:
            out = torch.empty(DCAMERA, dtype=torch.float32, device=self.device)
        lib = self._lib()
        with torch.cuda.device(self.device):
            _capi.check(lib.gh_camera_forward(self.n, _ptr(self.residuals), _ptr(self.base), _ptr(index), _ptr(out[0:16]),
                                              _ptr(out[16:32]), _ptr(out[32:35]), _ptr(out[35:37]),
                                              _ptr(self.status if status is None else status), 0, _stream(self.device)))
        return out

    def backward(self, index: torch.Tensor, d_camera: torch.Tensor, status: Optional[torch.Tensor] = None) -> None:
        """gh_camera_backward: the (37,) upstream gradients (gh_project_backward's d_camera layout) of the camera at
        `index` -> added to grad[index], touched[index] = 1, nan_flag OR-ed when a gradient is NaN."""
        lib = self._lib()
        with torch.cuda.device(self.device):
            _capi.check(lib.gh_camera_backward(self.n, _ptr(self.residuals), _ptr(self.base), _ptr(index), int(self.intrinsics),
                                               _ptr(d_camera), _ptr(self.grad), _ptr(self.touched), _ptr(self.nan_flag),
                                               _ptr(self.status if status is None else status), 0, _stream(self.device)))

    # ------------------------------------------------------------------------------------------ the reference's files
    def reference_dicts(self):
        """The three `{image_name: tensor}` dicts train_gaussians.py pickles (rotation (3), translation (3), fov (2);
        the last one empty without intrinsics)."""
        r = self.residuals.detach()
        rot = {n: r[i, 0:3].clone() for i, n in enumerate(self.names)}
        trans = {n: r[i, 3:6].clone() for i, n in enumerate(self.names)}
        fov = {n: r[i, 6:8].clone() for i, n in enumerate(self.names)} if self.intrinsics else {}
        return rot, trans, fov

    def write_back(self, cameras) -> None:
        """Set the `.data` of each Camera's residual parameters (matched by image_name) to the rig's values, so that
        the reference's own Camera properties, checkpoints and later stages see the trained cameras."""
        rot, trans, fov = self.reference_dicts()
        for cam in cameras:
            n = cam.image_name
            if n not in rot:
                raise KeyError(f"CameraRig.write_back: camera '{n}' is not in the rig")
            cam._rotation_res.data = rot[n].to(cam._rotation_res.device).reshape(cam._rotation_res.shape)
            cam._translation_res.data = trans[n].to(cam._translation_res.device).reshape(cam._translation_res.shape)
            if self.intrinsics:
                cam._fov_res.data = fov[n].to(cam._fov_res.device).reshape(cam._fov_res.shape)


class _CameraNode(torch.autograd.Function):
    """(residuals, index, rig) -> (viewmatrix, projmatrix, campos, tan_fov) of camera `index`.  The backward adds dL/dr
    into rig.grad (not into residuals.grad) and marks the row touched: CameraAdam steps exactly those rows."""

    @staticmethod
    def forward(ctx, residuals, index, rig):
        ctx.rig, ctx.index = rig, index
        out = rig.forward(index)
        return out[0:16].view(4, 4), out[16:32].view(4, 4), out[32:35], out[35:37]

    @staticmethod
    def backward(ctx, g_view, g_proj, g_campos, g_tan):
        d = torch.cat([g_view.reshape(-1), g_proj.reshape(-1), g_campos.reshape(-1), g_tan.reshape(-1)]).float()
        ctx.rig.backward(ctx.index, d)
        return None, None, None


class CameraView:
    """A rig camera with the attributes the reference renderers read: world_view_transform, full_proj_transform,
    camera_center, FoVx / FoVy, image_width / image_height, image_name, and tan_fov = tan(FoV / 2) (x, y) as a (2,)
    device tensor (renderer.py uses it instead of reading FoVx / FoVy back)."""

    def __init__(self, rig: CameraRig, index: int, requires_grad: bool):
        self.rig, self.index, self.requires_grad = rig, index, bool(requires_grad)
        self.image_width, self.image_height = rig.sizes[index]
        self.image_name = rig.names[index]
        self.znear, self.zfar = 0.01, 100.0
        self._out = None

    def _outputs(self):
        if self._out is None:
            idx = self.rig.indices[self.index:self.index + 1]
            if self.requires_grad:
                self._out = _CameraNode.apply(self.rig.residuals, idx, self.rig)
            else:
                with torch.no_grad():
                    out = self.rig.forward(idx)
                self._out = (out[0:16].view(4, 4), out[16:32].view(4, 4), out[32:35], out[35:37])
        return self._out

    @property
    def world_view_transform(self):
        return self._outputs()[0]

    @property
    def full_proj_transform(self):
        return self._outputs()[1]

    @property
    def camera_center(self):
        return self._outputs()[2]

    @property
    def tan_fov(self):
        return self._outputs()[3]

    @property
    def FoVx(self):
        return (self.rig.base[self.index, 16] + self.rig.residuals.detach()[self.index, 6]).reshape(1)

    @property
    def FoVy(self):
        return (self.rig.base[self.index, 17] + self.rig.residuals.detach()[self.index, 7]).reshape(1)


class CameraAdam:
    """The reference's camera optimizer, torch.optim.Adam(groups, lr=0.0, eps=1e-15) over every camera's
    _rotation_res / _translation_res / _fov_res, on a CameraRig.  `param_groups` are named "rotation", "translation"
    and "fov" (the reference's learning-rate schedule loop sets the translation 'lr' unchanged); each camera keeps its
    own step count and moments, and only cameras whose view received a gradient since the last step move.
    `capturable=True`: step() neither reads the host learning rates nor synchronises while a CUDA graph is captured --
    call load_lrs() before each replay (graphs.CapturedTrainStep does)."""

    def __init__(self, rig: CameraRig, lr_rotation: float, lr_translation: float, lr_fov: float = 0.0, eps: float = 1e-15,
                 betas=(0.9, 0.999), capturable: bool = False):
        self.rig = rig
        self.param_groups: List[Dict] = [{"name": "rotation", "lr": float(lr_rotation), "params": [rig.residuals]},
                                         {"name": "translation", "lr": float(lr_translation), "params": [rig.residuals]},
                                         {"name": "fov", "lr": float(lr_fov), "params": [rig.residuals]}]
        self.betas, self.eps, self.capturable = betas, float(eps), bool(capturable)
        f = dict(dtype=torch.float32, device=rig.device)
        self.exp_avg = torch.zeros(rig.n, ROW, **f)
        self.exp_avg_sq = torch.zeros(rig.n, ROW, **f)
        self.steps = torch.zeros(rig.n, dtype=torch.int32, device=rig.device)
        self.lrs = torch.zeros(3, **f)
        self._lrs_host = None          # pinned staging buffer of load_lrs, and the event of its last copy
        self._lrs_copied = None

    def load_lrs(self) -> None:
        """Copy the groups' 'lr' (rotation, translation, fov) into the device tensor `lrs`, through a pinned buffer on
        the current stream (no synchronisation: only the previous copy out of the buffer is waited for)."""
        if self._lrs_host is None:
            self._lrs_host = torch.zeros(3, dtype=torch.float32).pin_memory()
        if self._lrs_copied is not None:
            self._lrs_copied.synchronize()
        self._lrs_host.numpy()[:] = [float(g["lr"]) for g in self.param_groups]
        stream = torch.cuda.current_stream(self.rig.device)
        with torch.cuda.stream(stream):
            self.lrs.copy_(self._lrs_host, non_blocking=True)
        self._lrs_copied = torch.cuda.Event()
        self._lrs_copied.record(stream)

    def step(self, skip_flag: Optional[torch.Tensor] = None) -> None:
        """gh_camera_adam_step: update the touched cameras, then clear their gradients.  Skipped on the device when the
        rig's NaN flag or `skip_flag` (device int32 (1,), e.g. the binning status word) is set."""
        if not (self.capturable and torch.cuda.is_current_stream_capturing()):
            self.load_lrs()
        r, lib = self.rig, self.rig._lib()
        with torch.cuda.device(r.device):
            _capi.check(lib.gh_camera_adam_step(r.n, int(r.intrinsics), _ptr(r.residuals), _ptr(r.grad), _ptr(r.touched),
                                                _ptr(self.exp_avg), _ptr(self.exp_avg_sq), _ptr(self.steps), _ptr(self.lrs),
                                                float(self.betas[0]), float(self.betas[1]), self.eps, _ptr(r.nan_flag),
                                                _ptr(skip_flag), 0, _stream(r.device)))

    def zero_grad(self, set_to_none: bool = True) -> None:
        """Drop every accumulated camera gradient (step() already cleared the rows it consumed)."""
        self.rig.grad.zero_()
        self.rig.touched.zero_()
