"""The appearance-stage training iteration captured in one CUDA graph (DESIGN §16).

`CapturedTrainStep.step()` runs the iteration that `tools/train_loop.py` runs for `src/train_gaussians.py` --
fused render -> hair_image_loss -> backward -> FusedAdam -> densification statistics -- as one graph replay instead of
a few dozen Python-driven launches.  Per step the camera, the supervision maps and the learning rates are copied into
static device buffers, the graph is replayed, and one small pinned read returns the status word and the losses (the
same synchronisation a trainer's `loss.item()` costs).

R, the number of tile instances, never reaches the host inside the graph: the binning buffer has a fixed capacity, and
a frame whose R exceeds it sets the overflow bit of the status word, renders nothing and skips the Adam step on the
device (include/gh_rasterizer.h).  `step()` then reruns that iteration through the eager path -- so the run stays what
eager training computes -- raises the capacity (capacity_for: the largest R seen + 25 % + 256) and recaptures on the
next step.  A change of the model size (densify.densify_and_prune, which stays eager), of the image size, of the active
SH degree, of the deterministic switch or of the storage of any parameter, moment or statistic also recaptures.

Trainable cameras (DESIGN §17): with `cameras=rig` (cameras.CameraRig) and `camera_optimizer=CameraAdam(rig, ...,
capturable=True)`, `step(rig.view(i), ..., train_cameras=True)` copies only the camera index and the three camera
learning rates; the graph runs camera forward -> render (camera gradients into a static buffer) -> loss -> backward ->
camera backward -> FusedAdam (skipped on the status word) -> camera Adam (skipped on the status word or the camera NaN
flag).  `train_cameras=False` (the trainer passes `iteration < opt.iterations_cam`) renders the rig's cameras frozen;
the flag is part of the capture key.

Not captured: render_hair / render_hair_strands (head block, strand models), the multi-GPU gradient all-reduce
(gh_allreduce_p2p takes its epoch as a host argument).
"""
from __future__ import annotations

import types
from typing import Optional, Sequence

import torch

from . import _C, densify, losses as ghl, projection, renderer
from ._C import capacity_for
from .cameras import CameraAdam, CameraView, STATUS_CAMERA_INDEX
from .optim import FusedAdam

__all__ = ["CapturedTrainStep", "capture_key", "capacity_for", "STATUS_BINNING_OVERFLOW", "STATUS_CAMERA_INDEX"]

STATUS_BINNING_OVERFLOW = 1      # GH_STATUS_BINNING_OVERFLOW
WARMUP_ITERS = 2                 # eager iterations (on a side stream) before each capture


def capture_key(model, optimizer, width: int, height: int, cameras=None, camera_optimizer=None,
                train_cameras: bool = False) -> tuple:
    """What a captured iteration is specialised to: the model size P, the image size, the active SH degree,
    torch.are_deterministic_algorithms_enabled(), the storage of every parameter, Adam moment and densification
    statistic (a captured launch keeps the addresses it was recorded with) and, when the iteration renders a view of a
    cameras.CameraRig, the storage of the rig's and its optimizer's tables and whether the cameras train.  A different
    key means a new capture."""
    ptrs = []
    for g in optimizer.param_groups:
        for p in g["params"]:
            ptrs.append(p.data_ptr())
            st = optimizer.state.get(p) or {}
            ptrs.extend(st[k].data_ptr() for k in ("exp_avg", "exp_avg_sq") if k in st)
    for name in ("xyz_gradient_accum", "denom", "max_radii2D"):
        t = getattr(model, name, None)
        ptrs.append(t.data_ptr() if t is not None else 0)
    cam = ()
    if cameras is not None:
        tables = [cameras.base, cameras.residuals, cameras.grad, cameras.touched, cameras.nan_flag, cameras.indices]
        if camera_optimizer is not None:
            tables += [camera_optimizer.exp_avg, camera_optimizer.exp_avg_sq, camera_optimizer.steps, camera_optimizer.lrs]
        cam = (bool(train_cameras),) + tuple(t.data_ptr() for t in tables)
    return (int(model._xyz.shape[0]), int(width), int(height), int(model.active_sh_degree),
            bool(torch.are_deterministic_algorithms_enabled()), tuple(ptrs), cam)


def _check_no_arena() -> None:
    if projection._GRAD_ARENA["storage"] is not None:
        raise RuntimeError("CapturedTrainStep: a gradient arena is installed (projection.set_gradient_arena); the captured "
                           "iteration is single-GPU -- remove it with set_gradient_arena(None)")


def _check_camera(camera) -> None:
    for name in ("world_view_transform", "full_proj_transform", "camera_center", "FoVx", "FoVy"):
        t = getattr(camera, name)
        if isinstance(t, torch.Tensor) and t.requires_grad:
            raise RuntimeError(f"CapturedTrainStep: camera.{name} requires grad; trainable cameras are not supported "
                               "(use renderer.render_raw eagerly)")


class CapturedTrainStep:
    """One `train_gaussians.py` iteration per `step()`, replayed from a CUDA graph.

    model: a GaussianModel-shaped object (`_xyz ... _orient_conf`, `active_sh_degree`, and `xyz_gradient_accum`,
      `denom`, `max_radii2D` when `densification_stats`); optimizer: FusedAdam(..., capturable=True) over its
      parameters, every one of which receives a gradient; bg: the (10,) background; lambdas: (l1, ssim, mask, orient)
      loss weights; capacity: the initial binning capacity in records (None: seeded from the warm-up iterations);
      pipe: the trainer's pipeline options (`debug` must be off); cameras: a cameras.CameraRig whose views step()
      receives (None: cameras are plain objects with fixed tensors); camera_optimizer: CameraAdam(cameras, ...,
      capturable=True), needed for `train_cameras=True`.
    """

    def __init__(self, model, optimizer, width: int, height: int, bg: torch.Tensor, lambdas: Sequence[float],
                 densification_stats: bool = True, capacity: Optional[int] = None, pipe=None, cameras=None,
                 camera_optimizer=None):
        if getattr(pipe, "debug", False):
            raise RuntimeError("CapturedTrainStep: debug mode synchronises after every stage and cannot be captured")
        if not isinstance(optimizer, FusedAdam) or not optimizer.capturable:
            raise RuntimeError("CapturedTrainStep needs FusedAdam(..., capturable=True)")
        _check_no_arena()
        if camera_optimizer is not None and (not isinstance(camera_optimizer, CameraAdam) or not camera_optimizer.capturable
                                             or camera_optimizer.rig is not cameras):
            raise RuntimeError("CapturedTrainStep: camera_optimizer must be CameraAdam(cameras, ..., capturable=True)")
        self.cameras, self.camera_optimizer = cameras, camera_optimizer
        self.model, self.optimizer = model, optimizer
        self.W, self.H = int(width), int(height)
        self.bg = bg
        self.lambdas = tuple(float(x) for x in lambdas)
        self.densification_stats = bool(densification_stats)
        self.pipe = pipe if pipe is not None else types.SimpleNamespace(debug=False)
        self.capacity = int(capacity or 0)
        self.r_max = 0                     # the largest R seen (eager iterations and replays)
        self.captures = self.replays = self.overflows = 0
        dev = model._xyz.device
        self.device = dev
        f = dict(dtype=torch.float32, device=dev)
        self._camera = {"viewmatrix": torch.zeros(4, 4, **f), "projmatrix": torch.zeros(4, 4, **f),
                        "campos": torch.zeros(3, **f), "tan_fov": torch.ones(2, **f)}
        # rig views: the device index of the view, the camera forward's outputs and the render's camera gradients
        self._cam_index = torch.zeros(1, dtype=torch.int32, device=dev)
        self._cam_out = torch.zeros(37, **f)
        self._d_camera = torch.zeros(37, **f)
        H, W = self.H, self.W
        self._gt = [torch.zeros(c, H, W, **f) for c in (3, 2, 1, 1)]
        # status word, R, and the float32 bits of the eight losses: read back together after every replay
        self._io = torch.zeros(10, dtype=torch.int32, device=dev)
        self._host = torch.zeros(10, dtype=torch.int32).pin_memory()
        self._nan_flag = torch.zeros(1, dtype=torch.int32, device=dev)
        self._ws = torch.empty(ghl.workspace_elems(W, H), dtype=torch.float64, device=dev)
        self._graph = None
        self._binning = None
        self._key = None
        self._warm = 0
        self._train_cameras = False

    # ------------------------------------------------------------------------------------------ the iteration
    def _tail(self, renders, radii, viewspace, gts, skip, camera_backward=None):
        """loss -> backward (-> camera backward) -> densification statistics -> Adam, shared by the eager and the
        captured iteration."""
        losses8, dL = ghl.image_loss_forward_backward(renders.detach(), *gts, *self.lambdas, workspace=self._ws)
        renders.backward(dL)
        if camera_backward is not None:
            camera_backward()
        if self.densification_stats:
            with torch.no_grad():
                densify.update_max_radii(self.model, radii)
                densify.add_densification_stats(self.model, viewspace, radii > 0)
        self.optimizer.step(skip_flags=skip, nan_flag_in=self._nan_flag)
        self.optimizer.zero_grad(set_to_none=True)
        return losses8

    def _with_nan_flag(self, fn):
        prev = renderer._NAN_FLAG["t"]
        renderer.set_nan_flag(self._nan_flag)
        try:
            return fn()
        finally:
            renderer.set_nan_flag(prev)

    def _eager(self, camera, gts) -> torch.Tensor:
        """The eager iteration (renderer.render_raw), on a side stream like every warm-up before a capture.  A rig view
        is rendered through its autograd node (camera gradients when the step trains the cameras) and the camera Adam
        follows."""
        train_cameras = self._train_cameras
        cur = torch.cuda.current_stream(self.device)
        side = torch.cuda.Stream(self.device)
        side.wait_stream(cur)
        with torch.cuda.stream(side):
            if isinstance(camera, CameraView):
                camera = camera.rig.view(camera.index, requires_grad=train_cameras)
            renders, radii, viewspace = renderer.render_raw(camera, self.model, self.pipe, self.bg)
            losses8 = self._with_nan_flag(lambda: self._tail(renders, radii, viewspace, gts, ()))
            if train_cameras:
                self.camera_optimizer.step()
        cur.wait_stream(side)
        key = (self.device.index, int(self.model._xyz.shape[0]), self.W, self.H)
        self.r_max = max(self.r_max, _C.last_num_rendered(key))
        return losses8.cpu()

    def _captured(self, rig_view: bool, train_cameras: bool):
        status, n_rendered = self._io[0:1], self._io[1:2]
        status.zero_()
        camera, d_camera, camera_backward = self._camera, None, None
        if rig_view:
            rig, out = self.cameras, self._cam_out
            rig.forward(self._cam_index, out=out, status=status)
            camera = {"viewmatrix": out[0:16].view(4, 4), "projmatrix": out[16:32].view(4, 4), "campos": out[32:35],
                      "tan_fov": out[35:37]}
            if train_cameras:
                d_camera = self._d_camera
                camera_backward = lambda: rig.backward(self._cam_index, d_camera, status=status)  # noqa: E731
        renders, radii, viewspace = renderer.render_raw_capturable(camera, self.model, self.bg, self.W, self.H,
                                                                   self._binning, self.capacity, status, n_rendered,
                                                                   d_camera=d_camera)
        losses8 = self._tail(renders, radii, viewspace, self._gt, (status,), camera_backward)
        if train_cameras:
            self.camera_optimizer.step(skip_flag=status)
        self._io[2:].copy_(losses8.view(torch.int32))

    def _current_key(self, rig_view: bool, train_cameras: bool) -> tuple:
        if not rig_view:
            return capture_key(self.model, self.optimizer, self.W, self.H)
        return capture_key(self.model, self.optimizer, self.W, self.H, self.cameras, self.camera_optimizer, train_cameras)

    def _capture(self, rig_view: bool, train_cameras: bool) -> None:
        self.capacity = max(self.capacity, capacity_for(self.r_max))
        self._graph = None
        self._binning = _C.binning_workspace(self.capacity, self.device)
        self.optimizer.zero_grad(set_to_none=True)
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            self._with_nan_flag(lambda: self._captured(rig_view, train_cameras))
        self._graph = g
        self.captures += 1

    def _load(self, camera, gts, rig_view: bool, train_cameras: bool) -> None:
        if rig_view:
            self._cam_index.copy_(camera.rig.indices[camera.index:camera.index + 1])
            if train_cameras:
                self.camera_optimizer.load_lrs()
        else:
            c = self._camera
            c["viewmatrix"].copy_(camera.world_view_transform)
            c["projmatrix"].copy_(camera.full_proj_transform)
            c["campos"].copy_(camera.camera_center)
            # the same values the eager path passes: a camera's own tan_fov (renderer._static), else the host values of
            # renderer._tan_half (cached per FoV tensor)
            tan = getattr(camera, "tan_fov", None)
            if tan is None:
                tan = torch.tensor([renderer._tan_half(camera.FoVx), renderer._tan_half(camera.FoVy)], dtype=torch.float32)
            c["tan_fov"].copy_(tan)
        for dst, src in zip(self._gt, gts):
            dst.copy_(src)
        self.optimizer.load_lrs()

    # ------------------------------------------------------------------------------------------ public
    def step(self, camera, gt_image, gt_mask, gt_orient_angle, gt_orient_conf, train_cameras: bool = False) -> torch.Tensor:
        """One training iteration on `camera` -> the eight losses of hair_image_loss (float32 CPU tensor: total, Ll1,
        Lssim, Lmask, Lorient, sum of orientation weights, Lorient-was-NaN, 0).  `camera`: a view of `cameras` (the
        rig) or a camera with fixed tensors; `train_cameras`: also train the rig's camera (src/train_gaussians.py:183:
        `iteration < opt.iterations_cam`)."""
        rig_view = self.cameras is not None and isinstance(camera, CameraView) and camera.rig is self.cameras
        if not rig_view:
            _check_camera(camera)
        train_cameras = bool(train_cameras)
        if train_cameras and (not rig_view or self.camera_optimizer is None):
            raise RuntimeError("CapturedTrainStep: train_cameras=True needs a view of the step's CameraRig and a camera_optimizer")
        _check_no_arena()
        self._train_cameras = train_cameras
        gts = (gt_image, gt_mask, gt_orient_angle, gt_orient_conf)
        key = self._current_key(rig_view, train_cameras)
        if key != self._key:
            self._graph, self._binning, self._key, self._warm = None, None, key, 0
        if self._graph is None and self._warm < WARMUP_ITERS:
            self._warm += 1
            losses = self._eager(camera, gts)
            self._key = self._current_key(rig_view, train_cameras)   # the first step creates the moments
            return losses
        if self._graph is None:
            self._capture(rig_view, train_cameras)
            self._key = self._current_key(rig_view, train_cameras)
        self._load(camera, gts, rig_view, train_cameras)
        self._graph.replay()
        self.replays += 1
        self._host.copy_(self._io, non_blocking=True)
        torch.cuda.current_stream(self.device).synchronize()
        status, R = int(self._host[0]), int(self._host[1])
        self.r_max = max(self.r_max, R)
        if status & STATUS_CAMERA_INDEX:
            raise RuntimeError("CapturedTrainStep: the camera index was outside the rig (nothing was updated)")
        if status & STATUS_BINNING_OVERFLOW:
            # the replay rendered nothing and left parameters, moments, step counts and statistics untouched
            self.overflows += 1
            self.capacity = capacity_for(self.r_max)
            self._graph, self._binning = None, None
            return self._eager(camera, gts)
        return self._host[2:].view(torch.float32).clone()
