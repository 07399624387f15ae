"""Training iterations captured in one CUDA graph (DESIGN §16, §19).

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

`CapturedStrandStep.step()` does the same for the `src/train_strands.py` iteration (DESIGN §19):
render_hair_strands_capturable (frozen head block + strand model) -> strand_image_loss -> backward (+ the prior's
`_dirs` gradient, computed outside the graph) -> FusedAdam.  The two classes share the warm-up on a side stream, the
capacity seeding, the overflow rerun and recapture, and the pinned read-back (_CapturedStep).

`CapturedLatentStrandStep.step()` captures the part of the `src/train_latent_strands.py` iteration that runs in this
package (DESIGN §20): render_hair_segments_capturable (frozen head block + the decoder's segment rows) ->
latent_strand_image_loss -> backward into static gradients of the five decoder outputs.  The strand networks, their
prior term and their AdamW stay eager, outside the graph: step() returns a loss tensor whose backward hands the static
gradients to them.

Not captured: the multi-GPU gradient all-reduce (gh_allreduce_p2p takes its epoch as a host argument).
"""
from __future__ import annotations

import types
from typing import Callable, Optional, Sequence

import torch

from . import _C, densify, losses as ghl, projection, renderer
from ._C import capacity_for
from .cameras import CameraAdam, CameraView, STATUS_CAMERA_INDEX
from .optim import FusedAdam

__all__ = ["CapturedTrainStep", "CapturedStrandStep", "CapturedLatentStrandStep", "capture_key", "strand_capture_key",
           "latent_capture_key", "check_dirs_grad", "capacity_for", "STATUS_BINNING_OVERFLOW", "STATUS_CAMERA_INDEX"]

STATUS_BINNING_OVERFLOW = 1      # GH_STATUS_BINNING_OVERFLOW
WARMUP_ITERS = 2                 # eager iterations (on a side stream) before each capture


def _rig_tables(cameras, camera_optimizer=None) -> tuple:
    tables = [cameras.base, cameras.residuals, cameras.grad, cameras.touched, cameras.nan_flag, cameras.indices]
    if camera_optimizer is not None:
        tables += [camera_optimizer.exp_avg, camera_optimizer.exp_avg_sq, camera_optimizer.steps, camera_optimizer.lrs]
    return tuple(t.data_ptr() for t in tables)


def _optimizer_storage(optimizer) -> list:
    ptrs = []
    for g in optimizer.param_groups:
        for p in g["params"]:
            ptrs.append(p.data_ptr())
            st = optimizer.state.get(p) or {}
            ptrs.extend(st[k].data_ptr() for k in ("exp_avg", "exp_avg_sq") if k in st)
    return ptrs


def capture_key(model, optimizer, width: int, height: int, cameras=None, camera_optimizer=None,
                train_cameras: bool = False) -> tuple:
    """What a captured iteration is specialised to: the model size P, the image size, the active SH degree,
    torch.are_deterministic_algorithms_enabled(), the storage of every parameter, Adam moment and densification
    statistic (a captured launch keeps the addresses it was recorded with) and, when the iteration renders a view of a
    cameras.CameraRig, the storage of the rig's and its optimizer's tables and whether the cameras train.  A different
    key means a new capture."""
    ptrs = _optimizer_storage(optimizer)
    for name in ("xyz_gradient_accum", "denom", "max_radii2D"):
        t = getattr(model, name, None)
        ptrs.append(t.data_ptr() if t is not None else 0)
    cam = ()
    if cameras is not None:
        cam = (bool(train_cameras),) + _rig_tables(cameras, camera_optimizer)
    return (int(model._xyz.shape[0]), int(width), int(height), int(model.active_sh_degree),
            bool(torch.are_deterministic_algorithms_enabled()), tuple(ptrs), cam)


def strand_capture_key(pc, pc_hair, optimizer, width: int, height: int, use_gt_orient_conf: bool = True,
                       train_orient_conf: bool = True, cameras=None, dirs_grad: bool = False) -> tuple:
    """What a captured strand iteration is specialised to: S, L, the head block's size n_head, the image size, the
    strand model's active SH degree, torch.are_deterministic_algorithms_enabled(), the two loss options, whether a prior
    gradient is added to `_dirs`, and the storage of the optimizer's parameters and moments, of `pts_origins`, of
    `scale`, of the cached head block (renderer._head_block) and of the rig's tables when views of a
    cameras.CameraRig are rendered.  A different key means a new capture."""
    S, L = int(pc_hair._dirs.shape[0]), int(pc_hair._dirs.shape[1])
    head = renderer._head_block(pc) if pc is not None else None
    n_head = 0 if head is None else int(head["xyz"].shape[0])
    head_ptrs = () if head is None else tuple(head[k].data_ptr() for k in ("xyz", "scaling", "rotation", "opacity",
                                                                            "f_dc", "f_rest"))
    scale = pc_hair.scale
    ptrs = _optimizer_storage(optimizer) + [pc_hair.pts_origins.data_ptr(),
                                            scale.data_ptr() if isinstance(scale, torch.Tensor) else 0]
    cam = _rig_tables(cameras) if cameras is not None else ()
    return (S, L, n_head, int(width), int(height), int(pc_hair.active_sh_degree),
            bool(torch.are_deterministic_algorithms_enabled()), bool(use_gt_orient_conf), bool(train_orient_conf),
            bool(dirs_grad), tuple(ptrs), head_ptrs, cam)


def latent_capture_key(pc, pc_hair, width: int, height: int, use_gt_orient_conf: bool = True,
                       train_orient_conf: bool = True, cameras=None) -> tuple:
    """What a captured latent strand iteration is specialised to: the segment rows N, the head block's size n_head,
    the image size, the strand model's active SH degree, torch.are_deterministic_algorithms_enabled(), the two loss
    options, and the storage of `scale`, of the cached head block (renderer._head_block) and of the rig's tables when
    views of a cameras.CameraRig are rendered.  The decoder's outputs are copied into buffers the step owns, so their
    storage is not part of the key.  A different key means a new capture."""
    N = int(pc_hair._xyz.shape[0])
    head = renderer._head_block(pc) if pc is not None else None
    n_head = 0 if head is None else int(head["xyz"].shape[0])
    head_ptrs = () if head is None else tuple(head[k].data_ptr() for k in ("xyz", "scaling", "rotation", "opacity",
                                                                            "f_dc", "f_rest"))
    scale = pc_hair.scale
    cam = _rig_tables(cameras) if cameras is not None else ()
    return (N, n_head, int(width), int(height), int(pc_hair.active_sh_degree),
            bool(torch.are_deterministic_algorithms_enabled()), bool(use_gt_orient_conf), bool(train_orient_conf),
            scale.data_ptr() if isinstance(scale, torch.Tensor) else 0, head_ptrs, cam)


def check_dirs_grad(dirs_grad: torch.Tensor, dirs: torch.Tensor) -> None:
    """The prior gradient a strand trainer hands to CapturedStrandStep.step(): float32, on the device of `_dirs`, and
    of its (S, L, 3) shape."""
    if not isinstance(dirs_grad, torch.Tensor) or tuple(dirs_grad.shape) != tuple(dirs.shape):
        got = tuple(dirs_grad.shape) if isinstance(dirs_grad, torch.Tensor) else type(dirs_grad).__name__
        raise RuntimeError(f"CapturedStrandStep: dirs_grad must have the shape of _dirs {tuple(dirs.shape)}, got {got}")
    if dirs_grad.dtype != torch.float32 or dirs_grad.device != dirs.device:
        raise RuntimeError(f"CapturedStrandStep: dirs_grad must be float32 on {dirs.device}, got {dirs_grad.dtype} on "
                           f"{dirs_grad.device}")


def _check_no_arena(who: str = "CapturedTrainStep") -> None:
    if projection._GRAD_ARENA["storage"] is not None:
        raise RuntimeError(f"{who}: a gradient arena is installed (projection.set_gradient_arena); the captured "
                           "iteration is single-GPU -- remove it with set_gradient_arena(None)")


def _check_camera(camera, who: str = "CapturedTrainStep", eager: str = "renderer.render_raw") -> None:
    for name in ("world_view_transform", "full_proj_transform", "camera_center", "FoVx", "FoVy"):
        t = getattr(camera, name)
        if isinstance(t, torch.Tensor) and t.requires_grad:
            raise RuntimeError(f"{who}: camera.{name} requires grad; trainable cameras are not supported "
                               f"(use {eager} eagerly)")


def _on_side_stream(device, fn):
    """fn() on a fresh side stream, ordered after and before the current stream's work (every eager iteration runs
    like the warm-ups before a capture)."""
    cur = torch.cuda.current_stream(device)
    side = torch.cuda.Stream(device)
    side.wait_stream(cur)
    with torch.cuda.stream(side):
        out = fn()
    cur.wait_stream(side)
    return out


class _CapturedStep:
    """What the captured iterations share: the static status / R / loss words and their pinned read-back, the NaN flag,
    the loss workspace, the capacity policy, the warm-up iterations before a capture, the capture itself, and the
    replay that falls back to the eager iteration on a binning overflow."""

    def __init__(self, who: str, optimizer, width: int, height: int, bg: torch.Tensor, lambdas: Sequence[float],
                 capacity: Optional[int], pipe, device, needs_optimizer: bool = True):
        """`needs_optimizer=False`: the iteration has no optimizer inside the graph (`optimizer` must then be None)."""
        if getattr(pipe, "debug", False):
            raise RuntimeError(f"{who}: debug mode synchronises after every stage and cannot be captured")
        if needs_optimizer and (not isinstance(optimizer, FusedAdam) or not optimizer.capturable):
            raise RuntimeError(f"{who} needs FusedAdam(..., capturable=True)")
        if not needs_optimizer and optimizer is not None:
            raise RuntimeError(f"{who}: the iteration has no optimizer inside the graph")
        _check_no_arena(who)
        self.optimizer = optimizer
        self.W, self.H = int(width), int(height)
        self.bg = bg
        self.lambdas = tuple(float(x) for x in lambdas)
        self.pipe = pipe if pipe is not None else types.SimpleNamespace(debug=False)
        self.capacity = int(capacity or 0)
        self.r_max = 0                     # the largest R seen (eager iterations and replays)
        self.captures = self.replays = self.overflows = 0
        self.device = device
        f = dict(dtype=torch.float32, device=device)
        self._camera = {"viewmatrix": torch.zeros(4, 4, **f), "projmatrix": torch.zeros(4, 4, **f),
                        "campos": torch.zeros(3, **f), "tan_fov": torch.ones(2, **f)}
        self._cam_index = torch.zeros(1, dtype=torch.int32, device=device)
        self._gt = [torch.zeros(c, self.H, self.W, **f) for c in (3, 2, 1, 1)]
        # status word, R, and the float32 bits of the eight losses: read back together after every replay
        self._io = torch.zeros(10, dtype=torch.int32, device=device)
        self._host = torch.zeros(10, dtype=torch.int32).pin_memory()
        self._nan_flag = torch.zeros(1, dtype=torch.int32, device=device)
        self._ws = torch.empty(ghl.workspace_elems(self.W, self.H), dtype=torch.float64, device=device)
        self._graph = None
        self._binning = None
        self._key = None
        self._warm = 0

    def _with_nan_flag(self, fn):
        prev = renderer._NAN_FLAG["t"]
        renderer.set_nan_flag(self._nan_flag)
        try:
            return fn()
        finally:
            renderer.set_nan_flag(prev)

    def _record_r(self, P: int) -> None:
        """After an eager iteration: the R its forward recorded for (device, P, W, H) (_C.binning_record)."""
        self.r_max = max(self.r_max, _C.last_num_rendered((self.device.index, int(P), self.W, self.H)))

    def _load_camera(self, camera) -> None:
        """A camera with fixed tensors into the static camera buffers: the values the eager path passes -- a camera's
        own tan_fov (renderer._static), else the host values of renderer._tan_half (cached per FoV tensor)."""
        c = self._camera
        c["viewmatrix"].copy_(camera.world_view_transform)
        c["projmatrix"].copy_(camera.full_proj_transform)
        c["campos"].copy_(camera.camera_center)
        tan = getattr(camera, "tan_fov", None)
        if tan is None:
            tan = torch.tensor([renderer._tan_half(camera.FoVx), renderer._tan_half(camera.FoVy)], dtype=torch.float32)
        c["tan_fov"].copy_(tan)

    def _capture(self, captured: Callable[[], None]) -> None:
        self.capacity = max(self.capacity, capacity_for(self.r_max))
        self._graph = None
        self._binning = _C.binning_workspace(self.capacity, self.device)
        if self.optimizer is not None:
            self.optimizer.zero_grad(set_to_none=True)
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            self._with_nan_flag(captured)
        self._graph = g
        self.captures += 1

    def _iterate(self, current_key: Callable[[], tuple], eager: Callable[[], torch.Tensor],
                 captured: Callable[[], None], load: Callable[[], None], who: str) -> torch.Tensor:
        """One iteration: eager while warming up after a key change, else (capture and) replay; an overflowed replay
        changed nothing and reruns eagerly with a raised capacity, recaptured on the next step."""
        key = current_key()
        if key != self._key:
            self._graph, self._binning, self._key, self._warm = None, None, key, 0
        if self._graph is None and self._warm < WARMUP_ITERS:
            self._warm += 1
            losses = eager()
            self._key = current_key()   # the first step creates the moments
            return losses
        if self._graph is None:
            self._capture(captured)
            self._key = current_key()
        load()
        self._graph.replay()
        self.replays += 1
        self._host.copy_(self._io, non_blocking=True)
        torch.cuda.current_stream(self.device).synchronize()
        status, R = int(self._host[0]), int(self._host[1])
        self.r_max = max(self.r_max, R)
        if status & STATUS_CAMERA_INDEX:
            raise RuntimeError(f"{who}: the camera index was outside the rig (nothing was updated)")
        if status & STATUS_BINNING_OVERFLOW:
            # the replay rendered nothing and left parameters, moments, step counts and statistics untouched
            self.overflows += 1
            self.capacity = capacity_for(self.r_max)
            self._graph, self._binning = None, None
            return eager()
        return self._host[2:].view(torch.float32).clone()


class CapturedTrainStep(_CapturedStep):
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
        super().__init__("CapturedTrainStep", optimizer, width, height, bg, lambdas, capacity, pipe, model._xyz.device)
        if camera_optimizer is not None and (not isinstance(camera_optimizer, CameraAdam) or not camera_optimizer.capturable
                                             or camera_optimizer.rig is not cameras):
            raise RuntimeError("CapturedTrainStep: camera_optimizer must be CameraAdam(cameras, ..., capturable=True)")
        self.cameras, self.camera_optimizer = cameras, camera_optimizer
        self.model = model
        self.densification_stats = bool(densification_stats)
        f = dict(dtype=torch.float32, device=self.device)
        # rig views: the camera forward's outputs and the render's camera gradients
        self._cam_out = torch.zeros(37, **f)
        self._d_camera = torch.zeros(37, **f)
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

    def _eager(self, camera, gts) -> torch.Tensor:
        """The eager iteration (renderer.render_raw), on a side stream like every warm-up before a capture.  A rig view
        is rendered through its autograd node (camera gradients when the step trains the cameras) and the camera Adam
        follows."""
        train_cameras = self._train_cameras

        def run():
            cam = camera
            if isinstance(cam, CameraView):
                cam = cam.rig.view(cam.index, requires_grad=train_cameras)
            renders, radii, viewspace = renderer.render_raw(cam, self.model, self.pipe, self.bg)
            losses8 = self._with_nan_flag(lambda: self._tail(renders, radii, viewspace, gts, ()))
            if train_cameras:
                self.camera_optimizer.step()
            return losses8

        losses8 = _on_side_stream(self.device, run)
        self._record_r(self.model._xyz.shape[0])
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

    def _load(self, camera, gts, rig_view: bool, train_cameras: bool) -> None:
        if rig_view:
            self._cam_index.copy_(camera.rig.indices[camera.index:camera.index + 1])
            if train_cameras:
                self.camera_optimizer.load_lrs()
        else:
            self._load_camera(camera)
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
        return self._iterate(lambda: self._current_key(rig_view, train_cameras),
                             lambda: self._eager(camera, gts),
                             lambda: self._captured(rig_view, train_cameras),
                             lambda: self._load(camera, gts, rig_view, train_cameras),
                             "CapturedTrainStep")


class CapturedStrandStep(_CapturedStep):
    """One `train_strands.py` iteration per `step()`, replayed from a CUDA graph (DESIGN §19).

    pc: the frozen head GaussianModel with the trainer's *_precomp attributes (renderer._head_block), or None for a
      hair-only model; pc_hair: the GaussianModelCurves (`_dirs` (S,L,3), `pts_origins`, `scale` a (1,) device
      tensor, `_features_dc`, `_features_rest`, `_orient_conf`, `active_sh_degree`); optimizer: FusedAdam(...,
      capturable=True) over those four parameters (its `_dirs` schedule reaches the graph through load_lrs()); bg: the
      (10,) background; lambdas: (l1, ssim, mask, orient) loss weights; use_gt_orient_conf / train_orient_conf: the
      trainer's options of strand_image_loss; capacity: the initial binning capacity in records (None: seeded from the
      warm-up iterations); pipe: the trainer's pipeline options (`debug` must be off); cameras: a cameras.CameraRig whose
      frozen views step() receives (None: cameras are plain objects with fixed tensors).

    The eager iteration (warm-ups and overflow reruns) is render_hair_strands -> image_loss_forward_backward(stage=
    "strands") -> backward (+ dirs_grad) -> FusedAdam.step(nan_flag_in=...); the captured one computes the same values
    (bit for bit under torch.use_deterministic_algorithms(True)).
    """

    def __init__(self, pc, pc_hair, optimizer, width: int, height: int, bg: torch.Tensor, lambdas: Sequence[float],
                 use_gt_orient_conf: bool = True, train_orient_conf: bool = True, capacity: Optional[int] = None,
                 pipe=None, cameras=None):
        super().__init__("CapturedStrandStep", optimizer, width, height, bg, lambdas, capacity, pipe,
                         pc_hair._dirs.device)
        if not isinstance(pc_hair.scale, torch.Tensor):
            raise RuntimeError("CapturedStrandStep: pc_hair.scale must be a (1,) device tensor")
        self.pc, self.pc_hair, self.cameras = pc, pc_hair, cameras
        self.use_gt_orient_conf, self.train_orient_conf = bool(use_gt_orient_conf), bool(train_orient_conf)
        self._cam_out = torch.zeros(37, dtype=torch.float32, device=self.device)
        self._dirs_grad = None          # the static copy of the prior's gradient (allocated on first use)

    def _dirs_grad_buffer(self, dirs_grad: Optional[torch.Tensor]) -> Optional[torch.Tensor]:
        if dirs_grad is None:
            return None
        check_dirs_grad(dirs_grad, self.pc_hair._dirs)
        shape = tuple(self.pc_hair._dirs.shape)
        if self._dirs_grad is None or tuple(self._dirs_grad.shape) != shape:
            self._dirs_grad = torch.zeros(shape, dtype=torch.float32, device=self.device)
        return self._dirs_grad

    # ------------------------------------------------------------------------------------------ the iteration
    def _tail(self, renders, gts, skip, dirs_grad):
        """loss -> backward -> (+ the prior's _dirs gradient) -> Adam, shared by the eager and the captured iteration."""
        losses8, dL = ghl.image_loss_forward_backward(renders.detach(), *gts, *self.lambdas, workspace=self._ws,
                                                      stage="strands", use_gt_orient_conf=self.use_gt_orient_conf,
                                                      train_orient_conf=self.train_orient_conf)
        renders.backward(dL)
        if dirs_grad is not None:
            g = self.pc_hair._dirs.grad
            g.add_(dirs_grad)
            # the reference's `_dirs.grad.isnan()` guard on the sum
            torch.maximum(self._nan_flag, g.isnan().any().to(torch.int32).reshape(1), out=self._nan_flag)
        self.optimizer.step(skip_flags=skip, nan_flag_in=self._nan_flag)
        self.optimizer.zero_grad(set_to_none=True)
        return losses8

    def _eager(self, camera, gts, dirs_grad) -> torch.Tensor:
        """The eager iteration (renderer.render_hair_strands) on a side stream.  A rig view is rendered frozen."""

        def run():
            cam = camera
            if isinstance(cam, CameraView):
                cam = cam.rig.view(cam.index, requires_grad=False)
            pkg = renderer.render_hair_strands(cam, self.pc, self.pc_hair, self.pipe, self.bg)
            return self._with_nan_flag(lambda: self._tail(pkg["raw"], gts, (), dirs_grad))

        losses8 = _on_side_stream(self.device, run)
        self._record_r(self._rows())
        return losses8.cpu()

    def _rows(self) -> int:
        head = renderer._head_block(self.pc) if self.pc is not None else None
        n_head = 0 if head is None else int(head["xyz"].shape[0])
        return n_head + int(self.pc_hair._dirs.shape[0]) * int(self.pc_hair._dirs.shape[1])

    def _captured(self, rig_view: bool, dirs_grad: Optional[torch.Tensor]):
        status, n_rendered = self._io[0:1], self._io[1:2]
        status.zero_()
        camera = self._camera
        if rig_view:
            out = self._cam_out
            self.cameras.forward(self._cam_index, out=out, status=status)
            camera = {"viewmatrix": out[0:16].view(4, 4), "projmatrix": out[16:32].view(4, 4), "campos": out[32:35],
                      "tan_fov": out[35:37]}
        renders, _radii = renderer.render_hair_strands_capturable(camera, self.pc, self.pc_hair, self.bg, self.W, self.H,
                                                                  self._binning, self.capacity, status, n_rendered)
        losses8 = self._tail(renders, self._gt, (status,), dirs_grad)
        self._io[2:].copy_(losses8.view(torch.int32))

    def _current_key(self, rig_view: bool, has_dirs_grad: bool) -> tuple:
        return strand_capture_key(self.pc, self.pc_hair, self.optimizer, self.W, self.H, self.use_gt_orient_conf,
                                  self.train_orient_conf, self.cameras if rig_view else None, has_dirs_grad)

    def _load(self, camera, gts, rig_view: bool, dirs_grad, static_dirs_grad) -> None:
        if rig_view:
            self._cam_index.copy_(camera.rig.indices[camera.index:camera.index + 1])
        else:
            self._load_camera(camera)
        for dst, src in zip(self._gt, gts):
            if src is not None:
                dst.copy_(src)
        if dirs_grad is not None:
            static_dirs_grad.copy_(dirs_grad)
        self.optimizer.load_lrs()

    # ------------------------------------------------------------------------------------------ public
    def step(self, camera, gt_image, gt_mask, gt_orient_angle, gt_orient_conf,
             dirs_grad: Optional[torch.Tensor] = None) -> torch.Tensor:
        """One training iteration on `camera` -> the eight losses of strand_image_loss (float32 CPU tensor: total,
        Ll1, Lssim, Lmask, Lorient, sum of orientation weights, Lorient-was-NaN, 0; the total without the prior term).
        `camera`: a (frozen) view of `cameras` or a camera with fixed tensors.  `dirs_grad`: None, or the (S, L, 3)
        gradient of the prior term (`Lsds * lambda_dsds`) w.r.t. `_dirs`, computed by the trainer outside the graph; it
        is added to the render's gradient before Adam, and a NaN in the sum skips the step."""
        rig_view = self.cameras is not None and isinstance(camera, CameraView) and camera.rig is self.cameras
        if not rig_view:
            _check_camera(camera, "CapturedStrandStep", "renderer.render_hair_strands")
        _check_no_arena("CapturedStrandStep")
        static_dirs_grad = self._dirs_grad_buffer(dirs_grad)
        if gt_orient_conf is None and self.use_gt_orient_conf:
            raise RuntimeError("CapturedStrandStep: gt_orient_conf is required with use_gt_orient_conf=True")
        gts = (gt_image, gt_mask, gt_orient_angle, gt_orient_conf)
        has = dirs_grad is not None
        return self._iterate(lambda: self._current_key(rig_view, has),
                             lambda: self._eager(camera, gts, dirs_grad),
                             lambda: self._captured(rig_view, static_dirs_grad),
                             lambda: self._load(camera, gts, rig_view, dirs_grad, static_dirs_grad),
                             "CapturedStrandStep")


SEGMENT_TENSORS = ("_xyz", "_dir", "_features_dc", "_features_rest", "_orient_conf")


class _StaticGradients(torch.autograd.Function):
    """(total, step, generation, xyz, dirs, f_dc, f_rest, conf) -> the 0-dim image loss of one CapturedLatentStrandStep
    step, connected to the five decoder outputs: the backward returns grad_output times the step's gradients (exact
    for grad_output = 1), and raises when a later step has overwritten them."""

    @staticmethod
    def forward(ctx, total, step, generation, *tensors):
        ctx.step, ctx.generation = step, generation
        return total.clone()

    @staticmethod
    def backward(ctx, g):
        step = ctx.step
        if ctx.generation != step._generation or step._grads is None:
            raise RuntimeError(f"CapturedLatentStrandStep: this loss is from step {ctx.generation}, but its gradients "
                               f"were overwritten by step {step._generation}; call backward() before the next step()")
        need = ctx.needs_input_grad
        return (None, None, None) + tuple(gr * g if need[3 + i] else None for i, gr in enumerate(step._grads))


class CapturedLatentStrandStep(_CapturedStep):
    """The render, loss and backward of one `train_latent_strands.py` iteration per `step()`, replayed from a CUDA
    graph (DESIGN §20).  The strand networks stay outside the graph: the trainer runs their forward
    (`pc_hair.generate_strands(iteration)`), hands the model to step(), adds its prior term to the returned loss,
    calls backward() and steps its AdamW.

    pc: the frozen head GaussianModel with the trainer's *_precomp attributes (renderer._head_block), or None for a
      hair-only model; bg: the (10,) background; lambdas: (l1, mask, orient) loss weights (opt.lambda_dl1,
      lambda_dmask, lambda_dorient); use_gt_orient_conf / train_orient_conf: the trainer's options of
      latent_strand_image_loss; capacity: the initial binning capacity in records (None: seeded from the warm-up
      iterations); pipe: the trainer's pipeline options (`debug` must be off); cameras: a cameras.CameraRig whose
      frozen views step() receives (None: cameras are plain objects with fixed tensors).

    The eager iteration (warm-ups and overflow reruns) is render_hair_segments -> image_loss_forward_backward(stage=
    "latent_strands") -> backward; the captured one computes the same values (bit for bit under
    torch.use_deterministic_algorithms(True)).  Both end in the same gradient contract.
    """

    def __init__(self, pc, width: int, height: int, bg: torch.Tensor, lambdas: Sequence[float],
                 use_gt_orient_conf: bool = True, train_orient_conf: bool = True, capacity: Optional[int] = None,
                 pipe=None, cameras=None):
        if len(lambdas) != 3:
            raise RuntimeError("CapturedLatentStrandStep: lambdas are (l1, mask, orient)")
        super().__init__("CapturedLatentStrandStep", None, width, height, bg, lambdas, capacity, pipe, bg.device,
                         needs_optimizer=False)
        self.pc, self.cameras = pc, cameras
        self.use_gt_orient_conf, self.train_orient_conf = bool(use_gt_orient_conf), bool(train_orient_conf)
        self._cam_out = torch.zeros(37, dtype=torch.float32, device=self.device)
        self._inputs = None             # the static copies of the five decoder outputs (leaves of the captured render)
        self._static_grads = None       # their gradients, written by every replay
        self._grads = None              # the gradients of the latest step (static or eager)
        self._generation = 0

    # ------------------------------------------------------------------------------------------ the iteration
    def _tail(self, renders, gts):
        """loss -> backward, shared by the eager and the captured iteration; the 8 losses land in the static words."""
        l1, lmask, lorient = self.lambdas          # (latent_strand_image_loss: no SSIM term)
        losses8, dL = ghl.image_loss_forward_backward(renders.detach(), *gts, l1, 0.0, lmask, lorient, workspace=self._ws,
                                                      stage="latent_strands", use_gt_orient_conf=self.use_gt_orient_conf,
                                                      train_orient_conf=self.train_orient_conf)
        renders.backward(dL)
        self._io[2:].copy_(losses8.view(torch.int32))
        return losses8

    def _model(self, pc_hair, tensors):
        return types.SimpleNamespace(scale=pc_hair.scale, active_sh_degree=pc_hair.active_sh_degree,
                                     **dict(zip(SEGMENT_TENSORS, tensors)))

    def _eager(self, camera, gts, pc_hair) -> torch.Tensor:
        """The eager iteration (renderer.render_hair_segments) on a side stream, on leaves that share the decoder
        outputs' storage.  A rig view is rendered frozen."""
        leaves = [getattr(pc_hair, n).detach().requires_grad_(True) for n in SEGMENT_TENSORS]

        def run():
            cam = camera
            if isinstance(cam, CameraView):
                cam = cam.rig.view(cam.index, requires_grad=False)
            pkg = renderer.render_hair_segments(cam, self.pc, self._model(pc_hair, leaves), self.pipe, self.bg)
            return self._with_nan_flag(lambda: self._tail(pkg["raw"], gts))

        losses8 = _on_side_stream(self.device, run)
        self._grads = tuple(t.grad for t in leaves)
        self._record_r(self._rows(pc_hair))
        return losses8.cpu()

    def _rows(self, pc_hair) -> int:
        head = renderer._head_block(self.pc) if self.pc is not None else None
        return (0 if head is None else int(head["xyz"].shape[0])) + int(pc_hair._xyz.shape[0])

    def _captured(self, rig_view: bool, pc_hair):
        status, n_rendered = self._io[0:1], self._io[1:2]
        status.zero_()
        camera = self._camera
        if rig_view:
            out = self._cam_out
            self.cameras.forward(self._cam_index, out=out, status=status)
            camera = {"viewmatrix": out[0:16].view(4, 4), "projmatrix": out[16:32].view(4, 4), "campos": out[32:35],
                      "tan_fov": out[35:37]}
        for t in self._inputs:
            t.grad = None
        renders, _radii = renderer.render_hair_segments_capturable(camera, self.pc, self._model(pc_hair, self._inputs),
                                                                   self.bg, self.W, self.H, self._binning, self.capacity,
                                                                   status, n_rendered)
        self._tail(renders, self._gt)
        self._static_grads = tuple(t.grad for t in self._inputs)

    def _static_inputs(self, tensors) -> None:
        """The step's own copies of the decoder outputs, reallocated (and the graph dropped) when a shape changes."""
        shapes = tuple(tuple(t.shape) for t in tensors)
        if self._inputs is None or tuple(tuple(t.shape) for t in self._inputs) != shapes:
            self._inputs = tuple(torch.zeros(sh, dtype=torch.float32, device=self.device, requires_grad=True)
                                 for sh in shapes)
            self._static_grads = None
            self._graph, self._binning, self._key = None, None, None

    def _load(self, camera, gts, rig_view: bool, tensors) -> None:
        if rig_view:
            self._cam_index.copy_(camera.rig.indices[camera.index:camera.index + 1])
        else:
            self._load_camera(camera)
        for dst, src in zip(self._gt, gts):
            if src is not None:
                dst.copy_(src)
        with torch.no_grad():
            for dst, src in zip(self._inputs, tensors):
                dst.copy_(src)
        self._grads = self._static_grads

    # ------------------------------------------------------------------------------------------ public
    def step(self, camera, gt_image, gt_mask, gt_orient_angle, gt_orient_conf, pc_hair):
        """Render, loss and backward of one iteration on `camera` for the segment rows `pc_hair` holds now (after
        `generate_strands`: `_xyz`, `_dir`, `_features_dc`, `_features_rest`, `_orient_conf`, `scale` a (1,) device
        tensor, `active_sh_degree`) -> (loss, losses).  `loss`: the 0-dim total of the image terms on the device,
        connected to the five tensors -- its backward adds grad_output times their gradients, which stay valid until
        the next step() (a backward after it raises); `losses`: the eight losses of latent_strand_image_loss (float32
        CPU tensor: total, Ll1, 0, LCE, LOR, sum of orientation weights, LOR-was-NaN, the other replaced terms).
        `camera`: a (frozen) view of `cameras` or a camera with fixed tensors."""
        self._generation += 1
        self._grads = None
        rig_view = self.cameras is not None and isinstance(camera, CameraView) and camera.rig is self.cameras
        if not rig_view:
            _check_camera(camera, "CapturedLatentStrandStep", "renderer.render_hair_segments")
        _check_no_arena("CapturedLatentStrandStep")
        if not isinstance(pc_hair.scale, torch.Tensor):
            raise RuntimeError("CapturedLatentStrandStep: pc_hair.scale must be a (1,) device tensor")
        if renderer._segment_rows(pc_hair, "CapturedLatentStrandStep") < 1:
            raise RuntimeError("CapturedLatentStrandStep: the model has no segment rows")
        if gt_orient_conf is None and self.use_gt_orient_conf:
            raise RuntimeError("CapturedLatentStrandStep: gt_orient_conf is required with use_gt_orient_conf=True")
        tensors = tuple(getattr(pc_hair, n) for n in SEGMENT_TENSORS)
        self._static_inputs(tensors)
        gts = (gt_image, gt_mask, gt_orient_angle, gt_orient_conf)
        losses8 = self._iterate(lambda: latent_capture_key(self.pc, pc_hair, self.W, self.H, self.use_gt_orient_conf,
                                                           self.train_orient_conf, self.cameras if rig_view else None),
                                lambda: self._eager(camera, gts, pc_hair),
                                lambda: self._captured(rig_view, pc_hair),
                                lambda: self._load(camera, gts, rig_view, tensors),
                                "CapturedLatentStrandStep")
        total = self._io[2:3].view(torch.float32).reshape(())
        return _StaticGradients.apply(total, self, self._generation, *tensors), losses8
