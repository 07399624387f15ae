"""Rendering and evaluation without a backward: the reference's render scripts and the trainers' `training_report`.

    render_gaussians.py  render_set (src/render_gaussians.py:31-68)     write_render_set(..., ViewRenderer(pc, pipe, bg))
    render_strands.py    render_set (src/render_strands.py:32-69)       write_render_set(..., ViewRenderer(pc, pipe, bg, pc_hair))
    training_report      (src/train_gaussians.py:232-293 and the two    evaluate_views(views, renderer, stage)
                         strand trainers' copies)

`ViewRenderer` is the forward of `renderer.render*` with nothing kept for a backward: no autograd node, no
`viewspace_points` leaf, one set of buffers reused for every view, and the sync-free first phase of the CUDA-graph
paths (DESIGN.md §16/§19/§20) with the binning capacity carried from view to view (it starts at 0: the first view
is rendered twice).  `gh_render_maps` turns the raw
(10,H,W) image into the maps the scripts save -- the bytes of `torchvision.utils.save_image` included -- in one kernel,
`gh_eval_metrics` into the numbers `training_report` prints, and `gh_eval_ssim` (`eval_ssim`, `evaluate_views(...,
ssim=True)`) adds the SSIM of loss_utils.ssim.  There is no CPU path: CPU tensors raise.
"""
from __future__ import annotations

import ctypes as C
import os
from typing import Dict, Iterable, Iterator, Optional, Sequence, Tuple

import torch

from . import _C, _capi, projection, renderer
from ._alloc import empty_rows
from ._capi import _f32, _ptr, _stream
from .graphs import STATUS_BINNING_OVERFLOW
from .losses import STAGES

__all__ = ["ViewRenderer", "sweep", "write_render_set", "maps_to_supervision", "evaluate_views", "eval_metrics",
           "eval_ssim", "MAP_NAMES", "RENDER_SET_MAPS", "METRIC_NAMES"]

# gh_render_maps' outputs in argument order: name -> (dtype, trailing shape after (H, W); floats are (1,H,W))
MAP_NAMES = ("orient_angle", "orient_conf_masked", "render_u8", "hair_mask_u8", "head_mask_u8", "orient_u8",
             "orient_vis_u8", "orient_conf_vis_u8")
_RGB = ("render_u8", "orient_vis_u8", "orient_conf_vis_u8")
_FLOAT = ("orient_angle", "orient_conf_masked")
# what render_set writes: directory -> map
RENDER_SET_MAPS = {"renders": "render_u8", "hair_masks": "hair_mask_u8", "head_masks": "head_mask_u8",
                   "orients": "orient_u8", "orients_vis": "orient_vis_u8", "orient_confs": "orient_conf_masked",
                   "orient_confs_vis": "orient_conf_vis_u8"}
# gh_eval_metrics' row
METRIC_NAMES = ("l1", "mask", "or", "psnr", "ssim", "mse_r", "mse_g", "mse_b")
MODES = ("gaussians", "strands", "segments", "hair")


def _check_want(want: Sequence[str]) -> Tuple[str, ...]:
    want = tuple(want)
    for k in want:
        if k not in MAP_NAMES:
            raise RuntimeError(f"inference: unknown map {k!r} (one of {', '.join(MAP_NAMES)})")
    return want


class ViewRenderer:
    """A forward-only renderer for one model: `render_raw(view)` is bit-identical to the raw image of

        mode "gaussians"   renderer.render(view, pc, pipe, bg)                       pc_hair is None
        mode "strands"     renderer.render_hair_strands(view, pc, pc_hair, pipe, bg)   pc_hair has `_dirs` (GaussianModelCurves)
        mode "segments"    renderer.render_hair_segments(view, pc, pc_hair, pipe, bg)  pc_hair has no `_rotation` of its own
        mode "hair"        renderer.render_hair(view, pc, pc_hair, pipe, bg)           pc_hair brings `_rotation`

    (`mode="auto"` picks by those rules).  It runs under torch.no_grad() whatever the caller's mode, and owns one set of
    buffers for (P, W, H) -- projection outputs, workspaces, the raw image, the maps -- that every view reuses; they are
    re-allocated only when the model size or the resolution changes or the binning capacity has to grow.

    The first three modes run the capturable first phase: R stays on the device, and a view whose R exceeds the
    capacity sets the overflow bit of the status word and renders nothing.  With `check=True` (the default) the status
    word is read back after the launches (one small synchronising copy) and an overflowed view is rendered again,
    once, with a capacity for the R it reported.  With `check=False` nothing is read: the caller reads `io` (int32:
    status word, R) where it reads the results anyway and hands them to `after_readback` (sweep and evaluate_views do).  Mode "hair" has
    no capturable first phase: it runs renderer.render_hair's two-phase forward, with one R read-back per view.

    The tensors returned by render_raw and render_maps are this object's buffers: the next call overwrites them."""

    def __init__(self, pc, pipe, bg: torch.Tensor, pc_hair=None, mode: str = "auto", scaling_modifier: float = 1.0):
        if mode == "auto":
            if pc_hair is None:
                mode = "gaussians"
            elif hasattr(pc_hair, "_dirs"):
                mode = "strands"
            else:
                mode = "hair" if getattr(pc_hair, "_rotation", None) is not None else "segments"
        if mode not in MODES:
            raise RuntimeError(f"ViewRenderer: unknown mode {mode!r} (one of {', '.join(MODES)}, or 'auto')")
        if (mode == "gaussians") != (pc_hair is None):
            raise RuntimeError(f"ViewRenderer: mode {mode!r} " + ("takes no pc_hair" if pc_hair is not None else "needs pc_hair"))
        self.pc, self.pc_hair, self.pipe, self.bg, self.mode = pc, pc_hair, pipe, bg, mode
        self.mod = float(scaling_modifier)
        self.device = bg.device
        if self.device.type != "cuda":
            raise RuntimeError("ViewRenderer: tensors must live on a CUDA device (there is no CPU path)")
        f = dict(dtype=torch.float32, device=self.device)
        self._camera = {"viewmatrix": torch.zeros(4, 4, **f), "projmatrix": torch.zeros(4, 4, **f),
                        "campos": torch.zeros(3, **f), "tan_fov": torch.ones(2, **f)}
        self.io = torch.zeros(2, dtype=torch.int32, device=self.device)          # status word, R
        self._io_host = torch.zeros(2, dtype=torch.int32).pin_memory()
        self.capacity = 0
        self.r_max = 0
        self.retries = 0                  # views rendered twice because their R exceeded the capacity
        self.allocations = 0              # times the per-(P, W, H) buffers were (re)allocated
        self._key = None
        self._bufs: Dict[str, object] = {}
        self._binning = None
        self._maps: Dict[str, torch.Tensor] = {}
        self._tan: Dict[tuple, torch.Tensor] = {}

    # ------------------------------------------------------------------------------------------------- buffers
    def _rows(self) -> int:
        if self.mode == "gaussians":
            return int(self.pc._xyz.shape[0])
        head = renderer._head_block(self.pc) if self.pc is not None else None
        n_head = 0 if head is None else int(head["xyz"].shape[0])
        if self.mode == "strands":
            d = self.pc_hair._dirs
            return n_head + int(d.shape[0]) * int(d.shape[1])
        return n_head + int(self.pc_hair._xyz.shape[0])

    def _ensure(self, W: int, H: int) -> None:
        P = self._rows()
        if P == 0:
            raise RuntimeError("ViewRenderer: empty model")
        key = (P, W, H)
        if key != self._key:
            dev = self.device
            geom, img, radii = _C.alloc_forward_workspaces(P, W, H, dev)
            self._bufs = {"out": projection.alloc_outputs(P, dev), "geom": geom, "img": img, "radii": radii,
                          "raw": torch.empty((_C.NUM_CHANNELS, H, W), dtype=torch.float32, device=dev)}
            if self.mode == "strands":
                self._bufs["mid"] = empty_rows(P, (3,), torch.float32, dev)       # segment midpoints (the strand rows)
            self._maps = {}
            self._key = key
            self.allocations += 1
        if self._binning is None:
            self._binning = _C.binning_workspace(self.capacity, self.device)

    def _load_camera(self, view) -> None:
        c = self._camera
        c["viewmatrix"].copy_(view.world_view_transform)
        c["projmatrix"].copy_(view.full_proj_transform)
        c["campos"].copy_(view.camera_center)
        tan = getattr(view, "tan_fov", None)             # a cameras.CameraRig view: tan(FoV / 2) on the device
        if tan is None:
            host = (renderer._tan_half(view.FoVx), renderer._tan_half(view.FoVy))
            tan = self._tan.get(host)
            if tan is None:
                if len(self._tan) > 4096:
                    self._tan.clear()
                tan = self._tan[host] = torch.tensor(host, dtype=torch.float32, device=self.device)
        c["tan_fov"].copy_(tan)

    # ------------------------------------------------------------------------------------------------- the forward
    def _launch(self, W: int, H: int) -> None:
        """First phase (projection + binning, R on the device) and gh_forward_render_capturable into the owned buffers."""
        lib = _capi.load()
        dev, b, c = self.device, self._bufs, self._camera
        out, status, n_rendered = b["out"], self.io[0:1], self.io[1:2]
        tail = (_ptr(out["means2D"]), _ptr(out["colors"]), _ptr(out["opacity"]), _ptr(out["conic"]), _ptr(out["visible"]),
                _ptr(b["radii"]), _ptr(b["geom"]), _ptr(b["img"]), _ptr(self._binning), int(self.capacity), _ptr(status),
                _ptr(n_rendered), 0, _stream(dev))
        cam = (c["viewmatrix"], c["projmatrix"], c["campos"], c["tan_fov"])
        head_cfg = (projection.encode_flags(projection.HEAD_PRECOMP), float(projection.HEAD_PRECOMP["det_eps"]))
        if self.mode == "gaussians":
            pc = self.pc
            pi = projection.pack_inputs(pc._xyz, pc._scaling, pc._rotation, None, pc._features_dc, pc._features_rest,
                                        pc._opacity, pc._label, pc._orient_conf, *cam[:3], 0.0, 0.0, W, H,
                                        pc.active_sh_degree, self.mod, projection.GAUSSIAN_MODEL)
            _capi.check(lib.gh_project_forward_binned_capturable(*projection._common_args_capturable(pi, cam[3]), *tail))
            P = pi.P
        else:
            hair = self.pc_hair
            scale = hair.scale
            if not isinstance(scale, torch.Tensor):
                scale = torch.full((1,), float(scale), dtype=torch.float32, device=dev)
            head = renderer._head_block(self.pc) if self.pc is not None else None
            if self.mode == "strands":
                sp = projection.pack_strand_inputs(head, hair.pts_origins, hair._dirs, scale, hair._features_dc,
                                                   hair._features_rest, hair._orient_conf, *cam, W, H,
                                                   hair.active_sh_degree, self.mod)
                rows, mid = (sp.n_head, sp.S, sp.L, W, H), (_ptr(sp.origins), *sp.common(), _ptr(b["mid"]))
                fn = lib.gh_hair_strands_forward_binned_capturable
            else:
                renderer._segment_rows(hair, "ViewRenderer")
                sp = projection.pack_segment_inputs(head, hair._xyz, hair._dir, scale, hair._features_dc,
                                                    hair._features_rest, hair._orient_conf, *cam, W, H,
                                                    hair.active_sh_degree, self.mod)
                rows, mid = (sp.n_head, sp.N, W, H), sp.common()
                fn = lib.gh_hair_segments_forward_binned_capturable
            hd = sp.head or {}
            _capi.check(fn(*rows, *(_ptr(hd.get(k)) for k in ("xyz", "scaling", "rotation", "f_dc", "f_rest", "opacity")),
                           *head_cfg, *mid, *tail))
            P = sp.P
        _capi.check(lib.gh_forward_render_capturable(
            P, W, H, int(self.capacity), _ptr(_f32(self.bg, "background", dev)), _ptr(out["colors"]), _ptr(b["geom"]),
            _ptr(self._binning), _ptr(b["img"]), _ptr(b["raw"]), 0, _stream(dev)))

    def _grow(self, R: int) -> None:
        self.r_max = max(self.r_max, int(R))
        self.capacity = _C.capacity_for(self.r_max)
        self._binning = None

    def _render(self, view, check: bool) -> torch.Tensor:
        W, H = int(view.image_width), int(view.image_height)
        with torch.no_grad(), torch.cuda.device(self.device):
            if self.mode == "hair":
                raw = renderer.render_hair(view, self.pc, self.pc_hair, self.pipe, self.bg, self.mod)["raw"]
                self._bufs = {"raw": raw.detach()}
                if self._key != ("hair", W, H):
                    self._key, self._maps = ("hair", W, H), {}
                return self._bufs["raw"]
            self._ensure(W, H)
            self._load_camera(view)
            self.io.zero_()
            self._launch(W, H)
            if check:
                self._io_host.copy_(self.io, non_blocking=True)
                torch.cuda.current_stream(self.device).synchronize()
                self.after_readback(view, int(self._io_host[0]), int(self._io_host[1]), render=True)
        return self._bufs["raw"]

    def after_readback(self, view, status: int, R: int, render: bool = False) -> bool:
        """What a caller of `check=False` does with the (status word, R) it read back for `view`: records R, and on
        overflow raises the capacity (and, with `render`, renders the view again).  -> whether the view overflowed."""
        self.r_max = max(self.r_max, int(R))
        if not status & STATUS_BINNING_OVERFLOW:
            return False
        self.retries += 1
        self._grow(R)
        if render:
            W, H = int(view.image_width), int(view.image_height)
            with torch.no_grad(), torch.cuda.device(self.device):
                self._ensure(W, H)
                self._load_camera(view)
                self.io.zero_()
                self._launch(W, H)
        return True

    def render_raw(self, view, check: bool = True) -> torch.Tensor:
        """The raw (10,H,W) image of `view` (image 0..2, mask 3..4, dir 5..7, orientation confidence 8, depth 9) -- this
        object's buffer, overwritten by the next call."""
        return self._render(view, check)

    def render_maps(self, view, want: Sequence[str] = MAP_NAMES, check: bool = True) -> Dict[str, torch.Tensor]:
        """`view` rendered and reduced to the maps named in `want` (MAP_NAMES; include/gh_rasterizer.h, gh_render_maps):
        float maps (1,H,W), grey byte maps (H,W), colour byte maps (H,W,3).  Device tensors owned by this object,
        overwritten by the next call."""
        want = _check_want(want)
        raw = self._render(view, check)
        return self.maps_of(raw, want)

    def maps_of(self, raw: torch.Tensor, want: Sequence[str] = MAP_NAMES) -> Dict[str, torch.Tensor]:
        """gh_render_maps on a raw (10,H,W) image, into this object's map buffers."""
        H, W = int(raw.shape[1]), int(raw.shape[2])
        dev = self.device
        for k in want:
            t = self._maps.get(k)
            shape = (1, H, W) if k in _FLOAT else ((H, W, 3) if k in _RGB else (H, W))
            if t is None or tuple(t.shape) != shape:
                self._maps[k] = torch.empty(shape, dtype=torch.float32 if k in _FLOAT else torch.uint8, device=dev)
        with torch.cuda.device(dev):
            _capi.check(_capi.load().gh_render_maps(W, H, _ptr(raw), *(_ptr(self._maps[k]) if k in want else None
                                                                       for k in MAP_NAMES), _stream(dev)))
        return {k: self._maps[k] for k in want}


# ------------------------------------------------------------------------------------------------------- the sweep
def sweep(view_renderer, views: Iterable, want: Sequence[str] = MAP_NAMES, depth: int = 2) -> Iterator[Tuple[object, Dict[str, torch.Tensor]]]:
    """Render `views` and yield (view, maps on the host) one view behind the GPU: the maps of view i are copied into one
    of `depth` rotating pinned host buffer sets on a copy stream while the caller still works on view i - 1 (its PNG
    encoding, say), and the render of view i + 1 is launched as soon as the caller asks for the next item.  One host
    wait per step (on the copy's event) replaces the blocking copy per saved map.  The yielded tensors are this
    generator's buffers: valid until `depth - 1` further items have been taken.  No threads, no processes; the stream,
    events and pinned buffers are released when the generator is exhausted or closed.

    An overflowed view (ViewRenderer's status word, copied with the maps) is rendered again before it is yielded."""
    want = _check_want(want)
    if depth < 2:
        raise RuntimeError("sweep: depth must be at least 2 (one buffer set with the caller, one being filled)")
    on_gpu = getattr(view_renderer, "device", torch.device("cpu")).type == "cuda"
    slots, copy_stream = [], None
    try:
        pending = None                     # (view, slot) whose copy is in flight
        for i, view in enumerate(views):
            # (nothing is known about R before the first view: check it at once instead of overflowing twice)
            maps = view_renderer.render_maps(view, want, check=getattr(view_renderer, "capacity", 1) == 0)
            if len(slots) < depth:
                slots.append({"maps": {}, "io": torch.zeros(2, dtype=torch.int32, pin_memory=on_gpu),
                              "done": torch.cuda.Event() if on_gpu else None})
            slot = slots[i % depth]
            if on_gpu and copy_stream is None:
                copy_stream = torch.cuda.Stream(device=view_renderer.device)
            _copy_out(view_renderer, maps, slot, copy_stream)
            if pending is not None:
                yield _finish(view_renderer, *pending, want, copy_stream)
            pending = (view, slot)
        if pending is not None:
            yield _finish(view_renderer, *pending, want, copy_stream)
            pending = None
    finally:
        if copy_stream is not None:
            copy_stream.synchronize()
        for s in slots:
            s.clear()
        slots.clear()
        copy_stream = None


def _copy_out(view_renderer, maps, slot, copy_stream) -> None:
    """The device maps and the status words into `slot` on the copy stream; the render stream then waits for the copy,
    because the next render overwrites the device maps."""
    host = slot["maps"]
    for k, t in maps.items():
        h = host.get(k)
        if h is None or h.shape != t.shape:
            host[k] = torch.empty(t.shape, dtype=t.dtype, pin_memory=copy_stream is not None)
    for k in [k for k in host if k not in maps]:
        del host[k]
    if copy_stream is None:
        for k, t in maps.items():
            host[k].copy_(t)
        slot["io"].copy_(view_renderer.io)
        return
    main = torch.cuda.current_stream(view_renderer.device)
    copy_stream.wait_stream(main)
    with torch.cuda.stream(copy_stream):
        for k, t in maps.items():
            host[k].copy_(t, non_blocking=True)
        slot["io"].copy_(view_renderer.io, non_blocking=True)
        slot["done"].record(copy_stream)
    main.wait_event(slot["done"])


def _finish(view_renderer, view, slot, want, copy_stream):
    if slot["done"] is not None:
        slot["done"].synchronize()
    status, R = int(slot["io"][0]), int(slot["io"][1])
    if view_renderer.after_readback(view, status, R):
        maps = view_renderer.render_maps(view, want, check=True)
        _copy_out(view_renderer, maps, slot, copy_stream)
        if slot["done"] is not None:
            slot["done"].synchronize()
    return view, slot["maps"]


# ------------------------------------------------------------------------------------------------- the render scripts
def _basename(view) -> str:
    return os.path.basename(view.image_name).split(".")[0]


def save_png(u8: torch.Tensor, path: str) -> None:
    """A byte map as torchvision.utils.save_image writes it: (H,W,3) as RGB, (H,W) as RGB with three equal channels."""
    from PIL import Image
    a = u8.numpy()
    if a.ndim == 2:
        a = a[:, :, None].repeat(3, axis=2)
    Image.fromarray(a).save(path)


def write_render_set(model_path: str, name: str, iteration, views, view_renderer, scene_suffix: str = "") -> str:
    """The body of the reference's render_set (src/render_gaussians.py:31-68, src/render_strands.py:32-69):
    <model_path>/<name><scene_suffix>/ours_<iteration>/{renders,hair_masks,head_masks,orients,orients_vis,
    orient_confs_vis}/<view>.png and orient_confs/<view>.pth (the float (1,H,W) orient_conf * hair_mask), rendered by
    `view_renderer` through `sweep`.  -> the ours_<iteration> directory."""
    root = os.path.join(model_path, f"{name}{scene_suffix}", "ours_{}".format(iteration))
    for d in RENDER_SET_MAPS:
        os.makedirs(os.path.join(root, d), exist_ok=True)
    for view, maps in sweep(view_renderer, views, tuple(RENDER_SET_MAPS.values())):
        base = _basename(view)
        for d, k in RENDER_SET_MAPS.items():
            if k in _FLOAT:
                torch.save(maps[k].clone(), os.path.join(root, d, base + ".pth"))
            else:
                save_png(maps[k], os.path.join(root, d, base + ".png"))
    return root


def maps_to_supervision(maps: Dict[str, torch.Tensor], binarize_masks: bool = False) -> Dict[str, torch.Tensor]:
    """The ground truth tensors the reference's loadCam builds from a render set at the resolution it was rendered at
    (src/utils/camera_utils.py:51-78 with --load_synthetic_rgba --load_synthetic_geom): bytes / 255, the first channel
    of the grey maps, masks optionally thresholded at 0.5, the confidence as it is.  `maps`: render_u8, hair_mask_u8,
    head_mask_u8, orient_u8 and orient_conf_masked of render_maps or sweep (any device).  -> image (3,H,W), mask_hair,
    mask_body, orient_angle, orient_conf (1,H,W) float32, the same values as after the PNG round trip."""
    unit = lambda u8: u8 / 255.0  # noqa: E731
    out = {"image": unit(maps["render_u8"]).permute(2, 0, 1), "mask_hair": unit(maps["hair_mask_u8"])[None],
           "mask_body": unit(maps["head_mask_u8"])[None], "orient_angle": unit(maps["orient_u8"])[None],
           "orient_conf": maps["orient_conf_masked"].float().clone()}
    if binarize_masks:
        out["mask_hair"], out["mask_body"] = (out["mask_hair"] >= 0.5).float(), (out["mask_body"] >= 0.5).float()
    return out


# --------------------------------------------------------------------------------------------------------- evaluation
def eval_workspace(W: int, H: int, device: torch.device) -> torch.Tensor:
    nbytes = C.c_size_t()
    _capi.check(_capi.load().gh_eval_metrics_workspace_size(int(W), int(H), C.byref(nbytes)))
    return torch.empty((nbytes.value + 7) // 8, dtype=torch.float64, device=device)


def eval_metrics(raw: torch.Tensor, gt_image: torch.Tensor, gt_mask: torch.Tensor, gt_orient_angle: torch.Tensor,
                 gt_orient_conf: torch.Tensor, stage: str, row: torch.Tensor, workspace: Optional[torch.Tensor] = None) -> None:
    """gh_eval_metrics: the METRIC_NAMES of one view from its raw (10,H,W) render and ground truth maps ((3,H,W),
    (2,H,W) hair then head, (1,H,W), (1,H,W), device float32) into `row`, a contiguous float32 (8,) device tensor such
    as one row of an (N,8) buffer.  `stage`: "appearance", "strands" or "latent_strands".  No host synchronisation."""
    if stage not in STAGES:
        raise RuntimeError(f"eval_metrics: unknown stage {stage!r} (one of {', '.join(STAGES)})")
    dev = raw.device
    H, W = int(raw.shape[1]), int(raw.shape[2])
    gts = []
    for name, t, c in (("gt_image", gt_image, 3), ("gt_mask", gt_mask, 2), ("gt_orient_angle", gt_orient_angle, 1),
                       ("gt_orient_conf", gt_orient_conf, 1)):
        if tuple(t.shape) != (c, H, W):
            raise RuntimeError(f"eval_metrics: {name} must have shape {(c, H, W)}, got {tuple(t.shape)}")
        gts.append(_f32(t, name, dev))
    if row.dtype != torch.float32 or row.numel() != 8 or not row.is_contiguous() or row.device != dev:
        raise RuntimeError("eval_metrics: row must be a contiguous float32 (8,) tensor on the render's device")
    if workspace is None:
        workspace = eval_workspace(W, H, dev)
    with torch.cuda.device(dev):
        _capi.check(_capi.load().gh_eval_metrics(W, H, STAGES[stage], _ptr(_f32(raw, "render", dev)), *(_ptr(g) for g in gts),
                                                 _ptr(workspace), workspace.numel() * workspace.element_size(), _ptr(row),
                                                 _stream(dev)))


def ssim_workspace(B: int, W: int, H: int, device: torch.device) -> torch.Tensor:
    nbytes = C.c_size_t()
    _capi.check(_capi.load().gh_eval_ssim_workspace_size(int(B), int(W), int(H), C.byref(nbytes)))
    return torch.empty((nbytes.value + 7) // 8, dtype=torch.float64, device=device)


_DTYPES = {torch.float32: 0, torch.uint8: 1}          # GH_DTYPE_FLOAT32, GH_DTYPE_UINT8
_CLAMP1, _CLAMP2, _CLAMP_MASK = 1, 2, 4               # GH_SSIM_CLAMP_IMG1, _IMG2, _MASK


def _pairs(t: torch.Tensor, name: str, dev: torch.device, C_: int) -> Tuple[torch.Tensor, int]:
    """`t` as B planar (C_,H,W) blocks: (B,C_,H,W), or (C_,H,W) for B = 1; each block contiguous, the pair stride free
    (so raw[:3] of a (10,H,W) render or x[:, :3] of a (B,10,H,W) stack is read in place).  -> (tensor, pair stride)."""
    if not t.is_cuda:
        raise RuntimeError(f"eval_ssim: '{name}' must be a CUDA tensor (there is no CPU path)")
    if t.device != dev:
        raise RuntimeError(f"eval_ssim: '{name}' is on {t.device}, expected {dev}")
    if t.dim() == 3:
        t = t.unsqueeze(0)
    if t.dim() != 4 or t.shape[1] != C_:
        raise RuntimeError(f"eval_ssim: '{name}' must have shape (B,{C_},H,W) or ({C_},H,W), got {tuple(t.shape)}")
    if t.requires_grad:
        t = t.detach()
    H, W = int(t.shape[2]), int(t.shape[3])
    if t.stride()[1:] != (H * W, W, 1) and not (C_ == 1 and t.stride()[2:] == (W, 1)):
        t = t.contiguous()
    if t.data_ptr() % t.element_size():
        t = t.clone()
    return t, (int(t.stride(0)) if t.shape[0] > 1 else C_ * H * W)


def _out_vec(t: Optional[torch.Tensor], name: str, B: int, dev: torch.device) -> Tuple[Optional[torch.Tensor], int]:
    if t is None:
        return None, 0
    if t.dtype != torch.float32 or t.dim() != 1 or t.numel() != B or t.device != dev:
        raise RuntimeError(f"eval_ssim: {name} must be a float32 ({B},) tensor on {dev} (any stride, e.g. rows[:, 4])")
    return t, int(t.stride(0))


def eval_ssim(img1: torch.Tensor, img2: torch.Tensor, out_ssim: torch.Tensor, out_psnr: Optional[torch.Tensor] = None,
              clamp1: bool = False, mask: Optional[torch.Tensor] = None, workspace: Optional[torch.Tensor] = None,
              clamp2: bool = False, clamp_mask: bool = False, debug: bool = False) -> None:
    """gh_eval_ssim: loss_utils.ssim(img1[i], img2[i]) into out_ssim[i] and image_utils.psnr(img1[i], img2[i]) into
    out_psnr[i] (optional) for B pairs, in one launch.

    img1, img2: (B,3,H,W) or (3,H,W) device tensors, float32 or uint8 (x / 255 as torchvision's to_tensor rounds it; a
    uint8 image and its to_tensor conversion give the same bits); each (3,H,W) block contiguous, the pair stride free.
    clamp1 / clamp2 clamp that image to [0, 1].  mask: (B,1,H,W) or (1,H,W) float32, multiplied into both images
    (clamped to [0, 1] first with clamp_mask).  out_ssim, out_psnr: float32 (B,) device tensors of any stride, such as
    rows[:, 4] and rows[:, 3] of an (N,8) metrics buffer.  workspace: ssim_workspace(B, W, H, device) or None.
    No host synchronisation (unless debug)."""
    dev = img1.device
    for name, t in (("img1", img1), ("img2", img2)):
        if t.dtype not in _DTYPES:
            raise RuntimeError(f"eval_ssim: '{name}' must be float32 or uint8, got {t.dtype}")
    a, s1 = _pairs(img1, "img1", dev, 3)
    b, s2 = _pairs(img2, "img2", dev, 3)
    if a.shape != b.shape:
        raise RuntimeError(f"eval_ssim: img1 {tuple(a.shape)} and img2 {tuple(b.shape)} differ")
    B, H, W = int(a.shape[0]), int(a.shape[2]), int(a.shape[3])
    sm = 0
    if mask is not None:
        if mask.dtype != torch.float32:
            raise RuntimeError(f"eval_ssim: mask must be float32, got {mask.dtype}")
        mask, sm = _pairs(mask, "mask", dev, 1)
        if tuple(mask.shape) != (B, 1, H, W):
            raise RuntimeError(f"eval_ssim: mask must have shape {(B, 1, H, W)}, got {tuple(mask.shape)}")
    o_s, ss = _out_vec(out_ssim, "out_ssim", B, dev)
    if o_s is None:
        raise RuntimeError("eval_ssim: out_ssim is required")
    o_p, sp = _out_vec(out_psnr, "out_psnr", B, dev)
    if workspace is None:
        workspace = ssim_workspace(B, W, H, dev)
    flags = (_CLAMP1 if clamp1 else 0) | (_CLAMP2 if clamp2 else 0) | (_CLAMP_MASK if clamp_mask else 0)
    with torch.cuda.device(dev):
        _capi.check(_capi.load().gh_eval_ssim(B, W, H, _ptr(a), _DTYPES[a.dtype], s1, _ptr(b), _DTYPES[b.dtype], s2,
                                              _ptr(mask), sm, flags, _ptr(o_s), ss, _ptr(o_p), sp, _ptr(workspace),
                                              workspace.numel() * workspace.element_size(), int(bool(debug)),
                                              _stream(dev)))


def _gt_of(view, dev):
    g = lambda t: t.to(dev, non_blocking=True)  # noqa: E731
    return g(view.original_image), g(view.original_mask), g(view.original_orient_angle), g(view.original_orient_conf)


def evaluate_views(views, view_renderer: ViewRenderer, stage: str, ssim: bool = False) -> Dict[str, float]:
    """training_report's loop over `views` (src/train_gaussians.py:246-281 and the strand trainers' copies): per view the
    ground truth maps go to the device (`original_image`, `original_mask`, `original_orient_angle`,
    `original_orient_conf`), the view is rendered and gh_eval_metrics fills row i of an (N,8) device buffer; the buffer
    and the views' status words are read back once after the last view, an overflowed view is redone, and the means
    over the views are taken in float64 on the host.  -> {"l1", "mask" ("ce" in the latent strand stage), "or", "psnr"}
    plus "mse_r", "mse_g", "mse_b".

    ssim=True adds "ssim": gh_eval_ssim writes slot 4 of each row, on the same stream after gh_eval_metrics, from the
    pair the row's l1 term uses -- the render's image channels and gt_image, both clamped to [0, 1], and in the
    latent strand stage both multiplied by the clamped gt_mask[:1].  The other slots are the same bits as without it."""
    if not isinstance(ssim, bool):
        raise TypeError(f"evaluate_views: ssim must be True or False, got {ssim!r}")
    views = list(views)
    if not views:
        return {}
    dev = view_renderer.device
    rows = torch.zeros(len(views), 8, dtype=torch.float32, device=dev)
    ios = torch.zeros(len(views), 2, dtype=torch.int32, device=dev)
    ws = None

    def one(i, view, check):
        nonlocal ws
        raw = view_renderer.render_raw(view, check=check)
        if ws is None or ws[0] != tuple(raw.shape):
            H, W = int(raw.shape[1]), int(raw.shape[2])
            ws = (tuple(raw.shape), eval_workspace(W, H, dev), ssim_workspace(1, W, H, dev) if ssim else None)
        gts = _gt_of(view, dev)
        eval_metrics(raw, *gts, stage, rows[i], ws[1])
        if ssim:
            eval_ssim(raw[:3], gts[0], rows[i, 4:5], clamp1=True, clamp2=True, workspace=ws[2],
                      mask=gts[1][:1] if stage == "latent_strands" else None, clamp_mask=True)
        ios[i].copy_(view_renderer.io)

    for i, view in enumerate(views):
        one(i, view, view_renderer.capacity == 0)       # nothing is known about R before the first view: check it at once
    host_io = ios.cpu()                                     # the one synchronisation of the sweep
    redo = [i for i, v in enumerate(views)
            if view_renderer.after_readback(v, int(host_io[i, 0]), int(host_io[i, 1]))]
    for i in redo:
        one(i, views[i], True)
    m = rows.cpu().double().mean(dim=0)
    names = list(METRIC_NAMES)
    if stage == "latent_strands":
        names[1] = "ce"
    return {k: float(m[j]) for j, k in enumerate(names) if k != "ssim" or ssim}
