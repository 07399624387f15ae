"""Fused projection preamble ("next" row 1 of SURVEY.md 8f): the PyTorch code the reference runs before every
rasterizer call, as one forward and one backward kernel (csrc/gh_project.cu) behind the C ABI
(`gh_project_forward` / `gh_project_backward`, include/gh_rasterizer.h).

Replaces, for one camera, on the RAW parameters a model stores:

    GaussianModel.get_conic / get_covariance_2d / get_covariance      src/scene/gaussian_model.py:230-315
    get_mean_2d :317-337, get_depths :339-342, get_direction_2d :344-393, filter_points :143-228
    the activations get_scaling / get_opacity / get_label / get_orient_conf   :106-141
    eval_sh + clamp, the 10-channel feature concatenation, the mask gathers    src/gaussian_renderer/__init__.py:29-83
    (and the strand models' copies of the same functions, src/scene/gaussian_model_latent_strands.py:109-440)

including the gradients w.r.t. the camera matrices, which the reference gets from autograd because cameras are
trainable (src/scene/cameras.py:124-150).  `renderer.py` builds `render()` / `render_hair()` on top of it.
There is no CPU path: CPU tensors raise.
"""
from __future__ import annotations

import ctypes as C
from typing import Dict, Optional

import torch

from . import _capi
from ._alloc import carve_segments, empty_rows, segments_floats
from ._capi import _f32, _ptr, _stream

# activation / mode codes (GhProjArgs in csrc/gh_project_math.h)
GAUSSIAN_MODEL = dict(scale_act=1, opacity_act=1, label_act=1, conf_act=1, dir_mode=0, det_eps=1e-12)   # gaussian_model.py
HAIR_MODEL = dict(scale_act=0, opacity_act=2, label_act=2, conf_act=1, dir_mode=1, det_eps=1e-7)         # gaussian_model_latent_strands.py
# the frozen head Gaussians inside render_hair(): activated scales / opacities, label = dir2D = confidence = 0
HEAD_PRECOMP = dict(scale_act=0, opacity_act=0, label_act=3, conf_act=3, dir_mode=2, det_eps=1e-12)
# GaussianModelCurves (gaussian_model_strands.py) rendered from its polylines: HAIR_MODEL semantics, but every Gaussian is
# a segment whose scales / rotation the kernels derive from dirs[i]; `scaling` is the (1,) strand thickness, no rotation
HAIR_STRANDS = dict(HAIR_MODEL, strands=1)


def encode_flags(cfg: Dict[str, object]) -> int:
    return (int(cfg["scale_act"]) & 3) | ((int(cfg["opacity_act"]) & 3) << 2) | ((int(cfg["label_act"]) & 3) << 4) | \
           ((int(cfg["conf_act"]) & 3) << 6) | ((int(cfg["dir_mode"]) & 3) << 8) | ((int(cfg.get("strands", 0)) & 1) << 10)


class ProjectionInputs:
    """The (detached, contiguous) tensors of one projection call, kept between forward and backward."""
    __slots__ = ("P", "W", "H", "xyz", "scaling", "rotation", "dirs", "f_dc", "f_rest", "opacity", "label", "conf",
                 "V", "Pm", "campos", "tanx", "tany", "mod", "sh_degree", "flags", "det_eps", "device")


def pack_inputs(xyz, scaling, rotation, dirs, f_dc, f_rest, opacity, label, conf, viewmatrix, projmatrix, campos,
                tanfovx: float, tanfovy: float, width: int, height: int, sh_degree: int, scaling_modifier: float,
                cfg: Dict[str, object]) -> ProjectionInputs:
    if xyz.ndim != 2 or xyz.size(1) != 3:
        raise RuntimeError("means3D must have dimensions (num_points, 3)")
    dev = xyz.device
    pi = ProjectionInputs()
    pi.device = dev
    pi.P, pi.W, pi.H = int(xyz.size(0)), int(width), int(height)
    pi.xyz = _f32(xyz, "xyz", dev)
    pi.scaling = _f32(scaling, "scaling", dev)
    pi.rotation = _f32(rotation, "rotation", dev, align=16)
    pi.dirs = _f32(dirs, "dirs", dev)
    pi.f_dc = _f32(f_dc, "features_dc", dev)
    pi.f_rest = _f32(f_rest, "features_rest", dev)
    pi.opacity = _f32(opacity, "opacity", dev)
    pi.label = _f32(label, "label", dev)
    pi.conf = _f32(conf, "orient_conf", dev)
    pi.V = _f32(viewmatrix, "viewmatrix", dev)
    pi.Pm = _f32(projmatrix, "projmatrix", dev)
    pi.campos = _f32(campos, "campos", dev)
    pi.tanx, pi.tany = float(tanfovx), float(tanfovy)
    pi.mod, pi.sh_degree = float(scaling_modifier), int(sh_degree)
    pi.flags, pi.det_eps = encode_flags(cfg), float(cfg["det_eps"])
    n = pi.P
    if cfg.get("strands", 0):
        if pi.scaling is None or pi.scaling.numel() != 1 or pi.rotation is not None:
            raise RuntimeError("projection: strand mode takes the strand thickness as a (1,) 'scaling' tensor and no rotation")
        per_row = (("dirs", pi.dirs, 3), ("features_dc", pi.f_dc, 3), ("orient_conf", pi.conf, 1))
    else:
        per_row = (("scaling", pi.scaling, 3), ("rotation", pi.rotation, 4), ("features_dc", pi.f_dc, 3))
    for name, t, per in per_row:
        if t is None or t.numel() != n * per:
            raise RuntimeError(f"projection: '{name}' must have {per} floats per Gaussian")
    if pi.sh_degree > 0 and (pi.f_rest is None or pi.f_rest.numel() != n * 45):
        raise RuntimeError("projection: 'features_rest' must be (P, 15, 3) for sh_degree > 0")
    return pi


def _common_args(pi: ProjectionInputs):
    return (pi.P, pi.W, pi.H, _ptr(pi.xyz), _ptr(pi.scaling), _ptr(pi.rotation), _ptr(pi.dirs), _ptr(pi.f_dc), _ptr(pi.f_rest),
            _ptr(pi.opacity), _ptr(pi.label), _ptr(pi.conf), _ptr(pi.V), _ptr(pi.Pm), _ptr(pi.campos),
            pi.tanx, pi.tany, pi.mod, pi.sh_degree, pi.flags, pi.det_eps)


def _common_args_capturable(pi: ProjectionInputs, tan_fov: torch.Tensor):
    """_common_args with tan(fov / 2) from the device float[2] `tan_fov` (the capturable entry points)."""
    return (pi.P, pi.W, pi.H, _ptr(pi.xyz), _ptr(pi.scaling), _ptr(pi.rotation), _ptr(pi.dirs), _ptr(pi.f_dc), _ptr(pi.f_rest),
            _ptr(pi.opacity), _ptr(pi.label), _ptr(pi.conf), _ptr(pi.V), _ptr(pi.Pm), _ptr(pi.campos),
            _ptr(_f32(tan_fov, "tan_fov", pi.device)), pi.mod, pi.sh_degree, pi.flags, pi.det_eps)


def alloc_outputs(P: int, dev: torch.device, want_cov3D: bool = False, means2D_out: Optional[torch.Tensor] = None):
    f32 = torch.float32
    return {"means2D": means2D_out if means2D_out is not None else empty_rows(P, (3,), f32, dev),
            "colors": empty_rows(P, (10,), f32, dev), "opacity": empty_rows(P, (1,), f32, dev), "conic": empty_rows(P, (3,), f32, dev),
            "visible": empty_rows(P, (), torch.uint8, dev),
            "cov3D": empty_rows(P, (6,), f32, dev) if want_cov3D else None}


def project_forward(pi: ProjectionInputs, want_cov3D: bool = False, means2D_out: Optional[torch.Tensor] = None,
                    out: Optional[Dict[str, torch.Tensor]] = None):
    """-> dict(means2D (P,3) NDC, colors (P,10), opacity (P,1), conic (P,3) [zeros where culled], visible (P) uint8,
    cov3D (P,6) or None).  `means2D_out`: write the NDC means into this (P,3) float32 tensor instead of allocating;
    `out`: write everything into these preallocated tensors (e.g. row slices of larger buffers)."""
    lib = _capi.load()
    dev, P = pi.device, pi.P
    if out is None:
        out = alloc_outputs(P, dev, want_cov3D, means2D_out)
    else:
        for k, v in out.items():
            if v is not None and (not v.is_contiguous() or v.shape[0] != P):
                raise RuntimeError(f"projection: preallocated output '{k}' must be contiguous with {P} rows")
    if P == 0:
        return out
    with torch.cuda.device(dev):
        _capi.check(lib.gh_project_forward(*_common_args(pi), _ptr(out["means2D"]), _ptr(out["colors"]), _ptr(out["opacity"]),
                                           _ptr(out["conic"]), _ptr(out["cov3D"]), _ptr(out["visible"]), _stream(dev)))
    return out


def project_forward_binned(pi: ProjectionInputs, means2D_out: Optional[torch.Tensor] = None, binning: bool = False):
    """project_forward AND the rasterizer's first phase in one pass over the Gaussians (gh_project_forward_binned):
    -> (out dict as project_forward, radii (P,) int32, geomBuffer, imgBuffer, num_rendered, max_tile_len).  Continue
    with `_C.forward_render`.  Bit-identical to project_forward followed by `_C.rasterize_gaussians` on its outputs
    with prefiltered=False (tests/test_gpu_projection.py).

    `binning=True` also runs the bucket scatter in the first phase when the capacity hint of `_C.binning_hint` covers R,
    and appends the binning buffer it filled (or None) to the tuple: hand it to `_C.forward_render(..., binned=...)`."""
    from . import _C
    lib = _capi.load()
    dev, P = pi.device, pi.P
    if P == 0:
        raise RuntimeError("project_forward_binned: empty model (use project_forward + rasterize_gaussians)")
    out = alloc_outputs(P, dev, False, means2D_out)
    geom, img, radii = _C.alloc_forward_workspaces(P, int(pi.W), int(pi.H), dev)
    key = (dev.index, P, int(pi.W), int(pi.H))
    buf, capacity = _C.binning_hint(key) if binning else (None, 0)
    n_rendered, max_len, emitted = C.c_int(0), C.c_int(0), C.c_int(0)
    with torch.cuda.device(dev):
        _capi.check(lib.gh_project_forward_binned(
            *_common_args(pi), _ptr(out["means2D"]), _ptr(out["colors"]), _ptr(out["opacity"]), _ptr(out["conic"]), None,
            _ptr(out["visible"]), _ptr(radii), _ptr(geom), _ptr(img), _ptr(buf), capacity,
            C.byref(n_rendered), C.byref(max_len), C.byref(emitted), _stream(dev)))
    R = int(n_rendered.value)
    if not binning:
        return out, radii, geom, img, R, int(max_len.value)
    _C.binning_record(key, R)
    return out, radii, geom, img, R, int(max_len.value), (buf if emitted.value else None)


def project_forward_binned_capturable(pi: ProjectionInputs, tan_fov: torch.Tensor, binning: torch.Tensor, capacity: int,
                                      status: torch.Tensor, num_rendered: Optional[torch.Tensor] = None,
                                      means2D_out: Optional[torch.Tensor] = None):
    """gh_project_forward_binned_capturable: project_forward_binned with tan(fov / 2) from the device (2,) tensor
    `tan_fov`, emit into the caller's `binning` buffer of `capacity` records (_C.binning_workspace) and R left on the
    device (written to the int32 (1,) `num_rendered` when given).  R > capacity sets bit 0 of the int32 (1,) `status`
    and renders an empty frame (include/gh_rasterizer.h).  -> (out dict as project_forward, radii, geomBuffer,
    imgBuffer); continue with `_C.forward_render_capturable`.  No host synchronisation."""
    from . import _C
    lib = _capi.load()
    dev, P = pi.device, pi.P
    if P == 0:
        raise RuntimeError("project_forward_binned_capturable: empty model")
    out = alloc_outputs(P, dev, False, means2D_out)
    geom, img, radii = _C.alloc_forward_workspaces(P, int(pi.W), int(pi.H), dev)
    with torch.cuda.device(dev):
        _capi.check(lib.gh_project_forward_binned_capturable(
            *_common_args_capturable(pi, tan_fov), _ptr(out["means2D"]), _ptr(out["colors"]), _ptr(out["opacity"]),
            _ptr(out["conic"]), _ptr(out["visible"]), _ptr(radii), _ptr(geom), _ptr(img), _ptr(binning), int(capacity),
            _ptr(status), _ptr(num_rendered), 0, _stream(dev)))
    return out, radii, geom, img


_CAM_WS: Dict[tuple, torch.Tensor] = {}


def _camera_workspace(P: int, dev: torch.device) -> torch.Tensor:
    nbytes = C.c_size_t()
    _capi.check(_capi.load().gh_project_workspace_size(P, C.byref(nbytes)))
    key = (dev.index, torch.cuda.current_stream(dev).cuda_stream)
    ws = _CAM_WS.get(key)
    if ws is None or ws.numel() < nbytes.value:
        ws = torch.zeros(nbytes.value, dtype=torch.uint8, device=dev)
        _CAM_WS[key] = ws
    return ws


# the parameter gradients of project_backward, in the order of the flat gradient arena (segment padding:
# _alloc.segments_floats); `dirs` is last and only there for models that have direction vectors
GRAD_SEGMENTS = (("rotation", 4, (4,)), ("xyz", 3, (3,)), ("scaling", 3, (3,)), ("f_dc", 3, (1, 3)), ("f_rest", 45, (15, 3)),
                 ("opacity", 1, (1,)), ("label", 1, (1,)), ("conf", 1, (1,)), ("dirs", 3, (3,)))


def _grad_layout(with_dirs: bool):
    return GRAD_SEGMENTS if with_dirs else GRAD_SEGMENTS[:-1]


def grad_arena_floats(P: int, with_dirs: bool = False) -> int:
    """float32 elements of the model-gradient arena for P Gaussians (61 per Gaussian + padding; +3 with `dirs`)."""
    return segments_floats(P, _grad_layout(with_dirs))


def carve_grad_arena(storage: torch.Tensor, P: int, with_dirs: bool = False) -> Dict[str, torch.Tensor]:
    need = grad_arena_floats(P, with_dirs)
    if storage.dtype != torch.float32 or not storage.is_contiguous() or storage.numel() < need:
        raise RuntimeError(f"projection: gradient arena must be a contiguous float32 tensor of at least {need} elements")
    return carve_segments(storage.view(-1), P, _grad_layout(with_dirs))


# process-wide, like rasterizer.set_gradient_arena (autograd's backward thread must see it)
_GRAD_ARENA = {"storage": None}


def _check_no_strand_arena() -> None:
    """The strand model has no gradient-arena layout: an installed arena raises (render_hair_strands checks before it
    launches anything, project_backward again for direct callers)."""
    if _GRAD_ARENA["storage"] is not None:
        raise RuntimeError("projection: the strand model has no gradient-arena layout; remove the arena (set_gradient_arena(None))")


def set_gradient_arena(storage):
    """Install (or remove with None) a caller-owned flat float32 buffer -- e.g. dist.PeerAllReduce(...).buffer -- into
    which the next projection backward writes every parameter gradient (`carve_grad_arena` layout), so that a
    data-parallel trainer reduces the whole model gradient with ONE collective over `flat[:grad_arena_floats(P)]`."""
    prev = _GRAD_ARENA["storage"]
    _GRAD_ARENA["storage"] = storage
    return prev


def project_backward(pi: ProjectionInputs, visible: torch.Tensor, geom_buffer: Optional[torch.Tensor] = None,
                     dL_dmeans2D=None, dL_dconic4=None, dL_dcolors=None, dL_dopacity=None,
                     camera_grads: bool = True, want_means2D_grad: bool = False, nan_flag: Optional[torch.Tensor] = None,
                     tan_fov: Optional[torch.Tensor] = None, d_camera: Optional[torch.Tensor] = None):
    """Incoming gradients: either the rasterizer's geometry workspace after `gh_backward` (its accumulation records are
    read directly) or the four API-shaped tensors (dL_dmeans2D (P,3), dL_dconic (P,2,2) native layout, dL_dcolors
    (P,10), dL_dopacity (P,1)).  -> dict of parameter gradients (+ 'viewmatrix' (4,4), 'projmatrix' (4,4), 'campos' (3),
    'tanfov' (2) when `camera_grads`, + 'means2D' (P,3) = the incoming NDC gradient when `want_means2D_grad`).
    `nan_flag` (device int32[1], zeroed by the caller): OR-ed with 1 when a parameter gradient is NaN.
    `tan_fov`: tan(fov / 2) as a device (2,) tensor instead of the floats in `pi` (gh_project_backward_capturable).
    `d_camera`: with `camera_grads`, a caller-owned contiguous float32 (37,) buffer for the camera gradients."""
    lib = _capi.load()
    dev, P = pi.device, pi.P
    f = dict(dtype=torch.float32, device=dev)
    strand = bool(pi.flags >> 10 & 1)
    if strand:
        _check_no_strand_arena()
    # which gradients this model configuration has: the strand model folds scaling and rotation into dirs
    has = {"scaling": not strand, "rotation": not strand, "dirs": pi.dirs is not None, "opacity": pi.opacity is not None,
           "label": pi.label is not None, "conf": pi.conf is not None}
    if _GRAD_ARENA["storage"] is not None:
        views = carve_grad_arena(_GRAD_ARENA["storage"], P, with_dirs=has["dirs"])
    else:
        views = {k: empty_rows(P, shape, torch.float32, dev) for k, _, shape in GRAD_SEGMENTS if has.get(k, True)}
    g = {k: views[k] if has.get(k, True) else None for k, _, _ in GRAD_SEGMENTS}
    del views
    g["means2D"] = empty_rows(P, (3,), torch.float32, dev) if want_means2D_grad else None
    cam = None
    if camera_grads:
        cam = torch.zeros(37, **f) if d_camera is None else d_camera
        if d_camera is not None and P == 0:
            cam.zero_()
    if P != 0:
        with torch.cuda.device(dev):
            ws = _camera_workspace(P, dev) if camera_grads else None
            conic4 = _f32(dL_dconic4, "dL_dconic", dev, align=16)
            args = (_ptr(visible), _ptr(geom_buffer),
                    _ptr(_f32(dL_dmeans2D, "dL_dmeans2D", dev)), _ptr(conic4), _ptr(_f32(dL_dcolors, "dL_dcolors", dev, align=8)),
                    _ptr(_f32(dL_dopacity, "dL_dopacity", dev)),
                    _ptr(g["xyz"]), _ptr(g["scaling"]), _ptr(g["rotation"]), _ptr(g["dirs"]), _ptr(g["f_dc"]), _ptr(g["f_rest"]),
                    _ptr(g["opacity"]), _ptr(g["label"]), _ptr(g["conf"]), _ptr(g["means2D"]), _ptr(cam), _ptr(nan_flag), _ptr(ws))
            if tan_fov is None:
                _capi.check(lib.gh_project_backward(*_common_args(pi), *args, _stream(dev)))
            else:
                _capi.check(lib.gh_project_backward_capturable(*_common_args_capturable(pi, tan_fov), *args, 0, _stream(dev)))
    if camera_grads:
        g["viewmatrix"], g["projmatrix"] = cam[0:16].view(4, 4), cam[16:32].view(4, 4)
        g["campos"], g["tanfov"] = cam[32:35], cam[35:37]
    return g


# ------------------------------------------------------------------------------------------------- strand geometry
def strand_midpoints(origins: torch.Tensor, dirs: torch.Tensor, out: torch.Tensor) -> torch.Tensor:
    """Segment midpoints of S polylines (gh_strand_midpoints): origins (S,1,3), dirs (S,L,3) -> `out` (S*L,3), a
    contiguous float32 buffer (e.g. a row block of a larger means3D buffer); what initialize_gaussians_hair() computes
    as `_xyz` (gaussian_model_strands.py:436-438), up to the summation order of the scan."""
    lib = _capi.load()
    S, L = int(dirs.shape[0]), int(dirs.shape[1])
    dev = out.device
    o = _f32(origins, "pts_origins", dev)
    d = _f32(dirs, "dirs", dev)
    if not out.is_contiguous() or out.shape != (S * L, 3):
        raise RuntimeError(f"strand_midpoints: 'out' must be a contiguous ({S * L}, 3) tensor")
    with torch.cuda.device(dev):
        _capi.check(lib.gh_strand_midpoints(S, L, _ptr(o), _ptr(d), _ptr(out), _stream(dev)))
    return out


def strand_backward(S: int, L: int, d_xyz: torch.Tensor, d_dirs: torch.Tensor, nan_flag: Optional[torch.Tensor] = None):
    """gh_strand_backward: d_dirs (S*L,3), holding the direct terms of the strand-mode projection backward, becomes
    dL/d_dirs IN PLACE (the midpoint gradients d_xyz chained through the cumulative sum); returns it as (S,L,3)."""
    lib = _capi.load()
    dev = d_dirs.device
    with torch.cuda.device(dev):
        _capi.check(lib.gh_strand_backward(S, L, _ptr(d_xyz), _ptr(d_dirs), _ptr(nan_flag), _stream(dev)))
    return d_dirs.view(S, L, 3)


# ------------------------------------------------------------------------------------------------- capturable strands
class StrandInputs:
    """The (detached, contiguous) tensors of one capturable strand render (head block + strand model), kept between the
    forward and the backward."""
    __slots__ = ("n_head", "S", "L", "W", "H", "head", "origins", "dirs", "scale", "f_dc", "f_rest", "conf", "V", "Pm",
                 "campos", "tan_fov", "mod", "sh_degree", "device")

    @property
    def P(self) -> int:
        return self.n_head + self.S * self.L

    def common(self):
        """The arguments shared by the two gh_hair_strands_*_capturable entry points after the row counts."""
        return (_ptr(self.dirs), _ptr(self.scale), _ptr(self.f_dc), _ptr(self.f_rest), _ptr(self.conf),
                encode_flags(HAIR_STRANDS), float(HAIR_STRANDS["det_eps"]), _ptr(self.V), _ptr(self.Pm), _ptr(self.campos),
                _ptr(self.tan_fov), self.mod, self.sh_degree)


def pack_strand_inputs(head, origins, dirs, scale, f_dc, f_rest, conf, viewmatrix, projmatrix, campos, tan_fov,
                       width: int, height: int, sh_degree: int, scaling_modifier: float) -> StrandInputs:
    """`head`: the frozen head block (renderer._head_block: xyz, scaling, rotation, opacity, f_dc, f_rest) or None;
    `dirs` (S,L,3) segment vectors, `origins` (S,1,3), `scale` the (1,) strand thickness, f_dc / f_rest / conf with
    S*L rows; the camera tensors and the (2,) `tan_fov` on the device."""
    dev = dirs.device
    if dirs.ndim != 3 or dirs.shape[-1] != 3:
        raise RuntimeError(f"projection: dirs must be (S, L, 3), got {tuple(dirs.shape)}")
    sp = StrandInputs()
    sp.device = dev
    sp.S, sp.L, sp.W, sp.H = int(dirs.shape[0]), int(dirs.shape[1]), int(width), int(height)
    sp.head = None
    if head is not None and int(head["xyz"].shape[0]) > 0:
        sp.head = {k: _f32(head[k], "head " + k, dev, align=16 if k == "rotation" else 4)
                   for k in ("xyz", "scaling", "rotation", "f_dc", "f_rest", "opacity")}
    sp.n_head = 0 if sp.head is None else int(sp.head["xyz"].shape[0])
    sp.origins, sp.dirs = _f32(origins, "pts_origins", dev), _f32(dirs, "dirs", dev)
    sp.scale = _f32(scale, "scale", dev)
    sp.f_dc, sp.f_rest, sp.conf = _f32(f_dc, "features_dc", dev), _f32(f_rest, "features_rest", dev), _f32(conf, "orient_conf", dev)
    sp.V, sp.Pm, sp.campos = _f32(viewmatrix, "viewmatrix", dev), _f32(projmatrix, "projmatrix", dev), _f32(campos, "campos", dev)
    sp.tan_fov = _f32(tan_fov, "tan_fov", dev)
    sp.mod, sp.sh_degree = float(scaling_modifier), int(sh_degree)
    n = sp.S * sp.L
    if sp.origins is None or sp.origins.numel() != 3 * sp.S:
        raise RuntimeError(f"projection: pts_origins must be (S, 1, 3) = ({sp.S}, 1, 3)")
    if sp.scale is None or sp.scale.numel() != 1:
        raise RuntimeError("projection: the strand thickness must be a (1,) tensor")
    for name, t, per in (("features_dc", sp.f_dc, 3), ("orient_conf", sp.conf, 1)):
        if t is None or t.numel() != n * per:
            raise RuntimeError(f"projection: '{name}' must have {per} floats per segment (S*L = {n} rows)")
    if sp.sh_degree > 0 and (sp.f_rest is None or sp.f_rest.numel() != n * 45):
        raise RuntimeError("projection: 'features_rest' must be (S*L, 15, 3) for sh_degree > 0")
    return sp


def hair_strands_forward_binned_capturable(sp: StrandInputs, binning: torch.Tensor, capacity: int, status: torch.Tensor,
                                           num_rendered: Optional[torch.Tensor] = None):
    """gh_hair_strands_forward_binned_capturable: the capturable first phase of render_hair_strands over P = n_head +
    S*L rows (head rows first).  -> (out dict as project_forward with P rows, radii, geomBuffer, imgBuffer, midpoints
    (S*L,3)); continue with `_C.forward_render_capturable`.  No host synchronisation."""
    from . import _C
    lib = _capi.load()
    dev, P = sp.device, sp.P
    out = alloc_outputs(P, dev)
    geom, img, radii = _C.alloc_forward_workspaces(P, sp.W, sp.H, dev)
    mid = empty_rows(sp.S * sp.L, (3,), torch.float32, dev)
    hd = sp.head or {}
    h = lambda k: _ptr(hd.get(k))  # noqa: E731
    with torch.cuda.device(dev):
        _capi.check(lib.gh_hair_strands_forward_binned_capturable(
            sp.n_head, sp.S, sp.L, sp.W, sp.H, h("xyz"), h("scaling"), h("rotation"), h("f_dc"), h("f_rest"), h("opacity"),
            encode_flags(HEAD_PRECOMP), float(HEAD_PRECOMP["det_eps"]), _ptr(sp.origins), *sp.common(), _ptr(mid),
            _ptr(out["means2D"]), _ptr(out["colors"]), _ptr(out["opacity"]), _ptr(out["conic"]), _ptr(out["visible"]),
            _ptr(radii), _ptr(geom), _ptr(img), _ptr(binning), int(capacity), _ptr(status), _ptr(num_rendered), 0,
            _stream(dev)))
    return out, radii, geom, img, mid


def hair_strands_backward_capturable(sp: StrandInputs, midpoints: torch.Tensor, visible: torch.Tensor,
                                     geom_buffer: torch.Tensor, nan_flag: Optional[torch.Tensor] = None):
    """gh_hair_strands_backward_capturable, after `_C.backward_records_capturable` over all P rows: the gradients of the
    strand model's parameters from the accumulation records of its rows -> dict(dirs (S,L,3), f_dc (S*L,1,3), f_rest
    (S*L,15,3), conf (S*L,1)).  `nan_flag` as in project_backward."""
    _check_no_strand_arena()
    lib = _capi.load()
    dev, n = sp.device, sp.S * sp.L
    g = {k: empty_rows(n, shape, torch.float32, dev) for k, shape in (("xyz", (3,)), ("dirs", (3,)), ("f_dc", (1, 3)),
                                                                      ("f_rest", (15, 3)), ("conf", (1,)))}
    with torch.cuda.device(dev):
        _capi.check(lib.gh_hair_strands_backward_capturable(
            sp.n_head, sp.S, sp.L, sp.W, sp.H, _ptr(midpoints), *sp.common(), _ptr(visible), _ptr(geom_buffer),
            _ptr(g["xyz"]), _ptr(g["dirs"]), _ptr(g["f_dc"]), _ptr(g["f_rest"]), _ptr(g["conf"]), _ptr(nan_flag), 0,
            _stream(dev)))
    g["dirs"] = g["dirs"].view(sp.S, sp.L, 3)
    del g["xyz"]
    return g


# ------------------------------------------------------------------------------------------------ capturable segments
class SegmentInputs:
    """The (detached, contiguous) tensors of one capturable segment render (head block + the latent strand model's N
    given segment rows), kept between the forward and the backward."""
    __slots__ = ("n_head", "N", "W", "H", "head", "xyz", "dirs", "scale", "f_dc", "f_rest", "conf", "V", "Pm", "campos",
                 "tan_fov", "mod", "sh_degree", "device")

    @property
    def P(self) -> int:
        return self.n_head + self.N

    def common(self):
        """The arguments shared by the two gh_hair_segments_*_capturable entry points after the image size."""
        return (_ptr(self.xyz), _ptr(self.dirs), _ptr(self.scale), _ptr(self.f_dc), _ptr(self.f_rest), _ptr(self.conf),
                encode_flags(HAIR_STRANDS), float(HAIR_STRANDS["det_eps"]), _ptr(self.V), _ptr(self.Pm), _ptr(self.campos),
                _ptr(self.tan_fov), self.mod, self.sh_degree)


def pack_segment_inputs(head, xyz, dirs, scale, f_dc, f_rest, conf, viewmatrix, projmatrix, campos, tan_fov,
                        width: int, height: int, sh_degree: int, scaling_modifier: float) -> SegmentInputs:
    """`head`: the frozen head block (renderer._head_block) or None; `xyz` (N,3) segment midpoints and `dirs` (N,3)
    segment vectors (GaussianModelHair._xyz / _dir), `scale` the (1,) strand thickness, f_dc / f_rest / conf with N
    rows; the camera tensors and the (2,) `tan_fov` on the device."""
    dev = xyz.device
    if xyz.ndim != 2 or xyz.shape[-1] != 3 or tuple(dirs.shape) != tuple(xyz.shape):
        raise RuntimeError(f"projection: xyz and dirs must both be (N, 3), got {tuple(xyz.shape)} and {tuple(dirs.shape)}")
    sp = SegmentInputs()
    sp.device = dev
    sp.N, sp.W, sp.H = int(xyz.shape[0]), int(width), int(height)
    sp.head = None
    if head is not None and int(head["xyz"].shape[0]) > 0:
        sp.head = {k: _f32(head[k], "head " + k, dev, align=16 if k == "rotation" else 4)
                   for k in ("xyz", "scaling", "rotation", "f_dc", "f_rest", "opacity")}
    sp.n_head = 0 if sp.head is None else int(sp.head["xyz"].shape[0])
    sp.xyz, sp.dirs, sp.scale = _f32(xyz, "xyz", dev), _f32(dirs, "dirs", dev), _f32(scale, "scale", dev)
    sp.f_dc, sp.f_rest, sp.conf = _f32(f_dc, "features_dc", dev), _f32(f_rest, "features_rest", dev), _f32(conf, "orient_conf", dev)
    sp.V, sp.Pm, sp.campos = _f32(viewmatrix, "viewmatrix", dev), _f32(projmatrix, "projmatrix", dev), _f32(campos, "campos", dev)
    sp.tan_fov = _f32(tan_fov, "tan_fov", dev)
    sp.mod, sp.sh_degree = float(scaling_modifier), int(sh_degree)
    n = sp.N
    if sp.scale is None or sp.scale.numel() != 1:
        raise RuntimeError("projection: the strand thickness must be a (1,) tensor")
    for name, t, per in (("features_dc", sp.f_dc, 3), ("orient_conf", sp.conf, 1)):
        if t is None or t.numel() != n * per:
            raise RuntimeError(f"projection: '{name}' must have {per} floats per segment (N = {n} rows)")
    if sp.sh_degree > 0 and (sp.f_rest is None or sp.f_rest.numel() != n * 45):
        raise RuntimeError("projection: 'features_rest' must be (N, 15, 3) for sh_degree > 0")
    return sp


def hair_segments_forward_binned_capturable(sp: SegmentInputs, binning: torch.Tensor, capacity: int,
                                            status: torch.Tensor, num_rendered: Optional[torch.Tensor] = None):
    """gh_hair_segments_forward_binned_capturable: the capturable first phase of render_hair_segments over P = n_head +
    N rows (head rows first).  -> (out dict as project_forward with P rows, radii, geomBuffer, imgBuffer); continue
    with `_C.forward_render_capturable`.  No host synchronisation."""
    from . import _C
    lib = _capi.load()
    dev, P = sp.device, sp.P
    out = alloc_outputs(P, dev)
    geom, img, radii = _C.alloc_forward_workspaces(P, sp.W, sp.H, dev)
    hd = sp.head or {}
    h = lambda k: _ptr(hd.get(k))  # noqa: E731
    with torch.cuda.device(dev):
        _capi.check(lib.gh_hair_segments_forward_binned_capturable(
            sp.n_head, sp.N, sp.W, sp.H, h("xyz"), h("scaling"), h("rotation"), h("f_dc"), h("f_rest"), h("opacity"),
            encode_flags(HEAD_PRECOMP), float(HEAD_PRECOMP["det_eps"]), *sp.common(),
            _ptr(out["means2D"]), _ptr(out["colors"]), _ptr(out["opacity"]), _ptr(out["conic"]), _ptr(out["visible"]),
            _ptr(radii), _ptr(geom), _ptr(img), _ptr(binning), int(capacity), _ptr(status), _ptr(num_rendered), 0,
            _stream(dev)))
    return out, radii, geom, img


def hair_segments_backward_capturable(sp: SegmentInputs, visible: torch.Tensor, geom_buffer: torch.Tensor,
                                      nan_flag: Optional[torch.Tensor] = None):
    """gh_hair_segments_backward_capturable, after `_C.backward_records_capturable` over all P rows: the gradients of
    the segment rows from their accumulation records -> dict(xyz (N,3), dirs (N,3), f_dc (N,1,3), f_rest (N,15,3),
    conf (N,1)).  `nan_flag` as in project_backward."""
    _check_no_strand_arena()
    lib = _capi.load()
    dev, n = sp.device, sp.N
    g = {k: empty_rows(n, shape, torch.float32, dev) for k, shape in (("xyz", (3,)), ("dirs", (3,)), ("f_dc", (1, 3)),
                                                                      ("f_rest", (15, 3)), ("conf", (1,)))}
    with torch.cuda.device(dev):
        _capi.check(lib.gh_hair_segments_backward_capturable(
            sp.n_head, sp.N, sp.W, sp.H, *sp.common(), _ptr(visible), _ptr(geom_buffer),
            _ptr(g["xyz"]), _ptr(g["dirs"]), _ptr(g["f_dc"]), _ptr(g["f_rest"]), _ptr(g["conf"]), _ptr(nan_flag), 0,
            _stream(dev)))
    return g
