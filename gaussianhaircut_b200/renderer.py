"""Drop-in for the reference's `gaussian_renderer` module: `render()` and `render_hair()` with the same
signatures and the same returned dictionary (src/gaussian_renderer/__init__.py:23-114, :116-236), but one fused
autograd node from the models' RAW parameters to the rasterized 10-channel image:

    reference                                                    here
    ---------------------------------------------------------    -------------------------------------------------
    ~100 PyTorch kernels of model-side projection + autograd      gh_project_forward / gh_project_backward (1 launch each)
    six boolean-mask gathers (+ scatter of the radii)             none: culled Gaussians keep their index, conic = 0
    GaussianRasterizer forward / backward                         the same C-ABI rasterizer calls (rasterizer.py / _C.py)
    (P,2,2) conic gradient restack + per-tensor gradient buffers  none: the projection backward reads the blend backward's
                                                                  accumulation records in place

A trainer switches by importing `render` / `render_hair` from here instead of from `gaussian_renderer`; everything
it reads back afterwards is the same: the four maps, `viewspace_points` (+ its `.grad` for the densification
statistics), `visibility_filter`, `radii`, and `.grad` of every model parameter and of trainable camera tensors.
tests/test_gpu_projection.py checks all of that against the reference's own functions imported unmodified.
"""
from __future__ import annotations

import math
from typing import Dict, Optional

import torch
import torch.nn.functional as F

from . import _C, projection
from ._alloc import empty_rows

__all__ = ["render", "render_hair", "render_hair_segments", "render_hair_segments_capturable", "render_hair_strands",
           "render_hair_strands_capturable", "render_raw", "render_raw_capturable", "set_nan_flag"]

_EMPTY = torch.Tensor([])

# The optimizer's NaN guard (src/train_gaussians.py:174-181) without a pass over the gradients: when a flag tensor is
# installed, the projection backward ORs 1 into it if any parameter gradient is NaN; hand the same tensor to
# FusedAdam.step(nan_flag_in=...).  The caller zeroes it once per iteration (FusedAdam does, after reading it).
_NAN_FLAG = {"t": None}


def set_nan_flag(flag):
    """Install (or remove with None) the device int32[1] tensor that receives the NaN verdict of the next backward."""
    _NAN_FLAG["t"] = flag


_TAN_CACHE: Dict[int, tuple] = {}


def _tan_half(fov) -> float:
    """tan(fov / 2) as a host float.  The reference reads it back from the device on every call (`.item()`,
    __init__.py:43-44); here the value is cached per FoV tensor (identity + in-place version), so a camera whose
    field of view does not change costs one device read in total."""
    if isinstance(fov, torch.Tensor):
        key = id(fov)
        hit = _TAN_CACHE.get(key)
        if hit is not None and hit[0]() is fov and hit[1] == fov._version and not fov.requires_grad:
            return hit[2]
        val = float(torch.tan(fov.detach() * 0.5).item())
        if not fov.requires_grad:
            import weakref
            if len(_TAN_CACHE) > 4096:
                _TAN_CACHE.clear()
            try:
                _TAN_CACHE[key] = (weakref.ref(fov), fov._version, val)
            except TypeError:
                pass
        return val
    return math.tan(float(fov) * 0.5)


class _FusedRender(torch.autograd.Function):
    """(xyz, scaling, rotation, dirs, f_dc, f_rest, opacity, label, conf, viewspace, viewmatrix, projmatrix, campos, tanfov,
    static) -> (raw 10-channel image, radii).  `viewspace` is a (P,3) leaf: its storage receives the NDC means and its
    gradient the rasterizer's dL/dmeans2D (what `add_densification_stats` reads).  `static`: dict of non-tensors + the
    frozen head block of render_hair().
    Strand models (render_hair_strands, static["strands"] = polyline origins): xyz is None, `dirs` is the (S,L,3) segment
    vector parameter and `scaling` the (1,) strand thickness; the segment midpoints are computed into the means3D rows
    of this model and kept for the backward, which returns the gradient of `dirs` (S,L,3).
    Segment models (render_hair_segments: static["cfg"] = HAIR_STRANDS, no static["strands"]): `xyz` (N,3) are the given
    midpoints and `dirs` (N,3) the segment vectors; both gradients are returned as the projection backward writes them."""

    @staticmethod
    def forward(ctx, xyz, scaling, rotation, dirs, f_dc, f_rest, opacity, label, conf, viewspace, viewmatrix, projmatrix,
                campos, tanfov, static):
        st = static
        dev = viewspace.device
        head = st.get("head")
        n_head = 0 if head is None else int(head["xyz"].shape[0])
        strands = st.get("strands")
        P_own = int(dirs.shape[0] * dirs.shape[1]) if strands is not None else int(xyz.shape[0])
        P = n_head + P_own
        means3D = None
        if strands is not None:
            # segment midpoints straight into this model's rows of the means3D buffer (behind the head rows: no cat)
            means3D = empty_rows(P, (3,), torch.float32, dev)
            if n_head > 0:
                means3D[:n_head].copy_(head["xyz"])
            xyz = projection.strand_midpoints(strands["origins"], dirs, out=means3D[n_head:])
            dirs = dirs.reshape(P_own, 3)
        pi = projection.pack_inputs(xyz, scaling, rotation, dirs, f_dc, f_rest, opacity, label, conf, viewmatrix, projmatrix,
                                    campos, st["tanx"], st["tany"], st["W"], st["H"], st["sh_degree"], st["mod"], st["cfg"])
        bg = st["bg"]
        zero = any(ctx.needs_input_grad)    # only a forward with a backward needs cleared accumulation records
        if n_head == 0 and P_own > 0 and not st["debug"]:
            # one pass over the Gaussians does the projection AND the rasterizer's preprocess + tile histogram
            out, radii, geom, img, R, max_len, binned = projection.project_forward_binned(pi, means2D_out=viewspace.detach(),
                                                                                        binning=True)
            color, binning = _C.forward_render(bg, out["colors"], radii, geom, img, R, max_len, st["H"], st["W"], binned=binned,
                                               zero_records=zero)
            ctx.pi, ctx.st, ctx.R, ctx.n_head, ctx.hp = pi, st, R, 0, None
            ctx.bufs = (pi.xyz, out["colors"], out["conic"], out["visible"], radii, geom, binning, img)
            ctx.mark_non_differentiable(radii)
            return color, radii
        if n_head == 0:
            out = projection.project_forward(pi, means2D_out=viewspace.detach())
            means3D = pi.xyz
        else:
            # the frozen head Gaussians first, then this model's: both write row blocks of the same buffers
            out = projection.alloc_outputs(P, dev, means2D_out=viewspace.detach())
            hp = projection.pack_inputs(head["xyz"], head["scaling"], head["rotation"], None, head["f_dc"], head["f_rest"],
                                        head["opacity"], None, None, viewmatrix, projmatrix, campos, st["tanx"], st["tany"],
                                        st["W"], st["H"], st["sh_degree"], st["mod"], projection.HEAD_PRECOMP)
            sl = lambda a, b: {k: (v[a:b] if v is not None else None) for k, v in out.items()}  # noqa: E731
            projection.project_forward(hp, out=sl(0, n_head))
            projection.project_forward(pi, out=sl(n_head, P))
            if means3D is None:
                means3D = torch.cat([hp.xyz, pi.xyz], dim=0)
        R, color, radii, geom, binning, img = _C.rasterize_gaussians(
            bg, means3D, _EMPTY, out["colors"], out["opacity"], _EMPTY, _EMPTY, st["mod"], _EMPTY, out["conic"],
            pi.V, pi.Pm, st["tanx"], st["tany"], st["H"], st["W"], _EMPTY, st["sh_degree"], pi.campos,
            False, st["debug"], zero_records=zero)   # prefiltered=False: culled Gaussians are still in the list (conic = 0)
        ctx.pi, ctx.st, ctx.R, ctx.n_head = pi, st, R, n_head
        ctx.hp = hp if n_head > 0 else None
        ctx.bufs = (means3D, out["colors"], out["conic"], out["visible"], radii, geom, binning, img)
        ctx.mark_non_differentiable(radii)
        return color, radii

    @staticmethod
    def backward(ctx, g_color, _g_radii):
        pi, st, n_head = ctx.pi, ctx.st, ctx.n_head
        means3D, colors, conic, visible, radii, geom, binning, img = ctx.bufs
        need = ctx.needs_input_grad
        cam_grads = bool(need[10] or need[11] or need[12] or need[13])
        if n_head == 0:
            _C.rasterize_gaussians_backward_records(st["bg"], means3D, radii, colors, conic, pi.V, pi.Pm, st["tanx"], st["tany"],
                                                    g_color, pi.campos, geom, ctx.R, binning, img, st["debug"])
            g = projection.project_backward(pi, visible, geom_buffer=geom, camera_grads=cam_grads, want_means2D_grad=True,
                                            nan_flag=_NAN_FLAG["t"])
            g_view = g["means2D"]
        else:
            g9 = _C.rasterize_gaussians_backward(st["bg"], means3D, radii, colors, _EMPTY, _EMPTY, st["mod"], _EMPTY, conic,
                                                 pi.V, pi.Pm, st["tanx"], st["tany"], g_color, _EMPTY, st["sh_degree"],
                                                 pi.campos, geom, ctx.R, binning, img, st["debug"])
            g_m2, g_col, g_op, _g3, _gc3, g_conic = g9[0], g9[1], g9[2], g9[3], g9[4], g9[5]
            g = projection.project_backward(pi, visible[n_head:], dL_dmeans2D=g_m2[n_head:], dL_dconic4=g_conic[n_head:],
                                            dL_dcolors=g_col[n_head:], dL_dopacity=g_op[n_head:], camera_grads=cam_grads,
                                            nan_flag=_NAN_FLAG["t"])
            g_view = g_m2                  # `viewspace_points.grad` covers head rows too (retain_grad on the concatenation, :134-137)
            if cam_grads:
                # the head block is frozen, but its conic / depth / view direction still depend on the camera; only its
                # screen-space mean is detached (:132), so that path contributes nothing
                gh = projection.project_backward(ctx.hp, visible[:n_head], dL_dmeans2D=torch.zeros_like(g_m2[:n_head]), dL_dconic4=g_conic[:n_head],
                                                 dL_dcolors=g_col[:n_head], dL_dopacity=g_op[:n_head], camera_grads=True)
                for k in ("viewmatrix", "projmatrix", "campos", "tanfov"):
                    g[k] = g[k] + gh[k]
        strands = st.get("strands")
        if strands is not None:
            # the per-segment midpoint gradients, chained through the cumulative sum into the segment vectors
            g["dirs"] = projection.strand_backward(strands["S"], strands["L"], g["xyz"], g["dirs"], nan_flag=_NAN_FLAG["t"])
        pick = lambda k, idx: g.get(k) if need[idx] else None  # noqa: E731   (autograd rejects gradients for non-Variable inputs)
        return (pick("xyz", 0), pick("scaling", 1), pick("rotation", 2), pick("dirs", 3), pick("f_dc", 4), pick("f_rest", 5),
                pick("opacity", 6), pick("label", 7), pick("conf", 8), g_view if need[9] else None,
                pick("viewmatrix", 10), pick("projmatrix", 11), pick("campos", 12), pick("tanfov", 13), None)


class _CapturableRender(torch.autograd.Function):
    """The capturable twin of _FusedRender's fused path (n_head == 0, GaussianModel rows): (xyz, scaling, rotation, f_dc,
    f_rest, opacity, label, conf, viewspace, viewmatrix, projmatrix, campos, tan_fov, static) -> (raw image, radii), with
    the same gradients.  The camera tensors are static device inputs and R never leaves the device: `static` holds the
    caller's binning buffer, its capacity, the status word and the optional d_camera buffer that receives the camera
    gradients (render_raw_capturable)."""

    @staticmethod
    def forward(ctx, xyz, scaling, rotation, f_dc, f_rest, opacity, label, conf, viewspace, viewmatrix, projmatrix, campos,
                tan_fov, static):
        st = static
        # (tan fov is read from `tan_fov` on the device: the host floats of pack_inputs are unused placeholders)
        pi = projection.pack_inputs(xyz, scaling, rotation, None, f_dc, f_rest, opacity, label, conf, viewmatrix, projmatrix,
                                    campos, 0.0, 0.0, st["W"], st["H"], st["sh_degree"], st["mod"], st["cfg"])
        out, radii, geom, img = projection.project_forward_binned_capturable(
            pi, tan_fov, st["binning"], st["capacity"], st["status"], st["num_rendered"], means2D_out=viewspace.detach())
        color = _C.forward_render_capturable(st["bg"], out["colors"], geom, st["binning"], img, st["capacity"], st["H"], st["W"])
        ctx.pi, ctx.st, ctx.tan_fov = pi, st, tan_fov
        ctx.bufs = (out["colors"], out["visible"], radii, geom, img)
        ctx.mark_non_differentiable(radii)
        return color, radii

    @staticmethod
    def backward(ctx, g_color, _g_radii):
        pi, st = ctx.pi, ctx.st
        colors, visible, radii, geom, img = ctx.bufs
        _C.backward_records_capturable(st["bg"], colors, radii, geom, st["binning"], img, st["capacity"], g_color)
        d_camera = st.get("d_camera")
        g = projection.project_backward(pi, visible, geom_buffer=geom, camera_grads=d_camera is not None,
                                        want_means2D_grad=True, nan_flag=_NAN_FLAG["t"], tan_fov=ctx.tan_fov,
                                        d_camera=d_camera)
        need = ctx.needs_input_grad
        pick = lambda k, idx: g.get(k) if need[idx] else None  # noqa: E731
        return (pick("xyz", 0), pick("scaling", 1), pick("rotation", 2), pick("f_dc", 3), pick("f_rest", 4),
                pick("opacity", 5), pick("label", 6), pick("conf", 7), g["means2D"] if need[8] else None,
                None, None, None, None, None)


def render_raw_capturable(camera: Dict[str, torch.Tensor], pc, bg_color: torch.Tensor, width: int, height: int,
                          binning: torch.Tensor, capacity: int, status: torch.Tensor,
                          num_rendered: Optional[torch.Tensor] = None, scaling_modifier: float = 1.0,
                          d_camera: Optional[torch.Tensor] = None):
    """`render_raw` for CUDA-graph capture (graphs.CapturedTrainStep): no host synchronisation, and every value that
    changes between iterations is read on the device.  `camera`: device float32 tensors "viewmatrix" (4,4),
    "projmatrix" (4,4), "campos" (3) and "tan_fov" (2) = tan(FoV / 2) (x, y), none of which may require grad.
    `binning`: a buffer of `capacity` records (_C.binning_workspace); `status`: int32 (1,), zeroed by the caller,
    receives bit 0 when R exceeds the capacity -- the frame then renders as the background, with zero radii and zero
    gradients; `num_rendered`: int32 (1,) that receives R, or None; `d_camera`: None, or a device float32 (37,) buffer
    that the backward fills with the camera gradients in gh_project_backward's d_camera layout (dL/dviewmatrix,
    dL/dprojmatrix, dL/dcampos, dL/dtan_fov) -- the input of cameras.CameraRig.backward.
    -> (raw (10,H,W) image, radii, viewspace_points)."""
    for k in ("viewmatrix", "projmatrix", "campos", "tan_fov"):
        if camera[k].requires_grad:
            raise RuntimeError(f"render_raw_capturable: camera tensor '{k}' requires grad; trainable cameras are not supported")
    P = int(pc._xyz.shape[0])
    viewspace = empty_rows(P, (3,), torch.float32, pc._xyz.device).requires_grad_(True)
    st = {"W": int(width), "H": int(height), "bg": bg_color, "mod": float(scaling_modifier), "sh_degree": int(pc.active_sh_degree),
          "cfg": projection.GAUSSIAN_MODEL, "binning": binning, "capacity": int(capacity), "status": status,
          "num_rendered": num_rendered, "d_camera": d_camera}
    renders, radii = _CapturableRender.apply(
        pc._xyz, pc._scaling, pc._rotation, pc._features_dc, pc._features_rest, pc._opacity, pc._label, pc._orient_conf,
        viewspace, camera["viewmatrix"], camera["projmatrix"], camera["campos"], camera["tan_fov"], st)
    return renders, radii, viewspace


class _CapturableStrandRender(torch.autograd.Function):
    """The capturable twin of _FusedRender for render_hair_strands: (dirs, f_dc, f_rest, conf, static) -> (raw image,
    radii) over the head block and the strand rows, with the gradients of the four strand parameters.  `static` holds
    the packed inputs (projection.StrandInputs), the binning buffer, its capacity, the status word and num_rendered."""

    @staticmethod
    def forward(ctx, dirs, f_dc, f_rest, conf, static):
        st = static
        sp = projection.pack_strand_inputs(st["head"], st["origins"], dirs, st["scale"], f_dc, f_rest, conf,
                                           *st["camera"], st["W"], st["H"], st["sh_degree"], st["mod"])
        out, radii, geom, img, mid = projection.hair_strands_forward_binned_capturable(
            sp, st["binning"], st["capacity"], st["status"], st["num_rendered"])
        color = _C.forward_render_capturable(st["bg"], out["colors"], geom, st["binning"], img, st["capacity"], sp.H, sp.W)
        ctx.sp, ctx.st = sp, st
        ctx.bufs = (out["colors"], out["visible"], radii, geom, img, mid)
        ctx.mark_non_differentiable(radii)
        return color, radii

    @staticmethod
    def backward(ctx, g_color, _g_radii):
        st = ctx.st
        colors, visible, radii, geom, img, mid = ctx.bufs
        _C.backward_records_capturable(st["bg"], colors, radii, geom, st["binning"], img, st["capacity"], g_color)
        g = projection.hair_strands_backward_capturable(ctx.sp, mid, visible, geom, nan_flag=_NAN_FLAG["t"])
        need = ctx.needs_input_grad
        return (g["dirs"] if need[0] else None, g["f_dc"] if need[1] else None, g["f_rest"] if need[2] else None,
                g["conf"] if need[3] else None, None)


def render_hair_strands_capturable(camera: Dict[str, torch.Tensor], pc, pc_hair, bg_color: torch.Tensor, width: int,
                                   height: int, binning: torch.Tensor, capacity: int, status: torch.Tensor,
                                   num_rendered: Optional[torch.Tensor] = None, scaling_modifier: float = 1.0):
    """`render_hair_strands` for CUDA-graph capture (graphs.CapturedStrandStep): the frozen head block of `pc` (None or
    an empty block: hair only) followed by the segments of the strand model `pc_hair`, with no host synchronisation.
    `camera`, `binning`, `capacity`, `status` and `num_rendered` as in render_raw_capturable (no camera tensor may
    require grad: the strand stage does not train its cameras).  -> (raw (10,H,W) image, radii (n_head + S*L,)).
    Gradients land in `.grad` of `_dirs`, `_features_dc`, `_features_rest` and `_orient_conf`; set_nan_flag() works as
    with render_hair_strands.  With the same inputs, image, radii and (deterministic mode) gradients are bit-identical
    to render_hair_strands'."""
    for k in ("viewmatrix", "projmatrix", "campos", "tan_fov"):
        if camera[k].requires_grad:
            raise RuntimeError(f"render_hair_strands_capturable: camera tensor '{k}' requires grad; trainable cameras are "
                               "not supported")
    projection._check_no_strand_arena()
    dirs = pc_hair._dirs
    if dirs.ndim != 3 or dirs.shape[-1] != 3 or dirs.shape[0] < 1 or dirs.shape[1] < 1:
        raise RuntimeError(f"render_hair_strands_capturable: _dirs must be (S, L, 3) with S, L >= 1, got {tuple(dirs.shape)}")
    scale = pc_hair.scale
    if not isinstance(scale, torch.Tensor):
        raise RuntimeError("render_hair_strands_capturable: pc_hair.scale must be a (1,) device tensor (a captured "
                           "launch keeps its address)")
    head = _head_block(pc) if pc is not None else None
    st = {"W": int(width), "H": int(height), "bg": bg_color, "mod": float(scaling_modifier),
          "sh_degree": int(pc_hair.active_sh_degree), "head": head, "origins": pc_hair.pts_origins, "scale": scale.detach(),
          "camera": (camera["viewmatrix"], camera["projmatrix"], camera["campos"], camera["tan_fov"]),
          "binning": binning, "capacity": int(capacity), "status": status, "num_rendered": num_rendered}
    return _CapturableStrandRender.apply(dirs, pc_hair._features_dc, pc_hair._features_rest, pc_hair._orient_conf, st)


class _CapturableSegmentRender(torch.autograd.Function):
    """The capturable twin of _FusedRender for render_hair_segments: (xyz, dirs, f_dc, f_rest, conf, static) -> (raw
    image, radii) over the head block and the N segment rows, with the gradients of the five segment tensors.  `static`
    as in _CapturableStrandRender."""

    @staticmethod
    def forward(ctx, xyz, dirs, f_dc, f_rest, conf, static):
        st = static
        sp = projection.pack_segment_inputs(st["head"], xyz, dirs, st["scale"], f_dc, f_rest, conf, *st["camera"],
                                            st["W"], st["H"], st["sh_degree"], st["mod"])
        out, radii, geom, img = projection.hair_segments_forward_binned_capturable(
            sp, st["binning"], st["capacity"], st["status"], st["num_rendered"])
        color = _C.forward_render_capturable(st["bg"], out["colors"], geom, st["binning"], img, st["capacity"], sp.H, sp.W)
        ctx.sp, ctx.st = sp, st
        ctx.bufs = (out["colors"], out["visible"], radii, geom, img)
        ctx.mark_non_differentiable(radii)
        return color, radii

    @staticmethod
    def backward(ctx, g_color, _g_radii):
        st = ctx.st
        colors, visible, radii, geom, img = ctx.bufs
        _C.backward_records_capturable(st["bg"], colors, radii, geom, st["binning"], img, st["capacity"], g_color)
        g = projection.hair_segments_backward_capturable(ctx.sp, visible, geom, nan_flag=_NAN_FLAG["t"])
        need = ctx.needs_input_grad
        return tuple(g[k] if need[i] else None for i, k in enumerate(("xyz", "dirs", "f_dc", "f_rest", "conf"))) + (None,)


def _segment_rows(pc_hair, who: str) -> int:
    """N, the segment rows of a GaussianModelHair after generate_strands(): `_xyz`, `_dir` (N,3) and N-row features."""
    xyz, dirs = pc_hair._xyz, pc_hair._dir
    if xyz.ndim != 2 or xyz.shape[-1] != 3 or tuple(dirs.shape) != tuple(xyz.shape):
        raise RuntimeError(f"{who}: _xyz and _dir must both be (N, 3), got {tuple(xyz.shape)} and {tuple(dirs.shape)}")
    N = int(xyz.shape[0])
    for name in ("_features_dc", "_features_rest", "_orient_conf"):
        t = getattr(pc_hair, name)
        if t.shape[0] != N:
            raise RuntimeError(f"{who}: {name} must have N = {N} rows (strand-major), got {t.shape[0]}")
    return N


def render_hair_segments_capturable(camera: Dict[str, torch.Tensor], pc, pc_hair, bg_color: torch.Tensor, width: int,
                                    height: int, binning: torch.Tensor, capacity: int, status: torch.Tensor,
                                    num_rendered: Optional[torch.Tensor] = None, scaling_modifier: float = 1.0):
    """`render_hair_segments` for CUDA-graph capture (graphs.CapturedLatentStrandStep): the frozen head block of `pc`
    (None or an empty block: hair only) followed by the N segment rows of `pc_hair`, with no host synchronisation.
    `camera`, `binning`, `capacity`, `status` and `num_rendered` as in render_hair_strands_capturable.  -> (raw
    (10,H,W) image, radii (n_head + N,)).  Gradients flow to `_xyz`, `_dir`, `_features_dc`, `_features_rest` and
    `_orient_conf`; set_nan_flag() works as with render_hair_segments.  With the same inputs, image, radii and
    (deterministic mode) gradients are bit-identical to render_hair_segments'."""
    for k in ("viewmatrix", "projmatrix", "campos", "tan_fov"):
        if camera[k].requires_grad:
            raise RuntimeError(f"render_hair_segments_capturable: camera tensor '{k}' requires grad; trainable cameras "
                               "are not supported")
    projection._check_no_strand_arena()
    if _segment_rows(pc_hair, "render_hair_segments_capturable") < 1:
        raise RuntimeError("render_hair_segments_capturable: the model has no segment rows")
    scale = pc_hair.scale
    if not isinstance(scale, torch.Tensor):
        raise RuntimeError("render_hair_segments_capturable: pc_hair.scale must be a (1,) device tensor (a captured "
                           "launch keeps its address)")
    head = _head_block(pc) if pc is not None else None
    st = {"W": int(width), "H": int(height), "bg": bg_color, "mod": float(scaling_modifier),
          "sh_degree": int(pc_hair.active_sh_degree), "head": head, "scale": scale.detach(),
          "camera": (camera["viewmatrix"], camera["projmatrix"], camera["campos"], camera["tan_fov"]),
          "binning": binning, "capacity": int(capacity), "status": status, "num_rendered": num_rendered}
    return _CapturableSegmentRender.apply(pc_hair._xyz, pc_hair._dir, pc_hair._features_dc, pc_hair._features_rest,
                                          pc_hair._orient_conf, st)


def _post(renders: torch.Tensor, radii: torch.Tensor, viewspace: torch.Tensor) -> Dict[str, torch.Tensor]:
    """The reference's epilogue (gaussian_renderer/__init__.py:98-113)."""
    rendered_image, rendered_mask, rendered_cov2D, rendered_orient_conf, _ = renders.split([3, 2, 3, 1, 1], dim=0)
    rendered_dir2D = F.normalize(rendered_cov2D[:2], dim=0)
    to_mirror = torch.ones_like(rendered_dir2D[[0]])
    to_mirror[rendered_dir2D[[0]] < 0] *= -1
    rendered_orient_angle = torch.acos(rendered_dir2D[[1]].clamp(-1 + 1e-3, 1 - 1e-3) * to_mirror) / math.pi
    return {"render": rendered_image, "mask": rendered_mask, "orient_angle": rendered_orient_angle,
            "orient_conf": rendered_orient_conf, "viewspace_points": viewspace, "visibility_filter": radii > 0,
            "radii": radii, "raw": renders}


def _static(viewpoint_camera, bg_color, scaling_modifier, sh_degree, debug, cfg) -> Dict[str, object]:
    tan = getattr(viewpoint_camera, "tan_fov", None)        # a cameras.CameraRig view: tan(FoV / 2) on the device
    tanx, tany = (tan.tolist() if tan is not None else
                  (_tan_half(viewpoint_camera.FoVx), _tan_half(viewpoint_camera.FoVy)))
    return {"W": int(viewpoint_camera.image_width), "H": int(viewpoint_camera.image_height), "tanx": tanx, "tany": tany,
            "bg": bg_color, "mod": float(scaling_modifier), "sh_degree": int(sh_degree), "debug": bool(debug), "cfg": cfg}


def _tanfov_tensor(viewpoint_camera):
    """A differentiable (2,) tensor when the field of view is trainable (cameras.py:95-107), else None.  A camera with a
    `tan_fov` attribute (cameras.CameraRig views) hands that tensor over as it is."""
    tan = getattr(viewpoint_camera, "tan_fov", None)
    if tan is not None:
        return tan
    fx, fy = viewpoint_camera.FoVx, viewpoint_camera.FoVy
    if isinstance(fx, torch.Tensor) and isinstance(fy, torch.Tensor) and (fx.requires_grad or fy.requires_grad):
        return torch.stack([torch.tan(fx * 0.5).reshape(()), torch.tan(fy * 0.5).reshape(())])
    return None


def render_raw(viewpoint_camera, pc, pipe, bg_color: torch.Tensor, scaling_modifier: float = 1.0):
    """`render()` without the epilogue: (raw (10,H,W) image, radii, viewspace_points).  The raw image is what
    `losses.hair_image_loss` consumes (it contains the epilogue), so a trainer built on this repository never
    materialises the four separate maps."""
    P = int(pc._xyz.shape[0])
    viewspace = empty_rows(P, (3,), torch.float32, pc._xyz.device).requires_grad_(True)
    st = _static(viewpoint_camera, bg_color, scaling_modifier, pc.active_sh_degree, getattr(pipe, "debug", False),
                 projection.GAUSSIAN_MODEL)
    renders, radii = _FusedRender.apply(
        pc._xyz, pc._scaling, pc._rotation, None, pc._features_dc, pc._features_rest, pc._opacity, pc._label, pc._orient_conf,
        viewspace, viewpoint_camera.world_view_transform, viewpoint_camera.full_proj_transform, viewpoint_camera.camera_center,
        _tanfov_tensor(viewpoint_camera), st)
    return renders, radii, viewspace


def render(viewpoint_camera, pc, pipe, bg_color: torch.Tensor, scaling_modifier: float = 1.0):
    """Same contract as the reference's `render` (src/gaussian_renderer/__init__.py:23-114); `pc` is a GaussianModel
    (src/scene/gaussian_model.py:45) or anything with its raw parameter attributes."""
    renders, radii, viewspace = render_raw(viewpoint_camera, pc, pipe, bg_color, scaling_modifier)
    return _post(renders, radii, viewspace)


def _head_block(pc) -> Optional[Dict[str, torch.Tensor]]:
    """The frozen head Gaussians that render_hair() composites behind the hair (the *_precomp attributes the strand
    trainers attach, src/train_strands.py:67-73).  Cached on the model: they never change during strand training."""
    cache = getattr(pc, "_gh_head_block", None)
    if cache is not None and cache["key"] is pc.xyz_precomp:
        return cache
    with torch.no_grad():
        shs = pc.shs_view                                           # (n, 3, 16) channel-major
        feats = shs.transpose(1, 2).contiguous()                    # (n, 16, 3) like get_features
        blk = {"key": pc.xyz_precomp, "xyz": pc.xyz_precomp.contiguous(), "scaling": pc.scaling_precomp.contiguous(),
               "rotation": pc.rotation_precomp.contiguous(), "opacity": pc.opacity_precomp.contiguous(),
               "f_dc": feats[:, :1].contiguous(), "f_rest": feats[:, 1:].contiguous()}
    pc._gh_head_block = blk
    return blk


def render_hair(viewpoint_camera, pc, pc_hair, pipe, bg_color: torch.Tensor, scaling_modifier: float = 1.0):
    """Same contract as the reference's `render_hair` (src/gaussian_renderer/__init__.py:116-236): the frozen head
    Gaussians of `pc` (label < 0.5) followed by the strand Gaussians of `pc_hair`."""
    head = _head_block(pc)
    n_head = int(head["xyz"].shape[0])
    P = n_head + int(pc_hair.get_xyz.shape[0])
    dev = pc_hair.get_xyz.device
    viewspace = empty_rows(P, (3,), torch.float32, dev).requires_grad_(True)
    st = _static(viewpoint_camera, bg_color, scaling_modifier, pc_hair.active_sh_degree, getattr(pipe, "debug", False),
                 projection.HAIR_MODEL)
    st["head"] = head if n_head > 0 else None
    renders, radii = _FusedRender.apply(
        pc_hair.get_xyz, pc_hair.get_scaling, pc_hair._rotation, pc_hair._dir, pc_hair._features_dc, pc_hair._features_rest,
        None, None, pc_hair._orient_conf, viewspace, viewpoint_camera.world_view_transform,
        viewpoint_camera.full_proj_transform, viewpoint_camera.camera_center, _tanfov_tensor(viewpoint_camera), st)
    return _post(renders, radii, viewspace)


def render_hair_strands(viewpoint_camera, pc, pc_hair, pipe, bg_color: torch.Tensor, scaling_modifier: float = 1.0):
    """`render_hair` for a GaussianModelCurves (src/scene/gaussian_model_strands.py:31) rendered straight from its
    polylines: same contract and returned dictionary as render_hair, but the strand Gaussians are built inside the
    kernels from the trained segment vectors `pc_hair._dirs` (S,L,3) and `pc_hair.pts_origins` (S,1,3) -- midpoints,
    |d|/2 scales and parallel-transport rotations, what initialize_gaussians_hair() (:435-454) rebuilds in PyTorch --
    so the trainer drops its initialize_gaussians_hair() call.  Also read: `scale` (the strand thickness, a (1,) CUDA
    tensor or a float), `_features_dc`, `_features_rest`, `_orient_conf` (S*L rows, strand-major), `active_sh_degree`.
    Gradients land in `.grad` of `_dirs`, `_features_dc`, `_features_rest`, `_orient_conf`, of `viewspace_points`
    and of trainable camera tensors; set_nan_flag() works as with render_hair.  `pc` supplies the frozen head block
    like in render_hair (None or an empty block: hair only).

    This does NOT refresh `pc_hair._pts`, `_xyz` or `_rotation`: a trainer that calls `capture()` (which saves them)
    runs the model's own initialize_gaussians_hair() under torch.no_grad() first.  The strand model has no
    gradient-arena layout: an installed arena (projection.set_gradient_arena) raises.

    render_hair_strands_capturable is the CUDA-graph form (graphs.CapturedStrandStep captures the whole train_strands.py
    iteration with it): one first phase over the head and strand rows, a records-mode backward, and the same image,
    radii and deterministic-mode gradients as this function."""
    projection._check_no_strand_arena()
    dirs = pc_hair._dirs
    if dirs.ndim != 3 or dirs.shape[-1] != 3 or dirs.shape[1] < 1:
        raise RuntimeError(f"render_hair_strands: _dirs must be (S, L, 3), got {tuple(dirs.shape)}")
    S, L = int(dirs.shape[0]), int(dirs.shape[1])
    dev = dirs.device
    origins = pc_hair.pts_origins
    if origins.numel() != S * 3:
        raise RuntimeError(f"render_hair_strands: pts_origins must be (S, 1, 3) = ({S}, 1, 3), got {tuple(origins.shape)}")
    for name in ("_features_dc", "_features_rest", "_orient_conf"):
        t = getattr(pc_hair, name)
        if t.shape[0] != S * L:
            raise RuntimeError(f"render_hair_strands: {name} must have S*L = {S * L} rows (strand-major), got {t.shape[0]}")
    scale = pc_hair.scale
    if not isinstance(scale, torch.Tensor):
        scale = torch.full((1,), float(scale), dtype=torch.float32, device=dev)
    head = _head_block(pc) if pc is not None else None
    n_head = 0 if head is None else int(head["xyz"].shape[0])
    viewspace = empty_rows(n_head + S * L, (3,), torch.float32, dev).requires_grad_(True)
    st = _static(viewpoint_camera, bg_color, scaling_modifier, pc_hair.active_sh_degree, getattr(pipe, "debug", False),
                 projection.HAIR_STRANDS)
    st["head"] = head if n_head > 0 else None
    st["strands"] = {"origins": origins.detach(), "S": S, "L": L}
    renders, radii = _FusedRender.apply(
        None, scale.detach(), None, dirs, pc_hair._features_dc, pc_hair._features_rest, None, None, pc_hair._orient_conf,
        viewspace, viewpoint_camera.world_view_transform, viewpoint_camera.full_proj_transform,
        viewpoint_camera.camera_center, _tanfov_tensor(viewpoint_camera), st)
    return _post(renders, radii, viewspace)


def render_hair_segments(viewpoint_camera, pc, pc_hair, pipe, bg_color: torch.Tensor, scaling_modifier: float = 1.0):
    """`render_hair` for a GaussianModelHair (src/scene/gaussian_model_latent_strands.py:28) on the fused strand path:
    same contract and returned dictionary as render_hair, but the strand Gaussians' scales and rotations are derived
    inside the kernels from the segment vectors, so neither `get_scaling` nor `_rotation` is read.  Read: `_xyz` (N,3)
    segment midpoints, `_dir` (N,3) segment vectors, `scale` (the strand thickness, a (1,) CUDA tensor or a float),
    `_features_dc`, `_features_rest`, `_orient_conf` (N rows, strand-major) and `active_sh_degree`.  Autograd carries
    the gradients of the five tensors back to whatever produced them -- the strand decoder's parameters in training,
    or leaves -- and also fills `.grad` of `viewspace_points` and of trainable camera tensors; set_nan_flag() works as
    with render_hair.  `pc` supplies the frozen head block like in render_hair (None or an empty block: hair only).

    A train_latent_strands.py loop replaces `pc_hair.initialize_gaussians_hair(iteration)` -- generate_strands() plus
    the parallel-transport rotations this function does not need -- with

        diffusion_dict = pc_hair.generate_strands(iteration)
        pc_hair.LDiff = diffusion_dict.get("L_diff")

    and renders with this function.  The strand model has no gradient-arena layout: an installed arena
    (projection.set_gradient_arena) raises.

    render_hair_segments_capturable is the CUDA-graph form (graphs.CapturedLatentStrandStep captures render, loss and
    backward down to the five tensors with it)."""
    projection._check_no_strand_arena()
    N = _segment_rows(pc_hair, "render_hair_segments")
    dev = pc_hair._xyz.device
    scale = pc_hair.scale
    if not isinstance(scale, torch.Tensor):
        scale = torch.full((1,), float(scale), dtype=torch.float32, device=dev)
    head = _head_block(pc) if pc is not None else None
    n_head = 0 if head is None else int(head["xyz"].shape[0])
    viewspace = empty_rows(n_head + N, (3,), torch.float32, dev).requires_grad_(True)
    st = _static(viewpoint_camera, bg_color, scaling_modifier, pc_hair.active_sh_degree, getattr(pipe, "debug", False),
                 projection.HAIR_STRANDS)
    st["head"] = head if n_head > 0 else None
    renders, radii = _FusedRender.apply(
        pc_hair._xyz, scale.detach(), None, pc_hair._dir, pc_hair._features_dc, pc_hair._features_rest, None, None,
        pc_hair._orient_conf, viewspace, viewpoint_camera.world_view_transform, viewpoint_camera.full_proj_transform,
        viewpoint_camera.camera_center, _tanfov_tensor(viewpoint_camera), st)
    return _post(renders, radii, viewspace)
