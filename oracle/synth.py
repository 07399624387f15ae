"""Synthetic, seeded inputs for the rasterizer hot path (bench harness + parity tests).

Implements the scene / camera / caller-preamble specification of SURVEY.md section 8(d):

* scene "strands(S)": S strands x 100 segments -> P = 100*S strand-aligned Gaussians built the way
  `GaussianModelCurves.initialize_gaussians_hair` builds them
  (reference src/scene/gaussian_model_strands.py:435-454, src/utils/general_utils.py:150-160);
* K cameras on a ring, matrices in the reference's transposed row-vector convention
  (src/scene/cameras.py:72-81, src/utils/graphics_utils.py:51-72);
* the caller-side preamble of `render()` / `render_hair()` that turns model parameters into the
  tensors the rasterizer receives (src/gaussian_renderer/__init__.py:29-83, src/scene/gaussian_model.py:
  230-337, src/utils/sh_utils.py:57-112) -- written here from the math, device-agnostic, float32.

Everything is generated on the CPU from torch.Generator().manual_seed(seed) and moved afterwards, so
the same bytes reach every implementation under test.  There is no dataset and no checkpoint:
callers must label results "synthetic".
"""
from __future__ import annotations

import math
from typing import Dict, Optional

import torch
import torch.nn.functional as F

SH_C0 = 0.28209479177387814
SH_C1 = 0.4886025119029199
SH_C2 = (1.0925484305920792, -1.0925484305920792, 0.31539156525252005, -1.0925484305920792, 0.5462742152960396)
SH_C3 = (-0.5900435899266435, 2.890611442640554, -0.4570457994644658, 0.3731763325901154,
         -0.4570457994644658, 1.445305721320277, -0.5900435899266435)

NUM_CHANNELS = 10
BG_DEFAULT = (0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 100.0)   # depth background = 100 (train_gaussians.py:68)


# ----------------------------------------------------------------------------------------------- scene
def parallel_transport(a: torch.Tensor, b: torch.Tensor) -> torch.Tensor:
    """Quaternion (s, v) rotating unit a onto unit b, un-normalised (general_utils.py:150-160)."""
    a = F.normalize(a, dim=-1)
    b = F.normalize(b, dim=-1)
    s = 1 + (a * b).sum(dim=-1, keepdim=True)
    v = torch.cross(a, b, dim=-1)
    return torch.cat([s, v], dim=-1)


# torch's CPU elementwise kernels split a tensor of more than 32768 elements into one part per thread, and whether an
# element falls in a part's vectorised loop or in its scalar remainder -- which round sigmoid / exp differently --
# depends on where the parts start, so the float32 bits of a large scene would depend on the machine's thread count.  The
# scenes apply them part by part as torch does with 16 threads (the split the stored reference records were made with),
# each part on one thread: the same bits on every machine.
_GRAIN, _THREADS = 32768, 16


def _fixed_chunks(fn, x: torch.Tensor) -> torch.Tensor:
    flat = x.reshape(-1)
    n = flat.numel()
    size = -(-n // max(1, min(_THREADS, -(-n // _GRAIN))))
    prev = torch.get_num_threads()
    torch.set_num_threads(1)
    try:
        out = torch.cat([fn(flat[i:i + size]) for i in range(0, n, size)])
    finally:
        torch.set_num_threads(prev)
    return out.reshape(x.shape)


def make_strand_scene(num_strands: int, seed: int = 0, opacity_mode: str = "random",
                      segments: int = 100) -> Dict[str, torch.Tensor]:
    """CPU float32 tensors of the strands(S) scene: P = segments * num_strands Gaussians."""
    g = torch.Generator().manual_seed(seed)
    S = num_strands
    roots = 0.10 * F.normalize(torch.randn(S, 3, generator=g), dim=-1)
    d = F.normalize(roots, dim=-1)
    gravity = torch.tensor([0.0, 1.0, 0.0])
    dirs = []
    for _ in range(segments):
        d = F.normalize(d + 0.15 * torch.randn(S, 3, generator=g) + 0.02 * gravity, dim=-1)
        dirs.append(0.002 * d)
    dirs = torch.stack(dirs, dim=1)                                     # (S, seg, 3) segment vectors
    pts = roots[:, None, :] + torch.cat([torch.zeros(S, 1, 3), torch.cumsum(dirs, dim=1)], dim=1)
    xyz = ((pts[:, 1:] + pts[:, :-1]) * 0.5).reshape(-1, 3)            # strand-major
    dirv = dirs.reshape(-1, 3)
    P = xyz.shape[0]
    ex = torch.cat([torch.ones(P, 1), torch.zeros(P, 2)], dim=-1)
    rotation = F.normalize(parallel_transport(ex, dirv), dim=-1)        # get_rotation = normalize(_rotation)
    scaling = torch.full((P, 3), 2e-4)
    scaling[:, 0] = dirv.norm(dim=-1) * 0.5
    if opacity_mode == "random":
        opacity = _fixed_chunks(torch.sigmoid, 1 + torch.randn(P, 1, generator=g))
    elif opacity_mode == "ones":                                        # real hair: opacity == 1
        _ = torch.randn(P, 1, generator=g)
        opacity = torch.ones(P, 1)
    else:
        raise ValueError(opacity_mode)
    f_dc = (torch.rand(P, 1, 3, generator=g) - 0.5) / SH_C0
    f_rest = 0.1 * torch.randn(P, 15, 3, generator=g)
    label = _fixed_chunks(torch.sigmoid, torch.randn(P, 1, generator=g))
    orient_conf = _fixed_chunks(torch.exp, 0.1 * torch.randn(P, 1, generator=g))
    return {"xyz": xyz.contiguous(), "dir": dirv.contiguous(), "rotation": rotation.contiguous(),
            "scaling": scaling.contiguous(), "opacity": opacity.contiguous(),
            "f_dc": f_dc.contiguous(), "f_rest": f_rest.contiguous(),
            "label": label.contiguous(), "orient_conf": orient_conf.contiguous()}


def make_blob_scene(P: int, seed: int = 0, spread: float = 0.25, max_scale: float = 0.03) -> Dict[str, torch.Tensor]:
    """Generic anisotropic Gaussians (not strand-aligned): exercises large splats, un-normalised
    quaternions, long per-tile lists.  Used by parity tests only."""
    g = torch.Generator().manual_seed(seed)
    xyz = spread * torch.randn(P, 3, generator=g)
    scaling = max_scale * torch.rand(P, 3, generator=g) + 1e-4
    rotation = F.normalize(torch.randn(P, 4, generator=g), dim=-1) * (0.5 + torch.rand(P, 1, generator=g))
    opacity = _fixed_chunks(torch.sigmoid, torch.randn(P, 1, generator=g))
    f_dc = (torch.rand(P, 1, 3, generator=g) - 0.5) / SH_C0
    f_rest = 0.1 * torch.randn(P, 15, 3, generator=g)
    label = _fixed_chunks(torch.sigmoid, torch.randn(P, 1, generator=g))
    orient_conf = _fixed_chunks(torch.exp, 0.1 * torch.randn(P, 1, generator=g))
    dirv = F.normalize(torch.randn(P, 3, generator=g), dim=-1) * scaling.max(dim=-1, keepdim=True).values
    return {"xyz": xyz, "dir": dirv, "rotation": rotation.contiguous(), "scaling": scaling, "opacity": opacity,
            "f_dc": f_dc, "f_rest": f_rest, "label": label, "orient_conf": orient_conf}


# ---------------------------------------------------------------------------------------------- camera
def make_camera(k: int, width: int, height: int, num_cameras: int = 64, radius: float = 0.8,
                focal_factor: float = 1.2, znear: float = 0.01, zfar: float = 100.0) -> Dict[str, object]:
    """Camera k of a ring of `num_cameras` in the xz-plane looking at the origin (x right, y down,
    z forward).  Matrices are float32 and TRANSPOSED like the reference's (cameras.py:72-81)."""
    theta = 2.0 * math.pi * k / num_cameras
    c = torch.tensor([radius * math.sin(theta), 0.0, radius * math.cos(theta)], dtype=torch.float64)
    zc = -c / c.norm()
    yc = torch.tensor([0.0, 1.0, 0.0], dtype=torch.float64)
    xc = torch.linalg.cross(yc, zc)
    xc = xc / xc.norm()
    R = torch.stack([xc, yc, zc], dim=0)                 # world -> camera
    t = -R @ c
    w2c = torch.eye(4, dtype=torch.float64)
    w2c[:3, :3] = R
    w2c[:3, 3] = t
    focal = focal_factor * height
    fovx = 2.0 * math.atan(width / (2.0 * focal))
    fovy = 2.0 * math.atan(height / (2.0 * focal))
    tanx, tany = math.tan(fovx * 0.5), math.tan(fovy * 0.5)
    Pm = torch.zeros(4, 4, dtype=torch.float64)          # graphics_utils.py:51-72
    Pm[0, 0] = 1.0 / tanx
    Pm[1, 1] = 1.0 / tany
    Pm[3, 2] = 1.0
    Pm[2, 2] = zfar / (zfar - znear)
    Pm[2, 3] = -(zfar * znear) / (zfar - znear)
    world_view = w2c.t().contiguous()
    full_proj = world_view @ Pm.t()
    return {
        "image_width": int(width), "image_height": int(height),
        "FoVx": fovx, "FoVy": fovy, "tanfovx": tanx, "tanfovy": tany,
        "world_view_transform": world_view.float().contiguous(),
        "full_proj_transform": full_proj.float().contiguous(),
        "camera_center": c.float().contiguous(),
    }


# -------------------------------------------------------------------------------------- caller preamble
def eval_sh(deg: int, sh: torch.Tensor, dirs: torch.Tensor) -> torch.Tensor:
    """sh: (P, 3, (deg_max+1)^2), dirs: (P, 3) unit -> (P, 3)   (sh_utils.py:57-112, deg <= 3)."""
    res = SH_C0 * sh[..., 0]
    if deg > 0:
        x, y, z = dirs[..., 0:1], dirs[..., 1:2], dirs[..., 2:3]
        res = res - SH_C1 * y * sh[..., 1] + SH_C1 * z * sh[..., 2] - SH_C1 * x * sh[..., 3]
        if deg > 1:
            xx, yy, zz, xy, yz, xz = x * x, y * y, z * z, x * y, y * z, x * z
            res = (res + SH_C2[0] * xy * sh[..., 4] + SH_C2[1] * yz * sh[..., 5]
                   + SH_C2[2] * (2.0 * zz - xx - yy) * sh[..., 6] + SH_C2[3] * xz * sh[..., 7]
                   + SH_C2[4] * (xx - yy) * sh[..., 8])
            if deg > 2:
                res = (res + SH_C3[0] * y * (3 * xx - yy) * sh[..., 9] + SH_C3[1] * xy * z * sh[..., 10]
                       + SH_C3[2] * y * (4 * zz - xx - yy) * sh[..., 11]
                       + SH_C3[3] * z * (2 * zz - 3 * xx - 3 * yy) * sh[..., 12]
                       + SH_C3[4] * x * (4 * zz - xx - yy) * sh[..., 13]
                       + SH_C3[5] * z * (xx - yy) * sh[..., 14] + SH_C3[6] * x * (xx - 3 * yy) * sh[..., 15])
    return res


def build_rotation_glm(q: torch.Tensor) -> torch.Tensor:
    """(P,4) raw (r,x,y,z) -> (P,3,3) in the layout the CUDA code's glm::mat3 literal produces
    (i.e. the transpose of the textbook matrix; general_utils.py:79-109 WITHOUT its normalisation)."""
    r, x, y, z = q[:, 0], q[:, 1], q[:, 2], q[:, 3]
    R = torch.zeros(q.shape[0], 3, 3, dtype=q.dtype, device=q.device)
    R[:, 0, 0] = 1 - 2 * (y * y + z * z); R[:, 1, 0] = 2 * (x * y - r * z); R[:, 2, 0] = 2 * (x * z + r * y)
    R[:, 0, 1] = 2 * (x * y + r * z); R[:, 1, 1] = 1 - 2 * (x * x + z * z); R[:, 2, 1] = 2 * (y * z - r * x)
    R[:, 0, 2] = 2 * (x * z - r * y); R[:, 1, 2] = 2 * (y * z + r * x); R[:, 2, 2] = 1 - 2 * (x * x + y * y)
    return R


def covariance3d(scaling: torch.Tensor, rotation: torch.Tensor, modifier: float = 1.0):
    """(P,3,3) Sigma = (S R)^T (S R) and its 6-vector [xx,xy,xz,yy,yz,zz] (gaussian_model.py:230-250)."""
    s = scaling * modifier
    R = build_rotation_glm(rotation)
    M = s[:, :, None] * R                  # diag(s) @ R
    full = M.transpose(1, 2) @ M
    six = torch.stack([full[:, 0, 0], full[:, 0, 1], full[:, 0, 2], full[:, 1, 1], full[:, 1, 2], full[:, 2, 2]], dim=-1)
    return full, six


def _view_xyz(xyz, viewmatrix):
    return xyz @ viewmatrix[:3, :3] + viewmatrix[3:4, :3]


def _proj_transform_cov(xyz, cam):
    """T = W @ J of gaussian_model.py:252-297 (P,3,3)."""
    vm = cam["world_view_transform"].to(xyz)
    W, H = cam["image_width"], cam["image_height"]
    tanx, tany = cam["tanfovx"], cam["tanfovy"]
    fx, fy = W / (2.0 * tanx), H / (2.0 * tany)
    t = _view_xyz(xyz, vm)
    tx, ty, tz = t[:, 0], t[:, 1], t[:, 2]
    limx, limy = 1.3 * tanx, 1.3 * tany
    tx = torch.clamp(tx / tz, min=-limx, max=limx) * tz
    ty = torch.clamp(ty / tz, min=-limy, max=limy) * tz
    z0 = torch.zeros_like(tz)
    J = torch.stack([torch.stack([fx / tz, z0, -(fx * tx) / (tz * tz)], dim=-1),
                     torch.stack([z0, fy / tz, -(fy * ty) / (tz * tz)], dim=-1),
                     torch.stack([z0, z0, z0], dim=-1)], dim=-1)
    return vm[None, :3, :3] @ J


def caller_preamble(scene: Dict[str, torch.Tensor], cam: Dict[str, object], sh_degree: int = 3,
                    scaling_modifier: float = 1.0, strand_dir: bool = True) -> Dict[str, torch.Tensor]:
    """What `render()` / `render_hair()` compute in PyTorch before calling the rasterizer."""
    xyz = scene["xyz"]
    vm = cam["world_view_transform"].to(xyz)
    pm = cam["full_proj_transform"].to(xyz)
    cov_full, cov6 = covariance3d(scene["scaling"], scene["rotation"], scaling_modifier)
    T = _proj_transform_cov(xyz, cam)
    cov2d_full = T.transpose(1, 2) @ cov_full.transpose(1, 2) @ T
    a = cov2d_full[:, 0, 0] + 0.3
    b = cov2d_full[:, 0, 1]
    c = cov2d_full[:, 1, 1] + 0.3
    det = a * c - b * b
    conic = torch.stack([c, -b, a], dim=-1) * (1.0 / (det + 1e-12))[:, None]      # gaussian_model.py:303-315
    p_hom = xyz @ pm[:3, :] + pm[3:4, :]
    p_w = 1.0 / (p_hom[:, 3:4] + 0.0000001)
    means2D = p_hom[:, :3] * p_w                                                   # NDC (gaussian_model.py:317-337)
    depths = _view_xyz(xyz, vm)[:, 2:3]
    shs_view = torch.cat([scene["f_dc"], scene["f_rest"]], dim=1).transpose(1, 2)  # (P,3,16)
    dir_pp = xyz - cam["camera_center"].to(xyz)[None]
    dir_pp = dir_pp / dir_pp.norm(dim=1, keepdim=True)
    rgb = torch.clamp_min(eval_sh(sh_degree, shs_view, dir_pp) + 0.5, 0.0)
    if strand_dir:
        dir3d = F.normalize(scene["dir"], dim=-1)                                   # gaussian_model_strands.py:429-431
    else:
        dir3d = scene["dir"]
    dir2d = (dir3d[:, None, :] @ T)[:, 0]
    colors = torch.cat([rgb, scene["label"], torch.ones_like(scene["label"]), dir2d,
                        scene["orient_conf"], depths], dim=-1)                      # gaussian_renderer/__init__.py:64-74
    return {"means2D": means2D.contiguous(), "conic": conic.contiguous(), "cov3D": cov6.contiguous(),
            "colors": colors.contiguous(), "depths": depths.contiguous(),
            "cov2d": torch.stack([a, b, c], dim=-1)}


def filter_points(pre: Dict[str, torch.Tensor], scene, cam) -> torch.Tensor:
    """The caller's prefilter (gaussian_model.py:143-228): near cull, det != 0, non-empty tile rect."""
    W, H = cam["image_width"], cam["image_height"]
    vm = cam["world_view_transform"].to(scene["xyz"])
    z = _view_xyz(scene["xyz"], vm)[:, 2]
    a, b, c = pre["cov2d"][:, 0], pre["cov2d"][:, 1], pre["cov2d"][:, 2]
    det = a * c - b * b
    mask = (z > 0.2) & (det != 0)
    mid = 0.5 * (a + c)
    sq = torch.clamp(mid * mid - det, min=0.1) ** 0.5
    radius = torch.ceil(3 * torch.maximum(mid + sq, mid - sq) ** 0.5)
    px = ((pre["means2D"][:, 0] + 1) * W - 1.0) * 0.5
    py = ((pre["means2D"][:, 1] + 1) * H - 1.0) * 0.5
    gx, gy = (W + 15) // 16, (H + 15) // 16
    x0 = torch.clamp(((px - radius) / 16).int(), 0, gx); y0 = torch.clamp(((py - radius) / 16).int(), 0, gy)
    x1 = torch.clamp(((px + radius + 15) / 16).int(), 0, gx); y1 = torch.clamp(((py + radius + 15) / 16).int(), 0, gy)
    return mask & ((x1 - x0) * (y1 - y0) != 0)


def upstream_gradient(width: int, height: int, seed: int = 0) -> torch.Tensor:
    """dL/d(out) = rand(10, H, W): loss = sum(out * Wt)."""
    g = torch.Generator().manual_seed(1000 + seed)
    return torch.rand(NUM_CHANNELS, height, width, generator=g)


MODES = ("native", "render", "render_hair", "cov3d")


def rasterizer_inputs(scene, cam, mode: str = "native", sh_degree: int = 3,
                      device: Optional[torch.device] = None) -> Dict[str, object]:
    """Keyword arguments for `GaussianRasterizer.forward` + the settings fields, for one of:

    native       scales + rotations + colors_precomp, conic computed in-kernel   (all four stages)
    cov3d        cov3D_precomp + colors_precomp, conic computed in-kernel        (stock 3DGS shape)
    render       cov3D_precomp + conic_precomp + colors_precomp  (src/gaussian_renderer/__init__.py:87-96)
    render_hair  scales + rotations + conic_precomp + colors_precomp              (:188-197)
    """
    if mode not in MODES:
        raise ValueError(mode)
    pre = caller_preamble(scene, cam, sh_degree)
    if mode in ("render", "render_hair"):
        mask = filter_points(pre, scene, cam)
    else:
        mask = torch.ones(scene["xyz"].shape[0], dtype=torch.bool)
    sel = lambda t: t[mask].contiguous()   # noqa: E731
    kw = {"means3D": sel(scene["xyz"]), "means2D": sel(pre["means2D"]), "opacities": sel(scene["opacity"]),
          "shs": None, "colors_precomp": sel(pre["colors"]), "scales": None, "rotations": None,
          "cov3D_precomp": None, "conic_precomp": None}
    if mode in ("native", "render_hair"):
        kw["scales"], kw["rotations"] = sel(scene["scaling"]), sel(scene["rotation"])
    else:
        kw["cov3D_precomp"] = sel(pre["cov3D"])
    if mode in ("render", "render_hair"):
        kw["conic_precomp"] = sel(pre["conic"])
    settings = {
        "image_height": cam["image_height"], "image_width": cam["image_width"],
        "tanfovx": cam["tanfovx"], "tanfovy": cam["tanfovy"],
        "bg": torch.tensor(BG_DEFAULT, dtype=torch.float32), "scale_modifier": 1.0,
        "viewmatrix": cam["world_view_transform"], "projmatrix": cam["full_proj_transform"],
        "sh_degree": sh_degree, "campos": cam["camera_center"],
        "prefiltered": mode in ("render", "render_hair"), "debug": False,
    }
    if device is not None:
        kw = {k: (v.to(device) if isinstance(v, torch.Tensor) else v) for k, v in kw.items()}
        settings = {k: (v.to(device) if isinstance(v, torch.Tensor) else v) for k, v in settings.items()}
    return {"kwargs": kw, "settings": settings, "mask": mask}


# ------------------------------------------------------------------------- caller preamble from RAW model parameters
# Oracle of the fused projection op (gaussianhaircut_b200/projection.py, csrc/gh_project.cu): the whole preamble of
# `render()` / `render_hair()` as differentiable PyTorch, from the parameters the models store.  Restates
#   GaussianModel      scene/gaussian_model.py:106-141 (activations), :230-393, gaussian_renderer/__init__.py:29-83
#   GaussianModelHair  scene/gaussian_model_latent_strands.py:109-148, :237-440, gaussian_renderer/__init__.py:122-186
# and is pinned on the reference's own Python (tests/golden/pyref_project_*.npz, make_golden_pyref_project.py).
PROJECT_GAUSSIAN_MODEL = dict(scale_act=1, opacity_act=1, label_act=1, conf_act=1, dir_mode=0, det_eps=1e-12)
PROJECT_HAIR_MODEL = dict(scale_act=0, opacity_act=2, label_act=2, conf_act=1, dir_mode=1, det_eps=1e-7)


def build_rotation_ref(q: torch.Tensor) -> torch.Tensor:
    """general_utils.py:79-109: normalises q, fills the TRANSPOSED layout."""
    q = q / torch.sqrt((q * q).sum(dim=1, keepdim=True))
    return build_rotation_glm(q)


def project_reference(raw: Dict[str, torch.Tensor], cam: Dict[str, object], cfg: Dict[str, object],
                      sh_degree: int = 3, scaling_modifier: float = 1.0) -> Dict[str, torch.Tensor]:
    """raw: xyz (P,3), scaling (P,3), rotation (P,4), f_dc (P,1,3), f_rest (P,15,3), opacity / label / conf (P,1)
    [ignored when the activation says 'constant'], dirs (P,3) for dir_mode 1.  cam: synth.make_camera dict whose
    matrices may be autograd leaves; 'tanfovx'/'tanfovy' may be tensors."""
    xyz = raw["xyz"]
    vm, pm, cc = cam["world_view_transform"].to(xyz), cam["full_proj_transform"].to(xyz), cam["camera_center"].to(xyz)
    W, H = cam["image_width"], cam["image_height"]
    tanx, tany = cam["tanfovx"], cam["tanfovy"]
    s = (torch.exp(raw["scaling"]) if cfg["scale_act"] == 1 else raw["scaling"]) * scaling_modifier
    R = build_rotation_ref(raw["rotation"])
    M = s[:, :, None] * R
    cov_full = M.transpose(1, 2) @ M
    cov6 = torch.stack([cov_full[:, 0, 0], cov_full[:, 0, 1], cov_full[:, 0, 2], cov_full[:, 1, 1], cov_full[:, 1, 2],
                        cov_full[:, 2, 2]], dim=-1)
    fx, fy = W / (2.0 * tanx), H / (2.0 * tany)
    t = xyz @ vm[:3, :3] + vm[3:4, :3]
    tz = t[:, 2]
    limx, limy = 1.3 * tanx, 1.3 * tany
    if isinstance(limx, torch.Tensor):
        tx = torch.maximum(torch.minimum(t[:, 0] / tz, limx), -limx) * tz
        ty = torch.maximum(torch.minimum(t[:, 1] / tz, limy), -limy) * tz
    else:
        tx = torch.clamp(t[:, 0] / tz, min=-limx, max=limx) * tz
        ty = torch.clamp(t[:, 1] / tz, min=-limy, max=limy) * tz
    z0 = torch.zeros_like(tz)
    J = torch.stack([torch.stack([fx / tz, z0, -(fx * tx) / (tz * tz)], dim=-1),
                     torch.stack([z0, fy / tz, -(fy * ty) / (tz * tz)], dim=-1),
                     torch.stack([z0, z0, z0], dim=-1)], dim=-1)
    T = vm[None, :3, :3] @ J
    cov2d = T.transpose(1, 2) @ cov_full.transpose(1, 2) @ T
    a, b, c = cov2d[:, 0, 0] + 0.3, cov2d[:, 0, 1], cov2d[:, 1, 1] + 0.3
    det = a * c - b * b
    conic = torch.stack([c, -b, a], dim=-1) * (1.0 / (det + cfg["det_eps"]))[:, None]
    p_hom = xyz @ pm[:3, :] + pm[3:4, :]
    means2D = p_hom[:, :3] * (1.0 / (p_hom[:, 3:4] + 0.0000001))
    depths = t[:, 2:3]
    shs_view = torch.cat([raw["f_dc"], raw["f_rest"]], dim=1).transpose(1, 2)
    d = xyz - cc[None]
    d = d / d.norm(dim=1, keepdim=True)
    rgb = torch.clamp_min(eval_sh(sh_degree, shs_view, d) + 0.5, 0.0)
    if cfg["dir_mode"] == 0:
        j = s.argmax(dim=1)                                                 # argsort(descending)[:, 0]
        idx = torch.arange(s.shape[0], device=s.device)
        dir3 = R[idx, j] * s[idx, j][:, None]                               # gaussian_model.py:385-389
    elif cfg["dir_mode"] == 1:
        dir3 = F.normalize(raw["dirs"], dim=-1)
    else:
        dir3 = torch.zeros_like(xyz)
    dir2d = (dir3[:, None, :] @ T)[:, 0]
    ones = torch.ones_like(depths)
    act = lambda v, mode, f: f(v) if mode == 1 else (v if mode == 0 else (ones if mode == 2 else torch.zeros_like(ones)))  # noqa: E731
    opacity = act(raw.get("opacity"), cfg["opacity_act"], torch.sigmoid)
    label = act(raw.get("label"), cfg["label_act"], torch.sigmoid)
    conf = act(raw.get("conf"), cfg["conf_act"], torch.exp)
    colors = torch.cat([rgb, label, ones, dir2d, conf, depths], dim=-1)
    with torch.no_grad():                                                   # filter_points (gaussian_model.py:143-228)
        mask = (t[:, 2] > 0.2) & (det != 0)
        mid = 0.5 * (a + c)
        sq = torch.clamp(mid * mid - det, min=0.1) ** 0.5
        radius = torch.ceil(3 * torch.maximum(mid + sq, mid - sq) ** 0.5)
        px = ((means2D[:, 0] + 1) * W - 1.0) * 0.5
        py = ((means2D[:, 1] + 1) * H - 1.0) * 0.5
        gx, gy = (W + 15) // 16, (H + 15) // 16
        x0 = torch.clamp(((px - radius) / 16).int(), 0, gx); y0 = torch.clamp(((py - radius) / 16).int(), 0, gy)
        x1 = torch.clamp(((px + radius + 15) / 16).int(), 0, gx); y1 = torch.clamp(((py + radius + 15) / 16).int(), 0, gy)
        mask = mask & ((x1 - x0) * (y1 - y0) != 0)
    return {"means2D": means2D, "conic": conic, "colors": colors, "opacity": opacity, "cov3D": cov6, "mask": mask,
            "cov2d": torch.stack([a, b, c], dim=-1)}


def raw_params_from_scene(scene: Dict[str, torch.Tensor], flavour: str = "gaussian_model") -> Dict[str, torch.Tensor]:
    """The parameters a model would store for a synthetic scene (logit / log spaces for GaussianModel)."""
    logit = lambda p: torch.log(p / (1 - p))   # noqa: E731
    if flavour == "gaussian_model":
        return {"xyz": scene["xyz"].clone(), "scaling": torch.log(scene["scaling"]), "rotation": scene["rotation"].clone(),
                "f_dc": scene["f_dc"].clone(), "f_rest": scene["f_rest"].clone(),
                "opacity": logit(scene["opacity"].clamp(1e-6, 1 - 1e-6)), "label": logit(scene["label"].clamp(1e-6, 1 - 1e-6)),
                "conf": torch.log(scene["orient_conf"])}
    return {"xyz": scene["xyz"].clone(), "scaling": scene["scaling"].clone(), "rotation": scene["rotation"].clone(),
            "dirs": scene["dir"].clone(), "f_dc": scene["f_dc"].clone(), "f_rest": scene["f_rest"].clone(),
            "conf": torch.log(scene["orient_conf"])}
