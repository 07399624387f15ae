"""Strand-model test infrastructure: seeded polylines, the restated strand geometry of GaussianModelCurves, and a real
GaussianModelCurves built around them (reference src/scene/gaussian_model_strands.py:31, :435-454).

* `make_strand_polylines`: origins (S,1,3), segment vectors (S,L,3) and per-segment features (S*L rows, strand-major),
  drawn with the recipe of oracle/synth.py `make_strand_scene`;
* `strand_geometry_reference`: initialize_gaussians_hair() restated as differentiable PyTorch -- midpoints, |d|/2
  scales, parallel-transport rotations -- whose output feeds synth.project_reference (HAIR_MODEL semantics); pinned on
  the reference's own class by tests/golden/pyref_strands.npz;
* `make_curves_models`: the reference's GaussianModelCurves via __new__ (its __init__ loads networks that are absent),
  with setup_functions() called and use_sds = False, so that its own initialize_gaussians_hair() runs unmodified.
"""
from __future__ import annotations

import torch
import torch.nn.functional as F

import _util

synth = _util.synth


def make_strand_polylines(S: int, L: int, seed: int = 0):
    """-> dict(origins (S,1,3), dirs (S,L,3), f_dc (S*L,1,3), f_rest (S*L,15,3), conf (S*L,1) raw log-confidence,
    scale float): CPU float32, drawn from torch.Generator().manual_seed(seed) with the recipe of oracle/synth.py
    `make_strand_scene` (roots on a 0.1 sphere, a random walk of 2 mm segments with a slight pull along +y)."""
    g = torch.Generator().manual_seed(seed)
    roots = 0.10 * F.normalize(torch.randn(S, 3, generator=g), dim=-1)
    d = F.normalize(roots, dim=-1)
    gravity = torch.tensor([0.0, 1.0, 0.0])
    segs = []
    for _ in range(L):
        d = F.normalize(d + 0.15 * torch.randn(S, 3, generator=g) + 0.02 * gravity, dim=-1)
        segs.append(0.002 * d)
    P = S * L
    f_dc = (torch.rand(P, 1, 3, generator=g) - 0.5) / synth.SH_C0
    f_rest = 0.1 * torch.randn(P, 15, 3, generator=g)
    conf = 0.1 * torch.randn(P, 1, generator=g)
    return {"origins": roots[:, None, :].contiguous(), "dirs": torch.stack(segs, dim=1).contiguous(),
            "f_dc": f_dc.contiguous(), "f_rest": f_rest.contiguous(), "conf": conf.contiguous(), "scale": 2e-4}


def strand_geometry_reference(origins: torch.Tensor, dirs: torch.Tensor, scale):
    """initialize_gaussians_hair() (gaussian_model_strands.py:435-454) as differentiable PyTorch:
    -> dict(xyz (P,3) midpoints, scaling (P,3) = (|d|/2, scale, scale), rotation (P,4) un-normalised
    parallel_transport(e_x, d), dirs (P,3))."""
    S, L = dirs.shape[0], dirs.shape[1]
    pts = origins + torch.cat([torch.zeros_like(origins), torch.cumsum(dirs, dim=1)], dim=1)
    d = dirs.reshape(-1, 3)
    xyz = ((pts[:, 1:] + pts[:, :-1]) * 0.5).reshape(-1, 3)
    ex = torch.cat([torch.ones_like(d[:, :1]), torch.zeros_like(d[:, :2])], dim=-1)
    rotation = synth.parallel_transport(ex, d)
    sc = scale if isinstance(scale, torch.Tensor) else torch.tensor(float(scale), dtype=d.dtype, device=d.device)
    scaling = torch.cat([d.norm(dim=-1, keepdim=True) * 0.5, sc.reshape(1, 1).expand(S * L, 2)], dim=-1)
    return {"xyz": xyz, "scaling": scaling, "rotation": rotation, "dirs": d}


def project_strands_reference(origins, dirs, scale, f_dc, f_rest, conf, cam, sh_degree=3, scaling_modifier=1.0):
    """strand_geometry_reference + synth.project_reference with the HAIR_MODEL semantics."""
    geo = strand_geometry_reference(origins, dirs, scale)
    raw = dict(geo, f_dc=f_dc, f_rest=f_rest, conf=conf)
    return synth.project_reference(raw, cam, dict(synth.PROJECT_HAIR_MODEL), sh_degree=sh_degree,
                                   scaling_modifier=scaling_modifier), geo


def make_curves_models(head_scene, poly, device, sh_degree: int = 3):
    """(pc, pc_hair) for render_hair / render_hair_strands: `pc` the frozen head GaussianModel of
    oracle/ref_python.make_hair_models (None-free: an empty head scene gives an empty block) and `pc_hair` a real
    GaussianModelCurves whose trained parameters are leaves: _dirs (S,L,3), _features_dc, _features_rest, _orient_conf;
    pts_origins and scale are plain tensors as create_from_pcd leaves them (:538, :571-576)."""
    import ref_python
    from torch import nn
    ref_python.load_renderer("mine")                      # stubs + the reference's sources on sys.path
    from scene.gaussian_model_strands import GaussianModelCurves
    pc = ref_python.make_gaussian_model(head_scene, device, sh_degree)
    with torch.no_grad():
        pc.mask_precomp = pc.get_label[..., 0] < 0.5
        pc.xyz_precomp = pc.get_xyz[pc.mask_precomp].detach()
        pc.opacity_precomp = pc.get_opacity[pc.mask_precomp].detach()
        pc.scaling_precomp = pc.get_scaling[pc.mask_precomp].detach()
        pc.rotation_precomp = pc.get_rotation[pc.mask_precomp].detach()
        pc.shs_view = pc.get_features[pc.mask_precomp].detach().transpose(1, 2).view(-1, 3, (pc.max_sh_degree + 1) ** 2)
    hair = GaussianModelCurves.__new__(GaussianModelCurves)
    hair.setup_functions()
    hair.use_sds = False
    hair.active_sh_degree = hair.max_sh_degree = sh_degree
    P = lambda t: nn.Parameter(t.detach().clone().to(device).contiguous().requires_grad_(True))  # noqa: E731
    hair.pts_origins = poly["origins"].to(device)
    hair._dirs = P(poly["dirs"])
    hair._features_dc = P(poly["f_dc"])
    hair._features_rest = P(poly["f_rest"])
    hair._orient_conf = P(poly["conf"])
    hair.scale = poly["scale"] * torch.ones(1, device=device)
    return pc, hair


def empty_head_scene():
    """A head scene without any Gaussian (render_hair's head block is then empty)."""
    s = synth.make_blob_scene(1, seed=0)
    return {k: v[:0] for k, v in s.items()}


CURVES_PARAMS = ("_dirs", "_features_dc", "_features_rest", "_orient_conf")
