"""Golden vectors for the strand model rendered from its polylines (renderer.render_hair_strands) from the reference's
own Python.

The reference's GaussianModelCurves (src/scene/gaussian_model_strands.py:31) is imported UNMODIFIED (stubs + CPU
factory wrappers of make_golden_pyref.py), built via __new__ with setup_functions() and use_sds = False, given seeded
polylines (tests/_strands.py `make_strand_polylines`) and asked to run its own initialize_gaussians_hair() (:435-454)
and then for exactly what render_hair() asks it (src/gaussian_renderer/__init__.py:122-186): midpoints, scales,
rotations, conic, NDC mean, colour features, prefilter mask -- plus the gradients of a fixed random-weight loss w.r.t.
_dirs, the features, _orient_conf and the camera matrices.  Two models: (S=6, L=33) and (S=4, L=99), camera 7, 200x120.

    python tests/golden/make_golden_pyref_strands.py     (writes tests/golden/pyref_strands.npz)
"""
import os
import sys
import types

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import make_golden_pyref as base  # noqa: E402

MODELS = {"s6_l33": (6, 33, 11), "s4_l99": (4, 99, 12)}      # name -> (S, L, seed)


def main():
    base._cpu_factories()
    sys.path.insert(0, os.path.join(base.ROOT, "oracle"))
    sys.path.insert(0, os.path.join(base.ROOT, "tests"))
    import ref_python
    import synth
    import _strands
    ref_python.install_stubs()
    sys.path.insert(0, base.REF_SRC)
    from scene.gaussian_model_strands import GaussianModelCurves
    from utils.sh_utils import eval_sh

    W, H, cam_k = 200, 120, 7
    cam_d = synth.make_camera(cam_k, W, H)
    leaf = lambda t: t.detach().clone().requires_grad_(True)   # noqa: E731
    res = {"W": np.array(W), "H": np.array(H), "cam_k": np.array(cam_k)}
    for name, (S, L, seed) in MODELS.items():
        poly = _strands.make_strand_polylines(S, L, seed)
        vm, pm, cc = leaf(cam_d["world_view_transform"]), leaf(cam_d["full_proj_transform"]), leaf(cam_d["camera_center"])
        cam = types.SimpleNamespace(image_width=W, image_height=H, FoVx=torch.tensor(cam_d["FoVx"]), FoVy=torch.tensor(cam_d["FoVy"]),
                                    world_view_transform=vm, full_proj_transform=pm, camera_center=cc)
        hair = GaussianModelCurves.__new__(GaussianModelCurves)
        hair.setup_functions()
        hair.use_sds = False
        hair.active_sh_degree = hair.max_sh_degree = 3
        leaves = {"dirs": leaf(poly["dirs"]), "f_dc": leaf(poly["f_dc"]), "f_rest": leaf(poly["f_rest"]), "conf": leaf(poly["conf"])}
        hair.pts_origins = poly["origins"].clone()
        hair._dirs = leaves["dirs"]
        hair._features_dc, hair._features_rest, hair._orient_conf = leaves["f_dc"], leaves["f_rest"], leaves["conf"]
        hair.scale = poly["scale"] * torch.ones(1)
        hair.initialize_gaussians_hair()                          # the model's own geometry rebuild
        conic = hair.get_conic(cam)
        m2 = hair.get_mean_2d(cam)
        shs_view = hair.get_features.transpose(1, 2).view(-1, 3, 16)
        d = hair.get_xyz - cam.camera_center.repeat(hair.get_features.shape[0], 1)
        d = d / d.norm(dim=1, keepdim=True)
        rgb = torch.clamp_min(eval_sh(3, shs_view, d) + 0.5, 0.0)
        label = hair.get_label
        colors = torch.cat([rgb, label, torch.ones_like(label), hair.get_direction_2d(cam), hair.get_orient_conf,
                            hair.get_depths(cam)], dim=-1)
        mask = hair.filter_points(cam)
        out = {"conic": conic, "means2D": m2, "colors": colors}
        g = torch.Generator().manual_seed(100 + seed)
        Wt = {k: torch.rand(v.shape, generator=g) for k, v in out.items()}
        Wt["conic"] *= 1e-3
        Wt["means2D"][:, 2] = 0.0
        m = mask[:, None].float()
        loss = sum((out[k] * Wt[k] * m).sum() for k in out)
        loss.backward()
        p = name + "/"
        res.update({p + "S": np.array(S), p + "L": np.array(L), p + "seed": np.array(seed), p + "mask": mask.numpy(),
                    p + "xyz": hair._xyz.detach().numpy(), p + "scaling": hair._scaling.detach().numpy(),
                    p + "rotation": hair._rotation.detach().numpy()})
        res.update({p + k: v.detach().numpy() for k, v in out.items()})
        res.update({p + "W_" + k: v.numpy() for k, v in Wt.items()})
        res.update({p + "g_" + k: v.grad.numpy() for k, v in leaves.items()})
        res.update({p + "g_viewmatrix": vm.grad.numpy(), p + "g_projmatrix": pm.grad.numpy(), p + "g_campos": cc.grad.numpy()})
        print(name, "visible", int(mask.sum()), "of", mask.numel())
    path = os.path.join(HERE, "pyref_strands.npz")
    np.savez_compressed(path, **res)
    print("wrote", path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
