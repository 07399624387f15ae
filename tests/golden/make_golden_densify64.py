"""Regenerates densify64.npz: the reference's own `GaussianModel.densify_and_prune` (src/scene/gaussian_model.py:723-737)
run on the GPU (the reference allocates with device="cuda"), on the scenes of `scenes()` below.  Each scene stores its
inputs, the normal samples the reference drew (recorded from its torch.normal call) and every tensor it produced, so
tests/test_densify64_cpu.py can hold tests/_densify64.py to what the reference computes on the device.

The scenes put rows on the decision ties (exp(0) = 1 = percent_dense * extent, sigmoid(0) = 0.5 = min_opacity,
g = accum / denom = max_grad exactly), on denom = 0, on a NaN log-scale component and a NaN opacity logit, and give
quaternions of norm 1e-3 and 1e3, a negative real part and the zero quaternion.  `label` holds the source row index and
the moments hold row index + 0.25 / + 0.5, so the output layout can be read off any of them.

    python tests/golden/make_golden_densify64.py [out.npz]       (needs a GPU and the staged reference sources)
"""
import copy
import os
import sys
import types

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path[:0] = [os.path.join(ROOT, "tests"), os.path.join(ROOT, "oracle")]
from _densify64 import special_rows  # noqa: E402

TRAIN_ARGS = types.SimpleNamespace(percent_dense=0.01, position_lr_init=1.6e-4, position_lr_final=1.6e-6, position_lr_delay_mult=0.01,
                                   position_lr_max_steps=30000, feature_lr=2.5e-3, opacity_lr=0.05, label_lr=0.0025, scaling_lr=0.005,
                                   rotation_lr=0.001, train_orient_conf=True, orient_conf_lr=0.001)
OUT_NAMES = ("xyz", "scaling", "rotation", "opacity", "label")
MOMENT_NAMES = ("xyz", "scaling", "label")


def scenes():
    """{name: dict of inputs (float32 arrays) and parameters}."""
    out = {}
    for name, P, seed, kw in (("mixed", 400, 1, dict(max_grad=2e-4, min_opacity=0.005, extent=100.0, max_screen_size=20.0)),
                              ("no_screen", 200, 2, dict(max_grad=2e-4, min_opacity=0.005, extent=100.0, max_screen_size=None)),
                              ("tie_opacity", 200, 3, dict(max_grad=2e-4, min_opacity=0.5, extent=100.0, max_screen_size=20.0)),
                              ("max_grad_zero", 200, 4, dict(max_grad=0.0, min_opacity=0.005, extent=100.0, max_screen_size=20.0))):
        g = np.random.default_rng(seed)
        ls = g.normal(0.0, 1.2, (P, 3))
        op = g.normal(-1.0, 3.0, P)
        denom = g.integers(0, 4, P).astype(np.float64)
        accum = g.uniform(0, 6e-4, P) * np.maximum(denom, 1)
        rot = g.normal(0, 1, (P, 4))
        special = special_rows(kw["max_grad"] if kw["max_grad"] > 0 else 2e-4)
        idx = g.choice(P, len(special), replace=False)
        for k, (l, o, a, d, q) in zip(idx, special):
            ls[k], op[k], accum[k], denom[k], rot[k] = l, o, a, d, q
        if name == "tie_opacity":
            op[g.choice(P, 40, replace=False)] = 0.0
        out[name] = dict(xyz=g.normal(0, 1, (P, 3)).astype(np.float32), log_scaling=ls.astype(np.float32),
                         rotation=rot.astype(np.float32), opacity_logit=op.astype(np.float32),
                         accum=accum.astype(np.float32), denom=denom.astype(np.float32),
                         f_dc=g.normal(0, 1, (P, 1, 3)).astype(np.float32), orient_conf=g.normal(0, 1, (P, 1)).astype(np.float32),
                         percent_dense=TRAIN_ARGS.percent_dense, **kw)
    return out


def reference_outputs(sc, device):
    import ref_python
    from torch import nn
    ref_python.install_stubs()
    sys.path.insert(0, ref_python.ref_src_dir())
    from scene.gaussian_model import GaussianModel
    P = sc["xyz"].shape[0]
    pc = GaussianModel(0)
    prm = lambda a: nn.Parameter(torch.from_numpy(np.ascontiguousarray(a)).to(device).requires_grad_(True))  # noqa: E731
    pc._xyz, pc._scaling, pc._rotation = prm(sc["xyz"]), prm(sc["log_scaling"]), prm(sc["rotation"])
    pc._opacity = prm(sc["opacity_logit"][:, None])
    pc._features_dc, pc._features_rest = prm(sc["f_dc"]), prm(np.zeros((P, 0, 3), np.float32))
    pc._label = prm(np.arange(P, dtype=np.float32)[:, None])
    pc._orient_conf = prm(sc["orient_conf"])
    pc.spatial_lr_scale = 1.0
    pc.training_setup(copy.copy(TRAIN_ARGS))
    rid = torch.arange(P, dtype=torch.float32, device=device)
    for grp in pc.optimizer.param_groups:
        p = grp["params"][0]
        shape = (P,) + (1,) * (p.dim() - 1)
        pc.optimizer.state[p] = {"step": torch.tensor(3.0), "exp_avg": (rid.view(shape) + 0.25).expand_as(p).contiguous(),
                                 "exp_avg_sq": (rid.view(shape) + 0.5).expand_as(p).contiguous()}
    pc.xyz_gradient_accum = torch.from_numpy(sc["accum"][:, None]).to(device)
    pc.denom = torch.from_numpy(sc["denom"][:, None]).to(device)
    pc.max_radii2D = torch.zeros(P, device=device)
    drawn = []
    normal = torch.normal

    def recording_normal(*a, **k):
        s = normal(*a, **k)
        drawn.append(s.detach().cpu().numpy())
        return s
    torch.manual_seed(0)
    torch.normal = recording_normal
    try:
        pc.densify_and_prune(sc["max_grad"], sc["min_opacity"], sc["extent"], sc["max_screen_size"])
    finally:
        torch.normal = normal
    torch.cuda.synchronize()
    groups = {g["name"]: g["params"][0] for g in pc.optimizer.param_groups}
    out = {"samples": drawn[0] if drawn else np.zeros((0, 3), np.float32)}
    for n in OUT_NAMES:
        out[f"out_{n}"] = groups[n].detach().cpu().numpy().reshape(groups[n].shape[0], -1)
    for n in MOMENT_NAMES:
        st = pc.optimizer.state[groups[n]]
        out[f"out_{n}_exp_avg"] = st["exp_avg"].cpu().numpy().reshape(groups[n].shape[0], -1)
        out[f"out_{n}_exp_avg_sq"] = st["exp_avg_sq"].cpu().numpy().reshape(groups[n].shape[0], -1)
    return out


def main():
    path = sys.argv[1] if len(sys.argv) > 1 else os.path.join(HERE, "densify64.npz")
    dev = torch.device("cuda")
    out = {}
    for name, sc in scenes().items():
        for k in ("xyz", "log_scaling", "rotation", "opacity_logit", "accum", "denom"):
            out[f"{name}/{k}"] = sc[k]
        out[f"{name}/params"] = np.array([sc["max_grad"], sc["min_opacity"], sc["extent"],
                                          -1.0 if sc["max_screen_size"] is None else sc["max_screen_size"], sc["percent_dense"]])
        for k, v in reference_outputs(sc, dev).items():
            out[f"{name}/{k}"] = v
    np.savez_compressed(path, **out)
    print(path, len(out))


if __name__ == "__main__":
    main()
