"""Adaptive density control ("next" row 8f-3): gaussianhaircut_b200.densify against the reference's OWN
`GaussianModel.densify_and_prune` / `reset_opacity` (src/scene/gaussian_model.py:723-737, :516-519), imported unmodified
(oracle/ref_python.py) and run on the GPU with the same seed: every parameter tensor, both Adam moments of every group,
the statistics buffers and the resulting order of the Gaussians must agree -- with torch.optim.Adam (the reference's
optimizer) and with this repository's FusedAdam."""
import copy
import os
import sys
import types

import pytest
import torch

import _util
from _util import rel_err

pytestmark = pytest.mark.gpu

sys.path.insert(0, os.path.join(_util.ROOT, "oracle"))
import ref_python  # noqa: E402

TRAIN_ARGS = types.SimpleNamespace(percent_dense=0.01, position_lr_init=1.6e-4, position_lr_final=1.6e-6, position_lr_delay_mult=0.01,
                                   position_lr_max_steps=30000, feature_lr=2.5e-3, opacity_lr=0.05, label_lr=0.0025, scaling_lr=0.005,
                                   rotation_lr=0.001, train_orient_conf=True, orient_conf_lr=0.001)
NAMES = ("xyz", "f_dc", "f_rest", "opacity", "label", "scaling", "rotation", "orient_conf")


def _model(scene, device, train_orient_conf=True, fused=False, seed=0):
    """A reference GaussianModel with optimizer moments and densification statistics as after a stretch of training."""
    if not ref_python.available():
        pytest.skip("reference Python sources not staged")
    ref_python.install_stubs()
    src = ref_python.ref_src_dir()
    if src not in sys.path:
        sys.path.insert(0, src)
    pc = ref_python.make_gaussian_model(scene, device)
    pc.spatial_lr_scale = 1.0
    args = copy.copy(TRAIN_ARGS)
    args.train_orient_conf = train_orient_conf
    pc.training_setup(args)                                  # the reference's own optimizer construction (:423-448)
    if fused:
        from gaussianhaircut_b200.optim import FusedAdam
        pc.optimizer = FusedAdam([{"params": g["params"], "lr": g["lr"], "name": g["name"]} for g in pc.optimizer.param_groups], eps=1e-15)
    g = torch.Generator().manual_seed(seed)
    for it in range(3):                                      # populate exp_avg / exp_avg_sq
        for grp in pc.optimizer.param_groups:
            p = grp["params"][0]
            p.grad = (torch.randn(p.shape, generator=g) * 0.01).to(device)
        pc.optimizer.step()
    P = pc._xyz.shape[0]
    pc.xyz_gradient_accum = (torch.rand(P, 1, generator=g) * 6e-4).to(device)
    pc.denom = torch.randint(0, 3, (P, 1), generator=g).float().to(device)        # zeros included: 0/0 -> NaN -> 0
    pc.max_radii2D = (torch.rand(P, generator=g) * 40).to(device)
    return pc


def _scene(n, seed):
    synth = _util.synth
    sc = synth.make_blob_scene(n, seed=seed, spread=0.2, max_scale=0.02)
    g = torch.Generator().manual_seed(seed + 1)
    sc["scaling"] = sc["scaling"] * torch.exp(torch.randn(n, 1, generator=g))           # spread of sizes around the density threshold
    sc["opacity"] = torch.sigmoid(torch.randn(n, 1, generator=g) * 3 - 1)               # some below min_opacity
    return sc


def _compare(a, b):
    assert a._xyz.shape == b._xyz.shape, f"{tuple(a._xyz.shape)} vs {tuple(b._xyz.shape)}"
    ga = {g["name"]: g for g in a.optimizer.param_groups}
    gb = {g["name"]: g for g in b.optimizer.param_groups}
    for n in ga:
        pa, pb = ga[n]["params"][0], gb[n]["params"][0]
        assert pa.shape == pb.shape, n
        assert rel_err(pb.detach(), pa.detach()) <= 1e-6, f"{n}: {rel_err(pb.detach(), pa.detach())}"
        assert getattr(b, {"xyz": "_xyz", "f_dc": "_features_dc", "f_rest": "_features_rest", "opacity": "_opacity", "label": "_label",
                           "scaling": "_scaling", "rotation": "_rotation", "orient_conf": "_orient_conf"}[n]) is pb
        sa, sb = a.optimizer.state[pa], b.optimizer.state[pb]
        for k in ("exp_avg", "exp_avg_sq"):
            assert sa[k].shape == sb[k].shape == pa.shape
            assert rel_err(sb[k], sa[k]) <= 1e-6, f"{n}.{k}: {rel_err(sb[k], sa[k])}"
    for n in ("xyz_gradient_accum", "denom", "max_radii2D"):
        assert getattr(a, n).shape == getattr(b, n).shape and float(getattr(b, n).abs().sum()) == 0.0, n
    assert a._orient_conf.shape == b._orient_conf.shape and rel_err(b._orient_conf.detach(), a._orient_conf.detach()) <= 1e-6


@pytest.mark.parametrize("n,max_screen_size,train_conf,fused", [(20000, 20, True, False), (20000, None, True, False),
                                                                (20000, 20, False, False), (20000, 20, True, True),
                                                                (7, 20, True, False)])
def test_densify_and_prune_matches_the_reference(cuda_device, n, max_screen_size, train_conf, fused):
    from gaussianhaircut_b200 import densify
    scene = _scene(n, seed=3)
    extent = 2.0
    a = _model(scene, cuda_device, train_conf, fused=False, seed=7)
    b = _model(scene, cuda_device, train_conf, fused=fused, seed=7)
    torch.manual_seed(123); torch.cuda.manual_seed(123)
    a.densify_and_prune(2e-4, 0.005, extent, max_screen_size)                    # the reference's method, as shipped
    torch.manual_seed(123); torch.cuda.manual_seed(123)
    counts = densify.densify_and_prune(b, 2e-4, 0.005, extent, max_screen_size)
    torch.cuda.synchronize()
    assert counts["total"] == a._xyz.shape[0]
    if n >= 1000:
        assert counts["cloned"] > 0 and counts["children"] > 0 and counts["kept"] < n, counts     # every branch exercised
    _compare(a, b)
    # the models keep training identically afterwards (optimizer state re-keyed correctly)
    g = torch.Generator().manual_seed(99)
    for grp_a, grp_b in zip(a.optimizer.param_groups, b.optimizer.param_groups):
        gr = (torch.randn(grp_a["params"][0].shape, generator=g) * 0.01).to(cuda_device)
        grp_a["params"][0].grad = gr.clone(); grp_b["params"][0].grad = gr.clone()
    a.optimizer.step(); b.optimizer.step()
    torch.cuda.synchronize()
    for grp_a, grp_b in zip(a.optimizer.param_groups, b.optimizer.param_groups):
        assert rel_err(grp_b["params"][0].detach(), grp_a["params"][0].detach()) <= 1e-6, grp_a["name"]


def test_reserved_pools_are_used_and_change_nothing(cuda_device):
    """densify.reserve_pools: the rebuilt tensors live in the buffers allocated up front (no allocation inside the
    call), results identical to the un-reserved path."""
    from gaussianhaircut_b200 import densify
    scene = _scene(20000, seed=3)
    a = _model(scene, cuda_device, True, fused=True, seed=7)
    b = _model(scene, cuda_device, True, fused=True, seed=7)
    densify.reserve_pools(b, 400000)
    slots = {k: [t.data_ptr() for t in v] for k, v in b._gh_pools.items()}
    assert all(len(v) == 2 and v[0] != v[1] for v in slots.values()) and len(slots) == 3 * 8
    for rnd in range(3):                                   # source and destination alternate between the two slots
        for pc in (a, b):
            torch.manual_seed(5 + rnd); torch.cuda.manual_seed(5 + rnd)
            P = pc._xyz.shape[0]
            g = torch.Generator().manual_seed(rnd)
            pc.xyz_gradient_accum = (torch.rand(P, 1, generator=g) * 6e-4).to(cuda_device)
            pc.denom = torch.randint(1, 3, (P, 1), generator=g).float().to(cuda_device)
            densify.densify_and_prune(pc, 2e-4, 0.005, 2.0, 20)
        assert a._xyz.shape == b._xyz.shape
        for name in NAMES:
            pa = [g for g in a.optimizer.param_groups if g["name"] == name][0]["params"][0]
            pb = [g for g in b.optimizer.param_groups if g["name"] == name][0]["params"][0]
            assert torch.equal(pa.detach(), pb.detach()), name
            assert torch.equal(a.optimizer.state[pa]["exp_avg_sq"], b.optimizer.state[pb]["exp_avg_sq"]), name
            assert pb.data_ptr() in slots[name], name      # still inside the reserved buffers
            assert b.optimizer.state[pb]["exp_avg"].data_ptr() in slots[name + ".exp_avg"], name
    assert {k: [t.data_ptr() for t in v] for k, v in b._gh_pools.items()} == slots


def test_reset_opacity_matches_the_reference(cuda_device):
    from gaussianhaircut_b200 import densify
    scene = _scene(5000, seed=5)
    a = _model(scene, cuda_device, True, seed=2)
    b = _model(scene, cuda_device, True, seed=2)
    a.reset_opacity()
    densify.reset_opacity(b)
    assert rel_err(b._opacity.detach(), a._opacity.detach()) <= 1e-6
    pa = [g for g in a.optimizer.param_groups if g["name"] == "opacity"][0]["params"][0]
    pb = [g for g in b.optimizer.param_groups if g["name"] == "opacity"][0]["params"][0]
    assert pb is b._opacity and float(b.optimizer.state[pb]["exp_avg"].abs().sum()) == 0.0
    assert torch.equal(a.optimizer.state[pa]["exp_avg_sq"], b.optimizer.state[pb]["exp_avg_sq"])


def test_densify_at_config5_scale(cuda_device):
    """BASELINE config 5 scale (2M Gaussians): same outcome as the reference, and the time of both (informational)."""
    import time
    from gaussianhaircut_b200 import densify
    scene = _scene(2_000_000, seed=11)
    extent = 2.0
    a = _model(scene, cuda_device, True, seed=1)
    b = _model(scene, cuda_device, True, seed=1)
    torch.manual_seed(5); torch.cuda.manual_seed(5)
    torch.cuda.synchronize(); t0 = time.time()
    a.densify_and_prune(2e-4, 0.005, extent, 20)
    torch.cuda.synchronize(); t_ref = time.time() - t0
    torch.manual_seed(5); torch.cuda.manual_seed(5)
    torch.cuda.synchronize(); t0 = time.time()
    counts = densify.densify_and_prune(b, 2e-4, 0.005, extent, 20)
    torch.cuda.synchronize(); t_mine = time.time() - t0
    print(f"\\n[densify 2M] reference {t_ref * 1e3:.1f} ms, fused {t_mine * 1e3:.1f} ms, counts {counts}")
    _compare(a, b)
