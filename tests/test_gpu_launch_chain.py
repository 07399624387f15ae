"""GPU tests of the step's kernel chain: the accumulation records that the forward's blend clears for the fast blend
backward, and the kernels launched with programmatic dependent launch.

  * the first backward after a forward uses the records that forward cleared, and a second backward on the same
    forward (retain_graph=True) clears them itself: through `_C` and through autograd, both backward paths, the second
    result equal to the first (bit for bit under torch.use_deterministic_algorithms(True));
  * a forward that does not clear the records, followed by a backward that does, gives the same gradients.
"""
import os
import sys

import pytest
import torch

import _util

sys.path.insert(0, os.path.join(_util.ROOT, "oracle"))
import synth  # noqa: E402

pytestmark = pytest.mark.gpu

W, H = 320, 240


@pytest.fixture(params=[False, True], ids=["fast", "deterministic"])
def det(request):
    prev, warn = torch.are_deterministic_algorithms_enabled(), torch.is_deterministic_algorithms_warn_only_enabled()
    torch.use_deterministic_algorithms(request.param)
    yield request.param
    torch.use_deterministic_algorithms(prev, warn_only=warn)


def _inputs(mode="native"):
    dev = torch.device("cuda:0")
    scene = synth.make_strand_scene(300, seed=3)
    return synth.rasterizer_inputs(scene, synth.make_camera(5, W, H), mode=mode, device=dev), synth.upstream_gradient(W, H, 1).to(dev)


def _same(a, b, deterministic, what):
    if deterministic:
        assert torch.equal(a, b), what
    else:
        assert _util.rel_err(a, b) <= 1e-5, (what, _util.rel_err(a, b))


@pytest.mark.parametrize("mode", ["native", "render_hair"])
def test_second_backward_on_one_forward(det, mode):
    from gaussianhaircut_b200 import _C
    inp, dL = _inputs(mode)
    R, _color, radii, geom, binning, img = _C.rasterize_gaussians(*_util.native_args(inp))
    assert R > 0 and geom._gh_records_zeroed
    first = _C.rasterize_gaussians_backward(*_util.backward_args(inp, radii, dL, geom, R, binning, img))
    assert not geom._gh_records_zeroed
    second = _C.rasterize_gaussians_backward(*_util.backward_args(inp, radii, dL, geom, R, binning, img))
    # a forward that leaves the records alone, on a workspace that held garbage before: its backward clears them
    junk = torch.full((geom.untyped_storage().nbytes(),), 0xFF, dtype=torch.uint8, device=geom.device)
    del junk
    R2, _c2, radii2, geom2, binning2, img2 = _C.rasterize_gaussians(*_util.native_args(inp), zero_records=False)
    assert R2 == R and not getattr(geom2, "_gh_records_zeroed", False)
    cleared = _C.rasterize_gaussians_backward(*_util.backward_args(inp, radii2, dL, geom2, R2, binning2, img2))
    torch.cuda.synchronize()
    for name, a, b, c in zip(_util.GRAD_NAMES, first, second, cleared):
        if a.numel() == 0:
            continue
        assert a.abs().max() > 0 or name in ("dL_dsh", "dL_dcov3D", "dL_dmeans3D", "dL_dscales", "dL_drotations"), name
        _same(b, a, det, f"second backward: {name}")
        _same(c, a, det, f"backward after a forward that did not clear: {name}")


def test_retain_graph_gives_twice_the_gradient(det):
    import diff_gaussian_rasterization as dgr
    inp, dL = _inputs()
    kw, s = inp["kwargs"], inp["settings"]
    settings = dgr.GaussianRasterizationSettings(**{k: s[k] for k in dgr.GaussianRasterizationSettings._fields})
    names = [k for k in ("means3D", "colors_precomp", "opacities", "scales", "rotations") if kw[k] is not None]

    def leaves():
        return {k: (v.clone().requires_grad_(True) if k in names else v) for k, v in kw.items()}

    once = leaves()
    color, _radii = dgr.GaussianRasterizer(settings)(**once)
    (color * dL).sum().backward()
    twice = leaves()
    color, _radii = dgr.GaussianRasterizer(settings)(**twice)
    loss = (color * dL).sum()
    loss.backward(retain_graph=True)
    loss.backward()
    torch.cuda.synchronize()
    for k in names:
        g1, g2 = once[k].grad, twice[k].grad
        assert g1.abs().max() > 0, k
        _same(g2, 2 * g1, det, k)
