"""GPU tests of how the per-Gaussian kernels move their rows, and of emit in the forward's first phase.

  * preprocess_backward stages the array-of-structs rows of a CTA as contiguous spans through shared memory.  For P at
    every tail of those spans (1, 31, 127, 128, 129, 4097, 500 003), with the input and output tensors placed at every
    4-byte offset inside a 16-byte line, the image, radii, sorted keys and every gradient are bit-identical
    (deterministic backward), and NaN-prefilled gradient buffers come back fully written, with zero geometry gradients
    for the Gaussians that were not rendered;
  * the same for the cov3D_precomp input (a staged span of 6 floats per row) and the conic_precomp call shapes, and the
    prefiltered error raised by the first phase with and without a binning buffer;
  * binning-capacity hints that are exact, too large and too small, a buffer of capacity 0 and the first call without a
    hint all give byte-identical images, radii, sorted keys and gradients.
"""
import ctypes as C

import numpy as np
import pytest
import torch

import _util
import synth

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda:0")
W, H = 1920, 1080
# floats per Gaussian of each gradient the backward writes (the 4-float rows stay 16-byte aligned: the ABI requires it)
GRAD_ROWS = {"means2D": 3, "conic": 4, "opacity": 1, "colors": 10, "means3D": 3, "cov3D": 6, "scales": 3, "rotations": 4}
_SCENES = {}


@pytest.fixture
def det():
    prev, warn = torch.are_deterministic_algorithms_enabled(), torch.is_deterministic_algorithms_warn_only_enabled()
    torch.use_deterministic_algorithms(True)
    yield
    torch.use_deterministic_algorithms(prev, warn_only=warn)


def _inputs(P: int, mode: str, cam_k: int = 0):
    """The first P Gaussians of the strand bench scene (5001 strands: 500 100 Gaussians) in one call shape."""
    if mode not in _SCENES:
        scene = synth.make_strand_scene(5001, seed=0)
        _SCENES[mode] = synth.rasterizer_inputs(scene, synth.make_camera(cam_k, W, H), mode=mode, device=DEV)
    inp = _SCENES[mode]
    kw = {k: (v[:P].contiguous() if isinstance(v, torch.Tensor) else v) for k, v in inp["kwargs"].items()}
    return kw, inp["settings"]


def _at_offset(t, shift: int, fill=0.0):
    """A contiguous copy of `t` whose data starts `shift` floats past a 16-byte boundary (NaN or `fill` around it)."""
    if t is None:
        return None
    buf = torch.full((t.numel() + 8,), fill, dtype=torch.float32, device=DEV)
    out = buf[shift:shift + t.numel()].view(t.shape)
    out.copy_(t)
    assert out.data_ptr() % 16 == 4 * shift
    return out


def _run(kw, s, shift: int, backward: bool = True):
    """Forward + backward with every 1/3/6/10-float per-Gaussian tensor `shift` floats off 16-byte alignment (the colour
    rows, which must stay 8-byte aligned, by 2 * (shift % 2)).  -> dict of numpy arrays."""
    from gaussianhaircut_b200 import _C
    e = torch.Tensor([])
    P = kw["means3D"].shape[0]
    g = lambda k, sh=shift: e if kw[k] is None else _at_offset(kw[k], sh)  # noqa: E731
    means3D = g("means3D")
    colors = _at_offset(kw["colors_precomp"], 2 * (shift % 2))
    rotations = e if kw["rotations"] is None else kw["rotations"]
    R, color, radii, geom, binning, img = _C.rasterize_gaussians(
        s["bg"], means3D, kw["means2D"], colors, g("opacities"), g("scales"), rotations, 1.0, g("cov3D_precomp"),
        g("conic_precomp"), s["viewmatrix"], s["projmatrix"], s["tanfovx"], s["tanfovy"], H, W, e, 3, s["campos"],
        s["prefiltered"], False)
    out = {"color": color, "radii": radii, "keys": _C.debug_export(P, W, H, R, geom, binning, img)["keys"]}
    if backward and kw["conic_precomp"] is None:
        nan = float("nan")
        grads = {}
        for name, n in GRAD_ROWS.items():
            sh = 0 if n == 4 else (2 * (shift % 2) if name == "colors" else shift)
            grads[name] = _at_offset(torch.full((P, n), nan, device=DEV), sh, fill=nan)
        if kw["scales"] is None:
            grads["scales"] = grads["rotations"] = None
        _C._backward(s["bg"], means3D, radii, colors, g("scales"), rotations, 1.0, g("cov3D_precomp"), e,
                     s["viewmatrix"], s["projmatrix"], s["tanfovx"], s["tanfovy"], synth.upstream_gradient(W, H, 0).to(DEV),
                     None, 3, s["campos"], geom, R, binning, img, False, grads=grads)
        out.update({f"d_{k}": v for k, v in grads.items() if v is not None})
    torch.cuda.synchronize()
    return {k: v.detach().cpu().numpy() for k, v in out.items()}


def _same(a: dict, b: dict, what: str):
    assert a.keys() == b.keys()
    for k in a:
        assert a[k].shape == b[k].shape and a[k].tobytes() == b[k].tobytes(), f"{what}: {k} differs"


@pytest.mark.parametrize("P", [1, 31, 127, 128, 129, 4097, 500003])
def test_rows_do_not_depend_on_span_alignment(det, P):
    kw, s = _inputs(P, "native")
    ref = _run(kw, s, 0)
    for k, v in ref.items():
        if k.startswith("d_"):
            assert np.isfinite(v).all(), f"{k}: rows left unwritten (NaN prefill survived)"
    culled = ref["radii"] == 0
    for k in ("d_means3D", "d_cov3D", "d_scales", "d_rotations"):
        assert not ref[k][culled].any(), f"{k}: culled Gaussians must get zero geometry gradients"
    assert (ref["d_means2D"][:, 2] == 0).all() and (ref["d_conic"][:, 2] == 0).all()
    if P >= 4097:
        assert (~culled).sum() > 0 and ref["keys"].size > 0
    for shift in (1, 2, 3):
        _same(ref, _run(kw, s, shift), f"P={P} shift={shift}")


@pytest.mark.parametrize("P", [129, 4097])
def test_cov3d_precomp_rows(det, P):
    kw, s = _inputs(P, "cov3d")
    ref = _run(kw, s, 0)
    assert all(np.isfinite(v).all() for k, v in ref.items() if k.startswith("d_"))
    for shift in (1, 3):
        _same(ref, _run(kw, s, shift), f"cov3d P={P} shift={shift}")


@pytest.mark.parametrize("mode", ["render", "render_hair"])
def test_conic_precomp_rows(mode):
    kw, s = _inputs(4097, mode)
    ref = _run(kw, s, 0, backward=False)
    assert (ref["radii"] > 0).any()
    for shift in (1, 2, 3):
        _same(ref, _run(kw, s, shift, backward=False), f"{mode} shift={shift}")


def test_prefiltered_error_with_and_without_a_capacity_hint():
    from gaussianhaircut_b200 import _C, _capi
    kw, s = _inputs(4097, "render")
    bad = dict(kw)
    bad["means3D"] = kw["means3D"].clone()
    bad["means3D"][100] = 3.0 * s["campos"]          # the ring cameras look at the origin: this point is behind the camera
    key = (DEV.index, 4097, W, H)
    for hint in (None, 10 ** 6):
        _C._BIN_R.pop(key, None)
        if hint is not None:
            _C.binning_record(key, hint)
        with pytest.raises(_capi.GhError) as ei:
            _run(bad, s, 0, backward=False)
        assert ei.value.code == _capi.GH_E_PREFILTERED and "prefiltered" in str(ei.value)
    _run(kw, s, 0, backward=False)                                            # the next call is unaffected
    _C._BIN_R.pop(key, None)


def _forward_with_capacity(kw, s, capacity):
    """rasterize_gaussians + its backward with an explicit binning buffer of `capacity` records (None: no buffer)."""
    from gaussianhaircut_b200 import _C, _capi
    from gaussianhaircut_b200._capi import _ptr, _stream
    lib = _capi.load()
    e = torch.Tensor([])
    P = kw["means3D"].shape[0]
    geom, img, radii = _C.alloc_forward_workspaces(P, W, H, DEV)
    buf = None
    if capacity is not None:
        nb = C.c_size_t()
        _capi.check(lib.gh_binning_workspace_size(capacity, C.byref(nb)))
        buf = torch.full((nb.value,), 0xAB, dtype=torch.uint8, device=DEV)
    n, m, emitted = C.c_int(), C.c_int(), C.c_int(-1)
    _capi.check(lib.gh_forward_preprocess(
        P, 3, 0, W, H, _ptr(kw["means3D"]), None, None, _ptr(kw["colors_precomp"]), _ptr(kw["opacities"]),
        _ptr(kw["scales"]), 1.0, _ptr(kw["rotations"]), None, None, _ptr(s["viewmatrix"]), _ptr(s["projmatrix"]),
        _ptr(s["campos"]), s["tanfovx"], s["tanfovy"], 0, _ptr(radii), _ptr(geom), _ptr(img), _ptr(buf),
        capacity or 0, C.byref(n), C.byref(m), C.byref(emitted) if buf is not None else None, 0, _stream(DEV)))
    R = n.value
    color = torch.empty((10, H, W), dtype=torch.float32, device=DEV)
    binning = _C._render(s["bg"], kw["colors_precomp"], radii, geom, img, R, m.value, color, False,
                         buf if emitted.value == 1 else None)
    keys = _C.debug_export(P, W, H, R, geom, binning, img)["keys"]
    flat, _g, _ = _C.rasterize_gaussians_backward_arena(
        s["bg"], kw["means3D"], radii, kw["colors_precomp"], kw["scales"], kw["rotations"], 1.0, e, e, s["viewmatrix"],
        s["projmatrix"], s["tanfovx"], s["tanfovy"], synth.upstream_gradient(W, H, 0).to(DEV), e, 3, s["campos"], geom,
        R, binning, img, False)
    torch.cuda.synchronize()
    out = {"color": color, "radii": radii, "keys": keys, "grads": flat}
    return R, emitted.value, {k: v.cpu().numpy() for k, v in out.items()}


def test_binning_capacity_hints(det):
    from gaussianhaircut_b200 import _C
    kw, s = _inputs(500003, "native")
    R, _, ref = _forward_with_capacity(kw, s, None)
    assert R > 100000
    for capacity, expect in ((R, 1), (R + 100000, 1), (R - 1, 0), (0, 0)):
        R2, emitted, got = _forward_with_capacity(kw, s, capacity)
        assert R2 == R and emitted == expect, (capacity, emitted)
        _same(ref, got, f"capacity {capacity}")
    # the public path: the first call has no hint, the next ones size the buffer from it
    key = (DEV.index, 500003, W, H)
    _C._BIN_R.pop(key, None)
    pub = [_run(kw, s, 0) for _ in range(2)]
    assert _C.binning_capacity(key) >= R
    _same(pub[0], pub[1], "cache miss vs hint")
    assert pub[0]["color"].tobytes() == ref["color"].tobytes() and pub[0]["keys"].tobytes() == ref["keys"].tobytes()
    _C._BIN_R.pop(key, None)
