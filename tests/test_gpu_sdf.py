"""The mesh signed distance on the H100 (csrc/gh_sdf.cu, gaussianhaircut_b200.mesh, pysdf): every point of every case
within the float64 oracle's derived bounds (tests/_sdf64.py), the sign equal to the oracle's wherever it is decided,
NaN in NaN out, an out-of-range face index refused without a fault, bit-reproducible results independent of the
batch, the drop-in bit for bit, and the FLAME-intersection filter equal to its float64 replay on every Gaussian whose
corners clear the bounds -- also at the script's scale (500 k Gaussians, 6 M corners, the 10 k-face head)."""
import math

import numpy as np
import pytest
import torch

import _sdf64 as O
import _sdf_cases as K

pytestmark = pytest.mark.gpu

U = 2.0 ** -24


def _mesh(name, device):
    from gaussianhaircut_b200.mesh import MeshSDF
    v, f = K.MESHES[name]()
    return v, f, MeshSDF(torch.from_numpy(v).to(device), torch.from_numpy(f).to(device))


def _check(name, p, sdf, d, w, o):
    """Every finite point within the bounds; the sign where it is decided.  -> (largest error / bound of d, of w)."""
    fin = np.isfinite(p).all(1)
    assert np.isnan(sdf[~fin]).all() and np.isnan(d[~fin]).all() and np.isnan(w[~fin]).all(), name
    sdf, d, w = (x[fin].astype(np.float64) for x in (sdf, d, w))
    lo, hi, d64, w64, ew = (o[k][fin] for k in ("lo", "hi", "d", "w", "ew"))
    ok = (d >= lo) & (d <= hi)
    assert ok.all(), f"{name}: d outside its bound at {np.nonzero(~ok)[0][:5]}: {d[~ok][:5]} vs [{lo[~ok][:5]}, {hi[~ok][:5]}]"
    ew_out = ew + U * np.abs(w64)                       # + the float32 rounding of the written w
    bad = np.abs(w - w64) > ew_out
    assert not bad.any(), f"{name}: w outside its bound: {w[bad][:5]} vs {w64[bad][:5]} +- {ew_out[bad][:5]}"
    assert np.array_equal(np.abs(sdf), d), name
    decided = (np.abs(w64 - 0.5) > ew) & (lo > 0)
    assert (np.sign(sdf[decided]) == np.sign(o["sdf"][fin][decided])).all(), name
    r_d = np.max(np.abs(d - d64) / np.maximum(np.maximum(hi - d64, d64 - lo), 1e-300))
    r_w = np.max(np.abs(w - w64) / ew_out)
    print(f"{name}: {fin.sum()} points, sign decided at {decided.sum()}, largest error / bound: d {r_d:.3g}, "
          f"w {r_w:.3g}")
    return r_d, r_w


@pytest.mark.parametrize("name", list(K.MESHES))
def test_within_the_derived_bounds(cuda_device, name):
    v, f, mesh = _mesh(name, cuda_device)
    p = K.queries(v, f, 300 if name == "big" else 1500, 11)
    sdf, d, w = (t.cpu().numpy() for t in mesh(torch.from_numpy(p).to(cuda_device), return_parts=True))
    _check(name, p, sdf, d, w, O.query64(p, v, f))


def test_closed_meshes_are_inside_out(cuda_device):
    """A point well inside a closed mesh is positive, well outside negative (the reference's reading of the sign)."""
    for name in ("icosphere", "head", "big"):
        _, _, mesh = _mesh(name, cuda_device)
        p = torch.tensor([[0.0, 0.0, 0.0], [0.005, -0.01, 0.02], [0.5, 0.0, 0.0], [0.0, -3.0, 1.0]], device=cuda_device)
        sdf, _, w = mesh(p, return_parts=True)
        assert (sdf[:2] > 0).all() and (sdf[2:] < 0).all(), name
        assert torch.allclose(w, torch.tensor([1.0, 1.0, 0.0, 0.0], device=cuda_device), atol=1e-3), name


def test_out_of_range_face_index_raises(cuda_device):
    from gaussianhaircut_b200.mesh import MeshSDF
    v, f = K.MESHES["icosphere"]()
    for bad in (len(v), -1, 2 ** 31 - 1):
        g = f.copy()
        g[17, 1] = bad
        with pytest.raises(RuntimeError, match="face index"):
            MeshSDF(torch.from_numpy(v).to(cuda_device), torch.from_numpy(g).to(cuda_device))
    torch.cuda.synchronize()
    _, _, mesh = _mesh("icosphere", cuda_device)                         # the device is still sound
    assert torch.isfinite(mesh(torch.zeros(4, 3, device=cuda_device))).all()


def test_bit_reproducible_and_independent_of_the_batch(cuda_device):
    v, f, mesh = _mesh("head_holes", cuda_device)
    p = torch.from_numpy(K.queries(v, f, 20_000, 12)).to(cuda_device)
    a = [t.clone() for t in mesh(p, return_parts=True)]
    b = mesh(p, return_parts=True)
    for x, y in zip(a, b):
        assert torch.equal(x.view(torch.int32), y.view(torch.int32))
    for i in (0, 1, 4097, p.shape[0] - 7, p.shape[0] - 1):
        alone = mesh(p[i:i + 1].clone(), return_parts=True)
        for x, y in zip(a, alone):
            assert torch.equal(x[i:i + 1].view(torch.int32), y.view(torch.int32)), i
    side = torch.cuda.Stream(cuda_device)
    side.wait_stream(torch.cuda.current_stream(cuda_device))
    with torch.cuda.stream(side):
        c = mesh(p)
    torch.cuda.current_stream(cuda_device).wait_stream(side)
    assert torch.equal(c.view(torch.int32), a[0].view(torch.int32))


def test_pysdf_drop_in_is_mesh_sdf_bit_for_bit(cuda_device):
    from pysdf import SDF
    v, f, mesh = _mesh("head", cuda_device)
    p = K.queries(v, f, 2000, 13)
    with torch.cuda.device(cuda_device):
        s = SDF(v.astype(np.float64).tolist(), f.astype(np.int64))
        got = s(p.astype(np.float64))
        one = s(p[5])
    ref = mesh(torch.from_numpy(p).to(cuda_device)).cpu().numpy()
    assert got.dtype == np.float32 and got.shape == (len(p),)
    assert np.array_equal(got.view(np.int32), ref.view(np.int32))
    assert np.ndim(one) == 0 and np.float32(one).view(np.int32) == ref[5].view(np.int32)


def _filter_case(cuda_device, P, seed, sample=None):
    from gaussianhaircut_b200 import mesh as M
    v, f, mesh = _mesh("head_holes", cuda_device)
    xyz, scaling, rotation, label = K.gaussians(v, f, P, seed)
    dev = lambda a: torch.from_numpy(a).to(cuda_device)  # noqa: E731
    keep = M.flame_filter_keep(dev(xyz), dev(scaling), dev(rotation), dev(label), mesh).cpu().numpy()
    assert keep.dtype == bool and keep.shape == (P,)
    idx = np.arange(P) if sample is None else np.sort(np.random.default_rng(seed).choice(P, sample, replace=False))
    corners = M.flame_corners(dev(xyz[idx]), dev(scaling[idx]), dev(rotation[idx]))
    o = O.flame_filter_keep64(xyz[idx], scaling[idx], rotation[idx], label[idx], v, f)
    # the corners of the sampled Gaussians, queried on their own, against the oracle at the float64 corners
    ec = np.repeat(O.corner_bound(xyz[idx], scaling[idx]), 12)
    c32 = corners.cpu().numpy().astype(np.float64)
    assert (np.linalg.norm(c32 - o["corners"].reshape(-1, 3), axis=1) <= ec).all()
    clear = o["clear"]
    bad = np.nonzero(clear & (keep[idx] != o["keep"]))[0]
    print(f"filter P={P}: {len(idx)} Gaussians checked ({12 * len(idx)} corners), {int((~clear).sum())} excluded by "
          f"the margin, {int(keep.sum())} of {P} kept")
    assert bad.size == 0, f"filter differs from the float64 replay at {idx[bad][:5]}"
    assert (~clear).mean() < 0.05


def test_flame_filter_matches_the_float64_replay(cuda_device):
    _filter_case(cuda_device, 4000, 21)


def test_flame_filter_at_the_scripts_scale(cuda_device):
    """500 k Gaussians, 6 M corners against the 10 k-face head; the oracle checks a seeded sample of 20 k corners."""
    _filter_case(cuda_device, 500_000, 22, sample=20_000 // 12)


def test_corners_at_scale_within_the_bound_of_the_sample(cuda_device):
    """The 6 M-corner query itself: a seeded 20 k sample of the corners against the oracle's bounds."""
    from gaussianhaircut_b200 import mesh as M
    v, f, mesh = _mesh("head", cuda_device)
    xyz, scaling, rotation, _ = K.gaussians(v, f, 500_000, 23)
    dev = lambda a: torch.from_numpy(a).to(cuda_device)  # noqa: E731
    corners = M.flame_corners(dev(xyz), dev(scaling), dev(rotation))
    sdf, d, w = mesh(corners, return_parts=True)
    idx = np.sort(np.random.default_rng(23).choice(corners.shape[0], 20_000, replace=False))
    p = corners.cpu().numpy()[idx]
    _check("head, 6 M corners (20 k sample)", p, *(t.cpu().numpy()[idx] for t in (sdf, d, w)), O.query64(p, v, f))
