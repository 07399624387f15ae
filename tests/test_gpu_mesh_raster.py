"""The mesh rasterizer on the H100 (csrc/gh_mesh_raster.cu, `gaussianhaircut_b200.mesh`): pix_to_face equal to the
host harness's brute force bit for bit and to the float64 oracle at every decided pixel (admissible elsewhere),
bit-reproducible across calls, chunk sizes and B, the status bits, the `[1:]` rule, and `scalp_visibility` at the
script's scale (the 9 936-face head, 128 views, 1024 x 1024) against the numpy restatement of the script and the
float64 path."""
import numpy as np
import pytest
import torch

import _meshraster64 as O
import _sdf_cases as K
from test_mesh_raster_cpu import brute, check_view, host  # noqa: F401  (the harness fixture)

pytestmark = pytest.mark.gpu


def _dev(*a, device):
    return [torch.from_numpy(np.ascontiguousarray(x)).to(device) for x in a]


CASES = {"head": (96, 128, 4), "head_holes": (96, 128, 4), "degenerate": (96, 128, 4), "big": (72, 96, 2)}


@pytest.mark.parametrize("name", list(CASES))
def test_pix_to_face_equals_the_harness_and_the_oracle(cuda_device, host, name):  # noqa: F811
    from gaussianhaircut_b200.mesh import rasterize_faces
    H, W, B = CASES[name]
    v, f = K.MESHES[name]()
    Ks, Rs, ts = O.sphere_cameras(B, H, W, 41, radius=0.35 if name != "degenerate" else 0.4)
    got = rasterize_faces(*_dev(v, f, Ks, Rs, ts, device=cuda_device), H, W).cpu().numpy()
    ref, st = brute(host, v, f, Ks, Rs, ts, H, W)
    assert st == 0 and np.array_equal(got, ref), name
    worst = np.zeros(3)
    for b in range(B):
        r = check_view(host, v, f, Ks[b], Rs[b], ts[b], H, W, p2f=got[b])
        worst = np.maximum(worst, [r[0], r[1], 1 - r[2]])
    print(f"{name}: pix_to_face = brute force bit for bit; largest margin ratio (error / bound): edge functions "
          f"{worst[0]:.3g}, depth {worst[1]:.3g}; undecided pixels at most {worst[2]:.2%}")


def test_bit_reproducible_across_calls_chunks_and_B(cuda_device):
    from gaussianhaircut_b200.mesh import rasterize_faces, scalp_visibility
    H, W, B = 160, 200, 11
    v, f = K.MESHES["head_holes"]()
    Ks, Rs, ts = O.sphere_cameras(B, H, W, 43)
    dv = _dev(v, f, Ks, Rs, ts, device=cuda_device)
    a = rasterize_faces(*dv, H, W)
    assert torch.equal(a, rasterize_faces(*dv, H, W))
    for lo, hi in ((0, 1), (3, 10), (10, 11)):
        sub = rasterize_faces(dv[0], dv[1], dv[2][lo:hi], dv[3][lo:hi], dv[4][lo:hi], H, W)
        assert torch.equal(sub, a[lo:hi]), (lo, hi)
    rng = np.random.default_rng(3)
    head = torch.from_numpy(rng.random((B, H, W)) < 0.6).to(cuda_device)
    outs = []
    for chunk in (1, 7, B):
        vis = torch.empty((B, H, W), dtype=torch.bool, device=cuda_device)
        outs.append([x.clone() for x in scalp_visibility(*dv, head, chunk=chunk, vis_out=vis)] + [vis])
    for o in outs[1:]:
        for x, y in zip(outs[0], o):
            assert torch.equal(x, y)
    assert torch.equal(outs[0][3], head & (a >= 0))
    m, vm, vmh = O.script_visibility(a.cpu().numpy(), head.cpu().numpy(), f, len(v))
    assert np.array_equal(outs[0][0].cpu().numpy(), m)
    assert np.array_equal(outs[0][1].cpu().numpy(), vm) and np.array_equal(outs[0][2].cpu().numpy(), vmh)


def test_status_bits_and_skipped_faces(cuda_device, host):  # noqa: F811
    from gaussianhaircut_b200.mesh import rasterize_faces
    H, W = 64, 80
    v, f = K.MESHES["icosphere"]()
    Ks, Rs, ts = O.sphere_cameras(2, H, W, 45)
    for bad in (len(v), -1, 2 ** 31 - 1):
        g = f.copy()
        g[17, 1] = bad
        with pytest.raises(RuntimeError, match="face index"):
            rasterize_faces(*_dev(v, g, Ks, Rs, ts, device=cuda_device), H, W)
    torch.cuda.synchronize()
    ok = rasterize_faces(*_dev(v, f, Ks, Rs, ts, device=cuda_device), H, W)
    assert (ok >= 0).any()                                       # the device is still sound
    # NaN vertices: their faces are skipped, the rest drawn as the harness draws them
    vn = v.copy()
    vn[[3, 50]] = np.nan
    got = rasterize_faces(*_dev(vn, f, Ks, Rs, ts, device=cuda_device), H, W).cpu().numpy()
    ref, st = brute(host, vn, f, Ks, Rs, ts, H, W)
    nan_faces = np.nonzero(np.isin(f, [3, 50]).any(1))[0]
    assert st == 0 and np.array_equal(got, ref) and not np.isin(got, nan_faces).any()
    # a face across the z = 0 plane of view 0: skipped, with a warning
    tri = np.array([[0, 0, -0.5], [0.02, 0, 0.5], [0, 0.02, 0.5]], np.float32)
    R0, t0 = Rs[0].astype(np.float64), ts[0].astype(np.float64)
    world = ((tri - t0) @ R0).astype(np.float32)                  # camera coordinates -> world
    v2 = np.concatenate([v, world])
    f2 = np.concatenate([f, [[len(v), len(v) + 1, len(v) + 2]]]).astype(np.int32)
    with pytest.warns(RuntimeWarning, match="z = 0"):
        got = rasterize_faces(*_dev(v2, f2, Ks, Rs, ts, device=cuda_device), H, W).cpu().numpy()
    ref, st = brute(host, v2, f2, Ks, Rs, ts, H, W)
    assert st == 8 and np.array_equal(got, ref) and not (got[0] == len(f)).any()     # in front of view 1: drawn there
    # an empty view: the camera looks away from the mesh
    Ra, ta = O.look_at([0, 0, 1.0], [0, 0, 2.0])
    empty = rasterize_faces(*_dev(v, f, Ks[:1], Ra[None].astype(np.float32), ta[None].astype(np.float32),
                                  device=cuda_device), H, W)
    assert (empty == -1).all()


def test_the_drop_the_smallest_rule_when_every_pixel_is_covered(cuda_device):
    """A view the mesh fills completely (no -1): `[1:]` drops the smallest face, in the plain and the head variant; a
    view with an empty head mask; a view with background."""
    from gaussianhaircut_b200.mesh import rasterize_faces, scalp_visibility
    H, W = 48, 64
    v, f = K.MESHES["icosphere"]()
    Ks, Rs, ts = O.sphere_cameras(3, H, W, 47)
    Ks[0, 0, 0] = Ks[0, 1, 1] = 20 * W                            # view 0: zoomed into the sphere, every pixel covered
    Ks[1, 0, 0] = Ks[1, 1, 1] = 20 * W
    dv = _dev(v, f, Ks, Rs, ts, device=cuda_device)
    p2f = rasterize_faces(*dv, H, W)
    assert (p2f[0] >= 0).all() and (p2f[1] >= 0).all() and (p2f[2] < 0).any()
    head = torch.ones((3, H, W), dtype=torch.bool, device=cuda_device)
    head[1] = False                                               # view 1: an empty head mask
    head[2, : H // 2] = False
    m, vm, vmh = (x.cpu().numpy() for x in scalp_visibility(*dv, head, chunk=2))
    rm, rvm, rvmh = O.script_visibility(p2f.cpu().numpy(), head.cpu().numpy(), f, len(v))
    assert np.array_equal(vm, rvm) and np.array_equal(vmh, rvmh) and np.array_equal(m, rm)


def test_scalp_visibility_at_the_scripts_scale(cuda_device):
    """The 9 936-face head, 128 views on a sphere of cameras, 1024 x 1024."""
    from gaussianhaircut_b200.mesh import rasterize_faces, scalp_visibility
    H = W = 1024
    B = 128
    v, f = K.head()
    Ks, Rs, ts = O.sphere_cameras(B, H, W, 49, radius=0.45, f_scale=1.6)
    rng = np.random.default_rng(5)
    rows = np.arange(H)[:, None]
    cut = rng.uniform(0.3, 0.7, B)
    head = torch.from_numpy(np.broadcast_to(rows[None] >= (cut * H)[:, None, None], (B, H, W)).copy()).to(cuda_device)
    dv = _dev(v, f, Ks, Rs, ts, device=cuda_device)
    vis_mask, vis_maps, vis_maps_head = (x.cpu().numpy() for x in scalp_visibility(*dv, head, chunk=16))
    p2f = rasterize_faces(*dv, H, W)
    m, vm, vmh = O.script_visibility(p2f.cpu().numpy(), head.cpu().numpy(), f, len(v))
    assert np.array_equal(vis_maps, vm) and np.array_equal(vis_maps_head, vmh) and np.array_equal(vis_mask, m)
    # the float64 path: per view, the faces every admissible outcome shows and those some outcome may show
    F, V = len(f), len(v)
    fi = torch.from_numpy(f).long().to(cuda_device)
    counts = {k: torch.zeros(V, dtype=torch.long, device=cuda_device) for k in ("plain_lo", "plain_hi", "head_lo", "head_hi")}
    undecided_pixels = 0
    for b in range(B):
        o = O.raster64(v, f, Ks[b], Rs[b], ts[b], H, W, device=cuda_device)
        assert O.admissible(o, p2f[b], F).all(), b
        dec = o["decided"]
        assert torch.equal(p2f[b][dec].long(), o["answer"][dec]), b
        undecided_pixels += int((~dec).sum())
        for name, (lo, hi, neg) in O.face_sets(o, head[b], F).items():
            assert neg, "every view shows background and non-head pixels"        # so `[1:]` drops -1
            for tag, sel in (("lo", lo), ("hi", hi)):
                vf = torch.zeros(V, dtype=torch.bool, device=cuda_device)
                vf[fi[sel].reshape(-1)] = True
                counts[f"{name}_{tag}"] += vf.long()

    # vis_mask is not monotone in the counts (prob_hair > 0.5 rises with vis_maps, vis_maps / B < 0.1 falls), so a
    # vertex is decided when every (vis_maps, vis_maps_head) pair between its smallest and largest counts gives one mask
    c_lo, c_hi, h_lo, h_hi = (counts[k] for k in ("plain_lo", "plain_hi", "head_lo", "head_hi"))
    span = int(max((c_hi - c_lo).max(), (h_hi - h_lo).max()))
    first = None
    same = torch.ones(V, dtype=torch.bool, device=cuda_device)
    for dc in range(span + 1):
        for dh in range(span + 1):
            c = torch.minimum(c_lo + dc, c_hi).float()
            ch = torch.minimum(h_lo + dh, h_hi).float()
            mk = torch.logical_or(1 - ch / c > 0.5, c / B < 0.1)
            first = mk if first is None else first
            same &= mk == first
    same, first = same.cpu().numpy(), first.cpu().numpy()
    assert np.array_equal(vis_mask[same], first[same])
    und = ((c_lo != c_hi) | (h_lo != h_hi)).cpu().numpy()
    exact = ~und
    assert np.array_equal(vis_maps[exact], c_lo.cpu().numpy()[exact])
    assert np.array_equal(vis_maps_head[exact], h_lo.cpu().numpy()[exact])
    print(f"script scale: {B} views at {H}x{W}, {undecided_pixels} undecided pixels in all; {int(und.sum())} of {V} "
          f"vertices have undecided counts, {int((~same).sum())} an undecided vis_mask; {int(vis_mask.sum())} in "
          f"vis_mask")
