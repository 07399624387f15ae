"""GPU tests: the blend kernels per pixel and per Gaussian against the float64 replay (oracle/blend64.py), and the tile
sort per tile, on scenes built in screen space to reach the boundaries the kernels branch on:

  * image borders that cut pixel pairs (forward) and 2x2 blocks (backward);
  * the {alpha >= 1/255} band, where the forward's pair lists and the backward's block masks (both from the
    conservative span test, gh_span_level) must keep every pair that blends;
  * the 384-record staging windows of both kernels;
  * the test_T stop inside a pixel pair and a 2x2 block;
  * the in-CTA tile sort at its 1792-record limit, and equal depth keys in the in-CTA and the in-place sorts.

Each scene checks:
  * every tile's records are ordered by (depth bits, Gaussian index), and the keys equal Oracle-B's binning;
  * every reached blend decision is farther from its threshold than float32 can move it (the replay's margins),
    so that n_contrib has one right answer -- and it equals the replay's;
  * the image and final_T element by element, and every Gaussian's dL/d(mean2D, colour, opacity, conic)
    component by component: |x - x64| <= TOL (scale + FLOOR), scale = the replay's sum of term magnitudes.
Each scene also asserts what it exists to reach, so that an edit cannot quietly make it pointless.

TOL was calibrated by running the reference's own CUDA build through the same checks on the same scenes
(tools/blend_replay_calibrate.py): its worst ratio is recorded next to TOL, and TOL leaves it a factor 16.
"""
import os
import sys

import numpy as np
import pytest
import torch

import _util

sys.path.insert(0, os.path.join(_util.ROOT, "oracle"))
import blend64  # noqa: E402
import oracle  # noqa: E402

pytestmark = pytest.mark.gpu

# Worst ratio on these scenes, H100 80GB HBM3 at a 400 W power limit: the reference's CUDA build 1.25e-5
# (window-769-stop385), this repository's kernels 6.1e-5 (equal-depths-3000; the backward rebuilds T with
# rcp.approx over 3000 records).  tools/blend_replay_calibrate.py prints both.
TOL = 2e-4
FLOOR = 1e-30       # a component the replay leaves at zero must be exactly zero
SORT_MAX = 1792     # GH_INKERNEL_SORT_MAX: the longest bucket the forward CTA sorts itself


# ------------------------------------------------------------------------------------------------- scenes
def conics(sig_major, sig_minor, theta):
    """(P,3) conic (a, b, c) of the screen-space covariance R diag(s1^2, s2^2) R^T."""
    c, s = np.cos(theta), np.sin(theta)
    v1, v2 = sig_major ** 2, sig_minor ** 2
    cxx, cyy, cxy = c * c * v1 + s * s * v2, s * s * v1 + c * c * v2, c * s * (v1 - v2)
    det = cxx * cyy - cxy * cxy
    return np.stack([cyy / det, -cxy / det, cxx / det], axis=1)


def screen_scene(W, H, px, py, z, conic, op, seed=0):
    """Rasterizer inputs (the render() call shape: caller conics) for Gaussians placed at pixel (px, py) with view depth
    z, seen by camera 0 (x_cam = -x_w, y_cam = y_w, z_cam = 0.8 - z_w; focal length 1.2 H in both axes)."""
    P = len(px)
    px, py, z = (np.asarray(v, np.float64) for v in (px, py, z))
    f = 1.2 * H
    xyz = np.stack([-z * (2 * px + 1 - W) / (2 * f), z * (2 * py + 1 - H) / (2 * f), 0.8 - z], axis=1)
    g = torch.Generator().manual_seed(seed)
    cam = _util.synth.make_camera(0, W, H)
    kw = {"means3D": torch.from_numpy(xyz).float(), "means2D": torch.zeros(P, 3),
          "opacities": torch.from_numpy(np.asarray(op, np.float32).reshape(P, 1)), "shs": None,
          "colors_precomp": torch.rand(P, 10, generator=g), "scales": None, "rotations": None,
          "cov3D_precomp": torch.zeros(P, 6), "conic_precomp": torch.from_numpy(np.asarray(conic, np.float32))}
    settings = {"image_height": H, "image_width": W, "tanfovx": cam["tanfovx"], "tanfovy": cam["tanfovy"],
                "bg": torch.tensor(_util.synth.BG_DEFAULT, dtype=torch.float32), "scale_modifier": 1.0,
                "viewmatrix": cam["world_view_transform"], "projmatrix": cam["full_proj_transform"], "sh_degree": 3,
                "campos": cam["camera_center"], "prefiltered": False, "debug": False}
    return {"kwargs": kw, "settings": settings}


def distinct_depths(P, rng):
    """Distinct view depths in a random order: the tile sort has work to do."""
    return 0.5 + 1e-4 * rng.permutation(P)


def border_scene(W, H):
    """W, H = 1 (mod 16) and odd: the last tile row / column holds one pixel row / column, cutting pixel pairs and
    2x2 blocks; Gaussians of every size on and across the border."""
    rng = np.random.default_rng(W * 100 + H)
    P = 160
    px, py = rng.uniform(-6, W + 6, P), rng.uniform(-6, H + 6, P)
    px[:20], py[20:40] = W - 1 + rng.uniform(-0.5, 0.5, 20), H - 1 + rng.uniform(-0.5, 0.5, 20)
    con = conics(rng.uniform(0.7, 8, P), rng.uniform(0.6, 2.5, P), rng.uniform(0, np.pi, P))
    return screen_scene(W, H, px, py, distinct_depths(P, rng), con, rng.uniform(0.05, 1.0, P), seed=1)


NON_PD = (0.05, 0.3, 0.05)      # det < 0: no span bound, the pd == 0 all-pixels path


def band_scene():
    """Elongated, rotated Gaussians whose {alpha >= 1/255} ellipse only just reaches into the image: the mean
    sits inside a tile, on a tile edge, or tens to hundreds of pixels outside, and the ellipse overlaps a target
    pixel by a fraction of a pixel to a few pixels -- most of their pairs have alpha a little above 1/255.
    Opacities from just above 1/255 to 1, and one non-positive-definite conic."""
    W, H = 64, 48
    rng = np.random.default_rng(7)
    P = 420
    op = np.exp(rng.uniform(np.log(1.02 / 255), np.log(0.3), P))
    s1 = np.exp(rng.uniform(np.log(4), np.log(160), P))
    s2 = s1 / np.exp(rng.uniform(np.log(1.5), np.log(12), P))
    th = rng.uniform(0, np.pi, P)
    con = conics(s1, s2, th)
    q0 = 2 * np.log(255 * op)                                  # alpha = 1/255 on q = q0
    ang = rng.uniform(0, 2 * np.pi, P)
    n = np.stack([np.cos(ang), np.sin(ang)], axis=1)
    c, s = np.cos(th), np.sin(th)
    nsig = (n[:, 0] * c + n[:, 1] * s) ** 2 * s1 ** 2 + (-n[:, 0] * s + n[:, 1] * c) ** 2 * s2 ** 2
    reach = np.sqrt(q0 * nsig)                                  # support of the ellipse along n
    target = np.stack([rng.uniform(0, W - 1, P), rng.uniform(0, H - 1, P)], axis=1)
    mean = target - n * (reach - rng.uniform(0.2, 5.0, P))[:, None]
    # a quarter centred inside a tile or on a tile edge, with opacities up to 1 (pairs near 1/255 on their rim)
    k = P // 4
    mean[:k] = np.stack([rng.uniform(4, W - 4, k), rng.uniform(4, H - 4, k)], axis=1)
    mean[:k // 2, 0] = 16.0 * rng.integers(1, 4, k // 2) + rng.choice([-0.5, 0.0, 0.5], k // 2)
    op[:k] = np.exp(rng.uniform(np.log(1.005 / 255), 0.0, k))
    s1[:k] = rng.uniform(1.0, 12.0, k)
    con[:k] = conics(s1[:k], s1[:k] / rng.uniform(1.0, 6.0, k), th[:k])
    con[k] = NON_PD
    mean[k] = (W / 2 - 0.3, H / 2 + 0.2)
    op[k] = 0.5
    return screen_scene(W, H, mean[:, 0], mean[:, 1], distinct_depths(P, rng), con, op, seed=2)


FOG_OP = 0.006          # alpha ~ 0.006 on every pixel of the tile: 769 records leave T ~ 0.01, no pixel stops


def window_scene(n, stop_at=None):
    """One 16 x 16 image: n wide, faint Gaussians that every pixel blends ("fog"), depth-ordered as listed.  With
    stop_at = k, the records at list positions k - 1 and k (1-based) are two opaque Gaussians near the top-left
    corner: the pixels under their centre stop on record k.  The records after k are fog around the opposite
    corner that does not reach the opaque ones, so no pixel comes close to the stop threshold later."""
    rng = np.random.default_rng(n + (stop_at or 0))
    px, py = 8.0 + rng.uniform(-1, 1, n), 8.0 + rng.uniform(-1, 1, n)
    con = conics(np.full(n, 200.0), np.full(n, 150.0), rng.uniform(0, np.pi, n))
    op = np.full(n, FOG_OP)
    if stop_at is not None:
        for j in (stop_at - 2, stop_at - 1):
            px[j], py[j], op[j] = 2.3, 2.6, 1.0
            con[j] = conics(np.array([3.0]), np.array([2.5]), np.array([0.4]))[0]
        px[stop_at:], py[stop_at:] = 13.5, 13.5
        con[stop_at:] = (1 / 144.0, 0.0, 1 / 144.0)            # alpha >= 1/255 within 11 px of (13.5, 13.5)
    perm = rng.permutation(n)                                   # Gaussian i is the record at list position perm[i]
    return screen_scene(16, 16, px[perm], py[perm], 0.5 + 1e-4 * perm, con[perm], op[perm], seed=3)


def stop_scene():
    """Stacks of opacity-1 Gaussians (alpha capped at 0.99 near their centres) over a faint layer: the test_T stop
    cuts through pixel pairs and 2x2 blocks."""
    W, H = 32, 32
    rng = np.random.default_rng(11)
    px, py, op, s1, s2 = [], [], [], [], []
    for cx, cy in rng.uniform(3, 29, (10, 2)):
        k = int(rng.integers(3, 7))
        px += list(cx + rng.uniform(-1.5, 1.5, k)); py += list(cy + rng.uniform(-1.5, 1.5, k))
        op += [1.0] * k; s1 += list(rng.uniform(1.5, 5.0, k)); s2 += list(rng.uniform(1.0, 3.0, k))
    m = 60
    px += list(rng.uniform(0, W, m)); py += list(rng.uniform(0, H, m))
    op += list(rng.uniform(0.2, 0.6, m)); s1 += list(rng.uniform(6, 14, m)); s2 += list(rng.uniform(4, 8, m))
    P = len(px)
    con = conics(np.array(s1), np.array(s2), rng.uniform(0, np.pi, P))
    return screen_scene(W, H, px, py, distinct_depths(P, rng), con, op, seed=4)


TINY = (2.0, 0.0, 2.0)          # radius 3: a splat at a tile centre touches that tile only


def two_tile_scene(n_first, n_second):
    """n_first tiny splats in the middle of tile 0 and n_second in the middle of tile 1 of a 32 x 16 image, distinct
    depths descending with the index: bucket 1 starts at record n_first and holds n_second records."""
    P = n_first + n_second
    px = np.concatenate([np.full(n_first, 8.0), np.full(n_second, 24.0)])
    z = 0.5 + 1e-4 * np.arange(P)[::-1]
    return screen_scene(32, 16, px, np.full(P, 8.0), z, np.tile(TINY, (P, 1)), np.full(P, 0.02), seed=5)


def equal_depth_scene(n):
    """n tiny splats in one 16 x 16 tile, all at the same view depth: identical depth bits, ties ordered by index."""
    return screen_scene(16, 16, np.full(n, 8.0), np.full(n, 8.0), np.full(n, 0.5), np.tile(TINY, (n, 1)),
                        np.full(n, 0.02), seed=6)


# ------------------------------------------------------------------------------------------------- checks
def run(mod, inp, device, dL):
    """Forward + backward through `mod` (this repository's _C, or the reference's for calibration)."""
    s = inp["settings"]
    W, H = s["image_width"], s["image_height"]
    P = inp["kwargs"]["means3D"].shape[0]
    r = mod.rasterize_gaussians(*_util.native_args(inp))
    torch.cuda.synchronize()
    if hasattr(mod, "debug_export"):
        st = {k: v.cpu().numpy() for k, v in mod.debug_export(P, W, H, r[0], r[3], r[4], r[5]).items()}
    else:
        st = _util.parse_ref_buffers(P, W, H, r[0], r[3], r[4], r[5])
    g = mod.rasterize_gaussians_backward(*_util.backward_args(inp, r[2], dL, r[3], r[0], r[4], r[5]))
    torch.cuda.synchronize()
    return {"R": int(r[0]), "image": r[1], "radii": r[2].cpu().numpy(), "state": st, "grads": dict(zip(_util.GRAD_NAMES, g))}


def on(inp, device):
    return {"kwargs": {k: (v.to(device) if isinstance(v, torch.Tensor) else v) for k, v in inp["kwargs"].items()},
            "settings": {k: (v.to(device) if isinstance(v, torch.Tensor) else v) for k, v in inp["settings"].items()}}


def check(mod, inp, device, dL_seed=0):
    """Every check of the module docstring; returns (worst ratio per output, the replay, the run)."""
    s, kw = inp["settings"], inp["kwargs"]
    W, H = s["image_width"], s["image_height"]
    dL = _util.synth.upstream_gradient(W, H, dL_seed).to(device)
    o = run(mod, on(inp, device), device, dL)
    st = o["state"]
    ranges = st["ranges"].view(np.uint32).reshape(-1, 2).astype(np.int64)
    keys = st["keys"].view(np.uint64)
    plist = st["point_list"].view(np.uint32).astype(np.int64)
    # binning: the key multiset is Oracle-B's, and every tile is ordered by (depth bits, Gaussian index)
    npy = lambda t: None if t is None else t.numpy()   # noqa: E731
    fw = oracle.forward(npy(kw["means3D"]), npy(kw["opacities"]), npy(kw["colors_precomp"]), npy(s["viewmatrix"]),
                        npy(s["projmatrix"]), s["tanfovx"], s["tanfovy"], W, H, npy(s["bg"]),
                        cov3D_precomp=npy(kw["cov3D_precomp"]), conic_precomp=npy(kw["conic_precomp"]))
    assert o["R"] == fw["num_rendered"] == keys.size
    assert np.array_equal(np.sort(keys), fw["keys"]), "tile keys differ from Oracle-B's binning"
    assert np.array_equal(ranges, fw["ranges"].astype(np.int64))
    depth = (keys & np.uint64(0xFFFFFFFF)).astype(np.int64)
    for t in np.nonzero(ranges[:, 1] > ranges[:, 0])[0]:
        a, b = ranges[t]
        order = np.lexsort((plist[a:b], depth[a:b]))
        assert np.array_equal(order, np.arange(b - a)), f"tile {t}: records not ordered by (depth, index)"
        assert np.all((keys[a:b] >> np.uint64(32)) == t)
    # the blend against the replay
    rp = blend64.replay(st["means2D"], st["conic_opacity"], kw["colors_precomp"], s["bg"], plist, ranges, W, H, dL,
                        device=device)
    for k in ("alpha_ratio", "power_ratio", "stop_ratio"):
        assert rp[k] >= blend64.DECISION_SAFETY, f"scene has a decision within float32 error of its threshold: {k} {rp[k]}"
    nc = torch.from_numpy(st["n_contrib"].view(np.uint32).astype(np.int64)).to(device)
    assert torch.equal(nc, rp["n_contrib"]), f"n_contrib differs at {int((nc != rp['n_contrib']).sum())} pixels"
    worst = {"image": blend64.worst_ratio(o["image"], rp["image"], rp["image_scale"], FLOOR),
             "final_T": blend64.worst_ratio(torch.from_numpy(st["final_T"]), rp["final_T"], rp["final_T"], FLOOR)}
    for n in blend64.GRADS:
        worst[n] = blend64.worst_ratio(o["grads"][n], rp[n], rp["scale"][n], FLOOR)
    return worst, rp, o


def assert_within(worst):
    bad = {k: v for k, v in worst.items() if not v <= TOL}
    assert not bad, f"beyond {TOL} of the replay's scale: {bad}"


def _mine():
    import gaussianhaircut_b200._C as mine
    return mine


def n_blended(rp):
    return int(rp["n_contrib"].max())


# ------------------------------------------------------------------------------------------------- tests
@pytest.mark.parametrize("W,H", [(33, 17), (47, 31)])
def test_image_border(cuda_device, W, H):
    worst, rp, o = check(_mine(), border_scene(W, H), cuda_device)
    nc = rp["n_contrib"].reshape(H, W)
    assert bool((nc[-1] > 0).any()) and bool((nc[:, -1] > 0).any()), "nothing blends on the cut border row / column"
    assert_within(worst)


BAND_PAIRS = 1000       # reached (pixel, Gaussian) pairs with alpha in (1 + 1e-4, 1 + 1e-2) x 1/255


def test_alpha_band(cuda_device):
    inp = band_scene()
    worst, rp, o = check(_mine(), inp, cuda_device)
    rel = rp["alpha_rel"]
    near = int(((rel > 1e-4) & (rel < 1e-2)).sum())
    assert near >= BAND_PAIRS, f"only {near} pairs with alpha just above 1/255"
    con = inp["kwargs"]["conic_precomp"].double().numpy()
    non_pd = (con[:, 0] * con[:, 2] - con[:, 1] ** 2) <= 0
    assert int(non_pd.sum()) == 1 and int(o["radii"][non_pd][0]) > 0, "the non-positive-definite conic is not rendered"
    assert_within(worst)


WINDOW_CASES = [(383, None), (384, None), (385, None), (767, None), (768, None), (769, None), (769, 384), (769, 385)]


@pytest.mark.parametrize("n,stop_at", WINDOW_CASES, ids=[f"{n}" + (f"-stop{s}" if s else "") for n, s in WINDOW_CASES])
def test_window_boundaries(cuda_device, n, stop_at):
    worst, rp, o = check(_mine(), window_scene(n, stop_at), cuda_device)
    nc, stopped = rp["n_contrib"], rp["stopped"]
    if stop_at is None:
        assert not bool(stopped.any()) and bool((nc == n).all()), "every pixel must blend every record"
    else:
        assert bool((stopped & (nc == stop_at - 1)).any()), f"no pixel stops on record {stop_at}"
        assert bool((~stopped & (nc == n)).any())
    assert_within(worst)


def test_early_stop_in_pairs_and_blocks(cuda_device):
    worst, rp, o = check(_mine(), stop_scene(), cuda_device)
    s = rp["stopped"].reshape(32, 32).cpu().numpy()
    pair_mixed = s[0::2] != s[1::2]                                        # forward: vertical pixel pairs
    block = s.reshape(16, 2, 16, 2).transpose(0, 2, 1, 3).reshape(16, 16, 4)
    block_mixed = block.any(axis=2) & ~block.all(axis=2)                  # backward: 2x2 blocks
    assert int(pair_mixed.sum()) >= 10 and int(block_mixed.sum()) >= 10 and int((~s).sum()) >= 100
    assert_within(worst)


SORT_CASES = [(1, 1791), (2, 1791), (1, 1792), (2, 1792), (1, 1793), (2, 1793)]


@pytest.mark.parametrize("n_first,n_second", SORT_CASES)
def test_in_cta_sort_limit(cuda_device, n_first, n_second):
    """Buckets of 1791..1793 records starting at odd and even record indices: the in-CTA sort with the widened TMA
    copy, its load-loop fallback (1792 records from an odd index do not fit after widening), and the long-list
    kernels at 1793."""
    worst, rp, o = check(_mine(), two_tile_scene(n_first, n_second), cuda_device)
    rg = o["state"]["ranges"].view(np.uint32).reshape(-1, 2)
    assert int(rg[0, 1] - rg[0, 0]) == n_first and int(rg[1, 0]) == n_first and int(rg[1, 1] - rg[1, 0]) == n_second
    assert_within(worst)


@pytest.mark.parametrize("n", [1000, 3000])
def test_equal_depths(cuda_device, n):
    """1000 equal keys: one sub-bucket of the in-CTA sort.  3000: one long-list segment above SORT_MAX records,
    sorted in place in global memory.  Ties in Gaussian index order, like the reference's radix sort."""
    worst, rp, o = check(_mine(), equal_depth_scene(n), cuda_device)
    st = o["state"]
    keys = st["keys"].view(np.uint64)
    assert keys.size == n and np.unique(keys).size == 1 and (n <= SORT_MAX) == (n == 1000)
    assert np.array_equal(st["point_list"].view(np.uint32), np.arange(n, dtype=np.uint32))
    assert_within(worst)
