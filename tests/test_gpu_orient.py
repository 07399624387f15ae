"""Hair orientation maps on the H100 (csrc/gh_orient.cu) against the float64 replay (oracle/orient64.py), against the
reference's own `calc_orients` and `main()` imported unmodified from the staged copy, and for reproducibility.

A pixel's orientation index must equal the replay's wherever the replay calls it certain, and be one of its candidates
elsewhere; its variance must lie within TOL * scale of the replay's at that index (tests/_orient_cases.py)."""
import math
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import _orient_cases as OC

pytestmark = pytest.mark.gpu

import orient64  # noqa: E402  (oracle/, put on sys.path by _orient_cases)
import orient_ref  # noqa: E402

from gaussianhaircut_b200.orient import calc_orients, orientation_maps  # noqa: E402

DEFAULT_BANK = orient64.bank()


def _maps(img: np.ndarray, device, **kw):
    out = orientation_maps(torch.from_numpy(img).to(device), **kw)
    H, W = img.shape[:2]
    assert out["orients"].dtype == torch.int64 and out["var"].dtype == torch.float32 and out["dog"].dtype == torch.float64
    assert all(v.shape == (H, W) and v.device == device for v in out.values())
    return {k: v.cpu().numpy() for k, v in out.items()}


def _check(img, got, bank=DEFAULT_BANK, crop_list=None):
    b, t, G = bank
    dog32 = orient64.dog64(img).astype(np.float32)
    crop_list = crop_list or [None]
    certain = total = 0
    for crop in crop_list:
        rep = orient64.replay(dog32, b, t, G, crop=crop)
        res = orient64.check(got["orients"], got["var"], rep, OC.TOL)
        assert res["n_bad"] == 0, f"{res['n_bad']} of {res['n']} pixels outside the replay in crop {rep['crop']}: " \
                                  f"first {res['bad'][:8]}"
        certain += res["certain"]
        total += res["n"]
    assert np.all((got["orients"] >= 0) & (got["orients"] < len(t)))
    return certain, total


# ------------------------------------------------------------------------------------------------------------ DoG
@pytest.mark.parametrize("shape", [(1, 1, 3), (5, 5, 4), (97, 131, 3), (1080, 1920, 3)])
def test_dog_is_scipys(cuda_device, shape):
    img = OC.noise(*shape[:2], seed=shape[0], C=shape[2]) if shape[0] < 1000 else OC.strands(1080, 1920, 3)
    got = _maps(img, cuda_device)
    want = orient64.dog64(img)
    rel = np.abs(got["dog"] - want).max() / max(np.abs(want).max(), 1e-300)
    assert rel <= 1e-13, rel
    from gaussianhaircut_b200 import _capi
    lib = _capi.load()
    # the float32 copy the Gabor stage reads is float32(scipy's DoG), bit for bit
    H, W = img.shape[:2]
    import ctypes as C
    nbytes = C.c_size_t()
    _capi.check(lib.gh_orient_workspace_size(H, W, 180, 17, 180, C.byref(nbytes)))
    ws = torch.zeros(nbytes.value, dtype=torch.uint8, device=cuda_device)
    dog = torch.empty(H, W, dtype=torch.float64, device=cuda_device)
    from gaussianhaircut_b200.orient import gaussian_weights
    wl = torch.from_numpy(gaussian_weights(0.4)).to(cuda_device)
    wh = torch.from_numpy(gaussian_weights(10.0)).to(cuda_device)
    timg = torch.from_numpy(img).to(cuda_device)
    _capi.check(lib.gh_orient_dog(H, W, img.shape[2], _capi._ptr(timg), _capi._ptr(wl), 2, _capi._ptr(wh), 40,
                                  _capi._ptr(dog), _capi._ptr(ws), nbytes.value, _capi._stream(cuda_device)))
    dog32 = ws[:H * W * 4].view(torch.float32).reshape(H, W).cpu().numpy()
    assert np.array_equal(dog32.view(np.uint32), want.astype(np.float32).view(np.uint32))
    assert np.array_equal(dog.cpu().numpy(), got["dog"])


# ------------------------------------------------------------------------------------------- against the replay
@pytest.mark.parametrize("H,W", [(1, 1), (1, 17), (17, 1), (5, 5), (16, 16), (4099, 3), (3, 4099), (67, 45)])
def test_small_and_thin_images(cuda_device, H, W):
    img = OC.noise(H, W, seed=H * 7 + W)
    _check(img, _maps(img, cuda_device))


@pytest.mark.parametrize("value", [0, 255])
def test_constant_image_is_index_zero_variance_zero(cuda_device, value):
    img = np.full((40, 50, 3), value, np.uint8)
    got = _maps(img, cuda_device)
    assert np.all(got["dog"] == 0)                      # these two constants cancel exactly in the DoG
    assert np.all(got["orients"] == 0) and np.all(got["var"] == 0)


def test_other_constant_image(cuda_device):
    # 128 does not cancel exactly (the two Gaussians' weights sum to 1 only to rounding): a tiny constant DoG
    img = np.full((40, 50, 3), 128, np.uint8)
    _check(img, _maps(img, cuda_device))


def test_single_bright_pixel(cuda_device):
    img = np.zeros((41, 39, 3), np.uint8)
    img[20, 19] = 255
    _check(img, _maps(img, cuda_device))


def test_gratings_at_every_degree(cuda_device):
    """Each grating's interior takes one dominant index, within a degree of the stripes' normal, on at least 95 % of
    its pixels (uint8 quantisation and the real filters' zero crossings leave a few pixels elsewhere even in float64),
    and every pixel passes the replay."""
    interior = (44, 84, 44, 84)
    for deg in range(180):
        img = OC.grating(deg)
        got = _maps(img, cuda_device)
        _check(img, got, crop_list=[interior])
        o = got["orients"][44:84, 44:84]
        vals, cnt = np.unique(o, return_counts=True)
        mode = int(vals[np.argmax(cnt)])
        assert cnt.max() >= 0.95 * o.size, (deg, vals, cnt)
        want = (180 - deg) % 180
        assert min(abs(mode - want), 180 - abs(mode - want)) <= 1, (deg, mode)


@pytest.mark.parametrize("C", [3, 4])
def test_strand_picture_1080p(cuda_device, C):
    img = OC.strands(1080, 1920, seed=11, C=C)
    got = _maps(img, cuda_device)
    certain, total = _check(img, got, crop_list=OC.crops(1080, 1920, 160, seed=C, n=6))
    assert certain > 0.3 * total          # the flat background leaves many near-ties; the strands are decided
    if C == 4:
        rgb = _maps(np.ascontiguousarray(img[..., :3]), cuda_device)
        assert all(np.array_equal(rgb[k], got[k]) for k in got)          # alpha is ignored


def test_non_default_bank(cuda_device):
    kw = dict(num_sigmas_x=2, num_offsets=2)
    bank = orient64.bank(**kw)
    assert bank[0].shape == (720, 17, 17) and bank[2] == 4
    img = OC.strands(300, 400, seed=5)
    got = _maps(img, cuda_device, **kw)
    _check(img, got, bank=bank)
    # the argmin over groups matters: a single group would give other answers
    g0 = _maps(img, cuda_device)
    assert not np.array_equal(g0["var"], got["var"])


def test_4096_square_on_crops(cuda_device):
    img = OC.strands(4096, 4096, seed=21, n=8000)
    got = _maps(img, cuda_device)
    _check(img, got, crop_list=OC.crops(4096, 4096, 96, seed=4, n=8))


# ----------------------------------------------------------------------------------- the reference, unmodified
def _ref():
    try:
        return orient_ref.load()
    except RuntimeError as e:
        pytest.skip(str(e))


def test_reference_calc_orients_without_tf32(cuda_device):
    """cuDNN with TF32 off does not sum the taps one by one: its error is not bounded per pixel by sum|w||x| (at 360x480,
    1511 of its pixels lie outside the direct-summation bound the kernels meet, 724 still outside the TF32-wide one,
    on the flat background).  So the kernels are held to the strict replay, and the reference to: the same filtered
    image bit for bit, at most 1 % of pixels outside the TF32-wide replay, and the kernels' index wherever the strict
    replay is certain and the response is not negligible (146 k of the 173 k pixels)."""
    ref = _ref()
    img = OC.strands(360, 480, seed=2)
    prev = torch.backends.cudnn.allow_tf32
    torch.backends.cudnn.allow_tf32 = False
    try:
        ro, rv, rf = ref.calc_orients(img, 0.4, 10, 1, 180, 1, 1, 1, 64)
    finally:
        torch.backends.cudnn.allow_tf32 = prev
    mo, mv, mf = calc_orients(img, 0.4, 10, 1, 180, 1, 1, 1, 64)
    assert mo.dtype == ro.dtype == np.int64 and mv.dtype == rv.dtype == np.float32 and mf.dtype == rf.dtype == np.float64
    assert np.array_equal(mf, rf)
    b, t, G = DEFAULT_BANK
    ours = orient64.check(mo, mv, orient64.replay(rf.astype(np.float32), b, t, G), OC.TOL)
    assert ours["n_bad"] == 0
    wide = orient64.replay(rf.astype(np.float32), b, t, G, tf32=True)
    theirs = orient64.check(ro, rv, wide, OC.TOL_REF)
    assert theirs["n_bad"] <= 0.01 * theirs["n"], f"reference outside the wide replay at {theirs['n_bad']} pixels"
    # cuDNN's error scales with the patch rather than the pixel, so per-pixel certainty does not bind it; where the
    # strict replay is certain and the response is not negligible next to the picture's strongest, it must agree
    strict = orient64.replay(rf.astype(np.float32), b, t, G)
    c = ((strict["ncand"][:, 0] == 1) & (strict["fmax"][:, 0] >= 1e-2 * strict["fmax"].max())).reshape(mo.shape)
    assert c.sum() >= 0.5 * c.size
    assert np.array_equal(mo[c], ro[c])


def test_reference_calc_orients_with_tf32(cuda_device):
    """The reference's default: cuDNN in TF32.  It may only disagree with the kernels where the margin is within the
    TF32 bound, i.e. its index is a candidate of the replay with TF32 input rounding."""
    ref = _ref()
    img = OC.strands(360, 480, seed=2)
    prev = torch.backends.cudnn.allow_tf32
    torch.backends.cudnn.allow_tf32 = True
    try:
        ro, rv, rf = ref.calc_orients(img, 0.4, 10, 1, 180, 1, 1, 1, 64)
    finally:
        torch.backends.cudnn.allow_tf32 = prev
    mo, _, _ = calc_orients(img, 0.4, 10, 1, 180, 1, 1, 1, 64)
    b, t, G = DEFAULT_BANK
    rep = orient64.replay(rf.astype(np.float32), b, t, G, tf32=True)
    cand = set(zip(rep["pix"].tolist(), rep["idx"].tolist()))
    flat = ro.reshape(-1)
    differ = np.nonzero(flat != mo.reshape(-1))[0]
    outside = [p for p in differ if (int(p), int(flat[p])) not in cand]
    assert not outside, f"{len(outside)} of {differ.size} disagreements lie outside the TF32 candidate sets"


def test_cli_matches_the_reference_main(cuda_device, tmp_path):
    ref = _ref()
    import cv2
    from PIL import Image
    img_dir, mask_dir = tmp_path / "img", tmp_path / "mask"
    img_dir.mkdir()
    mask_dir.mkdir()
    pics = {"a.png": OC.strands(200, 260, seed=1), "b.png": OC.strands(150, 170, seed=2, C=4),
            "c.png": OC.noise(64, 90, seed=3)}
    for name, im in pics.items():
        Image.fromarray(im).save(img_dir / name)
        m = (np.random.default_rng(len(name)).random(im.shape[:2]) * 255).astype(np.uint8)
        Image.fromarray(m).save(mask_dir / name)

    def args(root):
        return ["--img_path", str(img_dir), "--mask_path", str(mask_dir), "--orient_dir", str(root / "o"),
                "--conf_dir", str(root / "c"), "--filtered_img_dir", str(root / "f"), "--vis_img_dir", str(root / "v")]

    mine, theirs = tmp_path / "mine", tmp_path / "ref"
    env = dict(os.environ, PYTHONPATH=OC.ROOT)
    r = subprocess.run([sys.executable, "-m", "gaussianhaircut_b200.orient"] + args(mine), cwd=OC.ROOT, env=env,
                       capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-3000:]
    prev = torch.backends.cudnn.allow_tf32
    torch.backends.cudnn.allow_tf32 = False
    try:
        import argparse
        ns = argparse.Namespace(img_path=str(img_dir), mask_path=str(mask_dir), orient_dir=str(theirs / "o"),
                                conf_dir=str(theirs / "c"), filtered_img_dir=str(theirs / "f"),
                                vis_img_dir=str(theirs / "v"), dog_low=0.4, dog_high=10, num_frequencies=1,
                                num_filters=180, num_sigmas_x=1, num_sigmas_y=1, num_offsets=1, crop_size=-1, patch_size=64)
        ref.main(ns)
    finally:
        torch.backends.cudnn.allow_tf32 = prev
    for sub in ("o", "c", "f", "v"):
        assert sorted(os.listdir(mine / sub)) == sorted(os.listdir(theirs / sub)), sub
    b, t, G = DEFAULT_BANK
    for name, im in pics.items():
        stem = name.split(".")[0]
        mo = cv2.imread(str(mine / "o" / f"{stem}.png"), cv2.IMREAD_UNCHANGED)
        ro = cv2.imread(str(theirs / "o" / f"{stem}.png"), cv2.IMREAD_UNCHANGED)
        assert mo.dtype == np.uint8 and mo.shape == im.shape[:2]
        rep = orient64.replay(orient64.dog64(im).astype(np.float32), b, t, G, tf32=True)   # the reference's cuDNN
        c = (rep["ncand"][:, 0] == 1).reshape(mo.shape)
        assert np.array_equal(mo[c], ro[c])
        mv = np.load(mine / "c" / f"{stem}.npy")
        rv = np.load(theirs / "c" / f"{stem}.npy")
        assert mv.dtype == rv.dtype == np.float16
        same = (mo == ro).reshape(-1)
        scale = np.full(mo.size, np.nan)
        hit = rep["idx"] == mo.reshape(-1)[rep["pix"]]
        scale[rep["pix"][hit]] = rep["scale"][hit]
        a, r_ = mv.reshape(-1).astype(np.float64)[same], rv.reshape(-1).astype(np.float64)[same]
        ulp16 = np.spacing(np.maximum(np.abs(a), np.abs(r_)).astype(np.float16)).astype(np.float64)
        assert np.all(np.abs(a - r_) <= (OC.TOL + OC.TOL_REF) * scale[same] + ulp16)
        for sub in ("f",):
            assert np.array_equal(cv2.imread(str(mine / sub / f"{stem}.png"), cv2.IMREAD_UNCHANGED),
                                  cv2.imread(str(theirs / sub / f"{stem}.png"), cv2.IMREAD_UNCHANGED))
        mvis = cv2.imread(str(mine / "v" / f"{stem}.png"), cv2.IMREAD_UNCHANGED)
        rvis = cv2.imread(str(theirs / "v" / f"{stem}.png"), cv2.IMREAD_UNCHANGED)
        agree = mo == ro
        assert np.array_equal(mvis[agree], rvis[agree])


# ---------------------------------------------------------------------------------- reproducibility and streams
def test_reproducible_across_runs_modes_and_streams(cuda_device):
    img = torch.from_numpy(OC.strands(540, 960, seed=8)).to(cuda_device)
    first = {k: v.cpu() for k, v in orientation_maps(img).items()}
    same = lambda out, why: [(torch.equal(out[k].cpu(), first[k]) or pytest.fail(f"{k} differs: {why}")) for k in first]  # noqa: E731
    same(orientation_maps(img), "second run")
    prev = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(True)
    try:
        same(orientation_maps(img), "deterministic mode")
    finally:
        torch.use_deterministic_algorithms(prev)
    side = torch.cuda.Stream(cuda_device)
    side.wait_stream(torch.cuda.current_stream(cuda_device))
    with torch.cuda.stream(side):
        busy = torch.randn(4096, 4096, device=cuda_device)
        out = orientation_maps(img)
        busy = busy @ busy
    side.synchronize()
    same(out, "side stream")


def test_no_host_synchronisation(cuda_device):
    img = torch.from_numpy(OC.strands(256, 256, seed=9)).to(cuda_device)
    orientation_maps(img)                       # constants cached, kernels loaded
    torch.cuda.synchronize()
    stream = torch.cuda.current_stream(cuda_device)
    torch.cuda._sleep(int(2e9))                 # about a second of device time ahead of the call
    gate = torch.cuda.Event()
    gate.record(stream)
    out = orientation_maps(img)
    assert not gate.query(), "orientation_maps waited for the device"
    done = torch.cuda.Event()
    done.record(stream)
    done.synchronize()
    assert out["orients"].shape == (256, 256)


def test_input_conventions(cuda_device):
    img = OC.strands(64, 80, seed=4)
    want = _maps(img, cuda_device)
    wide = torch.zeros(64, 80, 5, dtype=torch.uint8, device=cuda_device)
    wide[..., 1:4] = torch.from_numpy(img).to(cuda_device)
    got = orientation_maps(wide[..., 1:4])
    assert all(np.array_equal(got[k].cpu().numpy(), want[k]) for k in want)
    for bad in (torch.zeros(4, 4, 2, dtype=torch.uint8, device=cuda_device),
                torch.zeros(4, 4, 3, device=cuda_device), torch.zeros(4, 4, dtype=torch.uint8, device=cuda_device)):
        with pytest.raises(RuntimeError):
            orientation_maps(bad)
    with pytest.raises(RuntimeError, match="no CPU path"):
        orientation_maps(torch.from_numpy(img))
    o, v, f = calc_orients(img, 0.4, 10, 1, 180, 1, 1, 1, 17)            # patch_size changes nothing
    assert np.array_equal(o, want["orients"]) and np.array_equal(v, want["var"]) and np.array_equal(f, want["dog"])
    assert math.isfinite(float(v.max()))
