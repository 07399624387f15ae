"""CPU tests of the strand stages' image loss: pin the extended float64 replay (tests/_strand_loss64.py) on the
reference's own loss functions composed as the strand trainers compose them (tests/golden/loss64strands.npz,
tests/golden/make_golden_loss64_strands.py) and on float64 autograd of the restated compositions; check that stage 0
is the appearance replay; check that gh_image_loss_stage refuses bad stages, options and arguments before launching
anything, and that it is declared, exported and bound at ABI 6."""
import ctypes as C
import os
import re

import numpy as np
import pytest
import torch

import _strand_loss64 as sl
import loss64
import loss_oracle

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "loss64strands.npz")
PIN_TOL = 1e-12         # float64 against float64: a few units of 2^-53 of the scale
LAMBDAS = {1: (0.8, 0.2, 0.4, 0.1), 2: (0.8, 0.0, 0.4, 0.1)}
NAMES = ("out", "gt_image", "gt_mask", "gt_angle", "gt_conf")


def _worst(value, ref, scale):
    """max |value - ref| / scale; an element whose scale is 0 must match exactly."""
    value, ref, scale = (torch.as_tensor(np.asarray(a)).double() for a in (value, ref, scale))
    d = (value - ref).abs()
    assert bool((d[scale == 0] == 0).all()), "an element the replay calls exact differs"
    return float((d / scale.clamp(min=1e-300))[scale > 0].max())


def _check_losses(r, want):
    for k, v in zip(loss64.LOSSES, want):
        s = r["losses_scale"][k]
        assert (abs(r["losses"][k] - v) <= PIN_TOL * s) if s else r["losses"][k] == v, (k, r["losses"][k], v)


def _exact_channels(r, stage, options):
    sc = r["scale"]
    assert bool((sc[[7, 9]] == 0).all()) and bool((r["dL"][[7, 9]] == 0).all())
    if options & sl.NO_CONF:
        assert bool((r["dL"][8] == 0).all()) and bool((sc[8] == 0).all())
    if stage == 2:
        assert bool((r["dL"][4] == 0).all()) and bool((sc[4] == 0).all())


@pytest.mark.parametrize("options", sl.OPTION_SETS)
@pytest.mark.parametrize("stage", [1, 2])
@pytest.mark.parametrize("case", ["7x5", "1x13", "40x33"])
def test_replay_matches_reference_loss_utils_float64(case, stage, options):
    with np.load(GOLDEN) as z:
        ins = [z[f"{case}/{k}"] for k in NAMES]
        lam = z[f"lambdas{stage}"]
        want, dL = z[f"{case}/s{stage}o{options}/losses"], z[f"{case}/s{stage}o{options}/dL_dout"]
    r = sl.replay(*ins, [float(x) for x in lam], stage=stage, options=options, consts=loss64.CONST64)
    assert not r["nan"] and r["nan_terms"] == 0.0
    _check_losses(r, want)
    assert _worst(r["dL"], dL, r["scale"]) <= PIN_TOL
    _exact_channels(r, stage, options)
    if case != "1x13" and not options & sl.NO_CONF:
        assert float(r["dL"][6].abs().max()) > 1e6                                    # the eps gradient


def test_golden_covers_every_stage_and_option():
    with np.load(GOLDEN) as z:
        keys = set(z.files)
    for case in ("7x5", "1x13", "40x33"):
        for stage in (1, 2):
            for o in sl.OPTION_SETS:
                assert f"{case}/s{stage}o{o}/dL_dout" in keys
    assert {"nan9x8/s1o0/losses", "nan9x8/s2o0/losses"} <= keys


def test_replay_nan_image_pixel_matches_reference():
    """A NaN image pixel: stage 2 replaces Ll1 by 0 and zeroes channels 0..2; stage 1 keeps the NaN (Ll1, Lssim and the
    total are NaN, the SSIM window spreads NaN over the image gradient), like the reference."""
    with np.load(GOLDEN) as z:
        ins = [z[f"nan9x8/{k}"] for k in NAMES]
        g = {s: (z[f"nan9x8/s{s}o0/losses"], z[f"nan9x8/s{s}o0/dL_dout"]) for s in (1, 2)}
    r2 = sl.replay(*ins, LAMBDAS[2], stage=2, consts=loss64.CONST64)
    assert r2["nan_terms"] == 1.0 and not r2["nan"] and r2["losses"]["Ll1"] == 0.0
    _check_losses(r2, g[2][0])
    assert _worst(r2["dL"], g[2][1], r2["scale"]) <= PIN_TOL
    assert bool((r2["dL"][0:3] == 0).all()) and bool((r2["scale"][0:3] == 0).all())
    r1 = sl.replay(*ins, LAMBDAS[1], stage=1, consts=loss64.CONST64)
    want, dL = g[1]
    assert np.isnan(want[0]) and np.isnan(r1["losses"]["total"]) and np.isnan(r1["losses"]["Ll1"])
    for i, k in ((3, "Lmask"), (4, "Lorient")):
        assert abs(r1["losses"][k] - want[i]) <= PIN_TOL * r1["losses_scale"][k]
    dL = torch.from_numpy(dL)
    assert torch.equal(torch.isnan(r1["dL"]), torch.isnan(dL))
    fin = ~torch.isnan(dL)
    assert _worst(r1["dL"][fin], dL[fin], r1["scale"][fin]) <= PIN_TOL
    assert bool(torch.isnan(dL[0:3]).any()) and not bool(torch.isnan(dL[3:]).any())


@pytest.mark.parametrize("options", sl.OPTION_SETS)
@pytest.mark.parametrize("stage", [1, 2])
@pytest.mark.parametrize("W,H,seed", [(45, 37, 1), (20, 18, 3)])
def test_replay_matches_float64_autograd(W, H, seed, stage, options):
    ins = loss_oracle.synthetic_case(W, H, seed)
    lam = LAMBDAS[stage]
    r = sl.replay(*ins, lam, stage=stage, options=options, consts=loss64.CONST64)
    x = ins[0].double().requires_grad_(True)
    loss, parts = sl.training_loss(stage, options, x, *[t.double() for t in ins[1:]],
                                   [float(np.float32(v)) for v in lam])
    loss.backward()
    assert _worst(r["dL"], x.grad, r["scale"]) <= PIN_TOL
    _check_losses(r, [float(p.detach()) for p in parts])
    _exact_channels(r, stage, options)


def test_replay_stage0_is_the_appearance_replay():
    ins = loss64.edge_scene(40, 33, 3)
    lam = (0.8, 0.2, 0.4, 0.1)
    a, b = loss64.replay(*ins, lam), sl.replay(*ins, lam, stage=0, options=0)
    assert a["losses"] == b["losses"] and a["losses_scale"] == b["losses_scale"] and a["nan"] == b["nan"]
    assert torch.equal(a["dL"], b["dL"]) and torch.equal(a["scale"], b["scale"])
    assert a["alternatives"] == b["alternatives"]


def test_replay_unit_weight_ignores_gt_conf():
    """With unit weights the orientation weight map is never read: any gt_conf, or none, gives the same replay."""
    ins = list(loss64.edge_scene(20, 18, 7))
    a = sl.replay(*ins, LAMBDAS[1], stage=1, options=sl.UNIT_WEIGHT)
    ins[4] = None
    b = sl.replay(*ins, LAMBDAS[1], stage=1, options=sl.UNIT_WEIGHT)
    assert a["losses"] == b["losses"] and torch.equal(a["dL"], b["dL"])
    assert a["sum_w"] == (20.0 * 18.0, 0.0)


# ------------------------------------------------------------------------------------------------ the C entry point
@pytest.fixture(scope="module")
def lib():
    from gaussianhaircut_b200 import build, _capi
    build.build(verbose=False)
    return _capi.load()


FAKE = C.c_void_p(0x10000)


def _stage(lib, stage=1, options=0, W=4, H=4, ptrs=None, ws=FAKE, l_ssim=1.0):
    out, gi, gm, ga, gc, losses, dL = ptrs if ptrs is not None else [FAKE] * 7
    return lib.gh_image_loss_stage(W, H, stage, options, out, gi, gm, ga, gc, 1.0, l_ssim, 1.0, 1.0, ws, losses, dL,
                                   None, 0)


def test_stage_loss_rejects_before_launching(lib):
    """Every refusal of gh_image_loss_stage returns GH_E_INVALID_ARG with a message and calls nothing on the device;
    every call here fails one check, so no pointer is ever dereferenced."""
    from gaussianhaircut_b200 import _capi
    n0 = lib.gh_kernel_launch_count()
    cases = [
        (lambda: _stage(lib, stage=-1), "unknown stage"), (lambda: _stage(lib, stage=3), "unknown stage"),
        (lambda: _stage(lib, stage=0, options=1), "takes no options"),
        (lambda: _stage(lib, stage=0, options=2), "takes no options"),
        (lambda: _stage(lib, stage=1, options=4), "unknown option bits"),
        (lambda: _stage(lib, stage=2, options=0x80000003), "unknown option bits"),
        (lambda: _stage(lib, stage=2, l_ssim=0.2), "no SSIM term"),
        (lambda: _stage(lib, stage=2, l_ssim=float("nan")), "no SSIM term"),
        (lambda: _stage(lib, W=0), "bad size"), (lambda: _stage(lib, H=-2), "bad size"),
        (lambda: _stage(lib, ws=None), "missing pointer"),
        (lambda: _stage(lib, ws=C.c_void_p(0x10004)), "8-byte aligned"),
        (lambda: _stage(lib, W=1539, H=87211), "2^27"), (lambda: _stage(lib, W=1 << 16, H=1 << 16), "2^27"),
    ]
    for i in range(7):
        p = [FAKE] * 7
        p[i] = None
        for stage in (0, 1, 2):
            cases.append((lambda p=p, stage=stage: _stage(lib, stage=stage, ptrs=p, l_ssim=0.0), "missing pointer"))
    # gt_orient_conf (index 4) may be NULL only with unit weights
    p = [FAKE] * 7
    p[4] = None
    for stage, options in ((1, 2), (2, 0), (2, 2)):
        cases.append((lambda stage=stage, options=options: _stage(lib, stage, options, ptrs=p, l_ssim=0.0),
                      "missing pointer"))
    for call, msg in cases:
        assert call() == _capi.GH_E_INVALID_ARG
        err = lib.gh_last_error().decode()
        assert err.startswith("gh_image_loss_stage: ") and msg in err, err
    # a NULL gt_orient_conf with unit weights passes the pointer check: the next refusal (size) is what fails
    for stage, options in ((1, 1), (1, 3), (2, 1), (2, 3)):
        assert _stage(lib, stage, options, W=1539, H=87211, ptrs=p, l_ssim=0.0) == _capi.GH_E_INVALID_ARG
        assert "2^27" in lib.gh_last_error().decode()
    assert lib.gh_kernel_launch_count() == n0


def test_appearance_messages_unchanged(lib):
    """gh_image_loss keeps its own name in its messages."""
    from gaussianhaircut_b200 import _capi
    p = [FAKE] * 7
    assert lib.gh_image_loss(0, 4, *p[:5], 1.0, 1.0, 1.0, 1.0, FAKE, p[5], p[6], None, 0) == _capi.GH_E_INVALID_ARG
    assert lib.gh_last_error() == b"gh_image_loss: bad size or missing pointer"


def test_stage_entry_point_declared_exported_abi6(lib):
    from gaussianhaircut_b200 import _capi, losses
    src = open(os.path.join(ROOT, "include", "gh_rasterizer.h")).read()
    assert re.search(r"\bint gh_image_loss_stage\s*\(int width, int height, int stage, unsigned options,", src)
    for name, value in (("GH_LOSS_STAGE_APPEARANCE", "0"), ("GH_LOSS_STAGE_STRANDS", "1"),
                        ("GH_LOSS_STAGE_LATENT_STRANDS", "2"), ("GH_LOSS_ORIENT_UNIT_WEIGHT", "1u"),
                        ("GH_LOSS_ORIENT_NO_CONF", "2u")):
        assert re.search(rf"#define {name}\s+{value}\b", src), name
    assert losses.STAGES == {"appearance": 0, "strands": 1, "latent_strands": 2}
    assert (losses.ORIENT_UNIT_WEIGHT, losses.ORIENT_NO_CONF) == (sl.UNIT_WEIGHT, sl.NO_CONF) == (1, 2)
    assert hasattr(lib, "gh_image_loss_stage") and "gh_image_loss_stage" in _capi.SIGNATURES
    assert len(_capi.SIGNATURES["gh_image_loss_stage"][1]) == 18
    assert lib.gh_abi_version() == 6 and _capi.ABI_VERSION == 6


def test_python_layer_rejects_without_a_device():
    """The wrapper's own refusals come before anything touches a device."""
    from gaussianhaircut_b200 import losses
    x = torch.zeros(10, 4, 4)
    with pytest.raises(RuntimeError, match="unknown stage"):
        losses.image_loss_forward_backward(x, x[:3], x[:2], x[:1], x[:1], 1, 1, 1, 1, stage="hair")
    with pytest.raises(RuntimeError, match="options of the strand stages"):
        losses.image_loss_forward_backward(x, x[:3], x[:2], x[:1], x[:1], 1, 1, 1, 1, use_gt_orient_conf=False)
    with pytest.raises(RuntimeError, match="CUDA tensor"):
        losses.strand_image_loss(x, x[:3], x[:2], x[:1], None, 1, 1, 1, 1, use_gt_orient_conf=False)
