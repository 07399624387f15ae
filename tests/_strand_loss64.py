"""TEST INFRASTRUCTURE ONLY -- the strand stages' training losses, for gh_image_loss_stage.

Two parts, both built on the appearance-stage oracles in oracle/ and leaving them as they are:

  * `strand_training_loss` and `latent_strand_training_loss`: plain PyTorch compositions of the restated l1_loss /
    ssim / or_loss (oracle/loss_oracle.py), as SRC/train_strands.py:128-147 and SRC/train_latent_strands.py:130-152
    compose them, without the prior terms (Lsds, LDF) that come from external networks.  `fns` plugs in the
    reference's own (l1_loss, ssim, or_loss) (tests/golden/make_golden_loss64_strands.py);
  * `replay(..., stage, options)`: the float64 replay of oracle/loss64.py extended to those compositions, with the
    same error scales (see its docstring).  stage 0 with no options is loss64.replay itself.  Stage 1 is the replay
    with the image mask fixed to 1 (x * 1 is exact, so the image terms carry no mask rounding).  Stage 2 has no SSIM
    part, an L1 gradient sign(I - G) lambda_l1 / (3N) in channels 0..2, and a one-channel mask term
    LCE = mean |out[3] - gt_mask[0]|.  UNIT_WEIGHT sets the orientation weights to 1 and their sum to N exactly;
    NO_CONF drops the confidence factor and the log term (channel 8 is exactly 0, scale 0).  The NaN rules follow
    the trainers: stage 1 replaces only Lorient, stage 2 replaces each of Ll1, LCE and LOR and zeroes its channels.
"""
from __future__ import annotations

import math
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "oracle"))
import loss64  # noqa: E402
import loss_oracle  # noqa: E402
from loss64 import V  # noqa: E402

UNIT_WEIGHT = 1
NO_CONF = 2
OPTION_SETS = (0, UNIT_WEIGHT, NO_CONF, UNIT_WEIGHT | NO_CONF)


def opts(use_gt_orient_conf: bool, train_orient_conf: bool) -> int:
    return (0 if use_gt_orient_conf else UNIT_WEIGHT) | (0 if train_orient_conf else NO_CONF)


def flags(options: int):
    """(use_gt_orient_conf, train_orient_conf) of an option mask."""
    return not (options & UNIT_WEIGHT), not (options & NO_CONF)


# ------------------------------------------------------------------------------------------------ compositions
def _orient_term(f_or, orient_angle, orient_conf, gt_mask, gt_orient_angle, gt_orient_conf, use_gt_orient_conf,
                 train_orient_conf):
    orient_weight = torch.ones_like(gt_mask[:1])
    if use_gt_orient_conf:
        orient_weight = orient_weight * gt_orient_conf
    if not train_orient_conf:
        orient_conf = None
    return f_or(orient_angle, gt_orient_angle, orient_conf, weight=orient_weight, mask=gt_mask[:1])


def strand_training_loss(renders, gt_image, gt_mask, gt_orient_angle, gt_orient_conf, lambda_dl1, lambda_dssim,
                         lambda_dmask, lambda_dorient, use_gt_orient_conf=True, train_orient_conf=True, fns=None):
    """SRC/train_strands.py:128-147 without `Lsds * opt.lambda_dsds`."""
    f_l1, f_ssim, f_or = fns if fns is not None else (loss_oracle.l1_loss, loss_oracle.ssim, loss_oracle.or_loss)
    image, mask, orient_angle, orient_conf = loss_oracle.split_render(renders)
    Ll1 = f_l1(image, gt_image)
    Lssim = 1.0 - f_ssim(image, gt_image)
    Lmask = f_l1(mask, gt_mask)
    Lorient = _orient_term(f_or, orient_angle, orient_conf, gt_mask, gt_orient_angle, gt_orient_conf,
                           use_gt_orient_conf, train_orient_conf)
    if torch.isnan(Lorient).any():
        Lorient = torch.zeros_like(Ll1)
    loss = Ll1 * lambda_dl1 + Lssim * lambda_dssim + Lmask * lambda_dmask + Lorient * lambda_dorient
    return loss, {"Ll1": Ll1, "Lssim": Lssim, "Lmask": Lmask, "Lorient": Lorient}


def latent_strand_training_loss(renders, gt_image, gt_mask, gt_orient_angle, gt_orient_conf, lambda_dl1,
                                lambda_dmask, lambda_dorient, use_gt_orient_conf=True, train_orient_conf=True,
                                fns=None):
    """SRC/train_latent_strands.py:130-152 without `LDF * opt.lambda_dsds`."""
    f_l1, _, f_or = fns if fns is not None else (loss_oracle.l1_loss, loss_oracle.ssim, loss_oracle.or_loss)
    image, mask, orient_angle, orient_conf = loss_oracle.split_render(renders)
    LCE = f_l1(mask[:1], gt_mask[:1])
    Ll1 = f_l1(image, gt_image)
    LOR = _orient_term(f_or, orient_angle, orient_conf, gt_mask, gt_orient_angle, gt_orient_conf,
                       use_gt_orient_conf, train_orient_conf)
    if torch.isnan(Ll1).any():
        Ll1 = torch.zeros_like(Ll1)
    if torch.isnan(LCE).any():
        LCE = torch.zeros_like(Ll1)
    if torch.isnan(LOR).any():
        LOR = torch.zeros_like(Ll1)
    loss = Ll1 * lambda_dl1 + LCE * lambda_dmask + LOR * lambda_dorient
    return loss, {"Ll1": Ll1, "LCE": LCE, "LOR": LOR}


def training_loss(stage, options, renders, gt_image, gt_mask, gt_orient_angle, gt_orient_conf, lambdas, fns=None):
    """The composition of `stage` (0, 1, 2) with lambdas = (l1, ssim, mask, orient); returns (loss, [total, Ll1,
    Lssim, Lmask (LCE), Lorient (LOR)]) in the slot order of gh_image_loss_stage's losses."""
    u, t = flags(options)
    if stage == 0:
        assert options == 0
        loss, p = loss_oracle.training_loss(renders, gt_image, gt_mask, gt_orient_angle, gt_orient_conf, *lambdas,
                                            fns=fns)
        return loss, [loss, p["Ll1"], p["Lssim"], p["Lmask"], p["Lorient"]]
    if stage == 1:
        loss, p = strand_training_loss(renders, gt_image, gt_mask, gt_orient_angle, gt_orient_conf, *lambdas,
                                       use_gt_orient_conf=u, train_orient_conf=t, fns=fns)
        return loss, [loss, p["Ll1"], p["Lssim"], p["Lmask"], p["Lorient"]]
    assert lambdas[1] == 0
    loss, p = latent_strand_training_loss(renders, gt_image, gt_mask, gt_orient_angle, gt_orient_conf, lambdas[0],
                                          lambdas[2], lambdas[3], use_gt_orient_conf=u, train_orient_conf=t, fns=fns)
    return loss, [loss, p["Ll1"], torch.zeros_like(loss), p["LCE"], p["LOR"]]


# ------------------------------------------------------------------------------------------------ the replay
def _lmin(b):
    """pi min(l0, l1, l2) and its bound, as loss64._orient forms it."""
    inner = torch.minimum(b["l1"], b["l2"])
    e_inner = torch.where(b["l1"] < b["l2"], b["e_d1"], torch.where(b["l1"] > b["l2"], b["e_d2"],
                                                                     torch.maximum(b["e_d1"], b["e_d2"])))
    lmin = torch.minimum(b["l0"], inner)
    e_lmin_raw = torch.where(b["l0"] < inner, b["e_d0"], torch.where(b["l0"] > inner, e_inner,
                                                                     torch.maximum(b["e_d0"], e_inner)))
    return V(lmin * math.pi, math.pi * e_lmin_raw + 2.0 * lmin * math.pi)


def replay(out, gt_image, gt_mask, gt_angle, gt_conf, lambdas, stage=0, options=0, device=None,
           consts=loss64.CONST32) -> dict:
    """loss64.replay for gh_image_loss_stage(stage, options); the same result keys, plus `nan_terms` (slot 7 of the
    losses: 1 Ll1, 2 LCE replaced) in stage 2.  gt_conf may be None with UNIT_WEIGHT."""
    if stage == 0:
        assert options == 0, "the appearance stage has no options"
        return loss64.replay(out, gt_image, gt_mask, gt_angle, gt_conf, lambdas, device=device, consts=consts)
    assert stage in (1, 2) and options in OPTION_SETS
    if device is None:
        device = out.device if isinstance(out, torch.Tensor) else torch.device("cpu")
    unit_w, no_conf = bool(options & UNIT_WEIGHT), bool(options & NO_CONF)
    o, gi, gm, ga = (loss64._f64(a, device) for a in (out, gt_image, gt_mask, gt_angle))
    lam = [loss64._f32(x) for x in lambdas]
    if stage == 2:
        assert lam[1] == 0.0, "the latent-strand stage has no SSIM term"
    H, W = o.shape[1:]
    N = H * W
    m0 = gm[0]
    if unit_w:
        w = torch.ones(H, W, dtype=torch.float64, device=device)
        sum_w = (float(N), 0.0)                     # a float32 sum of N ones is exact below 2^24 (and in double)
    else:
        w = loss64._f64(gt_conf, device)[0]
        sum_w = (float(w.sum()), float((1.0 + math.log2(max(N, 1))) * w.abs().sum()))
    wnd = loss64.window(device)
    I, G = o[0:3], gi
    s_l1 = V.c(lam[0] / (3.0 * N), o[0])
    sgn = torch.sign(I - G)
    terms = {"w": V(w)}
    l1 = (I - G).abs()
    terms["l1"] = V(l1.sum(0), l1.sum(0))
    if stage == 1:
        # SSIM of the unmasked image: loss64.replay's arithmetic with m1 = 1 (exact products)
        x, y = V(I), V(G)
        mu1, mu2 = x.conv(wnd), y.conv(wnd)
        E11, E22, E12 = (x * x).conv(wnd), (y * y).conv(wnd), (x * y).conv(wnd)
        mu1_sq, mu2_sq, mu12 = mu1 * mu1, mu2 * mu2, mu1 * mu2
        s1, s2, s12 = E11 - mu1_sq, E22 - mu2_sq, E12 - mu12
        A1, A2 = 2.0 * mu12 + loss64.C1, 2.0 * s12 + loss64.C2
        B1, B2 = mu1_sq + mu2_sq + loss64.C1, s1 + s2 + loss64.C2
        BB = B1 * B2
        smap = A1 * A2 / BB
        D0 = 2.0 * mu2 * (A2 - A1) / BB - 2.0 * mu1 * smap * (B2 - B1) / BB
        D1 = -smap / B2
        D2 = 2.0 * A1 / BB
        s_ssim = V.c(-lam[1] / (3.0 * N), o[0])
        dS = D0.conv(wnd) + 2.0 * x * D1.conv(wnd) + y * D2.conv(wnd)
        g_img = s_ssim * dS + s_l1 * V(sgn)
        terms["ssim"] = V(smap.v.sum(0), smap.e.sum(0))
        dmk = o[3:5] - gm
        g_mask = lam[2] / (2.0 * N) * torch.sign(dmk)
        terms["mask"] = V(dmk.abs().sum(0), dmk.abs().sum(0))
    else:
        smap = None
        g_img = s_l1 * V(sgn)
        terms["ssim"] = V(torch.zeros(H, W, dtype=torch.float64, device=device))
        dmk = o[3:4] - gm[0:1]
        g_mask = lam[2] / float(N) * torch.sign(dmk)
        terms["mask"] = V(dmk.abs().sum(0), dmk.abs().sum(0))
    # orientation: with NO_CONF the gradient path is the confidence path at conf = 1 (an exact factor); the loss
    # term is pi min(...) * m0 * w and channel 8 is zero
    conf = torch.ones_like(o[8]) if no_conf else o[8]
    ori = loss64._orient(o[5].reshape(-1), o[6].reshape(-1), conf.reshape(-1), ga[0].reshape(-1), m0.reshape(-1),
                         w.reshape(-1), lam[3], sum_w[0], sum_w[1], consts)
    lp = _lmin(ori["base"]) * V(m0.reshape(-1)) * V(w.reshape(-1)) if no_conf else ori["lp"]
    terms["orient"] = V(lp.v.reshape(H, W), lp.e.reshape(H, W))
    sums, sums_scale = {}, {}
    for k in loss64.SUMS:
        sums[k], sums_scale[k] = loss64._sum(terms[k], N)
    if unit_w:
        sums["w"], sums_scale["w"] = float(N), 0.0
    if stage == 1:
        losses, losses_scale, nan = loss64._finish(sums, sums_scale, N, lam)
        nan_l1 = nan_ce = False
    else:
        losses, losses_scale, nan, nan_l1, nan_ce = _finish_latent(sums, sums_scale, N, lam)
    dL = torch.zeros(10, H, W, dtype=torch.float64, device=device)
    sc = torch.zeros_like(dL)
    if not nan_l1:
        dL[0:3], sc[0:3] = g_img.v, g_img.e
    if stage == 1:
        dL[3:5], sc[3:5] = g_mask, g_mask.abs()
    elif not nan_ce:
        dL[3:4], sc[3:4] = g_mask, g_mask.abs()
    if not nan:
        dL[5], sc[5] = ori["g5"].reshape(H, W), ori["e5"].reshape(H, W)
        dL[6], sc[6] = ori["g6"].reshape(H, W), ori["e6"].reshape(H, W)
        if not no_conf:
            dL[8], sc[8] = ori["g8"].v.reshape(H, W), ori["g8"].e.reshape(H, W)
        ratios = {k: v.reshape(H, W) for k, v in ori["ratios"].items()}
        alts = loss64._alternatives(ori, H, W)
    else:
        ratios = {k: torch.full((H, W), math.inf, dtype=torch.float64, device=device) for k in loss64.DECISIONS}
        alts = {}
    return dict(sums=sums, sums_scale=sums_scale, losses=losses, losses_scale=losses_scale, nan=nan, dL=dL, scale=sc,
                ratios=ratios, alternatives=alts, ssim_map=smap.v if smap is not None else None, terms=terms,
                sum_w=sum_w, nan_terms=(1.0 if nan_l1 else 0.0) + (2.0 if nan_ce else 0.0))


def _finish_latent(sums, sums_scale, N, lam):
    """Loss values of stage 2 from the sums (SRC/train_latent_strands.py:142-152): Lssim 0, LCE in the Lmask slot,
    each NaN term replaced by an exact 0."""
    n = float(N)
    with np.errstate(all="ignore"):
        Ll1 = np.float64(sums["l1"]) / (3 * n)
        LCE = np.float64(sums["mask"]) / n
        Lo = np.float64(sums["orient"]) / np.float64(sums["w"])
    nan_l1, nan_ce, nan = bool(np.isnan(Ll1)), bool(np.isnan(LCE)), bool(np.isnan(Lo))
    L = {"Ll1": 0.0 if nan_l1 else float(Ll1), "Lssim": 0.0, "Lmask": 0.0 if nan_ce else float(LCE),
         "Lorient": 0.0 if nan else float(Lo)}
    S = {"Ll1": 0.0 if nan_l1 else sums_scale["l1"] / (3 * n) + abs(L["Ll1"]), "Lssim": 0.0,
         "Lmask": 0.0 if nan_ce else sums_scale["mask"] / n + abs(L["Lmask"]),
         "Lorient": 0.0 if nan else (sums_scale["orient"] + abs(Lo) * sums_scale["w"]) / abs(sums["w"]) + abs(Lo)}
    keys = ("Ll1", "Lmask", "Lorient")
    lams = (lam[0], lam[2], lam[3])
    L["total"] = sum(l * L[k] for l, k in zip(lams, keys))
    S["total"] = sum(abs(l) * (S[k] + abs(L[k])) for l, k in zip(lams, keys))
    return L, S, nan, nan_l1, nan_ce
