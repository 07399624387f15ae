"""Fused image-space losses of the appearance stage ('next' row 4, SURVEY.md 8f).

One native call computes the reference's training loss from the rasterizer's raw (10,H,W) output and
its gradient w.r.t. that output (the tensor `gh_backward` consumes as dL_dpix):

    Ll1     = l1_loss(image, gt_image, mask=gt_mask[1:])            src/train_gaussians.py:126
    Lssim   = 1 - ssim(image * gt_mask[1:], gt_image * gt_mask[1:])   :127
    Lmask   = l1_loss(mask, gt_mask)                                 :128
    Lorient = or_loss(orient_angle, gt_orient_angle, orient_conf,
                      weight=gt_orient_conf, mask=gt_mask[:1])       :130-133 (NaN -> 0)
    loss    = lambda_dl1 Ll1 + lambda_dssim Lssim + lambda_dmask Lmask + lambda_dorient Lorient   :135-140

with orient_angle derived from channels 5..6 exactly like src/gaussian_renderer/__init__.py:100-105.
The loss functions themselves are src/utils/loss_utils.py:19-48 and :73-121.  No CPU path: CPU
tensors raise.

The two strand stages compose the same functions differently, and run in the same kernels
(`gh_image_loss_stage`):

    strand_image_loss          src/train_strands.py:128-147         Ll1 and Lssim unmasked
    latent_strand_image_loss   src/train_latent_strands.py:130-152  Ll1 unmasked, no SSIM,
                                                                    LCE = l1_loss(mask[:1], gt_mask[:1]),
                                                                    Ll1 / LCE / LOR each NaN -> 0

Both take the trainer's `opt.use_gt_orient_conf` and `opt.train_orient_conf`.  The prior term
(`Lsds * opt.lambda_dsds`, `LDF * opt.lambda_dsds`) comes from networks outside this package: add it to
the returned loss, autograd flows through the sum.
"""
from __future__ import annotations

import ctypes as C
from typing import Dict, Tuple

import torch

from . import _capi
from ._capi import _ptr, _stream

__all__ = ["hair_image_loss", "strand_image_loss", "latent_strand_image_loss", "HairImageLoss",
           "image_loss_forward_backward", "workspace_elems"]

# gh_image_loss_stage's stages and option bits (include/gh_rasterizer.h)
STAGES = {"appearance": 0, "strands": 1, "latent_strands": 2}
ORIENT_UNIT_WEIGHT = 1
ORIENT_NO_CONF = 2


def _check(name: str, t: torch.Tensor, shape) -> torch.Tensor:
    if not t.is_cuda:
        raise RuntimeError(f"hair_image_loss: {name} must be a CUDA tensor (there is no CPU path)")
    if tuple(t.shape) != tuple(shape):
        raise RuntimeError(f"hair_image_loss: {name} must have shape {tuple(shape)}, got {tuple(t.shape)}")
    if t.dtype != torch.float32:
        t = t.float()
    return t.contiguous()


def image_loss_forward_backward(out: torch.Tensor, gt_image: torch.Tensor, gt_mask: torch.Tensor,
                                gt_orient_angle: torch.Tensor, gt_orient_conf: torch.Tensor,
                                l_dl1: float, l_dssim: float, l_dmask: float, l_dorient: float,
                                workspace: torch.Tensor | None = None, stage: str = "appearance",
                                use_gt_orient_conf: bool = True, train_orient_conf: bool = True):
    """The native call itself (no autograd): returns (losses float32[8], dL_dout (10,H,W)).
    `workspace` (float64 tensor of at least `workspace_elems(W, H)` elements) can be passed to reuse it.
    Under `torch.use_deterministic_algorithms(True)` the loss sums are formed in a fixed order (bit-reproducible).

    `stage`: "appearance" (gh_image_loss, the default), "strands" or "latent_strands" (gh_image_loss_stage);
    `use_gt_orient_conf` / `train_orient_conf` are the strand trainers' options of the same names (False: unit
    orientation weights, where gt_orient_conf may be None / no confidence term).  The appearance stage has neither."""
    lib = _capi.load()
    if stage not in STAGES:
        raise RuntimeError(f"hair_image_loss: unknown stage {stage!r} (one of {', '.join(STAGES)})")
    options = (0 if use_gt_orient_conf else ORIENT_UNIT_WEIGHT) | (0 if train_orient_conf else ORIENT_NO_CONF)
    if stage == "appearance" and options:
        raise RuntimeError("hair_image_loss: use_gt_orient_conf / train_orient_conf are options of the strand stages")
    if out.dim() != 3 or out.shape[0] != 10:
        raise RuntimeError("hair_image_loss: the render must have shape (10, H, W)")
    H, W = int(out.shape[1]), int(out.shape[2])
    out_c = _check("render", out, (10, H, W))
    gi = _check("gt_image", gt_image, (3, H, W))
    gm = _check("gt_mask", gt_mask, (2, H, W))
    ga = _check("gt_orient_angle", gt_orient_angle, (1, H, W))
    if gt_orient_conf is None and not use_gt_orient_conf:
        gc = None                                   # not read with unit weights
    else:
        gc = _check("gt_orient_conf", gt_orient_conf, (1, H, W))
    dev = out.device
    need = workspace_elems(W, H)
    if workspace is None or workspace.numel() < need or workspace.dtype != torch.float64 or workspace.device != dev:
        workspace = torch.empty(need, dtype=torch.float64, device=dev)
    losses = torch.empty(8, dtype=torch.float32, device=dev)
    dL = torch.empty_like(out_c)
    det = int(torch.are_deterministic_algorithms_enabled())
    with torch.cuda.device(dev):
        if stage == "appearance":
            _capi.check(lib.gh_image_loss(W, H, _ptr(out_c), _ptr(gi), _ptr(gm), _ptr(ga), _ptr(gc),
                                          float(l_dl1), float(l_dssim), float(l_dmask), float(l_dorient),
                                          _ptr(workspace), _ptr(losses), _ptr(dL), _stream(dev), det))
        else:
            _capi.check(lib.gh_image_loss_stage(W, H, STAGES[stage], options, _ptr(out_c), _ptr(gi), _ptr(gm),
                                                _ptr(ga), _ptr(gc), float(l_dl1), float(l_dssim), float(l_dmask),
                                                float(l_dorient), _ptr(workspace), _ptr(losses), _ptr(dL),
                                                _stream(dev), det))
    return losses, dL


def workspace_elems(W: int, H: int) -> int:
    """Workspace size of gh_image_loss in float64 elements."""
    nbytes = C.c_size_t()
    _capi.check(_capi.load().gh_image_loss_workspace_size(W, H, C.byref(nbytes)))
    return (nbytes.value + 7) // 8


class HairImageLoss(torch.autograd.Function):
    """(total, parts) = HairImageLoss.apply(out10, gt_image, gt_mask, gt_orient_angle, gt_orient_conf,
    lambda_dl1, lambda_dssim, lambda_dmask, lambda_dorient[, stage, use_gt_orient_conf, train_orient_conf]).
    `parts` = float32[8] (detached): total, Ll1, Lssim, Lmask, Lorient, sum of orientation weights, Lorient-was-NaN
    flag, 0 (latent strands: Lssim 0, LCE in place of Lmask, the NaN-replaced terms in the last slot)."""

    @staticmethod
    def forward(ctx, out, gt_image, gt_mask, gt_orient_angle, gt_orient_conf, l_dl1, l_dssim, l_dmask, l_dorient,
                stage="appearance", use_gt_orient_conf=True, train_orient_conf=True):
        losses, dL = image_loss_forward_backward(out, gt_image, gt_mask, gt_orient_angle, gt_orient_conf,
                                                 l_dl1, l_dssim, l_dmask, l_dorient, stage=stage,
                                                 use_gt_orient_conf=use_gt_orient_conf,
                                                 train_orient_conf=train_orient_conf)
        ctx.save_for_backward(dL)
        ctx.mark_non_differentiable(losses)
        return losses[0].clone(), losses

    @staticmethod
    def backward(ctx, g_total, _g_parts):
        (dL,) = ctx.saved_tensors
        return (dL * g_total,) + (None,) * 11


def hair_image_loss(render: torch.Tensor, gt_image: torch.Tensor, gt_mask: torch.Tensor,
                    gt_orient_angle: torch.Tensor, gt_orient_conf: torch.Tensor,
                    lambda_dl1: float, lambda_dssim: float, lambda_dmask: float,
                    lambda_dorient: float) -> Tuple[torch.Tensor, Dict[str, torch.Tensor]]:
    """Training loss of src/train_gaussians.py:126-140 on the raw (10,H,W) rasterizer output.

    Returns (loss, parts); `loss` is differentiable w.r.t. `render`, `parts` holds the detached
    components the reference logs (Ll1, Lssim, Lmask, Lorient) as 0-dim device tensors: no host sync.
    """
    total, p = HairImageLoss.apply(render, gt_image, gt_mask, gt_orient_angle, gt_orient_conf,
                                   lambda_dl1, lambda_dssim, lambda_dmask, lambda_dorient)
    return total, {"Ll1": p[1], "Lssim": p[2], "Lmask": p[3], "Lorient": p[4], "orient_nan": p[6]}


def strand_image_loss(render: torch.Tensor, gt_image: torch.Tensor, gt_mask: torch.Tensor,
                      gt_orient_angle: torch.Tensor, gt_orient_conf: torch.Tensor | None,
                      lambda_dl1: float, lambda_dssim: float, lambda_dmask: float, lambda_dorient: float,
                      use_gt_orient_conf: bool = True,
                      train_orient_conf: bool = True) -> Tuple[torch.Tensor, Dict[str, torch.Tensor]]:
    """Training loss of src/train_strands.py:128-147 without its prior term, on the raw (10,H,W) output of
    `render_hair_strands(...)["raw"]` or `render_hair(...)["raw"]`:

        Ll1 = l1_loss(image, gt_image)            Lssim = 1 - ssim(image, gt_image)      (both unmasked)
        Lmask = l1_loss(mask, gt_mask)            Lorient as the appearance stage, NaN -> 0

    `use_gt_orient_conf` / `train_orient_conf` are the trainer's `opt` fields; with use_gt_orient_conf=False
    gt_orient_conf may be None.  Returns (loss, parts): `loss` is differentiable w.r.t. `render`; `parts` holds Ll1,
    Lssim, Lmask, Lorient and orient_nan as 0-dim device tensors (no host sync).  A NaN Ll1 or Lssim stays NaN in
    the loss, as in the reference.  Add `Lsds * opt.lambda_dsds` to the loss for the reference's total.
    graphs.CapturedStrandStep runs this loss inside the captured train_strands.py iteration; there the trainer passes
    the prior term's `_dirs` gradient to step(dirs_grad=...) instead."""
    total, p = HairImageLoss.apply(render, gt_image, gt_mask, gt_orient_angle, gt_orient_conf,
                                   lambda_dl1, lambda_dssim, lambda_dmask, lambda_dorient, "strands",
                                   use_gt_orient_conf, train_orient_conf)
    return total, {"Ll1": p[1], "Lssim": p[2], "Lmask": p[3], "Lorient": p[4], "orient_nan": p[6]}


def latent_strand_image_loss(render: torch.Tensor, gt_image: torch.Tensor, gt_mask: torch.Tensor,
                             gt_orient_angle: torch.Tensor, gt_orient_conf: torch.Tensor | None,
                             lambda_dl1: float, lambda_dmask: float, lambda_dorient: float,
                             use_gt_orient_conf: bool = True,
                             train_orient_conf: bool = True) -> Tuple[torch.Tensor, Dict[str, torch.Tensor]]:
    """Training loss of src/train_latent_strands.py:130-152 without its prior term, on the raw (10,H,W) output of
    `render_hair(...)["raw"]`:

        Ll1 = l1_loss(image, gt_image)            (unmasked; no SSIM term)
        LCE = l1_loss(mask[:1], gt_mask[:1])      LOR as the appearance stage's Lorient
        each of Ll1, LCE, LOR -> 0 when NaN (its gradient is then exactly 0)

    Returns (loss, parts): `parts` holds Ll1, LCE, LOR (the names the trainer logs) and nan_terms, the replaced
    terms as a float bitmask (1 Ll1, 2 LCE, 4 LOR), as 0-dim device tensors.  Add `LDF * opt.lambda_dsds` to the
    loss for the reference's total."""
    total, p = HairImageLoss.apply(render, gt_image, gt_mask, gt_orient_angle, gt_orient_conf,
                                   lambda_dl1, 0.0, lambda_dmask, lambda_dorient, "latent_strands",
                                   use_gt_orient_conf, train_orient_conf)
    return total, {"Ll1": p[1], "LCE": p[3], "LOR": p[4], "nan_terms": p[7] + 4.0 * p[6]}
