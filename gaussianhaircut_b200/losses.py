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
"""
from __future__ import annotations

import ctypes as C
from typing import Dict, Tuple

import torch

from . import _capi
from ._capi import _ptr, _stream

__all__ = ["hair_image_loss", "HairImageLoss", "image_loss_forward_backward", "workspace_elems"]


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
                                workspace: torch.Tensor | None = None):
    """The native call itself (no autograd): returns (losses float32[8], dL_dout (10,H,W)).
    `workspace` (float64 tensor of at least `workspace_elems(W, H)` elements) can be passed to reuse it.
    Under `torch.use_deterministic_algorithms(True)` the loss sums are formed in a fixed order (bit-reproducible)."""
    lib = _capi.load()
    if out.dim() != 3 or out.shape[0] != 10:
        raise RuntimeError("hair_image_loss: the render must have shape (10, H, W)")
    H, W = int(out.shape[1]), int(out.shape[2])
    out_c = _check("render", out, (10, H, W))
    gi = _check("gt_image", gt_image, (3, H, W))
    gm = _check("gt_mask", gt_mask, (2, H, W))
    ga = _check("gt_orient_angle", gt_orient_angle, (1, H, W))
    gc = _check("gt_orient_conf", gt_orient_conf, (1, H, W))
    dev = out.device
    need = workspace_elems(W, H)
    if workspace is None or workspace.numel() < need or workspace.dtype != torch.float64 or workspace.device != dev:
        workspace = torch.empty(need, dtype=torch.float64, device=dev)
    losses = torch.empty(8, dtype=torch.float32, device=dev)
    dL = torch.empty_like(out_c)
    with torch.cuda.device(dev):
        _capi.check(lib.gh_image_loss(W, H, _ptr(out_c), _ptr(gi), _ptr(gm), _ptr(ga), _ptr(gc),
                                      float(l_dl1), float(l_dssim), float(l_dmask), float(l_dorient),
                                      _ptr(workspace), _ptr(losses), _ptr(dL), _stream(dev),
                                      int(torch.are_deterministic_algorithms_enabled())))
    return losses, dL


def workspace_elems(W: int, H: int) -> int:
    """Workspace size of gh_image_loss in float64 elements."""
    nbytes = C.c_size_t()
    _capi.check(_capi.load().gh_image_loss_workspace_size(W, H, C.byref(nbytes)))
    return (nbytes.value + 7) // 8


class HairImageLoss(torch.autograd.Function):
    """(total, parts) = HairImageLoss.apply(out10, gt_image, gt_mask, gt_orient_angle, gt_orient_conf,
    lambda_dl1, lambda_dssim, lambda_dmask, lambda_dorient).  `parts` = float32[8] (detached):
    total, Ll1, Lssim, Lmask, Lorient, sum of orientation weights, Lorient-was-NaN flag, 0."""

    @staticmethod
    def forward(ctx, out, gt_image, gt_mask, gt_orient_angle, gt_orient_conf, l_dl1, l_dssim, l_dmask, l_dorient):
        losses, dL = image_loss_forward_backward(out, gt_image, gt_mask, gt_orient_angle, gt_orient_conf,
                                                 l_dl1, l_dssim, l_dmask, l_dorient)
        ctx.save_for_backward(dL)
        ctx.mark_non_differentiable(losses)
        return losses[0].clone(), losses

    @staticmethod
    def backward(ctx, g_total, _g_parts):
        (dL,) = ctx.saved_tensors
        return (dL * g_total, None, None, None, None, None, None, None, None)


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
