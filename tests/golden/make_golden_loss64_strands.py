"""Golden vectors for the strand stages' float64 loss replay (tests/_strand_loss64.py): the reference's OWN loss
functions (src/utils/loss_utils.py: l1_loss, ssim, or_loss, imported unmodified from /root/reference) composed as
src/train_strands.py:128-147 and src/train_latent_strands.py:130-152 compose them, evaluated in float64 with autograd
on the edge scenes of loss64.edge_scene at 7x5, 1x13 and 40x33: both stages x the four settings of
(use_gt_orient_conf, train_orient_conf), plus one scene per stage with a NaN image pixel.  The float32 inputs are
stored in the file.  The file name has no underscore, so the rasterizer (*_*.npz) and loss (loss_*.npz) golden
collectors do not pick it up.

    python tests/golden/make_golden_loss64_strands.py        (build container only: needs /root/reference)
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "oracle"))
sys.path.insert(0, "/root/reference/src")
import _strand_loss64 as sl  # noqa: E402
import loss64  # noqa: E402
from utils import loss_utils as ref  # noqa: E402  (the reference module itself)

LAMBDAS = {1: (0.8, 0.2, 0.4, 0.1), 2: (0.8, 0.0, 0.4, 0.1)}
CASES = {"7x5": (7, 5, 1), "1x13": (1, 13, 2), "40x33": (40, 33, 3)}
NAN_PIXEL = (1, 3, 4)                     # (channel, y, x) of the NaN image pixel on a 9x8 scene


def evaluate(stage, options, ins):
    r64 = ins[0].double().requires_grad_(True)
    lam = [float(np.float32(x)) for x in LAMBDAS[stage]]
    loss, parts = sl.training_loss(stage, options, r64, *[t.double() for t in ins[1:]], lam,
                                   fns=(ref.l1_loss, ref.ssim, ref.or_loss))
    loss.backward()
    return np.array([float(p.detach()) for p in parts]), r64.grad.numpy()


arrays = {f"lambdas{s}": np.array(l, np.float32) for s, l in LAMBDAS.items()}
scenes = {name: loss64.edge_scene(W, H, seed) for name, (W, H, seed) in CASES.items()}
nan_ins = list(loss64.edge_scene(9, 8, 4, specials=False))
nan_ins[0][NAN_PIXEL] = float("nan")
scenes["nan9x8"] = tuple(nan_ins)
for name, ins in scenes.items():
    for k, t in zip(("out", "gt_image", "gt_mask", "gt_angle", "gt_conf"), ins):
        arrays[f"{name}/{k}"] = t.numpy()
    for stage in (1, 2):
        for options in (sl.OPTION_SETS if name != "nan9x8" else (0,)):
            losses, grad = evaluate(stage, options, ins)
            arrays[f"{name}/s{stage}o{options}/losses"] = losses
            arrays[f"{name}/s{stage}o{options}/dL_dout"] = grad
            print(name, stage, options, losses)
np.savez_compressed(os.path.join(HERE, "loss64strands.npz"), **arrays)
