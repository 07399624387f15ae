"""Golden vectors for the float64 loss replay (oracle/loss64.py): the reference's OWN loss functions
(src/utils/loss_utils.py: l1_loss, ssim, or_loss, imported unmodified from /root/reference) evaluated in float64 with
autograd on the edge scenes of loss64.edge_scene (ties, clamps, zero and tiny directions, background pixels, image and
mask equalities, a masked-out block and a constant block), 7x5, 1x13 and 40x33.  The float32 inputs are stored in the
file, so the test does not depend on the scene builder staying the same.  The file name has no underscore: the
rasterizer goldens are collected as tests/golden/*_*.npz and the loss goldens as loss_*.npz, and this file is
neither.

    python tests/golden/make_golden_loss64.py        (build container only: needs /root/reference)
"""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.join(ROOT, "oracle"))
sys.path.insert(0, "/root/reference/src")
import loss64  # noqa: E402
import loss_oracle  # noqa: E402
from utils import loss_utils as ref  # noqa: E402  (the reference module itself)

LAMBDAS = (0.8, 0.2, 0.4, 0.1)   # dl1, dssim, dmask, dorient (all terms active)
CASES = {"7x5": (7, 5, 1), "1x13": (1, 13, 2), "40x33": (40, 33, 3)}

arrays = {"lambdas": np.array(LAMBDAS, np.float32)}
for name, (W, H, seed) in CASES.items():
    ins = loss64.edge_scene(W, H, seed)
    r64 = ins[0].double().requires_grad_(True)
    loss, parts = loss_oracle.training_loss(r64, *[t.double() for t in ins[1:]], *[float(np.float32(x)) for x in LAMBDAS],
                                            fns=(ref.l1_loss, ref.ssim, ref.or_loss))
    loss.backward()
    for k, t in zip(("out", "gt_image", "gt_mask", "gt_angle", "gt_conf"), ins):
        arrays[f"{name}/{k}"] = t.numpy()
    arrays[f"{name}/losses"] = np.array([float(loss)] + [float(parts[k]) for k in ("Ll1", "Lssim", "Lmask", "Lorient")])
    arrays[f"{name}/dL_dout"] = r64.grad.numpy()
    print(name, float(loss), {k: float(v) for k, v in parts.items()})
np.savez_compressed(os.path.join(os.path.dirname(os.path.abspath(__file__)), "loss64edges.npz"), **arrays)
