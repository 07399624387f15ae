"""Regenerates mapsref.npz: the reference's own vis_orient, psnr, l1_loss, or_loss, ce_loss and save_image arithmetic
(src/utils/image_utils.py, src/utils/loss_utils.py, torchvision.utils.save_image's mul(255).add_(0.5).clamp_(0, 255))
run on CPU float32 tensors, for the seeded inputs of tests/test_render_maps_cpu.py::_case.  Needs the reference
sources (oracle/ref_python.ref_src_dir()).

    python tests/golden/make_golden_maps.py
"""
import math
import os
import sys

import numpy as np
import torch
import torch.nn.functional as F

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path[:0] = [os.path.join(ROOT, "tests"), os.path.join(ROOT, "oracle")]


def save_u8(x):
    return x.mul(255).add_(0.5).clamp_(0, 255).to(torch.uint8).numpy()


def reference_outputs(raw, gts):
    """{name: array} from the reference's functions on the case (raw (10,H,W), gts) as CPU float32 tensors."""
    import ref_python
    ref_python.install_stubs()
    sys.path.insert(0, ref_python.ref_src_dir())
    from utils.image_utils import psnr, vis_orient
    from utils.loss_utils import ce_loss, l1_loss, or_loss
    raw = torch.from_numpy(raw)
    gi, gm, ga, gc = (torch.from_numpy(g) for g in gts)
    image, mask, cov, conf, _ = raw.split([3, 2, 3, 1, 1], dim=0)
    d2 = F.normalize(cov[:2], dim=0)                                   # gaussian_renderer/__init__.py:100-105
    mirror = torch.ones_like(d2[[0]])
    mirror[d2[[0]] < 0] *= -1
    ang = torch.acos(d2[[1]].clamp(-1 + 1e-3, 1 - 1e-3) * mirror) / math.pi
    hair = mask[:1]
    conf_m = conf * hair                                               # render_gaussians.py:52-59
    out = {"orient_angle": ang.numpy(), "orient_u8": save_u8(ang * hair)[0],
           "orient_vis_u8": save_u8(vis_orient(ang, hair)).transpose(1, 2, 0),
           "orient_conf_vis_u8": save_u8(vis_orient(ang, 1 - 1 / (conf_m + 1))).transpose(1, 2, 0),
           "render_u8": save_u8(image.clone()).transpose(1, 2, 0), "hair_mask_u8": save_u8(hair.clone())[0]}
    cl = lambda t: torch.clamp(t, 0.0, 1.0)  # noqa: E731             # train_gaussians.py:254-277
    im, mk, an, ggi, ggm, gga = cl(image), cl(mask), cl(ang), cl(gi), cl(gm), cl(ga)
    out["row_stage0"] = np.array([float(l1_loss(im, ggi).mean().double()), float(l1_loss(mk, ggm).mean().double()),
                                  float(or_loss(an, gga, mask=ggm[:1], weight=gc).mean().double()),
                                  float(psnr(im, ggi).mean().double())])
    out["row_stage2"] = np.array([float(l1_loss(im * ggm[:1], ggi * ggm[:1]).mean().double()),   # train_latent_strands.py:255-258
                                  float(ce_loss(mk[:1], ggm[:1]).mean().double()),
                                  float(or_loss(an, gga, mask=ggm[:1], weight=gc).mean().double()),
                                  float(psnr(im * ggm[:1], ggi * ggm[:1]).mean().double())])
    return out


if __name__ == "__main__":
    import test_render_maps_cpu as t
    raw, gts = t._case()
    np.savez_compressed(os.path.join(HERE, "mapsref.npz"), **reference_outputs(raw, gts))
    print("wrote mapsref.npz")
