"""Regenerates ssim64.npz: the reference's own loss_utils.ssim and image_utils.psnr (src/utils/loss_utils.py:72-121,
src/utils/image_utils.py:17-19) run in float64 on the CPU, on the cases of tests/_ssim64.py (the masked case
multiplied in float64, as the replay does).  Needs the reference sources (oracle/ref_python.ref_src_dir()).

    python tests/golden/make_golden_ssim64.py
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path[:0] = [os.path.join(ROOT, "tests"), os.path.join(ROOT, "oracle")]


def reference_outputs(img1, img2, mask):
    import ref_python
    sys.path.insert(0, ref_python.ref_src_dir())
    from utils.image_utils import psnr
    from utils.loss_utils import ssim
    a, b = (torch.from_numpy(x).double()[None] for x in (img1, img2))
    if mask is not None:
        m = torch.from_numpy(mask).double()[None]
        a, b = a * m, b * m
    return float(ssim(a, b)), float(psnr(a, b).reshape(()))


def main():
    import _ssim64
    out = {}
    for name, (a, b, m) in _ssim64.cases().items():
        s, p = reference_outputs(a, b, m)
        out[f"{name}/ssim"], out[f"{name}/psnr"] = np.float64(s), np.float64(p)
    path = os.path.join(HERE, "ssim64.npz")
    np.savez_compressed(path, **out)
    print(path, len(out))


if __name__ == "__main__":
    main()
