"""The counterpart of the reference's `metrics.py` (src/metrics.py): SSIM, PSNR and, given a function for it, LPIPS of
every render set under `<scene>/test/<method>/{renders,gt}`, written to `<scene>/results.json` and
`<scene>/per_view.json` in the reference's layout.

    python -m gaussianhaircut_b200.metrics -m <scene> [<scene> ...]

The PNGs are decoded by PIL on the host and kept as bytes (RGB: the first three channels, as `[:, :3]` does); the
bytes go to the device through one pinned buffer per chunk of views, and `gh_eval_ssim` evaluates the chunk in one
launch, reading x / 255 as torchvision's `to_tensor` rounds it.  The per-view numbers of a method are read back once.
LPIPS needs VGG weights this package does not ship: it is computed only when the caller passes
`lpips_fn(render, gt) -> tensor` (both (1,3,H,W) float32 in [0, 1] on the device, as the reference hands them to
`lpips(..., net_type='vgg')`); otherwise the LPIPS entries are left out and a notice says so.
"""
from __future__ import annotations

import json
import os
from argparse import ArgumentParser
from pathlib import Path
from typing import Callable, Dict, List, Optional, Sequence

import numpy as np
import torch

from . import inference

CHUNK = 16          # views per gh_eval_ssim launch (same size only)


def read_png(path) -> np.ndarray:
    """One 8-bit PNG as planar (3,H,W) uint8: the first three channels of what to_tensor would see."""
    from PIL import Image
    with Image.open(path) as im:
        a = np.asarray(im)
    if a.dtype != np.uint8 or a.ndim != 3 or a.shape[2] < 3:
        raise RuntimeError(f"metrics: {path} is not an 8-bit RGB or RGBA image (mode {im.mode})")
    return np.ascontiguousarray(a[:, :, :3].transpose(2, 0, 1))


def read_images(renders_dir, gt_dir):
    """readImages (src/metrics.py:24-34) on the host: -> renders, gts (lists of (3,H,W) uint8 arrays), image names in
    os.listdir order."""
    renders, gts, names = [], [], []
    for fname in os.listdir(renders_dir):
        renders.append(read_png(Path(renders_dir) / fname))
        gts.append(read_png(Path(gt_dir) / fname))
        names.append(fname)
    return renders, gts, names


def _chunks(renders: Sequence[np.ndarray], chunk: int):
    """Runs of consecutive views of one size, at most `chunk` long: (start, stop)."""
    i = 0
    while i < len(renders):
        j = i + 1
        while j < len(renders) and j - i < chunk and renders[j].shape == renders[i].shape:
            j += 1
        yield i, j
        i = j


def ssim_psnr(renders: Sequence[np.ndarray], gts: Sequence[np.ndarray], device: torch.device,
              chunk: int = CHUNK) -> tuple:
    """SSIM and PSNR of each (render, gt) pair of (3,H,W) uint8 arrays: one pinned upload and one gh_eval_ssim launch
    per chunk, one read-back at the end.  -> two float32 CPU tensors (N,)."""
    n = len(renders)
    ssim = torch.empty(n, dtype=torch.float32, device=device)
    psnr = torch.empty(n, dtype=torch.float32, device=device)
    for i, j in _chunks(renders, chunk):
        host = torch.empty((2, j - i) + renders[i].shape, dtype=torch.uint8, pin_memory=True)
        for k in range(i, j):
            if gts[k].shape != renders[k].shape:
                raise RuntimeError(f"metrics: render {renders[k].shape} and gt {gts[k].shape} sizes differ")
            host[0, k - i].copy_(torch.from_numpy(renders[k]))
            host[1, k - i].copy_(torch.from_numpy(gts[k]))
        # (the caching host allocator keeps the pinned buffer until the copy has read it)
        dev = host.to(device, non_blocking=True)
        inference.eval_ssim(dev[0], dev[1], ssim[i:j], psnr[i:j])
    return ssim.cpu(), psnr.cpu()     # the one synchronisation


def _lpips(renders, gts, lpips_fn, device) -> List[float]:
    to = lambda a: torch.from_numpy(a).float().div(255).unsqueeze(0).to(device)  # noqa: E731  (to_tensor's rounding)
    return [float(torch.as_tensor(lpips_fn(to(r), to(g))).reshape(-1)[0]) for r, g in zip(renders, gts)]


def evaluate(model_paths: Sequence[str], lpips_fn: Optional[Callable] = None, device=None,
             chunk: int = CHUNK) -> Dict[str, dict]:
    """evaluate (src/metrics.py:36-97): for each scene, for each method under <scene>/test, the mean SSIM, PSNR (and
    LPIPS with `lpips_fn`) printed and written to <scene>/results.json, the per-view values to <scene>/per_view.json.
    A scene that fails prints the reference's message and is skipped.  -> {scene: results dict}."""
    device = torch.device("cuda", torch.cuda.current_device()) if device is None else torch.device(device)
    full_dict, per_view_dict = {}, {}
    print("")
    if lpips_fn is None:
        print("LPIPS not computed: pass lpips_fn (it needs VGG weights this package does not ship)")
    for scene_dir in model_paths:
        try:
            print("Scene:", scene_dir)
            full_dict[scene_dir] = {}
            per_view_dict[scene_dir] = {}
            test_dir = Path(scene_dir) / "test"
            for method in os.listdir(test_dir):
                print("Method:", method)
                method_dir = test_dir / method
                renders, gts, names = read_images(method_dir / "renders", method_dir / "gt")
                ssims, psnrs = ssim_psnr(renders, gts, device, chunk)
                means = {"SSIM": ssims.mean(), "PSNR": psnrs.mean()}
                per_view = {"SSIM": ssims, "PSNR": psnrs}
                if lpips_fn is not None:
                    lp = torch.tensor(_lpips(renders, gts, lpips_fn, device))
                    means["LPIPS"], per_view["LPIPS"] = lp.mean(), lp
                for k, v in means.items():
                    print("  {:<5}: {:>12.7f}".format(k, float(v)))
                print("")
                full_dict[scene_dir][method] = {k: v.item() for k, v in means.items()}
                per_view_dict[scene_dir][method] = {k: {name: x for x, name in zip(v.tolist(), names)}
                                                    for k, v in per_view.items()}
            with open(scene_dir + "/results.json", "w") as fp:
                json.dump(full_dict[scene_dir], fp, indent=True)
            with open(scene_dir + "/per_view.json", "w") as fp:
                json.dump(per_view_dict[scene_dir], fp, indent=True)
        except Exception:
            print("Unable to compute metrics for model", scene_dir)
    return full_dict


def main(argv=None) -> None:
    parser = ArgumentParser(description="SSIM / PSNR of render sets (src/metrics.py)")
    parser.add_argument("--model_paths", "-m", required=True, nargs="+", type=str, default=[])
    args = parser.parse_args(argv)
    torch.cuda.set_device(torch.device("cuda:0"))
    evaluate(args.model_paths)


if __name__ == "__main__":
    main()
