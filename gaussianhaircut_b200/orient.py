"""Hair orientation maps: the reference's `calc_orients` (src/preprocessing/calc_orientation_maps.py:53-97) on the GPU,
and its command line (:100-179).  Every training stage's orientation loss reads the two maps this writes per view (an
angle PNG and a float16 variance `.npy`, src/utils/camera_utils.py:66-68).

* `gabor_bank(...)`            the real Gabor filter bank and its angles, on the host (float32);
* `orientation_maps(image)`    uint8 (H,W,3|4) CUDA tensor -> {"orients", "var", "dog"} device tensors, no host sync;
* `calc_orients(...)`          drop-in with the reference's signature: numpy in, numpy (int64, float32, float64) out;
* `python -m gaussianhaircut_b200.orient --img_path ... --mask_path ...` writes the same four files per image.

The contract is in include/gh_rasterizer.h and DESIGN §15; the kernels are csrc/gh_orient.cu.  Importing this module
neither loads the native library nor touches CUDA.
"""
from __future__ import annotations

import argparse
import ctypes as C
import math
import os

import numpy as np
import torch

from . import _capi
from ._capi import _ptr, _stream


# ------------------------------------------------------------------------------------------------------------ bank
def gabor_kernel_real(frequency: float, theta: float, sigma_x: float, sigma_y: float, offset: float,
                      n_stds: float = 3) -> np.ndarray:
    """Real part of scikit-image 0.20's `skimage.filters.gabor_kernel(frequency, theta, sigma_x=, sigma_y=, offset=)`
    (skimage/filters/_gabor.py), float64, shape (2*y0+1, 2*x0+1), evaluated with the same complex128 arithmetic:
    x0 = ceil(max(|n sx cos t|, |n sy sin t|, 1)), y0 = ceil(max(|n sy cos t|, |n sx sin t|, 1)),
    g = exp(-(xr^2/sx^2 + yr^2/sy^2)/2) / (2 pi sx sy) * exp(i (2 pi f xr + offset)), xr = x cos t + y sin t,
    yr = -x sin t + y cos t."""
    ct, st = math.cos(theta), math.sin(theta)
    x0 = math.ceil(max(abs(n_stds * sigma_x * ct), abs(n_stds * sigma_y * st), 1))
    y0 = math.ceil(max(abs(n_stds * sigma_y * ct), abs(n_stds * sigma_x * st), 1))
    y = np.arange(-y0, y0 + 1)[:, None]
    x = np.arange(-x0, x0 + 1)[None, :]
    rotx = x * ct + y * st
    roty = -x * st + y * ct
    g = np.empty(roty.shape, dtype=np.complex128)
    np.exp(-0.5 * (rotx ** 2 / sigma_x ** 2 + roty ** 2 / sigma_y ** 2), out=g)
    g /= 2 * np.pi * sigma_x * sigma_y
    g *= np.exp(1j * (2 * np.pi * frequency * rotx + offset))
    return np.real(g)


def bank_parameters(num_frequencies: int = 1, num_filters: int = 180, num_sigmas_x: int = 1, num_sigmas_y: int = 1,
                    num_offsets: int = 1):
    """The reference's parameter grids (calc_orientation_maps.py:24-30): thetas, sigmas_x, sigmas_y, offsets and
    frequencies; the group index g runs over (sigma_x, sigma_y, offset, frequency) with frequency fastest."""
    thetas = np.linspace(0, math.pi * (num_filters - 1) / num_filters, num_filters)
    offsets = np.linspace(0, math.pi * (num_offsets - 1) / num_offsets, num_offsets)
    sigmas_x = [1.8] if num_sigmas_x == 1 else 2 ** np.arange(num_sigmas_x)
    sigmas_y = [2.4] if num_sigmas_y == 1 else 2 ** np.arange(num_sigmas_y)
    frequencies = [0.23] if num_frequencies == 1 else 2.0 ** (-np.arange(num_frequencies))
    groups = [(sx, sy, off, f) for sx in sigmas_x for sy in sigmas_y for off in offsets for f in frequencies]
    return thetas, groups


def gabor_bank(num_frequencies: int = 1, num_filters: int = 180, num_sigmas_x: int = 1, num_sigmas_y: int = 1,
               num_offsets: int = 1):
    """-> (bank float32 (N, K, K), thetas float32 (num_filters,)), N = num_filters * G: filter j*G + g is the real Gabor
    kernel at theta = pi - thetas[j] with group g's parameters, centred in the odd K x K square (K = the largest
    kernel side, rounded up to odd), computed in float64 and rounded to float32 once."""
    for name, v in (("num_frequencies", num_frequencies), ("num_filters", num_filters), ("num_sigmas_x", num_sigmas_x),
                    ("num_sigmas_y", num_sigmas_y), ("num_offsets", num_offsets)):
        if int(v) != v or v < 1:
            raise ValueError(f"{name} must be a positive integer, got {v!r}")
    thetas, groups = bank_parameters(num_frequencies, num_filters, num_sigmas_x, num_sigmas_y, num_offsets)
    kernels = [gabor_kernel_real(f, math.pi - t, sx, sy, off) for t in thetas for (sx, sy, off, f) in groups]
    K = max(max(k.shape) for k in kernels)
    K += 1 - K % 2
    bank = np.zeros((len(kernels), K, K))
    for i, k in enumerate(kernels):
        py, px = (K - k.shape[0]) // 2, (K - k.shape[1]) // 2
        bank[i, py:py + k.shape[0], px:px + k.shape[1]] = k
    return bank.astype(np.float32), thetas.astype(np.float32)


def gaussian_weights(sigma: float, truncate: float = 4.0) -> np.ndarray:
    """scipy.ndimage.gaussian_filter1d's weights (order 0): radius int(truncate * sigma + 0.5),
    exp(-0.5 / sigma^2 * x^2) normalised by numpy's sum, float64 (symmetric, so reversing them changes nothing)."""
    r = int(truncate * float(sigma) + 0.5)
    x = np.arange(-r, r + 1)
    phi = np.exp(-0.5 / (sigma * sigma) * x ** 2)
    return phi / phi.sum()


# --------------------------------------------------------------------------------------------------- device side
_consts: dict = {}


def _device_constants(device: torch.device, dog_low: float, dog_high: float, bank_args: tuple):
    """Bank, angles and Gaussian weights on `device`, built once per parameter set and uploaded from pinned memory
    without a host synchronisation."""
    key = (device, float(dog_low), float(dog_high), bank_args)
    c = _consts.get(key)
    if c is None:
        bank, thetas = gabor_bank(*bank_args)
        if bank.shape[1] > _MAX_K or len(thetas) > _MAX_FILTERS or bank.shape[0] > _MAX_N:
            raise RuntimeError(f"orientation_maps: a bank of {bank.shape[0]} filters of {bank.shape[1]}x{bank.shape[2]} "
                               f"with {len(thetas)} angles exceeds the kernels' caps (K <= {_MAX_K}, num_filters <= "
                               f"{_MAX_FILTERS}, N <= {_MAX_N})")
        up = lambda a: torch.from_numpy(np.ascontiguousarray(a)).pin_memory().to(device, non_blocking=True)  # noqa: E731
        c = {"bank": up(bank), "thetas": up(thetas), "w_low": up(gaussian_weights(dog_low)),
             "w_high": up(gaussian_weights(dog_high)), "N": bank.shape[0], "K": bank.shape[1], "nf": len(thetas)}
        _consts[key] = c
    return c


# gh_rasterizer.h: GH_ORIENT_MAX_K, GH_ORIENT_MAX_FILTERS, GH_ORIENT_MAX_N
_MAX_K, _MAX_FILTERS, _MAX_N = 17, 256, 4096


def orientation_maps(image: torch.Tensor, dog_low: float = 0.4, dog_high: float = 10., num_frequencies: int = 1,
                     num_filters: int = 180, num_sigmas_x: int = 1, num_sigmas_y: int = 1, num_offsets: int = 1) -> dict:
    """uint8 CUDA tensor (H, W, 3) or (H, W, 4) (alpha ignored) -> {"orients": (H,W) int64 in [0, num_filters),
    "var": (H,W) float32, "dog": (H,W) float64}, on the image's device, produced on the current stream without a host
    synchronisation; bit-reproducible."""
    if not isinstance(image, torch.Tensor):
        raise RuntimeError(f"orientation_maps: 'image' must be a torch.Tensor, got {type(image).__name__}")
    if image.dim() != 3 or image.shape[2] not in (3, 4) or image.shape[0] < 1 or image.shape[1] < 1:
        raise RuntimeError(f"orientation_maps: 'image' must have shape (H, W, 3) or (H, W, 4), got {tuple(image.shape)}")
    if image.dtype != torch.uint8:
        raise RuntimeError(f"expected scalar type Byte but found {image.dtype} for argument 'image'")
    if not image.is_cuda:
        raise RuntimeError("orientation_maps: 'image' must be a CUDA tensor (there is no CPU path)")
    if not (0 < dog_low <= dog_high) or not math.isfinite(dog_high):
        raise ValueError(f"orientation_maps: need 0 < dog_low <= dog_high < inf, got {dog_low}, {dog_high}")
    H, W, Cn = (int(s) for s in image.shape)
    if H * W >= 1 << 31:
        raise RuntimeError(f"orientation_maps: H*W must stay below 2^31, got {H}x{W}")
    dev = image.device
    lib = _capi.load()
    with torch.cuda.device(dev):
        c = _device_constants(dev, dog_low, dog_high, (num_frequencies, num_filters, num_sigmas_x, num_sigmas_y, num_offsets))
        img = image.contiguous()
        nbytes = C.c_size_t()
        _capi.check(lib.gh_orient_workspace_size(H, W, c["N"], c["K"], c["nf"], C.byref(nbytes)))
        ws = torch.empty(nbytes.value, dtype=torch.uint8, device=dev)
        dog = torch.empty(H, W, dtype=torch.float64, device=dev)
        orients = torch.empty(H, W, dtype=torch.int64, device=dev)
        var = torch.empty(H, W, dtype=torch.float32, device=dev)
        stream = _stream(dev)
        rl, rh = (c["w_low"].numel() - 1) // 2, (c["w_high"].numel() - 1) // 2
        _capi.check(lib.gh_orient_dog(H, W, Cn, _ptr(img), _ptr(c["w_low"]), rl, _ptr(c["w_high"]), rh, _ptr(dog),
                                      _ptr(ws), nbytes.value, stream))
        _capi.check(lib.gh_orient_gabor(H, W, _ptr(c["bank"]), c["N"], c["K"], c["nf"], _ptr(c["thetas"]),
                                        _ptr(orients), _ptr(var), _ptr(ws), nbytes.value, stream))
    return {"orients": orients, "var": var, "dog": dog}


def calc_orients(img, dog_low, dog_high, num_frequencies, num_filters, num_sigmas_x, num_sigmas_y, num_offsets,
                 patch_size=64):
    """The reference's `calc_orients` (calc_orientation_maps.py:53): numpy uint8 (H,W,3|4) -> (orients int64, var
    float32, filtered float64) numpy arrays.  `patch_size` is accepted and changes nothing: the maps are the whole-image
    correlation either way."""
    a = np.asarray(img)
    if a.dtype != np.uint8:
        raise RuntimeError(f"calc_orients: expected a uint8 image, got {a.dtype}")
    out = orientation_maps(torch.from_numpy(np.ascontiguousarray(a)).cuda(), dog_low, dog_high, num_frequencies,
                           num_filters, num_sigmas_x, num_sigmas_y, num_offsets)
    return out["orients"].cpu().numpy(), out["var"].cpu().numpy(), out["dog"].cpu().numpy()


# -------------------------------------------------------------------------------------------------- command line
def normalise_filtered(dog: np.ndarray) -> np.ndarray:
    """The DoG stretched linearly so that its minimum maps to 0 and its maximum to 255 (float64; the caller truncates
    to uint8 when writing)."""
    lo, hi = dog.min(), dog.max()
    return (dog - lo) / (hi - lo) * 255


def visualise(angles: np.ndarray, mask: np.ndarray) -> np.ndarray:
    """BGR float64 picture of the angle map (degrees, 0..179) for cv2.imwrite: four triangular hue ramps 45 degrees wide
    centred on 0/180 (red), 90 (green), 45 (magenta) and 135 (teal), clipped to [0, 1], scaled by the mask in [0, 1]
    and by 255."""
    def ramp(centre):
        return np.clip(1 - np.abs(angles - float(centre)) / 45., 0, 1)
    red, green, magenta, teal = ramp(0) + ramp(180), ramp(90), ramp(45), ramp(135)
    bgr = np.stack([magenta + teal, green + teal, red + magenta], axis=-1)
    return np.clip(bgr, 0, 1) * mask[..., None] * 255.


def main(args) -> None:
    import cv2
    from PIL import Image
    for d in (args.orient_dir, args.conf_dir, args.filtered_img_dir, args.vis_img_dir):
        os.makedirs(d, exist_ok=True)
    for name in sorted(os.listdir(args.mask_path)):
        stem = name.split('.')[0]
        img = np.array(Image.open(os.path.join(args.img_path, name)))
        orients, var, dog = calc_orients(img, args.dog_low, args.dog_high, args.num_frequencies, args.num_filters,
                                         args.num_sigmas_x, args.num_sigmas_y, args.num_offsets, args.patch_size)
        angles = orients.astype(np.uint8)
        mask = np.asarray(Image.open(os.path.join(args.mask_path, name))) / 255.
        cv2.imwrite(os.path.join(args.orient_dir, f"{stem}.png"), angles)
        np.save(os.path.join(args.conf_dir, f"{stem}.npy"), var.astype(np.float16))
        cv2.imwrite(os.path.join(args.filtered_img_dir, f"{stem}.png"), normalise_filtered(dog).astype(np.uint8))
        cv2.imwrite(os.path.join(args.vis_img_dir, f"{stem}.png"), visualise(angles, mask).astype(np.uint8))


def parser() -> argparse.ArgumentParser:
    p = argparse.ArgumentParser(description="Hair orientation, variance, filtered and visualisation maps per image",
                                conflict_handler="resolve")
    p.add_argument("--img_path", default="./implicit-hair-data/data/h3ds/00141/image/", type=str)
    p.add_argument("--mask_path", default="./implicit-hair-data/data/h3ds/00141/image/", type=str)
    p.add_argument("--orient_dir", default="./implicit-hair-data/data/h3ds/00141/orientation_maps/", type=str)
    p.add_argument("--conf_dir", default="./implicit-hair-data/data/h3ds/00141/confidence_maps/", type=str)
    p.add_argument("--filtered_img_dir", default="./implicit-hair-data/data/h3ds/00141/filtered_imgs/", type=str)
    p.add_argument("--vis_img_dir", default="./implicit-hair-data/data/h3ds/00141/vis_imgs/", type=str)
    p.add_argument("--dog_low", default=0.4, type=float)
    p.add_argument("--dog_high", default=10, type=float)
    p.add_argument("--num_frequencies", default=1, type=int)
    p.add_argument("--num_filters", default=180, type=int)
    p.add_argument("--num_sigmas_x", default=1, type=int)
    p.add_argument("--num_sigmas_y", default=1, type=int)
    p.add_argument("--num_offsets", default=1, type=int)
    p.add_argument("--crop_size", default=-1, type=int)
    p.add_argument("--patch_size", default=64, type=int)
    return p


if __name__ == "__main__":
    main(parser().parse_known_args()[0])
