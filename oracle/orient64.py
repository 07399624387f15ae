"""TEST INFRASTRUCTURE ONLY -- a float64 replay of the reference's `calc_orients`
(src/preprocessing/calc_orientation_maps.py:53-97) that says, for every pixel, which answers a float32 evaluation may
give, and how far its variance may lie from the exact one.

* `gray64`, `difference_of_gaussians`: the grayscale and the DoG through scipy.ndimage.gaussian_filter (mode 'nearest',
  truncate 4), which is what scikit-image 0.20's `difference_of_gaussians` calls;
* `gabor_kernel`, `bank`: scikit-image 0.20's complex Gabor kernel and the reference's bank, restated here on their own
  (not imported from the product), float64 then float32;
* `replay(dog32, bank32, thetas32, G, crop)`: the correlation in float64 over the same float32 DoG and float32 bank the
  kernel receives, per pixel and group: the responses F_j, a first-order float32 error bound e_j = gamma_T sum|w||x|
  (T = K*K bounds the taps summed: taps with a zero weight add nothing), the top-two margin, the candidate set
  {j : F_j >= F_max - e_max - e_j}, and for every candidate the variance and its error scale (`var_scale`: the kernel's
  float32 variance lies within about u * var_scale of the exact one, u = 2^-24; TOL in the tests is measured by
  tools/orient_replay_calibrate.py).  Large images are replayed in bands of rows, or on crops;
* `check(orients, var, rep, tol)`: the per-pixel verdicts the GPU tests assert on.
Only tests/, tools/ and oracle/ref_python.py import this module.
"""
from __future__ import annotations

import math
import types

import numpy as np

U32 = 2.0 ** -24
U_TF32 = 2.0 ** -10          # TF32 keeps 10 explicit mantissa bits; rounding or truncation, either is bounded by this


def gray64(img: np.ndarray) -> np.ndarray:
    img = np.asarray(img)
    return 0.2989 * img[:, :, 0] + 0.5870 * img[:, :, 1] + 0.1140 * img[:, :, 2]


def difference_of_gaussians(image, low_sigma, high_sigma=None, *, mode="nearest", cval=0, channel_axis=None,
                            truncate=4.0):
    """skimage.filters.difference_of_gaussians (0.20) for a 2-D float64 image: gaussian(low) - gaussian(high), each
    scipy.ndimage.gaussian_filter with the given mode and truncate."""
    from scipy import ndimage
    image = np.asarray(image, dtype=np.float64)
    if high_sigma is None:
        high_sigma = 1.6 * low_sigma
    a = ndimage.gaussian_filter(image, float(low_sigma), mode=mode, cval=cval, truncate=truncate)
    b = ndimage.gaussian_filter(image, float(high_sigma), mode=mode, cval=cval, truncate=truncate)
    return a - b


def dog64(img: np.ndarray, low: float = 0.4, high: float = 10.0) -> np.ndarray:
    return difference_of_gaussians(gray64(img), low, high)


def gabor_kernel(frequency, theta=0, bandwidth=1, sigma_x=None, sigma_y=None, n_stds=3, offset=0,
                 dtype=np.complex128):
    """skimage.filters.gabor_kernel (0.20, skimage/filters/_gabor.py): complex kernel of shape (2*y0+1, 2*x0+1)."""
    if sigma_x is None or sigma_y is None:
        b = 1.0 / np.pi * np.sqrt(np.log(2) / 2.0) * (2.0 ** bandwidth + 1) / (2.0 ** bandwidth - 1)
        sigma_x = b / frequency if sigma_x is None else sigma_x
        sigma_y = b / frequency if sigma_y is None else sigma_y
    c, s = math.cos(theta), math.sin(theta)
    half_x = math.ceil(max(abs(n_stds * sigma_x * c), abs(n_stds * sigma_y * s), 1))
    half_y = math.ceil(max(abs(n_stds * sigma_y * c), abs(n_stds * sigma_x * s), 1))
    yy, xx = np.meshgrid(np.arange(-half_y, half_y + 1), np.arange(-half_x, half_x + 1), indexing="ij", sparse=True)
    u = xx * c + yy * s
    v = -xx * s + yy * c
    out = np.empty(v.shape, dtype=dtype)
    np.exp(-0.5 * (u ** 2 / sigma_x ** 2 + v ** 2 / sigma_y ** 2), out=out)
    out /= 2 * np.pi * sigma_x * sigma_y
    out *= np.exp(1j * (2 * np.pi * frequency * u + offset))
    return out


def support(sigma_x: float, sigma_y: float, theta: float, n_stds: float = 3) -> tuple:
    """(x0, y0): the kernel spans 2*y0+1 rows and 2*x0+1 columns."""
    c, s = math.cos(theta), math.sin(theta)
    return (math.ceil(max(abs(n_stds * sigma_x * c), abs(n_stds * sigma_y * s), 1)),
            math.ceil(max(abs(n_stds * sigma_y * c), abs(n_stds * sigma_x * s), 1)))


def bank(num_frequencies=1, num_filters=180, num_sigmas_x=1, num_sigmas_y=1, num_offsets=1):
    """-> (bank float32 (N,K,K), thetas float32, G): the reference's loops (calc_orientation_maps.py:24-50)."""
    thetas = np.linspace(0, math.pi * (num_filters - 1) / num_filters, num_filters)
    offs = np.linspace(0, math.pi * (num_offsets - 1) / num_offsets, num_offsets)
    sxs = [1.8] if num_sigmas_x == 1 else list(2 ** np.arange(num_sigmas_x))
    sys_ = [2.4] if num_sigmas_y == 1 else list(2 ** np.arange(num_sigmas_y))
    fs = [0.23] if num_frequencies == 1 else list(2.0 ** (-np.arange(num_frequencies)))
    ks = []
    for t in thetas:
        for sx in sxs:
            for sy in sys_:
                for o in offs:
                    for f in fs:
                        ks.append(np.real(gabor_kernel(f, theta=math.pi - t, sigma_x=sx, sigma_y=sy, offset=o)))
    side = max(max(k.shape) for k in ks)
    if side % 2 == 0:
        side += 1
    out = np.zeros((len(ks), side, side))
    for i, k in enumerate(ks):
        oy, ox = (side - k.shape[0]) // 2, (side - k.shape[1]) // 2
        out[i, oy:oy + k.shape[0], ox:ox + k.shape[1]] = k
    G = len(sxs) * len(sys_) * len(offs) * len(fs)
    return out.astype(np.float32), thetas.astype(np.float32), G


# ---------------------------------------------------------------------------------------------------- the replay
def _gamma(n: int, u: float = U32) -> float:
    return n * u / (1 - n * u)


def _dist32(idx: np.ndarray, thetas32: np.ndarray, nf: int) -> np.ndarray:
    """(n,) indices -> (n, nf) float32 wrap-around distances, the reference's float32 expressions."""
    pi = np.float32(math.pi)
    a = (idx.astype(np.float32) / np.float32(nf)) * pi
    t = a[:, None] - thetas32[None, :]
    return np.minimum(np.abs(t), np.minimum(np.abs(t - pi), np.abs(t + pi)))


def _windows(dog32: np.ndarray, K: int, y0: int, y1: int, x0: int, x1: int) -> np.ndarray:
    """(npix, K*K) float64 input windows of output pixels [y0,y1) x [x0,x1) (zero padding K//2)."""
    P = K // 2
    H, W = dog32.shape
    pad = np.zeros((y1 - y0 + K - 1, x1 - x0 + K - 1))
    ya, yb, xa, xb = max(y0 - P, 0), min(y1 + P, H), max(x0 - P, 0), min(x1 + P, W)
    pad[ya - (y0 - P):yb - (y0 - P), xa - (x0 - P):xb - (x0 - P)] = dog32[ya:yb, xa:xb]
    win = np.lib.stride_tricks.sliding_window_view(pad, (K, K))
    return win.reshape(-1, K * K)


def replay(dog32: np.ndarray, bank32: np.ndarray, thetas32: np.ndarray, G: int, crop=None, band_pixels: int = 65536,
           tf32: bool = False) -> dict:
    """Replay output pixels crop = (y0, y1, x0, x1) (default: the whole image).  Returns arrays over the crop's pixels
    (row-major) and groups: argmax (n, G) of the float64 responses |R|, fmax (n, G) their maximum, ncand (n, G) the
    candidate count, margin (n, G) the top-two gap over the sum of the two largest error bounds, and the candidate pairs
    (pix, g, idx, var64, var_scale).  With
    tf32=True the error bound also covers inputs rounded to TF32 (the reference's cuDNN default)."""
    H, W = dog32.shape
    y0, y1, x0, x1 = crop if crop is not None else (0, H, 0, W)
    N, K, _ = bank32.shape
    nf = N // G
    T = K * K
    coef = _gamma(T) + ((1 + U_TF32) ** 2 - 1 if tf32 else 0.0)
    Wm = bank32.reshape(N, T).astype(np.float64)
    Wa = np.abs(Wm)
    rows_per_band = max(1, band_pixels // max(1, x1 - x0))
    keep = {"argmax": [], "ncand": [], "margin": [], "fmax": []}
    pairs = []
    base = 0
    for ya in range(y0, y1, rows_per_band):
        yb = min(ya + rows_per_band, y1)
        X = _windows(dog32, K, ya, yb, x0, x1)
        F = np.abs(X @ Wm.T).reshape(-1, nf, G).transpose(0, 2, 1)          # (n, G, nf): channel j*G + g
        A = (np.abs(X) @ Wa.T).reshape(-1, nf, G).transpose(0, 2, 1) * T   # T * sum|w||x|
        e = A * (coef / T)
        fmax = F.max(axis=2, keepdims=True)
        cand = F >= fmax - e.max(axis=2, keepdims=True) - e
        if nf > 1:
            top2 = np.partition(F, nf - 2, axis=2)[..., -2:]
            e2 = np.partition(e, nf - 2, axis=2)[..., -2:]
            margin = (top2[..., 1] - top2[..., 0]) / np.maximum(e2.sum(axis=2), 1e-300)
        else:
            margin = np.full(F.shape[:2], np.inf)
        keep["argmax"].append(F.argmax(axis=2))
        keep["ncand"].append(cand.sum(axis=2))
        keep["margin"].append(margin)
        keep["fmax"].append(fmax[..., 0])
        p, g, j = np.nonzero(cand)
        d = _dist32(j, thetas32, nf).astype(np.float64)
        Fp, Ap = F[p, g], A[p, g]
        S = np.maximum(Fp.sum(axis=1), 1e-12)
        var = (d * d * Fp).sum(axis=1) / S
        scale = ((d * d * Ap).sum(axis=1) + var * Ap.sum(axis=1)) / S + var * (2 * nf + 8)
        pairs.append((p + base, g, j, var, scale))
        base += F.shape[0]
    cat = lambda k: np.concatenate([q[k] for q in pairs])  # noqa: E731
    out = {k: np.concatenate(v) for k, v in keep.items()}
    out.update({"crop": (y0, y1, x0, x1), "G": G, "nf": nf,
                "pix": cat(0), "g": cat(1), "idx": cat(2), "var": cat(3), "scale": cat(4)})
    return out


def check(orients: np.ndarray, var: np.ndarray, rep: dict, tol: float) -> dict:
    """Verdicts for the kernel's maps (full-image arrays) on the replayed crop.  A pixel passes when
      * its index is a candidate of some group g whose variance at that index is within tol * scale of var, and
      * var is no larger than min over groups of the largest candidate variance + tol * scale (the argmin over groups);
      * where every group has one candidate and the groups' variance intervals do not overlap, the index is the
        replay's exactly (`certain`).
    Returns counts and the flat indices (into the crop) of failing pixels."""
    y0, y1, x0, x1 = rep["crop"]
    o = orients[y0:y1, x0:x1].reshape(-1).astype(np.int64)
    v = var[y0:y1, x0:x1].reshape(-1).astype(np.float64)
    n = o.size
    pix, g, idx, pv, ps = rep["pix"], rep["g"], rep["idx"], rep["var"], rep["scale"]
    tolv = tol * ps
    match = (idx == o[pix]) & (np.abs(v[pix] - pv) <= tolv)
    ok_pair = np.zeros(n, bool)
    np.logical_or.at(ok_pair, pix[match], True)
    # the largest variance each group may report, then the smallest over groups
    G = rep["G"]
    hi = np.full((n, G), -np.inf)
    np.maximum.at(hi, (pix, g), pv + tolv)
    ok_min = v <= hi.min(axis=1) * (1 + 1e-12) + 1e-30
    # certain pixels: one candidate per group, and one group clearly smallest
    ncand = rep["ncand"]
    single = (ncand == 1).all(axis=1)
    lo = np.full((n, G), np.inf)
    np.minimum.at(lo, (pix, g), pv - tolv)
    best_g = np.argmin(hi, axis=1)
    lo_other = np.where(np.arange(G)[None, :] == best_g[:, None], np.inf, lo).min(axis=1) if G > 1 else np.full(n, np.inf)
    certain = single & (hi[np.arange(n), best_g] < lo_other)
    want = rep["argmax"][np.arange(n), best_g]
    ok_certain = ~certain | (o == want)
    bad = np.nonzero(~(ok_pair & ok_min & ok_certain))[0]
    # per pixel, the group that explains its variance best; then the worst pixel
    same = idx == o[pix]
    ratio = np.full(n, np.inf)
    np.minimum.at(ratio, pix[same], np.abs(v[pix[same]] - pv[same]) / np.maximum(ps[same], 1e-300))
    fin = np.isfinite(ratio)
    return {"n": n, "certain": int(certain.sum()), "bad": bad, "n_bad": int(bad.size),
            "worst_ratio": float(ratio[fin].max()) if fin.any() else 0.0, "certain_mask": certain}


def skimage_filters_module() -> types.ModuleType:
    """A `skimage.filters` carrying this module's gabor_kernel and difference_of_gaussians (the two names the
    reference's calc_orientation_maps.py imports from it)."""
    m = types.ModuleType("skimage.filters")
    m.gabor_kernel = gabor_kernel
    m.difference_of_gaussians = difference_of_gaussians
    return m
