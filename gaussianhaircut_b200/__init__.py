"""gaussianhaircut_b200 -- H100-native (sm_90a) strand-aligned differentiable Gaussian rasterizer.

A from-scratch replacement for the one hot path of eth-ait/GaussianHaircut: the extension
`ext/diff_gaussian_rasterization_hair` behind `src/gaussian_renderer`.  The public surface mirrors
the reference package `diff_gaussian_rasterization` (see `rasterizer.py`); the compute lives in
hand-written CUDA kernels behind the C ABI declared in `include/gh_rasterizer.h`.

There is no CPU fallback: importing the binding without the built library raises.
"""
__version__ = "0.1.0"

from .rasterizer import (  # noqa: F401
    GaussianRasterizationSettings,
    GaussianRasterizer,
    rasterize_gaussians,
    set_gradient_arena,
    last_gradient_arena,
)
