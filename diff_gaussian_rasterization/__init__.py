"""Drop-in name.  `src/gaussian_renderer/__init__.py:15` of the reference does

    from diff_gaussian_rasterization import GaussianRasterizationSettings, GaussianRasterizer

Putting this repository's root on `sys.path` makes that import resolve to the H100-native
implementation in `gaussianhaircut_b200` -- nothing in the reference's Python needs to change.
"""
from gaussianhaircut_b200.rasterizer import (  # noqa: F401
    GaussianRasterizationSettings,
    GaussianRasterizer,
    rasterize_gaussians,
    _RasterizeGaussians,
    set_gradient_arena,
    last_gradient_arena,
)
from gaussianhaircut_b200 import _C  # noqa: F401
