"""Drop-in name.  The reference does

    from pysdf import SDF
    f = SDF(mesh.vertices, mesh.faces)
    sdf = f(points)                      # (N,) float32, positive inside

(src/preprocessing/filter_flame_intersections.py:16,115-117, export_curves.py:17,41; imported at module scope by
src/scene/gaussian_model_strands.py:23).  Putting this repository's root on `sys.path` makes that import resolve to the
H100-native implementation in `gaussianhaircut_b200.mesh`; these two calls are the only ones the reference makes.  The
sign comes from the generalized winding number (DESIGN §23).  Importing this package neither loads the native library
nor touches CUDA; there is no CPU path.
"""
from __future__ import annotations

import numpy as np
import torch

from gaussianhaircut_b200.mesh import MeshSDF


class SDF:
    """SDF(vertices, faces): a mesh ((V,3) vertices, (F,3) vertex indices; numpy arrays or anything `np.asarray`
    accepts) prepared on the current CUDA device."""

    def __init__(self, vertices, faces):
        v = np.asarray(vertices, dtype=np.float32)
        f = np.asarray(faces)
        if v.ndim != 2 or v.shape[1] != 3 or f.ndim != 2 or f.shape[1] != 3:
            raise RuntimeError(f"SDF: vertices and faces must be (V, 3) and (F, 3), got {v.shape} and {f.shape}")
        if not np.issubdtype(f.dtype, np.integer):
            raise RuntimeError(f"SDF: faces must hold integer indices, got {f.dtype}")
        if f.size and (f.min() < 0 or f.max() >= v.shape[0]):
            raise RuntimeError(f"SDF: a face index lies outside [0, {v.shape[0]})")
        if not torch.cuda.is_available():
            raise RuntimeError("SDF: needs a CUDA device (there is no CPU path)")
        self._device = torch.device("cuda", torch.cuda.current_device())
        self._mesh = MeshSDF(torch.from_numpy(np.ascontiguousarray(v)).to(self._device),
                             torch.from_numpy(np.ascontiguousarray(f, dtype=np.int32)).to(self._device))

    def __call__(self, points):
        """(N,3) points -> (N,) float32 numpy array of signed distances (positive inside); a single (3,) point -> a
        float32 scalar."""
        p = np.asarray(points, dtype=np.float32)
        single = p.shape == (3,)
        if single:
            p = p.reshape(1, 3)
        if p.ndim != 2 or p.shape[1] != 3:
            raise RuntimeError(f"SDF: points must have shape (N, 3) or (3,), got {p.shape}")
        out = self._mesh(torch.from_numpy(np.ascontiguousarray(p)).to(self._device)).cpu().numpy()
        return out[0] if single else out
