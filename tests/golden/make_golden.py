"""Generate the golden vectors under tests/golden/ by RUNNING THE REFERENCE ITSELF.

The reference ships no tests, golden outputs or fixtures for this path (SURVEY.md section 4), so the
vectors are produced by Oracle-A -- the reference extension compiled in place from
/root/reference/ext/diff_gaussian_rasterization_hair (oracle/build_ref.py) -- executed on a GPU:

    python tests/golden/make_golden.py OUT_DIR          (on a GPU)

and then copied into tests/golden/.  Each .npz holds the exact argument tuple of the reference's
native `_C.rasterize_gaussians` / `_C.rasterize_gaussians_backward` calls (the reference's own
snapshot format, __init__.py:63-85,114-135) together with everything it returned, including the
contents of its opaque workspaces unpacked with its `obtain` layout (rasterizer_impl.cu:155-194).
The CPU tests pin oracle/ (the C restatement) against these files.
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import _util  # noqa: E402

CASES = [
    # name, scene, n, W, H, mode, opacity_mode, cam_k
    ("strands_native", "strands", 12, 96, 64, "native", "random", 3),
    ("strands_render", "strands", 12, 96, 64, "render", "random", 11),
    ("strands_render_hair", "strands", 12, 100, 70, "render_hair", "ones", 20),
    ("strands_cov3d", "strands", 12, 96, 64, "cov3d", "random", 40),
    ("blobs_native", "blobs", 500, 80, 48, "native", "random", 7),
]


def to_np(t):
    if isinstance(t, torch.Tensor):
        return t.detach().cpu().numpy()
    return np.asarray(t)


def main(outdir):
    os.makedirs(outdir, exist_ok=True)
    dev = torch.device("cuda:0")
    ref = _util.ref_module()._C
    for name, scene, n, W, H, mode, opm, cam_k in CASES:
        inp = _util.make_inputs(scene, n, W, H, mode, cam_k=cam_k, opacity_mode=opm, device=dev)
        args = _util.native_args(inp)
        R, color, radii, geom, binning, img = ref.rasterize_gaussians(*args)
        P = inp["kwargs"]["means3D"].shape[0]
        state = _util.parse_ref_buffers(P, W, H, R, geom, binning, img)
        dL = _util.synth.upstream_gradient(W, H, 5).to(dev)
        grads = ref.rasterize_gaussians_backward(*_util.backward_args(inp, radii, dL, geom, R, binning, img))
        torch.cuda.synchronize()
        kw, s = inp["kwargs"], inp["settings"]
        blob = {
            "mode": np.array(mode), "W": np.array(W), "H": np.array(H), "P": np.array(P), "R": np.array(R),
            "tanfovx": np.array(s["tanfovx"], dtype=np.float64), "tanfovy": np.array(s["tanfovy"], dtype=np.float64),
            "scale_modifier": np.array(s["scale_modifier"], dtype=np.float64),
            "bg": to_np(s["bg"]), "viewmatrix": to_np(s["viewmatrix"]), "projmatrix": to_np(s["projmatrix"]),
            "campos": to_np(s["campos"]), "prefiltered": np.array(bool(s["prefiltered"])),
            "dL_dout": to_np(dL),
            "out_color": to_np(color), "radii": to_np(radii),
        }
        for k in ("means3D", "means2D", "opacities", "colors_precomp", "scales", "rotations", "cov3D_precomp", "conic_precomp"):
            blob["in_" + k] = to_np(kw[k]) if kw[k] is not None else np.zeros((0,), dtype=np.float32)
        for k, v in state.items():
            blob["st_" + k] = v
        for nm, g in zip(_util.GRAD_NAMES, grads):
            blob["g_" + nm] = to_np(g)
        path = os.path.join(outdir, name + ".npz")
        np.savez_compressed(path, **blob)
        print(name, "P", P, "R", R, "->", path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main(sys.argv[1])
