"""Host-side mirror of the reference's native module `diff_gaussian_rasterization._C`.

Same three functions, same positional signatures, same return tuples and error behaviour as the
reference's torch/pybind binding (ext/diff_gaussian_rasterization_hair/ext.cpp:15-19,
rasterize_points.cu:35-123, :125-206, :208-227) -- but the work is done by libgh_raster.so through
its C ABI (include/gh_rasterizer.h).  PyTorch is used for device memory and the current stream only.
"""
from __future__ import annotations

import ctypes as C
from typing import Tuple

import torch

from . import _capi
from ._alloc import carve_segments, empty_rows, row_capacity, segments_floats
from ._capi import _f32 as _prep, _ptr, _stream

NUM_CHANNELS = 10  # reference cuda_rasterizer/config.h:15

# floats per Gaussian of each gradient the backward returns (rasterize_points.cu:160-168);
# they are views into ONE flat zero-filled arena so that a multi-GPU caller can all-reduce
# everything the op produced with a single collective and no packing copy.
# (rotations first: the native side stores them as one 16-byte vector per Gaussian; conic sits at a
# multiple of 4 floats per Gaussian for the same reason).  The first 21 floats per Gaussian are the
# gradients the optimizer consumes in the native call shape (scales+rotations, no conic): a multi-GPU
# caller only has to all-reduce `flat[:P * GRAD_FLOATS_TRAINABLE_NATIVE]`.  means2D follows: its gradient
# is only read for the densification statistics (per-view NORMS are accumulated, so it must not be
# summed over ranks as a gradient; dist.allreduce_densification_stats reduces the statistics instead).
# (segment padding: _alloc.segments_floats)
_GRAD_LAYOUT = tuple((k, n, (n,)) for k, n in (("rotations", 4), ("colors", NUM_CHANNELS), ("opacity", 1), ("means3D", 3),
                                                ("scales", 3), ("means2D", 3), ("conic", 4), ("cov3D", 6)))
_N_TRAINABLE_SEGMENTS = 5
GRAD_FLOATS_TRAINABLE_NATIVE = 4 + NUM_CHANNELS + 1 + 3 + 3
GRAD_FLOATS_PER_GAUSSIAN = sum(n for _, n, _ in _GRAD_LAYOUT)


def arena_floats(P: int) -> int:
    """float32 elements of the gradient arena for P Gaussians (34 * P when P % 4 == 0)."""
    return segments_floats(P, _GRAD_LAYOUT)


def trainable_floats(P: int) -> int:
    """Length of the arena prefix the optimizer consumes in the native call shape (21 * P when P % 4 == 0)."""
    return segments_floats(P, _GRAD_LAYOUT[:_N_TRAINABLE_SEGMENTS])


def rasterize_gaussians(
    background: torch.Tensor, means3D: torch.Tensor, means2D_precomp: torch.Tensor,
    colors: torch.Tensor, opacity: torch.Tensor, scales: torch.Tensor, rotations: torch.Tensor,
    scale_modifier: float, cov3D_precomp: torch.Tensor, conic_precomp: torch.Tensor,
    viewmatrix: torch.Tensor, projmatrix: torch.Tensor, tan_fovx: float, tan_fovy: float,
    image_height: int, image_width: int, sh: torch.Tensor, degree: int, campos: torch.Tensor,
    prefiltered: bool, debug: bool,
) -> Tuple[int, torch.Tensor, torch.Tensor, torch.Tensor, torch.Tensor, torch.Tensor]:
    """RasterizeGaussiansCUDA (rasterize_points.cu:35-123).

    Returns (num_rendered, out_color (C,H,W), radii (P,) int32, geomBuffer, binningBuffer, imgBuffer).
    """
    if means3D.ndim != 2 or means3D.size(1) != 3:
        raise RuntimeError("means3D must have dimensions (num_points, 3)")
    lib = _capi.load()
    device = means3D.device
    if device.type != "cuda":
        raise RuntimeError("gaussianhaircut_b200 rasterizer: tensors must live on a CUDA device (no CPU path)")
    P, H, W = int(means3D.size(0)), int(image_height), int(image_width)
    byte_opts = dict(dtype=torch.uint8, device=device)

    if P == 0:
        # reference: native call skipped, all-zero image (NOT background), R = 0 (rasterize_points.cu:86-87,122)
        return (0, torch.zeros((NUM_CHANNELS, H, W), dtype=torch.float32, device=device),
                torch.zeros((0,), dtype=torch.int32, device=device),
                torch.empty(0, **byte_opts), torch.empty(0, **byte_opts), torch.empty(0, **byte_opts))

    with torch.cuda.device(device):
        means3D = _prep(means3D, "means3D", device)
        colors = _prep(colors, "colors", device, align=8)
        opacity = _prep(opacity, "opacity", device)
        scales = _prep(scales, "scales", device)
        rotations = _prep(rotations, "rotations", device, align=16)
        cov3D_precomp = _prep(cov3D_precomp, "cov3D_precomp", device)
        conic_precomp = _prep(conic_precomp, "conic_precomp", device)
        viewmatrix = _prep(viewmatrix, "viewmatrix", device)
        projmatrix = _prep(projmatrix, "projmatrix", device)
        background = _prep(background, "background", device)
        M = int(sh.size(1)) if sh.numel() != 0 else 0

        geomBuffer, imgBuffer, radii = alloc_forward_workspaces(P, W, H, device)
        out_color = torch.empty((NUM_CHANNELS, H, W), dtype=torch.float32, device=device)
        n_rendered, max_len = C.c_int(0), C.c_int(0)
        _capi.check(lib.gh_forward_preprocess(
            P, int(degree), M, W, H,
            _ptr(means3D), _ptr(means2D_precomp), _ptr(sh), _ptr(colors), _ptr(opacity),
            _ptr(scales), float(scale_modifier), _ptr(rotations),
            _ptr(cov3D_precomp), _ptr(conic_precomp),
            _ptr(viewmatrix), _ptr(projmatrix), _ptr(campos),
            float(tan_fovx), float(tan_fovy), int(bool(prefiltered)),
            _ptr(radii), _ptr(geomBuffer), _ptr(imgBuffer),
            C.byref(n_rendered), C.byref(max_len), int(bool(debug)), _stream(device)))
        R = int(n_rendered.value)
        binningBuffer = _render(background, colors, radii, geomBuffer, imgBuffer, R, int(max_len.value), out_color, debug)
    return R, out_color, radii, geomBuffer, binningBuffer, imgBuffer


def alloc_forward_workspaces(P: int, W: int, H: int, device: torch.device):
    """(geomBuffer, imgBuffer, radii) of a forward pass, for the first phase to fill: gh_forward_preprocess
    (rasterize_gaussians) or gh_project_forward_binned (projection.project_forward_binned)."""
    lib = _capi.load()
    byte_opts = dict(dtype=torch.uint8, device=device)
    # the geometry workspace is allocated for the bucketed row capacity (see _alloc.py), so that a model that grows a
    # little keeps hitting the allocator's cached blocks; the view handed out has the size for P rows
    geom_bytes, img_bytes = [], C.c_size_t()
    for rows in (row_capacity(P), P):
        n = C.c_size_t()
        _capi.check(lib.gh_forward_workspace_sizes(rows, W, H, C.byref(n), C.byref(img_bytes)))
        geom_bytes.append(n.value)
    geomBuffer = torch.empty(geom_bytes[0], **byte_opts)[:geom_bytes[1]]
    imgBuffer = torch.empty(img_bytes.value, **byte_opts)
    radii = empty_rows(P, (), torch.int32, device)
    return geomBuffer, imgBuffer, radii


def forward_render(background: torch.Tensor, colors: torch.Tensor, radii: torch.Tensor, geomBuffer: torch.Tensor,
                   imgBuffer: torch.Tensor, num_rendered: int, max_tile_len: int, image_height: int, image_width: int,
                   debug: bool = False):
    """Second phase of the forward (emit, sort, blend) on workspaces whose first phase already ran
    (gh_forward_preprocess or gh_project_forward_binned).  -> (out_color (C,H,W), binningBuffer)."""
    device = colors.device
    with torch.cuda.device(device):
        out_color = torch.empty((NUM_CHANNELS, int(image_height), int(image_width)), dtype=torch.float32, device=device)
        binningBuffer = _render(_prep(background, "background", device), _prep(colors, "colors", device, align=8), radii,
                                geomBuffer, imgBuffer, num_rendered, max_tile_len, out_color, debug)
    return out_color, binningBuffer


def _render(background, colors, radii, geomBuffer, imgBuffer, num_rendered, max_tile_len, out_color, debug):
    """gh_forward_render into `out_color` on prepared tensors, inside their device's context -> binningBuffer.
    rasterize_gaussians calls this directly: between the first phase's read-back and this launch the GPU idles."""
    lib = _capi.load()
    device = colors.device
    H, W = int(out_color.size(1)), int(out_color.size(2))
    bin_bytes = C.c_size_t()
    _capi.check(lib.gh_binning_workspace_size(int(num_rendered), C.byref(bin_bytes)))
    binningBuffer = torch.empty(bin_bytes.value, dtype=torch.uint8, device=device)
    _capi.check(lib.gh_forward_render(
        int(colors.shape[0]), W, H, _ptr(background), _ptr(colors), _ptr(radii),
        _ptr(geomBuffer), _ptr(binningBuffer), _ptr(imgBuffer),
        int(num_rendered), int(max_tile_len), _ptr(out_color), int(bool(debug)), _stream(device)))
    return binningBuffer


def alloc_grad_arena(P: int, device: torch.device, zero: bool = True, storage: torch.Tensor | None = None):
    """One flat float32 buffer holding all per-Gaussian gradients + named (P, n) views.
    `zero=False` skips the fill: gh_backward writes every element itself.  `storage`: use (the head of)
    this float32 buffer instead of allocating, e.g. a symmetric-memory arena (dist.PeerAllReduce)."""
    n = arena_floats(P)
    if storage is not None:
        if storage.dtype != torch.float32 or storage.numel() < n or not storage.is_contiguous():
            raise RuntimeError("gradient arena storage must be a contiguous float32 tensor of at least _C.arena_floats(P) elements")
        flat = storage.view(-1)[:n]
        if zero:
            flat.zero_()
    else:
        alloc = torch.zeros if zero else torch.empty
        flat = alloc(n, dtype=torch.float32, device=device)
    return flat, carve_segments(flat, P, _GRAD_LAYOUT)


def _backward(background, means3D, radii, colors, scales, rotations, scale_modifier, cov3D_precomp, conic_precomp,
              viewmatrix, projmatrix, tan_fovx, tan_fovy, dL_dout_color, sh, degree, campos, geomBuffer, R, binningBuffer,
              imageBuffer, debug, grads=None, dL_dsh=None):
    """gh_backward on prepared tensors (P > 0), arguments in the order of rasterize_gaussians_backward.  `grads`: the
    alloc_grad_arena views that receive every per-Gaussian gradient; None leaves the blend's accumulation records in
    `geomBuffer` (records mode, conic_precomp call shape).

    Under `torch.use_deterministic_algorithms(True)` the deterministic blend backward runs (fixed summation order:
    bit-reproducible gradients, slower); otherwise the fast path, whose float sums depend on GPU scheduling."""
    device = means3D.device
    P = int(means3D.size(0))
    M = int(sh.size(1)) if sh is not None and sh.numel() != 0 else 0
    H, W = int(dL_dout_color.size(1)), int(dL_dout_color.size(2))
    g = grads or {}
    lib = _capi.load()
    det_buffer, det_bytes = None, 0
    if torch.are_deterministic_algorithms_enabled():
        n = C.c_size_t()
        _capi.check(lib.gh_backward_det_workspace_size(P, int(R), C.byref(n)))
        det_buffer, det_bytes = torch.empty(n.value, dtype=torch.uint8, device=device), n.value
    with torch.cuda.device(device):
        _capi.check(lib.gh_backward(
            P, int(degree), M, int(R), W, H,
            _ptr(background), _ptr(means3D), _ptr(sh), _ptr(colors),
            _ptr(scales), float(scale_modifier), _ptr(rotations),
            _ptr(cov3D_precomp), _ptr(conic_precomp),
            _ptr(viewmatrix), _ptr(projmatrix), _ptr(campos),
            float(tan_fovx), float(tan_fovy), _ptr(radii),
            _ptr(geomBuffer), _ptr(binningBuffer), _ptr(imageBuffer),
            _ptr(dL_dout_color),
            _ptr(g.get("means2D")), _ptr(g.get("conic")), _ptr(g.get("opacity")), _ptr(g.get("colors")),
            _ptr(g.get("means3D")), _ptr(g.get("cov3D")), _ptr(dL_dsh), _ptr(g.get("scales")), _ptr(g.get("rotations")),
            int(bool(debug)), _stream(device), _ptr(det_buffer), det_bytes))


def rasterize_gaussians_backward_arena(
    background, means3D, radii, colors, scales, rotations, scale_modifier, cov3D_precomp, conic_precomp,
    viewmatrix, projmatrix, tan_fovx, tan_fovy, dL_dout_color, sh, degree, campos,
    geomBuffer, R, binningBuffer, imageBuffer, debug, arena_storage=None,
):
    """Same work as `rasterize_gaussians_backward`, but returns (flat_arena, views, dL_dsh): every
    per-Gaussian gradient is a (P, n) view into ONE flat float32 buffer, which is what a multi-GPU
    caller all-reduces (one collective per step, no packing copy).  `arena_storage` places the arena
    in caller-owned memory (a symmetric-memory buffer for dist.PeerAllReduce)."""
    device = means3D.device
    P = int(means3D.size(0))
    M = int(sh.size(1)) if sh.numel() != 0 else 0
    flat, g = alloc_grad_arena(P, device, zero=False, storage=arena_storage)     # gh_backward writes every element
    dL_dsh = torch.zeros((P, M, 3), dtype=torch.float32, device=device)
    if P != 0:
        _backward(_prep(background, "background", device), _prep(means3D, "means3D", device), radii.contiguous(),
                  _prep(colors, "colors", device, align=8), _prep(scales, "scales", device),
                  _prep(rotations, "rotations", device, align=16), scale_modifier,
                  _prep(cov3D_precomp, "cov3D_precomp", device), _prep(conic_precomp, "conic_precomp", device),
                  _prep(viewmatrix, "viewmatrix", device), _prep(projmatrix, "projmatrix", device), tan_fovx, tan_fovy,
                  _prep(dL_dout_color, "dL_dout_color", device), sh, degree, campos, geomBuffer, R, binningBuffer,
                  imageBuffer, debug, g, dL_dsh)
    return flat, g, dL_dsh


def rasterize_gaussians_backward_records(background, means3D, radii, colors, conic_precomp, viewmatrix, projmatrix,
                                         tan_fovx, tan_fovy, dL_dout_color, campos, geomBuffer, R, binningBuffer,
                                         imageBuffer, debug) -> None:
    """Blend backward only, for the conic_precomp call shape: the per-Gaussian accumulation records (dL/d colour,
    2-D mean, conic, opacity) are LEFT in `geomBuffer` for `gh_project_backward` to consume directly -- no unpack
    pass, no intermediate gradient tensors (projection.project_backward(geom_buffer=...))."""
    if int(means3D.size(0)) == 0:
        return
    if conic_precomp is None or conic_precomp.numel() == 0:
        raise RuntimeError("rasterize_gaussians_backward_records needs the conic_precomp call shape")
    _backward(background, means3D, radii, colors, None, None, 1.0, None, conic_precomp, viewmatrix, projmatrix,
              tan_fovx, tan_fovy, _prep(dL_dout_color, "dL_dout_color", means3D.device), None, 0, campos,
              geomBuffer, R, binningBuffer, imageBuffer, debug)


def rasterize_gaussians_backward(
    background: torch.Tensor, means3D: torch.Tensor, radii: torch.Tensor, colors: torch.Tensor,
    scales: torch.Tensor, rotations: torch.Tensor, scale_modifier: float,
    cov3D_precomp: torch.Tensor, conic_precomp: torch.Tensor,
    viewmatrix: torch.Tensor, projmatrix: torch.Tensor, tan_fovx: float, tan_fovy: float,
    dL_dout_color: torch.Tensor, sh: torch.Tensor, degree: int, campos: torch.Tensor,
    geomBuffer: torch.Tensor, R: int, binningBuffer: torch.Tensor, imageBuffer: torch.Tensor,
    debug: bool,
):
    """RasterizeGaussiansBackwardCUDA (rasterize_points.cu:125-206).

    Returns (dL_dmeans2D (P,3), dL_dcolors (P,C), dL_dopacity (P,1), dL_dmeans3D (P,3), dL_dcov3D (P,6),
    dL_dconic (P,2,2), dL_dsh (P,M,3), dL_dscales (P,3), dL_drotations (P,4)).
    """
    _flat, g, dL_dsh = rasterize_gaussians_backward_arena(
        background, means3D, radii, colors, scales, rotations, scale_modifier, cov3D_precomp, conic_precomp,
        viewmatrix, projmatrix, tan_fovx, tan_fovy, dL_dout_color, sh, degree, campos,
        geomBuffer, R, binningBuffer, imageBuffer, debug)
    P = int(means3D.size(0))
    return (g["means2D"], g["colors"], g["opacity"], g["means3D"], g["cov3D"],
            g["conic"].view(P, 2, 2), dL_dsh, g["scales"], g["rotations"])


def mark_visible(means3D: torch.Tensor, viewmatrix: torch.Tensor, projmatrix: torch.Tensor) -> torch.Tensor:
    """markVisible (rasterize_points.cu:208-227): bool (P,) -- near-plane test only."""
    lib = _capi.load()
    device = means3D.device
    P = int(means3D.size(0))
    present = torch.zeros((P,), dtype=torch.bool, device=device)
    if P != 0:
        with torch.cuda.device(device):
            means3D = _prep(means3D, "means3D", device)
            viewmatrix = _prep(viewmatrix, "viewmatrix", device)
            projmatrix = _prep(projmatrix, "projmatrix", device)
            _capi.check(lib.gh_mark_visible(P, _ptr(means3D), _ptr(viewmatrix), _ptr(projmatrix),
                                            _ptr(present), _stream(device)))
    return present


def debug_export(P: int, W: int, H: int, R: int, geomBuffer, binningBuffer, imgBuffer):
    """Parity-test helper: unpack the opaque workspaces into reference-shaped arrays
    (keys, point_list, ranges, final_T, n_contrib, depths, means2D, conic_opacity)."""
    lib = _capi.load()
    device = geomBuffer.device
    T = ((W + 15) // 16) * ((H + 15) // 16)
    out = {
        "keys": torch.zeros(R, dtype=torch.int64, device=device),
        "point_list": torch.zeros(R, dtype=torch.int32, device=device),
        "ranges": torch.zeros((T, 2), dtype=torch.int32, device=device),
        "final_T": torch.zeros(H * W, dtype=torch.float32, device=device),
        "n_contrib": torch.zeros(H * W, dtype=torch.int32, device=device),
        "depths": torch.zeros(P, dtype=torch.float32, device=device),
        "means2D": torch.zeros((P, 2), dtype=torch.float32, device=device),
        "conic_opacity": torch.zeros((P, 4), dtype=torch.float32, device=device),
    }
    with torch.cuda.device(device):
        _capi.check(lib.gh_debug_export(
            P, W, H, R, _ptr(geomBuffer), _ptr(binningBuffer), _ptr(imgBuffer),
            _ptr(out["keys"]), _ptr(out["point_list"]), _ptr(out["ranges"]),
            _ptr(out["final_T"]), _ptr(out["n_contrib"]),
            _ptr(out["depths"]), _ptr(out["means2D"]), _ptr(out["conic_opacity"]), _stream(device)))
    return out
