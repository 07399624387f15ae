"""Shared helpers for the parity tests (test infrastructure)."""
from __future__ import annotations

import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

if os.path.join(ROOT, "oracle") not in sys.path:
    sys.path.insert(0, os.path.join(ROOT, "oracle"))
import synth  # noqa: E402  (oracle/synth.py: seeded scenes, cameras, the caller-preamble restatement)


def ref_module():
    """Oracle-A: the reference extension built in place under oracle/_ref (GPU only)."""
    sys.path.insert(0, os.path.join(ROOT, "oracle"))
    import build_ref
    return build_ref.load()


def ref_available() -> bool:
    sys.path.insert(0, os.path.join(ROOT, "oracle"))
    import build_ref
    return build_ref.is_built()


def _align(off: int, a: int = 128) -> int:
    return (off + a - 1) // a * a


def parse_ref_buffers(P: int, W: int, H: int, R: int, geom: torch.Tensor, binning: torch.Tensor, img: torch.Tensor):
    """Unpack the reference's three opaque byte buffers with its `obtain` arithmetic
    (rasterizer_impl.h:21-27, rasterizer_impl.cu:155-194).  Only the arrays in front of the
    CUB-sized temp regions are addressable without knowing CUB's temp size -- enough for the gates."""
    out = {}
    g = geom.cpu().numpy()
    base = geom.data_ptr()
    off = _align(base) - base
    out["depths"] = g[off:off + 4 * P].view(np.float32).copy(); off += 4 * P
    off = _align(base + off) - base; off += 3 * P                       # clamped bool[3P]
    off = _align(base + off) - base; off += 4 * P                       # internal_radii
    off = _align(base + off) - base
    out["means2D"] = g[off:off + 8 * P].view(np.float32).reshape(P, 2).copy(); off += 8 * P
    off = _align(base + off) - base; off += 24 * P                      # cov3D
    off = _align(base + off) - base
    out["conic_opacity"] = g[off:off + 16 * P].view(np.float32).reshape(P, 4).copy(); off += 16 * P
    off = _align(base + off) - base; off += 12 * P                      # rgb 3P
    off = _align(base + off) - base
    out["tiles_touched"] = g[off:off + 4 * P].view(np.uint32).copy()

    b = binning.cpu().numpy()
    base = binning.data_ptr()
    off = _align(base) - base
    out["point_list"] = b[off:off + 4 * R].view(np.uint32).copy(); off += 4 * R
    off = _align(base + off) - base; off += 4 * R                       # point_list_unsorted
    off = _align(base + off) - base
    out["keys"] = b[off:off + 8 * R].view(np.uint64).copy(); off += 8 * R

    i = img.cpu().numpy()
    base = img.data_ptr()
    N = W * H
    off = _align(base) - base
    out["final_T"] = i[off:off + 4 * N].view(np.float32).copy(); off += 4 * N
    off = _align(base + off) - base
    out["n_contrib"] = i[off:off + 4 * N].view(np.uint32).copy(); off += 4 * N
    off = _align(base + off) - base
    T = ((W + 15) // 16) * ((H + 15) // 16)
    out["ranges"] = i[off:off + 8 * T].view(np.uint32).reshape(T, 2).copy()
    return out


def settings_tuple(mod, s: dict):
    return mod.GaussianRasterizationSettings(
        image_height=s["image_height"], image_width=s["image_width"], tanfovx=s["tanfovx"], tanfovy=s["tanfovy"],
        bg=s["bg"], scale_modifier=s["scale_modifier"], viewmatrix=s["viewmatrix"], projmatrix=s["projmatrix"],
        sh_degree=s["sh_degree"], campos=s["campos"], prefiltered=s["prefiltered"], debug=s["debug"])


def native_args(inp: dict, empty_device=None):
    """The 21 positional args of `_C.rasterize_gaussians` (reference __init__.py:63-85)."""
    kw, s = inp["kwargs"], inp["settings"]
    e = torch.Tensor([])
    g = lambda k: e if kw[k] is None else kw[k]  # noqa: E731
    return (s["bg"], kw["means3D"], kw["means2D"], g("colors_precomp"), kw["opacities"], g("scales"), g("rotations"),
            s["scale_modifier"], g("cov3D_precomp"), g("conic_precomp"), s["viewmatrix"], s["projmatrix"],
            s["tanfovx"], s["tanfovy"], s["image_height"], s["image_width"], e, s["sh_degree"], s["campos"],
            s["prefiltered"], s["debug"])


def backward_args(inp: dict, radii, dL, geom, R, binning, img):
    kw, s = inp["kwargs"], inp["settings"]
    e = torch.Tensor([])
    g = lambda k: e if kw[k] is None else kw[k]  # noqa: E731
    return (s["bg"], kw["means3D"], radii, g("colors_precomp"), g("scales"), g("rotations"), s["scale_modifier"],
            g("cov3D_precomp"), g("conic_precomp"), s["viewmatrix"], s["projmatrix"], s["tanfovx"], s["tanfovy"],
            dL, e, s["sh_degree"], s["campos"], geom, R, binning, img, s["debug"])


GRAD_NAMES = ("dL_dmeans2D", "dL_dcolors", "dL_dopacity", "dL_dmeans3D", "dL_dcov3D", "dL_dconic",
              "dL_dsh", "dL_dscales", "dL_drotations")


def rel_err(a: torch.Tensor, b: torch.Tensor) -> float:
    """norm-relative error ||a-b|| / ||b|| (0 if both are zero)."""
    a = a.double().flatten(); b = b.double().flatten()
    nb = b.norm().item()
    d = (a - b).norm().item()
    if nb == 0.0:
        return 0.0 if d == 0.0 else float("inf")
    return d / nb


# ------------------------------------------------------------------ compact records of reference outputs
# The reference outputs the parity tests compare against are stored under tests/golden/ as records small enough
# to keep in the repository, whatever the size of the array:
#   digest  sha256 of the raw bytes (bit-exact comparisons),
#   norm    L2 norm, absmax, shape,
#   proj    SKETCH_K projections on pseudo-random +-1 vectors: the mean square of <r, a> - <r, ref> over the K
#           vectors estimates ||a - ref||^2 (Johnson-Lindenstrauss), i.e. the norm-relative error,
#   sample  the values at SAMPLE fixed positions (seeded by the size) plus the position of max|ref|,
#   blockmax  max|ref| over each of BLOCKS consecutive blocks of the flattened array: max|a| of every block must match
#           within the elementwise tolerance (implied by |a - ref| <= tol * max|ref| everywhere), so a few wrong
#           elements that change a block's extreme are caught wherever they are.
SKETCH_K = 16
SAMPLE = 24
BLOCKS = 64
_V_LEN = 3 + SKETCH_K + SAMPLE + 1          # norm, absmax, argmax, proj, sample (NaN padded)


def _signs(n: int, j: int, device) -> torch.Tensor:
    """+-1 vector j of length n from an integer hash of the index (the same on every device and torch version)."""
    i = torch.arange(n, dtype=torch.int64, device=device)
    h = (i * (2 * j + 0x9E3779B1) + 0x7F4A7C15 * (j + 1)) & 0xFFFFFFFF
    h = h ^ (h >> 15)
    h = (h * 0x2C1B3C6D) & 0xFFFFFFFF
    h = h ^ (h >> 12)
    return ((h >> 7) & 1).to(torch.float64) * 2.0 - 1.0


def digest(a) -> str:
    import hashlib
    if isinstance(a, torch.Tensor):
        a = a.detach().cpu().contiguous().numpy()
    a = np.ascontiguousarray(a)
    return hashlib.sha256(str(a.nbytes).encode() + a.tobytes()).hexdigest()


def _projections(x: torch.Tensor) -> np.ndarray:
    return np.array([float((x * _signs(x.numel(), j, x.device)).sum()) for j in range(SKETCH_K)])


def _sample_index(n: int, argmax: int) -> np.ndarray:
    idx = np.random.default_rng(n).choice(n, size=min(n, SAMPLE), replace=False)
    return np.unique(np.append(idx, argmax))


def _block_max(x: torch.Tensor) -> np.ndarray:
    n = x.numel()
    nb = min(BLOCKS, n)
    blk = torch.arange(n, dtype=torch.int64, device=x.device) * nb // n
    return torch.zeros(nb, dtype=x.dtype, device=x.device).scatter_reduce_(0, blk, x.abs(), "amax").cpu().numpy()


def sketch(t: torch.Tensor) -> dict:
    x = t.detach().reshape(-1).to(torch.float64)
    rec = {"digest": digest(t), "shape": tuple(t.shape)}
    if x.numel():
        am = int(x.abs().argmax())
        rec.update(norm=float(x.norm()), absmax=float(x.abs().max()), proj=_projections(x),
                   sample=x[torch.from_numpy(_sample_index(x.numel(), am)).to(x.device)].cpu().numpy(), argmax=am,
                   blockmax=_block_max(x))
    return rec


def sketch_rel_err(a: torch.Tensor, rec: dict) -> float:
    """Estimate of ||a - ref|| / ||ref|| from the record of ref (0 if both are zero)."""
    x = a.detach().reshape(-1).to(torch.float64)
    d = _projections(x) - rec["proj"]
    est = float(np.sqrt(np.mean(d * d)))
    if rec["norm"] == 0.0:
        return 0.0 if est == 0.0 and float(x.norm()) == 0.0 else float("inf")
    return est / rec["norm"]


def check_sketch(a: torch.Tensor, rec: dict, tol: float, name: str = "", elementwise: bool = True):
    """`a` against the stored record: same shape, norm-relative error <= tol and, with `elementwise`, every sampled
    element and the maximum of |a| over every block within tol * max|ref| (the tests' elementwise criterion on what is
    stored of ref)."""
    assert tuple(a.shape) == tuple(rec["shape"]), f"{name}: shape {tuple(a.shape)} vs {tuple(rec['shape'])}"
    if a.numel() == 0:
        return
    e = sketch_rel_err(a, rec)
    assert e <= tol, f"{name}: norm-relative error {e}"
    x = a.detach().reshape(-1).to(torch.float64)
    idx = _sample_index(x.numel(), int(rec["argmax"]))
    worst = float(np.max(np.abs(x[torch.from_numpy(idx).to(x.device)].cpu().numpy() - rec["sample"][:idx.size])))
    if elementwise and rec["absmax"] > 0:
        assert worst <= tol * rec["absmax"], f"{name}: elementwise error {worst / rec['absmax']} of max|ref|"
        bm = rec["blockmax"][:min(BLOCKS, x.numel())].astype(np.float64)
        bworst = float(np.max(np.abs(_block_max(x) - bm)))
        assert bworst <= tol * rec["absmax"], f"{name}: block maximum of |a| off by {bworst / rec['absmax']} of max|ref|"


def save_records(path: str, records: dict):
    """{case: {name: record or int}} -> one .npz, five arrays per case (names, digests, shapes, packed values,
    block maxima in float32)."""
    flat = {}
    for case, arrays in records.items():
        names, digests, shapes, vals, bmax = [], [], [], [], []
        for name, rec in arrays.items():
            if not isinstance(rec, dict):
                flat[f"{case}/{name}"] = np.asarray(rec)
                continue
            v = np.full(_V_LEN, np.nan)
            b = np.full(BLOCKS, np.nan, dtype=np.float32)
            if "norm" in rec:
                b[:rec["blockmax"].size] = rec["blockmax"]
                v[:3] = rec["norm"], rec["absmax"], rec["argmax"]
                v[3:3 + SKETCH_K] = rec["proj"]
                v[3 + SKETCH_K:3 + SKETCH_K + rec["sample"].size] = rec["sample"]
            names.append(name)
            digests.append(rec["digest"])
            shapes.append(",".join(str(int(d)) for d in rec.get("shape", ())) if "shape" in rec else "-")
            vals.append(v)
            bmax.append(b)
        flat[f"{case}/names"] = np.array(names, dtype="S")
        flat[f"{case}/digests"] = np.array(digests, dtype="S64")
        flat[f"{case}/shapes"] = np.array(shapes, dtype="S")
        flat[f"{case}/values"] = np.array(vals)
        flat[f"{case}/blockmax"] = np.array(bmax)
    np.savez_compressed(path, **flat)


def load_records(path: str, case: str) -> dict:
    out = {}
    with np.load(path) as z:
        keys = {k.split("/", 1)[1]: k for k in z.files if k.split("/", 1)[0] == case}
        assert keys, f"no stored reference record for {case} in {os.path.basename(path)}"
        for name, v, b in zip(z[keys["names"]], z[keys["values"]], z[keys["blockmax"]]):
            out[name.decode()] = rec = {}
            if not np.isnan(v[0]):
                rec.update(norm=float(v[0]), absmax=float(v[1]), argmax=int(v[2]), proj=v[3:3 + SKETCH_K], sample=v[3 + SKETCH_K:],
                           blockmax=b)
        for name, d, sh in zip(z[keys["names"]], z[keys["digests"]], z[keys["shapes"]]):
            out[name.decode()]["digest"] = d.decode()
            if sh != b"-":
                out[name.decode()]["shape"] = tuple(int(t) for t in sh.decode().split(",") if t)
        for k, full in keys.items():
            if k not in ("names", "digests", "shapes", "values", "blockmax"):
                out[k] = z[full].item()
    return out


def make_inputs(scene_kind: str, n: int, W: int, H: int, mode: str, cam_k: int = 0, seed: int = 0,
                opacity_mode: str = "random", device=None, **cam_kw):
    if scene_kind == "strands":
        scene = synth.make_strand_scene(n, seed=seed, opacity_mode=opacity_mode)
        strand_dir = True
    else:
        scene = synth.make_blob_scene(n, seed=seed)
        strand_dir = False
    cam = synth.make_camera(cam_k, W, H, **cam_kw)
    if not strand_dir:
        # blobs: dir feature is whatever; keep the same preamble code path
        pass
    inp = synth.rasterizer_inputs(scene, cam, mode=mode, device=device)
    return inp
