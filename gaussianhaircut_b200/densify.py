"""Adaptive density control ("next" row 3 of SURVEY.md 8f): `densify_and_prune` and `reset_opacity` with the
reference's semantics (src/scene/gaussian_model.py:723-737, :516-519; called from src/train_gaussians.py:160-171),
operating IN PLACE on a GaussianModel-shaped object (its `_xyz ... _orient_conf` parameters, `optimizer`,
`xyz_gradient_accum`, `denom`, `max_radii2D`, `percent_dense`) -- a trainer replaces

    gaussians.densify_and_prune(max_grad, min_opacity, extent, max_screen_size)
by  densify.densify_and_prune(gaussians, max_grad, min_opacity, extent, max_screen_size)

The reference runs three rounds (clone, split, prune) that each rebuild every parameter and both Adam moments with
boolean-mask gathers and torch.cat and then calls torch.cuda.empty_cache(); here one classification kernel decides the
fate of every Gaussian, a prefix sum assigns final row positions, and one compaction kernel writes every parameter and
both moments exactly once, in the reference's resulting order (csrc/gh_densify.cu).  The random offsets of split
children are drawn with the SAME torch call the reference makes (torch.normal on the same shapes), so a run seeded like
the reference produces the same children -- and ranks of a data-parallel job that seed identically stay identical.
Works with torch.optim.Adam and with gaussianhaircut_b200.optim.FusedAdam (same `param_groups` / `state` surface).
"""
from __future__ import annotations

import ctypes as C
from typing import Dict, List, Optional

import torch
from torch import nn

from . import _capi
from ._capi import _ptr, _stream

# optimizer group name -> model attribute (src/scene/gaussian_model.py:431-442, :621-628)
GROUPS = {"xyz": "_xyz", "f_dc": "_features_dc", "f_rest": "_features_rest", "opacity": "_opacity", "label": "_label",
          "scaling": "_scaling", "rotation": "_rotation", "orient_conf": "_orient_conf"}


def _pool_alloc(gaussians, key: str, rows: int, tail, dev, avoid: Optional[torch.Tensor]) -> torch.Tensor:
    """(rows, *tail) float32 view of a pooled buffer.  Every tensor that densification rebuilds has two pooled buffers
    (source and destination of a compaction alternate) sized with 25% headroom, so a model that grows a little every 100
    iterations does not hit cudaMalloc each time (the reference frees and re-allocates ~25 tensors three times per call
    and then empties the allocator cache)."""
    pools = getattr(gaussians, "_gh_pools", None)
    if pools is None:
        pools = {}
        gaussians._gh_pools = pools
    per_row = 1
    for d in tail:
        per_row *= int(d)
    need = rows * per_row
    slots = pools.setdefault(key, [None, None])
    avoid_ptr = avoid.data_ptr() if avoid is not None and avoid.numel() else -1
    pick = 0
    for k in (0, 1):
        b = slots[k]
        if b is not None and b.data_ptr() == avoid_ptr:
            pick = 1 - k
            break
    b = slots[pick]
    if b is None or b.numel() < need or b.device != dev:
        b = torch.empty(int(need * 1.25) + 1024, dtype=torch.float32, device=dev)
        slots[pick] = b
    return b[:need].view((rows,) + tuple(int(d) for d in tail))


def reserve_pools(gaussians, rows: int) -> None:
    """Allocate both pooled buffers of every tensor that densification rebuilds (parameters and Adam moments) for a
    model of up to `rows` Gaussians, so that no densification of the run has to go to cudaMalloc.  Optional: without it
    the pools are created by the first two calls of `densify_and_prune` -- which costs ~0.1 s per call at 2 M Gaussians
    on one GPU and ~1.5 s once NCCL has enabled peer access between 8 GPUs (every cudaMalloc then maps the block into
    all peers), measured with tools/train_loop.py."""
    opt = gaussians.optimizer
    dev = gaussians._xyz.device
    for group in opt.param_groups:
        name = group.get("name")
        if name not in GROUPS:
            continue
        p = group["params"][0]
        for key in (name, name + ".exp_avg", name + ".exp_avg_sq"):
            a = _pool_alloc(gaussians, key, rows, p.shape[1:], dev, None)
            _pool_alloc(gaussians, key, rows, p.shape[1:], dev, a)


def classify(gaussians, max_grad: float, min_opacity: float, extent: float, max_screen_size) -> torch.Tensor:
    """(P,4) int32 flags: [original survives, its clone survives, its two children survive, it is split]."""
    lib = _capi.load()
    xyz = gaussians._xyz
    dev, P = xyz.device, int(xyz.shape[0])
    if not xyz.is_cuda:
        raise RuntimeError("gaussianhaircut_b200.densify: tensors must live on a CUDA device (no CPU path)")
    flags = torch.empty((P, 4), dtype=torch.int32, device=dev)
    if P == 0:
        return flags
    acc = gaussians.xyz_gradient_accum.detach().reshape(-1).contiguous().float()
    den = gaussians.denom.detach().reshape(-1).contiguous().float()
    if acc.numel() != P or den.numel() != P:
        raise RuntimeError("densify: xyz_gradient_accum / denom must have one entry per Gaussian")
    ws_limit = float(0.1 * extent) if max_screen_size else 0.0
    with torch.cuda.device(dev):
        _capi.check(lib.gh_densify_classify(
            P, _ptr(acc), _ptr(den), _ptr(gaussians._scaling.detach().contiguous()), _ptr(gaussians._opacity.detach().contiguous()),
            float(max_grad), float(gaussians.percent_dense * extent), float(min_opacity), ws_limit, _ptr(flags), _stream(dev)))
    return flags


def densify_and_prune(gaussians, max_grad: float, min_opacity: float, extent: float, max_screen_size,
                      empty_cache: bool = False) -> Dict[str, int]:
    """In-place equivalent of GaussianModel.densify_and_prune.  Returns the counts
    {'kept', 'cloned', 'split', 'children', 'total'} (host ints; the one device->host read of the call)."""
    lib = _capi.load()
    opt = gaussians.optimizer
    dev = gaussians._xyz.device
    P = int(gaussians._xyz.shape[0])
    flags = classify(gaussians, max_grad, min_opacity, extent, max_screen_size)
    # inclusive prefix sums of the four flag columns (a scan along the CONTIGUOUS axis: torch's scan along dim 0 of a
    # (P,4) tensor is ~50x slower)
    prefix = torch.cumsum(flags.t().contiguous(), dim=1, dtype=torch.int32).t().contiguous()
    totals = [int(v) for v in (prefix[-1].tolist() if P > 0 else [0, 0, 0, 0])]
    nA, nB, nC, n_split_all = totals
    P_new = nA + nB + 2 * nC

    # the split children's offsets: exactly the reference's draw (gaussian_model.py:690-692)
    samples = None
    if n_split_all > 0:
        split_mask = flags[:, 3] != 0
        stds = torch.exp(gaussians._scaling.detach())[split_mask].repeat(2, 1)
        means = torch.zeros((stds.size(0), 3), device=dev)
        samples = torch.normal(mean=means, std=stds).contiguous()

    # tensor table: every optimizer group (parameter + its two moments) and, when it is not optimised, orient_conf
    by_name = {g["name"]: g for g in opt.param_groups}
    names: List[str] = [n for n in GROUPS if n in by_name]
    missing = [n for n in ("xyz", "f_dc", "f_rest", "opacity", "label", "scaling", "rotation") if n not in by_name]
    if missing:
        raise RuntimeError(f"densify: optimizer has no parameter group(s) {missing}")
    srcs, m1s, m2s, rows, dsts, d1s, d2s = [], [], [], [], [], [], []
    for n in names:
        p = by_name[n]["params"][0]
        if p.shape[0] != P or p.dtype != torch.float32 or not p.is_contiguous():
            raise RuntimeError(f"densify: parameter group '{n}' must be a contiguous float32 tensor with {P} rows")
        st = opt.state.get(p, None)
        row = 1
        for d in p.shape[1:]:
            row *= int(d)
        new_p = _pool_alloc(gaussians, n, P_new, p.shape[1:], dev, p)
        srcs.append(p.detach()); rows.append(row); dsts.append(new_p)
        if st is not None and "exp_avg" in st:
            for k in ("exp_avg", "exp_avg_sq"):
                if st[k].shape != p.shape or not st[k].is_contiguous():
                    raise RuntimeError(f"densify: optimizer state '{k}' of group '{n}' does not match its parameter")
            m1s.append(st["exp_avg"]); m2s.append(st["exp_avg_sq"])
            d1s.append(_pool_alloc(gaussians, n + ".exp_avg", P_new, p.shape[1:], dev, st["exp_avg"]))
            d2s.append(_pool_alloc(gaussians, n + ".exp_avg_sq", P_new, p.shape[1:], dev, st["exp_avg_sq"]))
        else:
            m1s.append(None); m2s.append(None); d1s.append(None); d2s.append(None)
    n = len(names)
    if P > 0:
        arr = lambda ts: (C.c_void_p * n)(*[(t.data_ptr() if t is not None else None) for t in ts])   # noqa: E731
        with torch.cuda.device(dev):
            _capi.check(lib.gh_densify_scatter(
                P, n, arr(srcs), arr(m1s), arr(m2s), arr(dsts), arr(d1s), arr(d2s), (C.c_int * n)(*rows),
                names.index("xyz"), names.index("scaling"), names.index("rotation"),
                _ptr(flags), _ptr(prefix), nA, nB, nC, _ptr(samples), n_split_all, _stream(dev)))

    # install the new tensors the way the reference does (new nn.Parameter per group, state re-keyed)
    for k, nme in enumerate(names):
        group = by_name[nme]
        old = group["params"][0]
        stored = opt.state.get(old, None)
        new_param = nn.Parameter(dsts[k].requires_grad_(True))
        if stored is not None:
            if d1s[k] is not None:
                stored["exp_avg"], stored["exp_avg_sq"] = d1s[k], d2s[k]
            del opt.state[old]
            opt.state[new_param] = stored
        group["params"][0] = new_param
        setattr(gaussians, GROUPS[nme], new_param)
    if "orient_conf" not in by_name:
        # the reference replaces a non-optimised orient_conf by zeros of the new size (:629, :671)
        gaussians._orient_conf = torch.zeros((P_new, 1), dtype=torch.float32, device=dev)
    gaussians.xyz_gradient_accum = torch.zeros((P_new, 1), device=dev)
    gaussians.denom = torch.zeros((P_new, 1), device=dev)
    gaussians.max_radii2D = torch.zeros((P_new,), device=dev)
    if empty_cache:
        torch.cuda.empty_cache()          # the reference always does (:737); it stalls the allocator, so it is opt-in here
    return {"kept": nA, "cloned": nB, "split": n_split_all, "children": 2 * nC, "total": P_new}


def reset_opacity(gaussians) -> None:
    """GaussianModel.reset_opacity (src/scene/gaussian_model.py:516-519): opacity <- min(opacity, 0.01) in logit space,
    optimizer moments of the group zeroed (replace_tensor_to_optimizer :581-593)."""
    opt = gaussians.optimizer
    with torch.no_grad():
        op = torch.sigmoid(gaussians._opacity)
        new = torch.minimum(op, torch.full_like(op, 0.01))
        new = torch.log(new / (1 - new))
    for group in opt.param_groups:
        if group.get("name") == "opacity":
            old = group["params"][0]
            stored = opt.state.get(old, None)
            new_param = nn.Parameter(new.contiguous().requires_grad_(True))
            if stored is not None:
                stored["exp_avg"] = torch.zeros_like(new_param)
                stored["exp_avg_sq"] = torch.zeros_like(new_param)
                del opt.state[old]
                opt.state[new_param] = stored
            group["params"][0] = new_param
            gaussians._opacity = new_param


def add_densification_stats(gaussians, viewspace_point_tensor, update_filter) -> None:
    """GaussianModel.add_densification_stats (:739-741) with the same arithmetic, but as dense element-wise updates:
    the reference's boolean-mask indexing synchronises with the host on every call."""
    g = viewspace_point_tensor.grad
    m = update_filter.reshape(-1, 1).to(g.dtype)
    gaussians.xyz_gradient_accum += torch.norm(g[:, :2], dim=-1, keepdim=True) * m
    gaussians.denom += m


def update_max_radii(gaussians, radii) -> None:
    """`max_radii2D[vis] = max(max_radii2D[vis], radii[vis])` (src/train_gaussians.py:163) without the mask: invisible
    Gaussians have radius 0, which never raises a non-negative maximum."""
    torch.maximum(gaussians.max_radii2D, radii.to(gaussians.max_radii2D.dtype), out=gaussians.max_radii2D)
