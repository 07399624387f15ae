"""The float64 replay of the projection kernels (tests/_project64.py) and its error bounds, proven without a GPU.

* The replay's values, with the reference's float64 constants, against float64 autograd of oracle/synth.py
  `project_reference` (itself pinned on the reference's Python by test_project_cpu.py): every output and every
  gradient element, camera gradients included, for both model flavours, SH degrees 0-3, every activation code and
  the strand form.
* The product's per-Gaussian arithmetic compiled for the host (tests/host_harness/project_host.cpp,
  strand_host.cpp: the very header the kernels call) lies within the replay's bound on every element and agrees
  with every decided branch: the same scenes the GPU test (test_gpu_project64.py) hands to the kernels, smaller.
* Hand-built rows at each decision edge take the decision they were built for."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import _project64 as p64

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "oracle"))
import synth  # noqa: E402

MATH_H = os.path.join(ROOT, "gaussianhaircut_b200", "csrc", "gh_project_math.h")
# unresolved elements (bound above 2^-10 of the value) allowed per case, as a fraction of the elements checked: the
# quaternion and scale gradients of un-normalised quaternions cancel on a few percent of their elements
UNRESOLVED_CAP = 0.05


def _harness(name):
    src = os.path.join(ROOT, "tests", "host_harness", f"{name}.cpp")
    so = os.path.join(ROOT, "tests", "host_harness", f"lib{name}.so")
    if not os.path.isfile(so) or os.path.getmtime(so) < max(os.path.getmtime(src), os.path.getmtime(MATH_H)):
        subprocess.run(["g++", "-O2", "-shared", "-fPIC", "-std=c++17", "-w", src, "-o", so], check=True)
    return C.CDLL(so)


@pytest.fixture(scope="module")
def host():
    return {"project": _harness("project_host"), "strand": _harness("strand_host")}


def _flags(cfg):
    from gaussianhaircut_b200.projection import encode_flags
    return encode_flags(cfg)


def _ptr(a):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


def _f(a, *shape):
    return None if a is None else np.ascontiguousarray(np.asarray(a, np.float32).reshape(*shape))


def run_host(host, sc, gi=None):
    """the header compiled for the host: forward, and with `gi` (p64.random_grads layout) the backward of the rows it
    found visible -> (forward dict, backward dict, d_camera (37,))"""
    P, cam, cfg = sc["P"], sc["cam"], sc["cfg"]
    strand = bool(cfg.get("strands"))
    xyz, dirs, fdc, rest, conf = _f(sc["xyz"], P, 3), _f(sc["dirs"], P, 3), _f(sc["f_dc"], P, 3), _f(sc["f_rest"], P, 45), _f(sc["conf"], P)
    head = (P, cam["W"], cam["H"], _ptr(xyz))
    tail = (_ptr(_f(cam["V"], 16)), _ptr(_f(cam["Pm"], 16)), _ptr(_f(cam["campos"], 3)), C.c_float(cam["tanx"]), C.c_float(cam["tany"]),
            C.c_float(sc["mod"]), sc["deg"], C.c_uint(_flags(cfg)), C.c_float(cfg["det_eps"]))
    keep = [xyz, dirs, fdc, rest, conf]
    if strand:
        scale = _f(sc["scaling"], 1)
        keep.append(scale)
        mid = (_ptr(scale), _ptr(dirs), _ptr(fdc), _ptr(rest), _ptr(conf))
        lib_f, lib_b = host["strand"].gh_host_strand_forward, host["strand"].gh_host_strand_backward
    else:
        sc_, rot, op, lab = _f(sc["scaling"], P, 3), _f(sc["rotation"], P, 4), _f(sc["opacity"], P), _f(sc["label"], P)
        keep += [sc_, rot, op, lab]
        mid = (_ptr(sc_), _ptr(rot), _ptr(dirs), _ptr(fdc), _ptr(rest), _ptr(op), _ptr(lab), _ptr(conf))
        lib_f, lib_b = host["project"].gh_host_project_forward, host["project"].gh_host_project_backward
    out = {"means2D": np.zeros((P, 3), np.float32), "colors": np.zeros((P, 10), np.float32), "opacity": np.zeros(P, np.float32),
           "conic": np.zeros((P, 3), np.float32), "cov3D": np.zeros((P, 6), np.float32), "visible": np.zeros(P, np.uint8)}
    lib_f(*head, *mid, *tail, *(_ptr(out[k]) for k in ("means2D", "colors", "opacity", "conic", "cov3D", "visible")))
    out["visible"] = out["visible"].astype(bool)
    if gi is None:
        return out, None, None
    m2 = np.zeros((P, 3), np.float32); m2[:, 0] = gi["m2x"]; m2[:, 1] = gi["m2y"]
    con, col, op_g = _f(gi["con"], P, 3), _f(gi["color"], P, 10), _f(gi["opacity"], P)
    d = {k: np.zeros((P, n), np.float32) for k, n in (("xyz", 3), ("scaling", 3), ("rotation", 4), ("dirs", 3), ("f_dc", 3),
                                                      ("rest", 45), ("opacity", 1), ("label", 1), ("conf", 1))}
    cam29 = np.zeros(29)
    vis8 = out["visible"].astype(np.uint8)
    if strand:
        sr = np.zeros((P, 7), np.float32)
        lib_b(*head, *mid, *tail, _ptr(vis8), _ptr(m2), _ptr(con), _ptr(col), _ptr(d["xyz"]), _ptr(d["dirs"]), _ptr(d["f_dc"]),
              _ptr(d["rest"]), _ptr(d["conf"]), _ptr(sr), _ptr(cam29))
        assert not sr.any(), "the strand form leaves scaling / rotation gradients at zero"
        for k in ("scaling", "rotation", "opacity", "label"):
            d[k] = None
    else:
        lib_b(*head, *mid, *tail, _ptr(vis8), _ptr(m2), _ptr(con), _ptr(col), _ptr(op_g), *(_ptr(d[k]) for k in
              ("xyz", "scaling", "rotation", "dirs", "f_dc", "rest", "opacity", "label", "conf")), _ptr(cam29))
    return out, d, p64.cam37(cam29)


def replay_and_check(sc, got_f, got_b=None, cam_got=None, gi=None):
    """the replay of scene `sc` against forward (and backward) outputs -> (Replay, Stats)"""
    A = p64.inputs(sc)
    rp = p64.Replay(A.P)
    o, g = p64.forward(rp, A)
    stats = p64.Stats()
    p64.check_forward(rp, o, got_f, stats, A.P)
    if got_b is not None:
        go, cam = p64.backward(rp, A, gi, got_f["visible"], g)
        p64.check_backward(rp, go, cam, got_b, stats, A.P, cam_got)
    return rp, stats


def _report(name, rp, stats):
    amb = {k: int(v.sum()) for k, v in rp.amb.items() if v.any()}
    print(f"\n[{name}] ambiguous {amb or 0}, unresolved rows {int(rp.unres.sum())}, "
          f"unresolved elements {stats.unresolved_fraction():.2e}\n  {stats}")
    assert stats.unresolved_fraction() <= UNRESOLVED_CAP, f"{name}: too many unresolved elements"


def test_build_keeps_division_and_sqrt_correctly_rounded():
    """the bound's model of `/` and sqrtf (correctly rounded) and of denormals (kept) holds only without these"""
    from gaussianhaircut_b200 import build
    flags = " ".join(build.NVCC_FLAGS)
    for bad in ("fast_math", "prec-div=false", "prec_div=false", "prec-sqrt=false", "prec_sqrt=false", "ftz=true"):
        assert bad not in flags, bad


# ------------------------------------------------------------------------------------- replay vs float64 autograd
def _torch_case(sc):
    t = lambda a: None if a is None else torch.from_numpy(np.asarray(a, np.float32).astype(np.float64))  # noqa: E731
    P = sc["P"]
    raw = {"xyz": t(sc["xyz"]), "f_dc": t(sc["f_dc"]).reshape(P, 1, 3), "f_rest": t(sc["f_rest"]).reshape(P, 15, 3),
           "opacity": t(sc["opacity"]).reshape(P, 1), "label": t(sc["label"]).reshape(P, 1), "conf": t(sc["conf"]).reshape(P, 1),
           "dirs": t(sc["dirs"])}
    if not sc["cfg"].get("strands"):
        raw.update(scaling=t(sc["scaling"]), rotation=t(sc["rotation"]))
    c = sc["cam"]
    cam = {"image_width": c["W"], "image_height": c["H"], "world_view_transform": t(c["V"]).requires_grad_(True),
           "full_proj_transform": t(c["Pm"]).requires_grad_(True), "camera_center": t(c["campos"]).requires_grad_(True),
           "tanfovx": torch.tensor(c["tanx"], dtype=torch.float64, requires_grad=True),
           "tanfovy": torch.tensor(c["tany"], dtype=torch.float64, requires_grad=True)}
    return raw, cam


def _close(name, a, b, tol=1e-11):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    a, b = a.reshape(a.shape[0], -1) if a.ndim else a.reshape(1, 1), b.reshape(b.shape[0], -1) if b.ndim else b.reshape(1, 1)
    scale = np.maximum(np.abs(b).max(axis=1, keepdims=True), 1e-300)
    err = np.abs(a - b) / scale
    assert err.max() <= tol, f"{name}: {err.max():.3g} at row {np.unravel_index(err.argmax(), err.shape)}"


AUTOGRAD_CASES = [("gaussian_model", d) for d in range(4)] + [("hair", 3), ("head", 2), ("identity", 1), ("strands", 3)]


@pytest.mark.parametrize("cfg_name,deg", AUTOGRAD_CASES)
def test_replay_matches_float64_autograd(cfg_name, deg):
    sc = p64.random_scene(300, 21 + deg, cfg_name, deg=deg, mod=1.0 if cfg_name == "strands" else 0.8)
    P, cfg = sc["P"], sc["cfg"]
    raw, cam = _torch_case(sc)
    leaves = {k: v.clone().requires_grad_(True) for k, v in raw.items() if v is not None}
    inp = dict(leaves)
    ref_cfg = dict(cfg)
    if cfg.get("strands"):
        d = leaves["dirs"]
        scale = float(np.float32(sc["scaling"][0]))
        inp["scaling"] = torch.cat([d.norm(dim=-1, keepdim=True) * 0.5, torch.full_like(d[:, :2], scale)], dim=-1)
        ex = torch.cat([torch.ones_like(d[:, :1]), torch.zeros_like(d[:, :2])], dim=-1)
        inp["rotation"] = synth.parallel_transport(ex, d)
        ref_cfg.pop("strands")
    ref = synth.project_reference(inp, cam, ref_cfg, sh_degree=deg, scaling_modifier=float(np.float32(sc["mod"])))
    A = p64.inputs(sc)
    rp = p64.Replay(P, f32=False)
    o, g = p64.forward(rp, A)
    mask = ref["mask"].numpy()
    st = lambda es: np.stack([np.broadcast_to(e.v, (P,)) for e in es], -1)  # noqa: E731
    _close("means2D", st(o["means2D"]), ref["means2D"].detach())
    _close("conic", st(o["conic"])[mask], ref["conic"].detach()[mask])
    _close("colors", st(o["color"]), ref["colors"].detach())
    _close("opacity", np.broadcast_to(o["opacity"].v, (P,)), ref["opacity"].detach().reshape(P))
    _close("cov3D", st(o["cov3D"]), ref["cov3D"].detach())
    if not (rp.rows("vis").any()):
        assert np.array_equal(o["visible"], mask)

    gi = p64.random_grads(P, 5)
    m = torch.from_numpy(mask)[:, None].double()
    m2 = torch.zeros(P, 3, dtype=torch.float64)
    m2[:, 0] = torch.from_numpy(gi["m2x"].astype(np.float64)); m2[:, 1] = torch.from_numpy(gi["m2y"].astype(np.float64))
    g64 = lambda a: torch.from_numpy(np.asarray(a, np.float32).astype(np.float64))  # noqa: E731
    loss = (ref["means2D"] * m2 * m).sum() + (ref["conic"] * g64(gi["con"]) * m).sum() + (ref["colors"] * g64(gi["color"]) * m).sum()
    if ref["opacity"].requires_grad:
        loss = loss + (ref["opacity"] * g64(gi["opacity"])[:, None] * m).sum()
    loss.backward()
    go, camr = p64.backward(rp, A, gi, mask, g)
    names = {"xyz": "xyz", "f_dc": "f_dc", "rest": "f_rest", "conf": "conf"}
    names.update({"dirs": "dirs"} if cfg["dir_mode"] == 1 else {})
    if not cfg.get("strands"):
        names.update(scaling="scaling", rotation="rotation", opacity="opacity", label="label")
    for key, leaf in names.items():
        gref = leaves[leaf].grad
        gref = torch.zeros_like(leaves[leaf]) if gref is None else gref
        val = go[key] if isinstance(go[key], list) else [go[key]]
        _close("d_" + key, st(val), gref.reshape(P, -1))
    cam_v = np.array([float(np.sum(e.v)) for e in camr])
    c37 = p64.cam37(cam_v)
    gr = lambda t: (torch.zeros_like(t) if t.grad is None else t.grad).reshape(-1)  # noqa: E731
    cref = torch.cat([gr(cam["world_view_transform"]), gr(cam["full_proj_transform"]), gr(cam["camera_center"]),
                      gr(cam["tanfovx"]), gr(cam["tanfovy"])]).detach()
    for name, sl in (("d_V", slice(0, 16)), ("d_Pm", slice(16, 32)), ("d_campos", slice(32, 35)), ("d_tan", slice(35, 37))):
        _close(name, c37[sl][None], cref[sl].numpy()[None])


# ------------------------------------------------------------------------------------- the host build within the bound
HOST_CASES = {
    "gaussian_model": lambda: p64.random_scene(20000, 1, "gaussian_model", deg=3),
    "gaussian_model_deg1_mod": lambda: p64.random_scene(5000, 2, "gaussian_model", deg=1, mod=0.7),
    "hair": lambda: p64.random_scene(20000, 3, "hair", deg=3),
    "head": lambda: p64.random_scene(5000, 4, "head", deg=0),
    "identity": lambda: p64.random_scene(5000, 5, "identity", deg=2),
    "strands": lambda: p64.random_scene(20000, 6, "strands", deg=3),
    "strand_edges": p64.strand_edge_scene,
    "edges": lambda: p64.edge_scene()[0],
}


@pytest.mark.parametrize("case", sorted(HOST_CASES))
def test_host_build_lies_within_the_bound(host, case):
    sc = HOST_CASES[case]()
    out, _, _ = run_host(host, sc)
    A = p64.inputs(sc)
    rp0 = p64.Replay(A.P)
    p64.forward(rp0, A)
    gi = p64.neutralize(rp0, p64.random_grads(sc["P"], 9))
    _, d, cam = run_host(host, sc, gi)
    rp, stats = replay_and_check(sc, out, d, cam, gi)
    _report(case, rp, stats)


def test_edge_rows_take_the_decision_they_were_built_for(host):
    sc, rows = p64.edge_scene()
    A = p64.inputs(sc)
    rp = p64.Replay(A.P)
    o, g = p64.forward(rp, A)
    for key, m in rp.amb.items():
        assert not m.any(), f"{key} ambiguous on edge rows {[n for n, r in rows.items() if m[r]]}"
    vis = {n: bool(o["visible"][r]) for n, r in rows.items()}
    assert not vis["near_below"] and not vis["near_on"] and vis["near_above"] and not vis["behind"]
    for n, r in rows.items():
        if n.startswith("clamp_"):
            ax = n[6]
            clamped = (g.clx if ax == "x" else g.cly)[r]
            assert vis[n] and clamped == n.endswith("_out"), n
            assert not (g.cly if ax == "x" else g.clx)[r], n
        if n.startswith("tile_"):
            assert vis[n] == n.endswith("_in"), n
        if n.startswith("needle"):
            assert vis[n], n
    assert g.jm[rows["tie01"]] == 0 and g.jm[rows["tie12"]] == 1 and g.jm[rows["tie012"]] == 0 and g.jm[rows["tie_after_mod"]] == 0
    s = sc["scaling"][rows["tie_after_mod"]]
    assert s[0] != s[1] and np.float32(s[0] * np.float32(sc["mod"])) == np.float32(s[1] * np.float32(sc["mod"]))
    # and the host build agrees on every one of them
    out, _, _ = run_host(host, sc)
    assert np.array_equal(out["visible"], o["visible"])


def test_colour_clamp_keeps_its_gradient_at_exactly_zero(host):
    """max(acc + 0.5, 0) passes the gradient at acc + 0.5 == 0 (torch.clamp_min), not one step below"""
    sc, accs, kk, B = p64.colour_tie_scene()
    assert accs[0] == -0.5 and accs[1] > -0.5 > accs[2]
    gi = p64.random_grads(sc["P"], 3)
    gi["color"][:] = 1.0
    out, d, _ = run_host(host, sc, gi)
    check_colour_tie(out, d, kk, B)


def check_colour_tie(out, d, kk, B):
    assert np.asarray(out["visible"]).all()
    rest = np.asarray(d["rest"]).reshape(-1, 45)
    fdc = np.asarray(d["f_dc"]).reshape(-1, 3)
    C0 = np.float32(p64.SH_C0)
    for row in range(rest.shape[0]):
        assert np.array_equal(rest[row, 3 * (kk - 1):3 * kk], [B, B, 0.0]), rest[row, 3 * (kk - 1):3 * kk]
        assert np.array_equal(fdc[row], [C0, C0, 0.0]), fdc[row]


# ------------------------------------------------------------------------------------- strand geometry kernels
def test_strand_replays_bound_float32_evaluations():
    """gh_strands.cu's midpoints (in segment order) and suffix-sum backward, evaluated in float32 numpy in the
    kernels' orders, lie within the replay's bounds"""
    rng = np.random.default_rng(4)
    S, L = 40, 100
    origins = rng.normal(0, 0.2, (S, 3)).astype(np.float32)
    dirs = (rng.normal(0, 1, (S, L, 3)) * 4e-3).astype(np.float32)
    v, e = p64.strand_midpoints(origins, dirs)
    acc = np.zeros((S, 3), np.float32)
    prev = origins + np.float32(0)
    for k in range(L):
        acc = acc + dirs[:, k]
        p = origins + acc
        m = (p + prev) * np.float32(0.5)
        assert np.all(np.abs(m - v[:, k]) <= e[:, k])
        prev = p
    gx = rng.normal(size=(S, L, 3)).astype(np.float32)
    direct = rng.normal(size=(S, L, 3)).astype(np.float32)
    v, e = p64.strand_backward(gx, direct)
    carry = np.zeros((S, 3), np.float32)
    for k in range(L - 1, -1, -1):
        t = (direct[:, k] + np.float32(0.5) * gx[:, k]) + carry
        assert np.all(np.abs(t - v[:, k]) <= e[:, k])
        carry = carry + gx[:, k]
