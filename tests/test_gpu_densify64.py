"""gh_densify_classify / gh_densify_scatter per element against the float64 replay of tests/_densify64.py, directly
through the C ABI with samples the test chooses and through `densify.densify_and_prune` with torch.optim.Adam and
FusedAdam: flags on every unambiguous row, the layout row by row, bit-exact copies of every tensor (row sizes 1, 3, 4
and 45) and of the kept originals' moments, exactly zero moments for clones and children, children's positions and
log-scales within the replay's bound (log-scales bit-identical to the reference's expression on the device), and NaN
where the replay has NaN.  Also `reset_opacity` against the reference's expression."""
import ctypes as C
import math
import types

import numpy as np
import pytest
import torch
from torch import nn

import _densify64 as D

pytestmark = pytest.mark.gpu

SHAPES = {"xyz": (3,), "f_dc": (1, 3), "f_rest": (15, 3), "opacity": (1,), "label": (1,), "scaling": (3,),
          "rotation": (4,), "orient_conf": (1,)}
NAMES = tuple(SHAPES)
ATTR = {"xyz": "_xyz", "f_dc": "_features_dc", "f_rest": "_features_rest", "opacity": "_opacity", "label": "_label",
        "scaling": "_scaling", "rotation": "_rotation", "orient_conf": "_orient_conf"}
PARAMS = dict(max_grad=2e-4, min_opacity=0.005, extent=100.0, max_screen_size=20.0, percent_dense=0.01)


def _inputs(P, seed, kind="mixed", specials=True):
    """float32 numpy inputs of the decisions and the child geometry for one scene."""
    g = np.random.default_rng(seed)
    ls = g.normal(0.0, 1.2, (P, 3))
    op = g.normal(-1.0, 3.0, P)
    denom = g.integers(0, 4, P).astype(np.float64)
    accum = g.uniform(0, 6e-4, P) * np.maximum(denom, 1)
    rot = g.normal(0, 1, (P, 4))
    if kind == "cold":
        accum[:] = 0.0
    elif kind in ("clone", "split", "pruned"):
        accum[:], denom[:] = 1e-2, 1.0
        ls = g.uniform(-6.0, -1.0, (P, 3)) if kind == "clone" else g.uniform(0.1, 1.5, (P, 3))
        op[:] = -30.0 if kind == "pruned" else 3.0
    elif kind == "denom_zero":
        denom[:] = 0.0
        accum[::2] = 0.0
    elif kind == "quaternions":
        accum[:], denom[:] = 1e-2, 1.0
        ls = g.uniform(0.1, 1.5, (P, 3))
        op[:] = 3.0
        for k, s in enumerate((1e-3, 1e3, 1.0, 0.0)):
            rot[k::4] *= s / np.linalg.norm(rot[k::4], axis=1, keepdims=True)
        rot[2::4, 0] = -np.abs(rot[2::4, 0])
    if specials and kind == "mixed" and P >= 32:
        rows = D.special_rows(PARAMS["max_grad"])
        idx = g.choice(P, len(rows), replace=False)
        for k, (l, o, a, d, q) in zip(idx, rows):
            ls[k], op[k], accum[k], denom[k], rot[k] = l, o, a, d, q
    f = lambda a: np.ascontiguousarray(a, dtype=np.float32)  # noqa: E731
    return dict(xyz=f(g.normal(0, 1, (P, 3))), log_scaling=f(ls), rotation=f(rot), opacity_logit=f(op), accum=f(accum),
                denom=f(denom))


def _tensors(inp, dev, seed):
    """The 8 parameter tensors (float32, device) and two non-zero moments for each."""
    P = inp["xyz"].shape[0]
    g = torch.Generator().manual_seed(seed)
    t = {n: torch.randn((P,) + SHAPES[n], generator=g) for n in NAMES}
    t["xyz"], t["scaling"], t["rotation"] = (torch.from_numpy(inp[k]) for k in ("xyz", "log_scaling", "rotation"))
    t["opacity"] = torch.from_numpy(inp["opacity_logit"])[:, None]
    t = {n: v.to(dev).contiguous() for n, v in t.items()}
    m = {n: (torch.rand(v.shape, generator=g).to(dev) + 0.5, torch.rand(v.shape, generator=g).to(dev) + 0.5) for n, v in t.items()}
    return t, m


def _bits(x):
    return x.contiguous().view(torch.int32)


def _run_kernels(t, m, inp, prm, samples_fn):
    """classify -> prefix -> samples_fn(n_split_all) -> scatter, through the C ABI.  -> flags, outputs, moments, samples."""
    from gaussianhaircut_b200 import _capi
    from gaussianhaircut_b200._capi import _ptr, _stream
    lib = _capi.load()
    dev = t["xyz"].device
    P = t["xyz"].shape[0]
    acc = torch.from_numpy(inp["accum"]).to(dev)
    den = torch.from_numpy(inp["denom"]).to(dev)
    ws = float(0.1 * prm["extent"]) if prm["max_screen_size"] else 0.0
    flags = torch.empty((P, 4), dtype=torch.int32, device=dev)
    _capi.check(lib.gh_densify_classify(P, _ptr(acc), _ptr(den), _ptr(t["scaling"]), _ptr(t["opacity"]), float(prm["max_grad"]),
                                        float(prm["percent_dense"] * prm["extent"]), float(prm["min_opacity"]), ws, _ptr(flags),
                                        _stream(dev)))
    prefix = torch.cumsum(flags.t().contiguous(), dim=1, dtype=torch.int32).t().contiguous()
    nA, nB, nC, nS = (int(v) for v in prefix[-1].tolist())
    samples = samples_fn(nS).to(dev).contiguous()
    P_new = nA + nB + 2 * nC
    out = {n: torch.full((P_new,) + SHAPES[n], float("nan"), device=dev) for n in NAMES}
    has_m = [n for n in NAMES if m.get(n) is not None]
    om = {n: (torch.full_like(out[n], float("nan")), torch.full_like(out[n], float("nan"))) for n in has_m}
    arr = lambda ts: (C.c_void_p * len(NAMES))(*[(x.data_ptr() if x is not None else None) for x in ts])  # noqa: E731
    rows = [math.prod(SHAPES[n]) for n in NAMES]
    _capi.check(lib.gh_densify_scatter(
        P, len(NAMES), arr([t[n] for n in NAMES]), arr([m[n][0] if n in om else None for n in NAMES]),
        arr([m[n][1] if n in om else None for n in NAMES]), arr([out[n] for n in NAMES]),
        arr([om[n][0] if n in om else None for n in NAMES]), arr([om[n][1] if n in om else None for n in NAMES]),
        (C.c_int * len(NAMES))(*rows), NAMES.index("xyz"), NAMES.index("scaling"), NAMES.index("rotation"),
        _ptr(flags), _ptr(prefix), nA, nB, nC, _ptr(samples), nS, _stream(dev)))
    torch.cuda.synchronize()
    return flags, out, om, samples


def _check(inp, prm, t, m, flags, out, om, samples, names=NAMES):
    """Every per-element property of the tensors `names` against the replay; returns the replay."""
    kf = flags.cpu().numpy()
    P = kf.shape[0]
    d = D.decide(inp["accum"], inp["denom"], inp["log_scaling"], inp["opacity_logit"], **prm)
    want, amb = D.flags_of(d), D.ambiguous(d)
    bad = np.nonzero((kf != want).any(axis=1) & ~amb)[0]
    assert bad.size == 0, (f"{bad.size} unambiguous rows with other flags, e.g. row {bad[0]}: kernel {kf[bad[0]].tolist()} "
                           f"replay {want[bad[0]].tolist()} (log-scale {inp['log_scaling'][bad[0]].tolist()}, "
                           f"g {d['g'][bad[0]]}, opacity logit {inp['opacity_logit'][bad[0]]})")
    rep = D.replay(inp, samples.cpu().numpy(), **prm, flags=kf)
    lay = rep["layout"]
    assert out["xyz"].shape[0] == lay["P_new"]
    dev = t["xyz"].device
    ix = lambda a: torch.from_numpy(np.ascontiguousarray(a, dtype=np.int64)).to(dev)  # noqa: E731
    o = np.nonzero(lay["dst_orig"] >= 0)[0]
    c = np.nonzero(lay["dst_clone"] >= 0)[0]
    k = rep["child_rows"]
    all_dst = np.concatenate([lay["dst_orig"][o], lay["dst_clone"][c], lay["dst_child0"][k], lay["dst_child1"][k]])
    assert np.array_equal(np.sort(all_dst), np.arange(lay["P_new"]))
    for n in names:
        w = math.prod(t[n].shape[1:])
        src = t[n].reshape(P, w)
        dst = out[n].reshape(lay["P_new"], w)
        pairs = [(lay["dst_orig"][o], o), (lay["dst_clone"][c], c)]
        if n not in ("xyz", "scaling"):
            pairs += [(lay["dst_child0"][k], k), (lay["dst_child1"][k], k)]
        for dr, sr in pairs:
            if len(dr):
                assert torch.equal(_bits(dst[ix(dr)]), _bits(src[ix(sr)])), f"{n}: a copied row differs"
        if n in om:
            for j in (0, 1):
                md, ms = om[n][j].reshape(lay["P_new"], w), m[n][j].reshape(P, w)
                if len(o):
                    assert torch.equal(_bits(md[ix(lay["dst_orig"][o])]), _bits(ms[ix(o)])), f"{n} moment {j}: kept original"
                new = np.concatenate([lay["dst_clone"][c], lay["dst_child0"][k], lay["dst_child1"][k]])
                if len(new):
                    assert int(_bits(md[ix(new)]).abs().max()) == 0, f"{n} moment {j}: clone / child moments are not +0"
    if len(k):
        msgs = D.check_children(out["xyz"].cpu().numpy(), out["scaling"].cpu().numpy(), rep)
        assert msgs == [], "\n".join(msgs)
        # scaling_inverse_activation(get_scaling[mask] / (0.8 * N)) evaluated by torch on the device
        ref_ls = torch.log(torch.exp(t["scaling"][ix(k)]) / (0.8 * 2))
        for w in ("dst_child0", "dst_child1"):
            assert torch.equal(_bits(out["scaling"][ix(lay[w][k])]), _bits(ref_ls)), "child log-scale differs from torch's"
    return rep


def _normal(seed, scale=1.0):
    def f(n):
        g = torch.Generator().manual_seed(seed)
        return torch.randn((2 * n, 3), generator=g) * scale
    return f


@pytest.mark.parametrize("P", [1, 127, 128, 129, 255, 256, 257, 1_000_003])
def test_kernels_at_block_tails(cuda_device, P):
    inp = _inputs(P, seed=P)
    t, m = _tensors(inp, cuda_device, seed=P)
    rep = _check(inp, PARAMS, t, m, *_run_kernels(t, m, inp, PARAMS, _normal(P)))
    if P >= 1000:
        lay = rep["layout"]
        assert lay["nB"] > 0 and lay["nC"] > 0 and lay["nC"] < lay["n_split_all"] and lay["nA"] < P


@pytest.mark.parametrize("kind,expect", [("cold", "none"), ("clone", "all_clone"), ("split", "all_split"), ("pruned", "empty"),
                                         ("denom_zero", None), ("quaternions", "all_split")])
def test_kernels_on_degenerate_scenes(cuda_device, kind, expect):
    P = 3000
    inp = _inputs(P, seed=11, kind=kind)
    t, m = _tensors(inp, cuda_device, seed=11)
    rep = _check(inp, PARAMS, t, m, *_run_kernels(t, m, inp, PARAMS, _normal(12)))
    lay = rep["layout"]
    got = {"none": (lay["nB"], lay["n_split_all"]) == (0, 0) and 0 < lay["nA"] < P,      # only the prune acts
           "all_clone": (lay["nA"], lay["nB"], lay["n_split_all"]) == (P, P, 0),
           "all_split": (lay["nA"], lay["nC"], lay["n_split_all"]) == (0, P, P),
           "empty": lay["P_new"] == 0 and lay["n_split_all"] == P}
    if expect is not None:
        assert got[expect], {k: lay[k] for k in ("nA", "nB", "nC", "n_split_all")}
    if kind == "quaternions":
        zero_q = np.nonzero((inp["rotation"] == 0).all(axis=1))[0]
        assert zero_q.size > 0 and np.isnan(rep["child_pos0"][np.searchsorted(rep["child_rows"], zero_q)]).all()


@pytest.mark.parametrize("samples", ["zeros", "large", "pruned_split_rows"])
def test_kernels_with_chosen_samples(cuda_device, samples):
    """Zero samples (children on the parent), samples of 1e4 (the position error is the product's), and a scene where
    most split rows are pruned, so every kept child must find its slot among ALL split rows."""
    P = 2000
    inp = _inputs(P, seed=21)
    prm = dict(PARAMS)
    if samples == "pruned_split_rows":
        prm["min_opacity"] = 0.5                      # about half the split rows lose their children
    fn = {"zeros": lambda n: torch.zeros((2 * n, 3)), "large": _normal(3, 1e4), "pruned_split_rows": _normal(4)}[samples]
    t, m = _tensors(inp, cuda_device, seed=21)
    rep = _check(inp, prm, t, m, *_run_kernels(t, m, inp, prm, fn))
    lay = rep["layout"]
    assert lay["nC"] > 0
    if samples == "pruned_split_rows":
        assert lay["n_split_all"] - lay["nC"] > lay["nC"] // 4


@pytest.mark.parametrize("max_grad,max_screen_size", [(0.0, 20.0), (2e-4, None), (2e-4, 0), (2e-4, 20.0)])
def test_kernels_thresholds(cuda_device, max_grad, max_screen_size):
    inp = _inputs(4000, seed=31)
    prm = dict(PARAMS, max_grad=max_grad, max_screen_size=max_screen_size)
    t, m = _tensors(inp, cuda_device, seed=31)
    _check(inp, prm, t, m, *_run_kernels(t, m, inp, prm, _normal(5)))


def test_kernels_without_moments_for_some_tensors(cuda_device):
    inp = _inputs(1500, seed=41)
    t, m = _tensors(inp, cuda_device, seed=41)
    for n in ("f_rest", "label", "scaling"):
        m[n] = None
    _check(inp, PARAMS, t, m, *_run_kernels(t, m, inp, PARAMS, _normal(6)))


def test_ties_and_nan_rows_are_decided_as_the_reference(cuda_device):
    """Every row on an exact tie or with a NaN input, against the hand-computed outcome (none of them is ambiguous)."""
    thr = np.float32(2e-4)
    big = math.log(20.0)
    rows = [  # log-scale, opacity logit, accum, denom, expected flags
        ([0, 0, 0], 2.0, 2 * thr, 2, [1, 1, 0, 0]),             # g = thr, smax = 1 = dense extent: cloned
        ([0, -1, -2], 0.0, 1e-2, 1, [1, 1, 0, 0]),              # sigmoid(0) = 0.5 is not < 0.5
        ([0.1, 0, 0], 2.0, 2 * thr, 2, [0, 0, 1, 1]),           # g = thr, smax > 1: split
        ([np.nan, big, big], 2.0, 1e-2, 1, [1, 0, 0, 0]),       # NaN scale: kept as it is
        ([big, np.nan, -3], 2.0, 1e-2, 1, [1, 0, 0, 0]),
        ([-3, -3, np.nan], 2.0, 1e-2, 1, [1, 0, 0, 0]),
        ([0.5, 0.5, 0.2], np.nan, 1e-2, 1, [0, 0, 1, 1]),       # NaN opacity: never pruned
        ([0.3, 0.2, 0.1], 2.0, 0.0, 0, [1, 0, 0, 0]),           # 0 / 0 -> 0
        ([0.3, 0.2, 0.1], 2.0, 1e-5, 0, [0, 0, 1, 1]),          # x / 0 = inf
        ([math.log(12.0), 0, 0], 2.0, 1e-2, 1, [0, 0, 1, 1]),   # parent over the world-size limit, children under it
        ([math.log(30.0), 0, 0], 2.0, 1e-2, 1, [0, 0, 0, 1]),   # both over it: split, nothing kept
    ]
    f = lambda a: np.asarray(a, np.float32)  # noqa: E731
    P = len(rows)
    g = np.random.default_rng(0)
    inp = dict(xyz=f(g.normal(0, 1, (P, 3))), log_scaling=f([r[0] for r in rows]), rotation=f(g.normal(0, 1, (P, 4))),
               opacity_logit=f([r[1] for r in rows]), accum=f([r[2] for r in rows]), denom=f([r[3] for r in rows]))
    prm = dict(PARAMS, min_opacity=0.5)
    t, m = _tensors(inp, cuda_device, seed=51)
    res = _run_kernels(t, m, inp, prm, _normal(7))
    assert res[0].cpu().numpy().tolist() == [r[4] for r in rows]
    d = D.decide(inp["accum"], inp["denom"], inp["log_scaling"], inp["opacity_logit"], **prm)
    assert not D.ambiguous(d).any()
    _check(inp, prm, t, m, *res)


# ------------------------------------------------------------------------------------------- densify.densify_and_prune
def _model(inp, dev, seed, fused, train_conf=True, stateless=()):
    """A GaussianModel-shaped object with an optimizer whose groups have state (one step with lr 0), except `stateless`."""
    t, _ = _tensors(inp, dev, seed)
    pc = types.SimpleNamespace(percent_dense=PARAMS["percent_dense"])
    for n in NAMES:
        setattr(pc, ATTR[n], nn.Parameter(t[n].clone()))
    groups = [{"params": [getattr(pc, ATTR[n])], "lr": 0.0, "name": n} for n in NAMES if n != "orient_conf" or train_conf]
    if fused:
        from gaussianhaircut_b200.optim import FusedAdam
        pc.optimizer = FusedAdam(groups, eps=1e-15)
    else:
        pc.optimizer = torch.optim.Adam(groups, lr=0.0, eps=1e-15)
    g = torch.Generator().manual_seed(seed + 1)
    for grp in pc.optimizer.param_groups:
        p = grp["params"][0]
        p.grad = None if grp["name"] in stateless else (torch.randn(p.shape, generator=g) * 0.01).to(dev)
    pc.optimizer.step()
    with torch.no_grad():                                  # keep the exact inputs (ties, NaN) whatever the step did
        for n in NAMES:
            getattr(pc, ATTR[n]).copy_(t[n])
    pc.xyz_gradient_accum = torch.from_numpy(inp["accum"])[:, None].to(dev)
    pc.denom = torch.from_numpy(inp["denom"])[:, None].to(dev)
    pc.max_radii2D = torch.rand(inp["xyz"].shape[0], generator=g).to(dev) * 40
    return pc


@pytest.mark.parametrize("fused,reserve,train_conf,stateless", [(False, False, True, ()), (True, False, True, ()),
                                                                (False, True, True, ()), (True, True, True, ()),
                                                                (False, False, False, ()),
                                                                (False, False, True, ("f_rest", "opacity", "scaling")),
                                                                (True, False, True, ("label", "xyz"))])
def test_densify_and_prune_per_element(cuda_device, fused, reserve, train_conf, stateless):
    from gaussianhaircut_b200 import densify
    P = 5000
    inp = _inputs(P, seed=61)
    pc = _model(inp, cuda_device, 61, fused, train_conf, stateless)
    if reserve:
        densify.reserve_pools(pc, 3 * P)
    t = {n: getattr(pc, ATTR[n]).detach().clone() for n in NAMES}
    st = {n: pc.optimizer.state.get(g["params"][0], {}) for g in pc.optimizer.param_groups for n in [g["name"]]}
    m = {n: (st[n]["exp_avg"].clone(), st[n]["exp_avg_sq"].clone()) if "exp_avg" in st.get(n, {}) else None for n in NAMES}
    args = (PARAMS["max_grad"], PARAMS["min_opacity"], PARAMS["extent"], PARAMS["max_screen_size"])
    flags = densify.classify(pc, *args)
    torch.manual_seed(77); torch.cuda.manual_seed(77)
    split = flags[:, 3] != 0
    stds = torch.exp(t["scaling"])[split].repeat(2, 1)
    samples = torch.normal(mean=torch.zeros((stds.size(0), 3), device=cuda_device), std=stds)
    torch.manual_seed(77); torch.cuda.manual_seed(77)
    counts = densify.densify_and_prune(pc, *args)
    torch.cuda.synchronize()
    by = {g["name"]: g["params"][0] for g in pc.optimizer.param_groups}
    out = {n: getattr(pc, ATTR[n]).detach() for n in NAMES}
    for n in by:
        assert by[n] is getattr(pc, ATTR[n])
    om = {n: (pc.optimizer.state[by[n]]["exp_avg"], pc.optimizer.state[by[n]]["exp_avg_sq"]) for n in by if m[n] is not None}
    for n in by:
        if m[n] is None:
            assert "exp_avg" not in pc.optimizer.state.get(by[n], {}), n
    if not train_conf:
        assert int(_bits(out["orient_conf"]).abs().max()) == 0 if out["orient_conf"].numel() else True
        out["orient_conf"] = None
    chk = {n: v for n, v in out.items() if v is not None}
    names = [n for n in NAMES if n in chk]
    rep = _check(inp, PARAMS, t, m, flags, chk, om, samples, names)
    lay = rep["layout"]
    assert counts == {"kept": lay["nA"], "cloned": lay["nB"], "split": lay["n_split_all"], "children": 2 * lay["nC"],
                      "total": lay["P_new"]}
    assert pc.xyz_gradient_accum.shape == (lay["P_new"], 1) and float(pc.denom.abs().sum()) == 0.0
    if reserve:
        assert all(p.data_ptr() in [b.data_ptr() for b in pc._gh_pools[n]] for n, p in by.items())


def test_reset_opacity_is_the_reference_expression(cuda_device):
    """GaussianModel.reset_opacity (:516-519): inverse_sigmoid(torch.min(get_opacity, ones_like * 0.01)), bit for bit,
    NaN included; the group's moments are zeroed."""
    from gaussianhaircut_b200 import densify
    inp = _inputs(4099, seed=71)
    inp["opacity_logit"][:5] = [0.0, np.nan, -np.inf, np.inf, -4.59512]      # around logit(0.01)
    pc = _model(inp, cuda_device, 71, fused=False)
    op = pc._opacity.detach().clone()
    densify.reset_opacity(pc)
    s = torch.sigmoid(op)
    m = torch.min(s, torch.ones_like(s) * 0.01)
    want = torch.log(m / (1 - m))
    assert torch.equal(_bits(pc._opacity.detach()), _bits(want))
    p = [g for g in pc.optimizer.param_groups if g["name"] == "opacity"][0]["params"][0]
    assert p is pc._opacity
    assert int(_bits(pc.optimizer.state[p]["exp_avg"]).abs().max()) == 0
    assert int(_bits(pc.optimizer.state[p]["exp_avg_sq"]).abs().max()) == 0
