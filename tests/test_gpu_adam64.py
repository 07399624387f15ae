"""GPU tests of the Adam kernels per element against the float64 replay of torch.optim.Adam (tests/_adam64.py):
gh_adam_step and gh_adam_step_capturable through optim.FusedAdam, gh_camera_adam_step through cameras.CameraAdam.
Every check starts from the kernel's own pre-step state (p, g, m, v and the step count).

The bound.  tests/test_adam64_cpu.py pins the replay to torch's float32 step: within 2 of its error units on both of
torch's paths.  The kernels compute, per element (gh_adam_math.cuh),
    m' = fma(w1, g - m, m)                         g - m rounded once, then m': at most 1 unit of scale_m
    v' = fma(v, b2, (w2 g) g)                      two roundings of w2 g^2, then v': at most 2 units of scale_v
    d  = fma(sqrt.approx(v'), 1 / bc2s, e)         sqrt.approx.f32 (PTX ISA: relative error <= 2^-23), the reciprocal
                                                   of bc2s rounded once, the fma rounded once
    p' = fma(-(ss m'), rcp.approx(d), p)           ss m' rounded once, rcp.approx.f32 (PTX ISA: <= 1 ulp, i.e. 2^-23)
To first order the relative errors of the update u add up: 1 (ss m') + 2 (sqrt.approx) + 1 (1 / bc2s) + 1 (d) + 2
(rcp.approx) = 7 units of 2^-24 |u|, plus half an ulp of p' from the final fma and the rounding of m' carried into u, which
is the second term of scale_p.  So p' must lie within BOUND_P = 8 units, m' and v' (no approximate instruction) within
BOUND_MV = 3 (2 plus the second-order terms).  The learning rates are float32 values, so that torch's double lr and the
float the kernels take are the same number.

The bound separates: with constants formed in float32 from float betas (1.0f - 0.999f is 1.29e-5 below torch's
(float)0.001, and powf(beta, step) stands in for the double power), exp_avg_sq after step 1 lies 110-146 units from the
replay and the parameters up to 56 units (measured on an H100); every test here except the eager-equals-capturable one
fails on such kernels.
"""
import numpy as np
import pytest
import torch

import _adam64 as A

pytestmark = pytest.mark.gpu

BOUND_P = 8.0
BOUND_MV = 3.0
LRS = [A.f32(x) for x in (1.6e-4, 2.5e-3, 1.25e-4, 5e-2, 2.5e-3, 5e-3, 1e-3, 1e-3)]
SIZE_CASES = {
    "small": [1, 2, 3, 5, 7, 1023, 4 * 1021 + 3],
    "eight": [1, 6, 255, 4096, 65537, 3, 1000, 513],       # GH_ADAM_MAX_GROUPS groups of mixed sizes
    "large": [3_000_001],                                    # > 1056 CTAs of 1024 elements: the grid-stride loop repeats
}


def _np(t: torch.Tensor) -> np.ndarray:
    return t.detach().float().cpu().numpy().reshape(-1)


def _make(sizes, capturable, rng, dev, lrs=None):
    from gaussianhaircut_b200.optim import FusedAdam
    lrs = lrs or LRS[:len(sizes)]
    ps = [torch.from_numpy(rng.standard_normal(n).astype(np.float32)).to(dev) for n in sizes]
    opt = FusedAdam([{"params": [p], "lr": lr} for p, lr in zip(ps, lrs)], eps=1e-15, capturable=capturable)
    return ps, lrs, opt


def _grads(rng, ps):
    """N(0,1) gradients scaled by 10^U(-3,3), one scale per group."""
    return [torch.from_numpy((rng.standard_normal(p.numel()) * 10.0 ** rng.uniform(-3, 3)).astype(np.float32)).to(p.device)
            for p in ps]


def _pre(opt, ps):
    out = []
    for p in ps:
        st = opt.state.get(p)
        m = _np(st["exp_avg"]) if st else np.zeros(p.numel(), np.float32)
        v = _np(st["exp_avg_sq"]) if st else np.zeros(p.numel(), np.float32)
        out.append((_np(p), m, v))
    return out


def _check(opt, ps, gs, pre, step, lrs, what):
    """p', m', v' of every group against the replay of step `step` from `pre`; -> the worst (p, m, v) units."""
    worst = np.zeros(3)
    for k, (p, g, (p0, m0, v0), lr) in enumerate(zip(ps, gs, pre, lrs)):
        r = A.adam_step(p0, _np(g), m0, v0, step, lr)
        st = opt.state[p]
        w = f"{what} group {k} (n={p.numel()}) step {step}"
        e = np.array([A.units(_np(p), r.p, r.scale_p, w + " p"), A.units(_np(st["exp_avg"]), r.m, r.scale_m, w + " m"),
                      A.units(_np(st["exp_avg_sq"]), r.v, r.scale_v, w + " v")])
        assert e[0] <= BOUND_P and max(e[1], e[2]) <= BOUND_MV, f"{w}: p / m / v off by {e} units"
        worst = np.maximum(worst, e)
    return worst


def _step_state(opt):
    return opt.step_state.cpu().tolist()


# ----------------------------------------------------------------------------------------------------- FusedAdam
@pytest.mark.parametrize("p_init", ["zero", "normal"])
@pytest.mark.parametrize("case", list(SIZE_CASES))
@pytest.mark.parametrize("capturable", [False, True], ids=["eager", "capturable"])
def test_fused_adam_per_element(cuda_device, capturable, case, p_init):
    """Every element of every group at steps 1, 2 and 10; p = 0 before each step (the update is not hidden under the
    rounding of p) or p ~ N(0,1)."""
    rng = np.random.default_rng([list(SIZE_CASES).index(case), int(p_init == "zero"), int(capturable)])
    ps, lrs, opt = _make(SIZE_CASES[case], capturable, rng, cuda_device)
    worst = np.zeros(3)
    for s in range(1, 11):
        if p_init == "zero":
            for p in ps:
                p.zero_()
        gs = _grads(rng, ps)
        pre = _pre(opt, ps) if s in (1, 2, 10) else None
        assert opt.step_count == s - 1
        opt.step(grads=gs)
        if pre is not None:
            worst = np.maximum(worst, _check(opt, ps, gs, pre, s, lrs, f"{case}/{p_init}/{'capturable' if capturable else 'eager'}"))
    print(f"FusedAdam {case}/{p_init}/{'capturable' if capturable else 'eager'}: worst p / m / v units {worst}")
    assert _step_state(opt) == [10, 0]


@pytest.mark.parametrize("late", [1000, 30000])
@pytest.mark.parametrize("capturable", [False, True], ids=["eager", "capturable"])
def test_fused_adam_late_state(cuda_device, capturable, late):
    """A state injected through load_state_dict at step `late`: the next steps use late + 1, late + 2, ...; a run of
    zero moments with a zero gradient leaves p bit-identical."""
    rng = np.random.default_rng(late)
    sizes = SIZE_CASES["small"]
    ps, lrs, opt = _make(sizes, capturable, rng, cuda_device)
    state = {}
    for i, n in enumerate(sizes):
        scale = (10.0 ** rng.uniform(-4, 2, n)).astype(np.float32)
        m = (rng.standard_normal(n) * scale * 0.3).astype(np.float32)
        v = (scale * scale * rng.uniform(0.5, 2.0, n)).astype(np.float32)
        m[:n // 4] = 0
        v[:n // 8] = 0
        state[i] = {"step": torch.tensor(float(late)), "exp_avg": torch.from_numpy(m), "exp_avg_sq": torch.from_numpy(v)}
    opt.load_state_dict({"state": state, "param_groups": [{"lr": lr, "params": [i]} for i, lr in enumerate(lrs)],
                         "steps_taken": late})
    for s in range(late + 1, late + 4):
        gs = _grads(rng, ps)
        if s == late + 1:
            for g in gs:
                g[:g.numel() // 4] = 0
        pre = _pre(opt, ps)
        opt.step(grads=gs)
        _check(opt, ps, gs, pre, s, lrs, f"late {late}")
        if s == late + 1:
            for p, (p0, _, _) in zip(ps, pre):
                n = p.numel() // 4
                assert np.array_equal(_np(p)[:n], p0[:n]), "m = 0 and g = 0 must leave p bit-identical"
    assert _step_state(opt) == [late + 3, 0]


@pytest.mark.parametrize("which", ["p", "g", "m", "v"])
@pytest.mark.parametrize("offset", [1, 2, 3])
def test_fused_adam_unaligned_views(cuda_device, which, offset):
    """One of p, g, m, v a view 1-3 floats into its storage (the others 16-byte aligned): the group takes the scalar
    path.  Same bound, and the floats in front of and behind each view are untouched."""
    from gaussianhaircut_b200.optim import FusedAdam
    rng = np.random.default_rng(offset * 7 + "pgmv".index(which))
    n, lr = 1031, LRS[1]
    start = {k: (offset if k == which else 4) for k in "pgmv"}
    bases = {k: torch.from_numpy(rng.standard_normal(n + 8).astype(np.float32)).to(cuda_device) for k in "pgmv"}
    bases["v"].abs_()
    view = {k: bases[k][start[k]:start[k] + n] for k in "pgmv"}
    assert all((view[k].data_ptr() % 16 != 0) == (k == which) for k in "pgmv")
    outside = {k: torch.cat([bases[k][:start[k]], bases[k][start[k] + n:]]) for k in "pgmv"}
    p = view["p"]
    opt = FusedAdam([{"params": [p], "lr": lr}], eps=1e-15)
    opt.state[p] = {"step": torch.zeros((), device=cuda_device), "exp_avg": view["m"], "exp_avg_sq": view["v"]}
    for s in (1, 2):
        view["g"].copy_(torch.from_numpy((rng.standard_normal(n) * 10.0 ** rng.uniform(-3, 3)).astype(np.float32)))
        pre = _pre(opt, [p])
        opt.step(grads=[view["g"]])
        assert opt.state[p]["exp_avg"].data_ptr() == view["m"].data_ptr()
        _check(opt, [p], [view["g"]], pre, s, [lr], f"{which}+{offset}")
    for k in "pgmv":
        assert torch.equal(torch.cat([bases[k][:start[k]], bases[k][start[k] + n:]]), outside[k]), \
            f"{k}: floats outside the view changed"


@pytest.mark.parametrize("capturable", [False, True], ids=["eager", "capturable"])
def test_fused_adam_edges(cuda_device, capturable):
    """Gradients of 0, subnormal w2 g^2, g^2 overflowing float32 with and without w2 g^2 overflowing, and +-inf: NaN and
    inf where the replay has them; a zero gradient on zero moments leaves p bit-identical; an lr = 0 group leaves p
    bit-identical and still updates its moments."""
    from gaussianhaircut_b200.optim import FusedAdam
    rng = np.random.default_rng(5)
    n = 2048
    ps = [torch.from_numpy(rng.standard_normal(n).astype(np.float32)).to(cuda_device) for _ in range(2)]
    lrs = [LRS[3], 0.0]
    opt = FusedAdam([{"params": [p], "lr": lr} for p, lr in zip(ps, lrs)], eps=1e-15, capturable=capturable)
    edges = [0.0, -0.0, 1e-21, -3e-22, 1e-24, 1e-19, 1e20, -1e20, 3e21, np.inf, -np.inf]
    for s in range(1, 4):
        g0 = rng.standard_normal(n).astype(np.float32)
        for k, x in enumerate(edges):
            g0[k * 32:(k + 1) * 32] = x
        gs = [torch.from_numpy(g0).to(cuda_device),
              torch.from_numpy(rng.standard_normal(n).astype(np.float32)).to(cuda_device)]
        pre = _pre(opt, ps)
        opt.step(grads=gs)
        assert int(opt.nan_flag.item()) == 0
        _check(opt, ps, gs, pre, s, lrs, "edges")
        assert not torch.isfinite(ps[0][9 * 32:11 * 32]).any(), "an infinite gradient must give a non-finite p"
        if s == 1:
            assert np.array_equal(_np(ps[0])[:64], pre[0][0][:64]), "m = 0 and g = 0 must leave p bit-identical"
        assert np.array_equal(_np(ps[1]), pre[1][0]), "an lr = 0 group must leave p bit-identical"
        assert not np.array_equal(_np(opt.state[ps[1]]["exp_avg_sq"]), pre[1][2]), "lr = 0 must still update the moments"


@pytest.mark.parametrize("how", ["nan", "skip_flag", "nan_flag_in"])
@pytest.mark.parametrize("capturable", [False, True], ids=["eager", "capturable"])
def test_fused_adam_skipped_step(cuda_device, capturable, how):
    """A single NaN in one group, a set `skip_flags` entry or a set `nan_flag_in` leaves every group's p, m, v and the
    step count bit-identical; the next clean step is step 3 for every element."""
    rng = np.random.default_rng(["nan", "skip_flag", "nan_flag_in"].index(how))
    ps, lrs, opt = _make(SIZE_CASES["eight"], capturable, rng, cuda_device)
    for _ in range(2):
        opt.step(grads=_grads(rng, ps))
    snap = [t.clone() for p in ps for t in (p, opt.state[p]["exp_avg"], opt.state[p]["exp_avg_sq"])]
    steps = opt.step_state.clone()
    gs = _grads(rng, ps)
    if how == "nan":
        gs[4][40000] = float("nan")
        opt.step(grads=gs)
        assert int(opt.nan_flag.item()) != 0
    elif how == "skip_flag":
        opt.step(grads=gs, skip_flags=(torch.ones(1, dtype=torch.int32, device=cuda_device),))
    else:
        flag = torch.ones(1, dtype=torch.int32, device=cuda_device)
        opt.step(grads=gs, nan_flag_in=flag)
        assert int(flag.item()) == 0, "nan_flag_in is consumed by the step"
    after = [t for p in ps for t in (p, opt.state[p]["exp_avg"], opt.state[p]["exp_avg_sq"])]
    assert all(torch.equal(a, b) for a, b in zip(after, snap)), "a skipped step changed a parameter or a moment"
    assert torch.equal(opt.step_state, steps)
    gs = _grads(rng, ps)
    pre = _pre(opt, ps)
    opt.step(grads=gs)
    _check(opt, ps, gs, pre, 3, lrs, f"after a skipped step ({how})")
    assert _step_state(opt) == [3, 0]


def test_fused_adam_eager_equals_capturable(cuda_device):
    """The two entry points apply the same arithmetic: bit-identical parameters and moments over 5 steps of 8 groups."""
    out = []
    for capturable in (False, True):
        rng = np.random.default_rng(21)
        ps, _, opt = _make(SIZE_CASES["eight"], capturable, rng, cuda_device)
        for _ in range(5):
            opt.step(grads=_grads(rng, ps))
        out.append([t.clone() for p in ps for t in (p, opt.state[p]["exp_avg"], opt.state[p]["exp_avg_sq"])])
        assert _step_state(opt) == [5, 0]
    assert all(torch.equal(a, b) for a, b in zip(*out))


@pytest.mark.parametrize("capturable", [False, True], ids=["eager", "capturable"])
def test_fused_adam_step_count(cuda_device, capturable):
    """After K steps of 8 groups of ~40 CTAs each the device step count is exactly [K, 0], and every element of the last
    step used step K.  This cannot prove the step-count election free of races (a race need not show in any run); it
    catches a count that is advanced more or less than once per step."""
    rng = np.random.default_rng(9)
    ps, lrs, opt = _make([40000 + 4 * k + (k % 4) for k in range(8)], capturable, rng, cuda_device)
    K = 40
    for s in range(1, K + 1):
        gs = _grads(rng, ps)
        pre = _pre(opt, ps) if s == K else None
        opt.step(grads=gs)
    _check(opt, ps, gs, pre, K, lrs, "step count")
    assert _step_state(opt) == [K, 0]


def test_fused_adam_matches_torch_gpu(cuda_device):
    """FusedAdam against the reference's construction, torch.optim.Adam(groups, lr=0.0, eps=1e-15) (the foreach path on
    CUDA), from identical state at every one of 10 steps: p', m', v' within the kernel bound of torch's, and torch's
    own step within 2 units of the replay."""
    from gaussianhaircut_b200.optim import FusedAdam
    rng = np.random.default_rng(17)
    sizes = [15000, 5000, 45000, 5000, 5000, 15000, 20000]
    lrs = LRS[:len(sizes)]
    p_ref = [torch.from_numpy(rng.standard_normal(n).astype(np.float32)).to(cuda_device).requires_grad_(True) for n in sizes]
    p_mine = [p.detach().clone() for p in p_ref]
    opt_ref = torch.optim.Adam([{"params": [p], "lr": lr} for p, lr in zip(p_ref, lrs)], lr=0.0, eps=1e-15)
    opt_mine = FusedAdam([{"params": [p], "lr": lr} for p, lr in zip(p_mine, lrs)], eps=1e-15)
    worst = np.zeros(3)
    for s in range(1, 11):
        gs = _grads(rng, p_ref)
        if s > 1:      # identical state: FusedAdam starts each step from torch's p, m, v
            for p, q in zip(p_ref, p_mine):
                q.copy_(p.detach())
                opt_mine.state[q]["exp_avg"].copy_(opt_ref.state[p]["exp_avg"])
                opt_mine.state[q]["exp_avg_sq"].copy_(opt_ref.state[p]["exp_avg_sq"])
        pre = _pre(opt_mine, p_mine)
        for p, g in zip(p_ref, gs):
            p.grad = g.clone()
        opt_ref.step()
        opt_mine.step(grads=gs)
        for k, (p, q, g, (p0, m0, v0), lr) in enumerate(zip(p_ref, p_mine, gs, pre, lrs)):
            r = A.adam_step(p0, _np(g), m0, v0, s, lr)
            w = f"group {k} step {s}"
            st, sq = opt_ref.state[p], opt_mine.state[q]
            t = [A.units(_np(p), r.p, r.scale_p, w), A.units(_np(st["exp_avg"]), r.m, r.scale_m, w),
                 A.units(_np(st["exp_avg_sq"]), r.v, r.scale_v, w)]
            assert max(t) <= 2.0, f"{w}: torch.optim.Adam is {t} units from the replay"
            k_rep = [A.units(_np(q), r.p, r.scale_p, w), A.units(_np(sq["exp_avg"]), r.m, r.scale_m, w),
                     A.units(_np(sq["exp_avg_sq"]), r.v, r.scale_v, w)]
            assert k_rep[0] <= BOUND_P and max(k_rep[1:]) <= BOUND_MV, f"{w}: FusedAdam is {k_rep} units from the replay"
            # the kernel against torch: within the kernel's bound plus torch's own 2 units
            e = np.array([A.units(_np(q), _np(p), r.scale_p, w + " p"),
                          A.units(_np(sq["exp_avg"]), _np(st["exp_avg"]), r.scale_m, w + " m"),
                          A.units(_np(sq["exp_avg_sq"]), _np(st["exp_avg_sq"]), r.scale_v, w + " v")])
            assert e[0] <= BOUND_P + 2.0 and max(e[1], e[2]) <= BOUND_MV + 2.0, f"{w}: FusedAdam is {e} units from torch"
            worst = np.maximum(worst, e)
    print(f"FusedAdam against torch.optim.Adam: worst p / m / v units {worst}")
    assert opt_mine.step_count == 10


# ----------------------------------------------------------------------------------------------------- CameraAdam
CAM_LRS = [A.f32(x) for x in (1e-3, 3e-4, 2e-3)]      # rotation, translation, fov


def _rig(n, intrinsics, rng, dev):
    from gaussianhaircut_b200.cameras import CameraRig
    base = torch.zeros(n, 18)
    res = torch.from_numpy((rng.standard_normal((n, 8)) * 0.01).astype(np.float32))
    return CameraRig(base.to(dev), res.to(dev), [f"c{i}" for i in range(n)], [(64, 48)] * n, intrinsics=intrinsics)


@pytest.mark.parametrize("intrinsics", [True, False], ids=["intrinsics", "no_intrinsics"])
def test_camera_adam_per_element(cuda_device, intrinsics):
    """n = 300 cameras (more rows than threads), rows touched on their own schedules so that each has its own step
    count: every updated element against the replay at its row's step with its column's learning rate; untouched rows
    (and columns 6-7 without intrinsics) bit-identical in residuals, moments and steps; after every call -- including a
    skipped one and a NaN one -- the gradients, `touched` and `nan_flag` are clear."""
    from gaussianhaircut_b200.cameras import CameraAdam
    rng = np.random.default_rng(int(intrinsics))
    n = 300
    rig = _rig(n, intrinsics, rng, cuda_device)
    opt = CameraAdam(rig, *CAM_LRS)
    cols = 8 if intrinsics else 6
    col_lr = np.array([CAM_LRS[0]] * 3 + [CAM_LRS[1]] * 3 + [CAM_LRS[2]] * 2)
    period, phase = 1 + np.arange(n) % 7, np.arange(n) // 7
    expected = np.zeros(n, np.int64)
    worst = np.zeros(3)
    for it in range(12):
        touched = ((it + phase) % period) == 0
        g = (rng.standard_normal((n, 8)) * 10.0 ** rng.uniform(-3, 3, (n, 1))).astype(np.float32)
        g[~touched] = 0
        rig.grad.copy_(torch.from_numpy(g))
        rig.touched.copy_(torch.from_numpy(touched.astype(np.int32)))
        mode = "skip" if it == 7 else ("nan" if it == 9 else "step")
        if mode == "nan":
            rig.nan_flag.fill_(1)
        r0, m0, v0 = (t.detach().cpu().numpy().copy() for t in (rig.residuals, opt.exp_avg, opt.exp_avg_sq))
        s0 = opt.steps.cpu().numpy().copy()
        opt.step(skip_flag=torch.ones(1, dtype=torch.int32, device=cuda_device) if mode == "skip" else None)
        r1, m1, v1 = (t.detach().cpu().numpy() for t in (rig.residuals, opt.exp_avg, opt.exp_avg_sq))
        s1 = opt.steps.cpu().numpy()
        assert not rig.grad.any() and not rig.touched.any() and int(rig.nan_flag.item()) == 0, f"iteration {it}: not cleared"
        moved = touched if mode == "step" else np.zeros(n, bool)
        expected += moved
        assert np.array_equal(s1, expected), f"iteration {it}: step counts"
        keep = ~moved
        for a, b in ((r1, r0), (m1, m0), (v1, v0)):
            assert np.array_equal(a[keep], b[keep]), f"iteration {it}: a row that did not step changed"
            assert np.array_equal(a[:, cols:], b[:, cols:]), f"iteration {it}: a column that is not trained changed"
        for i in np.flatnonzero(moved):
            for k in range(cols):
                rr = A.adam_step(r0[i, k:k + 1], g[i, k:k + 1], m0[i, k:k + 1], v0[i, k:k + 1], int(s1[i]), float(col_lr[k]))
                w = f"iteration {it} row {i} (step {s1[i]}) column {k}"
                e = (A.units(r1[i, k:k + 1], rr.p, rr.scale_p, w), A.units(m1[i, k:k + 1], rr.m, rr.scale_m, w),
                     A.units(v1[i, k:k + 1], rr.v, rr.scale_v, w))
                assert e[0] <= BOUND_P and max(e[1:]) <= BOUND_MV, f"{w}: p / m / v off by {e} units"
                worst = np.maximum(worst, e)
    print(f"CameraAdam intrinsics={intrinsics}: worst p / m / v units {worst}")
    assert len(set(expected.tolist())) >= 5, "the schedules should leave the rows at different step counts"
